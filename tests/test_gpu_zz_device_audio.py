"""Sound from device memory (htv_set_audio_device_source, Encoder.set_device_audio): k_pcm_ingest writes a strided
int16 or float32 stereo view into the sound ring, where a host source's copy would have put the same int16 pairs.
Everything after the ring is unchanged, so an encoder fed that way must render, byte for byte, what one fed the same
int16 values through read_audio renders: at every sound stage (FM + NICAM in the compiled-in form, AM + NICAM behind
the SECAM chain, FM with 75 us pre-emphasis), with blocks of 1, 7 and 8192 pairs and one block larger than a quarter
of the ring, for every layout the view can describe, for float32 under the header's rounding rule, for a source that
ends, for sound and pictures written on the render stream without a synchronise, through htv_render_host, htv_next_line
with prefetch and another sample type; and the refusals."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F = dict(vfilter=True)
# (id, mode, sample rate, overrides)
MODES = [
    ("pal-i-fm-nicam", "i", 16000000, F),           # the k_line form with the sound stages compiled in
    ("secam-l-am-nicam", "l", 16000000, F),         # AM + NICAM behind k_sec_raster and the chrominance chain
    ("ntsc-m-fm-75us", "m", 13500000, F),           # FM with 75 us pre-emphasis and its limiter
]
PIECES = [1, 2, 311, 1000, 625, 3, 2058]            # uneven calls, as in test_gpu_zz_line_widths.py
RING_QUARTER = (1 << 20) // 4                        # pairs: the largest piece of a block one pull takes


class _View:
    """A strided view of memory described by __cuda_array_interface__: torch has no view with a negative stride, and a
    host pointer described the same way is what the refusal test needs"""

    def __init__(self, keep, ptr, shape, strides, typestr="<i2"):
        self.keep = keep
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False),
                                         "strides": tuple(strides), "version": 3}


def _pcm(n, seed):
    return np.random.default_rng(seed).integers(-32768, 32768, size=(n, 2), dtype=np.int16)


def _pairs_for(lines, W, rate):
    """More pairs than `lines` lines take (the audio clock leads the lines by less than three)"""
    return (lines + 3) * W * 32000 // rate + 2


def _layout(audio, layout):
    """int16 pairs [n, 2] in device memory, laid out as `layout`"""
    import torch
    n = audio.shape[0]
    if layout == "interleaved":
        return torch.from_numpy(audio).cuda()
    if layout == "planar":
        return torch.from_numpy(np.ascontiguousarray(audio.T)).cuda()
    if layout == "r-before-l":
        t = torch.from_numpy(np.ascontiguousarray(audio[:, ::-1])).cuda()
        return _View(t, t.data_ptr() + 2, (n, 2), (4, -2))
    if layout == "strided":
        big = np.full((2 * n, 2), 0x2AAA, dtype=np.int16)
        big[::2] = audio
        return torch.from_numpy(big).cuda()[::2]
    raise ValueError(layout)


def _encoder(H, mode, rate, kw, sample_type=None):
    enc = H.Encoder(H.mode_config(mode, **kw) if isinstance(mode, str) else mode, rate)
    if sample_type:
        enc.set_sample_type(sample_type)
    return enc


def _render_host(H, mode, rate, kw, pieces, install, sample_type=None):
    enc = _encoder(H, mode, rate, kw, sample_type)
    install(enc)
    got = np.concatenate([enc.render_host(n) for n in pieces])
    enc.close()
    return got


def _render_device(H, mode, rate, kw, pieces, install):
    """htv_render into device memory on torch's current stream"""
    import torch
    enc = _encoder(H, mode, rate, kw)
    install(enc)
    per = 2 if enc.complex else 1
    buf = torch.empty(sum(pieces) * enc.width * per, dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    at = 0
    for n in pieces:
        enc.render(n, buf.data_ptr() + at * enc.width * per * 2, st)
        at += n
    torch.cuda.synchronize()
    enc.close()
    return buf


def _same(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    d = got != want
    assert not d.any(), f"{np.count_nonzero(d)} of {d.size} values differ from the host-fed encoder"


def _host_audio(audio, block=0):
    return lambda enc: enc.set_source(None, audio, audio_block=block)


def _device_audio(view, block=0):
    return lambda enc: enc.set_device_audio(view, audio_block=block)


@pytest.mark.parametrize("block", [1, 7, 8192])
@pytest.mark.parametrize("mode,rate,kw", [m[1:] for m in MODES], ids=[m[0] for m in MODES])
def test_every_sound_stage_device_fed_equals_host_fed(built, mode, rate, kw, block):
    H = built
    audio = _pcm(_pairs_for(sum(PIECES), 1024, 13500000) // 2, 1)        # half the stream: the source is reused
    got = _render_host(H, mode, rate, kw, PIECES, _device_audio(_layout(audio, "interleaved"), block))
    _same(got, _render_host(H, mode, rate, kw, PIECES, _host_audio(audio, block)))


def test_block_larger_than_a_quarter_of_the_ring(built):
    """Two blocks of 270 000 pairs each (a quarter of the ring is 262 144): each is taken in pieces over several calls
    and launch sequences, and the last call runs past the first block into the second"""
    import torch
    H = built
    mode, rate, kw = "i", 16000000, F
    blk = RING_QUARTER + 7856
    audio = _pcm(2 * blk, 2)
    pieces = PIECES + [150000]                                            # 9.6 s in all: 307 200 pairs
    assert _pairs_for(sum(pieces), 1024, rate) > blk
    got = _render_device(H, mode, rate, kw, pieces, _device_audio(_layout(audio, "interleaved"), blk))
    want = _render_device(H, mode, rate, kw, pieces, _host_audio(audio, blk))
    assert torch.equal(got, want), f"{int((got != want).sum())} of {got.numel()} values differ from the host-fed encoder"


@pytest.mark.parametrize("layout", ["interleaved", "planar", "r-before-l", "strided"])
def test_layouts(built, layout):
    H = built
    mode, rate, kw = "i", 16000000, F
    audio = _pcm(_pairs_for(sum(PIECES), 1024, rate), 3)
    got = _render_host(H, mode, rate, kw, PIECES, _device_audio(_layout(audio, layout), 1000))
    _same(got, _render_host(H, mode, rate, kw, PIECES, _host_audio(audio, 1000)))


def _float_pcm(n, seed):
    """float32 pairs: the range beyond [-1, 1], infinities, NaN, and exact ties (x * 32767 in float32 lands on k + 1/2)
    on both channels at once, so that the mono sum carries a tie's rounding to the sound carrier unhalved"""
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1.25, 1.25, size=(n, 2)).astype(np.float32)
    t = rng.integers(-32768, 32767, size=4 * n).astype(np.float64) + 0.5
    ties = (t / 32767.0).astype(np.float32)
    ties = ties[ties * np.float32(32767) == t.astype(np.float32)]
    ties = np.concatenate([ties, np.float32([0.5, -0.5, 1.5 / 32767, -2.5 / 32767])])
    ties = ties[ties * np.float32(32767) == np.floor(ties * np.float32(32767)) + np.float32(0.5)]
    assert ties.size > n // 4, ties.size
    at = rng.choice(n, size=min(n // 2, ties.size), replace=False)
    x[at, 0] = x[at, 1] = ties[:at.size]
    special = np.float32([np.nan, np.inf, -np.inf, 1.0, -1.0, 0.0, -0.0, 3e38, -3e38, 1e-30])
    x[:special.size, 0] = special
    x[:special.size, 1] = special[::-1]
    return x


def _float_rule(x, rounding=np.rint):
    """the header's HTV_PCM_FLOAT32 rule in numpy: the product in float32, rounded, clamped, NaN = 0"""
    with np.errstate(over="ignore", invalid="ignore"):
        p = x.astype(np.float32) * np.float32(32767)
        return np.where(np.isnan(p), 0, np.clip(rounding(p), -32768, 32767)).astype(np.int16)


def _half_away(p):
    return np.sign(p) * np.floor(np.abs(p) + np.float32(0.5))


def test_float32_follows_the_rounding_rule(built):
    import torch
    H = built
    mode, rate, kw = "i", 16000000, F
    x = _float_pcm(_pairs_for(sum(PIECES), 1024, rate), 4)
    got = _render_host(H, mode, rate, kw, PIECES, _device_audio(torch.from_numpy(x).cuda(), 999))
    _same(got, _render_host(H, mode, rate, kw, PIECES, _host_audio(_float_rule(x), 999)))


def test_float32_ties_reach_the_output(built):
    """Without pre-emphasis the FM carrier's step is looked up from each mono sample as it is, so a tie rounded away
    from zero instead of to even changes the stream: the comparison above cannot pass by the ties being lost"""
    import torch
    H = built
    rate = 16000000
    conf = H.mode_config("i", vfilter=True, nonicam=True)
    conf.fm_mono_preemph = 0
    x = _float_pcm(_pairs_for(sum(PIECES), 1024, rate), 5)
    even, away = _float_rule(x), _float_rule(x, _half_away)
    assert (even != away).any()
    got = _render_host(H, conf, rate, {}, PIECES, _device_audio(torch.from_numpy(x).cuda(), 4096))
    _same(got, _render_host(H, conf, rate, {}, PIECES, _host_audio(even, 4096)))
    assert (got != _render_host(H, conf, rate, {}, PIECES, _host_audio(away, 4096))).any()


@pytest.mark.parametrize("end", ["error", "null", "empty"])
def test_source_that_ends_equals_a_host_source_that_ends(built, end):
    """Blocks of 1000 pairs until 5 500 pairs, then an end of each kind: silence follows and the source is not pulled
    again; a host source that hands out the same blocks and then nothing renders the same"""
    import torch
    H = built
    mode, rate, kw = "i", 16000000, F
    audio = _pcm(5500, 6)
    dev = torch.from_numpy(audio).cuda()
    pulls = {"after_end": 0}

    def install_device(enc):
        state = {"at": 0}

        def read(ctx, blk):
            b = blk.contents
            at = state["at"]
            if at >= audio.shape[0]:
                pulls["after_end"] += at > audio.shape[0]
                state["at"] += 1
                if end == "error":
                    return H.HTV_ERROR
                b.data, b.npairs = (None, 1000) if end == "null" else (dev.data_ptr(), 0)
                b.format, b.stride_pair, b.stride_ch = H.HTV_PCM_INT16, 4, 2
                return H.HTV_OK
            b.data, b.npairs = dev.data_ptr() + at * 4, min(1000, audio.shape[0] - at)
            b.format, b.stride_pair, b.stride_ch = H.HTV_PCM_INT16, 4, 2
            state["at"] += b.npairs
            return H.HTV_OK
        cb = H._READ_AUDIO_DEVICE(read)
        enc._keep.append(cb)
        assert enc._L.htv_set_audio_device_source(enc._h, cb, None) == H.HTV_OK

    def install_host(enc):
        state = {"at": 0}

        def read(ctx, samples, n):
            at = state["at"]
            m = min(1000, max(audio.shape[0] - at, 0))
            samples[0] = audio[at:].ctypes.data if m else None
            n[0] = m
            state["at"] += m
            return H.HTV_OK
        cb = H._READ_AUDIO(read)
        enc._keep.append(cb)
        H.lib().htv_av(enc._h).contents.read_audio = cb

    got = _render_host(H, mode, rate, kw, PIECES, install_device)
    assert pulls["after_end"] == 0
    _same(got, _render_host(H, mode, rate, kw, PIECES, install_host))


def test_sound_and_pictures_written_on_the_render_stream_need_no_synchronise(built):
    """Before each call, on a side stream: a long sleep, then the pictures and the sound blocks that call pulls are
    written over a filler; htv_render on the same stream, never synchronised. An ingest that did not wait for the
    stream would read filler"""
    import torch
    H = built
    mode, rate, kw = "i", 16000000, F
    enc = _encoder(H, mode, rate, kw)
    L, W, per = enc.lines, enc.width, 2 if enc.complex else 1
    rng = np.random.default_rng(7)
    frames = rng.integers(0, 1 << 24, size=(19, enc.active_lines, enc.active_width), dtype=np.uint32)
    rgb = np.stack([(frames >> 16) & 255, (frames >> 8) & 255, frames & 255], axis=-1).astype(np.uint8)
    pieces = [L // 3, 2 * L + 17, 5 * L - 40, 1, 3 * L + 101, L - 78, 7 * L]
    blk = 512
    audio = _pcm(-(-_pairs_for(sum(pieces), W, rate) // blk) * blk + blk, 8)
    src_pics, src_pcm = torch.from_numpy(rgb).cuda(), torch.from_numpy(audio).cuda()
    pics, pcm = torch.full_like(src_pics, 0x55), torch.full_like(src_pcm, 0x1234)
    torch.cuda.synchronize()
    enc.set_device_source(pics)
    enc.set_device_audio(pcm, audio_block=blk)
    buf = torch.zeros(sum(pieces) * W * per, dtype=torch.int16, device="cuda")
    s = torch.cuda.Stream()
    at, written = 0, 0
    with torch.cuda.stream(s):
        for n in pieces:
            # frame f is pulled by the call that renders its first line; sound in whole blocks up to what the call needs
            new = sorted({f % 19 for f in range(-(-at // L), -(-(at + n) // L))})
            upto = min(-(-_pairs_for(at + n, W, rate) // blk) * blk, audio.shape[0])
            torch.cuda._sleep(20_000_000)
            for i in new:
                pics[i].copy_(src_pics[i])
            pcm[written:upto].copy_(src_pcm[written:upto])
            written = max(written, upto)
            enc.render(n, buf.data_ptr() + at * W * per * 2, s.cuda_stream)
            at += n
    torch.cuda.synchronize()
    got = buf.cpu().numpy()
    enc.close()

    def install_host(e):
        e.set_source(frames, audio, audio_block=blk)
    _same(got, _render_host(H, mode, rate, kw, pieces, install_host))


def test_render_host_with_another_sample_type(built):
    H = built
    mode, rate, kw = "i", 16000000, F
    audio = _pcm(_pairs_for(sum(PIECES), 1024, rate), 9)
    got = _render_host(H, mode, rate, kw, PIECES, _device_audio(_layout(audio, "planar"), 8192), sample_type="int8")
    assert got.dtype == np.int8
    _same(got, _render_host(H, mode, rate, kw, PIECES, _host_audio(audio, 8192), sample_type="int8"))


def test_next_line_with_prefetch(built):
    H = built
    mode, rate, kw = "l", 16000000, F
    audio = _pcm(20000, 10)

    def lines(install):
        enc = _encoder(H, mode, rate, kw)
        install(enc)
        enc.set_prefetch(True)
        out = np.concatenate([enc.next_line()[0] for _ in range(3 * enc.lines + 5)])
        enc.close()
        return out
    _same(lines(_device_audio(_layout(audio, "interleaved"), 777)), lines(_host_audio(audio, 777)))


def test_baseband_without_sound_never_pulls_the_source(built):
    import torch
    H = built
    mode, rate, kw = "pal", 16000000, dict(vfilter=True, noaudio=True)
    pulls = {"n": 0}
    dev = torch.zeros((64, 2), dtype=torch.int16, device="cuda")

    def install(enc):
        def read(ctx, blk):
            pulls["n"] += 1
            b = blk.contents
            b.data, b.npairs, b.format, b.stride_pair, b.stride_ch = dev.data_ptr(), 64, H.HTV_PCM_INT16, 4, 2
            return H.HTV_OK
        cb = H._READ_AUDIO_DEVICE(read)
        enc._keep.append(cb)
        assert enc._L.htv_set_audio_device_source(enc._h, cb, None) == H.HTV_OK
    got = _render_host(H, mode, rate, kw, PIECES, install)
    assert pulls["n"] == 0
    _same(got, _render_host(H, mode, rate, kw, PIECES, lambda enc: None))


def test_a_host_source_installed_afterwards_replaces_the_device_source(built):
    H = built
    mode, rate, kw = "i", 16000000, F
    audio = _pcm(9000, 11)
    enc_install = [_device_audio(_layout(_pcm(9000, 12), "interleaved")), _host_audio(audio)]
    got = _render_host(H, mode, rate, kw, PIECES, lambda enc: [f(enc) for f in enc_install])
    _same(got, _render_host(H, mode, rate, kw, PIECES, _host_audio(audio)))


def _refused(H, capfd, install, message):
    enc = _encoder(H, "i", 16000000, F)
    install(enc)
    with pytest.raises(RuntimeError):
        enc.render_host(10)
    enc.close()
    assert message in capfd.readouterr().err


def test_host_memory_is_refused(built, capfd):
    H = built
    host = np.zeros((4096, 2), dtype=np.int16)
    _refused(H, capfd, _device_audio(_View(host, host.ctypes.data, host.shape, host.strides)),
             "must be device or managed memory")


def test_another_devices_memory_is_refused(built, capfd):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    H = built
    other = torch.zeros((4096, 2), dtype=torch.int16, device="cuda:1")
    _refused(H, capfd, _device_audio(other), "must be device or managed memory")


@pytest.mark.parametrize("fmt,offset,message", [(7, 0, "unknown device PCM format 7"),
                                                (0, 1, "multiples of its 2-byte samples"),
                                                (1, 2, "multiples of its 4-byte samples")],
                         ids=["unknown-format", "misaligned-int16", "misaligned-float32"])
def test_bad_block_is_refused(built, capfd, fmt, offset, message):
    import torch
    H = built
    dev = torch.zeros((4096, 4), dtype=torch.int16, device="cuda")

    def install(enc):
        def read(ctx, blk):
            b = blk.contents
            b.data, b.npairs, b.format = dev.data_ptr() + offset, 4000, fmt
            b.stride_pair, b.stride_ch = 8, 4
            return H.HTV_OK
        cb = H._READ_AUDIO_DEVICE(read)
        enc._keep.append(cb)
        assert enc._L.htv_set_audio_device_source(enc._h, cb, None) == H.HTV_OK
    _refused(H, capfd, install, message)


def test_installing_after_the_first_line_is_refused(built, capfd):
    import torch
    H = built
    enc = _encoder(H, "i", 16000000, F)
    enc.set_source(None, _pcm(4096, 13))
    enc.render_host(10)
    with pytest.raises(RuntimeError):
        enc.set_device_audio(torch.zeros((64, 2), dtype=torch.int16, device="cuda"))
    assert enc._L.htv_set_audio_device_source(enc._h, H._READ_AUDIO_DEVICE(), None) == H.HTV_ERROR
    enc.close()
    assert "the sound source must be set before the first line" in capfd.readouterr().err
