"""Pictures from device memory (htv_set_video_device_source, Encoder.set_device_source): k_ingest converts a strided
view of three uint8 channels into a picture slot, and everything after the slot is what a host picture meets. So a
device-fed encoder must render, byte for byte, what one fed the same pixels as uint32 words through set_source renders,
on the same call pieces: at every slot reader (k_compose, the PS forms' k_picture, k_sec_raster, k_raster behind FM
video and --pixelrate, S-Video), for every layout the view can describe, with all 16 slots reused, a static picture
ingested once, a source that ends, pictures written on the render stream without a synchronise, and the refusals."""
import numpy as np
import pytest

import orc

pytestmark = pytest.mark.gpu

F = dict(vfilter=True)
# (id, mode, sample rate, pixel rate, overrides, a part of the line_kernel string the case is for)
READERS = [
    ("pal-i-bench", "i", 16000000, 0, F, "SND=37,WC=1024"),                        # composite store, sound stages
    ("pal-i", "i", 16000000, 0, dict(vfilter=True, noaudio=True), "SND=-1,WC=0"),  # composite store
    ("ntsc-m-16M", "m", 16000000, 0, F, "k_line<VF=1,HQ=1,FULL=0"),                # converted picture store (PS forms)
    ("secam-l", "l", 16000000, 0, F, "k_sec_raster"),
    ("pal-fm", "pal-fm", 16000000, 0, {}, "k_fmv_mod"),                            # k_raster behind FM video
    ("pal-i-pixelrate", "i", 16000000, 13500000, F, "k_resample"),                 # k_raster in the raster context
    ("pal-s-video", "pal", 16000000, 0, dict(s_video=True), ",SV>"),
]


class _View:
    """A strided uint8 view of a torch tensor's memory, described by __cuda_array_interface__ (torch has no view with a
    negative stride, and a host pointer described the same way is what the refusal test needs)."""

    def __init__(self, keep, ptr, shape, strides):
        self.keep = keep
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "|u1", "data": (int(ptr), False),
                                         "strides": tuple(strides), "version": 3}


def _pictures(enc, n, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 1 << 24, size=(n, enc.active_lines, enc.active_width), dtype=np.uint32)


def _rgb(frames):
    return np.stack([(frames >> 16) & 255, (frames >> 8) & 255, frames & 255], axis=-1).astype(np.uint8)


def _layout(frames, layout):
    """The pictures of `frames` (uint32 0x00RRGGBB) in device memory, laid out as `layout`"""
    import torch
    rgb = _rgb(frames)
    n, h, w, _ = rgb.shape
    if layout == "hwc-rgb":
        return torch.from_numpy(rgb).cuda()
    if layout == "hwc-rgba":
        alpha = np.full((n, h, w, 1), 255, dtype=np.uint8)
        return torch.from_numpy(np.concatenate([rgb, alpha], axis=-1)).cuda()
    if layout == "bgra":
        # B, G, R, A in memory: R of a pixel is its byte 2, G byte 1, B byte 0 - stride_c = -1
        t = torch.from_numpy(np.concatenate([rgb[..., ::-1], np.zeros((n, h, w, 1), np.uint8)], axis=-1).copy()).cuda()
        return _View(t, t.data_ptr() + 2, (n, h, w, 3), (h * w * 4, w * 4, 4, -1))
    if layout == "chw":
        return torch.from_numpy(np.ascontiguousarray(rgb.transpose(0, 3, 1, 2))).cuda()
    if layout == "crop":
        big = torch.full((n, h + 9, w + 53, 3), 77, dtype=torch.uint8)
        big[:, 5:5 + h, 11:11 + w, :] = torch.from_numpy(rgb)
        return big.cuda()[:, 5:5 + h, 11:11 + w, :]
    raise ValueError(layout)


def _encoder(H, mode, rate, prate, kw):
    return H.Encoder(H.mode_config(mode, **kw), rate, prate)


def _host_fed(H, mode, rate, prate, kw, frames, pieces, audio=None, static_video=False):
    enc = _encoder(H, mode, rate, prate, kw)
    enc.set_source(frames, audio, static_video=static_video)
    got = np.concatenate([enc.render_host(n) for n in pieces])
    launches = enc.kernel_launches
    enc.close()
    return got, launches


def _same(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    d = got != want
    assert not d.any(), f"{np.count_nonzero(d)} of {d.size} values differ from the host-fed encoder"


def _oracle(conf, rate, frames, nlines):
    o = orc.Oracle(conf, rate)
    o.set_source(frames, None)
    want = o.render(nlines)
    o.close()
    return want


@pytest.mark.parametrize("mode,rate,prate,kw,form", [r[1:] for r in READERS], ids=[r[0] for r in READERS])
def test_every_slot_reader_device_fed_equals_host_fed(built, mode, rate, prate, kw, form):
    """Five pictures used cyclically, with programme audio where the mode has sound, in calls that cut frames"""
    H = built
    enc = _encoder(H, mode, rate, prate, kw)
    frames = _pictures(enc, 5, 1)
    audio = H.test_tone()
    enc.set_device_source(_layout(frames, "hwc-rgb"))
    enc.set_source(None, audio)
    L = enc.lines
    pieces = [L // 3, 2 * L + 17, 3 * L - 40, 1, L + 101]
    got = np.concatenate([enc.render_host(n) for n in pieces])
    assert form in enc.line_kernel, enc.line_kernel
    enc.close()
    _same(got, _host_fed(H, mode, rate, prate, kw, frames, pieces, audio)[0])


@pytest.mark.parametrize("layout", ["hwc-rgb", "hwc-rgba", "bgra", "chw", "crop"])
@pytest.mark.parametrize("mode,rate,kw", [("i", 16000000, dict(vfilter=True, noaudio=True)), ("m", 16000000, F)],
                         ids=["composite-store", "picture-store"])
def test_layouts(built, layout, mode, rate, kw):
    H = built
    enc = _encoder(H, mode, rate, 0, kw)
    frames = _pictures(enc, 4, 2)
    enc.set_device_source(_layout(frames, layout))
    L = enc.lines
    pieces = [2 * L + 5, 3 * L - 5]
    got = np.concatenate([enc.render_host(n) for n in pieces])
    enc.close()
    _same(got, _host_fed(H, mode, rate, 0, kw, frames, pieces)[0])


@pytest.mark.parametrize("mode,rate,kw", [("i", 16000000, dict(vfilter=True, noaudio=True)),
                                          ("m", 16000000, dict(vfilter=True, noaudio=True))], ids=["pal-i", "ntsc-m-16M"])
def test_live_source_reuses_every_slot_bit_exact_against_the_oracle(built, mode, rate, kw):
    """19 pictures, one per frame, in the uneven calls of the picture-store test: all 16 slots are refilled while the
    calls before are in flight, runs of new pictures wrap around the slots, and pictures change inside a call"""
    H = built
    conf = H.mode_config(mode, **kw)
    enc = H.Encoder(conf, rate)
    frames = _pictures(enc, 19, 3)
    enc.set_device_source(_layout(frames, "hwc-rgb"))
    L = enc.lines
    pieces = [L // 3, 2 * L + 17, 5 * L - 40, 1, 3 * L + 101, L - 78, 7 * L]
    got = np.concatenate([enc.render_host(n) for n in pieces])
    enc.close()
    d = got.astype(np.int32) - _oracle(conf, rate, frames, sum(pieces)).astype(np.int32)
    assert not d.any(), f"{np.count_nonzero(d)} of {d.size} values differ from the oracle"


def test_static_source_is_ingested_once(built):
    """A constant serial: one k_ingest launch over the whole stream, and otherwise the launches of the host-fed run"""
    H = built
    mode, rate, kw = "i", 16000000, F
    enc = _encoder(H, mode, rate, 0, kw)
    frames = _pictures(enc, 1, 4)
    enc.set_device_source(_layout(frames, "hwc-rgb"), static_video=True)
    L = enc.lines
    pieces = [L + 3, 4 * L, 9 * L - 3, 2]
    got = np.concatenate([enc.render_host(n) for n in pieces])
    launches = enc.kernel_launches
    enc.close()
    want, host_launches = _host_fed(H, mode, rate, 0, kw, frames, pieces, static_video=True)
    _same(got, want)
    assert launches == host_launches + 1, (launches, host_launches)


def test_source_that_ends_falls_back_to_black(built):
    """Three pictures, then a read that fails, as a host source that ends"""
    import torch
    H = built
    conf = H.mode_config("i", vfilter=True, noaudio=True)
    enc = H.Encoder(conf, 16000000)
    frames = _pictures(enc, 3, 5)
    pics = torch.from_numpy(_rgb(frames)).cuda()
    state = {"f": 0}

    def read(ctx, fr):
        i = state["f"]
        if i >= 3:
            return H.HTV_ERROR
        f = fr.contents
        f.width, f.height, f.data = enc.active_width, enc.active_lines, pics[i].data_ptr()
        f.stride_x, f.stride_y, f.stride_c, f.serial = 3, 3 * enc.active_width, 1, i + 1
        state["f"] += 1
        return H.HTV_OK
    cb = H._READ_VIDEO_DEVICE(read)
    assert enc._L.htv_set_video_device_source(enc._h, cb, None) == H.HTV_OK
    L = enc.lines
    pieces = [L + 200, 2 * L, 3 * L - 200]
    got = np.concatenate([enc.render_host(n) for n in pieces])
    enc.close()
    padded = np.concatenate([frames, np.zeros((3,) + frames.shape[1:], dtype=np.uint32)])
    d = got.astype(np.int32) - _oracle(conf, 16000000, padded, sum(pieces)).astype(np.int32)
    assert not d.any(), f"{np.count_nonzero(d)} of {d.size} values differ from the oracle"


def test_pictures_written_on_the_render_stream_need_no_synchronise(built):
    """Before each call, on a side stream: a long sleep, then the pictures that call pulls are written over a filler;
    htv_render on the same stream, never synchronised. An ingest that did not wait for the stream would read filler."""
    import torch
    H = built
    conf = H.mode_config("i", vfilter=True, noaudio=True)
    enc = H.Encoder(conf, 16000000)
    frames = _pictures(enc, 19, 6)
    src = torch.from_numpy(_rgb(frames)).cuda()
    pics = torch.full_like(src, 0x55)
    torch.cuda.synchronize()
    enc.set_device_source(pics)
    L, W, per = enc.lines, enc.width, 2 if enc.complex else 1
    pieces = [L // 3, 2 * L + 17, 5 * L - 40, 1, 3 * L + 101, L - 78, 7 * L]
    buf = torch.zeros(sum(pieces) * W * per, dtype=torch.int16, device="cuda")
    s = torch.cuda.Stream()
    at = 0
    with torch.cuda.stream(s):
        for n in pieces:
            # frame f is pulled by the call that renders its first line
            new = sorted({f % 19 for f in range(-(-at // L), -(-(at + n) // L))})
            torch.cuda._sleep(20_000_000)
            for i in new:
                pics[i].copy_(src[i])
            enc.render(n, buf.data_ptr() + at * W * per * 2, s.cuda_stream)
            at += n
    torch.cuda.synchronize()
    got = buf.cpu().numpy()
    enc.close()
    d = got.astype(np.int32) - _oracle(conf, 16000000, frames, sum(pieces)).astype(np.int32)
    assert not d.any(), f"{np.count_nonzero(d)} of {d.size} values differ from the oracle"


def test_a_host_source_installed_afterwards_replaces_the_device_source(built):
    H = built
    kw = dict(vfilter=True, noaudio=True)
    enc = _encoder(H, "i", 16000000, 0, kw)
    frames = _pictures(enc, 3, 7)
    enc.set_device_source(_layout(_pictures(enc, 3, 8), "hwc-rgb"))
    enc.set_source(frames, None)
    pieces = [2 * enc.lines + 9]
    got = enc.render_host(pieces[0])
    enc.close()
    _same(got, _host_fed(H, "i", 16000000, 0, kw, frames, pieces)[0])


def test_host_memory_is_refused(built):
    H = built
    enc = _encoder(H, "i", 16000000, 0, dict(vfilter=True, noaudio=True))
    host = np.zeros((1, enc.active_lines, enc.active_width, 3), dtype=np.uint8)
    enc.set_device_source(_View(host, host.ctypes.data, host.shape, host.strides))
    with pytest.raises(RuntimeError):
        enc.render_host(10)
    enc.close()


def test_wrong_size_is_refused(built):
    import torch
    H = built
    enc = _encoder(H, "i", 16000000, 0, dict(vfilter=True, noaudio=True))
    enc.set_device_source(torch.zeros((1, enc.active_lines - 1, enc.active_width, 3), dtype=torch.uint8, device="cuda"))
    with pytest.raises(RuntimeError):
        enc.render_host(10)
    enc.close()


def test_installing_after_the_first_line_is_refused(built):
    import torch
    H = built
    enc = _encoder(H, "i", 16000000, 0, dict(vfilter=True, noaudio=True))
    frames = _pictures(enc, 1, 9)
    enc.set_source(frames, None)
    enc.render_host(10)
    with pytest.raises(RuntimeError):
        enc.set_device_source(_layout(frames, "hwc-rgb"))
    assert enc._L.htv_set_video_device_source(enc._h, H._READ_VIDEO_DEVICE(), None) == H.HTV_ERROR
    enc.close()
