"""GPU parity tests proper: the CUDA path, called through the C-ABI, against the oracle
on the same inputs. Bit-exact wherever the path is integer-only (video, chroma, VSB,
NICAM); within the +-1 LSB BASELINE.json states wherever an FM/AM sound carrier or the
offset mixer (closed-form NCOs) contributes."""
import numpy as np
import pytest

import orc

pytestmark = pytest.mark.gpu


def _diff(a, b):
    assert a.shape == b.shape
    return np.abs(a.astype(np.int32) - b.astype(np.int32))


def _pair(H, mode, rate, nlines, frames=None, audio=None, **kw):
    conf = H.mode_config(mode, **kw)
    enc = H.Encoder(conf, rate)
    o = orc.Oracle(conf, rate)
    if frames is None and audio is None:
        enc.open_test_source()
        o.open_test_source()
    else:
        enc.set_source(frames, audio)
        o.set_source(frames, audio)
    got = enc.render_host(nlines)
    want = o.render(nlines)
    launches = enc.kernel_launches
    enc.close()
    o.close()
    assert launches > 0
    return got, want


# (mode, rate, lines, overrides, tolerance): BASELINE.json configs 1-5 first
CASES = [
    ("pal", 16000000, 1300, dict(), 0),                                   # config 1
    ("i", 16000000, 1300, dict(vfilter=True), 1),                         # config 2
    ("m", 13500000, 1100, dict(vfilter=True), 1),                         # config 3
    ("i", 20000000, 700, dict(vfilter=True), 1),                          # config 5 (one channel)
    ("i", 16000000, 1300, dict(vfilter=True, noaudio=True), 0),           # video + VSB only: exact
    ("i", 16000000, 700, dict(vfilter=True, nonicam=True), 1),
    ("i", 16000000, 700, dict(), 1),                                      # no filter: no audio lead
    ("i", 16000000, 1300, dict(vfilter=True, noaudio=False, nocolour=True), 1),
    ("m", 13500000, 1100, dict(vfilter=True, noaudio=True), 0),
    ("ntsc", 13500000, 1100, dict(), 0),
    ("pal", 16000000, 700, dict(vfilter=True), 0),                        # real low-pass filter
    ("b", 16000000, 700, dict(vfilter=True), 1),
    ("pal-m", 13500000, 600, dict(vfilter=True), 1),
    ("pal-n", 16000000, 700, dict(vfilter=True), 1),
    ("l", 16000000, 1300, dict(vfilter=True), 1),                         # config 4: SECAM-L, AM sound + NICAM
    ("l", 16000000, 1300, dict(vfilter=True, noaudio=True), 0),           # SECAM chroma is exact
    ("secam", 16000000, 1300, dict(), 0),
    ("d", 16000000, 700, dict(vfilter=True), 1),
    ("secam-i", 16000000, 700, dict(vfilter=True, nonicam=True), 1),
    ("i", 16000000, 700, dict(vfilter=True, swap_iq=True), 1),
    ("i", 16000000, 700, dict(vfilter=True, invert_video=True, noaudio=True), 0),
    ("i", 16000000, 700, dict(vfilter=True, level=0.7, volume=2.0), 1),
    # FM video (SURVEY.md section 8f rank 2): closed-form phase = prefix sum over every sample. Without a
    # sound carrier the modulating signal is exact integer work, so the phase is exact: +-1 LSB for ever.
    ("pal-fm", 20000000, 700, dict(vfilter=True, noaudio=True), 1),
    ("pal-fm", 20000000, 700, dict(noaudio=True), 1),
    ("pal-fm", 20250000, 500, dict(vfilter=True, noaudio=True), 1),
    ("pal-fm", 14000000, 500, dict(vfilter=True, noaudio=True), 1),
    ("ntsc-fm", 18000000, 600, dict(vfilter=True, noaudio=True), 1),
    ("ntsc-fm", 20250000, 600, dict(vfilter=True, noaudio=True), 1),      # W = 1287, 71 taps
    ("secam-fm", 20250000, 500, dict(vfilter=True, noaudio=True), 1),
    ("pal-fm", 20000000, 500, dict(vfilter=True, noaudio=True, deviation=8e6, level=0.5), 1),
]


@pytest.mark.parametrize("mode,rate,nlines,kw,tol", CASES)
def test_test_pattern_parity(built, mode, rate, nlines, kw, tol):
    got, want = _pair(built, mode, rate, nlines, **kw)
    d = _diff(got, want)
    assert d.max() <= tol, f"max |diff| = {d.max()} at {np.argmax(d)}; {np.count_nonzero(d > tol)} samples out of tolerance"
    if tol:
        assert (d == 0).mean() > 0.97, f"only {(d == 0).mean():.4f} of samples exact"


def test_nicam_only_is_exact(built):
    """NICAM is integer-only end to end (frame encoder, DQPSK, pulse shaping, carrier LUT)."""
    H = built
    conf = H.mode_config("i", vfilter=True)
    conf.fm_mono_level = 0.0
    conf.fm_mono_carrier = 0.0
    enc = H.Encoder(conf, 16000000); o = orc.Oracle(conf, 16000000)
    enc.open_test_source(); o.open_test_source()
    got, want = enc.render_host(1300), o.render(1300)
    enc.close(); o.close()
    assert _diff(got, want).max() == 0


def test_random_pictures_and_loud_audio(built):
    """Random frames (a new one every frame) and full-scale noise audio: exercises the
    fp64 RGB->YUV path on arbitrary colours, the limiter's attack, and NICAM companding."""
    H = built
    rng = np.random.default_rng(1234)
    conf = H.mode_config("i", vfilter=True)
    enc = H.Encoder(conf, 16000000)
    frames = rng.integers(0, 1 << 24, size=(3, enc.active_lines, enc.active_width), dtype=np.uint32)
    audio = rng.integers(-32768, 32767, size=(40000, 2), dtype=np.int16)
    enc.close()
    got, want = _pair(H, "i", 16000000, 1900, frames=frames, audio=audio, vfilter=True)
    d = _diff(got, want)
    assert d.max() <= 1, f"max |diff| = {d.max()}; {np.count_nonzero(d > 1)} out of tolerance"


def test_chunking_is_invisible(built):
    """The stream is the same however the caller slices it into render calls."""
    H = built
    conf = H.mode_config("i", vfilter=True)
    a = H.Encoder(conf, 16000000); a.open_test_source()
    whole = a.render_host(1500); a.close()
    b = H.Encoder(conf, 16000000); b.open_test_source()
    parts = np.concatenate([b.render_host(n) for n in (1, 311, 313, 625, 250)]); b.close()
    assert np.array_equal(whole, parts)


def test_next_line_view_matches_batches(built):
    H = built
    conf = H.mode_config("pal")
    a = H.Encoder(conf, 16000000); a.open_test_source()
    ref = a.render_host(700).reshape(700, -1); a.close()
    b = H.Encoder(conf, 16000000); b.open_test_source()
    for k in range(700):
        iq, frame, line = b.next_line()
        assert frame == k // 625 + 1 and line == k % 625 + 1
        assert np.array_equal(iq[0::2], ref[k]) and not iq[1::2].any()
    b.close()


def test_secam_random_pictures_exact(built):
    """SECAM chroma on random pictures (a new one every frame), rendered in uneven pieces so
    the cross-line state (IIR state, the two aliased buffer words) crosses launch boundaries."""
    H = built
    rng = np.random.default_rng(99)
    conf = H.mode_config("l", vfilter=True, noaudio=True)
    enc = H.Encoder(conf, 16000000)
    frames = rng.integers(0, 1 << 24, size=(3, enc.active_lines, enc.active_width), dtype=np.uint32)
    enc.set_source(frames, None)
    got = np.concatenate([enc.render_host(n) for n in (1, 2, 23, 300, 625, 949)])
    enc.close()
    o = orc.Oracle(conf, 16000000)
    o.set_source(frames, None)
    want = o.render(1900)
    o.close()
    assert _diff(got, want).max() == 0


def test_offset_mixer(built):
    """--offset: the complex NCO multiply of ref video.c:3482-3515 incl. its INT16_MAX start-up
    (the first 32767 samples are scaled to ~0). Closed-form NCO: +-1 LSB on top of the sound carriers'."""
    got, want = _pair(built, "i", 16000000, 700, vfilter=True, offset=2000000)
    d = _diff(got, want)
    assert d.max() <= 2, f"max |diff| = {d.max()}"
    assert (d <= 1).mean() > 0.999
    got, want = _pair(built, "i", 16000000, 700, vfilter=True, offset=-3500000, noaudio=True)
    assert _diff(got, want).max() <= 1


def test_memory_source_equals_callback_source(built):
    """htv_av_memory_open (C) and Python callbacks feed the same stream."""
    H = built
    rng = np.random.default_rng(5)
    conf = H.mode_config("i", vfilter=True)
    a = H.Encoder(conf, 16000000)
    frames = rng.integers(0, 1 << 24, size=(2, a.active_lines, a.active_width), dtype=np.uint32)
    audio = rng.integers(-8000, 8000, size=(5000, 2), dtype=np.int16)
    a.set_source(frames, audio, audio_block=777)
    x = a.render_host(1400); a.close()
    b = H.Encoder(conf, 16000000)
    b.open_memory_source(frames, audio, audio_block=1000)
    y = b.render_host(1400); b.close()
    assert np.array_equal(x, y)


def test_fm_video_chunking_and_offset(built):
    """The FM video phase is carried across calls and sub-batches; the offset mixer follows it."""
    H = built
    conf = H.mode_config("pal-fm", vfilter=True)
    a = H.Encoder(conf, 20000000); a.open_test_source()
    whole = a.render_host(1400); a.close()
    b = H.Encoder(conf, 20000000); b.open_test_source()
    parts = np.concatenate([b.render_host(n) for n in (1, 311, 313, 625, 150)]); b.close()
    assert np.array_equal(whole, parts)
    # full-scale FM video (|IQ| reaches 32768.2 through the reference's floors) overflows int16 in the offset
    # mixer now and then, in the reference too: compare modulo the wrap
    got, want = _pair(H, "pal-fm", 20000000, 500, vfilter=True, noaudio=True, offset=-3000000, swap_iq=True)
    d = np.abs((got.astype(np.int32) - want.astype(np.int32) + 32768) % 65536 - 32768)
    assert d.max() <= 3 and (d <= 1).mean() > 0.999, (d.max(), (d <= 1).mean())     # +-1 turned by the mixer, +-1 of its NCO
    got, want = _pair(H, "pal-fm", 20000000, 500, vfilter=True, noaudio=True, offset=2500000, level=0.5)
    d = _diff(got, want)
    assert d.max() <= 2 and (d <= 1).mean() > 0.99, (d.max(), (d <= 1).mean())


def test_fm_video_long_run_stays_within_one_lsb(built):
    """> 9000 lines: several sub-batches, hundreds of renormalisation periods, no drift."""
    got, want = _pair(built, "pal-fm", 20000000, 9500, vfilter=True, noaudio=True)
    d = _diff(got, want)
    assert d.max() <= 1, d.max()


@pytest.mark.parametrize("mode,rate,nlines,kw", [
    ("pal-fm", 20000000, 2500, dict(vfilter=True)),
    ("pal-fm", 20000000, 700, dict()),
    ("ntsc-fm", 18000000, 1100, dict(vfilter=True)),
    ("secam-fm", 20250000, 700, dict(vfilter=True)),
])
def test_fm_video_with_sound_carrier(built, mode, rate, nlines, kw):
    """With a sound subcarrier the modulating signal inherits the carrier's +-1 LSB (closed-form NCO against
    the reference's Q31 recurrence), and an FM modulator INTEGRATES its input: every baseband sample that is
    1 LSB off turns everything after it by one LUT step (2 pi * deviation / 32767 / fs = 1.5e-4 rad, 5 LSB of
    arc at full scale), and because the 6.5 MHz carrier repeats every 40 samples at 20 Msps such samples come
    in runs inside one 32 kHz audio sample. No parallel formulation can avoid this - the reference's own
    truncation noise decides those samples (DESIGN.md section 2, FM video). Parity is therefore stated as:
    the same signal up to a slowly wandering common rotation (measured: a random walk of ~15 LUT steps =
    2e-3 rad over 700 lines), the instantaneous frequency identical except at < 0.5 % of the samples, a third to
    two thirds of the lines within 1 LSB once the line's mean rotation is removed. Without the sound carrier (above) the path is
    exact to +-1 LSB for ever."""
    got, want = _pair(built, mode, rate, nlines, **kw)
    g = got.astype(np.float64).reshape(nlines, -1, 2); g = g[..., 0] + 1j * g[..., 1]
    w = want.astype(np.float64).reshape(nlines, -1, 2); w = w[..., 0] + 1j * w[..., 1]
    rot = np.angle((g * np.conj(w)).sum(axis=1))
    res = g * np.exp(-1j * rot)[:, None] - w
    worst = np.maximum(np.abs(res.real), np.abs(res.imag)).max(axis=1)
    step = 2 * np.pi * 16e6 / 32767 / rate
    print(f"{mode} {rate}: worst residual {worst.max():.2f} LSB, lines within 1.5 LSB {(worst <= 1.5).mean():.4f}, "
          f"rotation after {nlines} lines {rot[-1] / step:.1f} LUT steps (max {np.abs(rot).max() / step:.1f})")
    # what is left after removing the common rotation of the carrier is small on most lines; the rotation itself stays
    # within a few tens of LUT steps over 700 - 2 500 lines
    assert (worst <= 1.5).mean() > 0.30, (worst <= 1.5).mean()
    assert worst.max() <= 90.0, worst.max()
    assert np.abs(rot).max() < step * (55 + 0.01 * nlines), np.abs(rot).max() / step
    df = np.angle(g[:, 1:] * np.conj(g[:, :-1])) - np.angle(w[:, 1:] * np.conj(w[:, :-1]))
    df = (df + np.pi) % (2 * np.pi) - np.pi
    assert (np.abs(df) > 0.6 * step).mean() < 0.005, (np.abs(df) > 0.6 * step).mean()


def test_audio_block_longer_than_a_ring_piece_is_not_dropped(built):
    """ADVICE r1: a source may hand over its PCM in one block of any size (ref video.c:3280). A block longer
    than a quarter of the device ring (262 144 pairs = 8.2 s) goes up in pieces across render calls; nothing
    of it is lost. 9.4 s of noise in ONE block vs the same audio in 8 192-pair blocks, compared behind
    the 8.2 s mark; the stream in between stays on the device."""
    import torch
    H = built
    rng = np.random.default_rng(5)
    audio = rng.integers(-20000, 20000, size=(300000, 2), dtype=np.int16)
    conf = H.mode_config("i", vfilter=True)
    outs = []
    for block in (0, 8192):
        enc = H.Encoder(conf, 16000000)
        enc.set_source(None, audio, audio_block=block)
        scratch = torch.empty(40000 * enc.width * 2, dtype=torch.int16, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        for _ in range(3):
            enc.render(40000, scratch.data_ptr(), st)            # 7.68 s
        enc.render(12000, scratch.data_ptr(), st)                # .. 8.45 s: the tail of the first piece and beyond
        torch.cuda.synchronize()
        outs.append(scratch[: 12000 * enc.width * 2].cpu().numpy().copy())
        outs.append(enc.render_host(3000))                       # 9.0 s .. 9.2 s: well into the second piece
        enc.close()
    assert np.array_equal(outs[0], outs[2]) and np.array_equal(outs[1], outs[3])
    assert np.count_nonzero(outs[1]) > 1000


def test_next_line_prefetch_is_invisible(built):
    """htv_set_prefetch: the frame after the one being handed out is rendered in the background (two pinned
    frames); the lines that come out are the same, frame and line numbers included."""
    H = built
    conf = H.mode_config("i", vfilter=True)
    outs = []
    for pf in (False, True):
        enc = H.Encoder(conf, 16000000); enc.open_test_source()
        enc.render_host(100)                                     # start in the middle of a frame
        enc.set_prefetch(pf)
        got = [enc.next_line() for _ in range(1500)]
        enc.close()
        outs.append(got)
    for (a, fa, la), (b, fb, lb) in zip(*outs):
        assert fa == fb and la == lb and np.array_equal(a, b)
    assert outs[0][0][2] == 101 and outs[0][525][1:] == (2, 1)
