"""--pixelrate on the GPU (SURVEY.md section 8f rank 4): raster in a second device context at the pixel
rate, k_resample (the reference's polyphase resampler in closed form), then the usual modulator - against the
oracle, which is pinned bit for bit to the reference's own --pixelrate output (tests/test_oracle_vs_ref.py).

This is the one path that runs the split modulators (k_mod_mma, k_mod_tma, k_mod) and so the sound stage's
four-consecutive-samples form. Each row of MATRIX states the W <- Wp it exists for and the `line_kernel` string it must
run, so that a change to the selection cannot move a row onto another path unnoticed; test_tables_and_abi.py checks the
same rows against the C selection without a GPU, and that together they reach every split modulator and CTA size.

Per row, as in test_gpu_zz_line_widths.py: with no sound bit-exact; with NICAM only bit-exact; with the mode's sound
within +-1 LSB and >= 97 % exact in every 128-sample tile column of the blanking lines and of the picture lines. With
--offset: the sound carriers (+-1 LSB each, closed-form NCOs) behind the offset mixer (its own NCO: +-1 LSB) stack to
2 LSB on a few samples per thousand lines - the relaxed tolerance include/hacktv_b200.h states."""
import os

import numpy as np
import pytest

import orc
from test_gpu_vbi import _overlays
from test_gpu_zz_line_widths import _check_sound, _has, _lines

pytestmark = pytest.mark.gpu

F = dict(vfilter=True)


def rs(mod, maxt, minb):
    return f"k_raster + k_resample + {mod}<{maxt},{minb}>"


MMA, MMA384 = rs("k_mod_mma", 256, 4), rs("k_mod_mma", 384, 2)
TMA, TMA384 = rs("k_mod_tma", 256, 4), rs("k_mod_tma", 384, 2)
MOD, MOD384 = rs("k_mod", 256, 4), rs("k_mod", 384, 2)

# (mode, sample rate, pixel rate, overrides, W, Wp, line_kernel); "pitched": 128 does not divide W, so k_mod_mma reads
# the pitched byte planes (htv_mma_fir.h); k_mod reads the int16 stream, where 4 does not divide W
MATRIX = [
    ("pal", 16000000, 13500000, {}, 1024, 864, TMA),                  # 32/27, real output
    ("i", 16000000, 13500000, F, 1024, 864, MMA),                     # VSB + FM + NICAM
    ("i", 16000000, 13500000, {}, 1024, 864, TMA),
    ("i", 20000000, 13500000, F, 1280, 864, MMA384),                  # 40/27
    ("i", 16000000, 14000000, F, 1024, 896, MMA),                     # 8/7
    ("pal", 20000000, 13500000, {}, 1280, 864, TMA384),               # the TMA modulator at 384 threads
    ("i", 13500000, 16000000, F, 864, 1024, MMA),                     # down-sampling 27/32, pitched: partial last tile
    ("pal", 13500000, 16000000, {}, 864, 1024, TMA),                  # down-sampling, real output
    ("i", 16000000, 20000000, F, 1024, 1280, MMA),                    # down-sampling 4/5 on whole tiles; 320-thread raster
    ("i", 10000000, 13500000, F, 640, 864, MMA),                      # 20/27; NICAM symbols < 33 samples: generic sum
    ("i", 20250000, 13500000, F, 1296, 864, MMA384),                  # 3/2, pitched at 384 threads
    ("m", 13500000, 9000000, F, 858, 572, MMA),                       # 525 lines, pitched, 4 does not divide W
    ("pal-m", 13500000, 9000000, F, 858, 572, MMA),                   # PAL on the 525-line raster
    ("ntsc", 13500000, 9000000, {}, 858, 572, MOD),                   # k_resample's int16 store, real output
    ("ntsc", 20250000, 13500000, {}, 1287, 858, MOD384),              # the same at 384 threads
    ("i", 16000000, 13515625, F, 1024, 865, MMA),                     # odd raster width, 1024 filter phases
    ("pal", 16000000, 13515625, {}, 1024, 865, TMA),
    ("i", 16000000, 13500000, dict(vfilter=True, nocolour=True), 1024, 864, MMA),   # mono raster
]
WHOLE = ("i", 16000000, 13500000)          # whole tiles: contiguous byte planes
PITCHED = ("i", 13500000, 16000000)        # partial last tile: pitched byte planes
NTSC = ("m", 13500000, 9000000)


def case_id(c):
    mode, rate, prate, kw = c[:4]
    return f"{mode}-{rate}-from-{prate}" + "".join(f"-{k}" for k, v in kw.items() if v)


def _render(H, conf, rate, prate, pieces, frames=None, audio=None, vbi=None, passthru=None):
    """The CUDA path's stream over calls of `pieces` lines, and the line kernel it ran."""
    enc = H.Encoder(conf, rate, prate)
    if frames is None:
        enc.open_test_source()
    else:
        enc.set_source(frames, audio)
    if vbi is not None:
        enc.set_vbi_lines(vbi)
    if passthru is not None:
        enc.set_passthru(passthru)
    got = np.concatenate([enc.render_host(n) for n in pieces])
    name = enc.line_kernel
    enc.close()
    return got, name


def _oracle(conf, rate, prate, nlines, frames=None, audio=None, vbi=None, passthru=None):
    o = orc.Oracle(conf, rate, prate)
    if frames is None:
        o.open_test_source()
    else:
        o.set_source(frames, audio)
    for line, add, rep in vbi or ():
        o.add_vbi_line(line, add, rep)
    if passthru is not None:
        o.set_passthru(passthru)
    want = o.render(nlines)
    o.close()
    return want


def _picture_lines(H, conf, rate, quiet):
    """Lines with picture content: the I samples over the middle half of the active width span more than 256 LSB. A
    resampled blanking line is flat but for the rounding of the filter phases, so it is not exactly constant."""
    g = H.Tables(conf, rate).get("geometry")
    W, al, aw = int(g[0]), int(g[2]), int(g[3])
    rows = quiet.reshape(-1, W, 2 if conf.output_type == 0 else 1)[:, al + aw // 4: al + 3 * aw // 4, 0].astype(np.int32)
    return rows.max(axis=1) - rows.min(axis=1) > 256


def _within(got, want, tol, what=""):
    d = np.abs(got.astype(np.int32) - want.astype(np.int32))
    assert d.max() <= tol, f"{what}: max |diff| {d.max()} at {np.argmax(d)}; {np.count_nonzero(d > tol)} values over {tol}"


def _row(mode, rate, prate):
    return next(c for c in MATRIX if c[:3] == (mode, rate, prate) and c[3] == F)


@pytest.mark.parametrize("mode,rate,prate,kw,W,Wp,kernel", MATRIX, ids=[case_id(c) for c in MATRIX])
def test_pixelrate_matrix_against_the_oracle(built, mode, rate, prate, kw, W, Wp, kernel):
    H = built
    conf = H.mode_config(mode, **kw)
    nlines = _lines(conf)
    quiet = H.mode_config(mode, noaudio=True, **kw)
    got, name = _render(H, quiet, rate, prate, [nlines])
    assert name == kernel, f"{mode} {rate} <- {prate} ran {name}, the row exists for {kernel}"
    want = _oracle(quiet, rate, prate, nlines)
    assert got.size == nlines * W * (2 if conf.output_type == 0 else 1)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"no sound: {bad.size} values differ, first at line {bad[0] // (got.size // nlines)}"
    if _has(conf, "nicam"):
        nic = H.mode_config(mode, **kw)
        nic.fm_mono_level = nic.fm_mono_carrier = nic.am_audio_level = nic.am_mono_carrier = 0.0
        got, name = _render(H, nic, rate, prate, [nlines])
        assert name == kernel
        bad = np.flatnonzero(got != _oracle(nic, rate, prate, nlines))
        assert bad.size == 0, f"NICAM only: {bad.size} values differ, first at line {bad[0] // (got.size // nlines)}"
    if _has(conf, "fm") or _has(conf, "am") or _has(conf, "nicam"):
        got, name = _render(H, conf, rate, prate, [nlines])
        assert name == kernel
        _check_sound(got, _oracle(conf, rate, prate, nlines), W, _picture_lines(H, conf, rate, want), "with sound")


OFFSET = [
    ("i", 16000000, 13500000, dict(vfilter=True, offset=2000000), 2),
    ("i", 16000000, 13500000, dict(vfilter=True, offset=2000000, noaudio=True), 1),
    ("i", 13500000, 16000000, dict(vfilter=True, offset=2000000), 2),
    ("i", 13500000, 16000000, dict(vfilter=True, offset=-1500000, swap_iq=True), 2),
]


@pytest.mark.parametrize("mode,rate,prate,kw,tol", OFFSET, ids=[case_id(c) for c in OFFSET])
def test_pixelrate_offset_mixer(built, mode, rate, prate, kw, tol):
    conf = built.mode_config(mode, **kw)
    got, _ = _render(built, conf, rate, prate, [500])
    _within(got, _oracle(conf, rate, prate, 500), tol)


def _random_source(H, mode, rate, prate, seed):
    """A new random picture every frame (three, used in turn) and full-scale noise audio."""
    e = H.Encoder(H.mode_config(mode), rate, prate); al, aw = e.active_lines, e.active_width; e.close()
    rng = np.random.default_rng(seed)
    frames = rng.integers(0, 1 << 24, size=(3, al, aw), dtype=np.uint32)
    audio = rng.integers(-32768, 32767, size=(40000, 2), dtype=np.int16)
    return frames, audio


@pytest.mark.parametrize("mode,rate,prate", [WHOLE, PITCHED, NTSC])
def test_pixelrate_random_pictures_loud_audio_and_uneven_calls(built, mode, rate, prate):
    """Random pictures bit-exact without sound and within +-1 LSB with full-scale noise audio; calls of 1, 2, 311, 313,
    625 lines and the rest give the stream one call gives."""
    H = built
    kernel = _row(mode, rate, prate)[6]
    frames, audio = _random_source(H, mode, rate, prate, 37)
    quiet = H.mode_config(mode, vfilter=True, noaudio=True)
    got, name = _render(H, quiet, rate, prate, [1300], frames, audio)
    assert name == kernel
    bad = np.flatnonzero(got != _oracle(quiet, rate, prate, 1300, frames, audio))
    assert bad.size == 0, f"no sound: {bad.size} values differ, first at value {bad[0]}"
    conf = H.mode_config(mode, vfilter=True)
    got, name = _render(H, conf, rate, prate, [1300], frames, audio)
    _within(got, _oracle(conf, rate, prate, 1300, frames, audio), 1, "with sound")
    parts, name = _render(H, conf, rate, prate, [1, 2, 311, 313, 625, 48], frames, audio)
    assert name == kernel
    assert np.array_equal(got, parts), f"{np.count_nonzero(got != parts)} values differ"


@pytest.mark.parametrize("mode,rate,prate", [WHOLE, PITCHED])
def test_pixelrate_call_longer_than_a_sub_batch(built, mode, rate, prate):
    """9000 lines in one device-resident call cross the 8192-line sub-batch (at W = 1024 the modulator's context sets it,
    at W = 864 the 1024-sample raster context's): the raster descriptors, raster rows and resampled rows of the second
    sub-batch equal the same lines rendered in pieces, and the oracle."""
    import torch
    H = built
    conf = H.mode_config(mode, vfilter=True)
    n = 9000
    enc = H.Encoder(conf, rate, prate); enc.open_test_source()
    W = enc.width
    buf = torch.zeros(n * W * 2, dtype=torch.int16, device="cuda")
    enc.render(n, buf.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    whole = buf.cpu().numpy()
    assert enc.line_kernel == _row(mode, rate, prate)[6]
    enc.close()
    parts, _ = _render(H, conf, rate, prate, [4000, 4000, 1000])
    assert np.array_equal(whole, parts), f"{np.count_nonzero(whole != parts)} values differ, first at line " \
        f"{np.flatnonzero(whole != parts)[0] // (2 * W)}"
    _within(whole, _oracle(conf, rate, prate, n), 1, "with sound")


@pytest.mark.parametrize("mode,rate,prate", [WHOLE, PITCHED, NTSC])
def test_pixelrate_vbi_overlays_at_the_raster_width(built, mode, rate, prate):
    """VBI overlays are drawn on the raster, at the pixel rate (the oracle's add_vbi_line): bit-exact without sound, also
    with an overlay that reaches the last sample of its line and a call boundary right behind it."""
    H = built
    conf = H.mode_config(mode, vfilter=True, noaudio=True)
    enc = H.Encoder(conf, rate, prate)
    Wr, lines = enc.raster_width, enc.lines
    enc.close()
    assert Wr == _row(mode, rate, prate)[5]
    ov = [(l, a, r) for (l, a, r) in _overlays(Wr, Wr // 2, 5) if lines == 625 or l < 300]
    end = np.zeros(Wr, dtype=np.int16); end[Wr - 300:] = 7000                  # non-zero up to sample Wr - 1
    ov += [(l, end, (0, 0, 0)) for l in (21, 22, 273)]
    ov.sort(key=lambda e: e[0])
    got, _ = _render(H, conf, rate, prate, [700], vbi=ov)
    want = _oracle(conf, rate, prate, 700, vbi=ov)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} values differ, first at line {bad[0] // (got.size // 700)}"
    plain, _ = _render(H, conf, rate, prate, [700])
    assert np.count_nonzero(got != plain) > 1000                            # the overlays are really there
    parts, _ = _render(H, conf, rate, prate, [21, 1, 1, 250, 427], vbi=ov)  # boundaries right behind lines 21, 22, 273
    assert np.array_equal(got, parts), f"{np.count_nonzero(got != parts)} values differ"


@pytest.mark.parametrize("mode,rate,prate", [WHOLE, PITCHED])
def test_pixelrate_passthru(built, mode, rate, prate):
    """An external stream summed behind the modulator; two fill lines in front of it (resampler + filter)."""
    H = built
    conf = H.mode_config(mode, vfilter=True, noaudio=True)
    enc = H.Encoder(conf, rate, prate); W = enc.width; enc.close()
    ext = np.random.default_rng(3).integers(-32768, 32767, size=(800 * W + W // 3, 2), dtype=np.int16)
    got, _ = _render(H, conf, rate, prate, [700], passthru=ext)
    want = _oracle(conf, rate, prate, 700, passthru=ext)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} values differ, first at line {bad[0] // (2 * W)}"


@pytest.mark.parametrize("mode,rate,prate", [WHOLE, PITCHED])
def test_pixelrate_render_add_into_a_device_buffer(built, mode, rate, prate):
    """htv_render_add into a stream already in device memory equals the oracle's passthru sum."""
    import torch
    H = built
    n = 400
    ca = H.mode_config(mode, vfilter=True, offset=-3000000, level=0.5)
    cb = H.mode_config(mode, vfilter=True, noaudio=True, level=0.5)
    a = H.Encoder(ca, rate); a.open_test_source()
    b = H.Encoder(cb, rate, prate); b.open_test_source()
    W = a.width
    delay = b.passthru_delay_lines
    buf = torch.zeros((n + delay) * W * 2, dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    a.render(n + delay, buf.data_ptr(), st)
    b.render_add(n, buf.data_ptr() + delay * W * 4, st)
    torch.cuda.synchronize()
    got = buf[delay * W * 2:].cpu().numpy()
    assert b.line_kernel == _row(mode, rate, prate)[6]
    a.close(); b.close()

    oa = orc.Oracle(ca, rate); oa.open_test_source()
    sa = oa.render(n + delay); oa.close()
    want = _oracle(cb, rate, prate, n, passthru=sa.reshape(-1, 2))
    d = (got.astype(np.int32) - want.astype(np.int32) + 32768) % 65536 - 32768
    assert np.abs(d).max() <= 2, np.abs(d).max()                  # channel A: sound + offset NCOs, +-1 LSB each
    assert np.count_nonzero(d) < d.size // 20


def test_pixelrate_chunking_and_scalar_filter(built):
    H = built
    conf = H.mode_config("i", vfilter=True)
    a = H.Encoder(conf, 16000000, 13500000); a.open_test_source(); whole = a.render_host(1500); a.close()
    b = H.Encoder(conf, 16000000, 13500000); b.open_test_source()
    parts = np.concatenate([b.render_host(n) for n in (1, 311, 313, 625, 250)]); b.close()
    assert np.array_equal(whole, parts)
    os.environ["HTV_FIR"] = "scalar"
    try:
        c = H.Encoder(conf, 16000000, 13500000); c.open_test_source(); scalar = c.render_host(1500); c.close()
    finally:
        os.environ.pop("HTV_FIR", None)
    assert np.array_equal(whole, scalar)
