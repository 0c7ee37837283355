"""The encoder below 10 Msps on the paths test_gpu_zz_low_rates.py does not reach, on the device, against the oracle:
  - the PS forms: k_line encoders whose colour subcarrier does not repeat within 4 frames (comp_phases P = 0), so that
    there is no composite store and k_picture converts each picture (RGB -> YUV, chroma_fir4<3|5|7>) for k_line. NTSC at
    most rates below 10 Msps, PAL60 at every rate and PAL at rounded widths (1.7 Msps: W = 109) take this path, at 3, 5
    and 7 chroma taps, with CSAT (NTSC at 7 Msps: the 7 taps sum to 32770) and in single-warp CTAs (W <= 128). The
    kernel name does not show PS, so every row states its P as well;
  - --pixelrate: k_raster in the pixel-rate context with 1, 3, 5 and 7 chroma taps (and 11 where the pixel rate is 13.5
    Msps), down to the 32-sample raster; k_resample at I / D from 32 / 1 to 5 / 54; the split modulators behind it at
    W <= 128, k_mod_mma on pitched planes (128 does not divide W) as on contiguous ones;
  - S-Video: the 3-, 5- and 7-tap low-pass, the single-warp CTA, the CSAT rate, the PS form (its chroma rows in shared
    memory) and SECAM's Q plane from 2 to 10 Msps.

Each row states its W (and Wp, the pixel-rate raster's width), its P or chroma taps, and the `line_kernel` string it must
run; test_low_rate_paths_host.py checks the same rows against the tables and the C selection without a GPU, and that
together they reach every path above. Composite and pixel-rate rows are checked as the line-width matrix does
(test_gpu_zz_line_widths.py): bit-exact without sound, bit-exact with NICAM only, and with the mode's sound within +-1 LSB
and >= 97 % exact in every tile column. S-Video rows are bit-exact against sv_oracle. test_oracle_vs_ref.py pins the
oracle to the reference at every composite and pixel-rate row, test_s_video_host.py sv_oracle at every S-Video row."""
import numpy as np
import pytest

import orc
import sv_oracle
import test_gpu_zz_pixelrate as PR
from test_gpu_zz_line_widths import _check_sound, _has, _lines, _oracle, _picture_lines, _render, kl, sec
from test_gpu_zz_pixelrate import MMA, MMA384, MOD, TMA

pytestmark = pytest.mark.gpu

F = dict(vfilter=True)
S = dict(s_video=True)
SF = dict(s_video=True, vfilter=True)


def sv(kernel):
    return kernel[:-1] + ",SV>"


# PS forms: (mode, rate, overrides, W, P, chroma taps, line_kernel)
PS = [
    ("ntsc", 1500000, {}, 95, 0, 3, kl(0, 0, 0, 0, 256)),            # one partial tile: a single-warp CTA
    ("ntsc", 2000000, {}, 127, 0, 3, kl(0, 0, 0, 0, 256)),
    ("m", 1500000, F, 95, 0, 3, kl(1, 1, 0, 0, 256)),                # VSB + FM
    ("m", 4000000, F, 254, 0, 3, kl(1, 1, 0, 0, 256)),
    ("pal60", 4500000, F, 286, 0, 5, kl(1, 0, 0, 0, 256)),
    ("ntsc", 7000000, F, 445, 0, 7, kl(1, 0, 0, 1, 256)),            # the 7 taps sum to 32770: PS with CSAT
    ("pal60-i", 8000000, F, 508, 0, 7, kl(1, 1, 0, 0, 256)),         # NICAM
    ("pal", 1700000, {}, 109, 0, 3, kl(0, 0, 0, 0, 256)),            # PAL at a rounded width
]

# --pixelrate: (mode, sample rate, pixel rate, overrides, W, Wp, chroma taps at the pixel rate, line_kernel); the
# modulator is k_mod_mma where the video filter runs (pitched planes where 128 does not divide W), else k_mod_tma where 4
# divides W, else k_mod
PIXELRATE = [
    ("i", 16000000, 2000000, F, 1024, 128, 3, MMA),                  # I / D = 8 / 1
    ("pal", 16000000, 500000, {}, 1024, 32, 1, TMA),                 # the raster at the 32-sample limit; 32 / 1
    ("i", 16000000, 1500000, F, 1024, 96, 3, MMA),                   # 32 / 3
    ("i", 20000000, 1250000, F, 1280, 80, 1, MMA384),
    ("i", 4000000, 13500000, F, 256, 864, 11, MMA),
    ("pal", 2000000, 13500000, {}, 128, 864, 11, TMA),               # 4 / 27
    ("i", 1250000, 13500000, F, 80, 864, 11, MMA),                   # 5 / 54, pitched
    ("i", 1250000, 2000000, F, 80, 128, 3, MMA),                     # FM + NICAM, 39 samples per audio sample
    ("pal", 500000, 2000000, {}, 32, 128, 3, TMA),
    ("i", 1500000, 1000000, F, 96, 64, 1, MMA),
    ("pal", 8000000, 7000000, {}, 512, 448, 7, TMA),                 # CSAT chroma at the pixel rate
    ("ntsc", 2250000, 4500000, {}, 143, 286, 5, MOD),
    ("ntsc", 13500000, 2250000, {}, 858, 143, 3, MOD),
    ("m", 4500000, 6750000, F, 286, 429, 5, MMA),
    ("m", 13500000, 2250000, F, 858, 143, 3, MMA),
]

# S-Video: (mode, rate, overrides, W, P, chroma taps, line_kernel); SECAM has no chroma low-pass in the line kernel
S_VIDEO = [
    ("pal", 1500000, S, 96, 4, 3, sv(kl(0, 0, 0, 0, 256))),          # a single-warp CTA
    ("pal", 2000000, SF, 128, 4, 3, sv(kl(1, 0, 1, 0, 256))),
    ("pal", 4000000, SF, 256, 4, 3, sv(kl(1, 0, 1, 0, 256))),
    ("pal", 6750000, SF, 432, 4, 5, sv(kl(1, 0, 0, 0, 256))),
    ("pal", 7000000, SF, 448, 4, 7, sv(kl(1, 0, 0, 1, 256))),         # CSAT
    ("pal", 8000000, SF, 512, 4, 7, sv(kl(1, 0, 1, 0, 256))),
    ("ntsc", 2000000, S, 127, 0, 3, sv(kl(0, 0, 0, 0, 256))),         # PS in a single-warp CTA
    ("ntsc", 2250000, S, 143, 2, 3, sv(kl(0, 0, 0, 0, 256))),
    ("ntsc", 4500000, SF, 286, 2, 5, sv(kl(1, 0, 0, 0, 256))),
    ("ntsc", 7000000, SF, 445, 0, 7, sv(kl(1, 0, 0, 1, 256))),        # PS + CSAT
    ("pal60", 6750000, SF, 429, 0, 5, sv(kl(1, 0, 0, 0, 256))),       # PS
    ("525pal", 4500000, S, 286, 4, 5, sv(kl(0, 0, 0, 0, 256))),
    ("secam", 2000000, S, 128, 1, None, sv(sec(0, 0, 1, 256))),
    ("secam", 4000000, S, 256, 1, None, sv(sec(0, 0, 1, 256))),
    ("secam", 6000000, SF, 384, 1, None, sv(sec(1, 0, 1, 256))),
    ("secam", 10000000, SF, 640, 1, None, sv(sec(1, 0, 1, 256))),
]

# the rows whose chroma taps sum to more than 32768, so that the low-pass saturates
CSAT = [("composite", "ntsc", 7000000, 0, F), ("s_video", "pal", 7000000, 0, SF), ("s_video", "ntsc", 7000000, 0, SF),
        ("pixelrate", "pal", 8000000, 7000000, {})]


def case_id(mode, rate, kw, prate=0):
    return f"{mode}-{rate}" + (f"-from-{prate}" if prate else "") + "".join(f"-{k}" for k, v in kw.items() if v)


def _sv_lines(conf):
    return 1300 if conf.lines == 625 else 1100          # two frames and a few lines: frame parity, V-switch, D'r / D'b


def _run(H, kind, conf, rate, prate, pieces, frames=None):
    """The device's stream over calls of `pieces` lines, and the line kernel it ran."""
    if kind == "pixelrate":
        return PR._render(H, conf, rate, prate, pieces, frames, None)
    return _render(H, conf, rate, pieces, frames, None)


def _want(kind, conf, rate, prate, nlines, frames=None):
    if kind == "s_video":
        return sv_oracle.render(conf, rate, nlines, None if frames is None else (frames, None))
    if kind == "pixelrate":
        return PR._oracle(conf, rate, prate, nlines, frames, None)
    return _oracle(conf, rate, nlines, frames, None)


def _against_the_oracle(H, kind, mode, rate, prate, kw, W, kernel):
    """No sound bit-exact, NICAM only bit-exact, the mode's sound +-1 LSB and >= 97 % exact in every tile column."""
    conf = H.mode_config(mode, **kw)
    nlines = _lines(conf)
    quiet = H.mode_config(mode, **dict(kw, noaudio=True))
    got, name = _run(H, kind, quiet, rate, prate, [nlines])
    assert name == kernel, f"{mode} {rate} <- {prate} ran {name}, the row exists for {kernel}"
    want = _want(kind, quiet, rate, prate, nlines)
    assert got.size == nlines * W * (2 if conf.output_type == 0 else 1)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"no sound: {bad.size} values differ, first at line {bad[0] // (got.size // nlines)}"
    if _has(conf, "nicam"):
        nic = H.mode_config(mode, **kw)
        nic.fm_mono_level = nic.fm_mono_carrier = nic.am_audio_level = nic.am_mono_carrier = 0.0
        got, name = _run(H, kind, nic, rate, prate, [nlines])
        assert name == kernel
        bad = np.flatnonzero(got != _want(kind, nic, rate, prate, nlines))
        assert bad.size == 0, f"NICAM only: {bad.size} values differ, first at line {bad[0] // (got.size // nlines)}"
    if _has(conf, "fm") or _has(conf, "am") or _has(conf, "nicam"):
        got, name = _run(H, kind, conf, rate, prate, [nlines])
        assert name == kernel
        picture = (PR._picture_lines if kind == "pixelrate" else _picture_lines)(H, conf, rate, want)
        _check_sound(got, _want(kind, conf, rate, prate, nlines), W, picture, "with sound")


@pytest.mark.parametrize("mode,rate,kw,W,P,taps,kernel", PS, ids=[case_id(*c[:3]) for c in PS])
def test_ps_forms_against_the_oracle(built, mode, rate, kw, W, P, taps, kernel):
    H = built
    assert int(H.Tables(H.mode_config(mode, **kw), rate).get("comp_phases")[0]) == P
    _against_the_oracle(H, "composite", mode, rate, 0, kw, W, kernel)


@pytest.mark.parametrize("mode,rate,prate,kw,W,Wp,taps,kernel", PIXELRATE,
                         ids=[case_id(c[0], c[1], c[3], c[2]) for c in PIXELRATE])
def test_low_pixelrate_against_the_oracle(built, mode, rate, prate, kw, W, Wp, taps, kernel):
    _against_the_oracle(built, "pixelrate", mode, rate, prate, kw, W, kernel)


@pytest.mark.parametrize("mode,rate,kw,W,P,taps,kernel", S_VIDEO, ids=[case_id(*c[:3]) for c in S_VIDEO])
def test_low_rate_s_video_against_the_oracle(built, mode, rate, kw, W, P, taps, kernel):
    H = built
    conf = H.mode_config(mode, **kw)
    assert int(H.Tables(conf, rate).get("comp_phases")[0]) == P
    n = _sv_lines(conf)
    got, name = _render(H, conf, rate, [n])
    assert name == kernel, f"{mode} {rate} ran {name}, the row exists for {kernel}"
    assert got.size == n * W * 2
    bad = np.flatnonzero(got != sv_oracle.render(conf, rate, n))
    assert bad.size == 0, f"{bad.size} values differ, first at line {bad[0] // (2 * W)}, {'IQ'[bad[0] % 2]}"


# every PS row, and the CSAT rows
RANDOM = [("composite", c[0], c[1], 0, c[2]) for c in PS] + [("s_video", c[0], c[1], 0, c[2]) for c in S_VIDEO if c[4] == 0]
RANDOM += [c for c in CSAT if c not in RANDOM]


@pytest.mark.parametrize("kind,mode,rate,prate,kw", RANDOM, ids=[f"{c[0]}-" + case_id(c[1], c[2], c[4], c[3]) for c in RANDOM])
def test_random_pictures(built, kind, mode, rate, prate, kw):
    """A new random picture every frame, bit-exact without sound: full-range U and V through k_picture's 3-, 5- and
    7-tap low-pass, the saturating one among them, and through the pixel-rate raster's."""
    H = built
    quiet = H.mode_config(mode, **dict(kw, noaudio=True))
    o = orc.Oracle(quiet, rate, prate); al, aw = o.active_lines, o.active_width; o.close()
    rng = np.random.default_rng(43)
    frames = rng.integers(0, 1 << 24, size=(3, al, aw), dtype=np.uint32)
    nlines = 2 * quiet.lines + 20
    got, name = _run(H, kind, quiet, rate, prate, [nlines], frames)
    rows = {"composite": PS, "s_video": S_VIDEO}.get(kind, PIXELRATE)
    assert name == next(c[-1] for c in rows if (c[0], c[1]) == (mode, rate) and (kind != "pixelrate" or c[2] == prate))
    bad = np.flatnonzero(got != _want(kind, quiet, rate, prate, nlines, frames))
    assert bad.size == 0, f"{bad.size} values differ, first at line {bad[0] // (got.size // nlines)}"


@pytest.mark.parametrize("kind,mode,rate,prate,kw", [("pixelrate", "i", 1250000, 2000000, F), ("composite", "m", 4000000, 0, F),
                                                     ("s_video", "ntsc", 2000000, 0, S)])
def test_uneven_calls(built, kind, mode, rate, prate, kw):
    """A pixel-rate row with FM + NICAM at W = 80, a PS row with FM, and the single-warp S-Video PS row: calls of any
    size give the stream one call gives."""
    H = built
    conf = H.mode_config(mode, **kw)
    whole, name = _run(H, kind, conf, rate, prate, [1400])
    parts, name2 = _run(H, kind, conf, rate, prate, [1, 2, 311, 700, 7, 379])
    assert name == name2 and name.startswith(("k_line", "k_raster"))
    assert np.array_equal(whole, parts), f"{np.count_nonzero(whole != parts)} values differ"


def test_call_longer_than_the_raster_sub_batch(built):
    """PAL at 2 Msps from 13.5 Msps: the sub-batch is the raster context's, 16 MiB / (864 x 2) = 9 709 lines, not the
    65 536 of the 128-sample line. 10 000 lines in one device-resident call cross it, and equal the same lines rendered in
    calls that do not, and the oracle."""
    import torch
    H = built
    mode, rate, prate = "pal", 2000000, 13500000
    conf = H.mode_config(mode)
    n = 10000
    enc = H.Encoder(conf, rate, prate)
    enc.open_test_source()
    W, per = enc.width, 2 if conf.output_type == 0 else 1
    assert (W, enc.raster_width) == (128, 864)
    buf = torch.zeros(n * W * per, dtype=torch.int16, device="cuda")
    enc.render(n, buf.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    whole = buf.cpu().numpy()
    assert enc.line_kernel == TMA
    enc.close()
    parts, _ = PR._render(H, conf, rate, prate, [5000, 4000, 1000])
    assert np.array_equal(whole, parts), f"{np.count_nonzero(whole != parts)} values differ, first at line " \
        f"{np.flatnonzero(whole != parts)[0] // (per * W)}"
    bad = np.flatnonzero(whole != PR._oracle(conf, rate, prate, n))
    assert bad.size == 0, f"{bad.size} values differ from the oracle, first at line {bad[0] // (per * W)}"


@pytest.mark.parametrize("mode,rate,prate,kw,msg", [
    ("pal", 2000000, 484375, {}, "the pixel-rate raster's line width 31 is below the kernels' 32-sample limit"),
    ("secam", 4750000, 0, SF, "SECAM with the video filter needs the burst window to start 25 samples or more into the "
                              "line (it starts at 24)"),
], ids=["pal-2000000-from-484375", "secam-4750000-s_video-vfilter"])
def test_low_rate_path_refusals(built, capfd, mode, rate, prate, kw, msg):
    """The tables accept these; htv_init refuses them with the kernels' limit, before anything is launched."""
    H = built
    conf = H.mode_config(mode, **kw)
    H.Tables(conf, rate, prate).close()
    with pytest.raises(RuntimeError):
        H.Encoder(conf, rate, prate)
    assert msg in capfd.readouterr().err
