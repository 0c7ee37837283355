"""The encoder below 10 Msps, on the device, against the oracle: every kernel form that only this band reaches.

Below 10 Msps the chroma low-pass has 7, 5, 3 and finally 1 tap, and the kernel selection changes with it:
  - k_compose's low-pass (chroma_lp4 / chroma_fir4<7|5|3>) fills the composite store k_line reads: every colour row
    here has P = 4 (PAL) or P = 2 (NTSC at multiples of 2.25 MHz), and at 7 Msps the taps sum to 32770 (CSAT). The
    encoders without a composite store (P = 0), where k_picture's low-pass feeds k_line, are test_gpu_zz_low_rate_paths.py's;
  - at W <= 128 k_line's CTA is a single warp, whose lanes fill both halos of a row, and W = 96 is one partial tile;
  - at 1 tap (1.25 Msps and below for PAL and NTSC) the split modulators run behind k_raster with chroma_fir4<1>:
    k_mod_tma (4 | W), k_mod_mma (pitched planes with the video filter), k_mod (NTSC W = 79);
  - SECAM keeps k_sec_raster + chain + k_line<SRC=1> down to W = 128.
The smallest line the kernels hold is 32 samples (40 for FM video), FM / AM sound needs 1.024 Msps, and SECAM takes the
video filter from 5 Msps, where the burst window starts 25 samples into the line (htv_kernels.cu plan_kernels): the
rows at W = 32 and SECAM-L at 5 Msps render at those limits, the refusals below them are tested without rendering.

Each row states the W it exists for and the `line_kernel` string it must run, and is checked as the line-width matrix
does (test_gpu_zz_line_widths.py): bit-exact without sound, bit-exact with NICAM only, and with the mode's sound within
+-1 LSB and >= 97 % exact in every tile column. test_oracle_vs_ref.py pins the oracle to the reference at every row.

SECAM between about 5 and 15 Msps: the reference's luma notch reads its line buffer's heap padding past the line's end,
where its subcarrier loop has added the burst window's last samples of earlier lines; the device, like the oracle by
default, reads zeros there (orc.Oracle ref_heap). Rows at 6, 8, 9 and 10 Msps, where the two differ, compare with the
default; test_oracle_vs_ref.py pins both to the reference's stream."""
import numpy as np
import pytest

from test_gpu_zz_line_widths import _check_sound, _has, _oracle, _picture_lines, _render, kl, sec

pytestmark = pytest.mark.gpu

F = dict(vfilter=True)
MONO = dict(vfilter=True, nocolour=True, noaudio=True)


def split(name, maxt=256, minb=4):
    return f"k_raster + {name}<{maxt},{minb}>"


# (mode, rate, overrides, W, line_kernel)
MATRIX = [
    # k_line at 3 chroma taps, one partial tile (W = 96) and one full tile (W = 128): a single-warp CTA
    ("pal", 1500000, {}, 96, kl(0, 0, 0, 0, 256)),
    ("pal", 1500000, F, 96, kl(1, 0, 0, 0, 256)),
    ("i", 1500000, F, 96, kl(1, 1, 0, 0, 256)),                     # FM + NICAM: the sound descriptor is wider than the CTA
    ("pal", 2000000, {}, 128, kl(0, 0, 1, 0, 256)),
    ("pal", 2000000, F, 128, kl(1, 0, 1, 0, 256)),
    ("i", 2000000, F, 128, kl(1, 1, 1, 0, 256)),
    # 3, 5 and 7 taps at two and more tiles; 7 Msps: the 7 taps sum to 32770
    ("i", 4000000, F, 256, kl(1, 1, 1, 0, 256)),
    ("i", 4500000, F, 288, kl(1, 1, 0, 0, 256)),                    # 5 taps
    ("pal", 6750000, F, 432, kl(1, 0, 0, 0, 256)),                  # 5 taps
    ("i", 8000000, F, 512, kl(1, 1, 1, 0, 256)),                    # 7 taps
    ("i", 7000000, F, 448, kl(1, 1, 0, 1, 256)),                    # CSAT
    # NTSC at multiples of 2.25 MHz
    ("ntsc", 2250000, {}, 143, kl(0, 0, 0, 0, 256)),
    ("m", 2250000, F, 143, kl(1, 1, 0, 0, 256)),
    ("ntsc", 4500000, {}, 286, kl(0, 0, 0, 0, 256)),
    ("m", 4500000, F, 286, kl(1, 1, 0, 0, 256)),
    ("ntsc", 6750000, {}, 429, kl(0, 0, 0, 0, 256)),
    ("m", 6750000, F, 429, kl(1, 1, 0, 0, 256)),
    # mono k_line below one tile, down to the 32-sample limit
    ("i", 1000000, MONO, 64, kl(1, 1, 0, 0, 256)),
    ("i", 500000, MONO, 32, kl(1, 1, 0, 0, 256)),
    # the split modulators at 1 chroma tap
    ("pal", 1250000, {}, 80, split("k_mod_tma")),
    ("pal", 1250000, F, 80, split("k_mod_mma")),                    # pitched planes: 128 does not divide 80
    ("ntsc", 1250000, {}, 79, split("k_mod")),                      # 4 does not divide 79
    ("i", 1250000, F, 80, split("k_mod_mma")),                      # FM + NICAM, 39 samples per audio sample
    # SECAM: k_sec_raster + chain + k_line<SRC=1>
    ("secam", 4000000, {}, 256, sec(0, 0, 1, 256)),
    ("secam", 6000000, {}, 384, sec(0, 0, 1, 256)),
    ("secam", 8000000, {}, 512, sec(0, 0, 1, 256)),
    ("secam", 9000000, {}, 576, sec(0, 0, 0, 256)),
    ("secam", 10000000, {}, 640, sec(0, 0, 1, 256)),
    ("l", 8000000, F, 512, sec(1, 1, 1, 256)),
    ("secam", 2000000, {}, 128, sec(0, 0, 1, 256)),                 # a single-warp CTA
    ("l", 5000000, F, 320, sec(1, 1, 0, 256)),                      # the lowest rate SECAM takes the video filter at
]


def case_id(c):
    mode, rate, kw, W, _ = c
    return f"{mode}-{rate}-W{W}" + "".join(f"-{k}" for k, v in kw.items() if v)


def _lines(conf):
    return 340 if conf.lines == 625 else 290       # first field, its picture and the second field's vertical blanking


@pytest.mark.parametrize("mode,rate,kw,W,kernel", MATRIX, ids=[case_id(c) for c in MATRIX])
def test_low_rate_forms_against_the_oracle(built, mode, rate, kw, W, kernel):
    H = built
    conf = H.mode_config(mode, **kw)
    nlines = _lines(conf)
    quiet = H.mode_config(mode, **dict(kw, noaudio=True))
    got, name = _render(H, quiet, rate, [nlines])
    assert name == kernel, f"{mode} {rate} ran {name}, the case exists for {kernel}"
    want = _oracle(quiet, rate, nlines)
    assert got.size == nlines * W * (2 if conf.output_type == 0 else 1)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"no sound: {bad.size} values differ, first at line {bad[0] // (got.size // nlines)}"
    if _has(conf, "nicam"):
        nic = H.mode_config(mode, **kw)
        nic.fm_mono_level = nic.fm_mono_carrier = nic.am_audio_level = nic.am_mono_carrier = 0.0
        got, name = _render(H, nic, rate, [nlines])
        assert name == kernel
        bad = np.flatnonzero(got != _oracle(nic, rate, nlines))
        assert bad.size == 0, f"NICAM only: {bad.size} values differ, first at line {bad[0] // (got.size // nlines)}"
    if _has(conf, "fm") or _has(conf, "am") or _has(conf, "nicam"):
        got, name = _render(H, conf, rate, [nlines])
        assert name == kernel
        _check_sound(got, _oracle(conf, rate, nlines), W, _picture_lines(H, conf, rate, want), "with sound")


COLOUR_KLINE = [c for c in MATRIX if c[4].startswith("k_line") and not c[2].get("nocolour")]


@pytest.mark.parametrize("mode,rate,kw,W,kernel", COLOUR_KLINE, ids=[case_id(c) for c in COLOUR_KLINE])
def test_low_rate_random_pictures(built, mode, rate, kw, W, kernel):
    """A new random picture every frame, bit-exact without sound: k_compose's 3-, 5- and 7-tap low-pass over full-range
    U and V."""
    H = built
    quiet = H.mode_config(mode, **dict(kw, noaudio=True))
    e = H.Encoder(quiet, rate); al, aw = e.active_lines, e.active_width; e.close()
    rng = np.random.default_rng(37)
    frames = rng.integers(0, 1 << 24, size=(3, al, aw), dtype=np.uint32)
    nlines = 2 * quiet.lines + 20
    got, name = _render(H, quiet, rate, [nlines], frames, None)
    assert name == kernel
    want = _oracle(quiet, rate, nlines, frames, None)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} values differ, first at line {bad[0] // (got.size // nlines)}"


@pytest.mark.parametrize("mode,rate,kw", [("i", 1500000, F), ("i", 1250000, F)])
def test_low_rate_uneven_calls(built, mode, rate, kw):
    """A single-warp k_line row and a split row, both with FM + NICAM: calls of any size give the stream one call gives."""
    H = built
    conf = H.mode_config(mode, **kw)
    kernel = next(c[4] for c in MATRIX if c[:3] == (mode, rate, kw))
    whole, name = _render(H, conf, rate, [1400])
    assert name == kernel
    parts, name = _render(H, conf, rate, [1, 2, 311, 700, 7, 379])
    assert name == kernel
    assert np.array_equal(whole, parts), f"{np.count_nonzero(whole != parts)} values differ"


@pytest.mark.parametrize("mode,rate,kw,msg", [
    ("i", 480000, MONO, "line width 31 is below the kernels' 32-sample limit"),
    ("i", 1000000, F, "FM / AM sound at 1000000 Hz is below the kernels' 1.024 MHz limit"),
    ("pal-fm", 609375, dict(vfilter=True, noaudio=True), "line width 39 is below FM video's 40-sample limit"),
    ("l", 4750000, F, "SECAM with the video filter needs the burst window to start 25 samples or more into the line"),
])
def test_line_narrower_than_the_kernels_is_refused(built, capfd, mode, rate, kw, msg):
    """The tables accept these; htv_init refuses them with the kernels' limit, before anything is launched."""
    H = built
    conf = H.mode_config(mode, **kw)
    H.Tables(conf, rate).close()
    with pytest.raises(RuntimeError):
        H.Encoder(conf, rate)
    assert msg in capfd.readouterr().err
