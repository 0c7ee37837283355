"""Every instantiation of the fused line kernel (k_line, htv_line.cuh) and of the SECAM raster (k_sec_raster) that the
host can select, at the line widths that select it, against the oracle.

The host picks one instantiation per encoder (htv_kernels.cu, htv_dev_render_lines) from
  VF    a video filter is on,               HQ    it has Q taps (VSB),
  FULL  128 divides W (no partial tile),    CSAT  the chroma low-pass needs saturation (sum of |taps| > 32768),
  MAXT  the CTA size 32 * ceil(W / 128) rounded up to 256, 320 or 384 threads,
  SRC   the SECAM form (k_sec_raster + chrominance chain + k_line<SRC=1>),
  SND / WC  PAL's VSB + FM + NICAM sound stages and W = 1024 compiled in (the 16 Msps form).
Each case states the W it exists for and the `line_kernel` string it must run, so that a change to the selection cannot
move a case onto another path unnoticed; test_tables_and_abi.py checks the same cases against the tables without a GPU
and that together they cover every class above.

Per case: with no sound the stream is bit-exact; with NICAM only (integer end to end) bit-exact; with the mode's sound
within +-1 LSB and >= 97 % exact in every 128-sample tile column of the blanking lines and of the picture lines, so
that an error confined to one tile (the last, partial one) cannot hide in the average."""
import contextlib
import os

import numpy as np
import pytest

import orc

pytestmark = pytest.mark.gpu


def kl(vf, hq, full, csat, maxt, src=0, snd=-1, wc=0):
    return f"k_line<VF={vf},HQ={hq},FULL={full},CSAT={csat},MAXT={maxt},SRC={src},SND={snd},WC={wc}>"


def sec(vf, hq, full, maxt):
    return f"k_sec_raster<FULL={full},MAXT={maxt}> + " + kl(vf, hq, full, 0, maxt, src=1)


F = dict(vfilter=True)
# (mode, rate, overrides, W, line_kernel); W % 128 is the last tile's width where it is not 0
MATRIX = [
    # 384 threads (W = 1281 .. 1536): PAL / NTSC from about 20.1 Msps, mono and SECAM up to 24 Msps
    ("i", 20250000, F, 1296, kl(1, 1, 0, 0, 384)),                  # last tile 16; NICAM on the generic path every line
    ("i", 20050000, F, 1283, kl(1, 1, 0, 1, 384)),                  # last tile 3, chroma taps sum to 32769
    ("i", 22500000, F, 1440, kl(1, 1, 0, 0, 384)),                  # 12 warps, 17 chroma taps
    ("i", 24000000, dict(vfilter=True, nocolour=True), 1536, kl(1, 1, 1, 0, 384)),   # the width limit
    ("m", 20250000, F, 1287, kl(1, 1, 0, 0, 384)),                  # last tile 7, 525 lines
    ("pal", 20250000, F, 1296, kl(1, 0, 0, 0, 384)),                # real low-pass
    ("ntsc", 20250000, {}, 1287, kl(0, 0, 0, 0, 384)),              # no filter, real output
    ("pal", 22000000, F, 1408, kl(1, 0, 1, 0, 384)),
    ("pal", 22000000, {}, 1408, kl(0, 0, 1, 0, 384)),
    ("pal", 20050000, F, 1283, kl(1, 0, 0, 1, 384)),
    ("pal", 20050000, {}, 1283, kl(0, 0, 0, 1, 384)),
    # 320 threads (W = 1025 .. 1280)
    ("i", 17734475, F, 1135, kl(1, 1, 0, 1, 320)),                  # 4 x the PAL subcarrier: taps sum to 32769
    ("pal", 17734475, {}, 1135, kl(0, 0, 0, 1, 320)),
    ("pal", 17734475, F, 1135, kl(1, 0, 0, 1, 320)),
    ("m", 18000000, F, 1144, kl(1, 1, 0, 0, 320)),                  # last tile 120
    ("ntsc", 18000000, {}, 1144, kl(0, 0, 0, 0, 320)),
    ("ntsc", 18000000, F, 1144, kl(1, 0, 0, 0, 320)),
    ("i", 20000000, F, 1280, kl(1, 1, 1, 0, 320)),
    ("pal", 20000000, {}, 1280, kl(0, 0, 1, 0, 320)),
    ("pal", 20000000, F, 1280, kl(1, 0, 1, 0, 320)),
    # 256 threads (W <= 1024)
    ("i", 10000000, F, 640, kl(1, 1, 1, 0, 256)),                   # 5 warps; NICAM symbols < 33 samples: generic path
    ("i", 15750000, F, 1008, kl(1, 1, 0, 1, 256)),                  # taps sum to 32769
    ("pal", 15750000, {}, 1008, kl(0, 0, 0, 1, 256)),
    ("pal", 15750000, F, 1008, kl(1, 0, 0, 1, 256)),
    ("m", 13500000, F, 858, kl(1, 1, 0, 0, 256)),
    ("ntsc", 13500000, {}, 858, kl(0, 0, 0, 0, 256)),
    ("ntsc", 13500000, F, 858, kl(1, 0, 0, 0, 256)),
    ("i", 16000000, dict(vfilter=True, nonicam=True), 1024, kl(1, 1, 1, 0, 256)),   # not the compiled-in sound form
    ("pal", 16000000, {}, 1024, kl(0, 0, 1, 0, 256)),
    ("pal", 16000000, F, 1024, kl(1, 0, 1, 0, 256)),
    # SECAM: k_sec_raster + chain + k_line<SRC=1>
    ("l", 20250000, F, 1296, sec(1, 1, 0, 384)),
    ("secam", 22500000, {}, 1440, sec(0, 0, 0, 384)),
    ("l", 24000000, F, 1536, sec(1, 1, 1, 384)),
    ("secam", 24000000, {}, 1536, sec(0, 0, 1, 384)),
    ("secam", 24000000, F, 1536, sec(1, 0, 1, 384)),
    ("secam", 20250000, F, 1296, sec(1, 0, 0, 384)),
    ("l", 20000000, F, 1280, sec(1, 1, 1, 320)),
    ("l", 18750000, F, 1200, sec(1, 1, 0, 320)),
    ("secam", 20000000, {}, 1280, sec(0, 0, 1, 320)),
    ("secam", 17500000, {}, 1120, sec(0, 0, 0, 320)),
    ("secam", 20000000, F, 1280, sec(1, 0, 1, 320)),
    ("secam", 17500000, F, 1120, sec(1, 0, 0, 320)),
    ("l", 16000000, F, 1024, sec(1, 1, 1, 256)),
    ("l", 13500000, F, 864, sec(1, 1, 0, 256)),
    ("secam", 16000000, {}, 1024, sec(0, 0, 1, 256)),
    ("secam", 13500000, {}, 864, sec(0, 0, 0, 256)),
    ("secam", 16000000, F, 1024, sec(1, 0, 1, 256)),
    ("secam", 13500000, F, 864, sec(1, 0, 0, 256)),
]
# the form with PAL's sound stages and W = 1024 compiled in, and what HTV_KL=general runs instead
FIXED = kl(1, 1, 1, 0, 256, snd=1 | 4 | 32, wc=1024)
GENERAL = kl(1, 1, 1, 0, 256)


def case_id(c):
    mode, rate, kw, W, _ = c
    return f"{mode}-{rate}-W{W}" + "".join(f"-{k}" for k, v in kw.items() if v)


@contextlib.contextmanager
def _env(**env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _render(H, conf, rate, pieces, frames=None, audio=None, audio_block=0, **env):
    """The CUDA path's stream over calls of `pieces` lines, and the line kernel it ran."""
    with _env(**env):
        enc = H.Encoder(conf, rate)
    if frames is None:
        enc.open_test_source()
    else:
        enc.set_source(frames, audio, audio_block=audio_block)
    got = np.concatenate([enc.render_host(n) for n in pieces])
    name = enc.line_kernel
    enc.close()
    return got, name


def _oracle(conf, rate, nlines, frames=None, audio=None):
    o = orc.Oracle(conf, rate)
    if frames is None:
        o.open_test_source()
    else:
        o.set_source(frames, audio)
    want = o.render(nlines)
    o.close()
    return want


def _lines(conf):
    return 340 if conf.lines == 625 else 290       # first field, its picture and the second field's vertical blanking


def _has(conf, what):
    level, carrier = {"fm": ("fm_mono_level", "fm_mono_carrier"), "am": ("am_audio_level", "am_mono_carrier"),
                      "nicam": ("nicam_level", "nicam_carrier")}[what]
    return getattr(conf, level) > 0 and getattr(conf, carrier) != 0


def _picture_lines(H, conf, rate, quiet):
    """Lines with picture content: the I samples over the middle half of the active width are not all equal."""
    g = H.Tables(conf, rate).get("geometry")
    W, al, aw = int(g[0]), int(g[2]), int(g[3])
    rows = quiet.reshape(-1, W, 2 if conf.output_type == 0 else 1)[:, al + aw // 4: al + 3 * aw // 4, 0]
    return rows.max(axis=1) != rows.min(axis=1)


def _check_sound(got, want, W, picture, what):
    """+-1 LSB, and >= 97 % of values exact in every 128-sample tile column of the blanking lines and of the
    picture lines; on failure name the worst column and the worst single (line, tile)."""
    d = np.abs(got.astype(np.int32) - want.astype(np.int32)).reshape(picture.size, W, -1)
    if d.max() > 1:
        ln, x, _ = np.unravel_index(np.argmax(d), d.shape)
        pytest.fail(f"{what}: |diff| {d.max()} at line {ln}, sample {x} (tile {x // 128}); "
                    f"{np.count_nonzero(d > 1)} values over 1")
    assert picture.any() and not picture.all(), "the window holds no blanking or no picture lines"
    worst = (2.0, None)
    for t in range(-(-W // 128)):
        exact = (d[:, 128 * t: 128 * t + 128] == 0).mean(axis=(1, 2))                 # per line
        for cls, m in (("blanking", ~picture), ("picture", picture)):
            worst = min(worst, (exact[m].mean(), (cls, t)))
    frac, (cls, t) = worst
    if frac < 0.97:
        exact = np.stack([(d[:, 128 * t: 128 * t + 128] == 0).mean(axis=(1, 2)) for t in range(-(-W // 128))], axis=1)
        ln, lt = np.unravel_index(np.argmin(exact), exact.shape)
        pytest.fail(f"{what}: only {frac:.4f} exact in tile {t} of the {cls} lines; worst (line, tile) = ({ln}, {lt}) "
                    f"with {exact[ln, lt]:.3f} exact")


@pytest.mark.parametrize("mode,rate,kw,W,kernel", MATRIX, ids=[case_id(c) for c in MATRIX])
def test_line_kernel_forms_against_the_oracle(built, mode, rate, kw, W, kernel):
    H = built
    conf = H.mode_config(mode, **kw)
    nlines = _lines(conf)
    quiet = H.mode_config(mode, noaudio=True, **kw)
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


@pytest.mark.parametrize("mode,rate", [("i", 20250000), ("l", 20250000)])
def test_wide_lines_random_pictures_loud_audio_and_uneven_calls(built, mode, rate):
    """At 384 threads with a partial last tile: random pictures (a new one every frame) bit-exact without sound and within
    +-1 LSB with full-scale noise audio; calls of any size give the stream one call gives."""
    H = built
    conf = H.mode_config(mode, vfilter=True)
    kernel = next(c[4] for c in MATRIX if c[:3] == (mode, rate, F))
    e = H.Encoder(conf, rate); al, aw = e.active_lines, e.active_width; e.close()
    rng = np.random.default_rng(29)
    frames = rng.integers(0, 1 << 24, size=(3, al, aw), dtype=np.uint32)
    audio = rng.integers(-32768, 32767, size=(40000, 2), dtype=np.int16)
    quiet = H.mode_config(mode, vfilter=True, noaudio=True)
    got, name = _render(H, quiet, rate, [900], frames, audio)
    assert name == kernel
    assert np.array_equal(got, _oracle(quiet, rate, 900, frames, audio))
    got, name = _render(H, conf, rate, [900], frames, audio)
    d = np.abs(got.astype(np.int32) - _oracle(conf, rate, 900, frames, audio).astype(np.int32))
    assert d.max() <= 1, f"max |diff| {d.max()}; {np.count_nonzero(d > 1)} values over 1"
    whole, _ = _render(H, conf, rate, [4000], frames, audio)
    parts, name = _render(H, conf, rate, [1, 2, 311, 1000, 7, 2679], frames, audio)
    assert name == kernel
    assert np.array_equal(whole, parts)


@pytest.mark.parametrize("mode", ["i", "b", "pal-d"])
def test_compiled_in_sound_form_equals_the_general_form(built, mode):
    """The instantiation with PAL's VSB + FM + NICAM stages and W = 1024 compiled in (16 Msps) against the general one
    (HTV_KL=general): bit-identical on the test card, on random pictures with full-scale noise audio, and over calls of
    uneven size."""
    H = built
    conf = H.mode_config(mode, vfilter=True)
    fixed, name = _render(H, conf, 16000000, [1300])
    assert name == FIXED
    general, name = _render(H, conf, 16000000, [1300], HTV_KL="general")
    assert name == GENERAL
    assert np.array_equal(fixed, general), f"{np.count_nonzero(fixed != general)} values differ"
    e = H.Encoder(conf, 16000000); al, aw = e.active_lines, e.active_width; e.close()
    rng = np.random.default_rng(31)
    frames = rng.integers(0, 1 << 24, size=(3, al, aw), dtype=np.uint32)
    audio = rng.integers(-32768, 32767, size=(40000, 2), dtype=np.int16)
    pieces = [1, 2, 311, 1000, 625, 3, 2058]
    fixed, name = _render(H, conf, 16000000, pieces, frames, audio)
    assert name == FIXED
    general, name = _render(H, conf, 16000000, [sum(pieces)], frames, audio, HTV_KL="general")
    assert name == GENERAL
    assert np.array_equal(fixed, general), f"{np.count_nonzero(fixed != general)} values differ"


def test_line_wider_than_the_kernels_is_refused(built, capfd):
    """W = 1542 (PAL-I at 24.1 Msps): the tables accept it, htv_init refuses it with the kernels' width limit."""
    H = built
    conf = H.mode_config("i", vfilter=True, nocolour=True)
    assert int(H.Tables(conf, 24100000).get("geometry")[0]) == 1542
    with pytest.raises(RuntimeError):
        H.Encoder(conf, 24100000)
    assert "line width 1542 exceeds the kernels' 1536-sample limit" in capfd.readouterr().err
