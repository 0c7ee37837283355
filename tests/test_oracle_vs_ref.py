"""The oracle against the reference itself: bit-exact, incl. inputs and options the golden fixtures of
test_oracle_golden.py do not cover. What the UNMODIFIED reference (the fsphil/hacktv sources compiled in place
into oracle/_ref/ref_harness) emitted for each case is stored as a sha256 of its int16 stream in
tests/golden/golden_ref.json, and the two scan lines the WSS overlay is recovered from in golden_ref_wss.npz;
tests/golden/make_golden_ref.py runs the reference and writes both. No GPU and no reference tree needed."""
import functools
import hashlib
import json
import os

import numpy as np
import pytest

import orc

HERE = os.path.dirname(os.path.abspath(__file__))


@functools.cache
def golden_ref():
    with open(os.path.join(HERE, "golden", "golden_ref.json")) as f:
        return json.load(f)


@functools.cache
def golden_wss_lines():
    return dict(np.load(os.path.join(HERE, "golden", "golden_ref_wss.npz")))


CASES = [
    ("pal", 16000000, 700, False, ()),
    ("i", 16000000, 700, True, ()),
    ("i", 16000000, 700, True, ("--nonicam",)),
    ("i", 16000000, 700, True, ("--noaudio", "--nocolour")),
    ("m", 13500000, 600, True, ()),
    ("l", 16000000, 700, True, ()),
    ("l", 16000000, 700, False, ()),
    ("i", 20000000, 400, True, ()),
    ("secam", 16000000, 700, False, ()),
    ("ntsc", 13500000, 600, False, ()),
    ("b", 16000000, 400, True, ()),
    ("pal-m", 13500000, 400, True, ()),
    ("d", 16000000, 400, True, ()),
    ("i", 16000000, 700, True, ("--offset", "2000000")),
    ("i", 16000000, 400, True, ("--swap-iq",)),
    ("pal", 16000000, 400, True, ()),
    # FM video (SURVEY.md section 8f rank 2): the pre-emphasis table differs per sample rate
    ("pal-fm", 20000000, 700, True, ()),
    ("pal-fm", 20250000, 400, True, ()),
    ("pal-fm", 14000000, 400, True, ("--noaudio",)),
    ("pal-fm", 28000000, 300, True, ()),
    ("pal-fm", 20000000, 700, False, ()),
    ("ntsc-fm", 18000000, 600, True, ()),
    ("ntsc-fm", 20250000, 400, True, ()),
    ("secam-fm", 20250000, 400, True, ()),
    ("pal-fm", 20000000, 400, True, ("--offset", "-3000000", "--swap-iq")),
]


def _line_width_cases():
    """Every mode, rate and option set the line kernel is held at by test_gpu_zz_line_widths.py, with the mode's sound
    and the lines it renders: the oracle those tests compare with is the reference there too."""
    from test_gpu_zz_line_widths import MATRIX
    out = []
    for mode, rate, kw, _, _ in MATRIX:
        extra = tuple(f"--{k}" for k in ("nocolour", "nonicam") if kw.get(k))
        case = (mode, rate, 290 if mode in ("m", "ntsc") else 340, bool(kw.get("vfilter")), extra)
        if case not in CASES and case not in out:
            out.append(case)
    return out


def _mode_matrix_cases():
    """Every row of the device's mode matrix (test_gpu_zz_modes.py), with the mode's sound and the lines it renders."""
    from test_gpu_zz_modes import MATRIX
    out = []
    for mode, rate, kw, _, _ in MATRIX:
        case = (mode, rate, 1100 if mode in ("ntsc-i", "pal60-i", "pal60", "525pal") else 1300, bool(kw.get("vfilter")), ())
        if case not in CASES and case not in out:
            out.append(case)
    return out


def _low_rate_cases():
    """Every row of the device's low-rate matrix (test_gpu_zz_low_rates.py), with the mode's sound and the lines it
    renders."""
    from test_gpu_zz_low_rates import MATRIX
    out = []
    for mode, rate, kw, _, _ in MATRIX:
        extra = tuple(f"--{k}" for k in ("nocolour", "nonicam", "noaudio") if kw.get(k))
        case = (mode, rate, 290 if mode in ("m", "ntsc") else 340, bool(kw.get("vfilter")), extra)
        if case not in CASES and case not in out:
            out.append(case)
    return out


def _low_rate_path_cases():
    """Every PS row of test_gpu_zz_low_rate_paths.py (k_line without a composite store below 10 Msps), with the mode's
    sound and the lines it renders."""
    from test_gpu_zz_low_rate_paths import PS
    out = []
    for mode, rate, kw, *_ in PS:
        case = (mode, rate, 290 if mode in ("m", "ntsc", "pal60", "pal60-i") else 340, bool(kw.get("vfilter")), ())
        if case not in CASES and case not in out:
            out.append(case)
    return out


CASES += _line_width_cases()
CASES += _mode_matrix_cases()
CASES += _low_rate_cases()
# SECAM with the video filter below 5 Msps: the filter's taps ahead reach the next line's burst window (the device
# refuses these; the oracle restates them)
CASES += [("l", 4000000, 340, True, ()), ("l", 2000000, 340, True, ())]
CASES += _low_rate_path_cases()


def ref_key(mode, rate, lines, *, skip=0, vfilter=False, extra=(), source="test", rawheap=False):
    """Names one reference run in golden_ref.json: its command line, with the input it was given instead of file
    names (`source`: the built-in test source, or which seeded random input / passthru stream)."""
    parts = [f"-m {mode} -s {rate} --skip {skip} --lines {lines}"] + (["--filter"] if vfilter else []) + list(extra)
    return " ".join(parts + [f"source={source}"] + (["rawheap"] if rawheap else []))


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def assert_reference(got, key):
    want = golden_ref()[key]
    assert got.size == want["size"], (got.size, want["size"])
    assert digest(got) == want["sha256"], f"the oracle's stream differs from the reference's ({key})"


def passthru_stream(width, ext_lines, seed=11, tail=None):
    """The external int16 IQ stream fed to --passthru (tail: complex samples past the last whole line)."""
    rng = np.random.default_rng(seed)
    return rng.integers(-32768, 32767, size=(ext_lines * width + (width // 3 if tail is None else tail), 2), dtype=np.int16)


def random_source(seed, active_lines, active_width):
    """Two random pictures and 30 000 random stereo sound samples (the reference reads the sound in blocks of 4000)."""
    rng = np.random.default_rng(seed)
    frames = rng.integers(0, 1 << 24, size=(2, active_lines, active_width), dtype=np.uint32)
    audio = rng.integers(-32768, 32767, size=(30000, 2), dtype=np.int16)
    return frames, audio


def programme_source(seed, active_lines, active_width):
    """Three random pictures and 2 711 stereo sound samples (an odd number, so that the loop's wrap falls inside an
    audio block) that reach the edges of the input range within the first 2 220, about 1 090 lines:
       0 ..  200  silence
     200 ..  900  uniform noise over the whole range, +32767 and -32768 included
     900 .. 1320  a full-scale square wave of period 4 .. 8 on both channels: through pre-emphasis it drives the FM
                  limiter hard
    1320 .. 1720  L = 2k + 1, R = -(2k + 2): L + R = -1, where the mono mix truncates toward zero
    1720 .. 1970  DC at -32768, then to 2 220 at +32767; after that noise again up to the wrap."""
    rng = np.random.default_rng(seed)
    frames = rng.integers(0, 1 << 24, size=(3, active_lines, active_width), dtype=np.uint32)
    audio = np.zeros((2711, 2), dtype=np.int16)
    audio[200:900] = rng.integers(-32768, 32767, size=(700, 2), endpoint=True)
    audio[200], audio[201] = (32767, -32768), (-32768, 32767)
    square = np.concatenate([np.where(np.arange(p) < p // 2, 32767, -32768) for p in np.tile(np.arange(4, 9), 14)])
    audio[900:1320] = square[:, None]
    k = rng.integers(-16384, 16383, size=400, endpoint=True)
    audio[1320:1720, 0], audio[1320:1720, 1] = 2 * k + 1, -(2 * k + 2)
    audio[1720:1970] = -32768
    audio[1970:2220] = 32767
    audio[2220:] = rng.integers(-32768, 32767, size=(491, 2), endpoint=True)
    return frames, audio


def _conf(H, mode, filt, extra):
    kw = dict(vfilter=filt)
    it = iter(extra)
    for e in it:
        if e == "--nonicam": kw["nonicam"] = True
        elif e == "--noaudio": kw["noaudio"] = True
        elif e == "--nocolour": kw["nocolour"] = True
        elif e == "--swap-iq": kw["swap_iq"] = True
        elif e == "--offset": kw["offset"] = int(next(it))
        elif e == "--volume": kw["volume"] = float(next(it))
    return H.mode_config(mode, **kw)


# SECAM cases whose reference stream depends on the heap padding past the line that the reference's luma notch reads
# (DESIGN.md section 2): there the oracle's default, which reads zeros as the CUDA path does, differs from it
HEAP_CASES = {("secam", 6000000), ("secam", 8000000), ("secam", 9000000), ("secam", 10000000), ("l", 8000000)}


@pytest.mark.parametrize("mode,rate,nlines,filt,extra", CASES)
def test_oracle_equals_reference(built, mode, rate, nlines, filt, extra):
    """The oracle's default is the reference's stream everywhere but HEAP_CASES, where it differs; with ref_heap (SECAM
    only) it is the reference's stream in every case."""
    conf = _conf(built, mode, filt, extra)
    key = ref_key(mode, rate, nlines, vfilter=filt, extra=extra)
    for ref_heap in (False, True) if conf.colour_mode == 3 else (False,):
        o = orc.Oracle(conf, rate, ref_heap=ref_heap)
        o.open_test_source()
        got = o.render(nlines)
        o.close()
        if ref_heap or (mode, rate) not in HEAP_CASES:
            assert_reference(got, key)
        else:
            assert digest(got) != golden_ref()[key]["sha256"], "the default no longer differs: is the case in HEAP_CASES?"


PASSTHRU_CASES = [
    ("pal", 16000000, False, (), 40),                    # real output: I only reaches the sink
    ("i", 16000000, True, ("--offset", "1250000"), 40),  # the README's two-channel recipe (second stage)
    ("l", 16000000, True, (), 40),
    ("i", 16000000, False, ("--noaudio",), 40),
    ("m", 13500000, True, (), 12),                       # external stream ends early, mid-line
]


def _post_stage_cases():
    """Every row of the device's post-modulation matrix (test_gpu_zz_post_stage.py), without sound as it renders them:
    (mode, rate, lines, vfilter, extra) of --offset f --swap-iq over its offset window on the complex rows, and (mode,
    rate, vfilter, extra, external lines) of --passthru over its calls, the external stream cut off mid-line inside them."""
    import test_gpu_zz_post_stage as P
    offset, passthru = [], []
    for i, (mode, rate, kw, W, _, _, cpx) in enumerate(P.ROWS):
        filt = bool(kw.get("vfilter"))
        quiet = ("--noaudio",) + (("--nocolour",) if kw.get("nocolour") else ())
        if cpx:
            offset.append((mode, rate, sum(P._offset_calls(W, kw)), filt,
                           quiet + ("--offset", str(P._offset(rate, i)), "--swap-iq")))
        passthru.append((mode, rate, filt, quiet, P._delay(kw) + P.PT_LINES))
    return offset, passthru


POST_OFFSET, POST_PASSTHRU = _post_stage_cases()
POST_LINES = 114                            # sum(test_gpu_zz_post_stage.PT_CALLS)


@pytest.mark.parametrize("mode,rate,nlines,filt,extra", POST_OFFSET)
def test_offset_and_swap_at_the_post_stage_rows(built, mode, rate, nlines, filt, extra):
    """The offset mixer's start-up window and the NCO after it, behind the IQ swap, at every complex row's width (in
    HEAP_CASES with the reference's SECAM heap padding, ref_heap)"""
    o = orc.Oracle(_conf(built, mode, filt, extra), rate, ref_heap=(mode, rate) in HEAP_CASES)
    o.open_test_source()
    got = o.render(nlines)
    o.close()
    assert_reference(got, ref_key(mode, rate, nlines, vfilter=filt, extra=extra))


@pytest.mark.parametrize("mode,rate,filt,extra,ext_lines", POST_PASSTHRU)
def test_passthru_at_the_post_stage_rows(built, mode, rate, filt, extra, ext_lines):
    import test_gpu_zz_post_stage as P
    assert sum(P.PT_CALLS) == POST_LINES
    o = orc.Oracle(_conf(built, mode, filt, extra), rate, ref_heap=(mode, rate) in HEAP_CASES)
    ext = passthru_stream(o.width, ext_lines)
    o.open_test_source()
    o.set_passthru(ext)
    got = o.render(POST_LINES)
    o.close()
    assert_reference(got, ref_key(mode, rate, POST_LINES, vfilter=filt, extra=tuple(extra) + ("--passthru",),
                                  source=f"passthru{ext_lines}"))


@pytest.mark.parametrize("mode,rate,filt,extra,ext_lines", PASSTHRU_CASES)
def test_passthru_alignment(built, mode, rate, filt, extra, ext_lines):
    """ref _vid_passthru_process video.c:3517-3541: line alignment (the external stream's first
    line is spent on the filter's fill line), int16 wrap, whole lines only at its end."""
    o = orc.Oracle(_conf(built, mode, filt, extra), rate)
    ext = passthru_stream(o.width, ext_lines)
    o.open_test_source()
    o.set_passthru(ext)
    got = o.render(30)
    o.close()
    assert_reference(got, ref_key(mode, rate, 30, vfilter=filt, extra=tuple(extra) + ("--passthru",), source=f"passthru{ext_lines}"))
    assert digest(got) != golden_ref()[ref_key(mode, rate, 30, vfilter=filt, extra=extra)]["sha256"]


def wss_overlay(built, mode, rate):
    """What the reference's WSS stage (--wss 16:9) does to line 23 (wss.c:154-193): part of the line set to black,
    then the bit waveform added. Recovered from the reference's own line 23 (I channel), unfiltered, no sound, no
    colour (the SECAM stage runs after WSS and would filter it), without and with --wss."""
    conf = built.mode_config(mode, noaudio=True)
    t = built.Tables(conf, rate)
    half = int(t.get("geometry")[1])
    black = int(t.get("levels")[1])
    t.close()
    plain = golden_wss_lines()[f"{mode}_{rate}_plain"].astype(np.int32)
    with_wss = golden_wss_lines()[f"{mode}_{rate}_wss"].astype(np.int32)
    blank_to = int(round(rate * 42.5e-6))
    base = plain.copy()
    base[half:blank_to] = black
    return (with_wss - base).astype(np.int16), (half, blank_to, black)


@pytest.mark.parametrize("mode,rate,filt,extra", [("i", 16000000, True, ()), ("pal", 16000000, False, ()),
                                                  ("l", 16000000, True, ()), ("secam", 16000000, False, ())])
def test_vbi_overlay_is_where_the_reference_puts_wss(built, mode, rate, filt, extra):
    """The overlay hook (after the raster, before SECAM / filter / sound) carries the reference's own WSS
    waveform to exactly the reference's --wss output, in modes other than the one it was recovered from."""
    add, rep = wss_overlay(built, mode, rate)
    assert np.count_nonzero(add) > 100
    o = orc.Oracle(_conf(built, mode, filt, extra), rate)
    o.open_test_source()
    o.add_vbi_line(23, add, rep)
    got = o.render(700)
    o.close()
    assert_reference(got, ref_key(mode, rate, 700, vfilter=filt, extra=tuple(extra) + ("--wss", "16:9")))


def test_oracle_equals_reference_on_random_input(built):
    conf = built.mode_config("i", vfilter=True)
    o = orc.Oracle(conf, 16000000)
    frames, audio = random_source(7, o.active_lines, o.active_width)
    o.set_source(frames, audio)
    got = o.render(1400)
    o.close()
    assert_reference(got, ref_key("i", 16000000, 1400, vfilter=True, source="random7"))


# low rates the random and the programme source are pinned at: 3 chroma taps on k_line, and 1 Msps (64 samples a
# line, a 32 kHz audio sample every 31.25 samples: the device refuses sound there, the oracle restates it)
LOW_RATE_SOURCES = [("i", 2000000, 700), ("i", 1000000, 700)]


@pytest.mark.parametrize("mode,rate,nlines", LOW_RATE_SOURCES)
def test_oracle_equals_reference_on_random_input_at_low_rates(built, mode, rate, nlines):
    o = orc.Oracle(built.mode_config(mode, vfilter=True), rate)
    frames, audio = random_source(13, o.active_lines, o.active_width)
    o.set_source(frames, audio)
    got = o.render(nlines)
    o.close()
    assert_reference(got, ref_key(mode, rate, nlines, vfilter=True, source="random13"))


@pytest.mark.parametrize("mode,rate,nlines", LOW_RATE_SOURCES)
def test_oracle_equals_reference_on_programme_audio_at_low_rates(built, mode, rate, nlines):
    o = orc.Oracle(built.mode_config(mode, vfilter=True), rate)
    o.set_source(*programme_source(17, o.active_lines, o.active_width))
    got = o.render(nlines)
    o.close()
    assert_reference(got, ref_key(mode, rate, nlines, vfilter=True, source="programme17"))


def test_secam_notch_reads_the_reference_heap_padding(built):
    """SECAM at 6 Msps: the reference's luma notch reads the padding past its line buffer, which holds what the
    subcarrier loop of earlier lines added past the burst window's end there. ref_heap restates that (the reference's
    stream); without it the notch reads zeros, as the CUDA path does, and the two streams differ only in the last 25
    samples of the picture."""
    conf = built.mode_config("secam")
    outs = []
    for ref_heap in (True, False):
        o = orc.Oracle(conf, 6000000, ref_heap=ref_heap)
        o.open_test_source()
        outs.append(o.render(340))
        aw, W = o.active_width, o.width
        o.close()
    assert_reference(outs[0], ref_key("secam", 6000000, 340))
    d = (outs[0] != outs[1]).reshape(340, W)
    assert d.any()
    x = np.flatnonzero(d.any(axis=0))
    t = built.Tables(conf, 6000000)
    end = int(t.get("geometry")[2]) + aw                      # the picture's end: 62 + 312
    t.close()
    assert x.min() >= end - 25 and x.max() < end, x


def programme_cases():
    """The programme-audio runs of the device (test_gpu_zz_modes.py): (mode, rate, vfilter, extra options, lines,
    audio block, seed)."""
    from test_gpu_zz_modes import PROGRAMME, PROGRAMME_BLOCK, PROGRAMME_LINES, PROGRAMME_SEED
    out = []
    for mode, rate, kw in PROGRAMME:
        extra = ("--volume", f"{kw['volume']:g}") if "volume" in kw else ()
        out.append((mode, rate, bool(kw.get("vfilter")), extra, PROGRAMME_LINES, PROGRAMME_BLOCK, PROGRAMME_SEED))
    return out


@pytest.mark.parametrize("mode,rate,filt,extra,nlines,block,seed", programme_cases())
def test_oracle_equals_reference_on_programme_audio(built, mode, rate, filt, extra, nlines, block, seed):
    """programme_source read in blocks of `block` pairs by the reference; the oracle takes it whole."""
    o = orc.Oracle(_conf(built, mode, filt, extra), rate)
    o.set_source(*programme_source(seed, o.active_lines, o.active_width))
    got = o.render(nlines)
    o.close()
    assert_reference(got, ref_key(mode, rate, nlines, vfilter=filt, extra=extra, source=f"programme{seed}"))


def test_unpatched_heap_differs_only_near_line_ends(built):
    """The stock allocator lets the chroma FIR read past its buffer (SURVEY.md §8c): the
    masked comparison with that build - everything further than 32 samples from a line boundary - is exact."""
    o = orc.Oracle(built.mode_config("i", vfilter=True), 16000000)
    o.open_test_source()
    got = o.render(700).reshape(700, 1024, 2)
    o.close()
    want = golden_ref()[ref_key("i", 16000000, 700, vfilter=True, rawheap=True)]
    assert digest(got[:, 32:-32]) == want["masked_32_sha256"]


# --pixelrate (SURVEY.md section 8f rank 4): raster at the pixel rate, the reference's polyphase resampler
# (video.c:3627-3651, fir.c:393-428) to the sample rate in front of the video filter. The oracle restates the
# rate pairs that keep the line width constant; the CUDA path takes them all except SECAM's and FM video's.
PIXELRATE_CASES = [
    ("pal", 16000000, 13500000, 700, False, ()),                 # 864 -> 1024 samples per line, I/D = 32/27
    ("i", 16000000, 13500000, 700, True, ()),                    # + VSB filter, FM + NICAM two lines ahead
    ("i", 16000000, 13500000, 400, False, ()),                   # resampler alone: one line ahead
    ("i", 16000000, 13500000, 400, True, ("--offset", "2000000")),
    ("i", 20000000, 13500000, 400, True, ()),                    # 40/27
    ("i", 13500000, 16000000, 400, True, ()),                    # resampling down, 27/32
    ("i", 16000000, 14000000, 300, True, ()),                    # 8/7
    ("m", 13500000, 9000000, 400, True, ()),                     # NTSC, 3/2
    ("l", 16000000, 13500000, 700, True, ()),                    # SECAM: the FIRs' reads past the line end find the blanking level
    ("l", 13500000, 16000000, 300, True, ()),
    ("secam", 16000000, 13500000, 400, False, ()),
    ("d", 20000000, 13500000, 300, True, ()),
]


def _pixelrate_matrix_cases():
    """Every mode, rate pair and option set the device's --pixelrate path is held at by test_gpu_zz_pixelrate.py, with the
    mode's sound and the lines it renders: the oracle those tests compare with is the reference there too."""
    from test_gpu_zz_pixelrate import MATRIX
    out = []
    for mode, rate, prate, kw, _, _, _ in MATRIX:
        extra = tuple(f"--{k}" for k in ("nocolour",) if kw.get(k))
        case = (mode, rate, prate, 290 if mode in ("m", "ntsc", "pal-m") else 340, bool(kw.get("vfilter")), extra)
        if case not in PIXELRATE_CASES and case not in out:
            out.append(case)
    return out


def _low_pixelrate_cases():
    """Every --pixelrate row of test_gpu_zz_low_rate_paths.py, with the mode's sound and the lines it renders, and PAL at
    2 Msps from 484 375 Hz: a 31-sample raster, which the oracle restates and the device refuses."""
    from test_gpu_zz_low_rate_paths import PIXELRATE
    out = []
    for mode, rate, prate, kw, *_ in PIXELRATE:
        case = (mode, rate, prate, 290 if mode in ("m", "ntsc") else 340, bool(kw.get("vfilter")), ())
        if case not in PIXELRATE_CASES and case not in out:
            out.append(case)
    return out + [("pal", 2000000, 484375, 340, False, ())]


PIXELRATE_CASES += _pixelrate_matrix_cases()
PIXELRATE_CASES += _low_pixelrate_cases()


@pytest.mark.parametrize("mode,rate,prate,nlines,filt,extra", PIXELRATE_CASES)
def test_pixelrate_resampler_equals_reference(built, mode, rate, prate, nlines, filt, extra):
    o = orc.Oracle(_conf(built, mode, filt, extra), rate, prate)
    o.open_test_source()
    got = o.render(nlines)
    o.close()
    assert_reference(got, ref_key(mode, rate, nlines, vfilter=filt, extra=tuple(extra) + ("--pixelrate", str(prate))))


def test_pixelrate_later_window_and_random_input(built):
    """A window two frames in (phase of the polyphase filter, NICAM frame counter) and random pictures + audio."""
    conf = built.mode_config("i", vfilter=True)
    o = orc.Oracle(conf, 16000000, 13500000)
    o.open_test_source()
    got = o.render(1700)[1400 * 2048:]
    o.close()
    assert_reference(got, ref_key("i", 16000000, 300, skip=1400, vfilter=True, extra=("--pixelrate", "13500000")))
    o = orc.Oracle(conf, 16000000, 13500000)
    frames, audio = random_source(5, o.active_lines, o.active_width)
    o.set_source(frames, audio)
    got = o.render(900)
    o.close()
    assert_reference(got, ref_key("i", 16000000, 900, vfilter=True, extra=("--pixelrate", "13500000"), source="random5"))


def test_pixelrate_with_passthru_and_wss(built):
    """Two fill lines in front of the stream (resampler + filter): the passthru stage spends two external
    lines on them; the VBI stages sit in front of the resampler."""
    conf = built.mode_config("i", vfilter=True)
    o = orc.Oracle(conf, 16000000, 13500000)
    ext = passthru_stream(o.width, 40, seed=3, tail=100)
    o.open_test_source()
    o.set_passthru(ext)
    got = o.render(30)
    o.close()
    assert_reference(got, ref_key("i", 16000000, 30, vfilter=True, extra=("--pixelrate", "13500000", "--passthru"), source="passthru40s3"))

    add, rep = wss_overlay(built, "pal", 13500000)               # the waveform at the pixel rate
    o = orc.Oracle(built.mode_config("pal"), 16000000, 13500000)
    o.open_test_source()
    o.add_vbi_line(23, add, rep)
    got = o.render(100)
    o.close()
    assert_reference(got, ref_key("pal", 16000000, 100, extra=("--pixelrate", "13500000", "--wss", "16:9")))


def test_pixelrate_pairs_the_oracle_does_not_restate(built):
    with pytest.raises(RuntimeError):
        orc.Oracle(built.mode_config("i", vfilter=True), 16000000, 13400000)    # line width would vary
    with pytest.raises(RuntimeError):
        orc.Oracle(built.mode_config("pal-fm", vfilter=True), 20000000, 13500000)
