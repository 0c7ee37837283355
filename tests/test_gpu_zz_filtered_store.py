"""The filtered store (k_vf_rows, htv_line.cuh): the k_line forms with a video filter and a composite store load each
line's filter output instead of filtering it. Lines 2 .. N - 1 of a frame come from the store's row of their (picture,
phase); the lines whose 51-tap window leaves one frame's rows or meets a VBI overlay (vf_exception, htv_kernels.cu) are
filtered per call. At every changed form and the widths that select it:
  - bit-exact against the oracle without sound: overlays on lines 1, 2, N - 1 and N of every frame and on two
    consecutive lines, 40 samples clear of the line ends; a live source with a new picture every frame, in calls that
    start at stream line 0 (a 1-line call), mid-frame and on frame boundaries, with the descriptors ahead of the
    caller's stream and with HTV_AHEAD=0; picture slots reused while other phases of them are still shown; S-Video;
  - overlays that reach both line ends, so that the filter windows of the lines on either side take overlaid samples
    (the neighbour half of vf_exception): on lines 1 and N, on a consecutive pair and on a line alone, against the
    51-tap filter run here over the oracle's unfiltered composite stream. The stream is filtered as one sequence of
    samples, every line with its overlay, as the reference's filter stage is fed (video.c _vid_filter_process) and as
    the line kernel has always filtered it; the oracle's own filtered path adds line t + 1's overlay only after it has
    filtered line t, so it is checked against this model only where the overlays stay clear of the line ends;
  - the forms with the sound stages and the width compiled in (bench form, int16 and int8) against the general form,
    and the int8 and run-time-typed stores against the converted int16 stream."""
import numpy as np
import pytest

import orc
import sv_oracle
from test_composite_store import _frames_shown, _held_source, _pictures
from test_gpu_zz_sample_types import _convert, _env

pytestmark = pytest.mark.gpu

# (id, mode, rate, overrides, what the form is)
FORMS = [
    ("i-16M", "i", 16000000, {}, "HQ=1,FULL=1,CSAT=0,MAXT=256"),
    ("m-13M5-W858", "m", 13500000, {}, "HQ=1,FULL=0,CSAT=0,MAXT=256"),
    ("i-20M25-W1296", "i", 20250000, {}, "HQ=1,FULL=0,CSAT=0,MAXT=384"),
    ("i-17M73-csat", "i", 17734475, {}, "HQ=1,FULL=0,CSAT=1,MAXT=320"),
    ("pal-16M-lowpass", "pal", 16000000, {}, "HQ=0,FULL=1,CSAT=0,MAXT=256"),
    ("ntsc-13M5-lowpass-W858", "ntsc", 13500000, {}, "HQ=0,FULL=0,CSAT=0,MAXT=256"),
    ("ntsc-13M5-s-video", "ntsc", 13500000, dict(s_video=True), "HQ=0,FULL=0,CSAT=0,MAXT=256"),
    ("i-20M-W1280", "i", 20000000, {}, "HQ=1,FULL=1,CSAT=0,MAXT=320"),               # cfg5's form
    ("pal-20M-lowpass-W1280", "pal", 20000000, {}, "HQ=0,FULL=1,CSAT=0,MAXT=320"),
    ("pal-20M25-lowpass-W1296", "pal", 20250000, {}, "HQ=0,FULL=0,CSAT=0,MAXT=384"),
]
NO_SV = [f for f in FORMS if not f[3].get("s_video")]


def _conf(H, mode, kw):
    return H.mode_config(mode, vfilter=True, noaudio=True, **kw)


def _overlays(W, N, seed):
    """Lines 1, 2, N - 1, N and 150, 151: random adds and a replaced run, 40 samples clear of the line ends."""
    rng = np.random.default_rng(seed)
    m = 40
    out = []
    for k, line in enumerate((1, 2, N - 1, N, 150, 151)):
        add = np.zeros(W, dtype=np.int16)
        add[m:W - m] = rng.integers(-6000, 6000, size=W - 2 * m, dtype=np.int16)
        rep = (m, m + 40, 3000) if k % 2 == 0 else (W - m - 40, W - m, -2000)
        out.append((line, add, rep))
    return out


def _edge_overlays(W, N, seed):
    """Lines 1 and N, the pair 150 / 151 and line 300 alone (299 and 301 have none): random adds over the whole line
    and replaced runs at either line end, inside the 25 samples the filter reaches into a neighbouring line."""
    rng = np.random.default_rng(seed)
    out = []
    for k, line in enumerate((1, 150, 151, 300, N)):
        add = rng.integers(-6000, 6000, size=W, dtype=np.int16)
        rep = (0, 12, 2500) if k % 2 == 0 else (W - 12, W, -2500)
        out.append((line, add, rep))
    return out


def _stream_filter(H, conf, rate, comp, n, W):
    """The video filter over the composite stream comp (n + 1 lines, zeros before the stream): I and Q of lines
    0 .. n - 1 as the reference's fir_int16 computes them (int32 sums with wrap-around, >> 15, saturated)."""
    t = H.Tables(conf, rate)
    ti = t.get("vsb_itaps").astype(np.int64)
    tq = t.get("vsb_qtaps")
    t.close()
    h = len(ti) // 2
    sp = np.concatenate([np.zeros(h, np.int64), comp.astype(np.int64)])
    win = np.lib.stride_tricks.sliding_window_view(sp, len(ti))

    def fir(taps):
        out = np.empty(n * W, np.int64)
        for a in range(0, n * W, 64 * W):
            b = min(a + 64 * W, n * W)
            out[a:b] = win[a:b] @ taps
        out = (out + (1 << 31)) % (1 << 32) - (1 << 31)
        return np.clip(out >> 15, -32768, 32767).astype(np.int16)
    return fir(ti), (fir(tq.astype(np.int64)) if tq is not None else None)


def _oracle_stream(H, conf, rate, frames, n, W, ov):
    """The oracle's composite stream without the video filter (each line with its overlay), filtered here."""
    plain = conf.copy()
    plain.vfilter = 0
    o = orc.Oracle(plain, rate)
    o.set_source(frames, None)
    for line, add, rep in ov:
        o.add_vbi_line(line, add, rep)
    raw = o.render(n + 1)
    o.close()
    comp = raw[::raw.size // ((n + 1) * W)]
    return _stream_filter(H, conf, rate, comp, n, W)


def _render(H, conf, rate, pictures, hold, pieces, ov, ahead="1", sample_type="int16"):
    with _env(HTV_AHEAD=ahead):
        enc = H.Encoder(conf, rate)
    _held_source(H, enc, pictures, hold)
    if ov:
        enc.set_vbi_lines(ov)
    if sample_type != "int16":
        enc.set_sample_type(sample_type)
    got = np.concatenate([enc.render_host(n) for n in pieces])
    name = enc.line_kernel
    enc.close()
    return got, name


def _oracle(conf, rate, frames, n, ov):
    if conf.s_video:
        return sv_oracle.render(conf, rate, n, source=(frames, None))
    o = orc.Oracle(conf, rate)
    o.set_source(frames, None)
    for line, add, rep in ov:
        o.add_vbi_line(line, add, rep)
    want = o.render(n)
    o.close()
    return want


@pytest.mark.parametrize("ahead", ["1", "0"])
@pytest.mark.parametrize("form", FORMS, ids=[f[0] for f in FORMS])
def test_overlays_and_frame_edges(built, form, ahead):
    H = built
    name, mode, rate, kw, what = form
    conf = _conf(H, mode, kw)
    N = conf.lines
    pictures = _pictures(H, conf, rate, 5, 61)
    enc = H.Encoder(conf, rate)
    W = enc.width
    enc.close()
    ov = [] if conf.s_video else _overlays(W, N, 3)
    pieces = [1, N // 2 - 1, N - N // 2, N, N + 7, 2 * N - 7]         # 5 frames
    got, kernel = _render(H, conf, rate, pictures, 1, pieces, ov, ahead)
    assert kernel.startswith("k_line<VF=1," + what), kernel
    n = sum(pieces)
    want = _oracle(conf, rate, _frames_shown(pictures, 1, n // N + 1), n, ov)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{name} HTV_AHEAD={ahead}: {bad.size} of {got.size} values differ, first at line {int(bad[0]) // (got.size // n)}"


def test_slots_reused(built):
    """20 new pictures, one a frame, in calls of 7 frames + 3 lines: the 16 slots are reused while the store still holds
    other phases of their previous pictures."""
    H = built
    conf = _conf(H, "i", {})
    N = conf.lines
    pictures = _pictures(H, conf, 16000000, 20, 67)
    pieces = [7 * N + 3, 7 * N + 3, 6 * N - 6]
    ov = _overlays(1024, N, 5)
    got, _ = _render(H, conf, 16000000, pictures, 1, pieces, ov)
    n = sum(pieces)
    want = _oracle(conf, 16000000, _frames_shown(pictures, 1, n // N + 1), n, ov)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} of {got.size} values differ, first at line {int(bad[0]) // (got.size // n)}"


TYPED = [("i-16M", "int8"), ("i-16M", "float"), ("m-13M5-W858", "int8"), ("i-20M-W1280", "uint16"),
         ("pal-20M25-lowpass-W1296", "float")]


@pytest.mark.parametrize("form_id,sample_type", TYPED, ids=[f"{f}-{t}" for f, t in TYPED])
def test_typed_stores(built, form_id, sample_type):
    """With overlays reaching the line ends: the typed stores are the conversion of the int16 stream."""
    H = built
    _, mode, rate, kw, what = next(f for f in FORMS if f[0] == form_id)
    conf = _conf(H, mode, kw)
    N = conf.lines
    pictures = _pictures(H, conf, rate, 3, 71)
    enc = H.Encoder(conf, rate)
    W = enc.width
    enc.close()
    pieces = [N // 3, N, N + 5]
    ov = _edge_overlays(W, N, 7)
    ref, _ = _render(H, conf, rate, pictures, 1, pieces, ov)
    got, kernel = _render(H, conf, rate, pictures, 1, pieces, ov, sample_type=sample_type)
    assert kernel.startswith("k_line<VF=1," + what) and f"ST=-1:{sample_type}" in kernel, kernel
    assert got.tobytes() == _convert(H, ref, sample_type)


def _interleave(i, q, per):
    if per == 1:
        return i
    return np.stack([i, q if q is not None else np.zeros_like(i)], axis=1).ravel()


@pytest.mark.parametrize("form", NO_SV, ids=[f[0] for f in NO_SV])
def test_overlays_reaching_the_line_ends(built, form):
    """Against the filter over the oracle's unfiltered stream, in one call and in calls that start on and right behind
    overlay lines and end right before them; first the model itself against the oracle's filtered path where the
    overlays stay clear of the line ends. No call ends on the last line of a frame: the host pulls a frame's overlays
    with its picture, so such a call's last line does not see the next frame's line-1 overlay (as before the filtered
    store)."""
    H = built
    name, mode, rate, kw, what = form
    conf = _conf(H, mode, kw)
    N = conf.lines
    pictures = _pictures(H, conf, rate, 4, 79)
    enc = H.Encoder(conf, rate)
    W = enc.width
    enc.close()
    n = 3 * N - 1
    frames = _frames_shown(pictures, 1, 4)
    clear = _overlays(W, N, 3)
    want = _oracle(conf, rate, frames, n, clear)
    per = want.size // (n * W)
    assert np.array_equal(_interleave(*_oracle_stream(H, conf, rate, frames, n, W, clear), per), want), name
    ov = _edge_overlays(W, N, 13)
    want = _interleave(*_oracle_stream(H, conf, rate, frames, n, W, ov), per)
    short = [1, 148, 1, 1, 148, 1, N - 298, N - 1, 3]               # ends at lines 1, 149 .. 151, 299, 300, N + 2, ...
    short.append(n - sum(short))
    for pieces, ahead in (([n], "1"), (short, "1"), (short, "0")):
        got, kernel = _render(H, conf, rate, pictures, 1, pieces, ov, ahead)
        assert kernel.startswith("k_line<VF=1," + what), kernel
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (f"{name} calls {pieces} HTV_AHEAD={ahead}: {bad.size} of {got.size} values differ, first "
                               f"at line {int(bad[0]) // (W * per)} sample {int(bad[0]) % (W * per) // per}")


def test_compiled_in_forms(built):
    """PAL-I at 16 Msps with FM and NICAM and overlays reaching the line ends: the forms with the sound stages and the
    width compiled in (int16, int8) equal the general form, and int8 is the conversion of int16."""
    H = built
    conf = H.mode_config("i", vfilter=True)
    N = conf.lines
    pictures = _pictures(H, conf, 16000000, 3, 83)
    ov = _edge_overlays(1024, N, 17)
    pieces = [N // 3, N, N + 5]
    fixed = "k_line<VF=1,HQ=1,FULL=1,CSAT=0,MAXT=256,SRC=0,SND=37,WC=1024"
    a, name = _render(H, conf, 16000000, pictures, 1, pieces, ov)
    assert name == fixed + ">", name
    with _env(HTV_KL="general"):
        b, name = _render(H, conf, 16000000, pictures, 1, pieces, ov)
    assert name.startswith("k_line<VF=1,HQ=1,FULL=1,CSAT=0,MAXT=256,SRC=0,SND=-1"), name
    assert np.array_equal(a, b)
    c, name = _render(H, conf, 16000000, pictures, 1, pieces, ov, sample_type="int8")
    assert name == fixed + ",ST=int8>", name
    assert c.tobytes() == _convert(H, a, "int8")
