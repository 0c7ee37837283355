"""Every colour-frame phase of the composite store (k_compose, htv_kernels.cu) at every fused-line-kernel form, and calls
that start on a frame boundary, against the oracle.

k_compose writes one finished row per (picture slot, phase f0 mod P) and k_line only loads it, so each colour line comes
from a row written at one of P phases: 4 for the PAL family, 2 for NTSC, 1 without colour (0: no composite store, the
PS forms). The device matrices render at most two frames and a few lines, which reaches phases 0 and 1 only. Here:
  - ROWS: every non-SECAM k_line row of the line-width, low-rate, mode and S-Video matrices, once per (mode, rate,
    overrides), with its P stated. A live source of 5 random full-range pictures, each up for 3 frames (3 is coprime with
    2 and 4, so a picture is converted at several phases, some of them in calls after the one that uploaded it), over
    2P + 2 frames (6 for P <= 1) in uneven calls: bit-exact without sound.
  - BOUNDARY: calls that start exactly on a frame boundary. A call rasterises lines L0 - 2 .. L0 - 1 again as the left
    neighbours of its first line; where L0 opens a frame they show the previous frame's picture, and on the progressive
    525-line raster the video filter reaches back into the last line's picture row from line 1. Whole-frame calls,
    through htv_render_host and htv_render, and one htv_render call of 9 new pictures that the host splits after 7.
  - The black slot at every phase (a source that ends), and the number of conversions: each (picture, phase) once.
Without a GPU: that the rows are what they are stated to be and together cover every form, and that the boundary rows'
line 1 depends on the previous frame's picture in the oracle exactly where stated, so that BOUNDARY is not vacuous."""
import numpy as np
import pytest

import orc
import sv_oracle
from test_composite_store import _frames_shown, _held_source, _pictures
from test_gpu_zz_line_widths import FIXED, GENERAL, MATRIX as WIDTHS
from test_gpu_zz_low_rates import MATRIX as LOW_RATES
from test_gpu_zz_modes import MATRIX as MODES
from test_gpu_zz_picture_store import _ended_source
from test_gpu_zz_s_video import MATRIX as S_VIDEO


def _rows():
    """(mode, rate, overrides, W, line_kernel without sound) of every non-SECAM k_line row of the four matrices, the
    first of each (mode, rate, overrides)."""
    rows, seen = [], set()
    for mode, rate, kw, W, kernel in WIDTHS + LOW_RATES + MODES + S_VIDEO:
        key = (mode, rate, tuple(sorted(kw.items())))
        if not kernel.startswith("k_line") or key in seen:       # SECAM (k_sec_raster) and the split modulators
            continue
        seen.add(key)
        rows.append((mode, rate, kw, W, GENERAL if kernel == FIXED else kernel))
    return rows


ROWS = _rows()

# P of each row by (mode, rate); rows without colour have P = 1
PHASES = {
    ("i", 20250000): 4, ("i", 20050000): 0, ("i", 22500000): 4, ("m", 20250000): 2, ("pal", 20250000): 4,
    ("ntsc", 20250000): 2, ("pal", 22000000): 4, ("pal", 20050000): 0, ("i", 17734475): 4, ("pal", 17734475): 4,
    ("m", 18000000): 2, ("ntsc", 18000000): 2, ("i", 20000000): 4, ("pal", 20000000): 4, ("i", 10000000): 4,
    ("i", 15750000): 4, ("pal", 15750000): 4, ("m", 13500000): 2, ("ntsc", 13500000): 2, ("i", 16000000): 4,
    ("pal", 16000000): 4,
    ("pal", 1500000): 4, ("i", 1500000): 4, ("pal", 2000000): 4, ("i", 2000000): 4, ("i", 4000000): 4,
    ("i", 4500000): 4, ("pal", 6750000): 4, ("i", 8000000): 4, ("i", 7000000): 4, ("ntsc", 2250000): 2,
    ("m", 2250000): 2, ("ntsc", 4500000): 2, ("m", 4500000): 2, ("ntsc", 6750000): 2, ("m", 6750000): 2,
    ("pal-d", 16000000): 4, ("pal-d", 20250000): 4, ("ntsc-i", 13500000): 2, ("ntsc-i", 18000000): 2,
    ("ntsc-i", 20250000): 2, ("pal60-i", 13500000): 0, ("pal60-i", 20250000): 0, ("pal60", 13500000): 0,
    ("pal60", 20250000): 0, ("525pal", 13500000): 4, ("525pal", 18000000): 4,
}


def _phases(mode, rate, kw):
    return 1 if kw.get("nocolour") else PHASES[(mode, rate)]


def case_id(c):
    mode, rate, kw, W, _ = c
    return f"{mode}-{rate}-W{W}" + "".join(f"-{k}" for k, v in kw.items() if v)


def _quiet(H, mode, kw):
    return H.mode_config(mode, **dict(kw, noaudio=True))


def _first_difference(got, want, lines, W, per, P):
    """None, or where got first differs from want: frame, its phase, line and sample."""
    bad = np.flatnonzero(got != want)
    if bad.size == 0:
        return None
    i = int(bad[0])
    L, x = divmod(i, W * per)
    f0 = L // lines
    phase = f"phase {f0 % P}" if P else "P = 0"
    part = f" ({'IQ'[x % 2]})" if per == 2 else ""
    return (f"{bad.size} of {got.size} values differ; first in frame {f0} ({phase}), line {L % lines + 1}, sample "
            f"{x // per}{part}: {got[i]} against {want[i]}")


def _oracle(conf, rate, frames, nlines, prate=0):
    if conf.s_video:
        return sv_oracle.render(conf, rate, nlines, source=(frames, None))
    o = orc.Oracle(conf, rate, prate)
    o.set_source(frames, None)
    want = o.render(nlines)
    o.close()
    return want


def _calls(L, P):
    """2P + 2 frames (6 for P <= 1): calls that start mid-frame, a 1-line call, a call that starts on a frame
    boundary, and one that starts mid-frame and spans more than P frames."""
    nframes = max(2 * P + 2, 6)
    a = L // 2
    pieces = [a, 1, L - a - 1, L // 3, (max(P, 1) + 1) * L]
    return pieces + [nframes * L - sum(pieces)]


# ---- without a GPU ------------------------------------------------------------------------------------------------

def test_rows_are_what_they_state(built):
    """Every row's W, P (comp_phases) and the C selection's kernel are what the row states; together the rows with a
    composite store (P > 0) cover VF / HQ / FULL 0 and 1, CSAT, MAXT 256 / 320 / 384, W <= 128, 4 not dividing W, the
    chroma low-pass at 3, 5, 7 and 17 taps, and S-Video."""
    from test_tables_and_abi import _plan_name
    H = built
    assert 60 <= len(ROWS) <= 90, len(ROWS)
    forms, narrow, odd4, taps, sv = set(), False, False, set(), False
    for mode, rate, kw, W, kernel in ROWS:
        t = H.Tables(_quiet(H, mode, kw), rate)
        w, P, ct = int(t.get("geometry")[0]), int(t.get("comp_phases")[0]), t.get("chroma_taps")
        t.close()
        what = (mode, rate, kw)
        assert w == W, (what, w)
        assert P == _phases(mode, rate, kw), (what, P)
        assert _plan_name(H, mode, rate, dict(kw, noaudio=True)) == kernel, what
        if P == 0:
            continue
        forms |= {f.strip() for f in kernel[len("k_line<"):-1].split(",")}
        narrow |= W <= 128
        odd4 |= W % 4 != 0
        if ct is not None and not kw.get("nocolour"):
            taps.add(len(ct))
        sv |= bool(kw.get("s_video"))
    want = {f"{k}={v}" for k in ("VF", "HQ", "FULL") for v in (0, 1)} | {"CSAT=1"} | \
        {f"MAXT={t}" for t in (256, 320, 384)} | {"SV"}
    assert not want - forms, sorted(want - forms)
    assert narrow and odd4 and sv, (narrow, odd4, sv)
    assert {3, 5, 7, 17} <= taps, sorted(taps)
    assert any(r[0] == "pal" and r[1] == 17734475 and _phases(*r[:3]) == 4 for r in ROWS)


# (id, mode, rate, pixel rate, overrides); all with the video filter, each at interlaced 0 and 1
BOUNDARY = [
    ("m-13.5M", "m", 13500000, 0, {}),                     # composite store, P = 2
    ("ntsc-13.5M", "ntsc", 13500000, 0, {}),               # baseband, P = 2
    ("pal-m-13.5M", "pal-m", 13500000, 0, {}),             # P = 4
    ("525pal-13.5M", "525pal", 13500000, 0, {}),           # P = 4
    ("m-2.25M", "m", 2250000, 0, {}),                      # W = 143
    ("m-16M", "m", 16000000, 0, {}),                       # P = 0: the converted picture store
    ("pal60-13.5M", "pal60", 13500000, 0, {}),             # P = 0
    ("m-1.25M", "m", 1250000, 0, {}),                      # k_raster + k_mod_mma
    ("ntsc-13.5M-s-video", "ntsc", 13500000, 0, dict(s_video=True)),
    ("m-13.5M-from-9M", "m", 13500000, 9000000, {}),       # --pixelrate: the raster context at 9 Msps
    ("i-16M", "i", 16000000, 0, {}),                       # the 625-line raster
]
# (id, interlaced) whose line 1 changes in the oracle when the previous frame's picture is black: the progressive
# 525-line raster's last line shows a source row, and the video filter reaches back into it (S-Video's on I). Not
# behind the 9 -> 13.5 Msps resampler, and not on the 625-line raster, whose last line has no source row.
DEPENDS = {("m-13.5M", 0), ("ntsc-13.5M", 0), ("pal-m-13.5M", 0), ("525pal-13.5M", 0), ("m-2.25M", 0), ("m-16M", 0),
           ("pal60-13.5M", 0), ("m-1.25M", 0), ("ntsc-13.5M-s-video", 0)}
BOUNDARY_CASES = [(b, il) for b in BOUNDARY for il in (0, 1)]
BOUNDARY_IDS = [f"{b[0]}-interlaced{il}" for b, il in BOUNDARY_CASES]


def _boundary_conf(H, mode, kw, interlaced):
    conf = H.mode_config(mode, vfilter=True, noaudio=True, **kw)
    conf.interlaced = interlaced
    return conf


def _source_geometry(conf, rate, prate):
    o = orc.Oracle(conf, rate, prate)
    g = (o.active_lines, o.active_width, o.width, 2 if o.complex or conf.s_video else 1)   # S-Video: I, Q pairs
    o.close()
    return g


@pytest.mark.parametrize("case,interlaced", BOUNDARY_CASES, ids=BOUNDARY_IDS)
def test_line_1_depends_on_the_previous_frame_where_stated(built, case, interlaced):
    """In the oracle, line 1 of frame 2 with frame 1's picture black against with it random."""
    name, mode, rate, prate, kw = case
    conf = _boundary_conf(built, mode, kw, interlaced)
    al, aw, W, per = _source_geometry(conf, rate, prate)
    pictures = np.random.default_rng(5).integers(0, 1 << 24, size=(3, al, aw), dtype=np.uint32)
    black = pictures.copy()
    black[0] = 0
    L = conf.lines
    a, b = (_oracle(conf, rate, p, L + 1, prate)[L * W * per:] for p in (pictures, black))
    changed = int(np.count_nonzero(a != b))
    assert (changed > 0) == ((name, interlaced) in DEPENDS), f"{changed} values of line 1 change"
    if interlaced == 0 and conf.lines == 525 and rate <= 13500000 and not prate and not kw:
        assert changed > 0


# ---- on the GPU ---------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("mode,rate,kw,W,kernel", ROWS, ids=[case_id(c) for c in ROWS])
def test_every_phase_of_every_form(built, mode, rate, kw, W, kernel):
    H = built
    conf = _quiet(H, mode, kw)
    P = _phases(mode, rate, kw)
    L = conf.lines
    pictures = _pictures(H, conf, rate, 5, 43)
    pieces = _calls(L, P)
    enc = H.Encoder(conf, rate)
    _held_source(H, enc, pictures, 3)
    got = np.concatenate([enc.render_host(n) for n in pieces])
    name = enc.line_kernel
    enc.close()
    assert name == kernel, f"{mode} {rate} ran {name}, the row exists for {kernel}"
    n = sum(pieces)
    want = _oracle(conf, rate, _frames_shown(pictures, 3, n // L + 1), n)
    diff = _first_difference(got, want, L, W, got.size // (n * W), P)
    assert diff is None, f"calls {pieces}: {diff}"


def _device_render(H, enc, pieces):
    """htv_render of each call into a buffer of its own (a whole frame is not a multiple of 16 bytes at every W)."""
    import torch
    st = torch.cuda.current_stream().cuda_stream
    bufs = []
    for n in pieces:
        buf = torch.zeros(n * enc.width * enc.bytes_per_sample // 2, dtype=torch.int16, device="cuda")
        enc.render(n, buf.data_ptr(), st)
        bufs.append(buf)
    torch.cuda.synchronize()
    return np.concatenate([b.cpu().numpy() for b in bufs])


@pytest.mark.gpu
@pytest.mark.parametrize("case,interlaced", BOUNDARY_CASES, ids=BOUNDARY_IDS)
def test_calls_that_start_on_a_frame_boundary(built, case, interlaced):
    """A new picture every frame. Whole-frame calls [L, L, 2L, L] through htv_render_host and through htv_render, and
    one htv_render call of 9 frames, which the host splits after 7 new pictures, on a frame boundary (htv_render_host
    would cut it into 8 MB pieces first)."""
    H = built
    name, mode, rate, prate, kw = case
    conf = _boundary_conf(H, mode, kw, interlaced)
    al, aw, W, per = _source_geometry(conf, rate, prate)
    L = conf.lines
    pictures = np.random.default_rng(47).integers(0, 1 << 24, size=(10, al, aw), dtype=np.uint32)
    P = int(H.Tables(conf, rate, prate).get("comp_phases")[0])
    failed = []
    for how, pieces in (("render_host", [L, L, 2 * L, L]), ("render", [L, L, 2 * L, L]), ("one call", [9 * L])):
        enc = H.Encoder(conf, rate, prate)
        enc.set_source(pictures, None)
        if how == "render_host":
            got = np.concatenate([enc.render_host(n) for n in pieces])
        else:
            got = _device_render(H, enc, pieces)
        enc.close()
        diff = _first_difference(got, _oracle(conf, rate, pictures, sum(pieces), prate), L, W, per, P)
        if diff:
            failed.append(f"{how} {pieces}: {diff}")
    assert not failed, "; ".join(failed)


# (mode, rate, overrides, P): the black slot and the conversion count
COMPOSITE = [("i", 16000000, dict(vfilter=True), 4),
             ("pal", 20250000, dict(vfilter=True), 4),          # W = 1296
             ("m", 13500000, dict(vfilter=True), 2)]
BLACK_CASES = [(c, k) for c in COMPOSITE for k in range(1, c[3] + 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("case,k", BLACK_CASES, ids=[f"{c[0]}-{c[1]}-after-{k}" for c, k in BLACK_CASES])
def test_black_slot_at_every_phase(built, case, k):
    """A source that ends after k frames, over 2P + 1 frames: the black slot's rows are shown at every phase, from frame
    k on, in calls that start mid-frame and on frame boundaries."""
    H = built
    mode, rate, kw, P = case
    conf = _quiet(H, mode, kw)
    L = conf.lines
    pictures = _pictures(H, conf, rate, k, 53 + k)
    enc = H.Encoder(conf, rate)
    W = enc.width
    _ended_source(H, enc, pictures)
    pieces = [L // 2, L - L // 2, 2 * L + 9]
    pieces.append((2 * P + 1) * L - sum(pieces))
    got = np.concatenate([enc.render_host(n) for n in pieces])
    enc.close()
    nf = 2 * P + 2
    frames = np.concatenate([pictures, np.zeros((nf - k,) + pictures.shape[1:], dtype=np.uint32)])
    diff = _first_difference(got, _oracle(conf, rate, frames, sum(pieces)), L, W, got.size // (sum(pieces) * W), P)
    assert diff is None, diff


def _launch_deltas(H, conf, rate, pictures, hold, ncalls):
    enc = H.Encoder(conf, rate)
    L = enc.lines
    if hold is None:
        enc.set_source(pictures[:1], None, static_video=True)
    else:
        _held_source(H, enc, pictures, hold)
    deltas, out = [], []
    for _ in range(ncalls):
        before = enc.kernel_launches
        out.append(enc.render_host(L))
        deltas.append(enc.kernel_launches - before)
    enc.close()
    return deltas, np.concatenate(out)


@pytest.mark.gpu
@pytest.mark.parametrize("case", COMPOSITE + [("i", 16000000, dict(vfilter=True, nocolour=True), 1)],
                         ids=["i-16000000", "pal-20250000", "m-13500000", "mono"])
def test_each_picture_is_converted_once_per_phase(built, case):
    """Whole-frame calls, without sound. A static source over 3P calls: each of the first P calls converts its phase
    (one k_compose launch more than the later calls), the later calls convert nothing. A source held for 2 frames:
    each call converts the (picture, phase) pairs it shows for the first time, and the stream equals the oracle's."""
    H = built
    mode, rate, kw, P = case
    conf = _quiet(H, mode, kw)
    pictures = _pictures(H, conf, rate, 3 * P, 59)
    deltas, _ = _launch_deltas(H, conf, rate, pictures, None, 3 * P)
    steady = deltas[P:]
    assert len(set(steady)) == 1, f"launches per call: {deltas}"
    assert deltas[:P] == [steady[0] + 1] * P, f"launches per call: {deltas}; a conversion per phase in the first {P}"
    deltas, got = _launch_deltas(H, conf, rate, pictures, 2, 3 * P)
    shown, want = set(), []
    for f in range(3 * P):
        new = (f // 2, f % P) not in shown
        shown.add((f // 2, f % P))
        want.append(steady[0] + new)
    assert deltas == want, f"launches per call {deltas}, expected {want}"
    L, frames = conf.lines, _frames_shown(pictures, 2, 3 * P + 1)
    W = int(H.Tables(conf, rate).get("geometry")[0])
    diff = _first_difference(got, _oracle(conf, rate, frames, 3 * P * L), L, W, got.size // (3 * P * L * W), P)
    assert diff is None, diff
