"""The stage after the modulator - IQ swap, the frequency-offset mixer from its start-up, the channel combiner
(--passthru, htv_render_add) and the store - at every kernel form, against the oracle.

Every emitted sample passes kl_mix + kl_post_store (htv_sound.cuh, htv_line.cuh) in k_line, SECAM's SRC form included, or
kl_mix<-1, 1> + mod_store (htv_kernels.cu) in k_mod, k_mod_tma, k_mod_mma and k_fmv_mod. Both have width-dependent
branches: the partial last tile, the single-warp CTA, mod_store's 128-bit branch (4 | W) and its per-sample one, and
`acc` stops at acc_rows, which can fall inside a persistent CTA's run of lines. The other device matrices render with the
stage idle. ROWS: the narrowest row of each (line_kernel, P = 0 or not, complex or real output) of the colour-phase,
line-width and low-rate matrices (no S-Video, no --pixelrate: their mixer and combiner rows are in their own files), the
narrowest of each W mod 4 those miss, and two FM-video rows. Without sound, so that every claim is sharp:
  - IQ swap: bit-exact.
  - --swap-iq --offset f in uneven calls, one boundary inside the offset mixer's start-up (audio-clock samples
    m < 32 767, where dt.offset_start replaces the NCO; the emitted stream starts at m = shift) and one on the line that
    holds m = 32 767: bit-exact before it (integer work), +-1 LSB after, and the one-call stream bit for bit.
  - --passthru of a full-range stream that ends mid-line inside the second of three calls: bit-exact (int16 wrap, I only
    for real output, whole lines only after the end).
  - htv_render_add into a stream already in device memory, passthru_delay_lines lines in (the reference's alignment):
    the oracle's passthru of that stream, the lines before it and the bytes around the buffer untouched.
  - htv_render at int16, int8 and float in uneven calls back to back, a guard right after the last byte: htv_convert of
    the int16 stream, guards intact (rows with a partial tile, a single warp or 4 not dividing W).
  - The typed store with the combiner; the mode's sound through both combiners on two rows; the two-channel recipe at
    W = 858.
FM video is +-1 LSB from the oracle before this stage (test_gpu_parity.py), so its rows take that tolerance, modulo the
int16 wrap. Without a GPU: the rows are what they state and cover what they exist for, and every offset row's start-up
window holds a call boundary and the line of sample 32 767."""
import numpy as np
import pytest

import orc
from test_gpu_zz_colour_phases import ROWS as PHASE_ROWS, _phases
from test_gpu_zz_line_widths import FIXED, MATRIX as WIDTHS, _check_sound, _picture_lines, kl
from test_gpu_zz_low_rates import MATRIX as LOW_RATES
from test_gpu_zz_sample_types import _convert

F = dict(vfilter=True)
# P of the split rows (the PAL and NTSC k_line rows take theirs from the colour-phase matrix); SECAM has one phase
SPLIT_PHASES = {("pal", 1250000): 4, ("i", 1250000): 4, ("ntsc", 1250000): 0}
REAL = {"pal", "ntsc", "secam", "pal60", "525pal", "pal-m"}      # baseband modes: the output is I only
FMV = "k_raster + k_fmv_base<{}> + k_fmv_scan + k_fmv_mod"
FM_VIDEO = [("ntsc-fm", 20250000, F, 1287, FMV.format(71), 2),     # mod_store's per-sample branch, pre-emphasis
            ("pal-fm", 20000000, {}, 1280, FMV.format(0), 4)]      # its 128-bit branch


def _sources():
    """(mode, rate, overrides, W, line_kernel, P) of every row the stage is derived from"""
    rows = [(m, r, kw, W, k, _phases(m, r, kw)) for m, r, kw, W, k in PHASE_ROWS if not kw.get("s_video")]
    for m, r, kw, W, k in WIDTHS + LOW_RATES:
        if k.startswith("k_sec_raster"):
            rows.append((m, r, kw, W, k, 1))
        elif not k.startswith("k_line"):
            rows.append((m, r, kw, W, k, SPLIT_PHASES[(m, r)]))
    return rows


def _rows():
    """(mode, rate, overrides, W, line_kernel, P, complex): the narrowest source row of each (line_kernel, P = 0,
    complex), then the narrowest of every W mod 4 none of those has, then the FM-video rows"""
    by_width = sorted(_sources(), key=lambda c: c[3])
    rows, keys = [], set()
    for c in by_width:
        key = (c[4], c[5] == 0, c[0] not in REAL)
        if key not in keys:
            keys.add(key)
            rows.append(c)
    for c in by_width:
        if c[3] % 4 not in {r[3] % 4 for r in rows}:
            rows.append(c)
    return [c + (c[0] not in REAL,) for c in rows + FM_VIDEO]


ROWS = _rows()
COMPLEX = [r for r in ROWS if r[6]]
# rows with a partial last tile, a single-warp CTA or 4 not dividing W: the buffer edges
EDGES = [r for r in ROWS if r[3] % 128 or r[3] <= 128 or r[3] % 4]
# the typed store with the combiner: ST = -1 k_line forms at a partial tile (complex) and single-warp rows, k_mod, and
# mod_store's complex typed store behind FM video
TYPED = [r for r in ROWS if (r[0], r[1]) in {("m", 20250000), ("i", 500000), ("pal", 1500000), ("ntsc", 1250000),
                                              ("ntsc-fm", 20250000)}]
ARGS = "mode,rate,kw,W,kernel,P,cpx"


def case_id(c):
    mode, rate, kw, W = c[:4]
    return f"{mode}-{rate}-W{W}" + "".join(f"-{k}" for k, v in kw.items() if v)


def _ids(rows):
    return [case_id(r) for r in rows]


def _delay(kw):
    """passthru_delay_lines = shift / W: one line with a video filter or FM pre-emphasis, else none"""
    return 1 if kw.get("vfilter") else 0


def _quiet(H, mode, kw, **more):
    return H.mode_config(mode, **dict(kw, noaudio=True, **more))


def _tol(kernel):
    return 1 if "k_fmv" in kernel else 0


def _lines(conf):
    return 290 if conf.lines == 525 else 340          # first field, its picture and the next vertical blanking


def _offset(rate, i):
    """about rate / 8, never a small rational fraction of it; the sign alternates over the rows"""
    return (rate // 8 + 12347) * (-1 if i % 2 else 1)


def _start_line(W, kw):
    """the line that holds audio-clock sample 32 767, the first the NCO serves (the stream starts at m = shift)"""
    return (32767 - _delay(kw) * W) // W


def _offset_calls(W, kw):
    """one boundary inside the start-up window, one on the line of sample 32 767, then two more calls"""
    s = _start_line(W, kw)
    a = max(1, s // 3)
    return [a, s - a, 3, 9]


PT_CALLS = [60, 45, 9]                      # the external stream ends 21 lines into the second call, mid-line
PT_LINES = PT_CALLS[0] + 21


def _wrap(d):
    return (d + 32768) % 65536 - 32768


def _where(i, pieces, W, per):
    L, x = divmod(int(i), W * per)
    starts = np.cumsum([0] + list(pieces))
    call = int(np.searchsorted(starts, L, side="right")) - 1
    part = f" ({'IQ'[x % 2]})" if per == 2 else ""
    return f"call {call} ({pieces[call]} lines from line {starts[call]}), line {L}, sample {x // per}{part}"


def _compare(got, want, tol, pieces, W, per, what, mask=None):
    """|got - want| modulo the int16 wrap <= tol where mask (all values by default); on failure the call, line, sample
    and component of the first value over"""
    assert got.size == want.size, (got.size, want.size)
    d = np.abs(_wrap(got.astype(np.int32) - want.astype(np.int32)))
    over = d > tol if mask is None else (d > tol) & mask
    bad = np.flatnonzero(over)
    if bad.size:
        i = bad[0]
        pytest.fail(f"{what}: {bad.size} of {int(over.size if mask is None else mask.sum())} values off by more than "
                    f"{tol}; first at {_where(i, pieces, W, per)}: {got[i]} against {want[i]}")


def _oracle(conf, rate, nlines, ext=None):
    o = orc.Oracle(conf, rate)
    o.open_test_source()
    if ext is not None:
        o.set_passthru(ext)
    want = o.render(nlines)
    o.close()
    return want


def _host(H, conf, rate, pieces, ext=None, sample_type=None):
    """htv_render_host over calls of `pieces` lines (bytes for another sample type), and the line kernel it ran"""
    enc = H.Encoder(conf, rate)
    enc.open_test_source()
    if ext is not None:
        enc.set_passthru(ext)
    if sample_type:
        enc.set_sample_type(sample_type)
    parts = [enc.render_host(n) for n in pieces]
    name = enc.line_kernel
    delay = enc.passthru_delay_lines
    enc.close()
    got = b"".join(p.tobytes() for p in parts) if sample_type else np.concatenate(parts)
    return got, name, delay


def _external(W, lines, seed):
    """a full-range int16 complex stream of `lines` lines and a third of one"""
    rng = np.random.default_rng(seed)
    return rng.integers(-32768, 32767, size=(lines * W + W // 3, 2), dtype=np.int16, endpoint=True)


def _typed_name(kernel, sample_type):
    return kernel[:-1] + f",ST=-1:{sample_type}>" if kernel.startswith("k_line") else None


# ---- without a GPU ------------------------------------------------------------------------------------------------

def test_rows_are_what_they_state(built):
    """Each row's W, P, output and the C selection's kernel (without sound, with --swap-iq --offset: the general forms
    test dp for both) are what it states. Together the rows cover every line-kernel string of the source matrices, P = 0,
    real output, W mod 4 = 0..3, the partial last tile, W <= 128, k_mod / k_mod_tma / k_mod_mma / k_fmv_mod and SRC."""
    from test_tables_and_abi import _plan_name
    H = built
    assert 40 <= len(ROWS) <= 70, len(ROWS)
    for i, (mode, rate, kw, W, kernel, P, cpx) in enumerate(ROWS):
        t = H.Tables(_quiet(H, mode, kw), rate)
        w, p = int(t.get("geometry")[0]), int(t.get("comp_phases")[0])
        t.close()
        what = (mode, rate, kw)
        assert (w, p) == (W, P), (what, w, p)
        assert (H.mode_config(mode).output_type == 0) == cpx, what
        assert _plan_name(H, mode, rate, dict(kw, noaudio=True)) == kernel, what
        if cpx:
            assert _plan_name(H, mode, rate, dict(kw, noaudio=True, swap_iq=True, offset=_offset(rate, i))) == kernel
    kernels = {r[4] for r in ROWS}
    assert {c[4] for c in _sources()} <= kernels
    assert {W % 4 for W in (r[3] for r in ROWS)} == {0, 1, 2, 3}
    assert any(r[5] == 0 for r in ROWS) and any(not r[6] for r in ROWS)
    assert any(r[3] % 128 and r[3] > 128 for r in ROWS) and any(r[3] <= 128 and r[3] % 128 for r in ROWS)
    for form in ("k_mod<", "k_mod_tma<", "k_mod_mma<", "k_fmv_mod", "SRC=1"):
        assert any(form in k for k in kernels), form
    assert any("k_fmv_mod" in r[4] and r[3] % 4 for r in ROWS) and any("k_fmv_mod" in r[4] and not r[3] % 4 for r in ROWS)
    for mode, rate, kw, W, kernel in [t[:5] for t in TYPED]:
        if kernel.startswith("k_line"):
            for st in ("int8", "float"):
                assert _plan_name(H, mode, rate, dict(kw, noaudio=True), sample_type=st) == _typed_name(kernel, st)
    assert {"k_mod<" in r[4] for r in TYPED} == {True, False}
    assert any(r[3] <= 128 for r in TYPED) and any(r[3] % 128 and r[3] > 128 and r[6] for r in TYPED)


def test_every_offset_window_holds_a_boundary_and_the_first_nco_line(built):
    """The start-up ends inside line _start_line (0-based, emitted): a call starts there and one starts before it
    inside the window, so that the bit-exact part of test_swap_and_offset_from_the_start_up is never vacuous."""
    for mode, rate, kw, W, *_ in COMPLEX:
        s = _start_line(W, kw)
        first = s * W + _delay(kw) * W                 # audio-clock sample of the line's first sample
        assert first <= 32767 < first + W, (mode, rate)
        starts = np.cumsum([0] + _offset_calls(W, kw))
        assert s in starts and any(0 < b < s for b in starts), (mode, rate, starts)
        assert starts[-1] > s + 1


# ---- on the GPU ---------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize(ARGS, COMPLEX, ids=_ids(COMPLEX))
def test_iq_swap(built, mode, rate, kw, W, kernel, P, cpx):
    H = built
    conf = _quiet(H, mode, kw, swap_iq=True)
    n = _lines(conf)
    got, name, _ = _host(H, conf, rate, [n])
    assert name == kernel, f"{mode} {rate} ran {name}, the row exists for {kernel}"
    _compare(got, _oracle(conf, rate, n), _tol(kernel), [n], W, 2, "--swap-iq")


@pytest.mark.gpu
@pytest.mark.parametrize(ARGS, COMPLEX, ids=_ids(COMPLEX))
def test_swap_and_offset_from_the_start_up(built, mode, rate, kw, W, kernel, P, cpx):
    H = built
    conf = _quiet(H, mode, kw, swap_iq=True, offset=_offset(rate, ROWS.index((mode, rate, kw, W, kernel, P, cpx))))
    pieces = _offset_calls(W, kw)
    n = sum(pieces)
    got, name, delay = _host(H, conf, rate, pieces)
    assert name == kernel, f"{mode} {rate} ran {name}, the row exists for {kernel}"
    assert delay == _delay(kw)
    want = _oracle(conf, rate, n)
    m = np.arange(got.size) // 2 + delay * W                 # audio-clock sample of every value
    fm = _tol(kernel)
    _compare(got, want, fm, pieces, W, 2, "the offset mixer's start-up (m < 32767)", m < 32767)
    _compare(got, want, 1 + 2 * fm, pieces, W, 2, "the offset mixer after its start-up", m >= 32767)
    whole, _, _ = _host(H, conf, rate, [n])
    _compare(got, whole, 0, pieces, W, 2, f"calls {pieces} against one call")


@pytest.mark.gpu
@pytest.mark.parametrize(ARGS, ROWS, ids=_ids(ROWS))
def test_passthru_that_ends_mid_line(built, mode, rate, kw, W, kernel, P, cpx):
    """The staging buffer's rows past the stream's end still hold the first call's lines: an add past acc_rows shows."""
    H = built
    conf = _quiet(H, mode, kw)
    ext = _external(W, _delay(kw) + PT_LINES, 61)
    got, name, _ = _host(H, conf, rate, PT_CALLS, ext)
    assert name == kernel, f"{mode} {rate} ran {name}, the row exists for {kernel}"
    want = _oracle(conf, rate, sum(PT_CALLS), ext)
    _compare(got, want, _tol(kernel), PT_CALLS, W, 2 if cpx else 1, "--passthru")
    plain = _oracle(conf, rate, sum(PT_CALLS))
    per = 2 if cpx else 1
    assert np.array_equal(want[PT_LINES * W * per:], plain[PT_LINES * W * per:]), "the oracle adds past the stream's end"
    assert not np.array_equal(want[:PT_LINES * W * per], plain[:PT_LINES * W * per])


SENTINEL = 64                               # guard bytes on either side of a device buffer


def _guarded(nbytes, seed):
    """a device buffer of nbytes between two guards, all of it a sentinel pattern; the payload starts 16-byte aligned"""
    import torch
    pattern = np.random.default_rng(seed).integers(0, 256, size=nbytes + 2 * SENTINEL, dtype=np.uint8)
    return torch.from_numpy(pattern).cuda(), pattern


def _check_guards(out, pattern, nbytes, what):
    for name, sl in (("before", slice(0, SENTINEL)), ("after", slice(SENTINEL + nbytes, None))):
        bad = np.flatnonzero(out[sl] != pattern[sl])
        assert bad.size == 0, f"{what}: {bad.size} guard bytes {name} the buffer changed, first at {bad[0]}"


@pytest.mark.gpu
@pytest.mark.parametrize(ARGS, ROWS, ids=_ids(ROWS))
def test_render_add_at_the_reference_alignment(built, mode, rate, kw, W, kernel, P, cpx):
    """Stream A (full-range) in device memory, this encoder added into it from line passthru_delay_lines on in uneven
    calls (the pointer 4, 8 or 12 bytes off 16 where 4 does not divide W): the oracle's --passthru of A."""
    import torch
    H = built
    conf = _quiet(H, mode, kw)
    pieces = [37, 1, 70]
    n = sum(pieces)
    enc = H.Encoder(conf, rate)
    enc.open_test_source()
    delay, bps, per = enc.passthru_delay_lines, enc.bytes_per_sample, 2 if cpx else 1
    ext = _external(W, n + delay, 67)[:(n + delay) * W]
    a = np.ascontiguousarray(ext if cpx else ext[:, 0]).reshape(-1)
    nbytes = a.size * 2
    buf, pattern = _guarded(nbytes, 71)
    pattern[SENTINEL:SENTINEL + nbytes] = a.view(np.uint8)
    buf.copy_(torch.from_numpy(pattern))
    st = torch.cuda.current_stream().cuda_stream
    ptr = buf.data_ptr() + SENTINEL + delay * W * bps
    done = 0
    for c in pieces:
        enc.render_add(c, ptr + done * W * bps, st)
        done += c
    torch.cuda.synchronize()
    name = enc.line_kernel
    enc.close()
    assert name == kernel, f"{mode} {rate} ran {name}, the row exists for {kernel}"
    out = buf.cpu().numpy()
    _check_guards(out, pattern, nbytes, "htv_render_add")
    got = out[SENTINEL:SENTINEL + nbytes].view(np.int16)
    assert np.array_equal(got[:delay * W * per], a[:delay * W * per]), "the lines before the pointer changed"
    _compare(got[delay * W * per:], _oracle(conf, rate, n, ext), _tol(kernel), pieces, W, per, "htv_render_add")


@pytest.mark.gpu
@pytest.mark.parametrize("sample_type", ["int16", "int8", "float"])
@pytest.mark.parametrize(ARGS, EDGES, ids=_ids(EDGES))
def test_render_buffer_edges(built, mode, rate, kw, W, kernel, P, cpx, sample_type):
    """htv_render in calls back to back (real int8 at odd W puts lines at odd addresses), the buffer's end right at the
    guard: htv_convert of the int16 stream, and no byte outside the buffer written."""
    import torch
    H = built
    conf = _quiet(H, mode, kw)
    pieces = [13, 1, 40, 7]
    n = sum(pieces)
    ref, _, _ = _host(H, conf, rate, [n])
    want = ref.tobytes() if sample_type == "int16" else _convert(H, ref, sample_type)
    enc = H.Encoder(conf, rate)
    enc.open_test_source()
    if sample_type != "int16":
        enc.set_sample_type(sample_type)
    bps = enc.bytes_per_sample
    nbytes = n * W * bps
    assert nbytes == len(want)
    buf, pattern = _guarded(nbytes, 73)
    st = torch.cuda.current_stream().cuda_stream
    done = 0
    for c in pieces:
        assert enc.render(c, buf.data_ptr() + SENTINEL + done * W * bps, st) == c * W
        done += c
    torch.cuda.synchronize()
    name = enc.line_kernel
    enc.close()
    if sample_type != "int16":
        assert f"ST=-1:{sample_type}" in name, name
    out = buf.cpu().numpy()
    _check_guards(out, pattern, nbytes, f"htv_render {sample_type}")
    got = out[SENTINEL:SENTINEL + nbytes].tobytes()
    if got != want:
        size = bps // (2 if cpx else 1)
        i = next(k for k in range(nbytes) if got[k] != want[k]) // size
        pytest.fail(f"htv_render {sample_type} differs from htv_convert of int16 first at "
                    f"{_where(i, pieces, W, 2 if cpx else 1)}")


@pytest.mark.gpu
@pytest.mark.parametrize("sample_type", ["int8", "float"])
@pytest.mark.parametrize(ARGS, TYPED, ids=_ids(TYPED))
def test_typed_store_with_passthru(built, mode, rate, kw, W, kernel, P, cpx, sample_type):
    """The typed combiners (kl_post_store, mod_store) add the staged int16 stream before the conversion: htv_convert
    of the int16 stream with the same --passthru."""
    H = built
    conf = _quiet(H, mode, kw)
    ext = _external(W, _delay(kw) + PT_LINES, 79)
    ref, _, _ = _host(H, conf, rate, PT_CALLS, ext)
    got, name, _ = _host(H, conf, rate, PT_CALLS, ext, sample_type)
    typed = _typed_name(kernel, sample_type)
    assert name == typed if typed else f"ST=-1:{sample_type}" in name, name
    want = _convert(H, ref, sample_type)
    if got != want:
        size = len(want) // ref.size
        i = next(k for k in range(len(want)) if got[k] != want[k]) // size
        pytest.fail(f"{sample_type} with --passthru differs from htv_convert of int16 first at "
                    f"{_where(i, PT_CALLS, W, 2 if cpx else 1)}")


# the form with PAL's sound stages compiled in, and a general 384-thread row with FM + NICAM
SOUND_ROWS = [("i", 16000000, F, 1024, FIXED), ("i", 20250000, F, 1296, kl(1, 1, 0, 0, 384))]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,rate,kw,W,kernel", SOUND_ROWS, ids=["fixed-W1024", "general-384-W1296"])
def test_combiners_with_sound(built, mode, rate, kw, W, kernel):
    """--passthru and htv_render_add with the mode's sound: +-1 LSB (modulo the wrap) and >= 97 % exact in every tile
    column of the blanking and of the picture lines."""
    import torch
    H = built
    conf = H.mode_config(mode, **kw)
    n = 340
    quiet = _oracle(H.mode_config(mode, noaudio=True, **kw), rate, n)
    picture = _picture_lines(H, conf, rate, quiet)
    ext = _external(W, n + 1, 83)
    want = _oracle(conf, rate, n, ext)
    pieces = [100, 3, 237]
    got, name, _ = _host(H, conf, rate, pieces, ext)
    assert name == kernel, name
    _check_sound(_wrap(got.astype(np.int32) - want), np.zeros(want.size, np.int32), W, picture, "--passthru")

    enc = H.Encoder(conf, rate)
    enc.open_test_source()
    a = ext[:(n + 1) * W].reshape(-1)
    buf = torch.from_numpy(a.copy()).cuda()
    st = torch.cuda.current_stream().cuda_stream
    done = 0
    for c in pieces:
        enc.render_add(c, buf.data_ptr() + (1 + done) * W * 4, st)
        done += c
    torch.cuda.synchronize()
    assert enc.line_kernel == kernel
    enc.close()
    got = buf.cpu().numpy()
    assert np.array_equal(got[:W * 2], a[:W * 2])
    _check_sound(_wrap(got[W * 2:].astype(np.int32) - want), np.zeros(want.size, np.int32), W, picture,
                 "htv_render_add")


@pytest.mark.gpu
def test_two_channel_recipe_at_858_samples_a_line(built):
    """`hacktv --offset -6.75e6 --level 0.5 --filter -o - | hacktv --offset 1.25e6 --level 0.5 --passthru /dev/stdin
    --filter` for NTSC-M at 13.5 Msps, device-resident: channel B added into channel A one line later, at a pointer
    8 bytes off 16. It equals the oracle's --passthru of channel A within +-1 LSB per channel's NCO."""
    import torch
    H = built
    rate, n = 13500000, 400
    ca = H.mode_config("m", vfilter=True, offset=-6750000, level=0.5)
    cb = H.mode_config("m", vfilter=True, offset=1250000, level=0.5)
    a = H.Encoder(ca, rate); a.open_test_source()
    b = H.Encoder(cb, rate); b.open_test_source()
    W = a.width
    assert W == 858 and b.passthru_delay_lines == 1 and (W * 4) % 16 == 8
    buf = torch.zeros((n + 1) * W * 2, dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    a.render(n + 1, buf.data_ptr(), st)
    b.render_add(n, buf.data_ptr() + W * 4, st)
    torch.cuda.synchronize()
    got = buf[W * 2:].cpu().numpy()
    a.close(); b.close()
    sa = _oracle(ca, rate, n + 1)
    want = _oracle(cb, rate, n, sa.reshape(-1, 2))
    d = np.abs(_wrap(got.astype(np.int32) - want))
    assert d.max() <= 2, d.max()
    assert np.count_nonzero(d) < d.size // 20


@pytest.mark.gpu
@pytest.mark.parametrize("mode,rate,kw,align", [
    ("m", 13500000, F, 4),                        # k_line: one complex int16 sample per access
    ("ntsc", 1250000, {}, 2),                     # k_mod at W = 79: its per-sample branch
    ("pal", 1250000, {}, 8),                      # k_mod_tma, real: four samples in 8 bytes
    ("i", 1250000, F, 16),                        # k_mod_mma, complex: four samples in 16 bytes
    ("pal-fm", 20000000, {}, 16),                 # k_fmv_mod at W = 1280
])
def test_output_alignment_is_the_stores_widest_access(built, capfd, mode, rate, kw, align):
    """htv_render and htv_render_add take a pointer one line into a 16-byte aligned buffer, and refuse one at half the
    alignment the store needs, before anything is launched."""
    import torch
    H = built
    conf = _quiet(H, mode, kw)
    enc = H.Encoder(conf, rate)
    enc.open_test_source()
    W, bps = enc.width, enc.bytes_per_sample
    buf = torch.zeros(8 * W * bps + 64, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    base = buf.data_ptr()
    for render in (enc.render, enc.render_add):
        with pytest.raises(RuntimeError):
            render(2, base + align // 2, st)
        assert f"the output buffer must be {align}-byte aligned" in capfd.readouterr().err
        render(2, base + W * bps, st)
    torch.cuda.synchronize()
    enc.close()
    assert (W * bps) % align == 0
