"""Every branch of the SECAM chain's fixed-point loop (htv_secam.cuh, htv_dev_render_lines) against the oracle.

The loop runs pass 0 from a guess, proposes better incoming states (k_sec_predict), then refinement passes until no
line's outgoing state changes. A pass re-runs the FM recurrence of its work list with one warp per line (k_sec_fm_list)
or, for more than 2048 lines, one thread per line (k_sec_fm_list_t); after a pass with a long list the predictor may
propose again. The fixed-point check makes the states right whatever the predictor proposed, but the FM inputs (yT),
phasor halves (phT) and checkpoints k_sec_out reads afterwards are only right if every recompute path left them in step
with the final state. Each test here forces or finds one such path, asserts from `Encoder.secam_chain` that it ran,
and compares the stream with the oracle rendering the same lines in one go: bit-exact without sound, within the +-1 LSB
of the sound carriers with it. Knob variants of one case must give identical streams.

HTV_SEC (read when an encoder is created, DESIGN §6) selects the paths: list=warp|thread, pred=<iterations>,
repredict=<budget>, repredict_min=<listed lines>, sub=<lines per launch>, passes=<limit>."""
import contextlib
import functools
import os

import numpy as np
import pytest

import orc

pytestmark = pytest.mark.gpu

F = dict(vfilter=True)
# (id, mode, rate, overrides, W, tolerance against the oracle: 0 bit-exact, 1 the sound carriers' +-1 LSB)
CASES = [
    ("l-13M5", "l", 13500000, F, 864, 1),                                         # AM + NICAM, 21 % of lines listed
    ("l-13M5-noaudio", "l", 13500000, dict(vfilter=True, noaudio=True), 864, 0),
    ("secam-W967", "secam", 15109375, {}, 967, 0),                                # chain tail of 7
    ("secam-W974", "secam", 15218750, {}, 974, 0),                                # chain tail of 14
    ("secam-24M", "secam", 24000000, {}, 1536, 0),                                # the width limit
    ("d-20M", "d", 20000000, F, 1280, 1),                                         # FM sound
    ("secam-fm", "secam-fm", 20250000, dict(vfilter=True, noaudio=True), 1296, 1),  # the chain behind the split raster
]
L16 = ("l-16M", "l", 16000000, F, 1024, 1)                                        # launch boundaries, fused and split
BY_ID = {c[0]: c for c in CASES + [L16]}
PIECES = [1, 2, 23, 300, 625, 2000]           # uneven calls: launches of 3 .. 2002 chain rows
# The cases whose work list is non-empty on random pictures. From 20 Msps on the FM range starts so far into the line
# that a corrected IIR start has decayed below half an LSB before it: no line is listed (l at 20 Msps: none in 64
# frames of the test card or of random pictures), and there forcing a list kernel must change nothing.
LISTING = {"l-13M5", "l-13M5-noaudio", "secam-W967", "secam-W974"}
LIST_MANY = 2048


@contextlib.contextmanager
def _env(**env):
    old = {k: os.environ.get(k) for k in env}
    for k, v in env.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@functools.lru_cache(maxsize=None)
def _random_source(cid):
    """Random pictures, a new one every frame (7 of them, used in turn), and full-scale noise audio."""
    _, mode, rate, kw, _, _ = BY_ID[cid]
    import hacktv_b200 as H
    o = orc.Oracle(H.mode_config(mode, **kw), rate)
    al, aw = o.active_lines, o.active_width
    o.close()
    rng = np.random.default_rng(sum(map(ord, cid)))
    frames = rng.integers(0, 1 << 24, size=(7, al, aw), dtype=np.uint32)
    audio = rng.integers(-32768, 32767, size=(40000, 2), dtype=np.int16)
    return frames, audio


def _source(cid, src):
    """None for the test card; else (frames, audio, static): "random" changes picture every frame, "still" holds the
    first random picture for the whole call. A call whose every frame is a new picture is cut into launches of the few
    pictures the encoder's frame slots hold; a still picture lets a 64-frame call be one launch."""
    if src == "card":
        return None
    frames, audio = _random_source(cid)
    return (frames[:1], audio, True) if src == "still" else (frames, audio, False)


def _render(H, cid, src, pieces, *, sec=None, path=None):
    """The stream over device-resident calls (htv_render) of `pieces` lines, what the chain did, and the kernels the
    last call ran. A call into device memory is one chain launch up to the launch size; htv_render_host would cut it
    into 8 MB pieces."""
    import torch
    _, mode, rate, kw, W, _ = BY_ID[cid]
    with _env(HTV_SEC=sec, HTV_PATH=path):
        enc = H.Encoder(H.mode_config(mode, **kw), rate)
    try:
        assert enc.width == W
        s = _source(cid, src)
        if s is None:
            enc.open_test_source()
        else:
            enc.set_source(s[0], s[1], static_video=s[2])
        st = torch.cuda.current_stream().cuda_stream
        got = []
        for n in pieces:
            buf = torch.empty(n * W * (2 if enc.complex else 1), dtype=torch.int16, device="cuda")
            enc.render(n, buf.data_ptr(), st)
            torch.cuda.synchronize()
            got.append(buf.cpu().numpy())
            del buf
        return np.concatenate(got), enc.secam_chain, enc.line_kernel
    finally:
        enc.close()


@functools.lru_cache(maxsize=None)
def _oracle(cid, src, nlines):
    _, mode, rate, kw, _, _ = BY_ID[cid]
    import hacktv_b200 as H
    o = orc.Oracle(H.mode_config(mode, **kw), rate)
    s = _source(cid, src)
    if s is None:
        o.open_test_source()
    else:
        o.set_source(s[0], s[1])
    want = o.render(nlines)
    o.close()
    return want


@functools.lru_cache(maxsize=None)
def _default(cid, src):
    """The stream with HTV_SEC unset over PIECES, reused by every knob variant of the case."""
    import hacktv_b200 as H
    return _render(H, cid, src, PIECES)


def _check_oracle(got, want, tol, what):
    assert got.size == want.size, (got.size, want.size)
    d = np.abs(got.astype(np.int32) - want.astype(np.int32))
    if tol == 0:
        bad = np.flatnonzero(d)
        assert bad.size == 0, f"{what}: {bad.size} values differ from the oracle, first at value {bad[0]}"
    else:
        assert d.max() <= tol, f"{what}: max |diff| {d.max()} at value {np.argmax(d)}; {np.count_nonzero(d > tol)} over {tol}"
        assert (d == 0).mean() > 0.97, f"{what}: only {(d == 0).mean():.4f} of values exact"


def _same(got, ref, what):
    assert got.size == ref.size
    bad = np.flatnonzero(got != ref)
    assert bad.size == 0, f"{what}: {bad.size} values differ, first at value {bad[0]}"


@pytest.mark.parametrize("src", ["card", "still"])
def test_long_work_list_at_production_size(built, src):
    """SECAM-L 13.5 Msps --filter, 64 frames (40 000 lines) in one call and one chain launch, on the test card and on a
    random picture: the work list is long enough for k_sec_fm_list_t, and the stream equals the oracle's."""
    H = built
    nlines = 40000
    got, cs, _ = _render(H, "l-13M5-noaudio", src, [nlines])
    assert cs["launches"] == 1, cs
    assert cs["listed_thread"] > 0 and cs["list_max"] > LIST_MANY, cs
    _check_oracle(got, _oracle("l-13M5-noaudio", src, nlines), 0, "no sound")
    del got
    if src == "card":
        got, cs, _ = _render(H, "l-13M5", src, [nlines])
        assert cs["listed_thread"] > 0 and cs["list_max"] > LIST_MANY, cs
        _check_oracle(got, _oracle("l-13M5", src, nlines), 1, "AM + NICAM")


@pytest.mark.parametrize("src", ["card", "random"])
@pytest.mark.parametrize("cid", [c[0] for c in CASES])
def test_both_list_kernels_give_the_same_bits(built, cid, src):
    """list=warp and list=thread put every listed line on one kernel; both streams equal the default one and the
    oracle. On random pictures the forced kernel must have had work where the rate lists lines at all (LISTING)."""
    H = built
    tol = BY_ID[cid][5]
    ref, cs, _ = _default(cid, src)
    _check_oracle(ref, _oracle(cid, src, sum(PIECES)), tol, "default")
    if cid not in LISTING:
        assert cs["listed_warp"] + cs["listed_thread"] == 0, cs
    for kind, other in (("warp", "thread"), ("thread", "warp")):
        got, cs, _ = _render(H, cid, src, PIECES, sec=f"list={kind}")
        assert cs[f"listed_{other}"] == 0, cs
        if src == "random" and cid in LISTING:
            assert cs[f"listed_{kind}"] > 0, cs
        _same(got, ref, f"list={kind}")


@pytest.mark.parametrize("cid", [c[0] for c in CASES])
def test_plain_iteration_reaches_the_same_fixed_point(built, cid):
    """pred=0, repredict=0: pass 1 starts from pass 0's states, so the loop iterates, lines are recomputed more than
    once, and launches end on odd and on even passes. The stream must still equal the default one and the oracle."""
    H = built
    ref, _, _ = _default(cid, "random")
    got, cs, _ = _render(H, cid, "random", PIECES, sec="pred=0,repredict=0")
    assert cs["passes_max"] >= 4, cs
    assert cs["final_odd"] > 0 and cs["final_even"] > 0, cs
    assert cs["repredict_odd"] == cs["repredict_even"] == 0, cs
    _same(got, ref, "pred=0")
    _check_oracle(got, _oracle(cid, "random", sum(PIECES)), BY_ID[cid][5], "pred=0")


@pytest.mark.parametrize("cid", [c[0] for c in CASES])
def test_reprediction_after_odd_and_even_passes(built, cid):
    """pred=1 leaves pass 1 far from the fixed point; with repredict_min=-1 the predictor proposes again after every
    pass that changed a state, up to 4 times: after passes 1 and 2, whose buffer copies go in opposite orders. The
    stream must equal the default one."""
    H = built
    ref, _, _ = _default(cid, "random")
    got, cs, _ = _render(H, cid, "random", PIECES, sec="pred=1,repredict=4,repredict_min=-1")
    assert cs["repredict_odd"] > 0 and cs["repredict_even"] > 0, cs
    _same(got, ref, "pred=1, repredict=4")


LAUNCH_CASES = [("l-16M", None), ("l-16M", "split"), ("secam-fm", None)]


@functools.lru_cache(maxsize=None)
def _one_launch(cid, path, nlines):
    import hacktv_b200 as H
    return _render(H, cid, "random", [nlines], path=path)


@pytest.mark.parametrize("sub", [64, 313])
@pytest.mark.parametrize("cid,path", LAUNCH_CASES, ids=[f"{c}-{p or 'fused'}" for c, p in LAUNCH_CASES])
def test_several_launches_per_call(built, cid, path, sub):
    """sub=64 / 313 lines per chain launch: one call of 2 000 lines crosses launch boundaries at offsets that fall
    differently against the field starts. The stream equals the one-launch stream and the oracle."""
    H = built
    nlines = 2000
    ref, cs1, name = _one_launch(cid, path, nlines)
    assert cs1["launches"] == 1, cs1
    if cid == "secam-fm":
        assert name.startswith("k_raster_secam + k_fmv_base"), name
    else:
        assert name.startswith("k_raster_secam + " if path == "split" else "k_sec_raster<"), name
    _check_oracle(ref, _oracle(cid, "random", nlines), BY_ID[cid][5], "one launch")
    got, cs, _ = _render(H, cid, "random", [nlines], sec=f"sub={sub}", path=path)
    assert cs["launches"] >= -(-nlines // sub), cs
    _same(got, ref, f"sub={sub}")


def test_render_add_across_launches(built):
    """htv_render_add with 313 lines per launch: each launch adds its lines at its own offset of the stream being
    summed into."""
    import torch
    H = built
    nlines = 2000
    ref, _, _ = _one_launch("l-16M", None, nlines)
    base = np.random.default_rng(3).integers(-32768, 32767, size=ref.size, dtype=np.int16)
    buf = torch.from_numpy(base.copy()).cuda()
    _, mode, rate, kw, _, _ = BY_ID["l-16M"]
    with _env(HTV_SEC="sub=313"):
        enc = H.Encoder(H.mode_config(mode, **kw), rate)
    try:
        enc.set_source(*_random_source("l-16M"))
        st = torch.cuda.current_stream().cuda_stream
        enc.render_add(nlines, buf.data_ptr(), st)
        torch.cuda.synchronize()
        cs = enc.secam_chain
    finally:
        enc.close()
    assert cs["launches"] >= -(-nlines // 313), cs
    want = (base.astype(np.int32) + ref.astype(np.int32)).astype(np.int16)     # int16 wrap
    _same(buf.cpu().numpy(), want, "render_add, sub=313")


def test_a_chain_that_does_not_converge_is_refused(built, capfd):
    """pred=0, repredict=0, passes=1 on a call that needs more passes: the render fails with a message, the encoder
    closes, and the next encoder renders the oracle's stream."""
    H = built
    _, mode, rate, kw, _, _ = BY_ID["l-13M5-noaudio"]
    with _env(HTV_SEC="pred=0,repredict=0,passes=1"):
        enc = H.Encoder(H.mode_config(mode, **kw), rate)
    enc.set_source(*_random_source("l-13M5-noaudio"))
    capfd.readouterr()
    import torch
    buf = torch.empty(2000 * enc.width * 2, dtype=torch.int16, device="cuda")
    with pytest.raises(RuntimeError):
        enc.render(2000, buf.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    cs = enc.secam_chain
    enc.close()
    assert "SECAM cross-line state did not converge in 1 passes" in capfd.readouterr().err
    assert cs["launches"] == 1 and cs["passes"] == 1 and cs["final_odd"] + cs["final_even"] == 0, cs
    got, cs, _ = _render(H, "l-13M5-noaudio", "random", [700])
    assert cs["final_odd"] + cs["final_even"] == cs["launches"] == 1, cs
    _check_oracle(got, _oracle("l-13M5-noaudio", "random", 700), 0, "after a refused chain")


@pytest.mark.parametrize("value,message", [
    ("lst=warp", "unknown key 'lst'"),
    ("list=both", "list=both is not auto, warp or thread"),
    ("pred=-1", "pred=-1 is not an integer"),
    ("repredict_min=-2", "repredict_min=-2 is not an integer"),
    ("pred=3x", "pred=3x is not an integer"),
    ("passes=0", "passes=0 is not an integer"),
    ("sub=63", "sub=63 is not an integer"),
    ("sub=1000000", "sub=1000000 is more than"),
    ("repredict", "'repredict' is not key=value"),
    ("list=warp,pred=", "pred= is not an integer"),
])
def test_bad_knobs_are_refused(built, capfd, value, message):
    """A typo in HTV_SEC fails the encoder with a message naming it, for SECAM and for every other mode."""
    H = built
    for mode, rate in (("l", 16000000), ("i", 16000000)):
        if "more than" in message and mode != "l":
            continue
        with _env(HTV_SEC=value), pytest.raises(RuntimeError):
            H.Encoder(H.mode_config(mode), rate)
        err = capfd.readouterr().err
        assert "HTV_SEC" in err and message in err, err


def test_counters_are_zero_without_secam(built):
    H = built
    enc = H.Encoder(H.mode_config("i", vfilter=True), 16000000)
    enc.open_test_source()
    enc.render_host(700)
    cs = enc.secam_chain
    assert enc.line_kernel.startswith("k_line<")
    enc.close()
    assert set(cs.values()) == {0}, cs
