"""The rows of test_gpu_zz_low_rate_paths.py without a GPU: each is what it states (W, Wp, P, the chroma low-pass and the
kernel the C selection names), together they reach the paths below 10 Msps that file exists for, each is pinned to the
reference (golden_ref.json, golden_s_video.json), and the configurations next to them that the kernels cannot hold are
refused with a message that names the limit."""
import json
import os

import numpy as np
import pytest

import orc
from test_gpu_zz_low_rate_paths import CSAT, PIXELRATE, PS, S_VIDEO, SF
from test_s_video_host import _plan_refusal
from test_tables_and_abi import _plan_name

HERE = os.path.dirname(os.path.abspath(__file__))


def _taps(t):
    ct = t.get("chroma_taps")
    return (None, 0) if ct is None else (len(ct), int(np.abs(ct).sum()))


def _raster_tables(H, mode, prate):
    """The raster context's tables of a --pixelrate encoder: the mode at the pixel rate, without sound or filter."""
    return H.Tables(H.mode_config(mode, noaudio=True), prate)


def test_rows_are_what_they_state(built):
    H = built
    csat = {(kind, mode, rate, prate) for kind, mode, rate, prate, _ in CSAT}
    for kind, rows in (("composite", PS), ("s_video", S_VIDEO)):
        for mode, rate, kw, W, P, taps, kernel in rows:
            what = (kind, mode, rate, kw)
            t = H.Tables(H.mode_config(mode, **kw), rate)
            n, tap_sum = _taps(t)
            assert (int(t.get("geometry")[0]), int(t.get("comp_phases")[0]), n) == (W, P, taps), what
            t.close()
            assert (tap_sum > 32768) == ((kind, mode, rate, 0) in csat), (what, tap_sum)
            assert _plan_name(H, mode, rate, kw) == kernel, what
    for mode, rate, prate, kw, W, Wp, taps, kernel in PIXELRATE:
        what = (mode, rate, prate, kw)
        t = H.Tables(H.mode_config(mode, **kw), rate, prate)
        assert (int(t.get("geometry")[0]), int(t.get("rs_geometry")[3])) == (W, Wp), what
        t.close()
        r = _raster_tables(H, mode, prate)
        n, tap_sum = _taps(r)
        assert (int(r.get("geometry")[0]), n) == (Wp, taps), what
        r.close()
        assert (tap_sum > 32768) == (("pixelrate", mode, rate, prate) in csat), (what, tap_sum)
        assert _plan_name(H, mode, rate, kw, prate) == kernel, what


def test_rows_reach_every_low_rate_path(built):
    """1, 3, 5 and 7 chroma taps at the pixel rate; a 32-sample raster and others below 128; k_resample at I = 32 and
    D = 54; k_mod_mma on contiguous and pitched planes, k_mod_tma and k_mod behind k_resample; PS at 3, 5 and 7 taps and
    with CSAT; single-warp PS rows with and without S-Video; S-Video at 3, 5 and 7 taps, CSAT and single-warp, and
    SECAM's from 2 Msps."""
    H = built
    taps, wp, ratios, mods = set(), set(), set(), set()
    for mode, rate, prate, kw, W, Wp, n, kernel in PIXELRATE:
        taps.add(n)
        wp.add(Wp)
        g = H.Tables(H.mode_config(mode, **kw), rate, prate).get("rs_geometry")
        ratios.add((int(g[0]), int(g[1])))
        mods.add(kernel.split(" + ")[-1].split("<")[0] + ("-pitched" if "k_mod_mma" in kernel and W % 128 else ""))
    assert {1, 3, 5, 7} <= taps, taps
    assert 32 in wp and len({w for w in wp if w < 128}) >= 3, wp
    assert any(i == 32 for i, _ in ratios) and any(d == 54 for _, d in ratios), ratios
    assert mods == {"k_mod_mma", "k_mod_mma-pitched", "k_mod_tma", "k_mod"}, mods
    ps = [(taps, W, kernel) for *_, W, P, taps, kernel in PS if P == 0]
    assert {t for t, _, _ in ps} == {3, 5, 7} and any("CSAT=1" in k for *_, k in ps)
    assert any(W <= 128 for _, W, _ in ps)
    sv_ps = [(W, kernel) for *_, W, P, taps, kernel in S_VIDEO if P == 0]
    assert any(W <= 128 for W, _ in sv_ps) and any("CSAT=1" in k for _, k in sv_ps)
    sv = [(taps, W, kernel) for *_, W, P, taps, kernel in S_VIDEO]
    assert {t for t, _, _ in sv if t} == {3, 5, 7} and any("CSAT=1" in k for *_, k in sv)
    assert min(W for t, W, _ in sv if t) <= 128 and min(W for t, W, _ in sv if t is None) <= 128


def test_rows_are_pinned_to_the_reference(built):
    """The oracle each row is compared with is the reference there: the PS rows are in test_oracle_vs_ref.CASES and the
    --pixelrate rows in PIXELRATE_CASES, with the lines the device renders, and every S-Video row has the reference's
    stream in golden_s_video.json."""
    from test_gpu_zz_line_widths import _lines
    import test_oracle_vs_ref as T
    H = built
    for mode, rate, kw, *_ in PS:
        conf = H.mode_config(mode, **kw)
        assert (mode, rate, _lines(conf), bool(kw.get("vfilter")), ()) in T.CASES, (mode, rate)
    for mode, rate, prate, kw, *_ in PIXELRATE:
        conf = H.mode_config(mode, **kw)
        assert (mode, rate, prate, _lines(conf), bool(kw.get("vfilter")), ()) in T.PIXELRATE_CASES, (mode, rate, prate)
    golden = json.load(open(os.path.join(HERE, "golden", "golden_s_video.json")))
    have = {(c["mode"], c["rate"], c["lines"], c["filter"]) for c in golden["cases"] if c["source"] == "test" and not c["extra"]}
    for mode, rate, kw, *_ in S_VIDEO:
        lines = 1300 if H.mode_config(mode).lines == 625 else 1100
        assert (mode, rate, lines, bool(kw.get("vfilter"))) in have, (mode, rate)


def test_pixel_rate_raster_narrower_than_the_kernels_is_refused(built, capfd):
    """PAL at 2 Msps from 484 375 Hz: a 128-sample line from a 31-sample raster. The tables and the oracle take it;
    htv_init plans the raster context's kernels before it touches the device, and refuses it there, naming the raster."""
    H = built
    conf = H.mode_config("pal")
    t = H.Tables(conf, 2000000, 484375)
    assert (int(t.get("geometry")[0]), int(t.get("rs_geometry")[3])) == (128, 31)
    t.close()
    o = orc.Oracle(conf, 2000000, 484375)
    assert (o.width, o.raster_width) == (128, 31)
    o.close()
    assert _plan_name(H, "pal", 2000000, {}, 484375) == "k_raster + k_resample + k_mod_tma<256,4>"
    with pytest.raises(RuntimeError):
        H.Encoder(conf, 2000000, 484375)
    err = capfd.readouterr().err
    assert "the pixel-rate raster's line width 31 is below the kernels' 32-sample limit" in err, err
    assert "no CUDA device" not in err


@pytest.mark.parametrize("rate,start", [(4750000, 24), (4000000, 20), (2000000, 10)])
def test_secam_s_video_with_the_filter_below_5_msps_is_refused(built, rate, start):
    """S-Video filters I only, but SECAM's chain still runs only through a call's last line: the limit of SECAM with the
    video filter holds for S-Video too. At 5 Msps the row is selected."""
    H = built
    assert _plan_refusal(H, "secam", rate, SF) == "SECAM with the video filter needs the burst window to start 25 " \
        f"samples or more into the line (it starts at {start})"
    assert _plan_name(H, "secam", 5000000, SF).endswith(",SV>")
