"""Host logic without a GPU: the product's table generation against the oracle's and
against the reference's known-answer values (SURVEY.md §9.2), the test source, and the
C-ABI surface (every symbol the header declares is exported; no compute is attempted)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLES = ["sync0", "sync1", "sync2", "sync3", "sync4", "sync_off", "burst_win", "chroma_taps", "vsb_itaps",
          "vsb_qtaps", "levels", "nicam_taps", "geometry", "secam_lpf", "secam_notch"]
MODES = [("i", 16000000, True), ("pal", 16000000, False), ("m", 13500000, True), ("l", 16000000, True),
         ("i", 20000000, True), ("b", 16000000, True), ("ntsc", 13500000, False), ("pal", 16000000, True),
         ("pal-n", 16000000, True), ("secam", 16000000, False), ("pal60", 13500000, False)]


@pytest.mark.parametrize("mode,rate,filt", MODES)
def test_product_tables_equal_oracle_tables(built, mode, rate, filt):
    conf = built.mode_config(mode, vfilter=filt)
    t, o = built.Tables(conf, rate), orc.Oracle(conf, rate)
    for name in TABLES:
        a, b = t.get(name), o.table(name)
        assert (a is None) == (b is None), name
        if a is not None:
            assert a.shape == b.shape and np.array_equal(a, b), name
    t.close(); o.close()


def test_known_answers_pal_i_16M(built):
    """Values dumped from the reference's vid_init (SURVEY.md §9.2)."""
    t = built.Tables(built.mode_config("i", vfilter=True), 16000000)
    assert list(t.get("geometry")) == [1024, 512, 166, 832, 87, 46]
    assert list(t.get("levels")) == [4653, 17681, 17681, 23265]
    assert list(t.get("sync0")[:8]) == [94, 558, 1508, 2791, 4075, 5025, 5489, 5583]
    assert list(t.get("sync0")[-4:]) == [1747, 711, 150, 3] and len(t.get("sync0")) == 83
    assert list(t.get("sync_off")) == [-3, -3, -3, 509, 509]
    assert [len(t.get(f"sync{i}")) for i in range(5)] == [83, 45, 444, 45, 444]
    assert list(t.get("chroma_taps")) == [3, 34, 249, 1179, 3583, 6978, 8715, 6978, 3583, 1179, 249, 34, 3]
    bw = t.get("burst_win")
    assert list(bw[:10]) == [0, -18, -138, -420, -865, -1409, -1950, -2388, -2663, -2776] and bw[20] == -2792
    assert list(t.get("vsb_itaps")[:26]) == [-1, 1, -8, -12, 3, -23, -3, 61, 3, 74, 165, -46, 46, 64, -431, -182,
                                              -151, -792, 153, 416, -317, 1956, 1975, -236, 6759, 13824]
    assert list(t.get("vsb_qtaps")[:26]) == [2, 2, -3, 7, -12, -34, 0, -50, -57, 74, -8, 56, 310, 43, 108, 340,
                                              -422, -328, -72, -1370, -529, 389, -1464, 2396, 7458, 0]
    nt = t.get("nicam_taps")
    assert len(nt) == 221 and list(nt[107:114]) == [1013, 1024, 1030, 1033, 1030, 1024, 1013] and list(nt[:3]) == [1, 1, 1]


def test_known_answers_ntsc_and_secam(built):
    t = built.Tables(built.mode_config("m", vfilter=True), 13500000)
    assert list(t.get("chroma_taps")) == [4, 70, 622, 2963, 7559, 10329, 7559, 2963, 622, 70, 4]
    assert list(t.get("burst_win")[:9]) == [0, -34, -250, -734, -1427, -2160, -2742, -3063, -3152]
    assert list(t.get("levels")) == [3154, 17740, 18923, 25231]
    t = built.Tables(built.mode_config("l", vfilter=True), 16000000)
    assert list(t.get("geometry"))[4:] == [82, 944]
    assert list(t.get("burst_win")[:10]) == [0, 6, 47, 157, 367, 705, 1195, 1854, 2693, 3719]
    assert list(t.get("secam_lpf")[:8]) == [-9, -68, -64, 400, 1810, 4138, 6456, 7440]
    assert list(t.get("secam_notch")[23:28]) == [4657, 680, 27307, 680, 4657]
    assert list(t.get("levels")) == [21140, 6342, 6342, 1057]


def test_known_answers_yuv(built):
    o = orc.Oracle(built.mode_config("i"), 16000000)
    for rgb, want in {0x000000: (17681, 0, 0), 0xFFFFFF: (4653, 0, 0), 0xBF0000: (14763, 1438, -5999),
                      0x00BF00: (11953, 2824, 5024), 0x0000BF: (16569, -4262, 976), 0x808080: (11141, 0, 0)}.items():
        assert tuple(o.yuv(rgb)) == want
    o.close()


def test_test_source_matches_oracle(built):
    for w, h in ((832, 576), (1039, 576), (715, 480)):
        assert np.array_equal(built.test_pattern(w, h), orc.test_pattern(w, h))
    assert np.array_equal(built.test_tone(), orc.test_tone())
    tone = built.test_tone()
    assert tone.shape == (204800, 2) and not tone[:20480, 0].any() and tone[1:20480, 1].any()


def test_mode_table(built):
    m = built.modes()
    for want in ("i", "pal", "l", "m", "b", "g", "ntsc", "secam", "pal-m", "pal-n"):
        assert want in m
    c, desc = m["i"]
    assert c.lines == 625 and c.colour_mode == 1 and c.modulation == 2 and c.fm_mono_carrier == 5999600
    assert "6.0 MHz FM audio" in desc
    assert m["m"][0].nicam_carrier == 0 and m["l"][0].am_mono_carrier == 6500000


def test_abi_exports_every_declared_symbol(built):
    hdr = open(os.path.join(ROOT, "include", "hacktv_b200.h")).read()
    names = set(re.findall(r"extern\s+[^;(]*?\b(htv_[a-z0-9_]+)\s*\(", hdr)) | {"htv_modes"}
    assert len(names) > 30
    L = C.CDLL(built.LIB_PATH)
    missing = [n for n in sorted(names) if not hasattr(L, n)]
    assert not missing, missing
    assert built.lib().htv_config_size() == C.sizeof(built.Config) == orc.lib().orc_params_size()


def test_product_never_links_the_oracle(built):
    import subprocess
    out = subprocess.run(["ldd", built.LIB_PATH], capture_output=True, text=True).stdout
    assert "oracle" not in out
    nm = subprocess.run(["nm", "-D", built.LIB_PATH], capture_output=True, text=True).stdout
    assert " orc_" not in nm


def test_unsupported_configs_fail_loudly(built):
    conf = built.mode_config("pal-fm")
    conf.fm_energy_dispersal = 0.0625    # FM energy dispersal: not on the accelerated path
    with pytest.raises(RuntimeError):
        built.Tables(conf, 20000000)
    conf = built.mode_config("i")
    conf.type = 3                # 819-line raster
    with pytest.raises(RuntimeError):
        built.Tables(conf, 16000000)


def test_encoder_needs_a_gpu_or_says_so(built):
    """No CPU fallback: on a box without CUDA, construction fails with an error."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(RuntimeError):
        built.Encoder("i", 16000000)


def test_fm_video_tables_match_the_oracle(built):
    """FM video (ref video.c:3678-3740, 4564-4570): pre-emphasis taps per sample rate."""
    for mode, rate, n in (("pal-fm", 20000000, 67), ("pal-fm", 20250000, 67), ("pal-fm", 14000000, 67),
                          ("ntsc-fm", 18000000, 67), ("ntsc-fm", 20250000, 71)):   # 28 Msps: line wider than the kernels' 1536
        conf = built.mode_config(mode, vfilter=True)
        t = built.Tables(conf, rate)
        o = orc.Oracle(conf, rate)
        a, b = t.get("fmv_taps"), o.table("vsb_itaps")
        assert a is not None and len(a) == n and np.array_equal(a, b), (mode, rate)
        o.close()


@pytest.mark.parametrize("mode,rate,prate,filt", [("i", 16000000, 13500000, True), ("i", 20000000, 13500000, False),
                                                  ("i", 13500000, 16000000, True), ("m", 13500000, 9000000, True),
                                                  ("i", 16000000, 14000000, True), ("l", 16000000, 13500000, True)])
def test_pixelrate_resampler_tables_equal_the_oracle(built, mode, rate, prate, filt):
    """htv_tables_create2: the --pixelrate resampler's polyphase taps and geometry (ref fir.c:263-295,
    393-428) against the oracle, which is pinned to the reference's --pixelrate output."""
    import orc
    conf = built.mode_config(mode, vfilter=filt)
    t = built.Tables(conf, rate, prate)
    o = orc.Oracle(conf, rate, prate)
    assert np.array_equal(t.get("rs_taps"), o.table("rs_taps"))
    g, og = t.get("rs_geometry"), o.table("rs_geometry")
    assert np.array_equal(g[:4], og)
    assert g[4] == (2 if filt else 1) * o.width          # sound carriers, offset mixer, passthru: lines of lead
    plain = built.Tables(conf, rate)
    for name in ("vsb_itaps", "vsb_qtaps", "nicam_taps", "levels"):
        a, b = t.get(name), plain.get(name)
        assert (a is None and b is None) or np.array_equal(a, b)
    t.close(); o.close(); plain.close()


def test_pixelrate_pairs_that_are_refused(built):
    with pytest.raises(RuntimeError):
        built.Tables(built.mode_config("i"), 16000000, 13400000)             # line width would vary
    with pytest.raises(RuntimeError):
        built.Tables(built.mode_config("pal-fm"), 20000000, 13500000)        # FM video
    t = built.Tables(built.mode_config("i"), 16000000, 16000000)             # no resampler at all
    assert t.get("rs_taps") is None
    t.close()


def _line_kernel_from_tables(H, mode, rate, kw):
    """The line kernel htv_dev_create / htv_dev_render_lines select for an encoder, from its tables alone, with the
    facts the selection rests on: W, its tiles of 128 samples, the last tile's width and the chroma taps' sum."""
    conf = H.mode_config(mode, **kw)
    t = H.Tables(conf, rate)
    W = int(t.get("geometry")[0])
    ct = t.get("chroma_taps")
    vf, hq = int(t.get("vsb_itaps") is not None), int(t.get("vsb_qtaps") is not None)
    t.close()
    tiles = -(-W // 128)
    maxt = 256 if tiles <= 8 else 320 if tiles <= 10 else 384
    tap_sum = 0 if ct is None else int(np.abs(ct).sum())
    if conf.colour_mode == 3:                                   # SECAM: no chroma low-pass in the line kernel
        full = int(W % 128 == 0)
        return W, tiles, W % 128, tap_sum, f"k_sec_raster<FULL={full},MAXT={maxt}> + " + \
            f"k_line<VF={vf},HQ={hq},FULL={full},CSAT=0,MAXT={maxt},SRC=1,SND=-1,WC=0>"
    assert conf.colour_mode == 0 or 3 <= len(ct) <= 17, "the chroma low-pass does not fit the line kernel"
    csat = int(tap_sum > 32768)
    full = int(W % 128 == 0 and not csat)
    return W, tiles, W % 128, tap_sum, f"k_line<VF={vf},HQ={hq},FULL={full},CSAT={csat},MAXT={maxt},SRC=0,SND=-1,WC=0>"


def test_line_width_matrix_selects_what_each_case_is_for(built):
    """The GPU line-width matrix (test_gpu_zz_line_widths.py) without a GPU: every case's W, tile count, last tile and
    chroma saturation condition are what the tables give, and the instantiation it names is the one they select."""
    from test_gpu_zz_line_widths import MATRIX
    for mode, rate, kw, W, kernel in MATRIX:
        w, tiles, residue, tap_sum, sel = _line_kernel_from_tables(built, mode, rate, kw)
        what = f"{mode} {rate} {kw}"
        assert w == W, (what, w)
        assert f"MAXT={256 if tiles <= 8 else 320 if tiles <= 10 else 384}" in kernel and tiles <= 12, (what, tiles)
        assert ("CSAT=1" in kernel) == (tap_sum > 32768), (what, tap_sum)
        assert ("FULL=1" in kernel) == (residue == 0 and tap_sum <= 32768), (what, residue)
        assert sel == kernel, (what, sel)


def test_line_width_matrix_covers_every_instantiation(built):
    """Together the matrix and the compiled-in sound form run every k_line and k_sec_raster instantiation
    htv_dev_create sets up: VF / HQ x {FULL, partial, CSAT} x MAXT, the SECAM SRC form's VF / HQ x FULL x MAXT and its
    raster's FULL x MAXT (SECAM has no chroma low-pass here, so no CSAT form), and the 16 Msps form with PAL's sound
    stages compiled in. No instantiation is unreachable from the modes and rates the tables accept."""
    from test_gpu_zz_line_widths import FIXED, MATRIX
    kl = "k_line<VF={},HQ={},FULL={},CSAT={},MAXT={},SRC={},SND=-1,WC=0>"
    want = {FIXED}
    for maxt in (256, 320, 384):
        for vf, hq in ((0, 0), (1, 0), (1, 1)):
            for full, csat in ((1, 0), (0, 0), (0, 1)):
                want.add(kl.format(vf, hq, full, csat, maxt, 0))
            for full in (0, 1):
                want.add(kl.format(vf, hq, full, 0, maxt, 1))
        for full in (0, 1):
            want.add(f"k_sec_raster<FULL={full},MAXT={maxt}>")
    ran = {FIXED} | {part for c in MATRIX for part in c[4].split(" + ")}
    assert not want - ran, sorted(want - ran)
    assert not ran - want, sorted(ran - want)


def _plan_name(H, mode, rate, kw, prate=0, sample_type="int16", **env):
    """htv_dev_plan_name: the line kernel(s) the C selection (plan_kernels in htv_kernels.cu, the code htv_dev_create
    runs) picks for an encoder of these tables writing this sample type, under the switches in `env`. No GPU needed."""
    from test_gpu_zz_line_widths import _env
    L = H.lib()
    L.htv_dev_plan_name.restype = C.c_int
    L.htv_dev_plan_name.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t]
    t = H.Tables(H.mode_config(mode, **kw), rate, prate)
    buf = C.create_string_buffer(256)
    with _env(**env):
        r = L.htv_dev_plan_name(t._t, H.SAMPLE_TYPES[sample_type], buf, len(buf))
    t.close()
    assert r == H.HTV_OK, buf.value.decode()
    return buf.value.decode()


def test_c_selection_runs_what_the_line_width_matrix_asserts(built):
    """The C selection itself names, for every case of the GPU line-width matrix, the instantiation the case asserts the
    encoder ran; so does it for the form with PAL's sound stages compiled in, and the general form under HTV_KL=general."""
    from test_gpu_zz_line_widths import FIXED, GENERAL, MATRIX
    for mode, rate, kw, _, kernel in MATRIX:
        assert _plan_name(built, mode, rate, kw) == kernel, (mode, rate, kw)
    for mode in ("i", "b"):
        assert _plan_name(built, mode, 16000000, dict(vfilter=True)) == FIXED
        assert _plan_name(built, mode, 16000000, dict(vfilter=True), HTV_KL="general") == GENERAL


def test_c_selection_runs_what_the_sample_type_cases_assert(built):
    """Every case of the GPU sample-type test, for each type: the names it asserts (the split modulators, FM video and
    --pixelrate among them), and the int8 form with PAL's sound stages compiled in, or the general one under HTV_KL=general."""
    from test_gpu_zz_sample_types import CASES, FIXED_INT8, TYPES
    for case, (mode, rate, prate, kw, env, _, kernel) in sorted(CASES.items()):
        for st in TYPES:
            name = _plan_name(built, mode, rate, kw, prate, st, **env)
            want = FIXED_INT8 if st == "int8" and case in ("i-16M-filter", "i-16M-filter-passthru") else kernel
            assert want.format(st=st) in name, (case, st, name)
            if "k_line" in want:
                assert name == want.format(st=st), (case, st, name)
            else:
                assert f"ST=-1:{st}" in name, (case, st, name)
    assert _plan_name(built, "i", 16000000, dict(vfilter=True), sample_type="int8") == FIXED_INT8
    assert _plan_name(built, "i", 16000000, dict(vfilter=True), sample_type="int8", HTV_KL="general") == \
        "k_line<VF=1,HQ=1,FULL=1,CSAT=0,MAXT=256,SRC=0,SND=-1,WC=0,ST=-1:int8>"


def test_c_selection_of_the_scalar_video_filter(built):
    """HTV_FIR=scalar: PAL-I falls back to the split kernels with the TMA-fed modulator, SECAM keeps k_line<SRC> behind
    the raster with the scalar notch."""
    F = dict(vfilter=True)
    assert _plan_name(built, "i", 16000000, F, HTV_FIR="scalar") == "k_raster + k_mod_tma<256,4>"
    assert _plan_name(built, "l", 16000000, F, HTV_FIR="scalar") == \
        "k_raster_secam + k_line<VF=1,HQ=1,FULL=1,CSAT=0,MAXT=256,SRC=1,SND=-1,WC=0>"
