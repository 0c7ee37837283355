"""S-Video (`--s-video`) without a GPU: sv_oracle.py against the reference's streams (golden_s_video.json, made by
tests/golden/make_golden_s_video.py), the configurations the encoder refuses, the line kernel the tables select for each
row of the device matrix (test_gpu_zz_s_video.py), and htv_cli's argument check."""
import ctypes as C
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import orc
import sv_oracle
from test_oracle_vs_ref import programme_source

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "golden_s_video.json")))
SV_MESSAGE = "S-Video is only available with PAL, SECAM, or NTSC baseband modes."


def _case_id(c):
    return "-".join([c["mode"], str(c["rate"]), "filter" if c["filter"] else "nofilter", c["source"]] + c["extra"])


def _conf(H, c):
    kw = dict(vfilter=c["filter"], s_video=True)
    it = iter(c["extra"])
    for e in it:
        if e == "--swap-iq": kw["swap_iq"] = True
        elif e == "--offset": kw["offset"] = int(next(it))
    return H.mode_config(c["mode"], **kw)


@pytest.mark.parametrize("case", GOLDEN["cases"], ids=[_case_id(c) for c in GOLDEN["cases"]])
def test_oracle_s_video_equals_reference(built, case):
    conf = _conf(built, case)
    source = None
    if case["source"] == "programme":
        o = orc.Oracle(conf, case["rate"])
        source = programme_source(GOLDEN["programme_seed"], o.active_lines, o.active_width)
        o.close()
    got = sv_oracle.render(conf, case["rate"], case["lines"], source)
    assert got.size == case["values"]
    assert hashlib.sha256(got.tobytes()).hexdigest() == case["sha256"]


def test_s_video_is_zero_in_every_mode(built):
    """s_video sits in htv_config_t's former padding word, which orc_params_t keeps as padding (reserved0)."""
    assert built.Config.s_video.offset == built.Config.fm_mono_preemph.offset + 4
    for mode in built.modes():
        assert built.mode_config(mode).s_video == 0, mode
    assert built.mode_config("pal", s_video=True).s_video == 1


@pytest.mark.parametrize("mode,kw,rate,prate,message", [
    ("i", {}, 16000000, 0, SV_MESSAGE),                                  # modulated, complex output
    ("pal", dict(nocolour=True), 16000000, 0, SV_MESSAGE),               # --nocolour --s-video
    ("pal-fm", {}, 16000000, 0, SV_MESSAGE),                             # FM video
    ("pal", {}, 16000000, 13500000, "--pixelrate with S-Video is not on the accelerated path"),
])
def test_unsupported_s_video_configs_are_refused(built, capfd, mode, kw, rate, prate, message):
    conf = built.mode_config(mode, s_video=True, **kw)
    L = built.lib()
    t = L.htv_tables_create2(C.byref(conf), rate, prate)
    assert not t
    assert message in capfd.readouterr().err


def _plan_refusal(H, mode, rate, kw, **env):
    """htv_dev_plan_name's message for a configuration the kernel selection refuses (plan_kernels, no GPU needed)."""
    from test_gpu_zz_line_widths import _env
    L = H.lib()
    L.htv_dev_plan_name.restype = C.c_int
    L.htv_dev_plan_name.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t]
    t = H.Tables(H.mode_config(mode, **kw), rate)
    buf = C.create_string_buffer(256)
    with _env(**env):
        r = L.htv_dev_plan_name(t._t, H.SAMPLE_TYPES["int16"], buf, len(buf))
    t.close()
    assert r == H.HTV_ERROR, buf.value.decode()
    return buf.value.decode()


def test_s_video_off_the_fused_line_kernels_is_refused(built):
    """At 1 Msps the chroma low-pass has a single tap and PAL runs on the split modulators, which have no S-Video form:
    the tables accept the configuration, the kernel selection refuses it and names the reason; so do the switches that
    select the split modulators or the scalar filters."""
    from test_tables_and_abi import _plan_name
    assert len(built.Tables(built.mode_config("pal", s_video=True), 1000000).get("chroma_taps")) == 1
    assert "k_mod" in _plan_name(built, "pal", 1000000, {})
    assert _plan_refusal(built, "pal", 1000000, dict(s_video=True)) == "S-Video runs on the fused line kernels only: " \
        "a chroma low-pass of 1 taps (k_line takes 3 .. 17) runs on the split modulators"
    assert _plan_refusal(built, "pal", 16000000, dict(s_video=True), HTV_PATH="split") == \
        "S-Video runs on the fused line kernels only: HTV_PATH=split selects the split modulators"
    assert _plan_refusal(built, "pal", 16000000, dict(s_video=True, vfilter=True), HTV_FIR="scalar") == \
        "S-Video runs on the fused line kernels only: HTV_FIR=scalar selects the scalar video filter"
    assert _plan_refusal(built, "secam", 16000000, dict(s_video=True), HTV_FIR="scalar") == \
        "S-Video runs on the fused line kernels only: HTV_FIR=scalar selects the scalar SECAM notch"


def test_s_video_matrix_selects_what_each_row_is_for(built):
    from test_gpu_zz_s_video import MATRIX
    from test_tables_and_abi import _plan_name
    for mode, rate, kw, W, kernel in MATRIX:
        assert int(built.Tables(built.mode_config(mode, **kw), rate).get("geometry")[0]) == W, (mode, rate)
        assert _plan_name(built, mode, rate, kw) == kernel, (mode, rate, kw)


def test_s_video_matrix_covers_every_form(built):
    """Every k_line class S-Video can select is a row: VF 0 / 1, FULL 0 / 1, CSAT, MAXT 256 / 320 / 384, SRC."""
    from test_gpu_zz_s_video import MATRIX
    import re
    seen = set()
    for *_, kernel in MATRIX:
        m = dict(re.findall(r"(VF|FULL|CSAT|MAXT|SRC)=(\d+)", kernel.split("k_line")[-1]))
        assert kernel.endswith(",SV>")
        seen |= {(k, v) for k, v in m.items()}
    for k, vs in (("VF", "01"), ("FULL", "01"), ("CSAT", "01"), ("SRC", "01")):
        for v in vs:
            assert (k, v) in seen, (k, v)
    for t in ("256", "320", "384"):
        assert ("MAXT", t) in seen


def _cli(built, *args):
    exe = os.path.join(os.path.dirname(built.LIB_PATH), "htv_cli")
    return subprocess.run([exe, *args], capture_output=True, text=True, timeout=60)


@pytest.mark.parametrize("args", [
    ("-m", "i", "--s-video"),
    ("-m", "pal", "--nocolour", "--s-video"),
    ("-m", "pal-fm", "--s-video"),
    ("-m", "l", "--s-video"),
])
def test_cli_refuses_s_video_outside_baseband_colour(built, args):
    r = _cli(built, *args, "-o", os.devnull, "--lines", "1", "test")
    assert r.returncode != 0
    assert SV_MESSAGE in r.stderr
    assert "initialise" not in r.stderr             # refused by the argument check, before the encoder


def test_cli_lists_s_video(built):
    r = _cli(built, "--help")
    assert "--s-video" in r.stderr
