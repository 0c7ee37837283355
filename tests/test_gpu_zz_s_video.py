"""S-Video (`--s-video`) on the device: luma and sync on I, the colour subcarrier and its burst on Q, for the PAL, NTSC
and SECAM baseband modes, against sv_oracle.py (the parity oracle's streams composed into S-Video's, pinned to the
reference by test_s_video_host.py).

MATRIX covers every k_line form S-Video can select - VF 0 / 1, FULL 0 / 1, CSAT, MAXT 256 / 320 / 384 and the SECAM SRC
form - at the widths that select each; every row states the W it exists for and the `line_kernel` string it must run
(",SV": the S-Video form ran), and is bit-exact over two frames and a few lines: burst-phase codes, PAL's V-switch and
SECAM's D'r / D'b alternation depend on frame parity. test_s_video_host.py checks the same strings against the kernel
selection without a GPU. The baseband modes have no sound carriers; --offset rows are within +-1 LSB as the other
offset cases are."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import sv_oracle
from test_gpu_zz_line_widths import _render, kl, sec

pytestmark = pytest.mark.gpu


def sv(kernel):
    return kernel[:-1] + ",SV>"


S = dict(s_video=True)
SF = dict(s_video=True, vfilter=True)
# (mode, rate, overrides, W, line_kernel); W % 128 is the last tile's width where it is not 0
MATRIX = [
    ("pal", 16000000, S, 1024, sv(kl(0, 0, 1, 0, 256))),
    ("pal", 16000000, SF, 1024, sv(kl(1, 0, 1, 0, 256))),
    ("pal", 20000000, S, 1280, sv(kl(0, 0, 1, 0, 320))),
    ("pal", 20000000, SF, 1280, sv(kl(1, 0, 1, 0, 320))),
    ("pal", 17734475, S, 1135, sv(kl(0, 0, 0, 1, 320))),            # 4 x the PAL subcarrier: chroma taps sum to 32769
    ("pal", 17734475, SF, 1135, sv(kl(1, 0, 0, 1, 320))),
    ("pal", 20050000, S, 1283, sv(kl(0, 0, 0, 1, 384))),            # last tile 3, CSAT
    ("pal", 20050000, SF, 1283, sv(kl(1, 0, 0, 1, 384))),
    ("pal", 20250000, SF, 1296, sv(kl(1, 0, 0, 0, 384))),           # last tile 16
    ("pal", 22000000, SF, 1408, sv(kl(1, 0, 1, 0, 384))),
    ("ntsc", 13500000, S, 858, sv(kl(0, 0, 0, 0, 256))),            # last tile 90
    ("ntsc", 13500000, SF, 858, sv(kl(1, 0, 0, 0, 256))),
    ("ntsc", 18000000, SF, 1144, sv(kl(1, 0, 0, 0, 320))),          # last tile 120
    ("525pal", 13500000, S, 858, sv(kl(0, 0, 0, 0, 256))),
    ("pal60", 13500000, SF, 858, sv(kl(1, 0, 0, 0, 256))),
    # SECAM: k_sec_raster (no luma notch) + chain (Q plane) + k_line<SRC=1>
    ("secam", 16000000, S, 1024, sv(sec(0, 0, 1, 256))),
    ("secam", 16000000, SF, 1024, sv(sec(1, 0, 1, 256))),
    ("secam", 13500000, SF, 864, sv(sec(1, 0, 0, 256))),
    ("secam", 17500000, S, 1120, sv(sec(0, 0, 0, 320))),
    ("secam", 20000000, SF, 1280, sv(sec(1, 0, 1, 320))),
    ("secam", 20250000, SF, 1296, sv(sec(1, 0, 0, 384))),
    ("secam", 24000000, S, 1536, sv(sec(0, 0, 1, 384))),
]


def case_id(c):
    mode, rate, kw, W, _ = c
    return f"{mode}-{rate}-W{W}" + ("-filter" if kw.get("vfilter") else "")


def _nlines(conf):
    return 1300 if conf.lines == 625 else 1100


@pytest.mark.parametrize("mode,rate,kw,W,kernel", MATRIX, ids=[case_id(c) for c in MATRIX])
def test_s_video_forms_against_the_oracle(built, mode, rate, kw, W, kernel):
    H = built
    conf = H.mode_config(mode, **kw)
    n = _nlines(conf)
    got, name = _render(H, conf, rate, [n])
    assert name == kernel, f"{mode} {rate} ran {name}, the row exists for {kernel}"
    assert got.size == n * W * 2
    want = sv_oracle.render(conf, rate, n)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} values differ, first at line {bad[0] // (2 * W)}, {'IQ'[bad[0] % 2]}"


@pytest.mark.parametrize("mode,rate,kw,tol", [
    ("pal", 16000000, dict(s_video=True, swap_iq=True), 0),
    ("pal", 16000000, dict(s_video=True, offset=2000000), 1),
    ("ntsc", 13500000, dict(s_video=True, vfilter=True, offset=-1500000), 1),
    ("secam", 16000000, dict(s_video=True, vfilter=True, swap_iq=True, offset=2000000), 1),
])
def test_s_video_mixers_act_on_the_luma_chroma_pair(built, mode, rate, kw, tol):
    H = built
    conf = H.mode_config(mode, **kw)
    n = _nlines(conf)
    got, name = _render(H, conf, rate, [n])
    assert name.endswith(",SV>")
    d = np.abs(got.astype(np.int32) - sv_oracle.render(conf, rate, n).astype(np.int32))
    assert d.max() <= tol, f"max |diff| {d.max()}, {np.count_nonzero(d > tol)} values over {tol}"


@pytest.mark.parametrize("mode,rate", [("pal", 16000000), ("ntsc", 13500000), ("pal60", 13500000)])
def test_q_carries_the_chroma(built, mode, rate):
    """Without a video filter I + Q (int16 wrap) is the composite stream, and Q is not zero on the colour lines."""
    H = built
    n = _nlines(H.mode_config(mode))
    got, _ = _render(H, H.mode_config(mode, s_video=True), rate, [n])
    composite, name = _render(H, H.mode_config(mode), rate, [n])
    assert ",SV" not in name
    iq = got.reshape(-1, 2)
    assert np.array_equal((iq[:, 0].astype(np.int32) + iq[:, 1]).astype(np.int16), composite)
    W = composite.size // n
    q = iq[:, 1].reshape(n, W)
    assert np.count_nonzero(q.any(axis=1)) > n // 2
    assert not np.array_equal(iq[:, 0], composite)


@pytest.mark.parametrize("mode,kw,env", [
    ("pal", SF, {}),
    ("ntsc", S, {}),
    ("secam", SF, dict(HTV_SEC="sub=64")),               # chain launches of 64 lines: the calls cut across them
    ("secam", S, dict(HTV_SEC="sub=64")),
])
def test_uneven_calls_give_the_one_call_stream(built, mode, kw, env):
    H = built
    rate = 13500000 if mode == "ntsc" else 16000000
    conf = H.mode_config(mode, **kw)
    pieces = [1, 2, 311, 1000, 7, 579]
    whole, _ = _render(H, conf, rate, [sum(pieces)])
    parts, name = _render(H, conf, rate, pieces, **env)
    assert name.endswith(",SV>")
    assert np.array_equal(whole, parts), f"{np.count_nonzero(whole != parts)} values differ"


@pytest.mark.parametrize("mode", ["pal", "secam"])
def test_next_line_equals_render(built, mode):
    H = built
    conf = H.mode_config(mode, **SF)
    n = 700
    want, _ = _render(H, conf, 16000000, [n])
    enc = H.Encoder(conf, 16000000)
    enc.open_test_source()
    lines = []
    for k in range(n):
        out, frame, line = enc.next_line()
        assert (frame, line) == (k // enc.lines + 1, k % enc.lines + 1)
        lines.append(out)
    enc.close()
    assert np.array_equal(np.concatenate(lines), want)


@pytest.mark.parametrize("mode,sample_type", [("pal", "int8"), ("pal", "float"), ("secam", "int8"), ("ntsc", "float")])
def test_sample_types_equal_the_converted_int16_stream(built, mode, sample_type):
    import torch
    H = built
    rate = 13500000 if mode == "ntsc" else 16000000
    conf = H.mode_config(mode, **SF)
    n = 700
    ref, _ = _render(H, conf, rate, [n])
    enc = H.Encoder(conf, rate)
    enc.open_test_source()
    enc.set_sample_type(sample_type)
    got = enc.render_host(n)
    name = enc.line_kernel
    enc.close()
    assert name.endswith(f",ST=-1:{sample_type},SV>")
    src = torch.from_numpy(ref).cuda()
    dst = torch.empty(ref.size, dtype={"int8": torch.int8, "float": torch.float32}[sample_type], device="cuda")
    H.convert(dst.data_ptr(), sample_type, src.data_ptr(), ref.size, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(got, dst.cpu().numpy())


def test_render_add_of_two_s_video_encoders_is_their_sum(built):
    import torch
    H = built
    a_conf, b_conf = H.mode_config("pal", **SF), H.mode_config("pal", s_video=True, offset=3000000)
    n = 900
    a_host, _ = _render(H, a_conf, 16000000, [n])
    b_host, _ = _render(H, b_conf, 16000000, [n])
    buf = torch.zeros(a_host.size, dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    for conf in (a_conf, b_conf):
        e = H.Encoder(conf, 16000000)
        e.open_test_source()
        e.render_add(n, buf.data_ptr(), st)
        torch.cuda.synchronize()
        e.close()
    assert np.array_equal(buf.cpu().numpy(), (a_host.astype(np.int32) + b_host).astype(np.int16))


@pytest.mark.parametrize("kw", [S, SF])
def test_vbi_overlays_land_on_i_only(built, kw):
    """A WSS-like line 23 (part of it set to black, then data added) and VITS-like test lines: I changes and equals the
    oracle with the same overlays, Q is the stream without them."""
    H = built
    conf = H.mode_config("pal", **kw)
    n = 1300
    enc = H.Encoder(conf, 16000000)
    W = enc.width
    ov = []
    for line, rep in ((23, (W // 2, int(W * 0.66), 1234)), (17, (0, 0, 0)), (330, (0, 0, 0))):
        add = np.zeros(W, dtype=np.int16)
        add[150: W - 60] = (np.sin(np.arange(W - 210) * 0.3) * 8000).astype(np.int16)
        ov.append((line, add, rep))
    enc.open_test_source()
    enc.set_vbi_lines(ov)
    got = enc.render_host(n)
    enc.close()
    want = sv_oracle.render(conf, 16000000, n, overlays=ov)
    plain, _ = _render(H, conf, 16000000, [n])
    assert np.array_equal(got, want)
    g, p = got.reshape(-1, 2), plain.reshape(-1, 2)
    assert np.array_equal(g[:, 1], p[:, 1])
    assert np.count_nonzero(g[:, 0] != p[:, 0]) > 1000


def test_cli_file_equals_the_reference_file(built, tmp_path):
    """htv_cli --s-video writes the file hacktv writes: I,Q interleaved, byte for byte the reference's over 2 500 lines
    (its sha256 in golden_s_video.json)."""
    H = built
    out = tmp_path / "out.bin"
    exe = os.path.join(os.path.dirname(H.LIB_PATH), "htv_cli")
    subprocess.run([exe, "-m", "pal", "-s", "16000000", "--s-video", "--filter", "-o", str(out), "--lines", "2500", "test"],
                   check=True, capture_output=True, timeout=300)
    golden = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_s_video.json")))
    want = next(c for c in golden["cases"] if (c["mode"], c["rate"], c["lines"], c["filter"], c["extra"], c["source"]) ==
                ("pal", 16000000, 2500, True, [], "test"))
    data = out.read_bytes()
    assert len(data) == 2 * want["values"] == 2500 * 1024 * 4
    assert hashlib.sha256(data).hexdigest() == want["sha256"]


def test_s_video_encoder_beside_a_plain_encoder_of_the_same_kernel(built):
    """An S-Video encoder asks its k_line instantiation for more shared memory than a plain encoder of the same one: a
    plain encoder created after it must not take that away (the limit is the function's, shared by the process)."""
    H = built
    conf = H.mode_config("pal", s_video=True)
    want, _ = _render(H, conf, 16000000, [700])
    enc = H.Encoder(conf, 16000000)
    plain = H.Encoder(H.mode_config("pal"), 16000000)
    enc.open_test_source()
    plain.open_test_source()
    got = enc.render_host(700)
    plain.render_host(1)
    assert enc.line_kernel == sv(plain.line_kernel)
    enc.close()
    plain.close()
    assert np.array_equal(got, want)
