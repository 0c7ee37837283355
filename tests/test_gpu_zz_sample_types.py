"""Sample types on the device (htv_set_sample_type, htv_convert, htv_cli -t): hacktv's file sink types (ref rf_file.c,
-t/--type) written by the line kernels' stores.

- Every store site and every instantiation that converts: each non-int16 type, rendered through htv_render (device)
  and htv_render_host with uneven calls, must equal htv_convert of the int16 stream of an identical encoder, bit for
  bit. Each case asserts the line kernel it exists for.
- htv_convert over every int16 value against the digests pinned from the reference's own rf_file.o.
- htv_cli -t T against the stock hacktv -t T.
- The refusals: htv_render_add, htv_next_line, a late htv_set_sample_type, an unknown type."""
import contextlib
import hashlib
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "hacktv_b200", "htv_cli")
STOCK = os.path.join(ROOT, "oracle", "_ref", "hacktv_ref")
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "golden_sample_types.json")))["streams"]
TYPES = ("uint8", "int8", "uint16", "int32", "float")
PIECES = (37, 300, 563)                       # uneven calls, 900 lines: more than one frame of either raster

pytestmark = pytest.mark.gpu

F = dict(vfilter=True)
# id: (mode, rate, pixel_rate, overrides, env, passthru, the line kernel, with {st} for the type's part)
KL = "k_line<VF={},HQ={},FULL={},CSAT={},MAXT={},SRC={},SND=-1,WC=0,ST=-1:{{st}}>"
CASES = {
    "i-16M-filter": ("i", 16000000, 0, F, {}, False, KL.format(1, 1, 1, 0, 256, 0)),
    "pal-16M-real": ("pal", 16000000, 0, {}, {}, False, KL.format(0, 0, 1, 0, 256, 0)),
    "m-13M5-filter-W858": ("m", 13500000, 0, F, {}, False, KL.format(1, 1, 0, 0, 256, 0)),
    "ntsc-13M5-real-W858": ("ntsc", 13500000, 0, {}, {}, False, KL.format(0, 0, 0, 0, 256, 0)),
    "i-20M25-filter-384": ("i", 20250000, 0, F, {}, False, KL.format(1, 1, 0, 0, 384, 0)),
    "i-17M73-filter-csat": ("i", 17734475, 0, F, {}, False, KL.format(1, 1, 0, 1, 320, 0)),
    "l-16M-filter-secam": ("l", 16000000, 0, F, {}, False, "k_sec_raster<FULL=1,MAXT=256> + " + KL.format(1, 1, 1, 0, 256, 1)),
    "secam-W967-real": ("secam", 15109375, 0, {}, {}, False, "k_sec_raster<FULL=0,MAXT=256> + " + KL.format(0, 0, 0, 0, 256, 1)),
    "pal-fm-20M-filter": ("pal-fm", 20000000, 0, F, {}, False, "k_fmv_base<"),
    "i-16M-pixelrate-13M5": ("i", 16000000, 13500000, F, {}, False, "k_raster + k_resample + "),
    "i-13M5-pixelrate-16M-W864": ("i", 13500000, 16000000, F, {}, False, "k_raster + k_resample + k_mod_mma"),   # pitched
    "i-16M-filter-split": ("i", 16000000, 0, F, {"HTV_PATH": "split"}, False, "k_raster + k_mod"),
    "ntsc-13M5-real-split-W858": ("ntsc", 13500000, 0, {}, {"HTV_PATH": "split"}, False, "k_raster + k_mod"),
    "i-16M-filter-offset-swap": ("i", 16000000, 0, dict(vfilter=True, offset=1250000, swap_iq=True), {}, False, KL.format(1, 1, 1, 0, 256, 0)),
    "i-16M-filter-passthru": ("i", 16000000, 0, F, {}, True, KL.format(1, 1, 1, 0, 256, 0)),
}

FIXED_INT8 = "k_line<VF=1,HQ=1,FULL=1,CSAT=0,MAXT=256,SRC=0,SND=37,WC=1024,ST=int8>"


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


def _encoder(H, case, sample_type):
    mode, rate, prate, kw, env, passthru, _ = CASES[case]
    with _env(**env):
        enc = H.Encoder(H.mode_config(mode, **kw), rate, prate)
    enc.open_test_source()
    if passthru:
        rng = np.random.default_rng(7)
        enc.set_passthru(rng.integers(-8000, 8000, size=(sum(PIECES) + 4) * enc.width * 2, dtype=np.int16).reshape(-1, 2))
    if sample_type != "int16":
        enc.set_sample_type(sample_type)
    return enc


def _convert(H, x: np.ndarray, sample_type: str) -> bytes:
    """htv_convert of an int16 array, through device memory"""
    import torch
    src = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    size = np.dtype(H.SAMPLE_DTYPES[sample_type]).itemsize
    dst = torch.empty(x.size * size + 16, dtype=torch.uint8, device="cuda")
    H.convert(dst.data_ptr(), sample_type, src.data_ptr(), x.size, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return dst[:x.size * size].cpu().numpy().tobytes()


_int16 = {}


def _int16_stream(H, case):
    if case not in _int16:
        enc = _encoder(H, case, "int16")
        _int16[case] = enc.render_host(sum(PIECES)).copy()
        enc.close()
    return _int16[case]


@pytest.mark.parametrize("sample_type", TYPES)
@pytest.mark.parametrize("case", sorted(CASES))
def test_typed_output_is_the_converted_int16_output(built, case, sample_type):
    import torch
    H = built
    want = _convert(H, _int16_stream(H, case), sample_type)
    kernel = CASES[case][6]

    # htv_render_host
    enc = _encoder(H, case, sample_type)
    assert enc.sample_type == sample_type
    per = 2 if enc.complex else 1
    size = np.dtype(H.SAMPLE_DTYPES[sample_type]).itemsize
    assert enc.bytes_per_sample == per * size
    parts = [enc.render_host(n) for n in PIECES]
    assert all(p.dtype == H.SAMPLE_DTYPES[sample_type] for p in parts)
    host = b"".join(p.tobytes() for p in parts)
    name = enc.line_kernel
    enc.close()

    # htv_render into device memory, one buffer per call
    enc = _encoder(H, case, sample_type)
    st = torch.cuda.current_stream().cuda_stream
    dev = []
    for n in PIECES:
        buf = torch.zeros(n * enc.width * enc.bytes_per_sample, dtype=torch.uint8, device="cuda")
        assert enc.render(n, buf.data_ptr(), st) == n * enc.width
        dev.append(buf)
    torch.cuda.synchronize()
    dev = b"".join(b.cpu().numpy().tobytes() for b in dev)
    enc.close()

    if sample_type == "int8" and case in ("i-16M-filter", "i-16M-filter-passthru"):
        kernel = FIXED_INT8                   # the sound stages, the width and the int8 store compiled in
    assert kernel.format(st=sample_type) in name, name
    if "k_line" not in kernel:
        assert f"ST=-1:{sample_type}" in name, name
    assert len(host) == len(want) and host == want, f"{case} {sample_type}: htv_render_host differs from htv_convert of int16"
    assert dev == want, f"{case} {sample_type}: htv_render differs from htv_convert of int16"


def test_compiled_in_int8_form(built):
    """PAL-I at 16 Msps with the VSB filter, FM and NICAM into int8 (a HackRF's format) runs the instantiation with the
    sound stages, the width and the int8 store compiled in, and equals int8 of the int16 stream; under HTV_KL=general
    the general form gives the same bytes."""
    H = built
    want = _convert(H, _int16_stream(H, "i-16M-filter"), "int8")
    for env, name in (({}, FIXED_INT8),
                      ({"HTV_KL": "general"}, "k_line<VF=1,HQ=1,FULL=1,CSAT=0,MAXT=256,SRC=0,SND=-1,WC=0,ST=-1:int8>")):
        with _env(**env):
            enc = H.Encoder(H.mode_config("i", vfilter=True), 16000000)
        enc.open_test_source()
        enc.set_sample_type("int8")
        got = b"".join(enc.render_host(n).tobytes() for n in PIECES)
        assert enc.line_kernel == name
        enc.close()
        assert got == want


def test_int16_names_are_unchanged(built):
    H = built
    enc = H.Encoder(H.mode_config("i", vfilter=True), 16000000)
    enc.open_test_source()
    enc.render_host(10)
    assert enc.line_kernel == "k_line<VF=1,HQ=1,FULL=1,CSAT=0,MAXT=256,SRC=0,SND=37,WC=1024>"
    assert enc.sample_type == "int16" and enc.bytes_per_sample == 4
    enc.close()


def test_convert_every_value_matches_the_reference_writers(built):
    H = built
    k = np.arange(65536)
    i = (k - 32768).astype(np.int16)
    iq = np.empty(65536 * 2, dtype=np.int16)
    iq[0::2] = i
    iq[1::2] = ~i
    for t in TYPES + ("int16",):
        for form, x in (("complex", iq), ("real", i)):
            data = _convert(H, x, t)
            g = GOLDEN[f"{t}_{form}"]
            assert len(data) == g["bytes"] and hashlib.sha256(data).hexdigest() == g["sha256"], f"{t}_{form}"
    # a tail that is not a whole group of eight, from an offset
    for t in TYPES:
        assert _convert(H, iq[8:8 + 1003], t) == _convert(H, iq[8:8 + 1008], t)[:1003 * np.dtype(H.SAMPLE_DTYPES[t]).itemsize]


def _cli(binary, args, nbytes):
    with tempfile.NamedTemporaryFile("r", suffix=".stderr") as err:
        cmd = f"timeout 120 {binary} {args} -o - test 2>{err.name} | head -c {nbytes}"
        out = subprocess.run(["bash", "-c", cmd], capture_output=True, timeout=180).stdout
        log = err.read()
    assert len(out) == nbytes, f"{binary} {args}: got {len(out)} of {nbytes} bytes\n{log[-500:]}"
    return out


@pytest.mark.skipif(not os.path.exists(STOCK), reason="the stock hacktv build is missing")
@pytest.mark.parametrize("sample_type", TYPES)
@pytest.mark.parametrize("args,per,exact", [
    ("-m i -s 16000000 --filter --noaudio", 2, True),
    ("-m pal -s 16000000", 1, True),
    ("-m i -s 16000000 --filter", 2, False),
])
def test_cli_type_against_stock_hacktv(built, sample_type, args, per, exact):
    H = built
    dtype = np.dtype(H.SAMPLE_DTYPES[sample_type])
    nbytes = 1300 * 1024 * per * dtype.itemsize
    a = _cli(CLI, f"{args} -t {sample_type}", nbytes)
    b = _cli(STOCK, f"{args} -t {sample_type}", nbytes)
    if exact:
        assert a == b
        return
    # the sound carriers' +-1 LSB of int16, through the type: +-1 for the 8- and 16-bit types, +-65537 for int32; a float
    # is compared as the int16 it was made from (x * 32767 rounds back to it), since two rounded quotients may lie a
    # little more than 1 / 32767 apart
    x, y = np.frombuffer(a, dtype=dtype).astype(np.float64), np.frombuffer(b, dtype=dtype).astype(np.float64)
    if sample_type == "float":
        x, y = np.rint(x * 32767), np.rint(y * 32767)
    tol = {"uint8": 1, "int8": 1, "uint16": 1, "int32": 65537, "float": 1}[sample_type]
    d = np.abs(x - y)
    assert d.max() <= tol, f"max |diff| {d.max()}"


def test_refusals(built, capfd):
    import torch
    H = built
    L = H.lib()
    enc = H.Encoder(H.mode_config("i", vfilter=True), 16000000)
    enc.open_test_source()
    assert L.htv_set_sample_type(enc._h, 9) == H.HTV_ERROR
    assert "unknown sample type 9" in capfd.readouterr().err
    with pytest.raises(ValueError):
        enc.set_sample_type("cf32")
    enc.set_sample_type("int8")
    buf = torch.zeros(64 * enc.width * 4, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError):
        enc.render_add(64, buf.data_ptr())
    assert "htv_render_add sums int16 streams" in capfd.readouterr().err
    assert enc.next_line() is None
    assert "htv_next_line hands out int16 lines" in capfd.readouterr().err
    enc.render_host(5)
    with pytest.raises(RuntimeError):
        enc.set_sample_type("float")
    assert "before the first line is rendered" in capfd.readouterr().err
    assert enc.sample_type == "int8" and L.htv_sample_type(enc._h) == 1
    enc.close()
    assert L.htv_convert(C_void(buf.data_ptr()), 6, C_void(buf.data_ptr()), 8, None) == H.HTV_ERROR
    assert "unknown sample type 6" in capfd.readouterr().err


def C_void(p):
    import ctypes
    return ctypes.c_void_p(p)
