"""The sample-type conversion of hacktv_b200/csrc/htv_sample_type.h on the CPU, the same functions the device stores and
htv_convert run: every int16 value through all twelve streams the reference's file sink writes (-t uint8 .. float,
complex and real), against the sizes and sha256 pinned from the reference's own rf_file.o
(tests/golden/make_golden_sample_types.py). tests/sample_type_emu.c writes the streams."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "golden_sample_types.json")))["streams"]


@pytest.fixture(scope="module")
def streams(tmp_path_factory):
    d = tmp_path_factory.mktemp("st")
    exe = str(d / "sample_type_emu")
    subprocess.check_call(["gcc", "-O2", "-Wall", "-Wextra", "-I", os.path.join(ROOT, "hacktv_b200", "csrc"),
                           "-I", os.path.join(ROOT, "include"), "-o", exe, os.path.join(ROOT, "tests", "sample_type_emu.c")])
    subprocess.check_call([exe, str(d)])
    return d


@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_header_conversion_matches_the_reference_writer(streams, name):
    data = (streams / f"{name}.bin").read_bytes()
    assert len(data) == GOLDEN[name]["bytes"]
    assert hashlib.sha256(data).hexdigest() == GOLDEN[name]["sha256"]


def test_the_two_traps(streams):
    """int32 wraps at -32768 as gcc's (x << 16) + x does; float is a double product rounded once, which a float
    multiply by (float) (1 / 32767) misses on 1 536 values."""
    i32 = np.frombuffer((streams / "int32_real.bin").read_bytes(), dtype=np.int32)
    assert i32[0] == 2147450880 and i32[1] == -32767 * 65537
    f = np.frombuffer((streams / "float_real.bin").read_bytes(), dtype=np.float32)
    x = np.arange(-32768, 32768, dtype=np.int64)
    assert np.array_equal(f, (x.astype(np.float64) * (1.0 / 32767.0)).astype(np.float32))
    single = x.astype(np.float32) * np.float32(1.0 / 32767.0)
    assert int(np.count_nonzero(single != f)) == 1536
