"""k_resample's arithmetic (hacktv_b200/csrc/htv_resample.h) on the CPU: the closed form per line against a
streaming restatement of the reference's resampler loop (ref fir.c:304-355), tests/resample_emu.c."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("rs") / "resample_emu")
    subprocess.check_call(["gcc", "-O2", "-Wall", "-I", os.path.join(ROOT, "hacktv_b200", "csrc"),
                           "-o", exe, os.path.join(ROOT, "tests", "resample_emu.c")])
    return exe


@pytest.mark.parametrize("Wp,I,D", [(864, 32, 27), (864, 40, 27), (1024, 27, 32), (572, 3, 2), (896, 8, 7), (832, 16, 13),
                                    (864, 20, 27), (1280, 4, 5), (865, 1024, 865), (864, 3, 2)])
def test_closed_form_equals_the_streaming_resampler(emu, Wp, I, D):
    for seed in (1, 2):
        out = subprocess.run([emu, str(Wp), str(I), str(D), str(seed)], capture_output=True, text=True)
        assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout
