"""k_line's per-lane sound feed (hacktv_b200/csrc/htv_line.cuh KlFeed) on the CPU: the state a lane advances by one
line's increments equals the closed forms of its audio-clock index - audio index and segment bounds, NICAM symbol and
its start, m mod 32767, m mod the NICAM carrier period - tests/sound_feed_emu.c."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("sf") / "sound_feed_emu")
    subprocess.check_call(["gcc", "-O2", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "sound_feed_emu.c")])
    return exe


# the sample rates the GPU tests render (W = 64 us of samples), from the stream start (segment j = -1, symbols s < 5)
RATES = [2_000_000, 4_000_000, 6_750_000, 8_000_000, 10_000_000, 12_000_000, 13_500_000, 14_000_000, 16_000_000,
         20_000_000, 20_250_000]


@pytest.mark.parametrize("rate", RATES)
def test_advance_equals_closed_form_from_stream_start(emu, rate):
    W = rate * 64 // 1_000_000
    # 700 lines pass segment boundaries at every lane and more than one renormalisation (m = 32766 mod 32767)
    out = subprocess.run([emu, str(rate), str(W), str(W), "0", "700"], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout


@pytest.mark.parametrize("rate", [10_000_000, 16_000_000, 20_250_000])
@pytest.mark.parametrize("line0", [1_000_003, (1 << 32) // 640 + 1, 1 << 23])
def test_advance_equals_closed_form_far_into_the_stream(emu, rate, line0):
    # past 2^32 samples: the 32-bit quotients wrap, their ring slots and the remainders must not
    W = rate * 64 // 1_000_000
    out = subprocess.run([emu, str(rate), str(W), str(2 * W), str(line0), "400"], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout
