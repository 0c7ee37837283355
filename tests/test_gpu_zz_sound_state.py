"""k_line's per-lane sound state (htv_line.cuh KlFeed) against the oracle and against the descriptor-fed forms.

The k_line forms with the sound stages compiled in (PAL-I and B/G at 16 Msps: VSB + FM + NICAM, int16 or int8 store)
derive each lane's audio segment, NICAM symbol, renormalisation count and carrier index from the lane's audio-clock
index, set up once per CTA and advanced by one line's increments, and read the per-symbol and per-audio-sample records
the pre-pass chains write; the general forms read LineA2. Each row renders in calls of 1, 2 and an odd number of lines
and calls that start mid-frame and mid-symbol, from the stream start (where NICAM takes the generic sum, symbols s < 5):
  - against the oracle, +-1 LSB (the FM carrier, as test_gpu_parity.py states);
  - against the general form of the same encoder (HTV_KL=general, which reads LineA2) bit for bit: the two feeds give
    the same state, and the per-lane choice between the NICAM pulse table and the generic sum the same sums;
  - the int8 store: htv_convert of the int16 stream, bit for bit."""
import os

import numpy as np
import pytest

import hacktv_b200 as H
import orc
from test_gpu_zz_sample_types import _convert

CALLS = [1, 2, 37, 311, 1, 626, 3, 333]          # 1314 lines: calls across frame boundaries, odd lengths, mid-frame starts
FED = "SND=37,WC=1024"


def _render(mode, env=None, sample_type="int16"):
    os.environ.pop("HTV_KL", None)
    if env:
        os.environ.update(env)
    try:
        enc = H.Encoder(H.mode_config(mode, vfilter=True), 16_000_000)
    finally:
        os.environ.pop("HTV_KL", None)
    enc.open_test_source()
    if sample_type != "int16":
        enc.set_sample_type(sample_type)
    got = [np.ascontiguousarray(enc.render_host(n)) for n in CALLS]
    kernel = enc.line_kernel
    enc.close()
    if sample_type == "int16":
        got = np.concatenate([g.reshape(-1) for g in got])
    else:
        got = b"".join(g.tobytes() for g in got)
    return got, kernel


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["i", "g"])
def test_fed_form_matches_oracle_and_descriptor_form(mode):
    got, kernel = _render(mode)
    assert FED in kernel, kernel
    o = orc.Oracle(H.mode_config(mode, vfilter=True), 16_000_000)
    o.open_test_source()
    want = np.asarray(o.render(sum(CALLS))).reshape(-1)
    o.close()
    d = np.abs(got.astype(np.int32) - want.astype(np.int32))
    d = np.minimum(d, 65536 - d)                  # int16 wrap-around
    assert d.max() <= 1, f"max |diff| {d.max()} at {int(np.argmax(d))} ({kernel})"
    gen, gkernel = _render(mode, {"HTV_KL": "general"})
    assert FED not in gkernel, gkernel
    assert np.array_equal(got, gen), f"fed form {kernel} differs from {gkernel} at {int(np.argmax(got != gen))}"


@pytest.mark.gpu
def test_fed_form_int8_store():
    ref, _ = _render("i")
    got, kernel = _render("i", sample_type="int8")
    assert FED in kernel and "int8" in kernel, kernel
    assert got == _convert(H, ref, "int8")
