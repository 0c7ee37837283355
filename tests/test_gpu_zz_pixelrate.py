"""--pixelrate on the GPU (SURVEY.md section 8f rank 4): raster in a second device context at the pixel
rate, k_resample (the reference's polyphase resampler in closed form), then the usual modulator - against the
oracle, which is pinned bit for bit to the reference's own --pixelrate output (tests/test_oracle_vs_ref.py).
"""
import os

import numpy as np
import pytest

import orc

pytestmark = pytest.mark.gpu

CASES = [
    ("pal", 16000000, 13500000, 700, dict(), 0),
    ("i", 16000000, 13500000, 700, dict(vfilter=True, noaudio=True), 0),
    ("i", 16000000, 13500000, 700, dict(vfilter=True), 1),
    ("i", 16000000, 13500000, 700, dict(), 1),
    ("i", 20000000, 13500000, 500, dict(vfilter=True), 1),
    ("i", 16000000, 14000000, 500, dict(vfilter=True), 1),
    # sound carriers (+-1 LSB each, closed-form NCOs) behind the offset mixer (its own NCO: +-1 LSB): the two
    # errors stack to 2 LSB on a few samples per thousand lines - the relaxed tolerance include/hacktv_b200.h states
    ("i", 16000000, 13500000, 500, dict(vfilter=True, offset=2000000), 2),
    ("i", 16000000, 13500000, 500, dict(vfilter=True, offset=2000000, noaudio=True), 1),
]


@pytest.mark.parametrize("mode,rate,prate,nlines,kw,tol", CASES)
def test_pixelrate_parity(built, mode, rate, prate, nlines, kw, tol):
    H = built
    conf = H.mode_config(mode, **kw)
    enc = H.Encoder(conf, rate, prate)
    enc.open_test_source()
    got = enc.render_host(nlines)
    enc.close()
    o = orc.Oracle(conf, rate, prate)
    o.open_test_source()
    want = o.render(nlines)
    o.close()
    d = np.abs(got.astype(np.int32) - want.astype(np.int32))
    assert d.max() <= tol, f"max |diff| = {d.max()} at {np.argmax(d)}"


def test_pixelrate_chunking_and_scalar_filter(built):
    H = built
    conf = H.mode_config("i", vfilter=True)
    a = H.Encoder(conf, 16000000, 13500000); a.open_test_source(); whole = a.render_host(1500); a.close()
    b = H.Encoder(conf, 16000000, 13500000); b.open_test_source()
    parts = np.concatenate([b.render_host(n) for n in (1, 311, 313, 625, 250)]); b.close()
    assert np.array_equal(whole, parts)
    os.environ["HTV_FIR"] = "scalar"
    try:
        c = H.Encoder(conf, 16000000, 13500000); c.open_test_source(); scalar = c.render_host(1500); c.close()
    finally:
        os.environ.pop("HTV_FIR", None)
    assert np.array_equal(whole, scalar)
