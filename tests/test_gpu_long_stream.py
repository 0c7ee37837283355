"""GPU parity far into the stream (SURVEY.md section 8d): BASELINE configs 2, 3 and 4 are rendered on the
device up to >= 10 s and >= 34 s of signal - past the wrap of every device-side ring (audio 2^20 pairs =
32.8 s, NICAM symbols 2^23 = 23 s, NICAM frames 2^14 = 16.4 s), through ~17 000 NCO renormalisations
and five loops of the 6.4 s test tone (ref av_test.c:156-196) - and the frame found there is compared with
lines of the UNMODIFIED reference's own output (tests/golden/long_*.npz, made by
tests/golden/make_golden_long.py). The stream in between is rendered into device memory and dropped.

What this test found (round 2): the reference's FM sound carrier is a Q31 phasor recurrence with a floor in every
step (ref video.c:2259-2276). Its phase follows the closed form used here - the sum of the exact angles of the
rounded LUT entries - to ~1e-5 rad over 10 s (tools/nco_drift.c) EXCEPT when the carrier sits at a small rational
fraction of the sample rate: NTSC-M at 13.5 Msps puts 4.5 MHz at exactly fs / 3, the phasor then revisits the same
three states, its floor errors stop averaging out and the reference's own carrier runs slow by ~1e-5 Hz
(6.6e-5 rad/s with the test tone, 6e-4 rad/s in silence). Reproducing that is a sample-serial problem (the drift
depends on the low bits of every state), so for config 3 the sound carrier is compared with an allowance of
0.35 LSB per second of signal on top of the +-1 LSB of BASELINE.json; everything else of config 3 (raster, chroma,
video filter - the "_noaudio" fixture) is integer work and is required to be bit-exact at 10 s and 34 s. The same
mode at 16 Msps, and PAL-I / SECAM-L at their rates, stay within +-1 LSB at 34 s (tools/drift_dbg.py)."""
import json
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "golden_long.json")))

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(GOLD))
def test_frames_at_10s_and_34s_match_the_reference(built, name):
    import torch
    H = built
    g = GOLD[name]
    z = np.load(os.path.join(HERE, "golden", "long_" + name + ".npz"))
    enc = H.Encoder(H.mode_config(g["mode"], vfilter=g["filter"], noaudio=g.get("noaudio", False)), g["rate"])
    enc.open_test_source()
    lpf, per = enc.lines, 2 if enc.complex else 1
    chunk = 64 * lpf                                             # 2.56 s (2.1 s at 525/59.94) per call
    scratch = torch.empty(chunk * enc.width * per, dtype=torch.int16, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    at = 0
    for tag in ("b", "c"):
        w = g["windows"][tag]
        assert w["values_per_line"] == enc.width * per
        while at < w["skip"]:
            n = min(chunk, w["skip"] - at)
            enc.render(n, scratch.data_ptr(), stream)
            at += n
        enc.render(lpf, scratch.data_ptr(), stream)
        at += lpf
        torch.cuda.synchronize()
        got = scratch[: lpf * enc.width * per].cpu().numpy().reshape(lpf, -1)[g["keep"]]
        d = np.abs(got.astype(np.int32) - z[tag].astype(np.int32))
        seconds = w["skip"] * enc.width / g["rate"]
        if g.get("noaudio"):
            assert d.max() == 0, f"{name} window {tag}: {np.count_nonzero(d)} values differ (integer-only configuration)"
            continue
        resonant = g["mode"] == "m" and g["rate"] == 13500000           # FM carrier at exactly fs / 3 (see above)
        tol = 1 + (int(np.ceil(0.35 * seconds)) if resonant else 0)
        # sound carriers are closed-form NCOs: +-1 LSB (BASELINE.json north_star); the rest is exact
        assert d.max() <= tol, f"{name} window {tag} (line {w['skip']}): max |diff| {d.max()} > {tol}, {np.count_nonzero(d > tol)} values out"
        # most values are exact (SECAM-L at 34 s, with AM + NICAM carriers, has the fewest); a model error would show as a drop
        if not resonant:
            assert (d == 0).mean() > 0.85, f"{name} window {tag}: only {(d == 0).mean():.3f} exact"
    enc.close()
