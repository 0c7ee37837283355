"""Pin S-Video (`--s-video`, ref hacktv.c:1136-1148, video.c:3031-3040, 3206-3228) to the reference: each case below is
rendered by tests/golden/s_video_harness.c, linked against the reference's own objects as the oracle build compiles
them in place (make -C oracle ref), and golden_s_video.json records the sha256 of its int16 I,Q stream.
tests/test_s_video_host.py renders the same cases with tests/sv_oracle.py and compares the hashes; the device's
htv_cli file is compared with the 2 500-line case. Run where the reference build exists, naming the reference tree
(the REF of oracle/Makefile):

    python tests/golden/make_golden_s_video.py <reference tree>

The windows are long enough for frame parity, PAL's V-switch and SECAM's D'r / D'b alternation: 1 300 lines of the
625-line modes, 1 100 of the 525-line ones. "programme" cases take their pictures from programme_source
(tests/test_oracle_vs_ref.py) with PROGRAMME_SEED; the baseband modes have no sound.
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
OBJ = os.path.join(os.path.dirname(TESTS), "oracle", "_ref", "obj")
# the reference modules the encoder core links against (oracle/Makefile REFMODS) and the zero-filling heap shim
REFMODS = ["common", "fir", "vbidata", "teletext", "wss", "video", "fifo", "mac", "dance", "eurocrypt", "videocrypt",
           "videocrypts", "syster", "syster-ca", "acp", "vits", "vitc", "nicam728", "sis", "av", "av_test", "rf", "rf_file",
           "spdif", "cc608", "ref_shim_zero"]
PROGRAMME_SEED = 41

# (mode, rate, lines, filter, extra, source)
CASES = [
    ("pal", 16000000, 1300, False, [], "test"),
    ("pal", 16000000, 1300, True, [], "test"),
    ("pal", 16000000, 2500, True, [], "test"),                  # htv_cli's file (test_gpu_zz_s_video.py)
    ("pal", 20050000, 1300, True, [], "test"),                  # chroma taps sum to 32769, partial last tile
    ("ntsc", 13500000, 1100, False, [], "test"),
    ("ntsc", 13500000, 1100, True, [], "test"),
    ("525pal", 13500000, 1100, False, [], "test"),
    ("pal60", 13500000, 1100, True, [], "test"),
    ("secam", 16000000, 1300, False, [], "test"),
    ("secam", 16000000, 1300, True, [], "test"),
    ("secam", 20250000, 1300, True, [], "test"),
    ("pal", 16000000, 1300, False, ["--swap-iq"], "test"),
    ("pal", 16000000, 1300, False, ["--offset", "2000000"], "test"),
    ("pal", 16000000, 1300, True, [], "programme"),
    ("secam", 16000000, 1300, True, [], "programme"),
]


def case_key(mode, rate, lines, filt, extra, source):
    return " ".join([mode, str(rate), str(lines), "filter" if filt else "nofilter", source] + list(extra))


def main(ref):
    sys.path.insert(0, TESTS)
    sys.path.insert(0, os.path.dirname(TESTS))
    import hacktv_b200 as H
    from test_oracle_vs_ref import programme_source
    cases = []
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "s_video_harness")
        subprocess.check_call(["gcc", "-O2", "-Wall", "-I", os.path.join(ref, "src"), "-o", exe,
                               os.path.join(HERE, "s_video_harness.c")] +
                              [os.path.join(OBJ, m + ".o") for m in REFMODS] + ["-Wl,--wrap=malloc", "-lm", "-pthread"])
        for mode, rate, lines, filt, extra, source in CASES:
            out = os.path.join(tmp, "out.bin")
            cmd = [exe, "-m", mode, "-s", str(rate), "--lines", str(lines), "-o", out] + (["--filter"] if filt else []) + extra
            if source == "programme":
                conf = H.mode_config(mode)
                t = H.Tables(conf, rate)
                aw = int(t.get("geometry")[3])
                t.close()
                frames, _ = programme_source(PROGRAMME_SEED, conf.active_lines, aw)
                fn = os.path.join(tmp, "frames.rgb32")
                np.ascontiguousarray(frames, dtype=np.uint32).tofile(fn)
                cmd += ["--frames", fn]
            subprocess.check_call(cmd, timeout=600)
            data = open(out, "rb").read()
            cases.append({"mode": mode, "rate": rate, "lines": lines, "filter": filt, "extra": extra, "source": source,
                          "values": len(data) // 2, "sha256": hashlib.sha256(data).hexdigest()})
            print(case_key(mode, rate, lines, filt, extra, source), len(data) // 2, cases[-1]["sha256"][:16])
    out = {"source": "tests/golden/s_video_harness.c on the unmodified reference: int16 I,Q interleaved",
           "programme_seed": PROGRAMME_SEED, "cases": cases}
    with open(os.path.join(HERE, "golden_s_video.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
