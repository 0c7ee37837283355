"""Pin the reference's file sink (ref rf_file.c, the twelve _rf_file_write_* writers behind hacktv's -t/--type) over
every int16 value: tests/golden/rf_file_harness.c, linked against the reference's own rf_file.o and rf.o as the oracle
build compiles them in place (make -C oracle ref), writes the twelve streams; this script records each stream's size
and sha256 in golden_sample_types.json. Run where the reference build exists, naming the reference tree (the
REF of oracle/Makefile; its src/rf.h declares the writers' interface):

    python tests/golden/make_golden_sample_types.py <reference tree>
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OBJ = os.path.join(ROOT, "oracle", "_ref", "obj")


def main(ref):
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "rf_file_harness")
        subprocess.check_call(["gcc", "-O2", "-Wall", "-I", os.path.join(ref, "src"), "-o", exe,
                               os.path.join(HERE, "rf_file_harness.c"),
                               os.path.join(OBJ, "rf_file.o"), os.path.join(OBJ, "rf.o")])
        subprocess.check_call([exe, tmp])
        streams = {}
        for t in ("uint8", "int8", "uint16", "int16", "int32", "float"):
            for form in ("complex", "real"):
                data = open(os.path.join(tmp, f"{t}_{form}.bin"), "rb").read()
                streams[f"{t}_{form}"] = {"bytes": len(data), "sha256": hashlib.sha256(data).hexdigest()}
    out = {"input": "65536 complex int16 samples, I = k - 32768, Q = ~I for k = 0..65535, interleaved I,Q; "
                    "real writers write I only",
           "source": "ref rf_file.c _rf_file_write_<type>_<complex|real> via rf_file_open + rf_write",
           "streams": streams}
    with open(os.path.join(HERE, "golden_sample_types.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps(streams, indent=1))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
