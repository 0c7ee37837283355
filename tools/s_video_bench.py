"""What S-Video costs on one GPU, and what its run-time test in the general k_line forms costs the other modes.

Device-resident time of one htv_render call of 64 frames (CUDA events around the call on its stream):
  - pal 16 Msps, ntsc 13.5 Msps and secam 16 Msps, each with and without S-Video (this build);
  - BASELINE configs 1 to 5 (tools/bench_configs.py) on this build and on another build of the library given by
    --parent-lib (the build before S-Video). Config 2 runs the instantiation with the sound stages compiled in, the
    others the general forms; config 5 (W = 1280) the 320-thread forms, where the run-time test moves the most spill code.
Each build runs in a worker process of its own (a library is chosen at import: HTV_LIB); --rounds rounds alternate the
two workers, parent first in odd rounds, this build first in even ones, and each worker times every case --reps times
after --warmup calls, cases interleaved call by call. Reported per case: the median over all calls, and the median of
each round. The card's name, power limit and maximum SM clock are read in the same run, before and after.

    python tools/s_video_bench.py --parent-lib PATH [--rounds 4] [--reps 8] [--warmup 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FRAMES = 64
SV_CASES = [(f"{m} {r}{' --s-video' if sv else ''}", m, r, dict(s_video=True) if sv else {})
            for m, r in (("pal", 16000000), ("ntsc", 13500000), ("secam", 16000000)) for sv in (False, True)]
CFG_CASES = [(f"{c} {m} {r}{' --filter' if f else ''}", m, r, dict(vfilter=f)) for c, m, r, f in
             (("cfg1", "pal", 16000000, False), ("cfg2", "i", 16000000, True), ("cfg3", "m", 13500000, True),
              ("cfg4", "l", 16000000, True), ("cfg5", "i", 20000000, True))]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def worker(with_sv, reps, warmup):
    """Times the cases on the library HTV_LIB names (or this tree's); one JSON line: case -> (line kernel, ms list)."""
    import torch
    sys.path.insert(0, ROOT)
    import hacktv_b200 as H
    cases = (SV_CASES if with_sv else []) + CFG_CASES
    encs = []
    for name, mode, rate, kw in cases:
        enc = H.Encoder(H.mode_config(mode, **kw), rate)
        enc.open_test_source()
        lines = FRAMES * enc.lines
        out = torch.empty(lines * enc.width * (2 if enc.complex else 1), dtype=torch.int16, device="cuda")
        encs.append((name, enc, lines, out, []))
    st = torch.cuda.current_stream()
    for i in range(warmup + reps):
        for name, enc, lines, out, ms in encs:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            enc.render(lines, out.data_ptr(), st.cuda_stream)
            e1.record(st)
            e1.synchronize()
            if i >= warmup:
                ms.append(e0.elapsed_time(e1))
    res = {name: (enc.line_kernel, ms) for name, enc, lines, out, ms in encs}
    for _, enc, _, _, _ in encs:
        enc.close()
    print(json.dumps(res))


def run_worker(lib, with_sv, reps, warmup):
    env = dict(os.environ)
    if lib:
        env["HTV_LIB"] = lib
    cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--reps", str(reps), "--warmup", str(warmup)]
    if with_sv:
        cmd.append("--with-sv")
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, check=True)
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", help="libhacktv_b200.so built from the commit before S-Video")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--with-sv", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        worker(a.with_sv, a.reps, a.warmup)
        return
    if not a.parent_lib:
        raise SystemExit("s_video_bench: --parent-lib is required")
    res = {"card": card(), "frames_per_call": FRAMES}
    runs = {"this": {}, "parent": {}}
    for rnd in range(a.rounds):
        order = ("parent", "this") if rnd % 2 == 0 else ("this", "parent")
        for build in order:
            got = run_worker(os.path.abspath(a.parent_lib) if build == "parent" else None, build == "this", a.reps, a.warmup)
            for name, (kernel, ms) in got.items():
                e = runs[build].setdefault(name, {"line_kernel": kernel, "ms": [], "round_medians": []})
                e["ms"] += ms
                e["round_medians"].append(round(float(np.median(ms)), 4))
    res["runs"] = []
    for build in ("this", "parent"):
        for name, e in runs[build].items():
            r = {"build": build, "case": name, "line_kernel": e["line_kernel"],
                 "ms_per_64_frames": round(float(np.median(e["ms"])), 4), "round_medians": e["round_medians"],
                 "calls": len(e["ms"])}
            res["runs"].append(r)
            print(json.dumps(r), flush=True)
    res["card_after"] = card()
    print(json.dumps({"card": res["card"], "card_after": res["card_after"]}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
