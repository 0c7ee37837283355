"""Cost of the sample types (htv_set_sample_type) at PAL-I 16 Msps --filter, 64-frame calls, on one GPU.

For each type, alternating with int16 in one process (int16, uint8, int16, int8, ...), it reports:
  - kline_ms: the line kernel's time per call (htv_last_line_kernel_ms, CUDA events around the launch);
  - step_ms: one device-resident htv_render call of 64 frames, CUDA events around the call on its stream;
  - host_ms / host_gsps: one htv_render_host call of 64 frames into pinned memory (wall clock, returns synchronised);
  - copy_floor_ms: a plain device-to-host copy of the same byte count into pinned memory (the floor
    tools/pcie_probe.py times for the int16 stream).
Medians over --reps calls after --warmup calls. The card's name and power limit are read in the same run.

    python tools/sample_type_bench.py [--reps 8] [--warmup 2] [--out results/sample_type_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hacktv_b200 as H  # noqa: E402

FRAMES = 64


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def measure(sample_type, reps, warmup):
    enc = H.Encoder(H.mode_config("i", vfilter=True), 16_000_000)
    enc.open_test_source()
    enc.set_sample_type(sample_type)
    enc.set_kernel_timing(True)
    lines = FRAMES * enc.lines
    nbytes = lines * enc.width * enc.bytes_per_sample
    dev = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    pinned = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    stream = torch.cuda.current_stream()
    kl, step = [], []
    for i in range(warmup + reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        enc.render(lines, dev.data_ptr(), stream.cuda_stream)
        e1.record(stream)
        e1.synchronize()
        if i >= warmup:
            step.append(e0.elapsed_time(e1))
            kl.append(enc.last_line_kernel_ms())
    host = []
    for i in range(warmup + reps):
        t = time.perf_counter()
        enc.render_host_ptr(lines, pinned.data_ptr())
        if i >= warmup:
            host.append((time.perf_counter() - t) * 1e3)
    name = enc.line_kernel
    samples = lines * enc.width
    enc.close()
    copy = []
    for i in range(warmup + reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        pinned.copy_(dev, non_blocking=True)
        e1.record(stream)
        e1.synchronize()
        if i >= warmup:
            copy.append(e0.elapsed_time(e1))
    med = lambda v: float(np.median(v))
    return {"type": sample_type, "line_kernel": name, "bytes_per_call": nbytes,
            "kline_ms": med(kl), "step_ms": med(step), "host_ms": med(host),
            "host_gsps": samples / (med(host) * 1e-3) / 1e9, "copy_floor_ms": med(copy),
            "kline_ms_range": [min(kl), max(kl)], "host_ms_range": [min(host), max(host)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sample_type_bench: no CUDA device")
    res = {"card": card(), "workload": "i 16 Msps --filter, test source, 64-frame calls", "runs": []}
    for t in ("uint8", "int8", "uint16", "int32", "float"):
        for st in ("int16", t):
            r = measure(st, a.reps, a.warmup)
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
