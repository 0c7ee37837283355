"""Where a bench-shaped step's time goes between line-kernel launches: one sequence of 64-frame htv_render calls of the
bench workload (PAL-I, VSB filter, FM + NICAM, 16 Msps) under torch.profiler with CUDA activities, in a run of its own.

Prints one JSON line per kernel (call, stream, name, start and end in us from the first kernel) and, per call, the gap
between the end of one k_line and the start of the next, with the side-stream kernels that ran in that gap and beside
k_line. The trace goes to --trace when given. Profiling slows the host: take step times from bench.py, not from here.

    python tools/step_timeline.py [--calls 8] [--warmup 3] [--trace out.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hacktv_b200 as H  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--trace", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        card = "unknown"
    enc = H.Encoder(H.mode_config("i", vfilter=True), 16_000_000)
    enc.open_test_source()
    lines = 64 * enc.lines
    out = torch.empty(lines * enc.width * enc.bytes_per_sample, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream()
    for _ in range(a.warmup):
        enc.render(lines, out.data_ptr(), s.cuda_stream)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.calls):
            enc.render(lines, out.data_ptr(), s.cuda_stream)
        torch.cuda.synchronize()
    name = enc.line_kernel
    enc.close()
    if a.trace:
        prof.export_chrome_trace(a.trace)

    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.time_range.end > e.time_range.start]
    ev = [e for e in ev if not e.name.startswith("Memcpy") and not e.name.startswith("Memset")]
    ev.sort(key=lambda e: e.time_range.start)
    t0 = ev[0].time_range.start if ev else 0
    kl = [e for e in ev if e.name.startswith("void k_line<") or e.name.startswith("k_line<")]
    print(json.dumps({"card": card, "line_kernel": name, "calls": a.calls, "kernels": len(ev)}), flush=True)
    for e in ev:
        # the call of a kernel: the first k_line that ends after it starts (side work runs ahead, for the next call)
        call = next((i for i, k in enumerate(kl) if k.time_range.end > e.time_range.start), len(kl))
        stream = getattr(e, "stream", None)
        if stream is None:
            stream = getattr(e, "device_resource_id", None)
        print(json.dumps({"call": call, "stream": stream, "name": e.name.split("(")[0][:80],
                          "start_us": round(e.time_range.start - t0, 2), "end_us": round(e.time_range.end - t0, 2)}))
    for c in range(1, len(kl)):
        g0, g1 = kl[c - 1].time_range.end, kl[c].time_range.start
        side = sorted({e.name.split("<")[0].split("(")[0].replace("void ", "") for e in ev
                       if e not in kl and e.time_range.end > g0 and e.time_range.start < g1})
        beside = sorted({e.name.split("<")[0].split("(")[0].replace("void ", "") for e in ev
                         if e not in kl and e.time_range.start < kl[c - 1].time_range.end and e.time_range.end > kl[c - 1].time_range.start})
        print(json.dumps({"gap_after_call": c - 1, "k_line_us": round(kl[c - 1].time_range.end - kl[c - 1].time_range.start, 2),
                          "gap_us": round(g1 - g0, 2), "in_gap": side, "beside_k_line": beside}))


if __name__ == "__main__":
    main()
