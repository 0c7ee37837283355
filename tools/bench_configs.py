#!/usr/bin/env python
"""Device-resident throughput of every BASELINE.json config on one GPU (not the graded
bench - that is bench.py, config 2). Prints one JSON line per config.
    python tools/bench_configs.py"""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import hacktv_b200 as H

CONFIGS = [("cfg1 pal 16M (real)", "pal", 16000000, False), ("cfg2 i 16M --filter", "i", 16000000, True),
           ("cfg3 m 13.5M --filter", "m", 13500000, True), ("cfg4 l 16M --filter (SECAM)", "l", 16000000, True),
           ("cfg5 i 20M --filter", "i", 20000000, True),
           ("next: pal-fm 20M --filter (FM video)", "pal-fm", 20000000, True)]
for name, mode, rate, filt in CONFIGS:
    enc = H.Encoder(H.mode_config(mode, vfilter=filt), rate)
    enc.open_test_source()
    frames = 64
    nlines = frames * enc.lines
    out = torch.empty(nlines * enc.width * 2, dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    for _ in range(3):
        enc.render(nlines, out.data_ptr(), st)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    K = 5
    for _ in range(K):
        enc.render(nlines, out.data_ptr(), st)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / K
    ms_ = nlines * enc.width / (ms / 1e3) / 1e6
    print(json.dumps({"config": name, "ms_per_64_frames": round(ms, 3), "msamples_per_s": round(ms_, 1),
                      "realtime_x": round(ms_ / (rate / 1e6), 1), "bytes_per_sample": enc.bytes_per_sample}))
    enc.close()
