"""Device-resident SECAM timing (64 frames per call) + pass statistics.

    python tools/sec_time.py [--random] [--digest] [--calls N]

Per mode: ms per 64-frame call, and what the chain did in the first such call (htv_secam_chain: launches, passes, the
most one launch needed, lines recomputed, listed lines and the list kernel that finished them, the longest work list,
re-predictions after odd / even passes). --random: random pictures, a new one every frame, instead of the test card.
--digest: the sha256 of the last call's IQ, to compare builds bit for bit. HTV_SEC applies as for any encoder."""
import argparse
import hashlib
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hacktv_b200 as H

ap = argparse.ArgumentParser()
ap.add_argument("--random", action="store_true")
ap.add_argument("--digest", action="store_true")
ap.add_argument("--calls", type=int, default=10, help="timed calls per mode")
args = ap.parse_args()
print("gpu", torch.cuda.get_device_name(), flush=True)
for mode, rate in (("l", 16000000), ("l", 13500000), ("l", 20000000)):
    enc = H.Encoder(H.mode_config(mode, vfilter=True), rate)
    if args.random:
        rng = np.random.default_rng(7)
        enc.set_source(rng.integers(0, 1 << 24, size=(7, enc.active_lines, enc.active_width), dtype=np.uint32),
                       rng.integers(-32768, 32767, size=(40000, 2), dtype=np.int16))
    else:
        enc.open_test_source()
    n = 64 * enc.lines
    out = torch.empty(n * enc.width * 2, dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    enc.render(n, out.data_ptr(), st)
    torch.cuda.synchronize()
    cs = enc.secam_chain
    for _ in range(2): enc.render(n, out.data_ptr(), st)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.calls): enc.render(n, out.data_ptr(), st)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.calls
    print(mode, rate, "W", enc.width, "ms per 64 frames", round(ms, 4), "realtime_x", round(64 / 25 / (ms / 1e3), 1))
    print("  first call (%d lines): launches %d, passes %d (at most %d per launch), recomputed %d, listed %d by k_sec_fm_list "
          "and %d by k_sec_fm_list_t, longest list %d, re-predictions %d after odd and %d after even passes" %
          (n, cs["launches"], cs["passes"], cs["passes_max"], cs["recomputed"], cs["listed_warp"], cs["listed_thread"],
           cs["list_max"], cs["repredict_odd"], cs["repredict_even"]))
    if args.digest:
        print("  sha256 of the last call", hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest())
    enc.close()
