"""What a live source costs per 64-frame step, fed from pinned host memory (uint32 words, open_memory_source: copies
across PCIe) against fed from device memory (uint8 HWC, set_device_source: k_ingest), with a new picture every frame.
PAL-I at 16 Msps with the video filter, as bench.py's workload, rendered with htv_render into device memory. The two
encoders take turns, step blocks alternating, so that both see the same machine; the step time is the host clock over a
block of steps that ends in a synchronise. Then, in a run of its own under torch.profiler, k_ingest's time per picture
and the host-to-device copy's. Prints the card's name and power limit, and one JSON line.
    python tools/device_source_time.py [rounds] [steps per block]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hacktv_b200 as H  # noqa: E402

PICTURES = 128          # cycled, one per frame: every frame brings a new picture


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def encoders():
    conf = H.mode_config("i", vfilter=True)
    host, dev = H.Encoder(conf, 16_000_000), H.Encoder(conf, 16_000_000)
    rng = np.random.default_rng(0)
    pics = rng.integers(0, 1 << 24, size=(PICTURES, host.active_lines, host.active_width), dtype=np.uint32)
    pinned = torch.empty(pics.shape, dtype=torch.int32, pin_memory=True).numpy().view(np.uint32)
    pinned[...] = pics
    host.open_memory_source(pinned, None)
    rgb = np.stack([(pics >> 16) & 255, (pics >> 8) & 255, pics & 255], axis=-1).astype(np.uint8)
    dev.set_device_source(torch.from_numpy(rgb).cuda())
    return host, dev, pinned


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 8
    gpu, watts = torch.cuda.get_device_name(0), power_limit()
    print(f"gpu: {gpu}, power limit: {watts} W", flush=True)
    host, dev, pinned = encoders()
    L, W = host.lines, host.width
    step = 64 * L
    buf = torch.empty(step * W * 2, dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    for enc in (host, dev):                                      # warm-up: every slot filled, every phase converted
        for _ in range(3):
            enc.render(step, buf.data_ptr(), st)
    torch.cuda.synchronize()
    times = {"host": [], "device": []}
    for _ in range(rounds):
        for name, enc in (("host", host), ("device", dev)):
            t0 = time.perf_counter()
            for _ in range(steps):
                enc.render(step, buf.data_ptr(), st)
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3 / steps)

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for enc in (host, dev):
            for _ in range(2):
                enc.render(step, buf.data_ptr(), st)
        torch.cuda.synchronize()
    ingest, copy = [], []
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        if "k_ingest" in e.name:
            ingest.append(e.device_time)
        elif "Memcpy HtoD" in e.name and e.device_time > 50:        # the picture copies, not the frame maps
            copy.append(e.device_time)
    host.close()
    dev.close()
    n = 2 * 64                                                   # pictures each encoder brought in the profiled run
    print(json.dumps({
        "gpu": gpu, "power_limit_w": watts, "workload": "PAL-I 16 Msps --filter, a new picture every frame",
        "rounds": rounds, "steps_per_block": steps,
        "host_pinned_step_ms_median": float(np.median(times["host"])), "host_pinned_step_ms_all": times["host"],
        "device_step_ms_median": float(np.median(times["device"])), "device_step_ms_all": times["device"],
        "k_ingest_launches": len(ingest), "k_ingest_us_per_picture": float(np.sum(ingest)) / n,
        "htod_us_per_picture": float(np.sum(copy)) / n,
        "picture_bytes_uint32": int(pinned[0].nbytes), "picture_bytes_uint8_rgb": int(pinned[0].size * 3)}))


if __name__ == "__main__":
    main()
