"""What a live source pays for the composite store: the time of k_compose per (picture, colour-frame phase) conversion,
and of k_vf_rows, which filters the converted rows into the filtered store once per call (where the build has it), beside
the host-to-device copy of the same picture, from torch.profiler over a run with a new picture every frame (one
conversion per picture: the phase of the frame that shows it). PAL-I at 16 Msps with the video filter, as bench.py's
workload. Prints one JSON line.
    python tools/picture_time.py [frames]"""
import json
import os
import sys

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import hacktv_b200 as H  # noqa: E402


def main():
    frames = int(sys.argv[1]) if len(sys.argv) > 1 else 128
    enc = H.Encoder(H.mode_config("i", vfilter=True), 16_000_000)
    rng = np.random.default_rng(0)
    pics = rng.integers(0, 1 << 24, size=(frames, enc.active_lines, enc.active_width), dtype=np.uint32)
    enc.open_memory_source(pics, None)
    L = enc.lines
    buf = torch.empty(64 * L * enc.width * 2, dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    enc.render(64 * L, buf.data_ptr(), st)                      # warm-up
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(frames // 64):
            enc.render(64 * L, buf.data_ptr(), st)
        torch.cuda.synchronize()
    conv, vf, copy = [], [], []
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        if "k_compose" in e.name:
            conv.append(e.device_time)
        elif "k_vf_rows" in e.name:
            vf.append(e.device_time)
        elif "Memcpy HtoD" in e.name and e.device_time > 50:
            copy.append(e.device_time)
    enc.close()
    pic_bytes = enc.active_lines * enc.active_width * 4
    # consecutive pictures go up as one copy (htv_host.c), so count per picture
    n = 64 * (frames // 64)
    print(json.dumps({"pictures": n, "k_compose_launches": len(conv), "k_compose_us_per_conversion": float(np.sum(conv)) / max(len(conv), 1),
                      "k_compose_us_per_picture": float(np.sum(conv)) / n,
                      "k_vf_rows_launches": len(vf), "k_vf_rows_us_per_conversion": float(np.sum(vf)) / max(len(conv), 1),
                      "htod_copies": len(copy), "htod_us_per_picture": float(np.sum(copy)) / n, "picture_bytes": pic_bytes,
                      "gpu": torch.cuda.get_device_name(0)}))


if __name__ == "__main__":
    main()
