"""What the sound source costs a programme that lives on the GPU, per 64-frame step: device pictures (set_device_source,
a new picture every frame) with the sound from host memory (pinned int16 pairs through read_audio: a copy across PCIe)
against the same pictures with the sound from device memory (set_device_audio: k_pcm_ingest). PAL-I at 16 Msps with the
video filter, FM + NICAM, as bench.py's workload, rendered with htv_render into device memory; the sound is pulled in
blocks of one video frame (1280 pairs). The two encoders take turns, step blocks alternating, so that both see the
same machine; the step time is the host clock over a block of steps that ends in a synchronise. Then, in a run of its
own under torch.profiler, k_pcm_ingest's time per block and the host-to-device copy's. Prints the card's name and power
limit, and one JSON line.
    python tools/device_audio_time.py [rounds] [steps per block]"""
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
BLOCK = 1280            # sound pairs per pull: one 25 Hz frame at 32 kHz
SECONDS = 64            # of sound, cycled


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
    pics = rng.integers(0, 256, size=(PICTURES, host.active_lines, host.active_width, 3), dtype=np.uint8)
    d_pics = torch.from_numpy(pics).cuda()
    pcm = rng.integers(-32768, 32768, size=(SECONDS * 32000, 2), dtype=np.int16)
    pinned = torch.empty(pcm.shape, dtype=torch.int16, pin_memory=True).numpy()
    pinned[...] = pcm
    host.set_device_source(d_pics)
    host.set_source(None, pinned, audio_block=BLOCK)            # a Python callback per block, as set_device_audio's
    dev.set_device_source(d_pics)
    dev.set_device_audio(torch.from_numpy(pcm).cuda(), audio_block=BLOCK)
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
        if "k_pcm_ingest" in e.name:
            ingest.append(e.device_time)
        elif "Memcpy HtoD" in e.name and "Pinned" in e.name:
            copy.append(e.device_time)
    host.close()
    dev.close()
    print(json.dumps({
        "gpu": gpu, "power_limit_w": watts,
        "workload": "PAL-I 16 Msps --filter, FM + NICAM, device pictures (a new one every frame), sound in 1280-pair blocks",
        "rounds": rounds, "steps_per_block": steps,
        "host_sound_step_ms_median": float(np.median(times["host"])), "host_sound_step_ms_all": times["host"],
        "device_sound_step_ms_median": float(np.median(times["device"])), "device_sound_step_ms_all": times["device"],
        "k_pcm_ingest_launches": len(ingest),
        "k_pcm_ingest_us_per_block": float(np.mean(ingest)) if ingest else None,
        "htod_pinned_copies": len(copy), "htod_pinned_us_per_copy": float(np.mean(copy)) if copy else None,
        "sound_bytes_per_step": int(64 * BLOCK * 4)}))


if __name__ == "__main__":
    main()
