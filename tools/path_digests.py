"""Byte identity of the device paths across builds: sha256 of each case's output, with its launch count.

Every case renders a fixed number of lines of the test source in uneven calls (1, 2, 23, 300, 625, 2000, ... lines),
so that sub-batch, descriptor-buffer and stream-start edges fall at different places, and prints one JSON line:
{"case", "line_kernel", "kernel_launches", "secam_chain", "lines", "sha256"}. Run it against two builds of the library
(HTV_LIB=<other .so>) and compare the lines: where the two builds are meant to compute the same stream in the same
launches, every line must match - the digest, the launch count and the SECAM chain's counters.

--time adds, for the timed cases, the device-resident ms of one 64-frame htv_render call (CUDA events around the
call on its stream, median of --reps calls after --warmup), with the card's name and power limit.

    python tools/path_digests.py [--time] [--reps 7] [--warmup 2] [--only NAME ...]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hacktv_b200 as H  # noqa: E402

PIECES = [1, 2, 23, 300, 625, 2000, 7, 1250]
SPLIT = {"HTV_PATH": "split"}

# name, mode, mode_config overrides, sample rate, pixel rate, environment, sample type, lines
CASES = [
    ("i_16M_filter_split_mma", "i", dict(vfilter=True), 16_000_000, 0, SPLIT, "int16", 1400),
    ("i_16M_filter_split_tma", "i", dict(vfilter=True), 16_000_000, 0, dict(SPLIT, HTV_FIR="scalar"), "int16", 1400),
    ("ntsc_13M5_split", "ntsc", dict(), 13_500_000, 0, SPLIT, "int16", 1100),
    ("m_13M5_filter_split", "m", dict(vfilter=True), 13_500_000, 0, SPLIT, "int16", 1100),
    ("l_16M_filter_split", "l", dict(vfilter=True), 16_000_000, 0, SPLIT, "int16", 1400),
    ("i_16M_filter_split_offset_swap", "i", dict(vfilter=True, offset=2_000_000, swap_iq=True), 16_000_000, 0, SPLIT,
     "int16", 1400),
    ("pal-fm_20M", "pal-fm", dict(), 20_000_000, 0, {}, "int16", 1400),
    ("pal-fm_20M_filter", "pal-fm", dict(vfilter=True), 20_000_000, 0, {}, "int16", 1400),
    ("secam-fm_20M25_filter", "secam-fm", dict(vfilter=True), 20_250_000, 0, {}, "int16", 900),
    ("i_16M_from_13M5_filter", "i", dict(vfilter=True), 16_000_000, 13_500_000, {}, "int16", 1400),
    ("i_16M_from_13M5", "i", dict(), 16_000_000, 13_500_000, {}, "int16", 1400),
    # a NICAM symbol shorter than 33 samples: every line takes the generic NICAM sum
    ("i_10M_split", "i", dict(), 10_000_000, 0, SPLIT, "int16", 1400),
    ("i_16M_filter_split_int8", "i", dict(vfilter=True), 16_000_000, 0, SPLIT, "int8", 1400),
    ("i_16M_filter_split_float", "i", dict(vfilter=True), 16_000_000, 0, SPLIT, "float", 1400),
    ("pal-fm_20M_filter_float", "pal-fm", dict(vfilter=True), 20_000_000, 0, {}, "float", 900),
    ("i_16M_filter_split_long", "i", dict(vfilter=True), 16_000_000, 0, SPLIT, "int16", 20_500),
    ("i_16M_filter_default", "i", dict(vfilter=True), 16_000_000, 0, {}, "int16", 1400),
    # the fused line kernel's sound pre-pass and descriptors in the caller's stream order
    ("i_16M_filter_default_no_ahead", "i", dict(vfilter=True), 16_000_000, 0, dict(HTV_AHEAD="0"), "int16", 1400),
    ("l_16M_filter_default", "l", dict(vfilter=True), 16_000_000, 0, {}, "int16", 1400),
    # SECAM: k_raster_secam + chain + k_line<SRC>; the same behind the split modulator; at 13.5 Msps the chain's
    # work-list kernels run; baseband (no video filter)
    ("l_16M_filter_scalar", "l", dict(vfilter=True), 16_000_000, 0, dict(HTV_FIR="scalar"), "int16", 1400),
    ("l_16M_filter_split_scalar", "l", dict(vfilter=True), 16_000_000, 0, dict(SPLIT, HTV_FIR="scalar"), "int16", 1400),
    ("l_13M5_filter_default", "l", dict(vfilter=True), 13_500_000, 0, {}, "int16", 1400),
    ("secam_16M", "secam", dict(), 16_000_000, 0, {}, "int16", 1400),
    ("pal_16M_from_13M5", "pal", dict(), 16_000_000, 13_500_000, {}, "int16", 1400),
    ("i_16M_from_14M_filter", "i", dict(vfilter=True), 16_000_000, 14_000_000, {}, "int16", 1400),
]

# render_add: the second channel added into the first one's stream, split and --pixelrate
ADD_CASES = [
    ("i_16M_filter_split_render_add", "i", dict(vfilter=True, offset=-3_000_000, level=0.5),
     dict(vfilter=True, offset=2_500_000, level=0.5), 16_000_000, 0, SPLIT, 1400),
    ("i_16M_from_13M5_filter_render_add", "i", dict(vfilter=True, offset=-3_000_000, level=0.5),
     dict(vfilter=True, offset=2_500_000, level=0.5), 16_000_000, 13_500_000, {}, 1400),
]

TIMED = ["i_16M_filter_split_mma", "i_16M_filter_split_tma", "pal-fm_20M", "pal-fm_20M_filter",
         "i_16M_from_13M5_filter", "i_16M_from_13M5", "l_16M_filter_split", "i_10M_split", "l_16M_filter_default",
         "i_16M_filter_default", "i_16M_filter_default_no_ahead"]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True).stdout.strip().splitlines()
    except OSError:
        q = []
    return q[0] if q else "unknown"


def encoder(mode, kw, rate, prate, env, sample_type):
    for k in ("HTV_PATH", "HTV_FIR", "HTV_AHEAD"):
        os.environ.pop(k, None)
    os.environ.update(env)                          # read once per encoder, when it is created
    enc = H.Encoder(H.mode_config(mode, **kw), rate, prate)
    enc.open_test_source()
    if sample_type != "int16":
        enc.set_sample_type(sample_type)
    return enc


def pieces(total):
    done, i = 0, 0
    while done < total:
        n = min(PIECES[i % len(PIECES)], total - done)
        yield n
        done += n
        i += 1


def digest(name, mode, kw, rate, prate, env, sample_type, lines):
    enc = encoder(mode, kw, rate, prate, env, sample_type)
    h = hashlib.sha256()
    for n in pieces(lines):
        h.update(np.ascontiguousarray(enc.render_host(n)).tobytes())
    r = {"case": name, "line_kernel": enc.line_kernel, "kernel_launches": enc.kernel_launches,
         "secam_chain": enc.secam_chain, "lines": lines, "sha256": h.hexdigest()}
    enc.close()
    return r


def digest_add(name, mode, kw_a, kw_b, rate, prate, env, lines):
    import torch
    a = encoder(mode, kw_a, rate, prate, env, "int16")
    b = encoder(mode, kw_b, rate, prate, env, "int16")
    per_line = a.width * (2 if a.complex else 1)
    buf = torch.zeros(lines * per_line, dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    done = 0
    for n in pieces(lines):
        p = buf.data_ptr() + done * per_line * 2
        a.render(n, p, st)
        b.render_add(n, p, st)
        done += n
    torch.cuda.synchronize()
    r = {"case": name, "line_kernel": b.line_kernel, "kernel_launches": [a.kernel_launches, b.kernel_launches],
         "secam_chain": [a.secam_chain, b.secam_chain], "lines": lines,
         "sha256": hashlib.sha256(buf.cpu().numpy().tobytes()).hexdigest()}
    a.close()
    b.close()
    return r


def time_case(name, mode, kw, rate, prate, env, sample_type, reps, warmup):
    import torch
    enc = encoder(mode, kw, rate, prate, env, sample_type)
    lines = 64 * enc.lines
    out = torch.empty(lines * enc.width * enc.bytes_per_sample, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream()
    ms = []
    for i in range(warmup + reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        enc.render(lines, out.data_ptr(), s.cuda_stream)
        e1.record(s)
        e1.synchronize()
        if i >= warmup:
            ms.append(e0.elapsed_time(e1))
    r = {"case": name, "line_kernel": enc.line_kernel, "lines_per_call": lines, "ms_median": float(np.median(ms)),
         "ms_range": [min(ms), max(ms)]}
    enc.close()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--time", action="store_true")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", nargs="*", default=None)
    a = ap.parse_args()
    want = lambda n: a.only is None or n in a.only
    print(json.dumps({"lib": H.LIB_PATH, "card": card()}), flush=True)
    for c in CASES:
        if want(c[0]):
            print(json.dumps(digest(*c)), flush=True)
    for c in ADD_CASES:
        if want(c[0]):
            print(json.dumps(digest_add(*c)), flush=True)
    if a.time:
        for c in CASES:
            if c[0] in TIMED and want(c[0]):
                print(json.dumps(time_case(*c[:7], a.reps, a.warmup)), flush=True)
        print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
