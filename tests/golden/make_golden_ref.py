#!/usr/bin/env python
"""Fixtures of tests/test_oracle_vs_ref.py from the UNMODIFIED reference (oracle/_ref/ref_harness and its
stock-allocator twin, built by `make -C oracle ref` where the reference tree is present): the sha256 and size
of the int16 stream of every reference run the tests compare with (golden_ref.json), and the two scan lines
per mode the WSS overlay is recovered from (golden_ref_wss.npz).

    python tests/golden/make_golden_ref.py
"""
import hashlib
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import orc  # noqa: E402
import test_oracle_vs_ref as T  # noqa: E402
import hacktv_b200 as H  # noqa: E402


def main():
    assert orc.have_ref(), "build the reference first: make -C oracle ref"
    index = {}

    def put(key, a, **more):
        index[key] = {"size": int(a.size), "sha256": hashlib.sha256(a.tobytes()).hexdigest(), **more}
        print(index[key]["sha256"][:16], key)

    def run(mode, rate, lines, *, skip=0, vfilter=False, extra=(), source="test", frames=None, audio=None, ext=None,
            audio_block=4000):
        with tempfile.TemporaryDirectory() as td:
            run_extra = tuple(extra)
            if ext is not None:
                fn = os.path.join(td, "ext.iq")
                ext.tofile(fn)
                run_extra += (fn,)                       # the value of the trailing --passthru
            a = orc.run_ref(mode, rate, lines, skip=skip, vfilter=vfilter, extra=run_extra, frames=frames, audio=audio,
                            audio_block=audio_block if audio is not None else 0)
        put(T.ref_key(mode, rate, lines, skip=skip, vfilter=vfilter, extra=extra, source=source), a)
        return a

    for mode, rate, nlines, filt, extra in T.CASES:
        run(mode, rate, nlines, vfilter=filt, extra=extra)
    for mode, rate, filt, extra, ext_lines in T.PASSTHRU_CASES:
        W = orc.Oracle(T._conf(H, mode, filt, extra), rate).width
        run(mode, rate, 30, vfilter=filt, extra=tuple(extra) + ("--passthru",), source=f"passthru{ext_lines}",
            ext=T.passthru_stream(W, ext_lines))
        run(mode, rate, 30, vfilter=filt, extra=extra)
    for mode, rate, nlines, filt, extra in T.POST_OFFSET:
        run(mode, rate, nlines, vfilter=filt, extra=extra)
    for mode, rate, filt, extra, ext_lines in T.POST_PASSTHRU:
        W = orc.Oracle(T._conf(H, mode, filt, extra), rate).width
        run(mode, rate, T.POST_LINES, vfilter=filt, extra=tuple(extra) + ("--passthru",), source=f"passthru{ext_lines}",
            ext=T.passthru_stream(W, ext_lines))

    lines = {}
    for mode, rate in (("i", 16000000), ("pal", 16000000), ("l", 16000000), ("secam", 16000000), ("pal", 13500000)):
        t = H.Tables(H.mode_config(mode, noaudio=True), rate)
        W = int(t.get("geometry")[0])
        t.close()
        per = 2 if H.mode_config(mode).output_type == 0 else 1
        for tag, extra in (("plain", ("--noaudio", "--nocolour")), ("wss", ("--noaudio", "--nocolour", "--wss", "16:9"))):
            lines[f"{mode}_{rate}_{tag}"] = orc.run_ref(mode, rate, 30, extra=extra).reshape(30, W, per)[22, :, 0].copy()
    for mode, rate, filt, extra in (("i", 16000000, True, ()), ("pal", 16000000, False, ()), ("l", 16000000, True, ()),
                                    ("secam", 16000000, False, ())):
        run(mode, rate, 700, vfilter=filt, extra=tuple(extra) + ("--wss", "16:9"))

    o = orc.Oracle(H.mode_config("i", vfilter=True), 16000000)
    frames, audio = T.random_source(7, o.active_lines, o.active_width)
    run("i", 16000000, 1400, vfilter=True, source="random7", frames=frames, audio=audio)

    for mode, rate, filt, extra, nlines, block, seed in T.programme_cases():
        o = orc.Oracle(T._conf(H, mode, filt, extra), rate)
        frames, audio = T.programme_source(seed, o.active_lines, o.active_width)
        run(mode, rate, nlines, vfilter=filt, extra=extra, source=f"programme{seed}", frames=frames, audio=audio,
            audio_block=block)

    for mode, rate, nlines in T.LOW_RATE_SOURCES:
        o = orc.Oracle(H.mode_config(mode, vfilter=True), rate)
        frames, audio = T.random_source(13, o.active_lines, o.active_width)
        run(mode, rate, nlines, vfilter=True, source="random13", frames=frames, audio=audio)
        frames, audio = T.programme_source(17, o.active_lines, o.active_width)
        run(mode, rate, nlines, vfilter=True, source="programme17", frames=frames, audio=audio)

    raw = orc.run_ref("i", 16000000, 700, vfilter=True, rawheap=True)
    put(T.ref_key("i", 16000000, 700, vfilter=True, rawheap=True), raw,
        masked_32_sha256=hashlib.sha256(np.ascontiguousarray(raw.reshape(700, 1024, 2)[:, 32:-32]).tobytes()).hexdigest())

    for mode, rate, prate, nlines, filt, extra in T.PIXELRATE_CASES:
        run(mode, rate, nlines, vfilter=filt, extra=tuple(extra) + ("--pixelrate", str(prate)))
    run("i", 16000000, 300, skip=1400, vfilter=True, extra=("--pixelrate", "13500000"))
    o = orc.Oracle(H.mode_config("i", vfilter=True), 16000000, 13500000)
    frames, audio = T.random_source(5, o.active_lines, o.active_width)
    run("i", 16000000, 900, vfilter=True, extra=("--pixelrate", "13500000"), source="random5", frames=frames, audio=audio)
    run("i", 16000000, 30, vfilter=True, extra=("--pixelrate", "13500000", "--passthru"), source="passthru40s3",
        ext=T.passthru_stream(o.width, 40, seed=3, tail=100))
    run("pal", 16000000, 100, extra=("--pixelrate", "13500000", "--wss", "16:9"))

    with open(os.path.join(HERE, "golden_ref.json"), "w") as f:
        json.dump(index, f, indent=1, sort_keys=True)
    np.savez_compressed(os.path.join(HERE, "golden_ref_wss.npz"), **lines)


if __name__ == "__main__":
    main()
