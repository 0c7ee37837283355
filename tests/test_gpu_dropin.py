"""hacktv's own, unmodified front end (hacktv.c + av_test.c + rf_file.c compiled in place from
the reference tree) linked against integration/video_b200.c + libhacktv_b200.so, run next to
the stock build: same command line, same bytes (within the +-1 LSB the sound carriers allow).
Both binaries are prebuilt by `make -C oracle ref dropin` and travel to the GPU box."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DROPIN = os.path.join(ROOT, "oracle", "_ref", "hacktv_b200_dropin")
STOCK = os.path.join(ROOT, "oracle", "_ref", "hacktv_ref")

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not (os.path.exists(DROPIN) and os.path.exists(STOCK)), reason="drop-in demo not built")]


def _run(binary, args, nbytes, env=""):
    """Also proves WHICH encoder ran: the adapter's vid_info prints `Encoder: hacktv_b200 ...` (integration/
    video_b200.c), the stock video.c does not - a bug in the adapter's _accelerated() that quietly sent a
    configuration to the renamed stock encoder would otherwise compare the reference with itself."""
    with tempfile.NamedTemporaryFile("r", suffix=".stderr") as err:
        cmd = f"{env}timeout 120 {binary} {args} -o - test 2>{err.name} | head -c {nbytes}"
        out = subprocess.run(["bash", "-c", cmd], capture_output=True, timeout=180).stdout
        log = err.read()
    assert len(out) == nbytes, f"{binary}: got {len(out)} of {nbytes} bytes"
    assert ("Encoder: hacktv_b200" in log) == (binary == DROPIN), f"{binary} {args}: wrong encoder ran\n{log[-500:]}"
    return np.frombuffer(out, dtype=np.int16)


@pytest.mark.parametrize("args,per,tol", [
    ("-m pal -s 16000000", 2, 0),
    ("-m i -s 16000000 --filter --noaudio", 4, 0),
    ("-m i -s 16000000 --filter", 4, 1),
    ("-m m -s 13500000 --filter", 4, 1),
    ("-m l -s 16000000 --filter", 4, 1),
    ("-m pal-fm -s 20000000 --filter --noaudio", 4, 1),
    # VBI: the stock WSS stage (wss.c) runs inside the adapter, its waveform rides the encoder's overlay hook
    ("-m i -s 16000000 --filter --noaudio --wss 16:9", 4, 0),
    ("-m l -s 16000000 --filter --wss auto", 4, 1),
    ("-m pal -s 16000000 --wss 14:9-letterbox", 2, 0),
    ("-m i -s 16000000 --filter --noaudio --vitc --wss 4:3", 4, 0),
    ("-m m -s 13500000 --filter --vitc", 4, 1),
    # VITS (chroma part mixed through the line's subcarrier table) and CEA-608 (run-in + null codes): stock stages too
    ("-m i -s 16000000 --filter --noaudio --vits", 4, 0),
    ("-m m -s 13500000 --filter --noaudio --vits --cc608", 4, 0),
    ("-m l -s 16000000 --filter --noaudio --vits", 4, 0),
    ("-m pal -s 16000000 --vits --cc608 --vitc --wss 16:9", 2, 0),
    # --pixelrate: raster at 13.5 MHz, the reference's polyphase resampler on the device, then the usual path
    ("-m i -s 16000000 --pixelrate 13500000 --filter --noaudio", 4, 0),
    ("-m i -s 16000000 --pixelrate 13500000 --filter", 4, 1),
    ("-m m -s 13500000 --pixelrate 9000000 --filter", 4, 1),          # W = 858 <- 572: pitched byte planes
    # HACKTV_B200_PREFETCH=1: the adapter's vid_next_line runs one frame ahead of the consumer
    ("PREFETCH -m i -s 16000000 --filter", 4, 1),
])
def test_same_cli_same_bytes(args, per, tol):
    env = ""
    if args.startswith("PREFETCH "):
        args, env = args[len("PREFETCH "):], "HACKTV_B200_PREFETCH=1 "
    w = 858 if "-s 13500000" in args else (1280 if "20000000" in args else 1024)
    lines = 1300 if w == 1024 else 1100
    a = _run(DROPIN, args, lines * w * per, env)
    b = _run(STOCK, args, lines * w * per)
    d = np.abs(a.astype(np.int32) - b.astype(np.int32))
    assert d.max() <= tol, f"max |diff| {d.max()}"


def test_readme_two_channel_pipeline():
    """README:89-90: one hacktv piped into another through --passthru; both stages on the GPU path
    against both stages stock."""
    def pipeline(binary, nbytes):
        with tempfile.NamedTemporaryFile("r", suffix=".stderr") as err:
            cmd = (f"timeout 120 {binary} -s 20000000 --offset -6750000 --level 0.5 --filter -o - test 2>>{err.name} | "
                   f"timeout 120 {binary} -s 20000000 --offset 1250000 --level 0.5 --passthru /dev/stdin --filter -o - test "
                   f"2>>{err.name} | head -c {nbytes}")
            out = subprocess.run(["bash", "-c", cmd], capture_output=True, timeout=300).stdout
            log = err.read()
        assert len(out) == nbytes, f"{binary}: got {len(out)} of {nbytes} bytes"
        assert log.count("Encoder: hacktv_b200") == (2 if binary == DROPIN else 0)
        return np.frombuffer(out, dtype=np.int16)
    n = 700 * 1280 * 4
    a = pipeline(DROPIN, n)
    b = pipeline(STOCK, n)
    d = np.abs(a.astype(np.int32) - b.astype(np.int32))
    assert d.max() <= 2, f"max |diff| {d.max()}"


def test_teletext_vitc_wss_through_the_stock_stages(tmp_path):
    """The reference's teletext (raw packet source: deterministic), VITC and WSS stages run inside the adapter in
    vid_init's order, vbialloc included (teletext skips the lines VITC took); 34 VBI lines per frame ride the
    encoder's overlay hook."""
    rng = np.random.default_rng(1)
    raw = tmp_path / "packets.t42"
    rng.integers(0, 256, size=42 * 500, dtype=np.uint8).tofile(raw)
    args = f"-m i -s 16000000 --filter --noaudio --teletext raw:{raw} --vitc --wss 16:9"
    n = 1900 * 1024 * 4
    a = _run(DROPIN, args, n)
    b = _run(STOCK, args, n)
    assert np.array_equal(a, b), f"{np.count_nonzero(a != b)} values differ"
    plain = _run(STOCK, "-m i -s 16000000 --filter --noaudio", n)
    changed = np.nonzero((b != plain).reshape(1900, -1).any(axis=1))[0]
    assert len(changed) > 90                                      # 3 frames x (32 teletext - 4 + 4 VITC + 1 WSS) lines
