"""The converted picture store of the fused line kernel (k_picture, htv_kernels.cu): every picture is converted once when
it arrives - line template, Y, and U / V through the chroma low-pass - and k_line reads each line's row of it. Against
the oracle, bit-exact without sound, with pictures that change every frame: through htv_render and htv_render_host, in
uneven calls that cut frames and reuse every one of the 16 picture slots, with a source that ends (its lines fall back
to the black slot), and with and without the interlaced raster's row shift (the half lines in every case)."""
import numpy as np
import pytest

import orc

pytestmark = pytest.mark.gpu

# (mode, rate, overrides, what the line kernel is)
CASES = [
    ("i", 16000000, dict(vfilter=True), "SND=37,WC=1024"),           # the bench form: PAL-I, VSB + FM + NICAM, W = 1024
    ("i", 16000000, dict(vfilter=True, noaudio=True), "MAXT=256"),   # the same picture path without sound: bit-exact
    ("m", 13500000, dict(vfilter=True, noaudio=True), "FULL=0"),     # NTSC-M, W = 858: a partial last tile
    ("i", 20000000, dict(vfilter=True, noaudio=True), "MAXT=320"),   # W = 1280, 320 threads
    ("i", 16000000, dict(vfilter=True, noaudio=True, nocolour=True), "MAXT=256"),   # mono: no chroma plane
]
IDS = ["pal-i-bench", "pal-i", "ntsc-m-858", "pal-i-20M", "mono"]


def _pictures(H, conf, rate, n, seed):
    t = H.Tables(conf, rate)
    aw, al = int(t.get("geometry")[3]), int(conf.active_lines)
    t.close()
    rng = np.random.default_rng(seed)
    return rng.integers(0, 1 << 24, size=(n, al, aw), dtype=np.uint32)


def _oracle(H, conf, rate, frames, nlines):
    o = orc.Oracle(conf, rate)
    o.set_source(frames, None)
    want = o.render(nlines)
    o.close()
    return want


def _check(got, want, sound):
    d = np.abs(got.astype(np.int32) - want.astype(np.int32))
    if sound:
        assert d.max() <= 1 and (d != 0).mean() < 0.01, (d.max(), (d != 0).mean())
    else:
        assert d.max() == 0, f"{np.count_nonzero(d)} of {d.size} values differ from the oracle"


def _ended_source(H, enc, frames):
    """A source that serves `frames` once, one per video frame, and then has no more pictures."""
    av = enc._L.htv_av(enc._h).contents
    state = {"f": 0}

    def read_video(ctx, fr):
        i = state["f"]
        if i >= frames.shape[0]:
            return H.HTV_ERROR
        fr.contents.width = enc.active_width
        fr.contents.height = enc.active_lines
        fr.contents.framebuffer = frames[i].ctypes.data
        fr.contents.serial = i + 1
        state["f"] += 1
        return H.HTV_OK
    cb = H._READ_VIDEO(read_video)
    av.read_video = cb
    enc._keep += [cb, frames]


@pytest.mark.parametrize("mode,rate,kw,form", CASES, ids=IDS)
def test_pictures_that_change_every_frame_in_uneven_calls(built, mode, rate, kw, form):
    """More than 16 distinct pictures, one per frame, in calls that start and end inside frames: every slot of the store
    is refilled while the calls before it are still in flight, and pictures change in the middle of a call."""
    H = built
    conf = H.mode_config(mode, **kw)
    enc = H.Encoder(conf, rate)
    frames = _pictures(H, conf, rate, 19, 1)
    enc.set_source(frames, None)
    L = enc.lines
    pieces = [L // 3, 2 * L + 17, 5 * L - 40, 1, 3 * L + 101, L - 78, 7 * L]
    got = np.concatenate([enc.render_host(n) for n in pieces])
    assert form in enc.line_kernel, enc.line_kernel
    enc.close()
    _check(got, _oracle(H, conf, rate, frames, sum(pieces)), "noaudio" not in kw)


@pytest.mark.parametrize("mode,rate,kw,form", CASES[1:4], ids=IDS[1:4])
def test_device_render_of_changing_pictures(built, mode, rate, kw, form):
    """htv_render into device memory, calls of uneven length on one stream, 18 pictures."""
    import torch
    H = built
    conf = H.mode_config(mode, **kw)
    enc = H.Encoder(conf, rate)
    frames = _pictures(H, conf, rate, 18, 2)
    enc.set_source(frames, None)
    L, W = enc.lines, enc.width
    per = 2 if enc.complex else 1
    # every call starts on a 16-byte boundary of the buffer: whole groups of 4 lines
    pieces = [n - n % 4 for n in (2 * L + 5, 3 * L - 11, L, 4 * L + 250, 9 * L - 244)]
    buf = torch.zeros(sum(pieces) * W * per, dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    at = 0
    for n in pieces:
        enc.render(n, buf.data_ptr() + at * W * per * 2, st)
        at += n
    torch.cuda.synchronize()
    got = buf.cpu().numpy()
    assert form in enc.line_kernel, enc.line_kernel
    enc.close()
    _check(got, _oracle(H, conf, rate, frames, sum(pieces)), False)


@pytest.mark.parametrize("mode,rate,kw,form", CASES, ids=IDS)
def test_source_that_ends_falls_back_to_black(built, mode, rate, kw, form):
    """Three pictures, then none: the rest of the stream is drawn from the black slot - which holds every line with a
    picture area, also those that show no source row."""
    H = built
    conf = H.mode_config(mode, **kw)
    enc = H.Encoder(conf, rate)
    frames = _pictures(H, conf, rate, 3, 3)
    _ended_source(H, enc, frames)
    L = enc.lines
    pieces = [L + 200, 2 * L, 3 * L - 200]
    got = np.concatenate([enc.render_host(n) for n in pieces])
    enc.close()
    # what the oracle renders for frames without a picture: black, as from an all-zero picture
    padded = np.concatenate([frames, np.zeros((3,) + frames.shape[1:], dtype=np.uint32)])
    _check(got, _oracle(H, conf, rate, padded, sum(pieces)), "noaudio" not in kw)


@pytest.mark.parametrize("mode,rate", [("i", 16000000), ("m", 13500000)], ids=["625", "525"])
def test_progressive_raster_rows_and_half_lines(built, mode, rate):
    """Every mode puts its picture on an interlaced raster, shifted down a row (the other tests); with `interlaced` off
    the rows are not shifted, and other rows and half lines carry the picture's edges. The 525-line raster still has
    lines with a picture area and no source row, drawn from the black slot's extra rows."""
    H = built
    conf = H.mode_config(mode, vfilter=True, noaudio=True)
    conf.interlaced = 0
    t = H.Tables(conf, rate)
    line_row = t.get("line_row")
    t.close()
    assert (line_row >= conf.active_lines).any() == (mode == "m")
    enc = H.Encoder(conf, rate)
    frames = _pictures(H, conf, rate, 5, 4)
    enc.set_source(frames, None)
    L = enc.lines
    pieces = [L - 3, 2 * L + 6, 2 * L - 3]
    got = np.concatenate([enc.render_host(n) for n in pieces])
    enc.close()
    _check(got, _oracle(H, conf, rate, frames, sum(pieces)), False)
