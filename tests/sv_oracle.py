"""S-Video (`--s-video`, ref video.c:3031-3040, 3206-3228) composed from the parity oracle (oracle/, tests/orc.py).
TEST INFRASTRUCTURE ONLY: tests/test_s_video_host.py pins it to the reference's own S-Video streams
(tests/golden/golden_s_video.json), tests/test_gpu_zz_s_video.py compares the device with it.

S-Video moves the colour subcarrier term from I to Q and changes nothing else the oracle computes, so its stream
follows from streams the oracle already renders:
  - I is the mode rendered without colour (colour_mode 0; the raster's luma, sync and VBI overlays are the same
    whatever the colour system) through the mode's video filter: the filter runs on I only (ref video.c:3235-3248,
    one channel);
  - Q is the line's own subcarrier, unfiltered (ref video.c:2935-2939 sets it to 0 when the line is blanked): for PAL
    and NTSC the colour stream less the colourless one, both without filter and overlays (int16 wrap). SECAM's colour
    stream also has the 51-tap luma notch applied to the picture area of every line that carries a subcarrier
    (ref video.c:3206), which S-Video skips: there Q is the colour stream less the notched colourless line. Those lines
    are the ones whose burst run (burst_left .. active_left, which the notch does not reach) differs;
  - then the IQ swap and the offset mixer (ref video.c:3466-3515) on the pair, as the oracle runs them on complex
    modes (oracle/htv_oracle.c offset_line: the Q31 phasor from INT16_MAX, renormalised every 32 767 samples; with a
    video filter one line of its state is spent on the pipeline's fill line first)."""
import math

import numpy as np

import orc

I16MAX, I32MAX = 32767, 2147483647


def _plain(conf, rate, nlines, source, colour, vfilter, overlays):
    c = conf.copy()
    c.s_video = 0
    c.swap_iq = 0
    c.offset = 0
    c.vfilter = int(vfilter)
    if not colour:
        c.colour_mode = 0
    o = orc.Oracle(c, rate)
    if source is None:
        o.open_test_source()
    else:
        o.set_source(*source)
    for line, add, rep in overlays:
        o.add_vbi_line(line, add, rep)
    g = o.table("geometry")
    notch = o.table("secam_notch")
    out = o.render(nlines).astype(np.int32)
    o.close()
    return out.reshape(nlines, -1), g, notch


def _notch(rows, taps, al, aw):
    """The oracle's fir_block over the picture area, step 1: centred, zero beyond the area's left edge, the line's own
    samples beyond its right edge, >> 15 and saturated."""
    h = len(taps) // 2
    out = rows.copy()
    x = np.zeros((rows.shape[0], aw + 2 * h), dtype=np.int64)
    seg = rows[:, al:al + aw + h]                 # past the line end: the buffer's zero padding
    x[:, h:h + seg.shape[1]] = seg
    acc = np.zeros((rows.shape[0], aw), dtype=np.int64)
    for y in range(len(taps)):
        acc += x[:, y:y + aw] * int(taps[y])
    acc = ((acc.astype(np.int32)) >> 15)
    out[:, al:al + aw] = np.clip(acc, -32768, 32767)
    return out


def _lround(v):
    return int(math.floor(v + 0.5)) if v >= 0 else -int(math.floor(-v + 0.5))


def _offset_carrier(offset, rate, n, skip):
    """(bi, bq) of the offset mixer for n samples after `skip` (oracle/htv_oracle.c offset_line)."""
    d = 2.0 * math.pi / rate * offset
    di, dq = _lround(math.cos(d) * I32MAX), _lround(math.sin(d) * I32MAX)
    pi, pq, counter = I16MAX, 0, I16MAX
    bi = np.empty(n, dtype=np.int32)
    bq = np.empty(n, dtype=np.int32)
    for k in range(skip + n):
        pi, pq = (pi * di - pq * dq) >> 31, (pi * dq + pq * di) >> 31
        if k >= skip:
            bi[k - skip], bq[k - skip] = pi >> 16, pq >> 16
        counter -= 1
        if counter == 0:
            ra = math.atan2(pq, pi)
            pi, pq = _lround(math.cos(ra) * I32MAX), _lround(math.sin(ra) * I32MAX)
            counter = I16MAX
    return bi, bq


def _wrap16(v):
    return v.astype(np.int64).astype(np.int16)


def render(conf, rate, nlines, source=None, overlays=()):
    """The emitted int16 I,Q stream of nlines lines of an S-Video configuration (conf.s_video set or not: the
    composition is S-Video's). source: None for the test source, else (frames, audio) as orc.Oracle.set_source takes
    them; overlays: (line, add, (from, to, value)) as orc.Oracle.add_vbi_line takes them."""
    secam = conf.colour_mode == 3
    i_rows, _, _ = _plain(conf, rate, nlines, source, False, conf.vfilter, overlays)
    colour, g, notch = _plain(conf, rate, nlines, source, True, False, ())
    luma, _, _ = _plain(conf, rate, nlines, source, False, False, ())
    W, al, aw, bl = int(g[0]), int(g[2]), int(g[3]), int(g[4])
    base = luma
    if secam:
        # lines with a subcarrier: their burst run differs from the colourless line
        sub = (colour[:, bl:al] != luma[:, bl:al]).any(axis=1)
        base = np.where(sub[:, None], _notch(luma, notch, al, aw), luma)
    q_rows = _wrap16(colour - base).astype(np.int32)
    i, q = i_rows.reshape(-1), q_rows.reshape(-1)
    if conf.swap_iq:
        i, q = q, i
    if conf.offset != 0:
        bi, bq = _offset_carrier(conf.offset, rate, i.size, W if conf.vfilter else 0)
        ai, aq = _wrap16(i).astype(np.int64), _wrap16(q).astype(np.int64)
        i = ((ai * bi - aq * bq).astype(np.int32) >> 15)
        q = ((ai * bq + aq * bi).astype(np.int32) >> 15)
    out = np.empty(2 * i.size, dtype=np.int16)
    out[0::2], out[1::2] = _wrap16(i), _wrap16(q)
    return out
