"""The composite store of the fused line kernel (k_compose, htv_kernels.cu): every line of the frame as the finished
composite row - template, Y, the low-passed chroma on the subcarrier, burst - per picture and per colour-frame phase
f0 mod P, converted when the frames of a call first show a (picture, phase) pair.

Without a GPU: P for every mode at the rates the line kernels take, and that a line's subcarrier offset, V-switch and
burst code are the same in every frame of one phase, so that one row stands for all of them. On the GPU, against the
oracle, bit-exact without sound: a live source whose pictures stay up for 1, 3, 5 and 9 frames, slots reused while
other phases of them are still shown, calls that start mid-frame, on frame boundaries and at stream line 0, S-Video,
NTSC (P = 2) and mono (P = 1)."""
import math

import numpy as np
import pytest

import orc
import sv_oracle

PAL, NTSC = 1, 2


def _rates(lines):
    """Whole-Msps rates across the line kernels' range, rates of a whole number of samples per line, and two that are
    neither (4 x the PAL subcarrier, 20.05 Msps)."""
    fh = 15625 if lines == 625 else 30000 / 1001 * 525
    return [6000000, 10000000, 13500000, 16000000, 20000000, 24000000, 17734475, 20050000] + \
        [int(round(W * fh)) for W in (400, 858, 1135)]


def _phase_fields(codes, lines, W, cw, colour, f0, line):
    """k_line_desc_r's V-switch and subcarrier offset of `line` (1-based) in 0-based frame f0 (ref video.c:2906-2910,
    3011-3040)."""
    frame, L = f0 + 1, f0 * lines + line - 1
    b = (int(codes[line]) >> 5) & 3
    pal = int(b == 1 or (b == 2 and frame % 2 == 0) or (b == 3 and frame % 2 == 1))
    if colour == PAL and pal and (frame + line) % 2:
        pal = -1
    return pal, (L * W) % cw


def test_colour_frame_phases_of_every_mode(built):
    """P = the period of lines W mod clut_width, with the frame parity of the V-switch and the burst codes: 4 for the
    PAL family, 2 for NTSC, 1 without colour, at every rate; and a row of phase p holds the subcarrier offset, V-switch
    and burst code of every frame f0 with f0 mod P = p. Where the line is no whole number of samples, or the carrier no
    quarter-line multiple of the line rate (PAL-60), the subcarrier does not repeat within 4 frames: P = 0, and the
    encoder keeps the converted picture store and the subcarrier stage in k_line."""
    H = built
    checked = aperiodic = 0
    for mode in sorted(H.modes()):
        conf = H.mode_config(mode)
        for rate in _rates(conf.lines):
            try:
                t = H.Tables(conf, rate)
            except RuntimeError:
                continue                                         # not on the accelerated path at this rate
            P, cw = (int(v) for v in t.get("comp_phases"))
            W = int(t.get("geometry")[0])
            codes = t.get("codes")
            t.close()
            if conf.colour_mode not in (PAL, NTSC):
                assert P == 1, (mode, rate, P)
                continue
            period = cw // math.gcd(cw, conf.lines * W % cw or cw)
            want = period if period % 2 == 0 else 2 * period
            assert P == (want if want <= 4 else 0), (mode, rate, P, period)
            if P == 0:
                aperiodic += 1                                   # no composite store: k_line's PS forms
                continue
            for line in range(1, conf.lines + 1, 7):
                for f0 in range(3 * P):
                    assert _phase_fields(codes, conf.lines, W, cw, conf.colour_mode, f0, line) == \
                        _phase_fields(codes, conf.lines, W, cw, conf.colour_mode, f0 % P, line), (mode, rate, f0, line)
            checked += 1
    assert checked >= 40 and aperiodic > 0


def test_ntsc_and_pal_phase_counts(built):
    H = built
    for mode, rate, want in (("i", 16000000, 4), ("pal", 20000000, 4), ("pal-m", 13500000, 4), ("m", 13500000, 2),
                             ("ntsc", 13500000, 2), ("pal60", 13500000, 0), ("ntsc", 16000000, 0), ("pal", 20050000, 0)):
        t = H.Tables(H.mode_config(mode), rate)
        assert int(t.get("comp_phases")[0]) == want, mode
        t.close()
    t = H.Tables(H.mode_config("i", nocolour=True), 16000000)
    assert int(t.get("comp_phases")[0]) == 1
    t.close()


# ---- on the GPU ---------------------------------------------------------------------------------------------------

def _pictures(H, conf, rate, n, seed):
    t = H.Tables(conf, rate)
    aw = int(t.get("geometry")[3])
    t.close()
    rng = np.random.default_rng(seed)
    return rng.integers(0, 1 << 24, size=(n, int(conf.active_lines), aw), dtype=np.uint32)


def _held_source(H, enc, pictures, hold):
    """A live source: picture k is up for frames k * hold .. k * hold + hold - 1 (a new serial when it changes); the
    pictures repeat after the last."""
    av = enc._L.htv_av(enc._h).contents
    state = {"f": 0}

    def read_video(ctx, fr):
        k = (state["f"] // hold) % pictures.shape[0]
        fr.contents.width = enc.active_width
        fr.contents.height = enc.active_lines
        fr.contents.framebuffer = pictures[k].ctypes.data
        fr.contents.serial = state["f"] // hold + 1
        state["f"] += 1
        return H.HTV_OK
    cb = H._READ_VIDEO(read_video)
    av.read_video = cb
    enc._keep += [cb, pictures]


def _frames_shown(pictures, hold, nframes):
    return np.stack([pictures[(f // hold) % pictures.shape[0]] for f in range(nframes)])


def _render_held(H, conf, rate, pictures, hold, pieces):
    enc = H.Encoder(conf, rate)
    _held_source(H, enc, pictures, hold)
    got = np.concatenate([enc.render_host(n) for n in pieces])
    name = enc.line_kernel
    enc.close()
    return got, name


def _oracle(conf, rate, frames, nlines):
    o = orc.Oracle(conf, rate)
    o.set_source(frames, None)
    want = o.render(nlines)
    o.close()
    return want


def _exact(got, want):
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} of {got.size} values differ from the oracle, first at {bad[0]}"


@pytest.mark.gpu
@pytest.mark.parametrize("hold", [1, 3, 5, 9])
def test_pictures_held_for_several_frames(built, hold):
    """Each picture is converted at the phases of the frames that show it, as they come: with hold 1 one phase per
    picture, with 5 and 9 every phase, some of them calls after the picture came up."""
    H = built
    conf = H.mode_config("i", vfilter=True, noaudio=True)
    rate = 16000000
    L = 625
    pictures = _pictures(H, conf, rate, 6, hold)
    pieces = [L + 11, 3 * L - 11, 2 * L + 300, 7 * L - 300, 1, 4 * L - 1, 6 * L]
    got, name = _render_held(H, conf, rate, pictures, hold, pieces)
    assert "k_line" in name
    nf = -(-sum(pieces) // L) + 1
    _exact(got, _oracle(conf, rate, _frames_shown(pictures, hold, nf), sum(pieces)))


@pytest.mark.gpu
def test_slots_reused_while_other_phases_are_shown(built):
    """21 pictures up for 2 frames each cycle through the 16 picture slots: a slot gets its next picture while the
    phases of the one before are still valid in other slots' neighbourhood, and calls of up to 7 new pictures convert
    two phases of each."""
    H = built
    conf = H.mode_config("i", vfilter=True, noaudio=True)
    rate = 16000000
    L = 625
    pictures = _pictures(H, conf, rate, 21, 7)
    pieces = [14 * L + 5, 3 * L, 9 * L - 5, L, 15 * L + 77, 2]
    got, _ = _render_held(H, conf, rate, pictures, 2, pieces)
    nf = -(-sum(pieces) // L) + 1
    _exact(got, _oracle(conf, rate, _frames_shown(pictures, 2, nf), sum(pieces)))


@pytest.mark.gpu
@pytest.mark.parametrize("pieces", [[1, 1, 623, 625, 1250], [625, 625, 1875, 1], [312, 313, 1251, 1250, 3]],
                         ids=["line0-single-lines", "frame-boundaries", "mid-frame"])
def test_calls_that_start_mid_frame_and_at_line_0(built, pieces):
    """The stream-start rows (the lines before the stream, stream line 0) and calls that begin on any line."""
    H = built
    conf = H.mode_config("i", vfilter=True, noaudio=True)
    rate = 16000000
    pictures = _pictures(H, conf, rate, 3, 11)
    got, _ = _render_held(H, conf, rate, pictures, 2, pieces)
    nf = -(-sum(pieces) // 625) + 1
    _exact(got, _oracle(conf, rate, _frames_shown(pictures, 2, nf), sum(pieces)))


@pytest.mark.gpu
@pytest.mark.parametrize("mode,rate,kw,P", [
    ("m", 13500000, dict(vfilter=True, noaudio=True), 2),
    ("ntsc", 13500000, dict(), 2),
    ("i", 16000000, dict(vfilter=True, noaudio=True, nocolour=True), 1),
    ("pal-m", 13500000, dict(vfilter=True, noaudio=True), 4),
], ids=["ntsc-m", "ntsc-baseband", "mono", "pal-m"])
def test_phase_counts_of_other_systems(built, mode, rate, kw, P):
    H = built
    conf = H.mode_config(mode, **kw)
    t = H.Tables(conf, rate)
    assert int(t.get("comp_phases")[0]) == P
    t.close()
    L = conf.lines
    pictures = _pictures(H, conf, rate, 4, 13)
    pieces = [L - 7, 2 * L + 7, 3 * L + 100, 3 * L - 100]
    got, _ = _render_held(H, conf, rate, pictures, 3, pieces)
    nf = -(-sum(pieces) // L) + 1
    _exact(got, _oracle(conf, rate, _frames_shown(pictures, 3, nf), sum(pieces)))


@pytest.mark.gpu
@pytest.mark.parametrize("mode,rate,kw", [("pal", 16000000, dict(s_video=True, vfilter=True)),
                                          ("ntsc", 13500000, dict(s_video=True))], ids=["pal", "ntsc"])
def test_s_video_chroma_plane_over_every_phase(built, mode, rate, kw):
    """S-Video reads Q from the store's chroma plane: held pictures over more frames than the phases."""
    H = built
    conf = H.mode_config(mode, **kw)
    L = conf.lines
    pictures = _pictures(H, conf, rate, 3, 17)
    pieces = [L + 3, 4 * L - 3, 2 * L + 50]
    got, name = _render_held(H, conf, rate, pictures, 2, pieces)
    assert name.endswith(",SV>"), name
    nf = -(-sum(pieces) // L) + 1
    want = sv_oracle.render(conf, rate, sum(pieces), source=(_frames_shown(pictures, 2, nf), None))
    _exact(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,rate,kw", [("m", 16000000, dict(vfilter=True, noaudio=True)),
                                          ("pal", 20050000, dict()),
                                          ("pal60", 13500000, dict(s_video=True))], ids=["ntsc-m-16M", "pal-20.05M", "pal60-sv"])
def test_subcarrier_that_does_not_repeat_within_4_frames(built, mode, rate, kw):
    """P = 0: no composite store, the converted picture store and the subcarrier in k_line. A live source over more than
    16 frames, so that picture slots are reused, in calls that cut frames."""
    H = built
    conf = H.mode_config(mode, **kw)
    t = H.Tables(conf, rate)
    assert int(t.get("comp_phases")[0]) == 0
    t.close()
    L = conf.lines
    pictures = _pictures(H, conf, rate, 19, 19)
    pieces = [L - 7, 5 * L + 7, 9 * L + 100, 6 * L - 100]
    got, name = _render_held(H, conf, rate, pictures, 1, pieces)
    nf = -(-sum(pieces) // L) + 1
    frames = _frames_shown(pictures, 1, nf)
    if kw.get("s_video"):
        assert name.endswith(",SV>"), name
        _exact(got, sv_oracle.render(conf, rate, sum(pieces), source=(frames, None)))
    else:
        _exact(got, _oracle(conf, rate, frames, sum(pieces)))
