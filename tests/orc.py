"""ctypes binding of the parity oracle (oracle/liboracle.so) and the runner for the
prebuilt reference harness (oracle/_ref/ref_harness). TEST INFRASTRUCTURE ONLY: nothing
under hacktv_b200/ imports this."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_SO = os.path.join(ROOT, "oracle", "liboracle.so")
REF_HARNESS = os.path.join(ROOT, "oracle", "_ref", "ref_harness")
REF_HARNESS_RAW = os.path.join(ROOT, "oracle", "_ref", "ref_harness_rawheap")

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(ORACLE_SO):
            subprocess.run(["make", "-C", os.path.join(ROOT, "oracle")], check=True, capture_output=True)
        L = C.CDLL(ORACLE_SO)
        vp = C.c_void_p
        L.orc_params_size.restype = C.c_size_t
        L.orc_open.restype = vp; L.orc_open.argtypes = [vp, C.c_uint]
        L.orc_open2.restype = vp; L.orc_open2.argtypes = [vp, C.c_uint, C.c_uint]
        L.orc_close.restype = None; L.orc_close.argtypes = [vp]
        L.orc_set_ref_heap.restype = None; L.orc_set_ref_heap.argtypes = [vp, C.c_int]
        L.orc_set_frames.restype = None; L.orc_set_frames.argtypes = [vp, vp, C.c_int]
        L.orc_set_audio.restype = None; L.orc_set_audio.argtypes = [vp, vp, C.c_size_t]
        L.orc_set_passthru.restype = None; L.orc_set_passthru.argtypes = [vp, vp, C.c_size_t]
        L.orc_add_vbi_line.restype = None; L.orc_add_vbi_line.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp]
        L.orc_render.restype = C.c_size_t; L.orc_render.argtypes = [vp, C.c_int, vp]
        for f in ("orc_width", "orc_raster_width", "orc_active_width", "orc_active_lines", "orc_is_complex"):
            getattr(L, f).restype = C.c_int; getattr(L, f).argtypes = [vp]
        L.orc_table.restype = C.POINTER(C.c_int32); L.orc_table.argtypes = [vp, C.c_char_p, C.POINTER(C.c_int)]
        L.orc_test_pattern.restype = None; L.orc_test_pattern.argtypes = [C.c_int, C.c_int, vp]
        L.orc_test_tone_pairs.restype = C.c_size_t
        L.orc_test_tone.restype = None; L.orc_test_tone.argtypes = [vp]
        L.orc_yuv.restype = None; L.orc_yuv.argtypes = [vp, C.c_uint32, vp]
        _lib = L
    return _lib


class Oracle:
    """orc_t. `conf` is a hacktv_b200.Config: htv_config_t and orc_params_t share one layout
    (checked against orc_params_size())."""

    def __init__(self, conf, sample_rate, pixel_rate=0, ref_heap=False):
        """ref_heap: SECAM's luma notch reads what the reference left in its line buffers' padding, not zeros
        (orc_set_ref_heap); the reference's stream, where the CUDA path's differs near the picture's right edge."""
        L = lib()
        assert C.sizeof(conf) == L.orc_params_size(), "orc_params_t / htv_config_t layouts differ"
        self._L = L
        self._o = L.orc_open2(C.byref(conf), sample_rate, pixel_rate)
        if not self._o:
            raise RuntimeError("orc_open failed")
        L.orc_set_ref_heap(self._o, int(ref_heap))
        self.width = L.orc_width(self._o)
        self.raster_width = L.orc_raster_width(self._o)    # differs from width with a --pixelrate resampler
        self.active_width = L.orc_active_width(self._o)
        self.active_lines = L.orc_active_lines(self._o)
        self.complex = bool(L.orc_is_complex(self._o))
        self._keep = []

    def set_source(self, frames, audio):
        if frames is not None:
            frames = np.ascontiguousarray(frames, dtype=np.uint32)
            assert frames.shape[1:] == (self.active_lines, self.active_width)
            self._L.orc_set_frames(self._o, frames.ctypes.data, frames.shape[0])
            self._keep.append(frames)
        if audio is not None:
            audio = np.ascontiguousarray(audio, dtype=np.int16)
            self._L.orc_set_audio(self._o, audio.ctypes.data, audio.shape[0])
            self._keep.append(audio)

    def set_passthru(self, iq):
        """iq: int16 [n, 2] complex samples added to the output (ref --passthru)."""
        iq = np.ascontiguousarray(iq, dtype=np.int16)
        self._L.orc_set_passthru(self._o, iq.ctypes.data, iq.shape[0])
        self._keep.append(iq)

    def add_vbi_line(self, line, add=None, replace=(0, 0, 0)):
        """A VBI overlay on `line` (1-based) of every frame: I[from:to] = value, then I += add."""
        p = None
        if add is not None:
            add = np.ascontiguousarray(add, dtype=np.int16)
            assert add.size == self.raster_width
            self._keep.append(add)
            p = add.ctypes.data
        self._L.orc_add_vbi_line(self._o, line, replace[0], replace[1], replace[2], p)

    def open_test_source(self):
        self.set_source(test_pattern(self.active_width, self.active_lines)[None], test_tone())

    def render(self, nlines):
        out = np.empty(nlines * self.width * (2 if self.complex else 1), dtype=np.int16)
        n = self._L.orc_render(self._o, nlines, out.ctypes.data)
        assert n == out.size
        return out

    def table(self, name):
        n = C.c_int(0)
        p = self._L.orc_table(self._o, name.encode(), C.byref(n))
        if not p:
            return None
        return np.ctypeslib.as_array(p, shape=(n.value,)).copy()

    def yuv(self, rgb):
        out = np.zeros(3, dtype=np.int16)
        self._L.orc_yuv(self._o, rgb, out.ctypes.data)
        return out

    def close(self):
        if self._o:
            self._L.orc_close(self._o)
            self._o = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def test_pattern(w, h):
    out = np.zeros((h, w), dtype=np.uint32)
    lib().orc_test_pattern(w, h, out.ctypes.data)
    return out


def test_tone():
    n = lib().orc_test_tone_pairs()
    out = np.zeros((n, 2), dtype=np.int16)
    lib().orc_test_tone(out.ctypes.data)
    return out


def have_ref():
    return os.path.exists(REF_HARNESS)


def run_ref(mode, rate, lines, *, skip=0, vfilter=False, extra=(), frames=None, audio=None,
            audio_block=0, rawheap=False, timeout=600):
    """Run the UNMODIFIED reference (oracle/_ref) and return its emitted int16 stream."""
    with tempfile.TemporaryDirectory() as td:
        out = os.path.join(td, "ref.bin")
        cmd = ["timeout", str(timeout), REF_HARNESS_RAW if rawheap else REF_HARNESS, "-m", mode, "-s", str(rate),
               "--skip", str(skip), "--lines", str(lines), "-o", out]
        if vfilter:
            cmd.append("--filter")
        cmd += list(extra)
        if frames is not None:
            fn = os.path.join(td, "frames.bin")
            np.ascontiguousarray(frames, dtype=np.uint32).tofile(fn)
            cmd += ["--frames", fn]
        if audio is not None:
            fn = os.path.join(td, "audio.bin")
            np.ascontiguousarray(audio, dtype=np.int16).tofile(fn)
            cmd += ["--audio", fn]
            if audio_block:
                cmd += ["--audio-block", str(audio_block)]
        subprocess.run(cmd, check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        return np.fromfile(out, dtype=np.int16)
