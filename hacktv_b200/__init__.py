"""hacktv_b200 - Python view of the C-ABI in include/hacktv_b200.h.

The product is the shared library ``libhacktv_b200.so`` (C host layer + sm_90a
CUDA kernels). This module only loads it with ctypes and mirrors the
reference-facing call sequence (reference hacktv.c:1440-1601):

    enc = Encoder("i", 16_000_000, vfilter=True)   # vid_configs lookup + vid_init
    enc.open_test_source()                          # av_test_open
    iq = enc.render_host(625)                       # 625 x vid_next_line + rf_write
    enc.close()                                     # vid_free

There is no CPU fallback: without the built library, or without a CUDA device,
construction raises. Nothing here imports or links anything under ``oracle/``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# HTV_LIB: another build of the same library (A/B runs of compile-time variants, tools/occ_ab.sh)
LIB_PATH = os.environ.get("HTV_LIB") or os.path.join(_HERE, "libhacktv_b200.so")

HTV_OK, HTV_ERROR, HTV_OUT_OF_MEMORY = 0, -1, -2

# sample types of the rendered stream, hacktv's -t/--type (include/hacktv_b200.h HTV_TYPE_*), and their numpy dtypes
SAMPLE_TYPES = {"uint8": 0, "int8": 1, "uint16": 2, "int16": 3, "int32": 4, "float": 5}
SAMPLE_DTYPES = {"uint8": np.uint8, "int8": np.int8, "uint16": np.uint16, "int16": np.int16, "int32": np.int32,
                 "float": np.float32}


def _type_code(sample_type: str) -> int:
    if sample_type not in SAMPLE_TYPES:
        raise ValueError(f"unknown sample type {sample_type!r}: one of {', '.join(SAMPLE_TYPES)}")
    return SAMPLE_TYPES[sample_type]


class Config(C.Structure):
    """htv_config_t (include/hacktv_b200.h) = the hot-path subset of vid_config_t."""

    _fields_ = [
        ("output_type", C.c_int32), ("modulation", C.c_int32),
        ("video_bw", C.c_double), ("vsb_upper_bw", C.c_double), ("vsb_lower_bw", C.c_double),
        ("level", C.c_double),
        ("swap_iq", C.c_int32), ("invert_video", C.c_int32), ("offset", C.c_int64),
        ("video_level", C.c_double), ("fm_mono_level", C.c_double),
        ("am_audio_level", C.c_double), ("nicam_level", C.c_double),
        ("type", C.c_int32), ("lines", C.c_int32),
        ("frame_rate_num", C.c_int64), ("frame_rate_den", C.c_int64),
        ("hline", C.c_int32), ("interlaced", C.c_int32), ("active_lines", C.c_int32), ("vfilter", C.c_int32),
        ("hsync_width", C.c_double), ("vsync_short_width", C.c_double),
        ("vsync_long_width", C.c_double), ("sync_rise", C.c_double),
        ("white_level", C.c_double), ("black_level", C.c_double),
        ("blanking_level", C.c_double), ("sync_level", C.c_double),
        ("active_width", C.c_double), ("active_left", C.c_double), ("gamma", C.c_double),
        ("rw_co", C.c_double), ("gw_co", C.c_double), ("bw_co", C.c_double),
        ("colour_mode", C.c_int32), ("volume", C.c_int32),
        ("colour_carrier_num", C.c_int64), ("colour_carrier_den", C.c_int64),
        ("colour_bw", C.c_double), ("burst_width", C.c_double), ("burst_left", C.c_double),
        ("burst_level", C.c_double), ("burst_rise", C.c_double),
        ("ev_co", C.c_double), ("eu_co", C.c_double),
        ("fm_mono_carrier", C.c_double), ("fm_mono_deviation", C.c_double),
        ("fm_mono_preemph", C.c_int32), ("reserved0", C.c_int32),
        ("nicam_carrier", C.c_double), ("nicam_beta", C.c_double), ("am_mono_carrier", C.c_double),
        ("fm_level", C.c_double), ("fm_deviation", C.c_double), ("fm_energy_dispersal", C.c_double),
    ]

    def copy(self) -> "Config":
        c = Config()
        C.memmove(C.byref(c), C.byref(self), C.sizeof(Config))
        return c


class _Mode(C.Structure):
    _fields_ = [("id", C.c_char_p), ("conf", C.POINTER(Config)), ("desc", C.c_char_p)]


class Frame(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("framebuffer", C.c_void_p), ("serial", C.c_uint64)]


_READ_VIDEO = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(Frame))
_READ_AUDIO = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t))
_PASSTHRU_READ = C.CFUNCTYPE(C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t)


class SecamChain(C.Structure):
    """htv_secam_chain_t"""
    _fields_ = [(n, C.c_int64) for n in ("launches", "passes", "final_odd", "final_even", "recomputed", "listed_warp",
                                         "listed_thread", "repredict_odd", "repredict_even")] + \
               [("passes_max", C.c_int32), ("list_max", C.c_int32)]


class VbiLine(C.Structure):
    """htv_vbi_line_t"""
    _fields_ = [("line", C.c_int), ("replace_from", C.c_int), ("replace_to", C.c_int), ("replace_value", C.c_int),
                ("add", C.c_void_p)]


_READ_VBI = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.POINTER(C.POINTER(VbiLine)), C.POINTER(C.c_int))
_CLOSE = C.CFUNCTYPE(C.c_int, C.c_void_p)


class AV(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("ctx", C.c_void_p),
                ("read_video", _READ_VIDEO), ("read_audio", _READ_AUDIO), ("close", _CLOSE)]


class Line(C.Structure):
    _fields_ = [("output", C.POINTER(C.c_int16)), ("width", C.c_int), ("frame", C.c_int), ("line", C.c_int)]


_lib = None


def build(verbose: bool = False) -> str:
    """Compile the C host layer and the sm_90a kernels in-tree (csrc/Makefile)."""
    r = subprocess.run(["make", "-C", os.path.join(_HERE, "csrc")], capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout[-4000:])
        print(r.stderr[-4000:])
    if r.returncode != 0:
        raise RuntimeError("hacktv_b200: build failed")
    return LIB_PATH


def lib() -> C.CDLL:
    """Load libhacktv_b200.so (raises if it has not been built - no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"hacktv_b200: {LIB_PATH} is missing - run `make -C hacktv_b200/csrc` "
                           "(or __graft_entry__.build()); there is no CPU fallback")
    L = C.CDLL(LIB_PATH)
    vp, i64, sz = C.c_void_p, C.c_int64, C.c_size_t
    L.htv_find_mode.restype = C.POINTER(Config); L.htv_find_mode.argtypes = [C.c_char_p]
    L.htv_config_size.restype = sz
    L.htv_init.restype = C.c_int; L.htv_init.argtypes = [C.POINTER(vp), C.c_uint, C.c_uint, C.POINTER(Config)]
    L.htv_init_on.restype = C.c_int; L.htv_init_on.argtypes = [C.POINTER(vp), C.c_int, C.c_uint, C.c_uint, C.POINTER(Config)]
    L.htv_device_count.restype = C.c_int; L.htv_device_count.argtypes = []
    L.htv_device.restype = C.c_int; L.htv_device.argtypes = [vp]
    L.htv_free.restype = None; L.htv_free.argtypes = [vp]
    L.htv_info.restype = None; L.htv_info.argtypes = [vp]
    L.htv_get_framebuffer_length.restype = sz; L.htv_get_framebuffer_length.argtypes = [vp]
    L.htv_av.restype = C.POINTER(AV); L.htv_av.argtypes = [vp]
    L.htv_av_test_open.restype = C.c_int; L.htv_av_test_open.argtypes = [C.POINTER(AV)]
    L.htv_av_close.restype = None; L.htv_av_close.argtypes = [C.POINTER(AV)]
    L.htv_av_memory_open.restype = C.c_int
    L.htv_av_memory_open.argtypes = [C.POINTER(AV), vp, sz, vp, sz, sz, C.c_int]
    L.htv_next_line.restype = C.POINTER(Line); L.htv_next_line.argtypes = [vp]
    L.htv_set_prefetch.restype = C.c_int; L.htv_set_prefetch.argtypes = [vp, C.c_int]
    L.htv_render.restype = C.c_int; L.htv_render.argtypes = [vp, C.c_int, vp, C.POINTER(sz), vp]
    L.htv_render_host.restype = C.c_int; L.htv_render_host.argtypes = [vp, C.c_int, vp, C.POINTER(sz)]
    L.htv_render_add.restype = C.c_int; L.htv_render_add.argtypes = [vp, C.c_int, vp, C.POINTER(sz), vp]
    L.htv_mix_add.restype = C.c_int; L.htv_mix_add.argtypes = [vp, vp, sz, vp]
    L.htv_set_sample_type.restype = C.c_int; L.htv_set_sample_type.argtypes = [vp, C.c_int]
    L.htv_sample_type.restype = C.c_int; L.htv_sample_type.argtypes = [vp]
    L.htv_convert.restype = C.c_int; L.htv_convert.argtypes = [vp, C.c_int, vp, sz, vp]
    L.htv_set_passthru.restype = C.c_int; L.htv_set_passthru.argtypes = [vp, _PASSTHRU_READ, vp]
    L.htv_passthru_delay_lines.restype = C.c_int; L.htv_passthru_delay_lines.argtypes = [vp]
    L.htv_set_vbi_source.restype = C.c_int; L.htv_set_vbi_source.argtypes = [vp, _READ_VBI, vp]
    for f in ("htv_samples_per_line", "htv_active_width", "htv_active_lines", "htv_lines_per_frame",
              "htv_sample_rate", "htv_is_complex", "htv_bytes_per_sample"):
        getattr(L, f).restype = C.c_int; getattr(L, f).argtypes = [vp]
    L.htv_lines_rendered.restype = i64; L.htv_lines_rendered.argtypes = [vp]
    L.htv_kernel_launches.restype = C.c_uint64; L.htv_kernel_launches.argtypes = [vp]
    L.htv_line_kernel.restype = C.c_char_p; L.htv_line_kernel.argtypes = [vp]
    L.htv_secam_chain.restype = C.c_int; L.htv_secam_chain.argtypes = [vp, C.POINTER(SecamChain)]
    L.htv_set_kernel_timing.restype = None; L.htv_set_kernel_timing.argtypes = [vp, C.c_int]
    L.htv_last_line_kernel_ms.restype = C.c_float; L.htv_last_line_kernel_ms.argtypes = [vp]
    L.htv_last_line_kernel_lines.restype = C.c_int; L.htv_last_line_kernel_lines.argtypes = [vp]
    L.htv_tables_create.restype = vp; L.htv_tables_create.argtypes = [C.POINTER(Config), C.c_uint]
    L.htv_tables_create2.restype = vp; L.htv_tables_create2.argtypes = [C.POINTER(Config), C.c_uint, C.c_uint]
    L.htv_tables_free.restype = None; L.htv_tables_free.argtypes = [vp]
    L.htv_tables_get.restype = C.POINTER(C.c_int32); L.htv_tables_get.argtypes = [vp, C.c_char_p, C.POINTER(C.c_int)]
    L.htv_test_pattern.restype = None; L.htv_test_pattern.argtypes = [C.c_int, C.c_int, vp]
    L.htv_test_tone_pairs.restype = sz
    L.htv_test_tone.restype = None; L.htv_test_tone.argtypes = [vp]
    L.htv_version.restype = C.c_char_p
    _lib = L
    return L


def modes() -> dict:
    """id -> (Config copy, description), the in-scope rows of the reference's vid_configs[]."""
    L = lib()
    arr = (_Mode * 64).in_dll(L, "htv_modes")
    out = {}
    for m in arr:
        if not m.id:
            break
        out[m.id.decode()] = (m.conf.contents.copy(), m.desc.decode())
    return out


def mode_config(mode: str, *, vfilter=False, nocolour=False, noaudio=False, nonicam=False,
                offset=0, swap_iq=False, level=1.0, volume=1.0, invert_video=False, deviation=0.0) -> Config:
    """Mode lookup + the command-line overrides of reference hacktv.c:1107-1437 (in-scope options)."""
    p = lib().htv_find_mode(mode.encode())
    if not p:
        raise ValueError(f"Unrecognised TV mode {mode!r}")
    c = p.contents.copy()
    if nocolour and c.colour_mode in (1, 2, 3):
        c.colour_mode = 0
    if noaudio:
        c.fm_mono_level = c.am_audio_level = c.nicam_level = 0.0
        c.fm_mono_carrier = c.nicam_carrier = c.am_mono_carrier = 0.0
    if nonicam:
        c.nicam_level = 0.0
        c.nicam_carrier = 0.0
    c.level *= float(np.float32(level))
    if vfilter:
        c.vfilter = 1
    c.swap_iq = int(bool(swap_iq))
    c.offset = int(offset)
    c.volume = int(float(np.float32(volume)) * 256 + 0.5)
    c.invert_video = int(bool(invert_video))
    if deviation > 0:
        c.fm_deviation = float(deviation)            # -D / --deviation, hacktv.c:1109-1113
    return c


class Tables:
    """Host-only table generation (no GPU needed) - htv_tables_* in the C-ABI."""

    def __init__(self, conf: Config, sample_rate: int, pixel_rate: int = 0):
        self._L = lib()
        self._t = self._L.htv_tables_create2(C.byref(conf), sample_rate, pixel_rate)
        if not self._t:
            raise RuntimeError("htv_tables_create failed")

    def get(self, name: str):
        n = C.c_int(0)
        p = self._L.htv_tables_get(self._t, name.encode(), C.byref(n))
        if not p:
            return None
        return np.ctypeslib.as_array(p, shape=(n.value,)).copy()

    def close(self):
        if self._t:
            self._L.htv_tables_free(self._t)
            self._t = None

    def __del__(self):
        self.close()


class Encoder:
    """htv_t: one RF channel on one CUDA device (htv_init_on; device None = the current one)."""

    def __init__(self, mode, sample_rate: int = 16_000_000, pixel_rate: int = 0, device: int | None = None, **overrides):
        """pixel_rate != 0 and != sample_rate: the raster is built at pixel_rate and resampled to
        sample_rate in front of the video filter (hacktv's --pixelrate)."""
        self._L = lib()
        self.conf = mode if isinstance(mode, Config) else mode_config(mode, **overrides)
        h = C.c_void_p()
        r = self._L.htv_init_on(C.byref(h), -1 if device is None else int(device), sample_rate, pixel_rate, C.byref(self.conf))
        if r != HTV_OK or not h:
            raise RuntimeError(f"htv_init failed ({r}): no CUDA device or unsupported configuration")
        self._h = h
        self.device = self._L.htv_device(h)
        self.width = self._L.htv_samples_per_line(h)
        self.lines = self._L.htv_lines_per_frame(h)
        self.active_width = self._L.htv_active_width(h)
        self.active_lines = self._L.htv_active_lines(h)
        self.complex = bool(self._L.htv_is_complex(h))
        self.bytes_per_sample = self._L.htv_bytes_per_sample(h)
        self._sample_type = "int16"
        self.sample_rate = sample_rate
        self._keep = []

    # ---- sources -------------------------------------------------------
    def open_test_source(self):
        r = self._L.htv_av_test_open(self._L.htv_av(self._h))
        if r != HTV_OK:
            raise RuntimeError("htv_av_test_open failed")

    def set_source(self, frames: np.ndarray | None, audio: np.ndarray | None, *, audio_block: int = 0,
                   static_video: bool = False):
        """Install numpy-backed callbacks: frames uint32 [n, active_lines, active_width] used
        cyclically one per video frame, audio int16 [n, 2] (32 kHz stereo) used cyclically."""
        av = self._L.htv_av(self._h).contents
        state = {"f": 0, "a": 0}
        if frames is not None:
            frames = np.ascontiguousarray(frames, dtype=np.uint32)
            assert frames.shape[1:] == (self.active_lines, self.active_width), frames.shape

            def read_video(ctx, fr):
                i = state["f"] % frames.shape[0]
                fr.contents.width = self.active_width
                fr.contents.height = self.active_lines
                fr.contents.framebuffer = frames[i].ctypes.data
                fr.contents.serial = 1 if static_video else state["f"] + 1
                state["f"] += 1
                return HTV_OK
            cb = _READ_VIDEO(read_video)
            av.read_video = cb
            self._keep += [cb, frames]
        if audio is not None:
            audio = np.ascontiguousarray(audio, dtype=np.int16)
            assert audio.ndim == 2 and audio.shape[1] == 2
            blk = audio_block or audio.shape[0]

            def read_audio(ctx, samples, n):
                at = state["a"]
                m = min(blk, audio.shape[0] - at)
                samples[0] = audio[at:].ctypes.data
                n[0] = m
                state["a"] = (at + m) % audio.shape[0]
                return HTV_OK
            cb = _READ_AUDIO(read_audio)
            av.read_audio = cb
            self._keep += [cb, audio]

    def open_memory_source(self, frames: np.ndarray | None, audio: np.ndarray | None, *, audio_block: int = 0,
                           static_video: bool = False):
        """htv_av_memory_open: the same as set_source but served by C code (no interpreter in the
        per-frame path). Arrays must stay alive and unchanged in place; they are used as they are."""
        fp, nf, ap, na = None, 0, None, 0
        if frames is not None:
            assert frames.dtype == np.uint32 and frames.flags["C_CONTIGUOUS"]
            assert frames.shape[1:] == (self.active_lines, self.active_width), frames.shape
            fp, nf = C.c_void_p(frames.ctypes.data), frames.shape[0]
            self._keep.append(frames)
        if audio is not None:
            assert audio.dtype == np.int16 and audio.flags["C_CONTIGUOUS"] and audio.shape[1] == 2
            ap, na = C.c_void_p(audio.ctypes.data), audio.shape[0]
            self._keep.append(audio)
        r = self._L.htv_av_memory_open(self._L.htv_av(self._h), fp, nf, ap, na, audio_block, int(static_video))
        if r != HTV_OK:
            raise RuntimeError("htv_av_memory_open failed")

    # ---- rendering -----------------------------------------------------
    def render(self, nlines: int, device_ptr: int, stream: int = 0) -> int:
        """htv_render: next nlines into DEVICE memory, asynchronous on `stream`."""
        n = C.c_size_t(0)
        r = self._L.htv_render(self._h, nlines, C.c_void_p(device_ptr), C.byref(n), C.c_void_p(stream))
        if r != HTV_OK:
            raise RuntimeError(f"htv_render failed ({r})")
        return n.value

    def render_add(self, nlines: int, device_ptr: int, stream: int = 0) -> int:
        """htv_render_add: next nlines ADDED (int16 wrap) into the stream already in DEVICE memory."""
        n = C.c_size_t(0)
        r = self._L.htv_render_add(self._h, nlines, C.c_void_p(device_ptr), C.byref(n), C.c_void_p(stream))
        if r != HTV_OK:
            raise RuntimeError(f"htv_render_add failed ({r})")
        return n.value

    def set_passthru(self, iq: np.ndarray):
        """htv_set_passthru over an in-memory int16 [n, 2] stream (ref --passthru <file>)."""
        iq = np.ascontiguousarray(iq, dtype=np.int16)
        assert iq.ndim == 2 and iq.shape[1] == 2
        state = {"at": 0}

        def read(ctx, dst, ncomplex):
            n = min(int(ncomplex), iq.shape[0] - state["at"])
            if n > 0:
                C.memmove(dst, iq[state["at"]:].ctypes.data, n * 4)
                state["at"] += n
            return max(n, 0)
        cb = _PASSTHRU_READ(read)
        self._keep += [cb, iq]
        r = self._L.htv_set_passthru(self._h, cb, None)
        if r != HTV_OK:
            raise RuntimeError("htv_set_passthru failed (it must precede the first rendered line)")

    def set_vbi_lines(self, lines, every=1):
        """htv_set_vbi_source with a fixed set of overlays: `lines` = [(line, add or None, (from, to, value))],
        reported for every `every`-th frame (1 = all frames)."""
        arr = (VbiLine * len(lines))()
        for i, (line, add, rep) in enumerate(lines):
            arr[i].line = line
            arr[i].replace_from, arr[i].replace_to, arr[i].replace_value = rep
            if add is not None:
                add = np.ascontiguousarray(add, dtype=np.int16)
                assert add.size == self.width
                self._keep.append(add)
                arr[i].add = add.ctypes.data
        n = len(lines)

        def read(ctx, frame, out, count):
            if (frame - 1) % every:
                count[0] = 0
                return HTV_OK
            out[0] = C.cast(arr, C.POINTER(VbiLine))
            count[0] = n
            return HTV_OK
        cb = _READ_VBI(read)
        self._keep += [cb, arr]
        if self._L.htv_set_vbi_source(self._h, cb, None) != HTV_OK:
            raise RuntimeError("htv_set_vbi_source failed")

    @property
    def passthru_delay_lines(self) -> int:
        return int(self._L.htv_passthru_delay_lines(self._h))

    def set_sample_type(self, sample_type: str):
        """htv_set_sample_type: what render / render_host write from now on ("uint8", "int8", "uint16", "int16",
        "int32" or "float", converted as hacktv's -t/--type converts). Only before the first rendered line."""
        if self._L.htv_set_sample_type(self._h, _type_code(sample_type)) != HTV_OK:
            raise RuntimeError("htv_set_sample_type failed (it must precede the first rendered line)")
        self._sample_type = sample_type
        self.bytes_per_sample = self._L.htv_bytes_per_sample(self._h)

    @property
    def sample_type(self) -> str:
        """The sample type render / render_host write (set_sample_type); "int16" by default."""
        return self._sample_type

    def render_host(self, nlines: int, out: np.ndarray | None = None) -> np.ndarray:
        """htv_render_host: next nlines into host memory (what `-o file -t <sample_type>` would hold), as an array of
        the sample type's dtype."""
        per = 2 if self.complex else 1
        dtype = SAMPLE_DTYPES[self._sample_type]
        if out is None:
            out = np.empty(nlines * self.width * per, dtype=dtype)
        assert out.dtype == dtype and out.size >= nlines * self.width * per
        r = self._L.htv_render_host(self._h, nlines, C.c_void_p(out.ctypes.data), None)
        if r != HTV_OK:
            raise RuntimeError(f"htv_render_host failed ({r})")
        return out

    def render_host_ptr(self, nlines: int, host_ptr: int):
        r = self._L.htv_render_host(self._h, nlines, C.c_void_p(host_ptr), None)
        if r != HTV_OK:
            raise RuntimeError(f"htv_render_host failed ({r})")

    def set_prefetch(self, on: bool = True):
        """htv_set_prefetch: htv_next_line renders the following frame while the current one is consumed."""
        if self._L.htv_set_prefetch(self._h, int(on)) != HTV_OK:
            raise RuntimeError("htv_set_prefetch failed")

    def next_line(self):
        p = self._L.htv_next_line(self._h)
        if not p:
            return None
        l = p.contents
        return np.ctypeslib.as_array(l.output, shape=(l.width * 2,)).copy(), l.frame, l.line

    @property
    def kernel_launches(self) -> int:
        return int(self._L.htv_kernel_launches(self._h))

    @property
    def line_kernel(self) -> str:
        """The line kernel(s) the most recent render launched, with their template arguments (htv_line_kernel)."""
        return self._L.htv_line_kernel(self._h).decode()

    @property
    def secam_chain(self) -> dict:
        """What the SECAM chain did since the encoder was created, summed over its launches (htv_secam_chain): launches,
        passes, passes_max, final_odd / final_even, recomputed, listed_warp / listed_thread, list_max,
        repredict_odd / repredict_even. All zero for other colour modes."""
        c = SecamChain()
        if self._L.htv_secam_chain(self._h, C.byref(c)) != HTV_OK:
            raise RuntimeError("htv_secam_chain failed")
        return {name: int(getattr(c, name)) for name, _ in SecamChain._fields_}

    def set_kernel_timing(self, on: bool):
        self._L.htv_set_kernel_timing(self._h, int(on))

    def last_line_kernel_ms(self) -> float:
        return float(self._L.htv_last_line_kernel_ms(self._h))

    def last_line_kernel_lines(self) -> int:
        return int(self._L.htv_last_line_kernel_lines(self._h))

    def close(self):
        if getattr(self, "_h", None):
            self._L.htv_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def mix_add(acc_ptr: int, in_ptr: int, nvalues: int, stream: int = 0):
    """htv_mix_add: acc[i] += in[i] (int16 wrap) over device memory."""
    r = lib().htv_mix_add(C.c_void_p(acc_ptr), C.c_void_p(in_ptr), nvalues, C.c_void_p(stream))
    if r != HTV_OK:
        raise RuntimeError(f"htv_mix_add failed ({r})")


def convert(dst_ptr: int, sample_type: str, src_ptr: int, nvalues: int, stream: int = 0):
    """htv_convert: dst[i] = src[i] (int16, device memory) as `sample_type`, stream-ordered on `stream`; both
    pointers 16-byte aligned. For a stream that already exists, e.g. a wideband sum built with render_add."""
    r = lib().htv_convert(C.c_void_p(dst_ptr), _type_code(sample_type), C.c_void_p(src_ptr), nvalues, C.c_void_p(stream))
    if r != HTV_OK:
        raise RuntimeError(f"htv_convert failed ({r})")


def test_pattern(width: int, height: int) -> np.ndarray:
    out = np.zeros((height, width), dtype=np.uint32)
    lib().htv_test_pattern(width, height, C.c_void_p(out.ctypes.data))
    return out


def test_tone() -> np.ndarray:
    n = lib().htv_test_tone_pairs()
    out = np.zeros((n, 2), dtype=np.int16)
    lib().htv_test_tone(C.c_void_p(out.ctypes.data))
    return out
