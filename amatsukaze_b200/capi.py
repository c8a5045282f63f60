"""ctypes binding of the C ABI in include/amtk_b200.h (libamtk_b200.so).

Python here is plumbing only (device memory via torch, launching, multi-GPU process group); all compute is in
the CUDA library.  Importing this module fails loudly when the native library has not been built; creating a
Context fails loudly when there is no H100: there is no CPU fallback.
"""
import ctypes as C
import os
import numpy as np

PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(PKG, "lib", "libamtk_b200.so")

c_float_p = C.POINTER(C.c_float)
c_i32_p = C.POINTER(C.c_int32)
c_u8_p = C.POINTER(C.c_uint8)


class AmtkError(RuntimeError):
    pass


class ClipDesc(C.Structure):
    _fields_ = [("base", C.c_void_p), ("frame_stride", C.c_int64), ("off_u", C.c_int64), ("off_v", C.c_int64),
                ("width", C.c_int32), ("height", C.c_int32), ("pitch_y", C.c_int32), ("pitch_uv", C.c_int32),
                ("log_uvx", C.c_int32), ("log_uvy", C.c_int32), ("bytes_per_sample", C.c_int32),
                ("bits_per_sample", C.c_int32), ("num_frames", C.c_int32), ("on_device", C.c_int32)]


class LogoInfo(C.Structure):
    _fields_ = [("w", C.c_int32), ("h", C.c_int32), ("log_uvx", C.c_int32), ("log_uvy", C.c_int32),
                ("imgw", C.c_int32), ("imgh", C.c_int32), ("imgx", C.c_int32), ("imgy", C.c_int32),
                ("maskpixels", C.c_int32), ("count", C.c_int32), ("black_score", C.c_float)]


class CombParams(C.Structure):
    _fields_ = [("th_move_y", C.c_int32), ("th_shima_y", C.c_int32), ("th_lshima_y", C.c_int32),
                ("th_move_c", C.c_int32), ("th_shima_c", C.c_int32), ("th_lshima_c", C.c_int32)]

    def as_list(self):
        return [self.th_move_y, self.th_shima_y, self.th_lshima_y, self.th_move_c, self.th_shima_c, self.th_lshima_c]


class LogoFindParams(C.Structure):
    _fields_ = [("block", C.c_int32), ("var_ratio", C.c_float), ("mean_delta", C.c_float), ("margin", C.c_int32),
                ("min_blocks", C.c_int32)]


class TnrParams(C.Structure):
    _fields_ = [("temporal_distance", C.c_int32), ("threshold", C.c_int32), ("interlaced", C.c_int32)]


# every symbol include/amtk_b200.h declares: (name, restype, argtypes)
V = C.c_void_p
VP = C.POINTER(C.c_void_p)
SIGNATURES = [
    ("amtk_last_error", C.c_char_p, []),
    ("amtk_version", C.c_int, []),
    ("amtk_device_count", C.c_int, []),
    ("amtk_ctx_create", C.c_int, [C.c_int, V, VP]),
    ("amtk_ctx_destroy", None, [V]),
    ("amtk_ctx_synchronize", C.c_int, [V]),
    ("amtk_ctx_launch_count", C.c_int64, [V]),
    ("amtk_ctx_last_h2d_bytes", C.c_int64, [V]),
    ("amtk_ctx_set_kernel_timing", C.c_int, [V, C.c_int]),
    ("amtk_ctx_get_kernel_timing", C.c_int, [V, C.POINTER(C.c_double), C.POINTER(C.c_int64), C.c_int]),
    ("amtk_probe_read_ms", C.c_int, [V, V, C.c_size_t, C.c_int, C.POINTER(C.c_double)]),
    ("amtk_host_alloc", C.c_int, [C.c_size_t, VP]),
    ("amtk_host_free", None, [V]),
    ("amtk_device_alloc", C.c_int, [V, C.c_size_t, VP]),
    ("amtk_device_free", None, [V, V]),
    ("amtk_memcpy_h2d", C.c_int, [V, V, V, C.c_size_t]),
    ("amtk_memcpy_d2h", C.c_int, [V, V, V, C.c_size_t]),
    ("amtk_memcpy_d2d", C.c_int, [V, V, V, C.c_size_t]),
    ("amtk_logo_create", C.c_int, [V, c_float_p] + [C.c_int] * 8 + [VP]),
    ("amtk_logo_load", C.c_int, [V, C.c_char_p, VP, V]),
    ("amtk_logo_save", C.c_int, [V, C.c_char_p, C.c_char_p, C.c_int]),
    ("amtk_logo_destroy", None, [V]),
    ("amtk_logo_deint", C.c_int, [V, VP]),
    ("amtk_logo_field", C.c_int, [V, C.c_int, VP]),
    ("amtk_logo_create_mask", C.c_int, [V, C.c_float]),
    ("amtk_logo_get_info", C.c_int, [V, C.POINTER(LogoInfo)]),
    ("amtk_logo_get_tables", C.c_int, [V, c_float_p, c_u8_p, c_float_p, c_float_p]),
    ("amtk_logo_scan_frames", C.c_int, [V, C.POINTER(ClipDesc), VP, C.c_int, C.c_int, C.c_int, C.c_int, V, C.c_int]),
    ("amtk_logo_analyze_frames", C.c_int, [V, C.POINTER(ClipDesc), V, V, V, C.c_int, C.c_int, V, C.c_int]),
    ("amtk_logo_eval_fades", C.c_int, [V, C.POINTER(ClipDesc), V, c_float_p, C.c_int, C.c_int, C.c_int, V, C.c_int]),
    ("amtk_comb_default_params", None, [C.POINTER(CombParams)]),
    ("amtk_comb_frames", C.c_int, [V, C.POINTER(ClipDesc), C.POINTER(CombParams), C.c_int, C.c_int, V, C.c_int]),
    ("amtk_scan_comb_frames", C.c_int, [V, C.POINTER(ClipDesc), VP, C.c_int, C.POINTER(CombParams), C.c_int, C.c_int, V, V, C.c_int]),
    ("amtk_scan_comb_frames_pitch", C.c_int, [V, C.POINTER(ClipDesc), VP, C.c_int, C.POINTER(CombParams), C.c_int, C.c_int, C.c_int,
                                              V, V, C.c_int]),
    ("amtk_scan_create", C.c_int, [V, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, VP]),
    ("amtk_scan_destroy", None, [V]),
    ("amtk_scan_add_frames", C.c_int, [V, C.POINTER(ClipDesc), C.c_int, C.c_int, C.c_int, C.c_int, c_u8_p, c_u8_p]),
    ("amtk_scan_num_valid", C.c_int, [V]),
    ("amtk_scan_get_sums", C.c_int, [V, C.POINTER(C.c_double)]),
    ("amtk_scan_get_logo", C.c_int, [V, C.c_int, C.c_int, c_float_p]),
    ("amtk_scan_logo", C.c_int, [V, C.POINTER(ClipDesc), C.c_int, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, V]),
    ("amtk_weave_frames", C.c_int, [V, C.POINTER(ClipDesc), C.POINTER(ClipDesc), C.c_int, c_i32_p, c_i32_p, C.c_int, C.c_int]),
    ("amtk_erase_logo_frames", C.c_int, [V, C.POINTER(ClipDesc), V, C.c_int, C.c_int, c_float_p]),
    ("amtk_calc_fade2", None, [c_float_p, C.c_int, C.c_int, C.c_int, c_float_p, c_float_p]),
    ("amtk_calc_fade2_index", C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int]),
    ("amtk_group_create", C.c_int, [C.c_int, c_i32_p, VP]),
    ("amtk_group_destroy", None, [V]),
    ("amtk_group_size", C.c_int, [V]),
    ("amtk_group_ctx", V, [V, C.c_int]),
    ("amtk_group_numa_cpus", C.c_int, [V, C.c_int]),
    ("amtk_group_nccl_version", C.c_int, [V]),
    ("amtk_group_host_alloc", C.c_int, [V, C.c_int, C.c_size_t, VP]),
    ("amtk_group_scan_comb_streams", C.c_int, [V, C.POINTER(ClipDesc), VP, C.POINTER(CombParams), C.c_int]),
    ("amtk_group_fetch_results", C.c_int, [V, C.c_int, C.c_int, V, V]),
    ("amtk_group_synchronize", C.c_int, [V]),
    ("amtk_group_mark", C.c_int, [V, C.c_int]),
    ("amtk_group_elapsed_ms", C.c_int, [V, C.c_int, C.c_int, C.POINTER(C.c_double)]),
    ("amtk_group_scan_add_frames", C.c_int, [V, VP, C.POINTER(ClipDesc), C.c_int, C.c_int, c_i32_p, c_i32_p]),
    ("amtk_calc_fade2_records", None, [c_float_p, c_float_p, c_float_p]),
    ("amtk_tnr_default_params", None, [C.POINTER(TnrParams)]),
    ("amtk_tnr_frames", C.c_int, [V, C.POINTER(ClipDesc), C.POINTER(ClipDesc), C.c_int, C.POINTER(TnrParams), C.c_int, C.c_int]),
    ("amtk_tnr_stream_create", C.c_int, [V, C.POINTER(TnrParams), C.c_int, C.c_int, VP]),
    ("amtk_tnr_stream_create_widening", C.c_int, [V, C.POINTER(TnrParams), C.c_int, C.c_int, C.c_int, VP]),
    ("amtk_tnr_stream_destroy", None, [V]),
    ("amtk_tnr_stream_send", C.c_int, [V, C.POINTER(ClipDesc), C.c_int32]),
    ("amtk_tnr_stream_recv", C.c_int, [V, C.POINTER(ClipDesc), c_i32_p, C.POINTER(C.c_int)]),
    ("amtk_tnr_stream_finish", C.c_int, [V]),
    ("amtk_scan_logo_stream_create", C.c_int, [V, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, V, VP]),
    ("amtk_scan_logo_stream_destroy", None, [V]),
    ("amtk_scan_logo_stream_send", C.c_int, [V, C.POINTER(ClipDesc), C.c_int64, C.c_int64, C.POINTER(C.c_int)]),
    ("amtk_scan_logo_stream_finish", C.c_int, [V, C.c_int, C.c_char_p]),
    ("amtk_scan_logo_stream_counts", C.c_int, [V, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int64)]),
    ("amtk_erase_logo_clip", C.c_int, [V, C.POINTER(ClipDesc), C.POINTER(ClipDesc), V, C.c_float, c_u8_p, C.c_int,
                                       C.c_int, C.c_int, c_float_p]),
    ("amtk_erase_logo_stream_create", C.c_int, [V, V, C.c_float, C.c_int, c_u8_p, C.c_int, C.c_int, VP]),
    ("amtk_erase_logo_stream_destroy", None, [V]),
    ("amtk_erase_logo_stream_send", C.c_int, [V, C.POINTER(ClipDesc)]),
    ("amtk_erase_logo_stream_recv", C.c_int, [V, C.POINTER(ClipDesc), C.POINTER(C.c_int), C.POINTER(C.c_int), c_float_p]),
    ("amtk_erase_logo_stream_counts", C.c_int, [V, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                                C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    ("amtk_logo_scan_stream_create", C.c_int, [V, VP, C.c_int, C.c_int, C.c_int, VP]),
    ("amtk_logo_scan_stream_destroy", None, [V]),
    ("amtk_logo_scan_stream_send", C.c_int, [V, C.POINTER(ClipDesc)]),
    ("amtk_logo_scan_stream_finish", C.c_int, [V]),
    ("amtk_logo_scan_stream_recv", C.c_int, [V, c_float_p, C.c_int, C.POINTER(C.c_int)]),
    ("amtk_logo_scan_stream_counts", C.c_int, [V, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int64),
                                               C.POINTER(C.c_int64)]),
    ("amtk_comb_stream_create", C.c_int, [V, C.POINTER(CombParams), C.c_int, VP]),
    ("amtk_comb_stream_destroy", None, [V]),
    ("amtk_comb_stream_send", C.c_int, [V, C.POINTER(ClipDesc)]),
    ("amtk_comb_stream_finish", C.c_int, [V]),
    ("amtk_comb_stream_recv", C.c_int, [V, c_i32_p, C.c_int, C.POINTER(C.c_int)]),
    ("amtk_comb_stream_counts", C.c_int, [V, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int64),
                                          C.POINTER(C.c_int64)]),
    ("amtk_scan_comb_stream_create", C.c_int, [V, VP, C.c_int, C.POINTER(CombParams), C.c_int, VP]),
    ("amtk_scan_comb_stream_create_pitch", C.c_int, [V, VP, C.c_int, C.POINTER(CombParams), C.c_int, C.c_int, VP]),
    ("amtk_scan_comb_stream_destroy", None, [V]),
    ("amtk_scan_comb_stream_send", C.c_int, [V, C.POINTER(ClipDesc)]),
    ("amtk_scan_comb_stream_finish", C.c_int, [V]),
    ("amtk_scan_comb_stream_recv", C.c_int, [V, c_float_p, c_i32_p, C.c_int, C.POINTER(C.c_int)]),
    ("amtk_scan_comb_stream_counts", C.c_int, [V, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int64),
                                              C.POINTER(C.c_int64)]),
    ("amtk_logo_find_create", C.c_int, [V, VP]),
    ("amtk_logo_find_destroy", None, [V]),
    ("amtk_logo_find_add_frames", C.c_int, [V, C.POINTER(ClipDesc), C.c_int, C.c_int]),
    ("amtk_logo_find_get_sums", C.c_int, [V, V, V, C.POINTER(C.c_int64)]),
    ("amtk_logo_find_default_params", None, [C.POINTER(LogoFindParams)]),
    ("amtk_logo_find_rects", C.c_int, [V, V, C.c_int64, C.c_int, C.c_int, C.c_int, C.POINTER(LogoFindParams), C.c_int,
                                       c_i32_p, c_float_p, C.POINTER(C.c_int)]),
]

LOGO_ANALYZE_CB = C.CFUNCTYPE(C.c_int, C.c_float, C.c_int, C.c_int, C.c_int)

_lib = None


def lib():
    """Load libamtk_b200.so (raises AmtkError when it has not been built -- no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise AmtkError("native library missing: %s (run `python -m amatsukaze_b200._build`); "
                            "there is no CPU fallback" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        for name, res, args in SIGNATURES:
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(ok):
    if not ok:
        raise AmtkError(lib().amtk_last_error().decode("utf-8", "replace"))


def default_comb_params():
    p = CombParams()
    lib().amtk_comb_default_params(C.byref(p))
    return p


def default_tnr_params():
    """(temporal_distance, threshold, interlaced) = (3, 1, 0): the product's KTemporalNR(3, 1)."""
    p = TnrParams()
    lib().amtk_tnr_default_params(C.byref(p))
    return p


def default_logo_find_params():
    """(block, var_ratio, mean_delta, margin, min_blocks) = (8, 0.5, 6, 8, 4)."""
    p = LogoFindParams()
    lib().amtk_logo_find_default_params(C.byref(p))
    return p


def logo_find_rects(s1, s2, nframes, bits, params=None, max_rects=16):
    """amtk_logo_find_rects on host sum maps (uint64 (height, width) each; no device needed): (rects int32 (n, 4) =
    imgx, imgy, w, h, best first; scores float32 (n,))."""
    a1 = np.ascontiguousarray(s1, np.uint64)
    a2 = np.ascontiguousarray(s2, np.uint64)
    assert a1.shape == a2.shape and a1.ndim == 2
    p = params if params is not None else default_logo_find_params()
    rects = np.zeros((max(int(max_rects), 0), 4), np.int32)
    scores = np.zeros(max(int(max_rects), 0), np.float32)
    n = C.c_int()
    check(lib().amtk_logo_find_rects(_ptr(a1), _ptr(a2), int(nframes), a1.shape[1], a1.shape[0], int(bits), C.byref(p),
                                     int(max_rects), rects.ctypes.data_as(c_i32_p), scores.ctypes.data_as(c_float_p), C.byref(n)))
    return rects[:n.value], scores[:n.value]


def tnr_params(temporal_distance=3, threshold=1, interlaced=False):
    return TnrParams(int(temporal_distance), int(threshold), int(bool(interlaced)))


def _ptr(x):
    """Device/host pointer of a torch tensor or numpy array (or a raw int)."""
    if isinstance(x, int):
        return C.c_void_p(x)
    if isinstance(x, np.ndarray):
        return C.c_void_p(x.ctypes.data)
    return C.c_void_p(x.data_ptr())


def yv12_clip(buf, width, height, num_frames, on_device, bits=8):
    """Descriptor for tightly packed planar 4:2:0 frames (Y, U, V back to back; pitch = row bytes)."""
    bps = 1 if bits == 8 else 2
    ysz = width * height * bps
    csz = (width // 2) * (height // 2) * bps
    d = ClipDesc()
    d.base = _ptr(buf).value
    d.frame_stride = ysz + 2 * csz
    d.off_u = ysz
    d.off_v = ysz + csz
    d.width, d.height = width, height
    d.pitch_y, d.pitch_uv = width * bps, (width // 2) * bps
    d.log_uvx = d.log_uvy = 1
    d.bytes_per_sample, d.bits_per_sample = bps, bits
    d.num_frames = num_frames
    d.on_device = 1 if on_device else 0
    return d


class Context:
    """One CUDA device + one stream (amtk_ctx)."""

    def __init__(self, device=0, stream=None):
        self.L = lib()
        h = C.c_void_p()
        check(self.L.amtk_ctx_create(int(device), C.c_void_p(stream) if stream else None, C.byref(h)))
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None) and not getattr(self, "borrowed", False):
            self.L.amtk_ctx_destroy(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def synchronize(self):
        check(self.L.amtk_ctx_synchronize(self.h))

    @property
    def launches(self):
        return int(self.L.amtk_ctx_launch_count(self.h))

    @property
    def last_h2d_bytes(self):
        return int(self.L.amtk_ctx_last_h2d_bytes(self.h))

    def set_kernel_timing(self, enable):
        check(self.L.amtk_ctx_set_kernel_timing(self.h, int(enable)))

    def probe_read_gbs(self, tensor, reps=3):
        """GB/s of a do-nothing streaming read of `tensor` (device) -- the read-only HBM ceiling on this GPU."""
        ms = C.c_double()
        nbytes = tensor.numel() * tensor.element_size()
        check(self.L.amtk_probe_read_ms(self.h, _ptr(tensor), nbytes, reps, C.byref(ms)))
        return nbytes / (ms.value * 1e-3) / 1e9

    def kernel_timing(self, reset=True):
        """(total ms, launches) of the comb kernel since the last reset, from CUDA events on the launch stream."""
        ms, n = C.c_double(), C.c_int64()
        check(self.L.amtk_ctx_get_kernel_timing(self.h, C.byref(ms), C.byref(n), int(reset)))
        return ms.value, n.value

    # ---- logos (host objects; uploaded to this context's device on first use) ----
    def logo(self, data, w, h, imgw, imgh, imgx, imgy, log_uvx=1, log_uvy=1):
        return Logo.create(data, w, h, imgw, imgh, imgx, imgy, log_uvx, log_uvy)

    def load_logo(self, path):
        return Logo.load(path)

    # ---- hot path ----
    def _out(self, out, shape, dtype, device_like):
        import torch
        if out is not None:
            return out, (1 if (not isinstance(out, np.ndarray) and out.is_cuda) else 0)
        if device_like:
            return torch.empty(shape, dtype=dtype, device="cuda:%d" % self.device), 1
        return np.empty(shape, np.float32 if dtype == torch.float32 else np.int32), 0

    def scan_frames(self, clip, logos, frame0=0, nframes=None, out=None, pitch_elems_override=0):
        import torch
        n = clip.num_frames - frame0 if nframes is None else nframes
        arr = (C.c_void_p * len(logos))(*[lg.h if lg is not None else None for lg in logos])
        out, on_dev = self._out(out, (n, len(logos), 2), torch.float32, clip.on_device)
        check(self.L.amtk_logo_scan_frames(self.h, C.byref(clip), arr, len(logos), frame0, n, pitch_elems_override, _ptr(out), on_dev))
        return out

    def analyze_frames(self, clip, deint, field_t, field_b, frame0=0, nframes=None, out=None):
        import torch
        n = clip.num_frames - frame0 if nframes is None else nframes
        out, on_dev = self._out(out, (n, 33), torch.float32, clip.on_device)
        check(self.L.amtk_logo_analyze_frames(self.h, C.byref(clip), deint.h, field_t.h, field_b.h, frame0, n, _ptr(out), on_dev))
        return out

    def eval_fades(self, clip, deint, fades, frame0=0, nframes=None, out=None):
        import torch
        n = clip.num_frames - frame0 if nframes is None else nframes
        f = np.ascontiguousarray(fades, np.float32)
        out, on_dev = self._out(out, (n, len(f)), torch.float32, clip.on_device)
        check(self.L.amtk_logo_eval_fades(self.h, C.byref(clip), deint.h, f.ctypes.data_as(c_float_p), len(f), frame0, n, _ptr(out), on_dev))
        return out

    def comb_frames(self, clip, params=None, frame0=0, nframes=None, out=None):
        import torch
        n = clip.num_frames - frame0 if nframes is None else nframes
        p = params or default_comb_params()
        out, on_dev = self._out(out, (n, 12), torch.int32, clip.on_device)
        check(self.L.amtk_comb_frames(self.h, C.byref(clip), C.byref(p), frame0, n, _ptr(out), on_dev))
        return out

    def scan_comb_frames(self, clip, logos, params=None, frame0=0, nframes=None, scores=None, counts=None,
                         pitch_elems_override=0):
        """The fused step: (scores (n, nlogos, 2), counters (n, 12)).  pitch_elems_override as for scan_frames (ScanFrame's
        byte-pitch row step on 2-byte samples: clip.pitch_y); 0 calls amtk_scan_comb_frames, any other value
        amtk_scan_comb_frames_pitch."""
        import torch
        n = clip.num_frames - frame0 if nframes is None else nframes
        p = params or default_comb_params()
        arr = (C.c_void_p * len(logos))(*[lg.h if lg is not None else None for lg in logos])
        scores, on_dev = self._out(scores, (n, len(logos), 2), torch.float32, clip.on_device)
        counts, on_dev2 = self._out(counts, (n, 12), torch.int32, clip.on_device)
        assert on_dev == on_dev2
        if pitch_elems_override:
            check(self.L.amtk_scan_comb_frames_pitch(self.h, C.byref(clip), arr, len(logos), C.byref(p), int(pitch_elems_override),
                                                     frame0, n, _ptr(scores), _ptr(counts), on_dev))
        else:
            check(self.L.amtk_scan_comb_frames(self.h, C.byref(clip), arr, len(logos), C.byref(p), frame0, n, _ptr(scores),
                                               _ptr(counts), on_dev))
        return scores, counts

    def erase_logo(self, clip, logo, fades, frame0=0, nframes=None):
        n = clip.num_frames - frame0 if nframes is None else nframes
        f = np.ascontiguousarray(fades, np.float32).reshape(n, 2)
        check(self.L.amtk_erase_logo_frames(self.h, C.byref(clip), logo.h, frame0, n, f.ctypes.data_as(c_float_p)))

    def scan_logo(self, clip, dstpath, imgx, imgy, w, h, thy, max_frames, service_id=0, cb=None):
        """The reference's ScanLogo pipeline (LogoScan.hpp:1058-1098) on a clip; cb(progress, nread, total, ngather)."""
        CB = C.CFUNCTYPE(C.c_int, C.c_float, C.c_int, C.c_int, C.c_int)
        fn = CB(lambda p, a, b, c: int(bool(cb(p, a, b, c)))) if cb else None
        check(self.L.amtk_scan_logo(self.h, C.byref(clip), service_id, dstpath.encode(), imgx, imgy, w, h, thy, max_frames,
                                    C.cast(fn, C.c_void_p) if fn else None))

    def weave_frames(self, src, dst, top_idx, bottom_idx, dst_frame0=0, src_is_nv12=False):
        """AMTSource::MergeField on the device: dst[k] even rows <- src[top_idx[k]], odd rows <- src[bottom_idx[k]]."""
        t = np.ascontiguousarray(top_idx, np.int32)
        b = np.ascontiguousarray(bottom_idx, np.int32)
        assert t.shape == b.shape
        check(self.L.amtk_weave_frames(self.h, C.byref(src), C.byref(dst), dst_frame0, t.ctypes.data_as(c_i32_p),
                                       b.ctypes.data_as(c_i32_p), int(t.size), int(bool(src_is_nv12))))

    def tnr_frames(self, src, dst, params=None, frame0=0, nframes=None, dst_frame0=0):
        """The reference's TemporalNRFilter (VideoFilter.hpp:27-212) over source frames [frame0, frame0+nframes) into
        dst frames dst_frame0..; each window clamps at the ends of the clip.  src/dst: ClipDesc, device or host.

        dst may also widen the clip (ConvertBits fused into the filter): a 2-byte dst whose bits_per_sample is above the
        source's (8, 10, 12 or 14 bits) receives the filter at dst's depth applied to the source frames shifted left by
        the difference, bit-exact against the reference's TemporalNRFilter on those shifted frames.  Narrowing, a 1-byte
        dst for a 2-byte source and a 2-byte dst at 8 bits are refused."""
        n = src.num_frames - frame0 if nframes is None else nframes
        p = params if params is not None else default_tnr_params()
        check(self.L.amtk_tnr_frames(self.h, C.byref(src), C.byref(dst), dst_frame0, C.byref(p), frame0, n))

    def tnr_stream(self, params=None, batch_size=8, reference_emission=False, out_bits=0):
        """The same filter fed one frame at a time (amtk_tnr_stream; the reference's cudaTNR* calls): send(frame, tag),
        recv(dst) -> tag or None, finish().  See include/amtk_b200.h for when outputs become available.

        out_bits in (10, 12, 14, 16) widens as it filters: frames are sent at their own size and every output is 2-byte
        samples at out_bits, the filter at out_bits on the frames shifted left by the difference; 0 keeps the frames'
        format."""
        p = params if params is not None else default_tnr_params()
        out = C.c_void_p()
        check(self.L.amtk_tnr_stream_create_widening(self.h, C.byref(p), int(out_bits), int(batch_size),
                                                     int(bool(reference_emission)), C.byref(out)))
        return TnrStream(self, out)

    def scan_logo_stream(self, imgx, imgy, w, h, thy, max_frames, cb=None):
        """The ScanLogo pipeline fed one decoded frame at a time (amtk_scan_logo_stream; InitialLogoCreator::onFrame):
        send(frame, pos, size) -> more, finish(dstpath, service_id=0), counts() -> (nread, ngather, h2d_bytes).
        cb(progress, nread, total, ngather) as for scan_logo; returning False cancels."""
        fn = LOGO_ANALYZE_CB(lambda p, a, b, c: int(bool(cb(p, a, b, c)))) if cb else None
        out = C.c_void_p()
        check(self.L.amtk_scan_logo_stream_create(self.h, int(imgx), int(imgy), int(w), int(h), int(thy), int(max_frames),
                                                  C.cast(fn, C.c_void_p) if fn else None, C.byref(out)))
        return ScanLogoStream(self, out, fn)

    def erase_logo_clip(self, src, logo, dst=None, frame_result=None, max_fade_length=16, frame0=0, nframes=None,
                        maskratio=0.35):
        """AMTEraseLogo(AMTAnalyzeLogo(src, logo), logo, logof, maxfade) over frames [frame0, frame0+nframes) of a whole clip
        in one call (amtk_erase_logo_clip): in place on src (dst None), or every output frame into dst (a device ClipDesc).
        Returns the fades, float32 (nframes, 2) = (fadeT, fadeB)."""
        n = src.num_frames - frame0 if nframes is None else nframes
        fr = None
        if frame_result is not None:
            fr = np.ascontiguousarray(frame_result, np.uint8)
            assert fr.size == src.num_frames
        fades = np.zeros((max(n, 0), 2), np.float32)
        check(self.L.amtk_erase_logo_clip(self.h, C.byref(src), C.byref(dst) if dst is not None else None, logo.h,
                                          C.c_float(maskratio), fr.ctypes.data_as(c_u8_p) if fr is not None else None,
                                          int(max_fade_length), int(frame0), int(n), fades.ctypes.data_as(c_float_p)))
        return fades

    def erase_logo_stream(self, logo, num_frames, frame_result=None, max_fade_length=16, batch_size=16, maskratio=0.35):
        """AMTEraseLogo(AMTAnalyzeLogo(src, logo), logo, logof, maxfade) fed one frame at a time (amtk_erase_logo_stream):
        send(frame), recv(dst) -> (n, (fadeT, fadeB)) or None, counts() -> (sent, received, analysed, h2d, d2h).
        logo: the raw Logo; frame_result: None or num_frames values in {0, 1, 2} (the logoframe file's frame states).
        See include/amtk_b200.h for when outputs become available."""
        fr = None
        if frame_result is not None:
            fr = np.ascontiguousarray(frame_result, np.uint8)
            assert fr.size == num_frames
        out = C.c_void_p()
        check(self.L.amtk_erase_logo_stream_create(self.h, logo.h, C.c_float(maskratio), int(num_frames),
                                                   fr.ctypes.data_as(c_u8_p) if fr is not None else None,
                                                   int(max_fade_length), int(batch_size), C.byref(out)))
        return EraseLogoStream(self, out)

    def logo_scan_stream(self, logos, batch_size=64, reference_pitch=False):
        """LogoFrame::ScanFrame over a recording fed one decoded frame at a time (amtk_logo_scan_stream): send(frame),
        finish(), recv(max_frames) -> float32 (n, nlogos, 2), counts() -> (sent, received, h2d, d2h).  logos: deint Logos
        with masks, or None.  See include/amtk_b200.h for when results become available."""
        arr = (C.c_void_p * len(logos))(*[lg.h if lg is not None else None for lg in logos])
        out = C.c_void_p()
        check(self.L.amtk_logo_scan_stream_create(self.h, arr, len(logos), int(batch_size), int(bool(reference_pitch)),
                                                  C.byref(out)))
        return LogoScanStream(self, out, len(logos))

    def comb_stream(self, params=None, batch_size=64):
        """The combing counters of a recording fed one decoded frame at a time (amtk_comb_stream): send(frame),
        finish(), recv(max_frames) -> int32 (n, 12), counts() -> (sent, received, h2d, d2h).  Row n equals row n of
        comb_frames on the clip of all frames sent.  See include/amtk_b200.h for when rows become available."""
        p = params or default_comb_params()
        out = C.c_void_p()
        check(self.L.amtk_comb_stream_create(self.h, C.byref(p), int(batch_size), C.byref(out)))
        return CombStream(self, out)

    def scan_comb_stream(self, logos, params=None, batch_size=16, reference_pitch=False):
        """The fused step (scan_comb_frames) over a recording fed one decoded frame at a time (amtk_scan_comb_stream):
        send(frame), finish(), recv(max_frames) -> (float32 (n, nlogos, 2) scores, int32 (n, 12) counters),
        counts() -> (sent, received, h2d, d2h).  Row n equals row n of scan_comb_frames on the clip of all frames sent.
        logos: deint Logos with masks, or None.  reference_pitch: ScanFrame's byte-pitch row step on 2-byte samples
        (amtk_scan_comb_stream_create_pitch; row n then equals scan_comb_frames(..., pitch_elems_override=clip.pitch_y)).
        See include/amtk_b200.h for when results become available."""
        p = params or default_comb_params()
        arr = (C.c_void_p * len(logos))(*[lg.h if lg is not None else None for lg in logos])
        out = C.c_void_p()
        if reference_pitch:
            check(self.L.amtk_scan_comb_stream_create_pitch(self.h, arr, len(logos), C.byref(p), int(batch_size), 1, C.byref(out)))
        else:
            check(self.L.amtk_scan_comb_stream_create(self.h, arr, len(logos), C.byref(p), int(batch_size), C.byref(out)))
        return ScanCombStream(self, out, len(logos))

    def logo_find(self):
        """The logo finder (amtk_logo_find): add_frames(clip, ...), sums() -> (s1, s2, nframes), rects(...)."""
        out = C.c_void_p()
        check(self.L.amtk_logo_find_create(self.h, C.byref(out)))
        return LogoFind(self, out)

    def logo_scan(self, scanw, scanh, thy, log_uvx=1, log_uvy=1):
        out = C.c_void_p()
        check(self.L.amtk_scan_create(self.h, scanw, scanh, log_uvx, log_uvy, thy, C.byref(out)))
        return LogoScanAcc(self, out, scanw, scanh, log_uvx, log_uvy)


class Group:
    """amtk_group: one process driving several devices (context + stream + host thread per device, NCCL for the final
    gather).  Python is plumbing only; bench.py --gpus N without torchrun goes through this."""

    def __init__(self, ndev, devices=None):
        self.L = lib()
        h = C.c_void_p()
        arr = None
        if devices is not None:
            arr = np.ascontiguousarray(devices, np.int32).ctypes.data_as(c_i32_p)
        check(self.L.amtk_group_create(int(ndev), arr, C.byref(h)))
        self.h = h
        self.n = self.L.amtk_group_size(h)

    def close(self):
        if getattr(self, "h", None):
            self.L.amtk_group_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def ctx(self, i):
        """Borrowed Context of member i (owned by the group: do not close it)."""
        c = Context.__new__(Context)
        c.L, c.h, c.device, c.borrowed = self.L, C.c_void_p(self.L.amtk_group_ctx(self.h, i)), i, True
        return c

    def numa_cpus(self, i):
        return int(self.L.amtk_group_numa_cpus(self.h, i))

    @property
    def nccl_version(self):
        return int(self.L.amtk_group_nccl_version(self.h))

    def host_alloc(self, i, nbytes):
        """Pinned, NUMA-local host buffer as a numpy uint8 array (freed with the process)."""
        p = C.c_void_p()
        check(self.L.amtk_group_host_alloc(self.h, i, nbytes, C.byref(p)))
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(nbytes,))

    def scan_comb_streams(self, clips, logos, params, nframes):
        carr = (ClipDesc * self.n)(*clips)
        larr = (C.c_void_p * self.n)(*[lg.h for lg in logos])
        check(self.L.amtk_group_scan_comb_streams(self.h, carr, larr, C.byref(params), nframes))

    def fetch_results(self, nframes, src=0):
        scores = np.empty((self.n, nframes, 2), np.float32)
        counts = np.empty((self.n, nframes, 12), np.int32)
        check(self.L.amtk_group_fetch_results(self.h, src, nframes, _ptr(scores), _ptr(counts)))
        return scores, counts

    def synchronize(self):
        check(self.L.amtk_group_synchronize(self.h))

    def mark(self, slot):
        check(self.L.amtk_group_mark(self.h, slot))

    def elapsed_ms(self, a, b):
        out = (C.c_double * self.n)()
        check(self.L.amtk_group_elapsed_ms(self.h, a, b, out))
        return list(out)

    def scan_add_frames(self, scans, clips, scanx, scany, frame0, nframes):
        sarr = (C.c_void_p * self.n)(*[s.h for s in scans])
        carr = (ClipDesc * self.n)(*clips)
        f0 = np.ascontiguousarray(frame0, np.int32)
        nf = np.ascontiguousarray(nframes, np.int32)
        check(self.L.amtk_group_scan_add_frames(self.h, sarr, carr, scanx, scany, f0.ctypes.data_as(c_i32_p), nf.ctypes.data_as(c_i32_p)))


class Logo:
    """amtk_logo: LogoData/LogoDataParam equivalent.  A host object (no GPU needed to build its tables)."""

    def __init__(self, h):
        self.L, self.h = lib(), h
        self.header = None

    @classmethod
    def create(cls, data, w, h, imgw, imgh, imgx, imgy, log_uvx=1, log_uvy=1):
        d = np.ascontiguousarray(data, np.float32)
        out = C.c_void_p()
        check(lib().amtk_logo_create(None, d.ctypes.data_as(c_float_p), w, h, log_uvx, log_uvy, imgw, imgh, imgx, imgy, C.byref(out)))
        return cls(out)

    @classmethod
    def load(cls, path):
        out = C.c_void_p()
        hdr = np.zeros(540, np.uint8)
        check(lib().amtk_logo_load(None, path.encode(), C.byref(out), hdr.ctypes.data_as(C.c_void_p)))
        lg = cls(out)
        lg.header = hdr
        return lg

    def __del__(self):
        try:
            if self.h:
                self.L.amtk_logo_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def deint(self):
        out = C.c_void_p()
        check(self.L.amtk_logo_deint(self.h, C.byref(out)))
        return Logo(out)

    def field(self, bottom):
        out = C.c_void_p()
        check(self.L.amtk_logo_field(self.h, int(bottom), C.byref(out)))
        return Logo(out)

    def create_mask(self, maskratio):
        check(self.L.amtk_logo_create_mask(self.h, C.c_float(maskratio)))
        return self

    def info(self):
        i = LogoInfo()
        check(self.L.amtk_logo_get_info(self.h, C.byref(i)))
        return i

    def save(self, path, name="No Name", service_id=0):
        check(self.L.amtk_logo_save(self.h, path.encode(), name.encode(), service_id))

    def tables(self):
        i = self.info()
        n = (i.w * i.h + (i.w >> i.log_uvx) * (i.h >> i.log_uvy) * 2) * 2
        data = np.zeros(n, np.float32)
        if i.maskpixels == 0:
            check(self.L.amtk_logo_get_tables(self.h, data.ctypes.data_as(c_float_p), None, None, None))
            return {"data": data}
        mask = np.zeros((i.h, i.w), np.uint8)
        kern = np.zeros((i.count, 25), np.float32)
        sc = np.zeros((i.count, 32, 2), np.float32)
        check(self.L.amtk_logo_get_tables(self.h, data.ctypes.data_as(c_float_p), mask.ctypes.data_as(c_u8_p),
                                          kern.ctypes.data_as(c_float_p), sc.ctypes.data_as(c_float_p)))
        return {"data": data, "mask": mask, "kernels": kern, "scales": sc, "black_score": i.black_score}


class _Stream:
    """A frame stream of the C ABI, amtk_<_prefix>_*: its handle and the Context, held so that the context outlives the
    stream."""
    _prefix = None

    def __init__(self, ctx, h):
        self.ctx, self.L, self.h = ctx, ctx.L, h

    def close(self):
        if getattr(self, "h", None) and getattr(self.ctx, "h", None):      # a closed context took the stream's memory with it
            getattr(self.L, "amtk_%s_destroy" % self._prefix)(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class TnrStream(_Stream):
    """amtk_tnr_stream: frames in one at a time, filtered frames out in order."""
    _prefix = "tnr_stream"

    def send(self, frame, index):
        """frame: a one-frame ClipDesc (host or device); index: the int32 tag recv returns with its output."""
        check(self.L.amtk_tnr_stream_send(self.h, C.byref(frame), int(index)))

    def recv(self, dst):
        """Writes the next output into dst (a one-frame ClipDesc) and returns its tag, or None when no output may be
        received yet."""
        idx, got = C.c_int32(), C.c_int()
        check(self.L.amtk_tnr_stream_recv(self.h, C.byref(dst), C.byref(idx), C.byref(got)))
        return idx.value if got.value else None

    def finish(self):
        check(self.L.amtk_tnr_stream_finish(self.h))


class ScanLogoStream(_Stream):
    """amtk_scan_logo_stream: one decoded frame per send, the logo file at finish.  Also holds the ctypes callback the
    library calls."""
    _prefix = "scan_logo_stream"

    def __init__(self, ctx, h, fn):
        super().__init__(ctx, h)
        self._fn = fn

    def send(self, frame, pos, size):
        """frame: a one-frame ClipDesc (host or device); pos, size: the reader's position and the source's size.
        Returns False once the reader should stop (max_frames valid frames were gathered)."""
        more = C.c_int(1)
        check(self.L.amtk_scan_logo_stream_send(self.h, C.byref(frame), int(pos), int(size), C.byref(more)))
        return bool(more.value)

    def finish(self, dstpath, service_id=0):
        check(self.L.amtk_scan_logo_stream_finish(self.h, int(service_id), dstpath.encode()))

    def counts(self):
        """(frames read up to the cut-off, frames gathered, payload bytes uploaded host->device)"""
        nr, ng, hb = C.c_int(), C.c_int(), C.c_int64()
        check(self.L.amtk_scan_logo_stream_counts(self.h, C.byref(nr), C.byref(ng), C.byref(hb)))
        return nr.value, ng.value, hb.value


class EraseLogoStream(_Stream):
    """amtk_erase_logo_stream: decoded frames in one at a time, their erased logo rectangles out in frame order."""
    _prefix = "erase_logo_stream"

    def send(self, frame):
        """frame: a one-frame ClipDesc (host or device), the next source frame."""
        check(self.L.amtk_erase_logo_stream_send(self.h, C.byref(frame)))

    def recv(self, dst):
        """Writes the next output's erased logo rectangles into dst (a one-frame ClipDesc holding that source frame's
        pixels) and returns (n, (fadeT, fadeB)), or None when no output may be received yet."""
        n, got = C.c_int(), C.c_int()
        fades = (C.c_float * 2)()
        check(self.L.amtk_erase_logo_stream_recv(self.h, C.byref(dst), C.byref(n), C.byref(got), fades))
        return (n.value, (fades[0], fades[1])) if got.value else None

    def counts(self):
        """(frames sent, outputs received, frames analysed, payload bytes host->device, payload bytes device->host)"""
        s, r, a, hb, db = C.c_int(), C.c_int(), C.c_int(), C.c_int64(), C.c_int64()
        check(self.L.amtk_erase_logo_stream_counts(self.h, C.byref(s), C.byref(r), C.byref(a), C.byref(hb), C.byref(db)))
        return s.value, r.value, a.value, hb.value, db.value


class _RowStream(_Stream):
    """A stream that takes decoded frames one at a time and returns one row of results per frame, in frame order: the
    functions amtk_<_prefix>_{send,finish,recv,counts}, rows of shape _row() and type _dtype."""
    _dtype = _ptr = None

    def _call(self, fn, *args):
        check(getattr(self.L, "amtk_%s_%s" % (self._prefix, fn))(self.h, *args))

    def send(self, frame):
        """frame: a one-frame ClipDesc (host or device), the next frame of the recording."""
        self._call("send", C.byref(frame))

    def finish(self):
        """End of input: launches the open partial batch; later sends fail."""
        self._call("finish")

    def recv(self, max_frames):
        """The next rows that may be received, at most max_frames: an array of shape (n,) + _row()."""
        out = np.empty((max(int(max_frames), 0),) + self._row(), self._dtype)
        got = C.c_int()
        self._call("recv", out.ctypes.data_as(self._ptr), int(max_frames), C.byref(got))
        return out[:got.value]

    def counts(self):
        """(frames sent, rows received, payload bytes host->device, result bytes device->host)"""
        s, r, hb, db = C.c_int(), C.c_int(), C.c_int64(), C.c_int64()
        self._call("counts", C.byref(s), C.byref(r), C.byref(hb), C.byref(db))
        return s.value, r.value, hb.value, db.value


class LogoScanStream(_RowStream):
    """amtk_logo_scan_stream: the frames' ScanFrame results, float32 (n, nlogos, 2) = (corr0, corr1)."""
    _prefix, _dtype, _ptr = "logo_scan_stream", np.float32, c_float_p

    def __init__(self, ctx, h, nlogos):
        super().__init__(ctx, h)
        self.nlogos = nlogos

    def _row(self):
        return (self.nlogos, 2)


class CombStream(_RowStream):
    """amtk_comb_stream: the frames' combing counters, int32 (n, 12), as comb_frames."""
    _prefix, _dtype, _ptr = "comb_stream", np.int32, c_i32_p

    def _row(self):
        return (12,)


class ScanCombStream(_RowStream):
    """amtk_scan_comb_stream: the frames' ScanFrame results and combing counters, as scan_comb_frames."""
    _prefix = "scan_comb_stream"

    def __init__(self, ctx, h, nlogos):
        super().__init__(ctx, h)
        self.nlogos = nlogos

    def recv(self, max_frames):
        """The next results that may be received, at most max_frames: (scores float32 (n, nlogos, 2), counts int32 (n, 12))."""
        m = max(int(max_frames), 0)
        scores, counts = np.empty((m, self.nlogos, 2), np.float32), np.empty((m, 12), np.int32)
        got = C.c_int()
        self._call("recv", scores.ctypes.data_as(c_float_p), counts.ctypes.data_as(c_i32_p), int(max_frames), C.byref(got))
        return scores[:got.value], counts[:got.value]


class LogoScanAcc:
    def __init__(self, ctx, h, scanw, scanh, lx, ly):
        self.ctx, self.L, self.h = ctx, ctx.L, h
        self.npix = scanw * scanh + 2 * (scanw >> lx) * (scanh >> ly)
        self.ndata = self.npix * 2

    def __del__(self):
        try:
            if self.h:
                self.L.amtk_scan_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def add_frames(self, clip, scanx, scany, frame0=0, nframes=None, select=None):
        n = clip.num_frames - frame0 if nframes is None else nframes
        valid = np.zeros(n, np.uint8)
        sel = None
        if select is not None:
            sel = np.ascontiguousarray(select, np.uint8)
        check(self.L.amtk_scan_add_frames(self.h, C.byref(clip), scanx, scany, frame0, n,
                                          sel.ctypes.data_as(c_u8_p) if sel is not None else None, valid.ctypes.data_as(c_u8_p)))
        return valid

    @property
    def num_valid(self):
        return self.L.amtk_scan_num_valid(self.h)

    def sums(self):
        out = np.zeros((self.npix, 5), np.float64)
        check(self.L.amtk_scan_get_sums(self.h, out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    def get_logo(self, maxv=255, clean=False):
        out = np.zeros(self.ndata, np.float32)
        ok = self.L.amtk_scan_get_logo(self.h, maxv, int(clean), out.ctypes.data_as(c_float_p))
        if not ok:
            msg = self.L.amtk_last_error().decode()
            if "Insufficient" in msg:
                return None
            raise AmtkError(msg)
        return out


class LogoFind:
    """amtk_logo_find: per-pixel temporal sums of the luma plane over the frames added, and the logo rectangles they
    show.  The first clip fixes the frame size and sample format."""

    def __init__(self, ctx, h):
        self.ctx, self.L, self.h = ctx, ctx.L, h
        self.width = self.height = self.bits = None

    def __del__(self):
        try:
            if self.h and getattr(self.ctx, "h", None):
                self.L.amtk_logo_find_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def add_frames(self, clip, frame0=0, nframes=None):
        n = clip.num_frames - frame0 if nframes is None else nframes
        check(self.L.amtk_logo_find_add_frames(self.h, C.byref(clip), int(frame0), int(n)))
        if self.width is None:
            self.width, self.height, self.bits = clip.width, clip.height, clip.bits_per_sample

    def sums(self):
        """(s1, s2, nframes): uint64 (height, width) each, None before the first clip."""
        n = C.c_int64()
        if self.width is None:
            check(self.L.amtk_logo_find_get_sums(self.h, None, None, C.byref(n)))
            return None, None, n.value
        s1 = np.zeros((self.height, self.width), np.uint64)
        s2 = np.zeros((self.height, self.width), np.uint64)
        check(self.L.amtk_logo_find_get_sums(self.h, _ptr(s1), _ptr(s2), C.byref(n)))
        return s1, s2, n.value

    def rects(self, params=None, max_rects=16):
        """The rectangles of the frames added so far: (rects int32 (n, 4) = imgx, imgy, w, h, best first; scores)."""
        s1, s2, n = self.sums()
        if s1 is None:
            return np.zeros((0, 4), np.int32), np.zeros(0, np.float32)
        return logo_find_rects(s1, s2, n, 8 if self.bits <= 8 else self.bits, params, max_rects)


def calc_fade2(records, num_frames, n):
    r = np.ascontiguousarray(records, np.float32).reshape(-1, 33)
    ft, fb = C.c_float(), C.c_float()
    lib().amtk_calc_fade2(r.ctypes.data_as(c_float_p), r.shape[0], num_frames, n, C.byref(ft), C.byref(fb))
    return ft.value, fb.value
