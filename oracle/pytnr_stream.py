"""oracle/pytnr_stream.py -- TEST INFRASTRUCTURE ONLY: the reference's own CudaTemporalNRFilter (VideoFilter.hpp:214-267)
driving the library's amtk_tnr_stream_* through the CudaFilter.h stand-in of oracle/ref_tnr_stream/.

  * oracle/_ref/libamtk_ref_tnr_stream.so -- built by oracle/build_ref_tnr_stream.sh where the reference tree is present
                                            (travels with the tree like the rest of oracle/_ref)
  * launched_batches / receivable / emitted -- the stream's launch and receive rule and its emission sets restated
                                               (DESIGN.md section 3.4), which the tests hold the library to

The product package never imports this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SO = os.path.join(HERE, "_ref", "libamtk_ref_tnr_stream.so")
REF_SRC = "/root/reference/Amatsukaze/VideoFilter.hpp"

_ref = None


def build_ref():
    """Run oracle/build_ref_tnr_stream.sh when the reference tree is present."""
    if os.path.exists(REF_SRC):
        srcs = [os.path.join(HERE, f) for f in ("build_ref_tnr_stream.sh", "ref_tnr_stream_glue.cpp",
                                                os.path.join("ref_tnr_stream", "CudaFilter.h"))]
        if not os.path.exists(REF_SO) or os.path.getmtime(REF_SO) < max(os.path.getmtime(f) for f in srcs):
            subprocess.check_call(["bash", os.path.join(HERE, "build_ref_tnr_stream.sh")])
    return REF_SO if os.path.exists(REF_SO) else None


def ref_available():
    return os.path.exists(REF_SO)


def _reflib():
    global _ref
    if _ref is None:
        if not os.path.exists(REF_SO):
            raise RuntimeError("reference CudaTemporalNRFilter not built (oracle/build_ref_tnr_stream.sh)")
        L = C.CDLL(REF_SO)
        L.ref_tnr_stream_run.restype = C.c_int
        L.ref_tnr_stream_run.argtypes = ([C.c_char_p, C.c_void_p] + [C.c_int] * 9 +
                                         [C.c_void_p, C.POINTER(C.c_int32), C.c_int, C.c_char_p, C.c_int])
        _ref = L
    return _ref


def ref_cuda_tnr_sequence(libpath, frames, W, H, bits, d, threshold, interlaced, batch):
    """The reference's CudaTemporalNRFilter over the whole clip on the library at `libpath`: (emitted frameIndex_ values,
    emitted frames).  Raises RuntimeError with the library's message if the filter threw."""
    frames = np.ascontiguousarray(frames)
    N = frames.shape[0]
    cap = N + 4                      # room for a filter that emits more frames than it received
    out = np.zeros((cap, frames.shape[1]), frames.dtype)
    idx = np.zeros(cap, np.int32)
    err = C.create_string_buffer(512)
    m = _reflib().ref_tnr_stream_run(libpath.encode(), frames.ctypes.data, N, W, H, frames.dtype.itemsize, bits, d,
                                     threshold, int(interlaced), batch, out.ctypes.data,
                                     idx.ctypes.data_as(C.POINTER(C.c_int32)), cap, err, len(err))
    if m < 0:
        raise RuntimeError("reference CudaTemporalNRFilter threw: " + err.value.decode("utf-8", "replace"))
    m = min(m, cap)
    return idx[:m].copy(), out[:m].copy()


def launched_batches(S, d, B, finished):
    """Batches of amtk_tnr_stream launched after S sends: batch k once S >= (k+1)B + d; after finish all ceil(S/B)."""
    if finished:
        return -(-S // B)
    return max(0, (S - d) // B)


def receivable(S, d, B, finished):
    """Outputs recv may have delivered in total after S sends (before finish: the newest launched batch is held back)."""
    if finished:
        return S
    return max(0, launched_batches(S, d, B, False) - 1) * B


def emitted(N, d, reference_emission):
    """Output frames the stream delivers for a clip of N frames: all of them, or the CPU TemporalNRFilter queue's set
    (frames N-d .. d-1 dropped when N < 2d)."""
    if not reference_emission:
        return list(range(N))
    return [n for n in range(N) if not (N < 2 * d and N - d <= n <= d - 1)]
