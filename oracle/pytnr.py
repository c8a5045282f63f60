"""oracle/pytnr.py -- TEST INFRASTRUCTURE ONLY: checkers for the temporal noise reduction (TemporalNRFilter,
VideoFilter.hpp:27-212).

  * oracle/_build/libamtk_tnr_oracle.so -- this repo's plain-C restatement (oracle/tnr_oracle.c)
  * oracle/_ref/libamtk_ref_tnr.so      -- the reference's own TemporalNRFilter, built by oracle/build_ref_tnr.sh where
                                           the reference tree is present (travels with the tree like oracle/_ref)
  * np_tnr_frame                        -- a numpy restatement of the same spec (float32 arithmetic, no contraction)

Frames are numpy arrays (N, frame_elems) of uint8 or uint16, packed planar 4:2:0: Y (H*W), U, V ((H/2)*(W/2)).
The product package never imports this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(HERE, "_build", "libamtk_tnr_oracle.so")
REF_SO = os.path.join(HERE, "_ref", "libamtk_ref_tnr.so")
REF_SRC = "/root/reference/Amatsukaze/VideoFilter.hpp"

_or = None
_ref = None


def build_oracle(force=False):
    """Compile oracle/tnr_oracle.c (gcc, no contraction, no fast-math)."""
    src = os.path.join(HERE, "tnr_oracle.c")
    if not force and os.path.exists(ORACLE_SO) and os.path.getmtime(ORACLE_SO) >= os.path.getmtime(src):
        return ORACLE_SO
    os.makedirs(os.path.dirname(ORACLE_SO), exist_ok=True)
    subprocess.check_call(["gcc", "-std=c99", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
                           "-o", ORACLE_SO, src])
    return ORACLE_SO


def build_ref():
    """Run oracle/build_ref_tnr.sh when the reference tree is present."""
    if os.path.exists(REF_SRC):
        srcs = [os.path.join(HERE, f) for f in ("build_ref_tnr.sh", "ref_tnr_glue.cpp")]
        if not os.path.exists(REF_SO) or os.path.getmtime(REF_SO) < max(os.path.getmtime(f) for f in srcs):
            subprocess.check_call(["bash", os.path.join(HERE, "build_ref_tnr.sh")])
    return REF_SO if os.path.exists(REF_SO) else None


def ref_available():
    return os.path.exists(REF_SO)


def _oracle():
    global _or
    if _or is None:
        build_oracle()
        L = C.CDLL(ORACLE_SO)
        L.or_tnr_frame.restype = None
        L.or_tnr_frame.argtypes = [C.POINTER(C.c_void_p), C.c_int] + [C.c_int] * 6 + [C.c_void_p]
        L.or_tnr_clip.restype = None
        L.or_tnr_clip.argtypes = [C.c_void_p] + [C.c_int] * 10 + [C.c_void_p]
        _or = L
    return _or


def _reflib():
    global _ref
    if _ref is None:
        if not os.path.exists(REF_SO):
            raise RuntimeError("reference TemporalNRFilter not built (oracle/build_ref_tnr.sh)")
        L = C.CDLL(REF_SO)
        L.ref_tnr_sequence.restype = C.c_int
        L.ref_tnr_sequence.argtypes = [C.c_void_p] + [C.c_int] * 8 + [C.c_void_p, C.POINTER(C.c_int32)]
        L.ref_tnr_window.restype = C.c_int
        L.ref_tnr_window.argtypes = [C.POINTER(C.c_void_p), C.c_int] + [C.c_int] * 6 + [C.c_void_p]
        _ref = L
    return _ref


def frame_elems(W, H):
    return W * H + 2 * (W // 2) * (H // 2)


def _bps(frames):
    return frames.dtype.itemsize


def _win_ptrs(win):
    return (C.c_void_p * len(win))(*[w.ctypes.data for w in win])


def or_tnr_frame(win, W, H, bits, threshold, interlaced):
    """C port: one output frame from the explicit window `win` (list of 2d+1 frames)."""
    win = [np.ascontiguousarray(w) for w in win]
    out = np.empty_like(win[0])
    _oracle().or_tnr_frame(_win_ptrs(win), len(win), W, H, _bps(win[0]), bits, threshold, int(interlaced), out.ctypes.data)
    return out


def or_tnr_clip(frames, W, H, bits, d, threshold, interlaced, frame0=0, nframes=None):
    """C port, the library's definition: frames [frame0, frame0+nframes) over windows clamped at the clip's ends."""
    frames = np.ascontiguousarray(frames)
    N = frames.shape[0]
    n = N - frame0 if nframes is None else nframes
    out = np.empty((n, frames.shape[1]), frames.dtype)
    _oracle().or_tnr_clip(frames.ctypes.data, N, W, H, _bps(frames), bits, d, threshold, int(interlaced), frame0, n, out.ctypes.data)
    return out


def sequence_windows(N, d):
    """The emission order of TemporalNRFilter::onFrame/finish (VideoFilter.hpp:45-89) restated on frame indices: a list of
    (frameIndex_, window) for a clip of N frames, window = the 2d+1 source frames TNRFilter receives."""
    nf, q, out = 2 * d + 1, [], []
    for n in range(N):                       # onFrame (:45-75)
        q.append(n)
        half = (nf + 1) // 2
        if len(q) < half:
            continue
        win = [q[max(f, 0)] for f in range(len(q) - nf, len(q))]
        out.append((q[len(q) - half], win))
        if len(q) >= nf:
            q.pop(0)
    half = nf // 2                           # finish (:76-88)
    while len(q) > half:
        out.append((q[half], [q[min(i, len(q) - 1)] for i in range(nf)]))
        q.pop(0)
    return out


def or_tnr_sequence(frames, W, H, bits, d, threshold, interlaced):
    """C port driven by the reference's own queue order: (frame indices, output frames)."""
    seq = sequence_windows(frames.shape[0], d)
    outs = [or_tnr_frame([frames[i] for i in win], W, H, bits, threshold, interlaced) for _, win in seq]
    idx = np.array([i for i, _ in seq], np.int32)
    return idx, (np.stack(outs) if outs else np.empty((0, frames.shape[1]), frames.dtype))


def ref_tnr_sequence(frames, W, H, bits, d, threshold, interlaced):
    """The reference's TemporalNRFilter over the whole clip: (emitted frameIndex_ values, emitted frames)."""
    frames = np.ascontiguousarray(frames)
    N = frames.shape[0]
    out = np.zeros_like(frames)
    idx = np.zeros(N, np.int32)
    m = _reflib().ref_tnr_sequence(frames.ctypes.data, N, W, H, _bps(frames), bits, d, threshold, int(interlaced),
                                   out.ctypes.data, idx.ctypes.data_as(C.POINTER(C.c_int32)))
    if m < 0:
        raise RuntimeError("reference TemporalNRFilter threw")
    assert m <= N
    return idx[:m].copy(), out[:m].copy()


def ref_tnr_frame(win, W, H, bits, threshold, interlaced):
    """The reference's TNRFilter on an explicit window."""
    win = [np.ascontiguousarray(w) for w in win]
    out = np.empty_like(win[0])
    if not _reflib().ref_tnr_window(_win_ptrs(win), len(win), W, H, _bps(win[0]), bits, threshold, int(interlaced), out.ctypes.data):
        raise RuntimeError("reference TemporalNRFilter threw")
    return out


def np_tnr_frame(win, W, H, bits, threshold, interlaced):
    """numpy restatement of the spec (DESIGN.md section 3.4), vectorised over pixels, float32 throughout."""
    nf = len(win)
    thresh = threshold << (bits - 8)
    ysz, cw, ch = W * H, W // 2, H // 2
    csz = cw * ch
    w = np.stack([np.asarray(f).astype(np.int64) for f in win])               # (nf, elems)
    Y = w[:, :ysz].reshape(nf, H, W)
    U = w[:, ysz:ysz + csz].reshape(nf, ch, cw)
    V = w[:, ysz + csz:].reshape(nf, ch, cw)
    y = np.arange(H)
    cy = (((y >> 1) & ~1) | (y & 1)) if interlaced else (y >> 1)
    cx = np.arange(W) >> 1
    Uf, Vf = U[:, cy][:, :, cx], V[:, cy][:, :, cx]                            # chroma seen by each luma pixel
    m = nf // 2
    diff = np.abs(Y - Y[m]) + np.abs(Uf - Uf[m]) + np.abs(Vf - Vf[m])
    inc = diff <= thresh
    k = inc.sum(axis=0).astype(np.float32)
    f = np.float32(1.0) / k
    dY = np.full((H, W), 0.5, np.float32)
    dU = np.full((H, W), 0.5, np.float32)
    dV = np.full((H, W), 0.5, np.float32)
    for i in range(nf):
        c = np.where(inc[i], f, np.float32(0.0)).astype(np.float32)
        dY = np.where(inc[i], dY + c * Y[i].astype(np.float32), dY).astype(np.float32)
        dU = np.where(inc[i], dU + c * Uf[i].astype(np.float32), dU).astype(np.float32)
        dV = np.where(inc[i], dV + c * Vf[i].astype(np.float32), dV).astype(np.float32)
    dt = np.asarray(win[0]).dtype
    out = np.empty(ysz + 2 * csz, dt)
    out[:ysz] = dY.astype(np.int32).astype(dt).ravel()
    wr = (((y >> 1) if interlaced else y) & 1) == 0                            # rows that write chroma
    oU = np.zeros((ch, cw), dt)
    oV = np.zeros((ch, cw), dt)
    rows = np.nonzero(wr)[0]
    oU[cy[rows]] = dU[rows][:, 0::2].astype(np.int32).astype(dt)
    oV[cy[rows]] = dV[rows][:, 0::2].astype(np.int32).astype(dt)
    out[ysz:ysz + csz] = oU.ravel()
    out[ysz + csz:] = oV.ravel()
    return out
