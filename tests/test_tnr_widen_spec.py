"""The two facts that let amtk_tnr_frames widen a clip inside the filter (DESIGN.md section 3.4), restated in numpy and
checked without a GPU:

1. inclusion: (dist << k) <= (t << (dst_bits - 8)) exactly when dist <= (t << (src_bits - 8));
2. average: in binary32 with every product and sum rounded on its own, 0.5f + sum f * (Y_i << k) equals
   2^k * (2^-k * 0.5f + sum f * Y_i).

Then the widening kernel's formulation (masks at src_bits, the sum on unshifted samples from 2^-k * 0.5f, times 2^k,
truncated through int32) against the C port of the reference's TemporalNRFilter run on the shifted frames, for random
clips at every (src_bits, dst_bits) pair."""
import numpy as np
import pytest

from oracle import pytnr as pt

PAIRS = [(s, d) for s in (8, 10, 12, 14) for d in (10, 12, 14, 16) if d > s]


@pytest.mark.parametrize("sb,db", PAIRS)
def test_inclusion_is_the_source_depth_test(sb, db):
    k = db - sb
    dist = np.arange(3 * ((1 << sb) - 1) + 1, dtype=np.int64)          # every |dY| + |dU| + |dV| at src_bits
    for t in list(range(0, 300)) + [1000, 4095, 65535]:
        assert np.array_equal((dist << k) <= (t << (db - 8)), dist <= (t << (sb - 8))), t


def _chains(Y, f, k):
    """Both float32 chains over a window Y (nf, n) of in-frame samples with weight f: on the shifted samples from 0.5f,
    and on the unshifted samples from 2^-k * 0.5f, scaled by 2^k."""
    a = np.full(Y.shape[1], 0.5, np.float32)
    b = np.full(Y.shape[1], np.float32(np.ldexp(0.5, -k)), np.float32)
    for i in range(Y.shape[0]):
        a = (a + (f * (Y[i] << k).astype(np.float32)).astype(np.float32)).astype(np.float32)
        b = (b + (f * Y[i].astype(np.float32)).astype(np.float32)).astype(np.float32)
    return a, (b * np.float32(2.0 ** k)).astype(np.float32)


@pytest.mark.parametrize("sb,db", PAIRS)
def test_scaled_float_chain_is_exact(sb, db):
    rng = np.random.default_rng(sb * 100 + db)
    k = db - sb
    for kk in range(1, 128):                                          # every in-frame count 2d+1 <= 127 allows
        f = np.float32(1.0) / np.float32(kk)
        Y = rng.integers(0, 1 << sb, size=(kk, 4096), dtype=np.int64)
        Y[:, :8] = (1 << sb) - 1                                       # all-maximum columns
        Y[:, 8:16] = 0
        a, b = _chains(Y, f, k)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), kk
        assert np.array_equal(a.astype(np.int32), b.astype(np.int32))


def np_tnr_widen_frame(win, W, H, sb, db, threshold, interlaced):
    """The widening kernel's formulation on one window of source frames (src_bits samples) -> dst_bits samples."""
    k = db - sb
    nf = len(win)
    ysz, cw, ch = W * H, W // 2, H // 2
    csz = cw * ch
    w = np.stack([np.asarray(f).astype(np.int64) for f in win])
    Y, U, V = w[:, :ysz].reshape(nf, H, W), w[:, ysz:ysz + csz].reshape(nf, ch, cw), w[:, ysz + csz:].reshape(nf, ch, cw)
    y = np.arange(H)
    cy = (((y >> 1) & ~1) | (y & 1)) if interlaced else (y >> 1)
    cx = np.arange(W) >> 1
    Uf, Vf = U[:, cy][:, :, cx], V[:, cy][:, :, cx]
    m = nf // 2
    inc = np.abs(Y - Y[m]) + np.abs(Uf - Uf[m]) + np.abs(Vf - Vf[m]) <= (threshold << (sb - 8))     # masks at src_bits
    f = np.float32(1.0) / inc.sum(axis=0).astype(np.float32)
    d0 = np.float32(np.ldexp(0.5, -k))
    dY, dU, dV = (np.full((H, W), d0, np.float32) for _ in range(3))
    for i in range(nf):
        c = np.where(inc[i], f, np.float32(0.0)).astype(np.float32)
        dY = (dY + (c * Y[i].astype(np.float32)).astype(np.float32)).astype(np.float32)
        dU = (dU + (c * Uf[i].astype(np.float32)).astype(np.float32)).astype(np.float32)
        dV = (dV + (c * Vf[i].astype(np.float32)).astype(np.float32)).astype(np.float32)
    s = np.float32(2.0 ** k)
    out = np.empty(ysz + 2 * csz, np.uint16)
    out[:ysz] = (dY * s).astype(np.int32).astype(np.uint16).ravel()
    rows = np.nonzero((((y >> 1) if interlaced else y) & 1) == 0)[0]          # rows that write chroma
    oU, oV = np.zeros((ch, cw), np.uint16), np.zeros((ch, cw), np.uint16)
    oU[cy[rows]] = (dU[rows][:, 0::2] * s).astype(np.int32).astype(np.uint16)
    oV[cy[rows]] = (dV[rows][:, 0::2] * s).astype(np.int32).astype(np.uint16)
    out[ysz:ysz + csz], out[ysz + csz:] = oU.ravel(), oV.ravel()
    return out


def _noisy(rng, N, W, H, bits):
    """Frames near a common base so that some window frames fall inside small thresholds and some do not."""
    n = W * H + 2 * (W // 2) * (H // 2)
    base = rng.integers(0, 1 << bits, size=n)
    step = 1 << (bits - 8)
    fr = base[None, :] + rng.integers(-3, 4, size=(N, n)) * step
    return np.clip(fr, 0, (1 << bits) - 1).astype(np.uint8 if bits == 8 else np.uint16)


@pytest.mark.parametrize("sb,db", PAIRS)
@pytest.mark.parametrize("il", [0, 1])
def test_kernel_formulation_matches_the_filter_on_shifted_frames(sb, db, il):
    rng = np.random.default_rng(1000 + 10 * sb + db + il)
    W, H, d, N = 24, 8, 3, 9
    fr = _noisy(rng, N, W, H, sb)
    wide = fr.astype(np.uint16) << (db - sb)
    for t in (0, 1, 2, 5, 65535):
        ref = pt.or_tnr_clip(wide, W, H, db, d, t, il)
        for n in range(N):
            win = [fr[min(max(n - d + i, 0), N - 1)] for i in range(2 * d + 1)]
            assert np.array_equal(np_tnr_widen_frame(win, W, H, sb, db, t, il), ref[n]), (t, n)
