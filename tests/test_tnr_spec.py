"""Temporal noise reduction spec (TemporalNRFilter, VideoFilter.hpp:27-212): the C port (oracle/tnr_oracle.c) against
the reference's own compiled filter (live where oracle/_ref was built, and through tests/golden/tnr_golden.json
everywhere), the numpy restatement against both, the reference's short-clip emission, and two cases that pin the
inclusion boundary and the interlaced chroma row mapping.  CPU only."""
import hashlib
import json
import os

import numpy as np
import pytest

from amatsukaze_b200 import synth
from oracle import pytnr as pt

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tnr_golden.json")
BITS = (8, 10, 12, 14, 16)


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


def _clamped(frames, n, d):
    N = frames.shape[0]
    return [frames[min(max(n - d + i, 0), N - 1)] for i in range(2 * d + 1)]


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_golden_covers_the_matrix():
    g = _golden()
    rows = g["cases"]
    assert {r[0] for r in rows} == set(BITS)
    assert {r[1] for r in rows} == {0, 1, 3, 7, 63}
    assert {r[2] for r in rows} == {0, 1, 4, 65535}
    assert {r[3] for r in rows} == {0, 1}
    for d in (0, 1, 3, 7):
        assert {r[4] for r in rows if r[1] == d} >= set(range(1, 2 * d + 3))


@pytest.mark.parametrize("bits", BITS)
def test_c_port_equals_reference_golden(bits):
    g = _golden()
    W, H = g["W"], g["H"]
    n = 0
    for b, d, t, il, N, seed, idx, sha_seq, sha_full in g["cases"]:
        if b != bits:
            continue
        fr = synth.noisy_clip(seed, N, W, H, bits)
        oidx, oseq = pt.or_tnr_sequence(fr, W, H, bits, d, t, il)
        assert oidx.tolist() == idx, (d, t, il, N)
        assert _sha(oseq) == sha_seq, ("emitted frames", d, t, il, N)
        assert _sha(pt.or_tnr_clip(fr, W, H, bits, d, t, il)) == sha_full, ("clamped windows", d, t, il, N)
        n += 1
    assert n > 0


@pytest.mark.skipif(not pt.ref_available(), reason="oracle/_ref (the reference's TemporalNRFilter) not built here")
@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("il", [0, 1])
def test_c_port_equals_reference_live(bits, il):
    W, H = 38, 20                                   # 38 % 4 == 2 luma, odd chroma width
    for d, t, N in ((0, 1, 3), (1, 0, 5), (2, 3, 4), (3, 1, 9), (3, 4, 5), (5, 65535, 12), (9, 2, 7)):
        fr = synth.noisy_clip(1000 + 7 * d + t + il, N, W, H, bits)
        ridx, rseq = pt.ref_tnr_sequence(fr, W, H, bits, d, t, il)
        oidx, oseq = pt.or_tnr_sequence(fr, W, H, bits, d, t, il)
        assert np.array_equal(ridx, oidx)
        assert np.array_equal(rseq, oseq), (d, t, N)
        lib = pt.or_tnr_clip(fr, W, H, bits, d, t, il)
        for n in range(N):
            assert np.array_equal(pt.ref_tnr_frame(_clamped(fr, n, d), W, H, bits, t, il), lib[n]), (d, t, n)


@pytest.mark.parametrize("bits", BITS)
def test_numpy_restatement_equals_c_port(bits):
    W, H = 20, 12
    for d, t, il in ((0, 1, 0), (1, 1, 1), (3, 1, 0), (3, 4, 1), (4, 0, 0), (2, 65535, 1)):
        fr = synth.noisy_clip(77 + d, 2 * d + 3, W, H, bits)
        lib = pt.or_tnr_clip(fr, W, H, bits, d, t, il)
        for n in range(fr.shape[0]):
            assert np.array_equal(pt.np_tnr_frame(_clamped(fr, n, d), W, H, bits, t, il), lib[n]), (d, t, il, n)


@pytest.mark.skipif(not pt.ref_available(), reason="oracle/_ref (the reference's TemporalNRFilter) not built here")
def test_numpy_restatement_equals_reference_live():
    W, H = 20, 12
    for bits in BITS:
        fr = synth.noisy_clip(5, 7, W, H, bits)
        for il in (0, 1):
            win = list(fr)
            assert np.array_equal(pt.np_tnr_frame(win, W, H, bits, 2, il), pt.ref_tnr_frame(win, W, H, bits, 2, il))


def test_short_clip_sequences_pinned():
    """The reference's queue drops frames of clips shorter than 2d (d = 3: N = 5 -> 0,1,3,4; N = 4 -> 0,3; N <= 3 -> none);
    from N = 2d on it emits every frame in order."""
    got = {N: [i for i, _ in pt.sequence_windows(N, 3)] for N in range(1, 9)}
    assert got == {1: [], 2: [], 3: [], 4: [0, 3], 5: [0, 1, 3, 4], 6: list(range(6)), 7: list(range(7)), 8: list(range(8))}
    for d in (0, 1, 2, 7):
        for N in range(2 * d, 2 * d + 4):
            if N == 0:
                continue
            seq = pt.sequence_windows(N, d)
            assert [i for i, _ in seq] == list(range(N))
            assert [w for _, w in seq] == [[min(max(n - d + i, 0), N - 1) for i in range(2 * d + 1)] for n in range(N)]


def _const_frames(nf, W, H, bits, y, u, v):
    dt = np.uint8 if bits == 8 else np.uint16
    ysz, csz = W * H, (W // 2) * (H // 2)
    f = np.empty((nf, ysz + 2 * csz), dt)
    f[:, :ysz], f[:, ysz:ysz + csz], f[:, ysz + csz:] = y, u, v
    return f


@pytest.mark.parametrize("bits", BITS)
def test_difference_equal_to_thresh_is_included(bits):
    """diff == thresh is in the average, thresh + 1 is not (VideoFilter.hpp:178, `diff <= thresh`)."""
    W, H, t = 4, 4, 3
    th = t << (bits - 8)
    c = 100 << (bits - 8)
    fr = _const_frames(3, W, H, bits, c, c, c)
    fr[0, :W * H] = c + th              # luma pixel differs by exactly thresh in frame 0 ...
    fr[2, :W * H] = c + th + 1          # ... and by thresh + 1 in frame 2
    out = pt.or_tnr_frame(list(fr), W, H, bits, t, 0)
    # k = 2: 0.5 + 0.5*(c+th) + 0.5*c
    want = int(np.float32(0.5) + np.float32(0.5) * np.float32(c + th) + np.float32(0.5) * np.float32(c))
    assert (out[:W * H] == want).all()
    assert np.array_equal(out, pt.np_tnr_frame(list(fr), W, H, bits, t, 0))
    if pt.ref_available():
        assert np.array_equal(out, pt.ref_tnr_frame(list(fr), W, H, bits, t, 0))
    fr[0, :W * H] = c + th + 1          # now neither is in: the centre frame alone
    assert (pt.or_tnr_frame(list(fr), W, H, bits, t, 0)[:W * H] == c).all()


@pytest.mark.parametrize("il", [0, 1])
def test_chroma_row_takes_the_mask_of_its_luma_row(il):
    """Frame 0 of the window breaks away in one luma row only; the chroma row whose output that luma row writes is the only
    one that loses frame 0's (distinct) chroma: (2cx, 2cy) progressive, (2cx, 4(cy>>1) + (cy&1)) interlaced."""
    W, H, bits, t = 8, 16, 8, 4
    ysz, csz = W * H, (W // 2) * (H // 2)
    for R in range(H):
        fr = _const_frames(3, W, H, bits, 100, 100, 100)
        fr[0, ysz:ysz + csz] = 102                                   # frame 0's U: in whenever its luma is
        fr[0, R * W:(R + 1) * W] = 160                               # luma row R of frame 0: out
        out = pt.or_tnr_frame(list(fr), W, H, bits, t, il)
        U = out[ysz:ysz + csz].reshape(H // 2, W // 2)
        writes = ((R >> 1) if il else R) & 1 == 0
        cyR = (((R >> 1) & ~1) | (R & 1)) if il else R >> 1
        distinct = [cy for cy in range(H // 2) if U[cy, 0] != U[(cy + 1) % (H // 2), 0] and U[cy, 0] == 100]
        assert distinct == ([cyR] if writes else []), (R, U[:, 0])
        assert np.array_equal(out, pt.np_tnr_frame(list(fr), W, H, bits, t, il))
        if pt.ref_available():
            assert np.array_equal(out, pt.ref_tnr_frame(list(fr), W, H, bits, t, il))


def test_d0_copies_the_frame():
    for bits in BITS:
        fr = synth.noisy_clip(3, 4, 10, 8, bits)
        assert np.array_equal(pt.or_tnr_clip(fr, 10, 8, bits, 0, 65535, 0), fr)
