"""amtk_tnr_stream widening as it filters (amtk_tnr_stream_create_widening: ConvertBits fused into the frame stream): frames
sent at 8, 10, 12 or 14 bits, outputs as 2-byte samples at out_bits.  Output n must equal amtk_tnr_frames' widening output
n over the whole clip and the C port of the reference's TemporalNRFilter on the frames shifted left by the difference,
byte for byte; the tags, the receive rule, the reference emission, layouts, the upload count, out_bits = 0 and equal bits
against amtk_tnr_stream_create, and the rejections."""
import ctypes as C

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth
from amatsukaze_b200.capi import check
from oracle import pytnr as pt
from oracle import pytnr_stream as ps
from test_gpu_tnr_stream import POISON, Frame, _desc, _drain, _layout, _pack1, _unpack1

pytestmark = pytest.mark.gpu

PAIRS = ((8, 10), (8, 12), (8, 14), (8, 16), (10, 12), (10, 14), (10, 16), (12, 14), (12, 16), (14, 16))
DS = (0, 1, 3, 7, 8)                  # register-window kernels (0, 1, 3, 7) and the general kernel (8)
BS = (1, 3, 16)


def shifted(frames, sb, db):
    return frames.astype(np.uint16) << (db - sb)


def drive(ctx, frames, W, H, sb, db, d, t, il, B, ref=False, src=None, dst=None, out_bits=None, stream=None):
    """Streams `frames` (at sb bits) into outputs at db bits.  src(n) -> (layout, where) of the n-th send; dst: (layout,
    where) of the one destination buffer.  Checks the receive rule after every send and the upload count of every host
    send.  Returns (tags, output frames) in delivery order."""
    st = stream or ctx.tnr_stream(ab.tnr_params(d, t, il), B, ref, out_bits=db if out_bits is None else out_bits)
    N = frames.shape[0]
    Ld, wd = dst or (_layout(W, H, db), "host")
    out = Frame(np.full(Ld["fs"], POISON, np.uint8), Ld, wd)
    assert st.recv(out.desc) is None
    outs = []
    for n in range(N):
        Ls, ws = src(n) if src else (_layout(W, H, sb), "host")
        f = Frame(_pack1(frames[n], Ls), Ls, ws)            # alive until send returns
        st.send(f.desc, n)
        if ws != "device":
            assert ctx.last_h2d_bytes == frames.shape[1] * Ls["bps"]       # uploaded once, at the source's size
        _drain(st, out, outs)
        assert len(outs) == ps.receivable(n + 1, d, B, False), (n, len(outs))
    st.finish()
    _drain(st, out, outs)
    st.close()
    if not outs:
        return [], np.empty((0, frames.shape[1]), np.uint16)
    return [t for t, _ in outs], np.stack([o for _, o in outs])


def tnr_frames_widened(ctx, frames, W, H, sb, db, d, t, il):
    """amtk_tnr_frames over the whole clip, device to device, widening into db bits."""
    Ls, Ld = _layout(W, H, sb), _layout(W, H, db)
    N = frames.shape[0]
    src = torch.from_numpy(np.concatenate([_pack1(f, Ls) for f in frames])).cuda()
    dst = torch.full((N * Ld["fs"],), POISON, dtype=torch.uint8, device="cuda")
    ctx.tnr_frames(_desc(src.data_ptr(), Ls, True, N), _desc(dst.data_ptr(), Ld, True, N), ab.tnr_params(d, t, il))
    torch.cuda.synchronize()
    raw = dst.cpu().numpy()
    return np.stack([_unpack1(raw[n * Ld["fs"]:(n + 1) * Ld["fs"]], Ld) for n in range(N)])


@pytest.mark.parametrize("sb,db", PAIRS)
@pytest.mark.parametrize("d", DS)
@pytest.mark.parametrize("il", [0, 1])
def test_pixels_match_tnr_frames_and_the_c_port(ctx, sb, db, d, il):
    """Every batch size, clips shorter than 2d and longer than the ring (R = 2d + 2B, so the ring wraps)."""
    W, H = 76, 12                     # a ragged last group
    t = (0, 1, 5)[(d + sb) % 3]
    for B in BS:
        R = 2 * d + 2 * B
        for N in sorted({max(1, 2 * d - 1), R + B + 3}):
            fr = synth.noisy_clip(9100 + 17 * d + sb + db + B + N + il, N, W, H, sb)
            tags, got = drive(ctx, fr, W, H, sb, db, d, t, il, B)
            assert tags == list(range(N)), (B, N)
            assert np.array_equal(got, pt.or_tnr_clip(shifted(fr, sb, db), W, H, db, d, t, il)), (B, N)
            assert np.array_equal(got, tnr_frames_widened(ctx, fr, W, H, sb, db, d, t, il)), (B, N)


@pytest.mark.parametrize("sb,db", [(8, 14), (12, 16)])
@pytest.mark.parametrize("d", [1, 3, 8])
def test_reference_emission(ctx, sb, db, d):
    W, H = 24, 8
    for B in (1, 3):
        for N in range(1, 2 * d + 3):
            fr = synth.noisy_clip(70 * d + N + sb + B, N, W, H, sb)
            tags, got = drive(ctx, fr, W, H, sb, db, d, 3, 0, B, ref=True)
            idx, want = pt.or_tnr_sequence(shifted(fr, sb, db), W, H, db, d, 3, 0)
            assert tags == list(idx) == ps.emitted(N, d, True), (B, N)
            assert np.array_equal(got, want), (B, N)


@pytest.mark.parametrize("sb,db", [(8, 14), (10, 16)])
def test_mixed_layouts_and_destinations(ctx, sb, db):
    """Sends alternate host (pageable, pinned) and device, packed and padded, U-first and V-first; destinations are
    padded, V-first and poisoned, on the host and on the device (the padding must stay poisoned)."""
    W, H, d, B, N = 50, 16, 3, 4, 23
    fr = synth.noisy_clip(188 + sb, N, W, H, sb)
    want = pt.or_tnr_clip(shifted(fr, sb, db), W, H, db, d, 2, 1)
    kinds = [(_layout(W, H, sb), "host"), (_layout(W, H, sb, pad=True, vfirst=True), "device"),
             (_layout(W, H, sb, pad=True), "pinned"), (_layout(W, H, sb, vfirst=True), "host"),
             (_layout(W, H, sb), "device")]
    for dst in ((_layout(W, H, db, pad=True, vfirst=True), "host"), (_layout(W, H, db, pad=True), "device"),
                (_layout(W, H, db, pad=True), "pinned"), (_layout(W, H, db), "device")):
        tags, got = drive(ctx, fr, W, H, sb, db, d, 2, 1, B, src=lambda n: kinds[n % len(kinds)], dst=dst)
        assert tags == list(range(N))
        assert np.array_equal(got, want), dst[1]


def _plain_stream(ctx, d, t, il, B):
    out = C.c_void_p()
    check(ctx.L.amtk_tnr_stream_create(ctx.h, C.byref(ab.tnr_params(d, t, il)), B, 0, C.byref(out)))
    return ab.TnrStream(ctx, out)


@pytest.mark.parametrize("bits", [8, 10, 12, 14, 16])
def test_out_bits_zero_and_equal_bits_are_the_plain_stream(ctx, bits):
    W, H, d, B = 40, 8, 3, 4
    fr = synth.noisy_clip(77 + bits, 2 * d + 2 * B + 7, W, H, bits)
    want = drive(ctx, fr, W, H, bits, bits, d, 1, 0, B, stream=_plain_stream(ctx, d, 1, 0, B))
    assert np.array_equal(want[1], pt.or_tnr_clip(fr, W, H, bits, d, 1, 0))
    variants = [0] + ([bits] if bits > 8 else [])
    for ob in variants:
        got = drive(ctx, fr, W, H, bits, bits, d, 1, 0, B, out_bits=ob)
        assert got[0] == want[0] and np.array_equal(got[1], want[1]), ob


def test_rejections(ctx):
    for ob in (-1, 1, 8, 9, 11, 15, 17, 32):
        with pytest.raises(ab.AmtkError, match="out_bits must be 0"):
            ctx.tnr_stream(ab.tnr_params(3, 1), 4, out_bits=ob)
    W, H, d, B, N = 32, 12, 3, 2, 17
    st = ctx.tnr_stream(ab.tnr_params(d, 1, 1), B, out_bits=10)
    narrowing = "fewer bits than the source; only widening is provided"
    for bits in (12, 16):                          # narrowing: the first send fixes no format and allocates no ring
        L = _layout(W, H, bits)
        with pytest.raises(ab.AmtkError, match=narrowing):
            f = Frame(_pack1(synth.noisy_clip(bits, 1, W, H, bits)[0], L), L, "host")
            st.send(f.desc, 0)
    fr = synth.noisy_clip(5, N, W, H, 8)            # ... so an 8-bit clip may follow
    Ls, Ld = _layout(W, H, 8), _layout(W, H, 10)
    dst = Frame(np.full(Ld["fs"], POISON, np.uint8), Ld, "host")
    outs = []
    for n in range(N):
        f = Frame(_pack1(fr[n], Ls), Ls, "host")
        st.send(f.desc, n)
        if n in (0, 9):
            for L in (Ls, _layout(W, H, 12)):      # the source's format, or another 2-byte depth: not the outputs'
                wrong = Frame(np.zeros(L["fs"], np.uint8), L, "host")
                with pytest.raises(ab.AmtkError, match="differs from the stream's output format"):
                    st.recv(wrong.desc)
            L16 = _layout(W, H, 16)                 # a later frame in another format
            with pytest.raises(ab.AmtkError, match="differs from the first frame's"):
                g = Frame(_pack1(synth.noisy_clip(1, 1, W, H, 16)[0], L16), L16, "host")
                st.send(g.desc, 99)
        _drain(st, dst, outs)
        assert len(outs) == ps.receivable(n + 1, d, B, False)
    st.finish()
    _drain(st, dst, outs)
    st.close()
    assert [t for t, _ in outs] == list(range(N))
    assert np.array_equal(np.stack([o for _, o in outs]), pt.or_tnr_clip(shifted(fr, 8, 10), W, H, 10, d, 1, 1))
