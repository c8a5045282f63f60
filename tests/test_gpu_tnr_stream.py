"""amtk_tnr_stream (temporal noise reduction one frame at a time: the reference's cudaTNRCreate / SendFrame / RecvFrame /
Finish) on the GPU, byte for byte against the C port of the reference's TemporalNRFilter (oracle/tnr_oracle.c) and
against amtk_tnr_frames on the same clip: a covering set of bit depths, d, batch sizes, interlace modes, thresholds and clip
lengths, the reference emission, the receive rule after every send, mixed layouts, the upload count, pending outputs,
independence, cleanup, every rejection, and the reference's own CudaTemporalNRFilter over the library."""
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth
from oracle import pytnr as pt
from oracle import pytnr_stream as ps

pytestmark = pytest.mark.gpu

POISON = 0xA5


def _layout(W, H, bits, pad=False, vfirst=False):
    bps = 1 if bits == 8 else 2
    ry, rc = W * bps, (W // 2) * bps
    py = (ry + 63) // 64 * 64 + 16 if pad else ry          # padded: rows of a 16-byte but not 64-byte multiple
    pc = (rc + 63) // 64 * 64 if pad else rc
    ysz, csz = py * H, pc * (H // 2)
    ou, ov = (ysz + csz, ysz) if vfirst else (ysz, ysz + csz)
    return dict(W=W, H=H, bits=bits, bps=bps, py=py, pc=pc, ou=ou, ov=ov, fs=ysz + 2 * csz + (24 if pad else 0))


def _planes(L):
    W, H, bps = L["W"], L["H"], L["bps"]
    return ((0, L["py"], H, W * bps), (L["ou"], L["pc"], H // 2, (W // 2) * bps), (L["ov"], L["pc"], H // 2, (W // 2) * bps))


def _pack1(frame, L):
    """One packed frame (elems,) -> poisoned byte buffer in layout L."""
    buf = np.full(L["fs"], POISON, np.uint8)
    fb = frame.view(np.uint8)
    pos = 0
    for off, pitch, rows, rb in _planes(L):
        for r in range(rows):
            buf[off + r * pitch: off + r * pitch + rb] = fb[pos:pos + rb]
            pos += rb
    return buf


def _unpack1(buf, L):
    dt = np.uint8 if L["bps"] == 1 else np.uint16
    return np.concatenate([buf[off + r * pitch: off + r * pitch + rb] for off, pitch, rows, rb in _planes(L)
                           for r in range(rows)]).view(dt)


def _padding_untouched(buf, L):
    mask = np.ones(L["fs"], bool)
    for off, pitch, rows, rb in _planes(L):
        for r in range(rows):
            mask[off + r * pitch: off + r * pitch + rb] = False
    return bool((buf[mask] == POISON).all())


def _desc(ptr, L, on_device, num_frames=1):
    d = ab.ClipDesc()
    d.base = ptr
    d.frame_stride, d.off_u, d.off_v = L["fs"], L["ou"], L["ov"]
    d.width, d.height, d.pitch_y, d.pitch_uv = L["W"], L["H"], L["py"], L["pc"]
    d.log_uvx = d.log_uvy = 1
    d.bytes_per_sample, d.bits_per_sample = L["bps"], L["bits"]
    d.num_frames, d.on_device = num_frames, int(on_device)
    return d


class Frame:
    """One frame buffer on the host (pageable or pinned) or the device, with its descriptor."""

    def __init__(self, raw, L, where):
        self.L, self.where = L, where
        if where == "device":
            self.mem = torch.from_numpy(raw).cuda()
            torch.cuda.synchronize()
            ptr = self.mem.data_ptr()
        elif where == "pinned":
            self.mem = torch.from_numpy(raw).pin_memory()
            ptr = self.mem.data_ptr()
        else:
            self.mem = raw.copy()
            ptr = self.mem.ctypes.data
        self.desc = _desc(ptr, L, where == "device")

    def raw(self):
        if self.where == "device":
            torch.cuda.synchronize()
            return self.mem.cpu().numpy()
        return self.mem.numpy().copy() if self.where == "pinned" else self.mem.copy()


def _drain(st, dst, outs):
    while True:
        tag = st.recv(dst.desc)
        if tag is None:
            return
        raw = dst.raw()
        assert _padding_untouched(raw, dst.L)
        outs.append((tag, _unpack1(raw, dst.L)))


def drive(ctx, frames, W, H, bits, d, t, il, B, ref=False, src=None, dst=None, tags=None, check_rule=True, drain=True):
    """Streams `frames` through a new stream.  src(n) -> (layout, where) of the n-th send; dst: (layout, where) of the one
    destination buffer.  After every send the number of outputs received must follow the receive rule.  Returns
    (tags, output frames) in delivery order."""
    st = ctx.tnr_stream(ab.tnr_params(d, t, il), B, ref)
    N = frames.shape[0]
    Ld, wd = dst or (_layout(W, H, bits), "host")
    out = Frame(np.full(Ld["fs"], POISON, np.uint8), Ld, wd)
    assert st.recv(out.desc) is None                           # nothing sent: nothing to receive
    tags = list(range(N)) if tags is None else tags
    outs = []
    for n in range(N):
        Ls, ws = src(n) if src else (_layout(W, H, bits), "host")
        f = Frame(_pack1(frames[n], Ls), Ls, ws)
        st.send(f.desc, tags[n])
        if ws != "device":
            assert ctx.last_h2d_bytes == frames.shape[1] * Ls["bps"]      # the frame's sample bytes, uploaded once
        if drain:
            _drain(st, out, outs)
            if check_rule:
                assert len(outs) == ps.receivable(n + 1, d, B, False), (n, len(outs))
    st.finish()
    _drain(st, out, outs)
    st.close()
    if not outs:
        return [], np.empty((0, frames.shape[1]), frames.dtype)
    return [t for t, _ in outs], np.stack([o for _, o in outs])


def _tnr_frames(ctx, frames, W, H, bits, d, t, il):
    """amtk_tnr_frames over the whole clip, device to device (packed)."""
    L = _layout(W, H, bits)
    N = frames.shape[0]
    src = torch.from_numpy(np.concatenate([_pack1(f, L) for f in frames])).cuda()
    dst = torch.full_like(src, POISON)
    ctx.tnr_frames(_desc(src.data_ptr(), L, True, N), _desc(dst.data_ptr(), L, True, N), ab.tnr_params(d, t, il))
    torch.cuda.synchronize()
    raw = dst.cpu().numpy()
    return np.stack([_unpack1(raw[n * L["fs"]:(n + 1) * L["fs"]], L) for n in range(N)])


# Covering set: every d <= 7 template and the general kernel (8, 63) at both sample sizes; every bit depth, batch size,
# interlace mode and threshold appears.
BITS16 = (10, 12, 14, 16)
BS = (1, 2, 5, 64)
TS = (0, 1, 65535)
CASES = []
for i, d in enumerate((0, 1, 2, 3, 4, 5, 6, 7, 8, 63)):
    CASES.append((8, d, BS[i % 4], i % 2, TS[i % 3]))
    CASES.append((BITS16[i % 4], d, BS[(i + 1) % 4], (i + 1) % 2, TS[(i + 1) % 3]))


@pytest.mark.parametrize("bits,d,B,il,t", CASES)
def test_pixels_match_the_c_port_and_tnr_frames(ctx, bits, d, B, il, t):
    W, H = 76, 12                 # a ragged last group at both sample sizes
    Ns = sorted({n for n in (1, d, 2 * d - 1, 2 * d, 2 * d + 1, B - 1, B, B + 1) if n >= 1})
    for N in Ns:
        fr = synth.noisy_clip(7000 + 31 * d + bits + N + B, N, W, H, bits)
        tags, got = drive(ctx, fr, W, H, bits, d, t, il, B)
        assert tags == list(range(N))
        want = pt.or_tnr_clip(fr, W, H, bits, d, t, il)
        assert np.array_equal(got, want), (N,)
        assert np.array_equal(got, _tnr_frames(ctx, fr, W, H, bits, d, t, il)), (N,)


@pytest.mark.parametrize("bits,d,B", [(8, 3, 5), (16, 8, 2), (14, 1, 1)])
def test_long_clip_wraps_the_ring(ctx, bits, d, B):
    W, H = 64, 8
    R = 2 * d + 2 * B
    N = 5 * R + B + 3
    fr = synth.noisy_clip(321 + d, N, W, H, bits)
    tags, got = drive(ctx, fr, W, H, bits, d, 2, 0, B, tags=[1000 + 3 * n for n in range(N)])
    assert tags == [1000 + 3 * n for n in range(N)]
    assert np.array_equal(got, pt.or_tnr_clip(fr, W, H, bits, d, 2, 0))


@pytest.mark.parametrize("d", [1, 3, 7, 8])
@pytest.mark.parametrize("B", [1, 3])
def test_reference_emission(ctx, d, B):
    W, H = 24, 8
    for bits in (8, 14):
        for N in range(1, 2 * d + 3):
            fr = synth.noisy_clip(50 * d + N + bits, N, W, H, bits)
            tags, got = drive(ctx, fr, W, H, bits, d, 3, 0, B, ref=True)
            idx, want = pt.or_tnr_sequence(fr, W, H, bits, d, 3, 0)
            assert tags == list(idx) == ps.emitted(N, d, True), (N,)
            assert np.array_equal(got, want), (N,)
            if pt.ref_available():
                ridx, rwant = pt.ref_tnr_sequence(fr, W, H, bits, d, 3, 0)
                assert tags == list(ridx) and np.array_equal(got, rwant), (N,)


def test_mixed_layouts_and_destinations(ctx):
    """Sends alternate host (pageable, pinned) and device, packed and padded, U-first and V-first; destinations are
    padded, V-first and poisoned, on the host and on the device."""
    W, H, d, B = 50, 16, 3, 4
    for bits in (8, 16):
        N = 23
        fr = synth.noisy_clip(88 + bits, N, W, H, bits)
        want = pt.or_tnr_clip(fr, W, H, bits, d, 2, 1)
        kinds = [(_layout(W, H, bits), "host"), (_layout(W, H, bits, pad=True, vfirst=True), "device"),
                 (_layout(W, H, bits, pad=True), "pinned"), (_layout(W, H, bits, vfirst=True), "host"),
                 (_layout(W, H, bits), "device")]
        for dst in ((_layout(W, H, bits, pad=True, vfirst=True), "host"), (_layout(W, H, bits, pad=True), "device"),
                    (_layout(W, H, bits, pad=True), "pinned")):
            tags, got = drive(ctx, fr, W, H, bits, d, 2, 1, B, src=lambda n: kinds[n % len(kinds)], dst=dst)
            assert tags == list(range(N))
            assert np.array_equal(got, want), dst[1]


def test_pending_outputs_stay_until_received(ctx):
    """Send everything, finish, then receive everything: the same as receiving as soon as allowed."""
    W, H, bits, d, B = 40, 8, 8, 3, 4
    for N in (1, 6, 37):
        fr = synth.noisy_clip(5 + N, N, W, H, bits)
        a = drive(ctx, fr, W, H, bits, d, 1, 0, B)
        b = drive(ctx, fr, W, H, bits, d, 1, 0, B, drain=False)
        assert a[0] == b[0] == list(range(N))
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[1], pt.or_tnr_clip(fr, W, H, bits, d, 1, 0))


def test_two_streams_on_one_context(ctx):
    W, H = 32, 8
    fa, fb = synth.noisy_clip(1, 30, W, H, 8), synth.noisy_clip(2, 25, W, H, 12)
    La, Lb = _layout(W, H, 8), _layout(W, H, 12)
    sa = ctx.tnr_stream(ab.tnr_params(3, 1, 0), 4)
    sb = ctx.tnr_stream(ab.tnr_params(8, 2, 1), 3)
    da, db = Frame(np.full(La["fs"], POISON, np.uint8), La, "host"), Frame(np.full(Lb["fs"], POISON, np.uint8), Lb, "device")
    oa, ob = [], []
    for n in range(30):
        sa.send(Frame(_pack1(fa[n], La), La, "host").desc, n)
        _drain(sa, da, oa)
        if n < 25:
            sb.send(Frame(_pack1(fb[n], Lb), Lb, "device").desc, 100 + n)
            _drain(sb, db, ob)
    sb.finish()
    _drain(sb, db, ob)
    sa.finish()
    _drain(sa, da, oa)
    assert [t for t, _ in oa] == list(range(30)) and [t for t, _ in ob] == list(range(100, 125))
    assert np.array_equal(np.stack([o for _, o in oa]), pt.or_tnr_clip(fa, W, H, 8, 3, 1, 0))
    assert np.array_equal(np.stack([o for _, o in ob]), pt.or_tnr_clip(fb, W, H, 12, 8, 2, 1))


def test_one_stream_from_two_threads(ctx):
    W, H, N = 32, 8, 29
    fr = synth.noisy_clip(9, N, W, H, 10)
    L = _layout(W, H, 10)
    st = ctx.tnr_stream(ab.tnr_params(3, 1, 0), 2)
    dst = Frame(np.full(L["fs"], POISON, np.uint8), L, "host")
    outs, names = [], set()
    ex = [ThreadPoolExecutor(1), ThreadPoolExecutor(1)]

    def step(n):
        names.add(threading.get_ident())
        st.send(Frame(_pack1(fr[n], L), L, "host").desc, n)
        _drain(st, dst, outs)

    for n in range(N):
        ex[n % 2].submit(step, n).result()
    ex[N % 2].submit(st.finish).result()
    ex[(N + 1) % 2].submit(_drain, st, dst, outs).result()
    for e in ex:
        e.shutdown()
    st.close()
    assert len(names) == 2
    assert [t for t, _ in outs] == list(range(N))
    assert np.array_equal(np.stack([o for _, o in outs]), pt.or_tnr_clip(fr, W, H, 10, 3, 1, 0))


def test_destroy_mid_clip_releases_memory(ctx):
    W, H = 1920, 1080
    L = _layout(W, H, 8)
    frames = [Frame(_pack1(f, L), L, "pinned") for f in synth.noisy_clip(3, 12, W, H, 8)]
    dst = Frame(np.zeros(L["fs"], np.uint8), L, "pinned")

    def one(k):
        st = ctx.tnr_stream(ab.tnr_params(3, 1, 0), 4)
        for n in range(5 + k % 7):
            st.send(frames[n].desc, n)
            st.recv(dst.desc)
        st.close()                          # mid-clip: frames in the ring, a batch in flight, outputs pending

    one(0)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for k in range(50):
        one(k)
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    assert abs(free1 - free0) <= 0.01 * free0, (free0, free1)


def _fmt_desc(mem, L, on_device=False):
    return _desc(mem.ctypes.data if not on_device else mem.data_ptr(), L, on_device)


def test_rejections_leave_the_stream_working(ctx):
    with pytest.raises(ab.AmtkError, match="temporal_distance"):
        ctx.tnr_stream(ab.tnr_params(64, 1))
    with pytest.raises(ab.AmtkError, match="temporal_distance"):
        ctx.tnr_stream(ab.tnr_params(-1, 1))
    for t in (-1, 65536):
        with pytest.raises(ab.AmtkError, match="threshold"):
            ctx.tnr_stream(ab.tnr_params(3, t))
    for B in (0, 257):
        with pytest.raises(ab.AmtkError, match="batch_size"):
            ctx.tnr_stream(ab.tnr_params(3, 1), B)
    ctx.tnr_stream(ab.tnr_params(63, 65535), 256).close()           # the edges are accepted

    W, H, N, d, B = 32, 12, 17, 3, 2                                 # H % 4 == 0 only for the interlaced checks below
    fr = synth.noisy_clip(4, N, W, H, 8)
    L = _layout(W, H, 8)
    st = ctx.tnr_stream(ab.tnr_params(d, 1, 1), B)
    dst = Frame(np.full(L["fs"], POISON, np.uint8), L, "host")
    outs = []

    def bad_send(desc, text):
        with pytest.raises(ab.AmtkError, match=text):
            st.send(desc, 999)

    def bad_recv(desc, text):
        with pytest.raises(ab.AmtkError, match=text):
            st.recv(desc)

    def check_first_frames_rejected():
        buf = _pack1(fr[0], L)
        for field, val, text in (("width", W - 1, "even"), ("height", H - 2, "multiple of 4"), ("log_uvy", 0, "4:2:0"),
                                 ("bits_per_sample", 10, "bits_per_sample"), ("num_frames", 2, "one frame")):
            dd = _fmt_desc(buf, L)
            setattr(dd, field, val)
            bad_send(dd, text)
        odd = _fmt_desc(buf, L)
        odd.height = H - 1
        bad_send(odd, "even")

    check_first_frames_rejected()                    # before the format is fixed
    for n in range(N):
        st.send(Frame(_pack1(fr[n], L), L, "host").desc, n)
        if n in (0, 7):
            check_first_frames_rejected()            # after it, too
            L2 = _layout(W + 2, H, 8)                # another size
            bad_send(_fmt_desc(_pack1(synth.noisy_clip(1, 1, W + 2, H, 8)[0], L2), L2), "differs")
            L16 = _layout(W, H, 16)                  # another sample format
            bad_send(_fmt_desc(_pack1(synth.noisy_clip(1, 1, W, H, 16)[0], L16), L16), "differs")
            bad_recv(Frame(np.zeros(L2["fs"], np.uint8), L2, "host").desc, "differs")
            bad_recv(Frame(np.zeros(L16["fs"], np.uint8), L16, "host").desc, "differs")
            d14 = Frame(np.zeros(L16["fs"], np.uint8), L16, "host").desc
            d14.bits_per_sample = 14
            bad_recv(d14, "differs")
        _drain(st, dst, outs)
        assert len(outs) == ps.receivable(n + 1, d, B, False)
    st.finish()
    bad_send(Frame(_pack1(fr[0], L), L, "host").desc, "after finish")
    with pytest.raises(ab.AmtkError, match="twice"):
        st.finish()
    _drain(st, dst, outs)
    st.close()
    assert [t for t, _ in outs] == list(range(N))
    assert np.array_equal(np.stack([o for _, o in outs]), pt.or_tnr_clip(fr, W, H, 8, d, 1, 1))


@pytest.mark.skipif(not ps.ref_available(), reason="oracle/_ref has no build of the reference's CudaTemporalNRFilter")
@pytest.mark.parametrize("bits", [8, 14])
@pytest.mark.parametrize("N", [1, 5, 40])
def test_reference_cuda_filter_drop_in(native_lib, bits, N):
    """The reference's own CudaTemporalNRFilter, its cudaTNR* calls mapped onto amtk_tnr_stream_*: it throws nothing
    (its frame-count checks hold), emits frameIndex_ 0..N-1, and the bytes equal the C port."""
    W, H, d, t = 48, 16, 3, 1
    fr = synth.noisy_clip(600 + N + bits, N, W, H, bits)
    for B in (1, 4):
        idx, got = ps.ref_cuda_tnr_sequence(ab.LIB_PATH, fr, W, H, bits, d, t, 0, B)
        assert list(idx) == list(range(N))
        assert np.array_equal(got, pt.or_tnr_clip(fr, W, H, bits, d, t, 0))
