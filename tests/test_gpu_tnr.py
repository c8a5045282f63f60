"""amtk_tnr_frames on the GPU, byte for byte against the C port of the reference's TemporalNRFilter (oracle/tnr_oracle.c,
itself pinned to the reference's compiled filter by tests/test_tnr_spec.py): every kernel template and the general
kernel, every bit depth, both interlace modes, thresholds at their edges, ragged widths, padded and V-first layouts,
range calls, host staging across chunk boundaries, short clips, and the rejections."""
import ctypes as C

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth
from oracle import pytnr as pt

pytestmark = pytest.mark.gpu

POISON = 0xA5


def _layout(W, H, bits, pad=False, vfirst=False, extra=0):
    bps = 1 if bits == 8 else 2
    ry, rc = W * bps, (W // 2) * bps
    py = (ry + 63) // 64 * 64 if pad else ry
    pc = (rc + 63) // 64 * 64 if pad else rc
    ysz, csz = py * H, pc * (H // 2)
    ou, ov = (ysz + csz, ysz) if vfirst else (ysz, ysz + csz)
    return dict(W=W, H=H, bits=bits, bps=bps, py=py, pc=pc, ou=ou, ov=ov, fs=ysz + 2 * csz + extra)


def _pack(frames, L):
    """(N, elems) samples -> poisoned byte buffer in layout L."""
    N, W, H, bps = frames.shape[0], L["W"], L["H"], L["bps"]
    buf = np.full(N * L["fs"], POISON, np.uint8)
    ysz, csz = W * H, (W // 2) * (H // 2)
    for n in range(N):
        fb = frames[n].view(np.uint8)
        base = n * L["fs"]
        for off, pitch, rows, rb, src in ((0, L["py"], H, W * bps, fb[:ysz * bps]),
                                          (L["ou"], L["pc"], H // 2, (W // 2) * bps, fb[ysz * bps:(ysz + csz) * bps]),
                                          (L["ov"], L["pc"], H // 2, (W // 2) * bps, fb[(ysz + csz) * bps:])):
            for r in range(rows):
                buf[base + off + r * pitch: base + off + r * pitch + rb] = src[r * rb:(r + 1) * rb]
    return buf


def _unpack(buf, L, N):
    W, H, bps = L["W"], L["H"], L["bps"]
    dt = np.uint8 if bps == 1 else np.uint16
    out = []
    for n in range(N):
        base = n * L["fs"]
        parts = []
        for off, pitch, rows, rb in ((0, L["py"], H, W * bps), (L["ou"], L["pc"], H // 2, (W // 2) * bps),
                                     (L["ov"], L["pc"], H // 2, (W // 2) * bps)):
            for r in range(rows):
                parts.append(buf[base + off + r * pitch: base + off + r * pitch + rb])
        out.append(np.concatenate(parts).view(dt))
    return np.stack(out)


def _desc(ptr, L, N, on_device):
    d = ab.ClipDesc()
    d.base = ptr
    d.frame_stride, d.off_u, d.off_v = L["fs"], L["ou"], L["ov"]
    d.width, d.height, d.pitch_y, d.pitch_uv = L["W"], L["H"], L["py"], L["pc"]
    d.log_uvx = d.log_uvy = 1
    d.bytes_per_sample, d.bits_per_sample = L["bps"], L["bits"]
    d.num_frames, d.on_device = N, int(on_device)
    return d


class Buf:
    """A clip buffer on the device (torch) or the host (numpy), with its descriptor."""

    def __init__(self, raw, L, N, on_device):
        self.L, self.N, self.dev = L, N, on_device
        self.mem = torch.from_numpy(raw).cuda() if on_device else raw
        ptr = self.mem.data_ptr() if on_device else self.mem.ctypes.data
        self.desc = _desc(ptr, L, N, on_device)

    def raw(self):
        torch.cuda.synchronize()
        return self.mem.cpu().numpy() if self.dev else self.mem.copy()


def run(ctx, frames, bits, d, t, il, W, H, frame0=0, nframes=None, src_dev=True, dst_dev=True, lsrc=None, ldst=None,
        dst_frames=None, dst_frame0=0):
    N = frames.shape[0]
    n = N - frame0 if nframes is None else nframes
    lsrc = lsrc or _layout(W, H, bits)
    ldst = ldst or _layout(W, H, bits)
    nd = dst_frames if dst_frames is not None else n
    src = Buf(_pack(frames, lsrc), lsrc, N, src_dev)
    dst = Buf(np.full(nd * ldst["fs"], POISON, np.uint8), ldst, nd, dst_dev)
    ctx.tnr_frames(src.desc, dst.desc, ab.tnr_params(d, t, il), frame0, n, dst_frame0)
    raw = dst.raw()
    return _unpack(raw, ldst, nd), raw


def _padding_untouched(raw, L, N):
    """Every byte of the destination outside the sample rows is still the poison."""
    mask = np.ones(N * L["fs"], bool)
    W, H, bps = L["W"], L["H"], L["bps"]
    for n in range(N):
        base = n * L["fs"]
        for off, pitch, rows, rb in ((0, L["py"], H, W * bps), (L["ou"], L["pc"], H // 2, (W // 2) * bps),
                                     (L["ov"], L["pc"], H // 2, (W // 2) * bps)):
            for r in range(rows):
                mask[base + off + r * pitch: base + off + r * pitch + rb] = False
    return bool((raw[mask] == POISON).all())


BITS = (8, 10, 12, 14, 16)
DS = (0, 1, 2, 3, 4, 7, 8, 15, 63)      # every register-window template (0..7) and the general kernel (8, 15, 63)


@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("d", DS)
@pytest.mark.parametrize("il", [0, 1])
def test_matrix(ctx, bits, d, il):
    W, H = 76, 12                         # 76: not a multiple of 16, 32 or 128 (a ragged last group at both sample sizes)
    N = min(2 * d + 3, 40)
    fr = synth.noisy_clip(900 + 13 * d + bits + il, N, W, H, bits)
    for t in (0, 1, 3, 65535):
        got, _ = run(ctx, fr, bits, d, t, il, W, H)
        assert np.array_equal(got, pt.or_tnr_clip(fr, W, H, bits, d, t, il)), (t,)


@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("d", DS)
@pytest.mark.parametrize("il", [0, 1])
def test_vector_path_with_ragged_edge(ctx, bits, d, il):
    """Layouts whose pitches, plane offsets and frame stride are multiples of 64 bytes take the 16-byte loads and stores
    (the path every 1080p clip runs); a 76-pixel width leaves a ragged last group on the element-wise path in the same
    launch, and a 128-pixel packed clip runs vector groups only."""
    H = 12
    N = min(2 * d + 3, 40)
    for W, pad in ((76, True), (128, False)):
        L = _layout(W, H, bits, pad=pad)
        assert L["py"] % 64 == 0 and L["pc"] % 64 == 0 and L["fs"] % 64 == 0
        fr = synth.noisy_clip(4100 + 7 * d + bits + il + W, N, W, H, bits)
        for t in (0, 1, 3, 65535):
            got, raw = run(ctx, fr, bits, d, t, il, W, H, lsrc=L, ldst=L)
            assert np.array_equal(got, pt.or_tnr_clip(fr, W, H, bits, d, t, il)), (W, t)
            assert _padding_untouched(raw, L, N)


@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("il", [0, 1])
def test_threshold_edges_and_maximum(ctx, bits, il):
    """Pixels exactly on thresh and thresh + 1 in every window frame; then a clip of all-maximum samples."""
    W, H, d, t = 40, 8, 3, 3
    th, maxv = t << (bits - 8), (1 << bits) - 1
    N = 2 * d + 4
    fr = synth.noisy_clip(31, N, W, H, bits).astype(np.int64)
    ysz = W * H
    c = fr[d].copy()
    for n in range(N):                    # luma = centre +- thresh / thresh+1 in alternating columns, chroma as the centre
        if n == d:
            continue
        delta = np.where(np.arange(ysz) % 4 < 2, th, th + 1) * np.where(np.arange(ysz) % 2 == 0, 1, -1)
        fr[n, :ysz] = np.clip(c[:ysz] + delta, 0, maxv)
        fr[n, ysz:] = c[ysz:]
    fr = fr.astype(np.uint8 if bits == 8 else np.uint16)
    got, _ = run(ctx, fr, bits, d, t, il, W, H)
    assert np.array_equal(got, pt.or_tnr_clip(fr, W, H, bits, d, t, il))
    full = np.full_like(fr, maxv)
    got, _ = run(ctx, full, bits, d, 0, il, W, H)
    assert np.array_equal(got, full)


@pytest.mark.parametrize("bits", [8, 14, 16])
@pytest.mark.parametrize("d", [3, 8])
@pytest.mark.parametrize("il", [0, 1])
@pytest.mark.parametrize("vfirst", [False, True])
def test_padded_and_v_first_layouts(ctx, bits, d, il, vfirst):
    W, H = 50, 16
    N = 2 * d + 3
    fr = synth.noisy_clip(55 + d, N, W, H, bits)
    ref = pt.or_tnr_clip(fr, W, H, bits, d, 2, il)
    lp = _layout(W, H, bits, pad=True, vfirst=vfirst, extra=24)      # rows padded to 64 bytes, a ragged frame stride
    for src_l, dst_l in ((lp, lp), (None, lp), (lp, None)):
        got, raw = run(ctx, fr, bits, d, 2, il, W, H, lsrc=src_l, ldst=dst_l)
        assert np.array_equal(got, ref)
        assert _padding_untouched(raw, dst_l or _layout(W, H, bits), N)


@pytest.mark.parametrize("bits", [8, 16])
@pytest.mark.parametrize("d", [1, 3, 8])
def test_range_calls_clamp_at_the_clip_ends(ctx, bits, d):
    W, H, N = 36, 8, 30
    fr = synth.noisy_clip(77, N, W, H, bits)
    full = pt.or_tnr_clip(fr, W, H, bits, d, 4, 0)
    for frame0, n in ((5, 7), (0, 3), (N - 4, 4), (d + 1, 1), (13, 17)):
        got, raw = run(ctx, fr, bits, d, 4, 0, W, H, frame0=frame0, nframes=n, dst_frames=n + 3, dst_frame0=2)
        assert np.array_equal(got[2:2 + n], full[frame0:frame0 + n]), (frame0, n)
        L = _layout(W, H, bits)
        assert (raw[:2 * L["fs"]] == POISON).all() and (raw[(2 + n) * L["fs"]:] == POISON).all()


@pytest.mark.parametrize("bits", [8, 16])
@pytest.mark.parametrize("d", [1, 3, 8])
@pytest.mark.parametrize("where", ["h2d", "d2h", "h2h"])
def test_host_staging_across_chunks(ctx, monkeypatch, bits, d, where):
    """AMTK_STAGE_MB=1 with 256x256 frames: a few frames per chunk, so every chunk needs halo frames from its neighbours."""
    monkeypatch.setenv("AMTK_STAGE_MB", "1")
    W, H, N = 256, 256, 2 * d + 20
    fr = synth.noisy_clip(99 + d, N, W, H, bits)
    full = pt.or_tnr_clip(fr, W, H, bits, d, 1, 1)
    src_dev, dst_dev = {"h2d": (False, True), "d2h": (True, False), "h2h": (False, False)}[where]
    got, _ = run(ctx, fr, bits, d, 1, 1, W, H, src_dev=src_dev, dst_dev=dst_dev)
    assert np.array_equal(got, full)
    got, _ = run(ctx, fr, bits, d, 1, 1, W, H, frame0=d + 3, nframes=11, src_dev=src_dev, dst_dev=dst_dev)
    assert np.array_equal(got, full[d + 3:d + 14])
    if not src_dev:
        L = _layout(W, H, bits)
        assert ctx.last_h2d_bytes > 11 * L["fs"]          # halo frames were staged too


@pytest.mark.parametrize("d", [1, 3, 7, 15])
def test_short_clips(ctx, d):
    """N = 1 and N < 2d: every frame is returned, over windows clamped at the clip's ends."""
    W, H = 24, 8
    for N in sorted({1, 2, max(1, 2 * d - 1)}):
        for bits in (8, 16):
            fr = synth.noisy_clip(3 * N + d, N, W, H, bits)
            got, _ = run(ctx, fr, bits, d, 4, 0, W, H)
            assert np.array_equal(got, pt.or_tnr_clip(fr, W, H, bits, d, 4, 0)), (N, bits)


def test_default_params():
    p = ab.default_tnr_params()
    assert (p.temporal_distance, p.threshold, p.interlaced) == (3, 1, 0)


def _expect_error(ctx, src, dst, prm, text, frame0=0, n=None):
    with pytest.raises(ab.AmtkError, match=text):
        ctx.tnr_frames(src, dst, prm, frame0, n if n is not None else src.num_frames)


def test_rejections(ctx):
    W, H, N = 32, 16, 4
    fr = synth.noisy_clip(1, N, W, H, 8)
    L = _layout(W, H, 8)
    src = Buf(_pack(fr, L), L, N, True)
    dst = Buf(np.zeros(N * L["fs"], np.uint8), L, N, True)
    _expect_error(ctx, src.desc, dst.desc, ab.tnr_params(64, 1), "temporal_distance")
    _expect_error(ctx, src.desc, dst.desc, ab.tnr_params(3, -1), "threshold")
    _expect_error(ctx, src.desc, dst.desc, ab.tnr_params(3, 65536), "threshold")
    for field, val, text in (("width", W - 1, "even"), ("height", H - 1, "even")):
        s2, d2 = _desc(src.desc.base, L, N, True), _desc(dst.desc.base, L, N, True)
        setattr(s2, field, val)
        setattr(d2, field, val)
        _expect_error(ctx, s2, d2, ab.tnr_params(3, 1), text)
    L2 = _layout(W, 18, 8)                                  # H % 4 == 2
    s2, d2 = Buf(np.zeros(N * L2["fs"], np.uint8), L2, N, True), Buf(np.zeros(N * L2["fs"], np.uint8), L2, N, True)
    ctx.tnr_frames(s2.desc, d2.desc, ab.tnr_params(3, 1, False))            # progressive: fine
    _expect_error(ctx, s2.desc, d2.desc, ab.tnr_params(3, 1, True), "multiple of 4")
    s422, d422 = _desc(src.desc.base, L, N, True), _desc(dst.desc.base, L, N, True)
    s422.log_uvy = d422.log_uvy = 0
    _expect_error(ctx, s422, d422, ab.tnr_params(3, 1), "4:2:0")
    _expect_error(ctx, src.desc, src.desc, ab.tnr_params(3, 1), "overlap")
    half = _desc(src.desc.base + L["fs"] * 2, L, N, True)                   # dst starting two frames into src
    _expect_error(ctx, src.desc, half, ab.tnr_params(3, 1), "overlap", n=2)
    hsrc = Buf(_pack(fr, L), L, N, False)
    _expect_error(ctx, hsrc.desc, hsrc.desc, ab.tnr_params(3, 1), "overlap")
    s16 = _desc(src.desc.base, L, N, True)
    s16.bits_per_sample = 10                                                # 1-byte samples at 10 bits
    _expect_error(ctx, s16, dst.desc, ab.tnr_params(3, 1), "bits_per_sample")
    _expect_error(ctx, src.desc, dst.desc, ab.tnr_params(3, 1), "frame range", frame0=2, n=3)
    assert C.sizeof(ab.TnrParams) == 12
