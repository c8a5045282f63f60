"""amtk_logo_find_add_frames / get_sums: the per-pixel temporal sums s1 = sum Y and s2 = sum Y*Y of the logo finder,
bit-exact against numpy in int64 at every depth, size, source and layout, on the TMA and plain-load kernels, whatever the
split of the frames into calls; the bytes it uploads, the launches it makes and the clips it refuses."""
import ctypes as C

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab

pytestmark = pytest.mark.gpu


def frames(seed, n, W, H, bits):
    """n packed 4:2:0 frames (numpy, uint8 or uint16): Y noise over the whole range, a band of samples at maxv, and for
    16 bits every sample of some frames at 0xFFFF (so that s2 carries past 2^32)."""
    rng = np.random.default_rng(seed)
    maxv = (1 << bits) - 1
    ysz, csz = W * H, (W // 2) * (H // 2)
    f = rng.integers(0, maxv + 1, (n, ysz + 2 * csz), dtype=np.int64)
    f[:, :W] = maxv
    if bits == 16:
        f[::3, :ysz] = 0xFFFF
    return f.astype(np.uint8 if bits == 8 else np.uint16)


def want(f, W, H, lo=0, hi=None):
    Y = f[lo:hi, :W * H].astype(np.int64).reshape(-1, H, W)
    return Y.sum(0), (Y * Y).sum(0)


def got(fd):
    s1, s2, n = fd.sums()
    return s1.astype(np.int64), s2.view(np.int64), n


def layout_buffer(f, W, H, bits, layout, device):
    """Copies packed frames f (numpy) into a buffer of `layout`; returns (buffer, ClipDesc without base set)."""
    bps = 1 if bits == 8 else 2
    n = f.shape[0]
    ysz, csz = W * H, (W // 2) * (H // 2)
    if layout == "packed":
        py, pc = W * bps, (W // 2) * bps
        offu, offv, extra = H * py, H * py + (H // 2) * pc, 0
    elif layout == "padded":
        py, pc = ((W * bps + 15) & ~15) + 64, (((W // 2) * bps + 15) & ~15) + 32
        offu = H * py + 128
        offv = offu + (H // 2) * pc + 64
        extra = 96
    elif layout == "vfirst":
        py, pc = ((W * bps + 15) & ~15) + 16, (((W // 2) * bps + 15) & ~15) + 16
        offv = H * py
        offu = offv + (H // 2) * pc
        extra = 0
    else:                                  # oddpitch: odd byte pitches (even at 2 bytes: sample-aligned but not 16-byte)
        py, pc = W * bps + (3 if bps == 1 else 6), (W // 2) * bps + (5 if bps == 1 else 10)
        offu = H * py + 2
        offv = offu + (H // 2) * pc + 2
        extra = 2 if bps == 2 else 1
    fs = offv + (H // 2) * pc + extra if layout != "vfirst" else offu + (H // 2) * pc
    if layout == "padded":
        fs = (fs + 15) & ~15
    rng = np.random.default_rng(99)
    raw = rng.integers(0, 256, n * fs + 64, dtype=np.uint8)          # poisoned padding
    dt = np.uint8 if bps == 1 else np.uint16
    for i in range(n):
        base = i * fs
        for off, pitch, rows, cols, src in ((0, py, H, W, f[i, :ysz]), (offu, pc, H // 2, W // 2, f[i, ysz:ysz + csz]),
                                            (offv, pc, H // 2, W // 2, f[i, ysz + csz:])):
            blk = src.reshape(rows, cols).astype(dt).view(np.uint8).reshape(rows, cols * bps)
            for r in range(rows):
                o = base + off + r * pitch
                raw[o:o + cols * bps] = blk[r]
    d = ab.ClipDesc()
    d.frame_stride, d.off_u, d.off_v = fs, offu, offv
    d.width, d.height, d.pitch_y, d.pitch_uv = W, H, py, pc
    d.log_uvx = d.log_uvy = 1
    d.bytes_per_sample, d.bits_per_sample, d.num_frames = bps, bits, n
    if device == "device":
        buf = torch.from_numpy(raw).cuda()
        d.on_device = 1
    elif device == "pinned":
        buf = torch.from_numpy(raw).pin_memory()
        d.on_device = 0
    else:
        buf = raw
        d.on_device = 0
    d.base = ab.capi._ptr(buf).value
    return buf, d


def fresh_device_clip(f, W, H, bits):
    t = torch.from_numpy(f.view(np.uint8).copy()).cuda()
    return t, ab.yv12_clip(t, W, H, f.shape[0], True, bits)


@pytest.mark.parametrize("bits", [8, 10, 12, 16])
@pytest.mark.parametrize("W,H", [(1920, 1080), (1440, 1080), (1918, 1078), (17, 16)])
def test_sums_exact(ctx, bits, W, H):
    n = 7 if W * H > 1e6 else 40
    f = frames(bits * 7 + W, n, W, H, bits)
    t, d = fresh_device_clip(f, W, H, bits)
    fd = ctx.logo_find()
    before = ctx.launches
    fd.add_frames(d)
    assert ctx.launches - before == 1
    s1, s2, got_n = got(fd)
    w1, w2 = want(f, W, H)
    assert got_n == n and np.array_equal(s1, w1) and np.array_equal(s2, w2)


def test_2160p_at_16_bits(ctx):
    W, H = 3840, 2160
    f = frames(3, 5, W, H, 16)
    t, d = fresh_device_clip(f, W, H, 16)
    fd = ctx.logo_find()
    fd.add_frames(d)
    s1, s2, _ = got(fd)
    w1, w2 = want(f, W, H)
    assert np.array_equal(s1, w1) and np.array_equal(s2, w2)
    assert s2.max() > 2 ** 32


def test_2160p_at_8_bits(ctx):
    W, H = 3840, 2160
    f = frames(4, 5, W, H, 8)
    t, d = fresh_device_clip(f, W, H, 8)
    fd = ctx.logo_find()
    fd.add_frames(d)
    s1, s2, _ = got(fd)
    w1, w2 = want(f, W, H)
    assert np.array_equal(s1, w1) and np.array_equal(s2, w2)


@pytest.mark.parametrize("bits", [8, 10, 16])
@pytest.mark.parametrize("layout", ["packed", "padded", "vfirst", "oddpitch"])
@pytest.mark.parametrize("source", ["device", "pinned", "pageable"])
def test_sources_and_layouts(ctx, bits, layout, source):
    W, H, n = 338, 190, 9
    f = frames(bits + len(layout) + len(source), n, W, H, bits)
    buf, d = layout_buffer(f, W, H, bits, layout, source)
    fd = ctx.logo_find()
    before = ctx.launches
    fd.add_frames(d)
    if source == "device":
        assert ctx.launches - before == 1
    else:
        assert ctx.last_h2d_bytes == n * W * H * (1 if bits == 8 else 2)
    s1, s2, _ = got(fd)
    w1, w2 = want(f, W, H)
    assert np.array_equal(s1, w1) and np.array_equal(s2, w2)


@pytest.mark.parametrize("bits", [8, 16])
@pytest.mark.parametrize("W,H,n", [(1918, 1078, 6), (640, 360, 240)])
def test_tma_and_plain_kernels_agree(ctx, bits, W, H, n):
    """The same frames through an aligned device layout (TMA kernel) and an odd-pitch one (plain loads).  At 640 x 360 x
    240 every CTA streams ~40 tile frames, so each ring slot is refilled several times."""
    f = frames(11, n, W, H, bits)
    out = []
    for layout in ("padded", "oddpitch"):
        buf, d = layout_buffer(f, W, H, bits, layout, "device")
        fd = ctx.logo_find()
        fd.add_frames(d)
        out.append(got(fd))
    w1, w2 = want(f, W, H)
    for s1, s2, _ in out:
        assert np.array_equal(s1, w1) and np.array_equal(s2, w2)


@pytest.mark.parametrize("bits", [8, 12])
def test_splits_agree(ctx, bits):
    W, H, n = 640, 360, 37
    f = frames(21, n, W, H, bits)
    t, d = fresh_device_clip(f, W, H, bits)
    host = f.view(np.uint8).copy()
    hd = ab.yv12_clip(host, W, H, n, False, bits)
    w1, w2 = want(f, W, H)
    rng = np.random.default_rng(5)
    for kind in ("one", "random", "single"):
        fd = ctx.logo_find()
        if kind == "one":
            fd.add_frames(d)
        elif kind == "single":
            for i in range(n):
                fd.add_frames(hd if i % 2 else d, i, 1)
        else:
            cuts = sorted(set(rng.integers(1, n, 6).tolist()))
            lo = 0
            for j, hi in enumerate(cuts + [n]):
                fd.add_frames(d if j % 2 else hd, lo, hi - lo)
                lo = hi
        s1, s2, got_n = got(fd)
        assert got_n == n and np.array_equal(s1, w1) and np.array_equal(s2, w2), kind


def test_host_chunks(ctx, monkeypatch):
    """A host clip larger than one staging buffer: one launch per chunk, the bytes of the Y rows only."""
    W, H, n = 1920, 1080, 9
    f = frames(31, n, W, H, 8)
    host = torch.from_numpy(f.copy()).pin_memory()
    d = ab.yv12_clip(host, W, H, n, False, 8)
    monkeypatch.setenv("AMTK_STAGE_MB", "5")                          # two 1080p Y planes per chunk
    fd = ctx.logo_find()
    before = ctx.launches
    fd.add_frames(d)
    assert ctx.launches - before == 5
    assert ctx.last_h2d_bytes == n * W * H
    s1, s2, _ = got(fd)
    w1, w2 = want(f, W, H)
    assert np.array_equal(s1, w1) and np.array_equal(s2, w2)


def test_refused_clips_leave_the_sums(ctx):
    W, H, n = 320, 180, 6
    f = frames(41, n, W, H, 8)
    t, d = fresh_device_clip(f, W, H, 8)
    fd = ctx.logo_find()
    fd.add_frames(d, 0, 3)
    before = got(fd)
    L = ab.lib()
    g10 = frames(42, 2, W, H, 10)
    t10, d10 = fresh_device_clip(g10, W, H, 10)
    other = frames(43, 2, W + 2, H, 8)
    to, do = fresh_device_clip(other, W + 2, H, 8)
    for clip, f0, nf, msg in ((d10, 0, 1, b"differs from the first clip"), (do, 0, 1, b"differs from the first clip"),
                              (d, 4, 3, b"frame range outside the clip"), (d, -1, 1, b"frame range outside the clip")):
        assert L.amtk_logo_find_add_frames(fd.h, C.byref(clip), f0, nf) == 0
        assert msg in L.amtk_last_error()
    small = frames(44, 1, 16, 15, 8)
    ts, ds = fresh_device_clip(small, 16, 16, 8)
    ds.height = 15
    fd2 = ctx.logo_find()
    assert L.amtk_logo_find_add_frames(fd2.h, C.byref(ds), 0, 1) == 0
    assert b"[16, 8192]" in L.amtk_last_error()
    after = got(fd)
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1]) and before[2] == after[2] == 3
    fd.add_frames(d, 3, 3)
    s1, s2, _ = got(fd)
    w1, w2 = want(f, W, H)
    assert np.array_equal(s1, w1) and np.array_equal(s2, w2)


def test_chroma_is_never_read(ctx):
    """Only the Y plane is read: chroma plane offsets pointing at unmapped memory do not matter."""
    W, H, n = 256, 144, 4
    f = frames(51, n, W, H, 8)
    t, d = fresh_device_clip(f, W, H, 8)
    d.off_u = d.off_v = 1 << 40
    fd = ctx.logo_find()
    fd.add_frames(d)
    s1, s2, _ = got(fd)
    w1, w2 = want(f, W, H)
    assert np.array_equal(s1, w1) and np.array_equal(s2, w2)


def test_get_sums_before_any_frame_and_partial_outputs(ctx):
    fd = ctx.logo_find()
    s1, s2, n = fd.sums()
    assert s1 is None and n == 0
    W, H = 64, 32
    f = frames(61, 3, W, H, 8)
    t, d = fresh_device_clip(f, W, H, 8)
    fd.add_frames(d)
    L = ab.lib()
    only2 = np.zeros((H, W), np.uint64)
    nn = C.c_int64()
    assert L.amtk_logo_find_get_sums(fd.h, None, only2.ctypes.data, C.byref(nn)) == 1
    assert nn.value == 3 and np.array_equal(only2.astype(np.int64), want(f, W, H)[1])
