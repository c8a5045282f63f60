"""LogoScan on 2-byte samples (9..16 bits): amtk_scan_add_frames / amtk_scan_get_logo against the reference's own
LogoScan::AddFrame<uint16_t>, Normalize and GetLogo (oracle.pyscan16.RefScan16, compiled into oracle/_ref; PyScan16, the
restatement tests/test_logoscan16_golden.py pins to the reference's golden vectors, where that was not built), and
amtk_scan_logo / amtk_scan_logo_stream against the ScanLogo composition at maxv = (1 << bits) - 1
(oracle.pyscan16.compose_scan_logo).

The frames come from amatsukaze_b200.synth.scan_frames16: every plane's border spans a chosen spread (at most thy, exactly
thy, or thy + 1), sits at maxv in some frames, and at 16 bits mostly holds samples >= 32768, which the reference keeps in
a std::vector<short> and so sees negative.  Chroma planes of one row are left out (the 8-bit kernel's handling of their
border is not settled)."""
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth
from oracle import pyscan16 as ps


def thy_of(bits):
    return 12 << (bits - 8)


def max_splits(w, h, lx, ly, sms):
    """Frame splits of an add_frames call with enough frames: (8 * SMs) / pixel blocks (amtk_scan_add_frames)."""
    npix = w * h + 2 * (w >> lx) * (h >> ly)
    return max(1, (sms * 8) // ((npix + 255) // 256))


def call_plan(w, h, lx, ly, sms):
    """add_frames calls: per = 1, per > 1 with empty trailing splits, per > 1 with a short last split (3, 5 and 16
    frames when a rectangle has one split)."""
    s = max_splits(w, h, lx, ly, sms)
    return [3, 5, 16] if s == 1 else [s, s + 1, 2 * s - 1]


# ---------------------------------------------------------------------------------------------------------------------
# frame layouts
# ---------------------------------------------------------------------------------------------------------------------
LAYOUTS = ("packed", "vfirst", "padded", "oddpitch")


def layout(frames, W, H, lx, ly, kind):
    """Packed uint16 frames (scan_frames16) rewritten into one of LAYOUTS: (uint8 array (n, frame_stride), ClipDesc with
    base 0).  vfirst: the V plane before the U plane; padded: rows 64 / 32 bytes longer, planes 256-byte aligned, frame
    stride padded; oddpitch: pitches of an odd number of samples."""
    n = frames.shape[0]
    W2, H2 = W >> lx, H >> ly
    py, pc = {"packed": (2 * W, 2 * W2), "vfirst": (2 * W, 2 * W2), "padded": (2 * W + 64, 2 * W2 + 32),
              "oddpitch": (2 * (W + 3 - W % 2), 2 * (W2 + 1 - W2 % 2))}[kind]
    al = 256 if kind == "padded" else 2
    o1 = -(-py * H // al) * al
    o2 = -(-(o1 + pc * H2) // al) * al
    fs = o2 + pc * H2 + (512 if kind == "padded" else 0)
    off_u, off_v = (o2, o1) if kind == "vfirst" else (o1, o2)
    out = np.zeros((n, fs), np.uint8)
    ysz, csz = W * H, W2 * H2
    for off, pitch, rows, cols, src in ((0, py, H, W, 0), (off_u, pc, H2, W2, ysz), (off_v, pc, H2, W2, ysz + csz)):
        plane = frames[:, src:src + rows * cols].reshape(n, rows, cols)
        dst = out[:, off:off + pitch * rows].reshape(n, rows, pitch)
        dst[:, :, :2 * cols] = plane.view(np.uint8).reshape(n, rows, 2 * cols)
    d = ab.ClipDesc()
    d.frame_stride, d.off_u, d.off_v = fs, off_u, off_v
    d.width, d.height, d.pitch_y, d.pitch_uv = W, H, py, pc
    d.log_uvx, d.log_uvy = lx, ly
    d.bytes_per_sample, d.bits_per_sample = 2, 0
    return out, d


def clip_on(buf, desc, bits, num_frames, first=0):
    """desc over buf (torch tensor or numpy array) from frame `first`."""
    d = ab.ClipDesc.from_buffer_copy(desc)
    on_dev = isinstance(buf, torch.Tensor) and buf.is_cuda
    ptr = buf.data_ptr() if isinstance(buf, torch.Tensor) else buf.ctypes.data
    d.base = ptr + first * desc.frame_stride
    d.bits_per_sample, d.num_frames, d.on_device = bits, num_frames, 1 if on_dev else 0
    return d


def packed_clip(frames, W, H, bits, lx=1, ly=1, device=True):
    buf, desc = layout(frames, W, H, lx, ly, "packed")
    t = torch.from_numpy(buf).cuda() if device else buf
    return t, clip_on(t, desc, bits, frames.shape[0])


# ---------------------------------------------------------------------------------------------------------------------
# accumulation
# ---------------------------------------------------------------------------------------------------------------------
def oracle_scan(frames, geom, bits, thy, lx, ly, select=None):
    W, H, x, y, w, h = geom
    sc = ps.scan16_class()(w, h, thy, lx, ly)
    Y, U, V = synth.scan_rects(frames, W, H, x, y, w, h, lx, ly)
    valid = [0 if select is not None and not select[i] else int(sc.add_frame_u16(Y[i], U[i], V[i]))
             for i in range(frames.shape[0])]
    return sc, valid


def assert_same(acc, valid, sc, ref_valid, maxv, where):
    assert list(map(int, valid)) == ref_valid, where
    assert acc.num_valid == sc.nframes == sum(ref_valid), where
    assert np.array_equal(acc.sums(), sc.sums()), where                  # exact integers in doubles
    got = []
    for clean in (False, True):
        a, b = acc.get_logo(maxv, clean), sc.get_logo(maxv, clean)
        assert (a is None) == (b is None), (where, clean)
        if a is not None:
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (where, clean)
        got.append(a)
    return got


# (frame W, H, scan x, y, w, h), log_uvx, log_uvy
GEOMETRIES = {
    "420-4x4": ((32, 16, 10, 6, 4, 4), 1, 1),
    "420-6x4": ((32, 16, 12, 8, 6, 4), 1, 1),
    "420-64x50": ((128, 96, 34, 22, 64, 50), 1, 1),
    "420-96x48": ((160, 64, 40, 8, 96, 48), 1, 1),
    "420-272x64": ((320, 96, 24, 16, 272, 64), 1, 1),
    "420-320x288": ((352, 320, 16, 16, 320, 288), 1, 1),
    "420-64x50-left": ((128, 96, 0, 20, 64, 50), 1, 1),
    "420-64x50-top": ((128, 96, 30, 0, 64, 50), 1, 1),
    "420-64x50-right": ((128, 96, 64, 20, 64, 50), 1, 1),
    "420-64x50-bottom": ((128, 96, 30, 46, 64, 50), 1, 1),
    "422-64x50": ((128, 96, 34, 22, 64, 50), 1, 0),
    "422-6x4": ((32, 16, 12, 8, 6, 4), 1, 0),
    "422-272x64": ((320, 96, 24, 16, 272, 64), 1, 0),
    "444-64x50": ((128, 96, 34, 22, 64, 50), 0, 0),
    "444-4x4": ((32, 16, 10, 6, 4, 4), 0, 0),
    "411-64x50": ((128, 96, 32, 22, 64, 50), 2, 0),
    "411-8x4": ((32, 16, 8, 6, 8, 4), 2, 0),
}
CASES = [(name, bits) for name in GEOMETRIES for bits in (10, 12, 16)] + [("420-1920x1080", 10)]
GEOMETRIES["420-1920x1080"] = ((1920, 1080, 0, 0, 1920, 1080), 1, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("name,bits", CASES, ids=["%s-%dbit" % c for c in CASES])
def test_add_frames_match_reference(ctx, name, bits):
    geom, lx, ly = GEOMETRIES[name]
    W, H, x, y, w, h = geom
    assert (w >> lx) >= 2 and (h >> ly) >= 2                               # no one-row chroma border
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    plan = call_plan(w, h, lx, ly, sms)
    n = sum(plan)
    thy, maxv = thy_of(bits), (1 << bits) - 1
    frames = synth.scan_frames16(zlib.crc32(("%s/%d" % (name, bits)).encode()), n, W, H, x, y, w, h, bits, thy, lx, ly)
    Y, U, V = synth.scan_rects(frames, W, H, x, y, w, h, lx, ly)
    assert max(Y.max(), U.max(), V.max()) == maxv                          # samples at maxv
    if bits == 16:
        assert (Y >= 32768).any() and (U >= 32768).any() and (V >= 32768).any()
    dev, clip = packed_clip(frames, W, H, bits, lx, ly)
    acc = ctx.logo_scan(w, h, thy, lx, ly)
    valid, f0 = [], 0
    for k in plan:                                                         # frame splits: see call_plan
        valid.append(acc.add_frames(clip, x, y, f0, k))
        f0 += k
    sc, rv = oracle_scan(frames, geom, bits, thy, lx, ly)
    assert 0 < sum(rv) < n
    logos = assert_same(acc, np.concatenate(valid), sc, rv, maxv, name)
    assert logos[0] is not None and logos[1] is not None, name


def border_spreads(frames, geom, lx, ly, bits):
    """max - min of each plane's border per frame, as the reference sees it (short samples)."""
    W, H, x, y, w, h = geom
    out = []
    for P in synth.scan_rects(frames, W, H, x, y, w, h, lx, ly):
        ph, pw = P.shape[1:]
        ys = np.concatenate([np.zeros(pw, int), np.full(pw, ph - 1), np.repeat(np.arange(1, ph - 1), 2)])
        xs = np.concatenate([np.arange(pw), np.arange(pw), np.tile([0, pw - 1], max(0, ph - 2))])
        b = np.ascontiguousarray(P[:, ys, xs]).view(np.int16).astype(np.int64)
        out.append(b.max(axis=1) - b.min(axis=1))
    return np.stack(out, axis=1)


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [10, 12, 16])
def test_threshold_edges(ctx, bits):
    """thy in sample units, with no scaling by depth: a frame whose plane's border spans exactly thy is valid, one that
    spans thy + 1 (thy one below its max - min) is not, in Y, U and V each."""
    geom, lx, ly = GEOMETRIES["420-64x50"]
    W, H, x, y, w, h = geom
    thy = thy_of(bits)
    frames = synth.scan_frames16(500 + bits, 240, W, H, x, y, w, h, bits, thy, lx, ly)
    d = border_spreads(frames, geom, lx, ly, bits)
    want = (d <= thy).all(axis=1).astype(int).tolist()
    for p in range(3):
        assert ((d[:, p] == thy) & (d <= thy).all(axis=1)).any() and (d[:, p] == thy + 1).any(), p
    dev, clip = packed_clip(frames, W, H, bits, lx, ly)
    acc = ctx.logo_scan(w, h, thy, lx, ly)
    valid = acc.add_frames(clip, x, y)
    assert valid.tolist() == want
    sc, rv = oracle_scan(frames, geom, bits, thy, lx, ly)
    assert_same(acc, valid, sc, rv, (1 << bits) - 1, bits)


@pytest.mark.gpu
def test_frame_select(ctx):
    geom, lx, ly = GEOMETRIES["420-64x50"]
    W, H, x, y, w, h = geom
    bits, n = 12, 150
    frames = synth.scan_frames16(77, n, W, H, x, y, w, h, bits, thy_of(bits))
    dev, clip = packed_clip(frames, W, H, bits)
    sel = (np.random.default_rng(5).random(n) < 0.5).astype(np.uint8)
    acc = ctx.logo_scan(w, h, thy_of(bits))
    valid = np.concatenate([acc.add_frames(clip, x, y, 0, 61, select=sel[:61]),
                            acc.add_frames(clip, x, y, 61, n - 61, select=sel[61:])])
    sc, rv = oracle_scan(frames, geom, bits, thy_of(bits), lx, ly, select=sel)
    assert 0 < sum(rv)
    assert_same(acc, valid, sc, rv, (1 << bits) - 1, "select")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", LAYOUTS)
def test_host_clips_and_layouts(ctx, monkeypatch, kind):
    """Device, pageable and pinned clips in each layout; AMTK_STAGE_MB=1 cuts host clips into many ROI windows."""
    W, H, x, y, w, h = 640, 360, 37, 23, 272, 64
    bits, n = 10, 130
    frames = synth.scan_frames16(900 + LAYOUTS.index(kind), n, W, H, x, y, w, h, bits, thy_of(bits))
    sc, rv = oracle_scan(frames, (W, H, x, y, w, h), bits, thy_of(bits), 1, 1)
    buf, desc = layout(frames, W, H, 1, 1, kind)
    monkeypatch.setenv("AMTK_STAGE_MB", "1")
    for where, b in (("device", torch.from_numpy(buf).cuda()), ("pageable", buf), ("pinned", torch.from_numpy(buf).pin_memory())):
        acc = ctx.logo_scan(w, h, thy_of(bits))
        clip = clip_on(b, desc, bits, n)
        valid = np.concatenate([acc.add_frames(clip, x, y, 0, 57), acc.add_frames(clip, x, y, 57, n - 57)])
        assert_same(acc, valid, sc, rv, (1 << bits) - 1, (kind, where))


# ---------------------------------------------------------------------------------------------------------------------
# format rules
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_format_rules_of_add_frames(ctx, tmp_path):
    W, H, x, y, w, h = 128, 96, 34, 22, 64, 50
    frames = synth.scan_frames16(3, 40, W, H, x, y, w, h, 10, thy_of(10))
    dev, c10 = packed_clip(frames, W, H, 10)
    acc = ctx.logo_scan(w, h, thy_of(10))
    acc.add_frames(c10, x, y, 0, 20)
    before = (acc.sums(), acc.num_valid)
    _, c12 = packed_clip(frames, W, H, 12)
    _, c2b8 = packed_clip(frames, W, H, 8)                                     # 2-byte samples at 8 bits
    u8 = torch.zeros((4, W * H * 3 // 2), dtype=torch.uint8, device="cuda")
    c8 = ab.yv12_clip(u8, W, H, 4, True)
    c1b10 = ab.yv12_clip(u8, W, H, 4, True)
    c1b10.bytes_per_sample, c1b10.bits_per_sample = 1, 10                      # 1-byte samples above 8 bits
    for bad, msg in ((c12, "differs from the first"), (c8, "differs from the first"), (c2b8, "bits_per_sample"),
                     (c1b10, "bits_per_sample")):
        with pytest.raises(ab.AmtkError, match=msg):
            acc.add_frames(bad, x, y)
    assert np.array_equal(acc.sums(), before[0]) and acc.num_valid == before[1]
    acc.add_frames(c10, x, y, 20, 20)
    sc, rv = oracle_scan(frames, (W, H, x, y, w, h), 10, thy_of(10), 1, 1)
    assert acc.num_valid == sum(rv) and np.array_equal(acc.sums(), sc.sums())
    for bad in (c2b8, c1b10):                                                  # refused as a first clip too
        with pytest.raises(ab.AmtkError, match="bits_per_sample"):
            ctx.logo_scan(w, h, 12).add_frames(bad, x, y)
        with pytest.raises(ab.AmtkError, match="bits_per_sample"):
            ctx.scan_logo(bad, str(tmp_path / "x.lgd"), x, y, w, h, 12, 100)
    c8.bits_per_sample = 8                                                     # an 8-bit scan refuses 2-byte clips
    acc8 = ctx.logo_scan(w, h, 12)
    acc8.add_frames(c8, x, y)
    with pytest.raises(ab.AmtkError, match="differs from the first"):
        acc8.add_frames(c10, x, y)


def one(buf, desc, bits, i):
    return clip_on(buf, desc, bits, 1, first=i)


@pytest.mark.gpu
def test_format_rules_of_the_stream(ctx, tmp_path):
    """The first frame fixes the sample format; a frame of another depth, a 2-byte frame at 8 bits and a 1-byte frame
    above 8 bits are refused and leave the stream as it was."""
    W, H, x, y, w, h = 128, 96, 34, 22, 64, 50
    n, bits = 90, 10
    frames = synth.scan_frames16(4, n, W, H, x, y, w, h, bits, thy_of(bits))
    buf, desc = layout(frames, W, H, 1, 1, "packed")
    dev = torch.from_numpy(buf).cuda()
    s = ctx.scan_logo_stream(x, y, w, h, thy_of(bits), 1000)
    for i in range(n):
        s.send(one(dev, desc, bits, i), i + 1, n)
    s.finish(str(tmp_path / "a.lgd"))
    want = open(str(tmp_path / "a.lgd"), "rb").read()
    u8 = torch.zeros((1, W * H * 3 // 2), dtype=torch.uint8, device="cuda")
    c1b10 = ab.yv12_clip(u8, W, H, 1, True)
    c1b10.bits_per_sample = 10
    bad = [one(dev, desc, 12, 0), one(dev, desc, 16, 0), ab.yv12_clip(u8, W, H, 1, True), one(dev, desc, 8, 0), c1b10]
    s = ctx.scan_logo_stream(x, y, w, h, thy_of(bits), 1000)
    for i in range(n):
        if i == 7:
            for b in bad:
                with pytest.raises(ab.AmtkError):
                    s.send(b, i + 1, n)
            assert s.counts()[0] == 7
        s.send(one(dev, desc, bits, i), i + 1, n)
    s.finish(str(tmp_path / "b.lgd"))
    assert open(str(tmp_path / "b.lgd"), "rb").read() == want
    for first in (one(dev, desc, 8, 0), c1b10):                                # refused as a first frame
        s = ctx.scan_logo_stream(x, y, w, h, thy_of(bits), 1000)
        with pytest.raises(ab.AmtkError, match="bits_per_sample"):
            s.send(first, 1, n)
        assert s.counts() == (0, 0, 0)
        s.close()


# ---------------------------------------------------------------------------------------------------------------------
# the whole pipeline and the frame stream
# ---------------------------------------------------------------------------------------------------------------------
PGEOM = (128, 96, 34, 22, 64, 50)
PIPE_N = 450


def pipeline_frames(bits):
    W, H, x, y, w, h = PGEOM
    return synth.scan_frames16(4000 + bits, PIPE_N, W, H, x, y, w, h, bits, thy_of(bits))


def compose(frames, bits, maxf):
    W, H, x, y, w, h = PGEOM
    Y, U, V = synth.scan_rects(frames, W, H, x, y, w, h)
    return ps.compose_scan_logo(Y, U, V, w, h, thy_of(bits), maxf, (1 << bits) - 1)


def cut_inside_a_batch(frames, bits):
    """max_frames whose cut-off frame is read inside the second batch of 200, not at its end."""
    _, rv = oracle_scan(frames, PGEOM, bits, thy_of(bits), 1, 1)
    cut = next(r for r in range(241, 290) if rv[r - 1])
    return sum(rv[:cut])


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [10, 12])
@pytest.mark.parametrize("maxf", [100000, 60, "inside a stack batch"])
def test_pipeline_and_stream(ctx, tmp_path, bits, maxf):
    W, H, x, y, w, h = PGEOM
    frames = pipeline_frames(bits)
    if maxf == "inside a stack batch":
        maxf = cut_inside_a_batch(frames, bits)
    want, stored = compose(frames, bits, maxf)
    assert want is not None and 0 < len(stored) <= maxf
    kinds = {100000: ("vfirst", "pinned"), 60: ("padded", "pageable")}.get(maxf, ("oddpitch", "pinned"))
    buf, desc = layout(frames, W, H, 1, 1, kinds[0])
    dev = torch.from_numpy(buf).cuda()
    host = torch.from_numpy(buf).pin_memory() if kinds[1] == "pinned" else buf
    files = {}
    for where, b in (("device", dev), ("host", host)):
        path = str(tmp_path / ("whole-%s.lgd" % where))
        ctx.scan_logo(clip_on(b, desc, bits, PIPE_N), path, x, y, w, h, thy_of(bits), maxf, service_id=21)
        files["whole-" + where] = open(path, "rb").read()
        s = ctx.scan_logo_stream(x, y, w, h, thy_of(bits), maxf)
        copied = 0
        for i in range(PIPE_N):
            copied += 1
            if not s.send(one(b, desc, bits, i), i + 1, PIPE_N):
                break
        path = str(tmp_path / ("stream-%s.lgd" % where))
        s.finish(path, 21)
        nread, ngather, h2d = s.counts()
        assert ngather == len(stored) and nread == (stored[-1] + 1 if len(stored) == maxf else PIPE_N)
        payload = (w * h + 2 * (w >> 1) * (h >> 1)) * 2
        assert h2d == (copied * payload if where == "host" else 0)
        s.close()
        files["stream-" + where] = open(path, "rb").read()
    got = ab.Logo.load(str(tmp_path / "whole-device.lgd"))
    gi = got.info()
    assert (gi.w, gi.h, gi.imgw, gi.imgh, gi.imgx, gi.imgy) == (w, h, W, H, x, y)
    assert np.array_equal(got.tables()["data"].view(np.uint32), want.view(np.uint32))
    assert len(set(files.values())) == 1, [k for k in files if files[k] != files["whole-device"]]


def callback_model(frames, bits, n):
    """The callback sequence of ScanLogo without a cut-off: (50 r / n, r, 0, gathered) at every 200 frames read
    (:905-910), (i / N * 25 + 50 + 25 k, i, N, N) every 100 stored frames of ReMakeLogo k (:976-982), (1, N, N, N)."""
    _, rv = oracle_scan(frames, PGEOM, bits, thy_of(bits), 1, 1)
    N = sum(rv)
    out = [(50.0 * r / n, r, 0, sum(rv[:r])) for r in range(200, n + 1, 200)]
    for k in range(2):
        out += [(i / N * 25 + 50 + 25 * k, i, N, N) for i in range(0, N, 100)]
    return out + [(1.0, N, N, N)]


def same_calls(got, want):
    assert [c[1:] for c in got] == [c[1:] for c in want]
    assert np.allclose([c[0] for c in got], [c[0] for c in want], rtol=1e-6, atol=0)


@pytest.mark.gpu
def test_callbacks_and_cancel(ctx, tmp_path):
    W, H, x, y, w, h = PGEOM
    bits = 10
    frames = pipeline_frames(bits)
    want = callback_model(frames, bits, PIPE_N)
    dev, clip = packed_clip(frames, W, H, bits)
    buf, desc = layout(frames, W, H, 1, 1, "packed")
    seen = []
    ctx.scan_logo(clip, str(tmp_path / "a.lgd"), x, y, w, h, thy_of(bits), 100000, cb=lambda *a: seen.append(a) or True)
    same_calls(seen, want)
    seen = []
    s = ctx.scan_logo_stream(x, y, w, h, thy_of(bits), 100000, cb=lambda *a: seen.append(a) or True)
    for i in range(PIPE_N):
        s.send(one(dev, desc, bits, i), i + 1, PIPE_N)
    s.finish(str(tmp_path / "b.lgd"))
    s.close()
    same_calls(seen, want)
    assert open(str(tmp_path / "a.lgd"), "rb").read() == open(str(tmp_path / "b.lgd"), "rb").read()
    # cancel at the second callback: the 400th frame read
    calls = []
    with pytest.raises(ab.AmtkError, match="Cancel requested"):
        ctx.scan_logo(clip, str(tmp_path / "c.lgd"), x, y, w, h, thy_of(bits), 100000, cb=lambda *a: calls.append(a) or len(calls) < 2)
    assert len(calls) == 2 and not os.path.exists(str(tmp_path / "c.lgd"))
    calls = []
    s = ctx.scan_logo_stream(x, y, w, h, thy_of(bits), 100000, cb=lambda *a: calls.append(a) or len(calls) < 2)
    for i in range(399):
        s.send(one(dev, desc, bits, i), i + 1, PIPE_N)
    with pytest.raises(ab.AmtkError, match="Cancel requested"):
        s.send(one(dev, desc, bits, 399), 400, PIPE_N)
    with pytest.raises(ab.AmtkError, match="closed"):
        s.send(one(dev, desc, bits, 400), 401, PIPE_N)
    s.close()
    assert len(calls) == 2


# ---------------------------------------------------------------------------------------------------------------------
# the host-side mirror: logo::LogoAnalyzer (tests/cpp/test_scan_logo_stream_deep.cpp)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("bits", [10, 12])
def test_mirror_logo_analyzer(ctx, tmp_path, bits):
    from amatsukaze_b200 import _build
    exe = _build.build_scan_logo_stream_deep_test() if os.path.exists("/usr/bin/g++") else _build.SCAN_LOGO_STREAM_DEEP_TEST
    W, H, x, y, w, h = PGEOM
    frames = pipeline_frames(bits)
    maxf = 250
    with open(tmp_path / "src.dat", "wb") as f:
        f.write(b"AMTSRAW1" + struct.pack("<6i", W, H, bits, PIPE_N, 30000, 1001))
        f.write(frames.tobytes())
    args = [tmp_path / "src.dat", x, y, w, h, thy_of(bits), maxf, 7, tmp_path / "cpu.lgd", tmp_path / "src.lgd"]
    r = subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "in_order=1" in r.stdout and ("source: bits=%d resident=1" % bits) in r.stdout, r.stdout
    dev, clip = packed_clip(frames, W, H, bits)
    ctx.scan_logo(clip, str(tmp_path / "w.lgd"), x, y, w, h, thy_of(bits), maxf, service_id=7)
    want = open(tmp_path / "w.lgd", "rb").read()
    assert open(tmp_path / "cpu.lgd", "rb").read() == want
    assert open(tmp_path / "src.lgd", "rb").read() == want
