"""amtk_logo_scan_stream: LogoFrame::ScanFrame fed one decoded frame at a time (DESIGN.md section 3.3.3).

The result for every sent frame must equal amtk_logo_scan_frames on the same frames as a resident clip (with the
byte-pitch override under reference_pitch at 2-byte samples), bit for bit, and the reference's own ScanFrame (oracle/_ref,
else the C port).  After every send and after finish, the results that can be received equal the restated receive rule."""

import ctypes
import gc

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth
from test_gpu_erase_logo_stream import Frame, H, W

pytestmark = pytest.mark.gpu

# name: (w, h, imgx, imgy, seed, imgw, imgh)
SPEC = {
    "tl": (64, 64, 1, 3, 3, W, H),                   # odd x, top left
    "ov": (48, 40, 31, 27, 5, W, H),                 # overlaps tl
    "br": (64, 64, W - 65, H - 65, 7, W, H),         # odd x, the opposite corner
    "other": (64, 64, 100, 100, 9, 1920, 1080),      # another image size -> (0, -1)
    "q1": (64, 64, 37, 5, 3, W, H),                  # upper half: inside the plane under the byte-pitch row step
    "q2": (48, 40, 181, 9, 5, W, H),
    "low": (64, 64, 37, 40, 7, W, H),                # lower half: leaves the plane under that row step
    "big": (160, 128, 16, 16, 11, W, H),             # fits the evaluation plan at 1-byte samples only
}
SETS = {"one": ["tl"], "three": ["tl", None, "other"], "mixed": ["tl", None, "other", "ov", "br"]}
_DATA = {}


def logo_data(nm):
    w, h, _, _, seed, _, _ = SPEC[nm]
    if (w, h, seed) not in _DATA:
        _DATA[(w, h, seed)] = synth.make_logo(w, h, seed=seed)["data"]
    return _DATA[(w, h, seed)]


def make_logos(names, cls=None, ratio=0.35):
    out = []
    for nm in names:
        if nm is None:
            out.append(None)
            continue
        w, h, x, y, _, iw, ih = SPEC[nm]
        out.append((cls or ab.Logo).create(logo_data(nm), w, h, iw, ih, x, y).deint().create_mask(ratio))
    return out


def make_frames(N, bits, seed=1):
    """(N, W*H*3/2) packed frames, uint8 or uint16, with the tl logo fading in and out."""
    lg = synth.make_logo(64, 64, seed=3)
    f = synth.make_frames(0, N, W, H, seed=0x5EED0200 + seed, logo=lg, imgx=1, imgy=3, logo_period=20).numpy()
    if bits == 8:
        return f
    low = np.random.default_rng(seed).integers(0, 1 << (bits - 8), f.shape)
    return ((f.astype(np.int64) << (bits - 8)) | low).astype(np.uint16)


def bits_of(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def resident(ctx, fr, bits, logos, quirk):
    """amtk_logo_scan_frames over the frames as one resident clip: (N, L, 2)."""
    t = torch.from_numpy(fr.view(np.int16) if bits > 8 else fr).cuda()
    clip = ab.yv12_clip(t, W, H, fr.shape[0], True, bits)
    return ctx.scan_frames(clip, logos, pitch_elems_override=clip.pitch_y if quirk and bits > 8 else 0).cpu().numpy()


def reference(po, names, fr, bits, quirk):
    """The reference's own ScanFrame (which addresses 2-byte planes with the byte pitch), else the C port."""
    N, maxv = fr.shape[0], float((1 << bits) - 1)
    if po.ref_has_drivers() and (bits == 8 or quirk):
        rl = make_logos(names, po.RefLogo)
        return np.stack([po.ref_scan_frame_code(rl, fr[i], W, H, bits) for i in range(N)])
    out = np.zeros((N, len(names), 2), np.float32)
    out[..., 1] = -1.0
    for j, ol in enumerate(make_logos(names, po.OracleLogo)):
        if ol is None or SPEC[names[j]][5:] != (W, H):
            continue
        for i in range(N):
            Y = fr[i, :W * H].reshape(H, W)
            out[i, j] = ol.scan_frame(Y.reshape(H // 2, 2 * W), pitch=2 * W, maxv=maxv) if quirk and bits > 8 else ol.scan_frame(Y, maxv=maxv)
    return out


def receivable(S, B, finished):
    """Results that can have been received after S sends: batch k once batch k+1 was launched (S >= (k+2)B), all after finish."""
    return S if finished else max(0, S // B - 1) * B


def run(ctx, logos, descs, B, quirk=False, chunk=1 << 20):
    """Sends every frame, receiving after each send and after finish; checks the receive rule throughout."""
    s = ctx.logo_scan_stream(logos, B, quirk)
    got = []
    for k, d in enumerate(descs):
        s.send(d)
        while True:
            r = s.recv(chunk)
            got.append(r)
            if len(r) < chunk:
                break
        assert sum(len(g) for g in got) == receivable(k + 1, B, False), (k, B)
    s.finish()
    got.append(s.recv(len(descs) + 1))
    assert sum(len(g) for g in got) == len(descs)
    assert len(s.recv(5)) == 0
    counts = s.counts()
    s.close()
    return np.concatenate(got).reshape(len(descs), len(logos), 2), counts


def host_desc(fr, bits, i):
    return ab.yv12_clip(fr[i], W, H, 1, False, bits)


@pytest.mark.parametrize("bits", [8, 10, 12, 16])
@pytest.mark.parametrize("B", [1, 7, 64, 256])
def test_results_bit_exact(ctx, oracle, bits, B):
    Nmax = 3 * B + 5
    fr = make_frames(Nmax, bits, seed=B + bits)
    for set_name in ("one", "three") if B in (1, 256) else ("one", "mixed"):
        names = SETS[set_name]
        logos = make_logos(names)
        exp = resident(ctx, fr, bits, logos, False)
        ref = reference(oracle, names, fr[:B + 1], bits, False)
        assert np.array_equal(bits_of(exp[:B + 1]), bits_of(ref)), (set_name, bits, B)
        for N in sorted({1, B - 1, B, B + 1, 3 * B + 5} - {0}):
            got, _ = run(ctx, logos, [host_desc(fr, bits, i) for i in range(N)], B)
            assert np.array_equal(bits_of(got), bits_of(exp[:N])), (set_name, bits, B, N)
    assert exp[:, 0, 0].max() > 0.5 and exp[:, 0, 0].min() < 0.2          # the logo is both on and off


@pytest.mark.parametrize("bits", [10, 16])
def test_reference_pitch_quirk(ctx, oracle, bits):
    """2-byte planes addressed with the byte pitch (rows two physical rows apart), as the reference's ScanFrame does."""
    N, B = 21, 8
    fr = make_frames(N, bits, seed=bits)
    names = ["q1", None, "q2"]
    logos = make_logos(names)
    exp = resident(ctx, fr, bits, logos, True)
    assert np.array_equal(bits_of(exp), bits_of(reference(oracle, names, fr, bits, True)))
    for mem in ("pageable", "device"):
        frames = [Frame(fr[i], bits, "packed", mem) for i in range(N)]
        got, _ = run(ctx, logos, [f.desc for f in frames], B, quirk=True)
        assert np.array_equal(bits_of(got), bits_of(exp)), mem
    # without reference_pitch the rows are addressed with the element pitch: a different (plain) result
    plain, _ = run(ctx, logos, [host_desc(fr, bits, i) for i in range(N)], B, quirk=False)
    assert np.array_equal(bits_of(plain), bits_of(resident(ctx, fr, bits, logos, False)))
    # a lower-half logo leaves the plane under the quirk: refused as amtk_logo_scan_frames refuses it, nothing changes
    low = make_logos(["q1", "low"])
    t = torch.from_numpy(fr.view(np.int16)).cuda()
    clip = ab.yv12_clip(t, W, H, N, True, bits)
    with pytest.raises(ab.AmtkError, match="outside the frame"):
        ctx.scan_frames(clip, low, pitch_elems_override=clip.pitch_y)
    s = ctx.logo_scan_stream(low, B, True)
    with pytest.raises(ab.AmtkError, match="logo rectangle lies outside the frame"):
        s.send(host_desc(fr, bits, 0))
    assert s.counts() == (0, 0, 0, 0)
    f8 = make_frames(N, 8, seed=bits)                 # the format is not fixed yet: 1-byte frames are taken
    for i in range(N):
        s.send(host_desc(f8, 8, i))
    s.finish()
    got = s.recv(N)
    assert np.array_equal(bits_of(got), bits_of(resident(ctx, f8, 8, low, True)))


def test_receive_rule_small_recv(ctx):
    """recv with small max_frames: results in frame order, never more than the rule allows."""
    N, B = 50, 8
    fr = make_frames(N, 8, seed=4)
    logos = make_logos(SETS["mixed"])
    exp = resident(ctx, fr, 8, logos, False)
    for chunk in (1, 3):
        got, counts = run(ctx, logos, [host_desc(fr, 8, i) for i in range(N)], B, chunk=chunk)
        assert np.array_equal(bits_of(got), bits_of(exp)) and counts[:2] == (N, N)
    s = ctx.logo_scan_stream(logos, B)
    recvd = 0
    for k in range(N):
        s.send(host_desc(fr, 8, k))
        r = s.recv(2)
        assert np.array_equal(bits_of(r), bits_of(exp[recvd:recvd + len(r)]))
        recvd += len(r)
        assert recvd <= receivable(k + 1, B, False) and s.counts()[1] == recvd
    assert len(s.recv(0)) == 0
    s.finish()
    rest = s.recv(N)
    assert recvd + len(rest) == N and np.array_equal(bits_of(rest), bits_of(exp[recvd:]))


@pytest.mark.parametrize("bits", [8, 10])
def test_layouts_and_sources_mixed(ctx, bits):
    """Padded pitches, V-plane-first frames, pinned, pageable and device frames mixed in one stream."""
    N, B = 45, 16
    fr = make_frames(N, bits, seed=20 + bits)
    logos = make_logos(SETS["mixed"])
    exp = resident(ctx, fr, bits, logos, False)
    combos = [(lay, mem) for lay in ("packed", "vfirst") for mem in ("pageable", "pinned", "device")]
    frames = [Frame(fr[i], bits, *combos[(i * 5) % len(combos)]) for i in range(N)]
    got, _ = run(ctx, logos, [f.desc for f in frames], B)
    assert np.array_equal(bits_of(got), bits_of(exp))
    for lay, mem in combos:                            # each kind alone
        frames = [Frame(fr[i], bits, lay, mem) for i in range(N)]
        got, _ = run(ctx, logos, [f.desc for f in frames], B)
        assert np.array_equal(bits_of(got), bits_of(exp)), (lay, mem)


@pytest.mark.parametrize("bits", [8, 16])
def test_counts_and_launches(ctx, bits):
    """h2d_bytes follows the payload formula (so no whole frame moves), d2h_bytes 8*nlogos per result, launches 2 per
    evaluated logo per batch plus 1 per device frame."""
    N, B = 37, 8
    bps = 1 if bits == 8 else 2
    fr = make_frames(N, bits, seed=30)
    names = ["q1", None, "other", "q2"]
    logos = make_logos(names)
    payload = sum(SPEC[n][0] * SPEC[n][1] * bps for n in ("q1", "q2"))
    dev = [i % 3 == 0 for i in range(N)]
    frames = [Frame(fr[i], bits, "packed", "device" if dev[i] else "pageable") for i in range(N)]
    s = ctx.logo_scan_stream(logos, B, True)
    l0 = ctx.launches
    for k in range(N):
        s.send(frames[k].desc)
        S = k + 1
        launched = S // B
        sent, received, h2d, d2h = s.counts()
        assert (sent, received) == (S, 0)
        assert h2d == payload * sum(1 for i in range(launched * B) if not dev[i])
        assert d2h == 8 * len(names) * launched * B
        assert ctx.launches - l0 == 2 * 2 * launched + sum(dev[:S])
    s.finish()
    nb = (N + B - 1) // B
    assert s.counts()[2:] == (payload * (N - sum(dev)), 8 * len(names) * N)
    assert ctx.launches - l0 == 2 * 2 * nb + sum(dev)
    got = s.recv(N)
    assert np.array_equal(bits_of(got), bits_of(resident(ctx, fr, bits, logos, True)))
    # logos that give (0, -1) cost no device work
    s2 = ctx.logo_scan_stream([None, make_logos(["other"])[0]], B)
    l1 = ctx.launches
    for k in range(N):
        s2.send(frames[k].desc)
    s2.finish()
    assert ctx.launches == l1 and s2.counts()[2] == 0
    r = s2.recv(N)
    assert np.all(r[..., 0] == 0.0) and np.all(r[..., 1] == -1.0)


# Rectangles for logo_rect_gather_kernel's copy widths: (w, h, imgx, imgy).  Byte x and the row tail (row bytes mod 16) at
# 8 bits | 16 bits: 16-aligned, no tail | 16-aligned; 8-aligned, 13 | 16-aligned, 10; 4-aligned, 5 | 8-aligned, 10;
# 2-aligned, 12 | 4-aligned, 8; odd, none | 2-aligned.  All lie in the upper half (the byte-pitch row step at 16 bits).
GATHER_RECTS = [(64, 40, 16, 2), (61, 37, 88, 6), (37, 33, 164, 8), (60, 30, 194, 12), (48, 36, 1, 40)]


def cropped_logo(w, h, x, y):
    """A w x h logo (any size) cut from a 64 x 64 one: LogoData planes aY, bY, aU, bU, aV, bV."""
    d = synth.make_logo(64, 64, seed=w + h)["data"]
    Yn, Cn = 64 * 64, 32 * 32
    planes = [d[:Yn].reshape(64, 64)[:h, :w], d[Yn:2 * Yn].reshape(64, 64)[:h, :w]]
    planes += [d[2 * Yn + k * Cn:2 * Yn + (k + 1) * Cn].reshape(32, 32)[:h >> 1, :w >> 1] for k in range(4)]
    data = np.concatenate([p.ravel() for p in planes]).astype(np.float32)
    return ab.Logo.create(data, w, h, W, H, x, y).deint().create_mask(0.35)


@pytest.mark.parametrize("bits", [8, 16])
@pytest.mark.parametrize("quirk", [False, True])
@pytest.mark.parametrize("pad", [0, 8])
def test_device_frames_every_copy_width(ctx, bits, quirk, pad):
    """Device frames through logo_rect_gather_kernel with rectangles whose source alignment and row tail select each of
    its copy widths (16-, 8-, 4-, 2- and 1-byte copies and the short row tail); pad = 8 makes the luma pitch 8 mod 16,
    so the alignment also changes from row to row.  Results equal the resident amtk_logo_scan_frames call on the same
    frames in the same layout."""
    N, B = 20, 7
    bps = 1 if bits == 8 else 2
    fr = make_frames(N, bits, seed=60 + bits + pad)
    py, pc = W * bps + pad, (W // 2) * bps
    total = py * H + 2 * pc * (H // 2)
    buf = np.zeros((N, total), np.uint8)
    raw = fr.view(np.uint8).reshape(N, -1)
    for i in range(N):
        buf[i, :py * H].reshape(H, py)[:, :W * bps] = raw[i, :W * H * bps].reshape(H, W * bps)
        buf[i, py * H:] = raw[i, W * H * bps:]
    dev = torch.from_numpy(buf).cuda()
    clip = ab.ClipDesc()
    clip.base, clip.frame_stride, clip.off_u, clip.off_v = dev.data_ptr(), total, py * H, py * H + pc * (H // 2)
    clip.width, clip.height, clip.pitch_y, clip.pitch_uv = W, H, py, pc
    clip.log_uvx = clip.log_uvy = 1
    clip.bytes_per_sample, clip.bits_per_sample, clip.num_frames, clip.on_device = bps, bits, N, 1
    logos = [cropped_logo(*r) for r in GATHER_RECTS]
    exp = ctx.scan_frames(clip, logos, pitch_elems_override=py if quirk and bps == 2 else 0).cpu().numpy()
    assert not np.any((exp[..., 0] == 0.0) & (exp[..., 1] == -1.0))      # every rectangle is evaluated
    descs = []
    for i in range(N):
        d = ab.ClipDesc.from_buffer_copy(clip)
        d.base, d.num_frames = dev.data_ptr() + i * total, 1
        descs.append(d)
    launches = ctx.launches
    got, counts = run(ctx, logos, descs, B, quirk=quirk)
    assert np.array_equal(bits_of(got), bits_of(exp)), (bits, quirk, pad)
    assert counts[2] == 0 and ctx.launches - launches == N + 2 * len(logos) * ((N + B - 1) // B)


def test_rejections_leave_the_stream_unchanged(ctx):
    N, B = 12, 4
    fr = make_frames(N, 8, seed=40)
    logos = make_logos(SETS["three"])
    exp = resident(ctx, fr, 8, logos, False)
    # create
    out = ctypes.c_void_p()
    assert not ctx.L.amtk_logo_scan_stream_create(ctx.h, None, 1, 4, 0, ctypes.byref(out))
    assert "bad argument" in ctx.L.amtk_last_error().decode()
    with pytest.raises(ab.AmtkError, match="batch_size"):
        ctx.logo_scan_stream(logos, 0)
    with pytest.raises(ab.AmtkError, match="batch_size"):
        ctx.logo_scan_stream(logos, 257)
    with pytest.raises(ab.AmtkError, match="bad argument"):
        ctx.logo_scan_stream([], 4)
    raw = ab.Logo.create(logo_data("tl"), 64, 64, W, H, 1, 3)
    with pytest.raises(ab.AmtkError, match="logo has no mask: call amtk_logo_create_mask first"):
        ctx.logo_scan_stream([raw.deint()], 4)
    # a flat logo at a small mask ratio: every mask pixel lies on the two-pixel border, where no feature is taken
    flat = ab.Logo.create(np.zeros_like(logo_data("tl")), 64, 64, W, H, 1, 3).deint().create_mask(0.03)
    assert flat.info().count == 0 and flat.info().maskpixels > 0
    with pytest.raises(ab.AmtkError, match="no feature pixels"):
        ctx.logo_scan_stream([flat], 4)
    with pytest.raises(ab.AmtkError, match="no feature pixels"):           # as amtk_logo_scan_frames refuses it
        ctx.scan_frames(ab.yv12_clip(fr, W, H, N, False, 8), [flat])
    huge = ab.Logo.create(synth.make_logo(256, 128, seed=9)["data"], 256, 128, W, H, 0, 16).deint().create_mask(0.1)
    with pytest.raises(ab.AmtkError, match="too large"):
        ctx.logo_scan_stream([huge], 4)
    # frames
    s = ctx.logo_scan_stream(logos, B)
    two = ab.yv12_clip(fr[:2], W, H, 2, False, 8)
    bad = [(two, "exactly one frame")]
    sent = 0
    for i in range(N):
        if i == 5:
            wide = host_desc(fr, 8, i)
            wide.width = W - 16
            bad.append((wide, "format differs"))
            deep = host_desc(fr, 8, i)
            deep.bits_per_sample = 10
            bad.append((deep, "format differs"))
        for d, msg in bad if i in (0, 5) else []:
            before = s.counts()
            with pytest.raises(ab.AmtkError, match=msg):
                s.send(d)
            assert s.counts() == before
        s.send(host_desc(fr, 8, i))
        sent += 1
    s.finish()
    assert np.array_equal(bits_of(s.recv(N)), bits_of(exp))
    # a first frame whose sample size the evaluation plan refuses; the stream then takes 1-byte frames
    big = make_logos(["big"])
    s = ctx.logo_scan_stream(big, B)
    f16 = make_frames(2, 16, seed=41)
    with pytest.raises(ab.AmtkError, match="too large"):
        s.send(host_desc(f16, 16, 0))
    assert s.counts() == (0, 0, 0, 0)
    for i in range(N):
        s.send(host_desc(fr, 8, i))
    s.finish()
    assert np.array_equal(bits_of(s.recv(N)), bits_of(resident(ctx, fr, 8, big, False)))


def test_lifetime(ctx):
    N, B = 30, 8
    fr = make_frames(N, 8, seed=50)
    names = SETS["mixed"]
    exp = resident(ctx, fr, 8, make_logos(names), False)
    # the caller destroys its logos right after create
    logos = make_logos(names)
    s = ctx.logo_scan_stream(logos, B)
    del logos
    gc.collect()
    for i in range(N):
        s.send(host_desc(fr, 8, i))
    s.finish()
    assert np.array_equal(bits_of(s.recv(N)), bits_of(exp))
    with pytest.raises(ab.AmtkError, match=r"closed \(finished\)"):
        s.send(host_desc(fr, 8, 0))
    with pytest.raises(ab.AmtkError, match=r"closed \(finished\)"):
        s.finish()
    s.close()
    # destroy at every stage: before the first frame, mid-batch, with results pending, after draining
    logos = make_logos(names)
    frames = [Frame(fr[i], 8, "packed", "device" if i % 2 else "pinned") for i in range(N)]
    for stop in (0, 3, 2 * B + 3, N):
        s = ctx.logo_scan_stream(logos, B)
        for i in range(stop):
            s.send(frames[i].desc)
        if stop == N:
            s.finish()
            assert len(s.recv(N)) == N
        s.close()
    ctx.synchronize()
    # two streams on one context, interleaved, with different batch sizes and logos
    a = ctx.logo_scan_stream(logos, 5)
    b = ctx.logo_scan_stream(make_logos(["br"]), 3)
    ga, gb = [], []
    rev = [Frame(fr[N - 1 - i], 8, "packed", "device") for i in range(N)]
    for i in range(N):
        a.send(host_desc(fr, 8, i))
        b.send(rev[i].desc)
        ga.append(a.recv(N))
        gb.append(b.recv(N))
    a.finish()
    b.finish()
    ga.append(a.recv(N))
    gb.append(b.recv(N))
    assert np.array_equal(bits_of(np.concatenate(ga)), bits_of(exp))
    exp_b = resident(ctx, np.ascontiguousarray(fr[::-1]), 8, make_logos(["br"]), False)
    assert np.array_equal(bits_of(np.concatenate(gb)), bits_of(exp_b))
