"""amtk_scan_comb_stream: the fused step (ScanFrame scores and combing counters) fed one decoded frame at a time (DESIGN.md
section 3.1e).

With C the clip of all frames sent, the results of sent frame n must equal row n of amtk_scan_comb_frames(C, 0, N) on a
resident clip of the same frames, and the results of the logo scan stream and the comb stream fed the same frames, byte
for byte.  After every send and after finish, the results that can be received equal the restated receive rule, and the
h2d / d2h bytes and the launches are the ones include/amtk_b200.h states."""

import ctypes

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth
from test_gpu_comb_stream import LAYOUTS, MEMS, Frame, params, receivable, slot_bytes

pytestmark = pytest.mark.gpu

W, H = 256, 160


def make_frames(N, w, h, bits, seed=1):
    """(N, w*h*3/2) packed 4:2:0 frames, uint8 or uint16 at `bits`: 3:2 pulldown, so that every counter moves, with a
    64x64 logo at (1, 3) fading in and out."""
    lg = synth.make_logo(64, 64, seed=3)
    f = synth.make_frames(0, N, w, h, seed=0x5EED0600 + seed, mode="telecine", logo=lg, imgx=1, imgy=3, logo_period=20).numpy()
    if bits == 8:
        return f
    low = np.random.default_rng(seed).integers(0, 1 << (bits - 8), f.shape)
    return ((f.astype(np.int64) << (bits - 8)) | low).astype(np.uint16)


def make_logos(names, w, h):
    """tl: the logo in the frames; br: 48x40 in the opposite corner (odd x); other: made for another frame size; None."""
    out = []
    for nm in names:
        if nm is None:
            out.append(None)
            continue
        lw, lh, x, y, iw, seed = {"tl": (64, 64, 1, 3, w, 3), "br": (48, 40, w - 49, h - 41, w, 5),
                                  "other": (64, 64, 1, 3, w + 2, 7)}[nm]
        out.append(ab.Logo.create(synth.make_logo(lw, lh, seed=seed)["data"], lw, lh, iw, h, x, y).deint().create_mask(0.35))
    return out


def device_clip(fr, w, h, bits):
    t = torch.from_numpy(fr.view(np.int16) if bits > 8 else fr).cuda()
    return ab.yv12_clip(t, w, h, fr.shape[0], True, bits), t


def resident(ctx, fr, w, h, bits, logos, prm=None):
    """amtk_scan_comb_frames over the frames as one resident clip: ((N, L, 2) scores, (N, 12) counters)."""
    clip, _t = device_clip(fr, w, h, bits)
    s, c = ctx.scan_comb_frames(clip, logos, prm)
    return s.cpu().numpy(), c.cpu().numpy()


def launches_of(ctx, fr, w, h, bits, logos, prm=None):
    """The launches amtk_scan_comb_frames makes on a device clip of these frames."""
    clip, _t = device_clip(fr, w, h, bits)
    n0 = ctx.launches
    ctx.scan_comb_frames(clip, logos, prm)
    return ctx.launches - n0


def bits_of(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def run(ctx, logos, fr, w, h, bits, B, prm=None, layouts=("packed",), mems=("pageable",), chunk=1 << 20):
    """Sends every frame (layouts and memory kinds cycling), receiving after each send and after finish; checks the
    receive rule throughout.  Returns (scores, counters, counts(), host frames sent, launches)."""
    s = ctx.scan_comb_stream(logos, prm, B)
    n0 = ctx.launches
    gs, gc, nhost = [], [], 0
    for k in range(fr.shape[0]):
        f = Frame(fr[k], w, h, bits, layouts[k % len(layouts)], mems[k % len(mems)])
        nhost += f.desc.on_device == 0
        s.send(f.desc)
        while True:
            sc, cn = s.recv(chunk)
            assert len(sc) == len(cn)
            gs.append(sc); gc.append(cn)
            if len(sc) < chunk:
                break
        assert sum(len(g) for g in gs) == receivable(k + 1, B, False), (k, B)
    s.finish()
    sc, cn = s.recv(fr.shape[0] + 1)
    gs.append(sc); gc.append(cn)
    assert sum(len(g) for g in gs) == fr.shape[0]
    assert len(s.recv(5)[0]) == 0
    launches = ctx.launches - n0
    counts = s.counts()
    s.close()
    return np.concatenate(gs).reshape(-1, len(logos), 2), np.concatenate(gc).reshape(-1, 12), counts, nhost, launches


def separate_streams(ctx, logos, fr, w, h, bits, B, prm=None):
    """The logo scan stream and the comb stream fed the same frames."""
    ls, cs = ctx.logo_scan_stream(logos, B), ctx.comb_stream(prm, B)
    for k in range(fr.shape[0]):
        f = Frame(fr[k], w, h, bits, mem=MEMS[k % 3])
        ls.send(f.desc); cs.send(f.desc)
    ls.finish(); cs.finish()
    out = ls.recv(fr.shape[0]), cs.recv(fr.shape[0])
    ls.close(); cs.close()
    return out


def lengths(B):
    return sorted({n for n in (1, 2, B - 1, B, B + 1, 2 * B - 1, 2 * B, 2 * B + 1, 3 * B + 5) if n >= 1})


# ---------------------------------------------------------------------------------------------------------------------
# the result rule
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 2, 16, 64, 256])
def test_every_length_around_the_batch_size(ctx, B):
    fr = make_frames(3 * B + 5, W, H, 8, seed=B)
    logos = make_logos(["tl"], W, H)
    es, ec = resident(ctx, fr, W, H, 8, logos)
    assert (ec != 0).any(axis=0).all() and es[:, 0, 0].max() > 0.5 and es[:, 0, 0].min() < 0.2
    for N in lengths(B):
        sc, cn, (sent, received, h2d, d2h), nhost, launches = run(ctx, logos, fr[:N], W, H, 8, B, mems=("pinned",))
        assert np.array_equal(bits_of(sc), bits_of(es[:N])) and np.array_equal(cn, ec[:N]), (B, N)
        assert (sent, received, d2h) == (N, N, (48 + 8) * N)
        assert h2d == nhost * slot_bytes(W, H, 8) == N * slot_bytes(W, H, 8)
        assert launches == (N + B - 1) // B           # one fused launch per batch: the scores come from its logo items


GEOMS = [(1920, 1080, 8), (1440, 1080, 8), (1920, 1080, 10), (720, 480, 12), (720, 480, 16), (202, 94, 8), (202, 94, 10)]


@pytest.mark.parametrize("w,h,bits", GEOMS)
def test_geometries_and_sample_sizes(ctx, w, h, bits):
    """Every bit depth and size, with all sources and layouts: equal to the resident call and to the two streams."""
    B = 7
    fr = make_frames(2 * B + 3, w, h, bits, seed=w + bits)
    logos = make_logos(["tl", None, "other", "br"], w, h)
    es, ec = resident(ctx, fr, w, h, bits, logos)
    sc, cn, (sent, received, h2d, d2h), nhost, launches = run(ctx, logos, fr, w, h, bits, B, layouts=tuple(LAYOUTS), mems=MEMS)
    assert np.array_equal(bits_of(sc), bits_of(es)) and np.array_equal(cn, ec)
    ls, cs = separate_streams(ctx, logos, fr, w, h, bits, B)
    assert np.array_equal(bits_of(sc), bits_of(ls)) and np.array_equal(cn, cs)
    assert np.all(sc[:, 1] == np.array([0.0, -1.0], np.float32)) and np.all(sc[:, 2] == np.array([0.0, -1.0], np.float32))
    assert (ec != 0).any()
    assert d2h == (48 + 8 * 4) * fr.shape[0] and h2d == nhost * slot_bytes(w, h, bits)
    assert launches == 3 * (1 + 2 + 2 + 1 + 1)       # per batch: comb + two evaluated logos + two (0, -1) fills


@pytest.mark.parametrize("names,bits,per_batch", [
    (["tl"], 8, 1), (["tl"], 10, 3), (["tl"], 16, 3), (["br"], 8, 1), (["tl", "br"], 8, 5), ([None], 8, 2),
    (["other"], 8, 2), ([None, "tl"], 8, 4), (["tl", None, "other", "br"], 8, 7)])
def test_logo_sets_and_launches(ctx, names, bits, per_batch):
    """1 to 4 logos, NULL and other-size logos: exact, and per batch exactly the launches of amtk_scan_comb_frames on a
    device clip of the batch's frames."""
    B = 6
    fr = make_frames(2 * B + 1, W, H, bits, seed=len(names) + bits)
    logos = make_logos(names, W, H)
    es, ec = resident(ctx, fr, W, H, bits, logos)
    sc, cn, (sent, received, h2d, d2h), nhost, launches = run(ctx, logos, fr, W, H, bits, B, mems=MEMS)
    assert np.array_equal(bits_of(sc), bits_of(es)) and np.array_equal(cn, ec)
    assert d2h == (48 + 8 * len(names)) * fr.shape[0]
    assert launches_of(ctx, fr[:B], W, H, bits, logos) == per_batch
    assert launches == 3 * per_batch


def test_device_frames_upload_nothing(ctx):
    B = 4
    fr = make_frames(11, W, H, 8, seed=5)
    logos = make_logos(["tl"], W, H)
    sc, cn, (sent, received, h2d, d2h), nhost, _ = run(ctx, logos, fr, W, H, 8, B, layouts=("vfirst", "odd"), mems=("device",))
    es, ec = resident(ctx, fr, W, H, 8, logos)
    assert np.array_equal(bits_of(sc), bits_of(es)) and np.array_equal(cn, ec)
    assert (nhost, h2d, d2h) == (0, 0, 56 * 11)


@pytest.mark.parametrize("chunk", [1, 3])
def test_receive_rule_partial_reads(ctx, chunk):
    B = 5
    fr = make_frames(4 * B + 2, W, H, 8, seed=7)
    logos = make_logos(["tl", "br"], W, H)
    es, ec = resident(ctx, fr, W, H, 8, logos)
    sc, cn, _, _, _ = run(ctx, logos, fr, W, H, 8, B, mems=MEMS, chunk=chunk)
    assert np.array_equal(bits_of(sc), bits_of(es)) and np.array_equal(cn, ec)


# ---------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_create_refusals(ctx):
    logos = make_logos(["tl"], W, H)
    for B in (0, 257):
        with pytest.raises(ab.AmtkError, match="batch_size"):
            ctx.scan_comb_stream(logos, None, B)
    with pytest.raises(ab.AmtkError, match="thresholds must be >= 1"):
        ctx.scan_comb_stream(logos, params(th_shima_y=0), 4)
    with pytest.raises(ab.AmtkError, match="bad argument"):
        ctx.scan_comb_stream([], None, 4)
    lg = synth.make_logo(64, 64, seed=3)
    with pytest.raises(ab.AmtkError, match="no mask"):
        ctx.scan_comb_stream([ab.Logo.create(lg["data"], 64, 64, W, H, 1, 3).deint()], None, 4)
    big = synth.make_logo(256, 128, seed=9)
    with pytest.raises(ab.AmtkError, match="too large"):
        ctx.scan_comb_stream([ab.Logo.create(big["data"], 256, 128, 1920, 1080, 8, 8).deint().create_mask(0.35)], None, 4)
    L, out, p = ctx.L, ctypes.c_void_p(), ab.default_comb_params()
    arr = (ctypes.c_void_p * 1)(logos[0].h)
    for args in ((None, arr, 1, ctypes.byref(p), 4, ctypes.byref(out)), (ctx.h, None, 1, ctypes.byref(p), 4, ctypes.byref(out)),
                 (ctx.h, arr, 1, None, 4, ctypes.byref(out)), (ctx.h, arr, 1, ctypes.byref(p), 4, None)):
        assert L.amtk_scan_comb_stream_create(*args) == 0
        assert "bad argument" in L.amtk_last_error().decode()


def test_rejections_leave_the_stream_unchanged(ctx):
    B = 3
    fr = make_frames(8, W, H, 8, seed=9)
    logos = make_logos(["tl", "br"], W, H)
    es, ec = resident(ctx, fr, W, H, 8, logos)
    s = ctx.scan_comb_stream(logos, None, B)
    clip2, _t = device_clip(fr[:2], W, H, 8)
    with pytest.raises(ab.AmtkError, match="exactly one frame"):
        s.send(clip2)
    s.send(Frame(fr[0], W, H, 8).desc)
    with pytest.raises(ab.AmtkError, match="format differs"):
        s.send(Frame(make_frames(1, W + 16, H, 8)[0], W + 16, H, 8).desc)
    with pytest.raises(ab.AmtkError, match="format differs"):
        s.send(Frame(make_frames(1, W, H, 10)[0], W, H, 10).desc)
    assert s.counts() == (1, 0, 0, 0)               # nothing launched yet: host frames are uploaded at launch
    for k in range(1, 8):
        s.send(Frame(fr[k], W, H, 8, mem=MEMS[k % 3]).desc)
    s.finish()
    with pytest.raises(ab.AmtkError, match=r"closed \(finished\)"):
        s.send(Frame(fr[0], W, H, 8).desc)
    with pytest.raises(ab.AmtkError, match=r"closed \(finished\)"):
        s.finish()
    sc, cn = s.recv(100)
    assert np.array_equal(bits_of(sc), bits_of(es)) and np.array_equal(cn, ec)
    s.close()


def test_first_frame_refusals_fix_no_format(ctx):
    """A first frame the thresholds refuse at its sample size, or on which a logo's rectangle leaves the frame, fixes no
    format; a frame the stream can take then starts it, exact."""
    prm = params(th_move_y=200, th_move_c=300)
    logos = make_logos(["tl"], W, H)
    s = ctx.scan_comb_stream(logos, prm, 4)
    with pytest.raises(ab.AmtkError, match=r"th_move must be in \[1,128\]"):
        s.send(Frame(make_frames(1, W, H, 8)[0], W, H, 8).desc)
    assert s.counts() == (0, 0, 0, 0)
    fr = make_frames(9, W, H, 16, seed=2)
    for k in range(9):
        s.send(Frame(fr[k], W, H, 16, mem=MEMS[k % 3]).desc)
    s.finish()
    sc, cn = s.recv(9)
    es, ec = resident(ctx, fr, W, H, 16, logos, prm)
    assert np.array_equal(bits_of(sc), bits_of(es)) and np.array_equal(cn, ec)
    s.close()
    lg = synth.make_logo(64, 64, seed=3)
    outside = ab.Logo.create(lg["data"], 64, 64, W, H, W - 40, 3).deint().create_mask(0.35)
    s = ctx.scan_comb_stream([outside], None, 4)
    with pytest.raises(ab.AmtkError, match="logo rectangle lies outside the frame"):
        s.send(Frame(make_frames(1, W, H, 8)[0], W, H, 8).desc)
    assert s.counts() == (0, 0, 0, 0)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# lifetime and sharing the context
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stage", ["created", "mid_batch", "launched", "finished"])
def test_destroy_at_every_stage(ctx, stage):
    B = 4
    fr = make_frames(2 * B + 2, W, H, 8)
    logos = make_logos(["tl"], W, H)
    s = ctx.scan_comb_stream(logos, None, B)
    n = {"created": 0, "mid_batch": 2, "launched": 2 * B + 1, "finished": 2 * B + 2}[stage]
    for k in range(n):
        s.send(Frame(fr[k], W, H, 8, mem=MEMS[k % 3]).desc)
    if stage == "finished":
        s.finish()
        assert len(s.recv(3)[0]) == 3
    s.close()
    del logos[0]                                     # the stream held its own copies
    logos = make_logos(["tl"], W, H)
    sc, cn = run(ctx, logos, fr, W, H, 8, B)[:2]
    es, ec = resident(ctx, fr, W, H, 8, logos)
    assert np.array_equal(bits_of(sc), bits_of(es)) and np.array_equal(cn, ec)


@pytest.mark.parametrize("bits", [8, 10])
def test_interleaved_with_other_calls_and_streams(ctx, bits):
    """comb_frames, scan_frames and scan_comb_frames on the stream's context between its batches, and a comb stream and a
    logo scan stream fed at the same time, share its cached plan and the band form's watchdog record: all exact."""
    B = 5
    fr = make_frames(3 * B + 2, W, H, bits, seed=31)
    other = make_frames(12, W, H, 8, seed=32)
    logos = make_logos(["tl", "br"] if bits == 8 else ["tl"], W, H)
    es, ec = resident(ctx, fr, W, H, bits, logos)
    oc, _t = device_clip(other, W, H, 8)
    one = make_logos(["tl"], W, H)
    os_, ocn = resident(ctx, other, W, H, 8, one)
    s, cs, ls = ctx.scan_comb_stream(logos, None, B), ctx.comb_stream(None, 4), ctx.logo_scan_stream(one, 3)
    gs, gc, gcs, gls = [], [], [], []
    for k in range(fr.shape[0]):
        s.send(Frame(fr[k], W, H, bits, mem=MEMS[k % 3]).desc)
        if k < other.shape[0]:
            f = Frame(other[k], W, H, 8, mem=MEMS[(k + 1) % 3])
            cs.send(f.desc); ls.send(f.desc)
            gcs.append(cs.recv(100)); gls.append(ls.recv(100))
        if k % 3 == 1:
            assert np.array_equal(ctx.comb_frames(oc).cpu().numpy(), ocn)
            assert np.array_equal(bits_of(ctx.scan_frames(oc, one).cpu().numpy()), bits_of(os_))
        if k % 4 == 2:
            sc, cn = ctx.scan_comb_frames(oc, one)
            assert np.array_equal(cn.cpu().numpy(), ocn) and np.array_equal(bits_of(sc.cpu().numpy()), bits_of(os_))
        sc, cn = s.recv(2)
        gs.append(sc); gc.append(cn)
    s.finish(); cs.finish(); ls.finish()
    sc, cn = s.recv(100)
    gs.append(sc); gc.append(cn); gcs.append(cs.recv(100)); gls.append(ls.recv(100))
    assert np.array_equal(bits_of(np.concatenate(gs)), bits_of(es)) and np.array_equal(np.concatenate(gc), ec)
    assert np.array_equal(np.concatenate(gcs), ocn) and np.array_equal(bits_of(np.concatenate(gls)), bits_of(os_))
    assert np.array_equal(ctx.comb_frames(oc).cpu().numpy(), ocn)    # the context's watchdog checks pass after the stream
    s.close(); cs.close(); ls.close()
