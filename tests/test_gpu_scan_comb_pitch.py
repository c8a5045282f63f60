"""The fused step with LogoFrame::ScanFrame's byte-pitch row step (DESIGN.md section 3.1e): amtk_scan_comb_frames_pitch and
amtk_scan_comb_stream_create_pitch.

The reference passes the Y plane's byte pitch as the element pitch (LogoScan.hpp:1547,1561), so on 2-byte samples element
row r of the evaluation is luma row 2r.  The clip call's scores must equal amtk_logo_scan_frames with the same override and
its counters amtk_comb_frames, with the launches of both; the stream's scores must equal the logo scan stream's with
reference_pitch = 1, its counters the comb stream's, and both row n of the clip call with override C.pitch_y on a resident
clip C of the frames sent.  Scores are compared as bits, counters as integers.  Where no byte step applies (8-bit
frames, override 0 or the clip's own element pitch, reference_pitch = 0) both entry points must be the existing ones
byte for byte, launches included."""

import ctypes

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth
from amatsukaze_b200.capi import ScanCombStream, check
from test_gpu_comb_stream import LAYOUTS, MEMS, Frame, params, receivable, slot_bytes
from test_gpu_scan_comb_stream import bits_of, device_clip, lengths, make_frames

pytestmark = pytest.mark.gpu

W, H = 256, 160


def make_logos(names, w, h):
    """tl: 64x64 at (1, 3); half: 48x40 ending on row h/2 at the right edge (the last rectangle the byte-pitch step
    accepts on even heights); over: the same one row lower (refused); other: made for another frame size; None."""
    out = []
    for nm in names:
        if nm is None:
            out.append(None)
            continue
        lw, lh, x, y, iw, seed = {"tl": (64, 64, 1, 3, w, 3), "half": (48, 40, w - 48, h // 2 - 40, w, 5),
                                  "over": (48, 40, w - 48, h // 2 - 39, w, 5), "other": (64, 64, 1, 3, w + 2, 7)}[nm]
        out.append(ab.Logo.create(synth.make_logo(lw, lh, seed=seed)["data"], lw, lh, iw, h, x, y).deint().create_mask(0.35))
    return out


def _arr(logos):
    return (ctypes.c_void_p * len(logos))(*[lg.h if lg is not None else None for lg in logos])


def pitch_call(ctx, clip, logos, override, prm=None):
    """amtk_scan_comb_frames_pitch into host arrays, and the launches it made: (scores, counters, launches)."""
    n = clip.num_frames
    p = prm or ab.default_comb_params()
    sc, cn = np.empty((n, len(logos), 2), np.float32), np.empty((n, 12), np.int32)
    n0 = ctx.launches
    check(ctx.L.amtk_scan_comb_frames_pitch(ctx.h, ctypes.byref(clip), _arr(logos), len(logos), ctypes.byref(p), int(override),
                                            0, n, sc.ctypes.data_as(ctypes.c_void_p), cn.ctypes.data_as(ctypes.c_void_p), 0))
    return sc, cn, ctx.launches - n0


def fused_call(ctx, clip, logos, prm=None):
    """amtk_scan_comb_frames into host arrays: (scores, counters, launches)."""
    n0 = ctx.launches
    out = (np.empty((clip.num_frames, len(logos), 2), np.float32), np.empty((clip.num_frames, 12), np.int32))
    sc, cn = ctx.scan_comb_frames(clip, logos, prm, scores=out[0], counts=out[1])
    return sc, cn, ctx.launches - n0


def two_calls(ctx, clip, logos, override, prm=None):
    """amtk_logo_scan_frames(override) and amtk_comb_frames on the same clip: (scores, counters, launches)."""
    n0 = ctx.launches
    sc = ctx.scan_frames(clip, logos, out=np.empty((clip.num_frames, len(logos), 2), np.float32), pitch_elems_override=override)
    cn = ctx.comb_frames(clip, prm, out=np.empty((clip.num_frames, 12), np.int32))
    return sc, cn, ctx.launches - n0


def laid_out_clip(fr, w, h, bits, layout, mem):
    """The frames as one clip with the padding of a Frame layout (pad8, vfirst, odd), in pageable, pinned or device
    memory.  The Y plane comes first in every frame, so that a host clip's frames are whole from its base; V-first layouts
    put V before U."""
    bps = 1 if bits == 8 else 2
    ey, ec, vfirst = LAYOUTS[layout]
    if bps == 2:
        ey, ec = ey + (ey & 1), ec + (ec & 1)
    ry, rc, hc = w * bps, (w // 2) * bps, h // 2
    py, pc = ry + ey, rc + ec
    first_c, second_c = py * h, py * h + pc * hc
    stride = py * h + 2 * pc * hc
    buf = np.full(fr.shape[0] * stride, 0xA5, np.uint8)
    for k in range(fr.shape[0]):
        b = np.ascontiguousarray(fr[k]).view(np.uint8)
        f = buf[k * stride:(k + 1) * stride]
        ysz, csz = ry * h, rc * hc
        f[:py * h].reshape(h, py)[:, :ry] = b[:ysz].reshape(h, ry)
        u, v = b[ysz:ysz + csz].reshape(hc, rc), b[ysz + csz:].reshape(hc, rc)
        for off, plane in ((first_c, v if vfirst else u), (second_c, u if vfirst else v)):
            f[off:off + pc * hc].reshape(hc, pc)[:, :rc] = plane
    keep = buf if mem == "pageable" else torch.from_numpy(buf).pin_memory() if mem == "pinned" else torch.from_numpy(buf).cuda()
    c = ab.ClipDesc()
    c.base = keep.ctypes.data if mem == "pageable" else keep.data_ptr()
    c.frame_stride = stride
    c.off_u, c.off_v = (second_c, first_c) if vfirst else (first_c, second_c)
    c.width, c.height, c.pitch_y, c.pitch_uv = w, h, py, pc
    c.log_uvx = c.log_uvy = 1
    c.bytes_per_sample, c.bits_per_sample = bps, bits
    c.num_frames, c.on_device = fr.shape[0], 1 if mem == "device" else 0
    c.keep = keep
    return c


def host_clip(fr, w, h, bits, pinned):
    t = torch.from_numpy(fr.view(np.int16) if bits > 8 else fr)
    t = t.pin_memory() if pinned else t.clone()
    c = ab.yv12_clip(t, w, h, fr.shape[0], False, bits)
    c.keep = t
    return c


def run(ctx, logos, fr, w, h, bits, B, prm=None, reference_pitch=True, layouts=("packed",), mems=("pageable",), chunk=1 << 20):
    """Sends every frame (layouts and memory kinds cycling), receiving after each send and after finish; checks the
    receive rule after every send.  Returns (scores, counters, counts(), host frames sent, launches)."""
    s = ctx.scan_comb_stream(logos, prm, B, reference_pitch=reference_pitch)
    n0 = ctx.launches
    gs, gc, nhost = [], [], 0
    for k in range(fr.shape[0]):
        f = Frame(fr[k], w, h, bits, layouts[k % len(layouts)], mems[k % len(mems)])
        nhost += f.desc.on_device == 0
        s.send(f.desc)
        while True:
            sc, cn = s.recv(chunk)
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


def separate_streams(ctx, logos, fr, w, h, bits, B, prm=None, layouts=("packed",)):
    """The logo scan stream with reference_pitch = 1 and the comb stream fed the same frames."""
    ls, cs = ctx.logo_scan_stream(logos, B, reference_pitch=True), ctx.comb_stream(prm, B)
    for k in range(fr.shape[0]):
        f = Frame(fr[k], w, h, bits, layouts[k % len(layouts)], MEMS[k % 3])
        ls.send(f.desc); cs.send(f.desc)
    ls.finish(); cs.finish()
    out = ls.recv(fr.shape[0]), cs.recv(fr.shape[0])
    ls.close(); cs.close()
    return out


def resident_pitch(ctx, fr, w, h, bits, logos, prm=None):
    """amtk_scan_comb_frames_pitch(C, C.pitch_y) on a resident packed clip C of the frames (2-byte: the byte step)."""
    clip, _t = device_clip(fr, w, h, bits)
    return pitch_call(ctx, clip, logos, clip.pitch_y, prm)


def same(a, b):
    return np.array_equal(bits_of(a[0]), bits_of(b[0])) and np.array_equal(a[1], b[1])


# ---------------------------------------------------------------------------------------------------------------------
# the clip call
# ---------------------------------------------------------------------------------------------------------------------
CLIP_GEOMS = [(1920, 1080, 10), (1920, 1080, 12), (1920, 1080, 16), (202, 142, 10), (718, 478, 12), (3840, 2160, 10)]


@pytest.mark.parametrize("w,h,bits", CLIP_GEOMS)
def test_clip_call_is_the_two_calls(ctx, w, h, bits):
    """Device, pinned and pageable clips: scores as amtk_logo_scan_frames(pitch_y), counters as amtk_comb_frames, and
    the launches of both."""
    N = 3 if w >= 3840 else 9
    fr = make_frames(N, w, h, bits, seed=w + h + bits)
    logos = make_logos(["tl", None, "other", "half"], w, h)
    dev, _t = device_clip(fr, w, h, bits)
    for clip in (dev, host_clip(fr, w, h, bits, True), host_clip(fr, w, h, bits, False)):
        got, want = pitch_call(ctx, clip, logos, clip.pitch_y), two_calls(ctx, clip, logos, clip.pitch_y)
        assert same(got, want), (w, h, bits, clip.on_device)
        if clip.on_device:
            assert got[2] == want[2] == 1 + 2 + 1 + 1 + 2     # comb + tl + (0, -1) fills for None and other + half
    sc = got[0]
    assert np.all(sc[:, 1] == np.array([0.0, -1.0], np.float32)) and np.all(sc[:, 2] == np.array([0.0, -1.0], np.float32))
    assert (got[1] != 0).any() and np.abs(sc[:, 0, 0]).max() > 0


@pytest.mark.parametrize("layout", ["pad8", "vfirst", "odd"])
@pytest.mark.parametrize("mem", ["device", "pinned", "pageable"])
def test_clip_call_on_every_layout(ctx, layout, mem):
    bits = 10
    fr = make_frames(7, W, H, bits, seed=11)
    logos = make_logos(["tl", "half"], W, H)
    clip = laid_out_clip(fr, W, H, bits, layout, mem)
    got, want = pitch_call(ctx, clip, logos, clip.pitch_y), two_calls(ctx, clip, logos, clip.pitch_y)
    assert same(got, want)
    assert same(got, resident_pitch(ctx, fr, W, H, bits, logos))     # the byte step picks the same samples at any pitch


def test_clip_call_boundary_and_refusals(ctx):
    """imgy + h = height / 2 is accepted, one row more refused with amtk_logo_scan_frames' message; the other refusals
    are those of amtk_scan_comb_frames."""
    bits = 12
    fr = make_frames(5, W, H, bits, seed=13)
    clip, _t = device_clip(fr, W, H, bits)
    assert same(pitch_call(ctx, clip, make_logos(["half"], W, H), clip.pitch_y), two_calls(ctx, clip, make_logos(["half"], W, H), clip.pitch_y))
    over = make_logos(["over"], W, H)
    with pytest.raises(ab.AmtkError, match="logo rectangle lies outside the frame"):
        ctx.scan_frames(clip, over, pitch_elems_override=clip.pitch_y)
    with pytest.raises(ab.AmtkError, match="logo rectangle lies outside the frame"):
        pitch_call(ctx, clip, over, clip.pitch_y)
    with pytest.raises(ab.AmtkError, match="logo rectangle lies outside the frame"):
        ctx.scan_comb_frames(clip, over, pitch_elems_override=clip.pitch_y)
    assert same(pitch_call(ctx, clip, over, 0), fused_call(ctx, clip, over))          # no byte step: inside the frame
    with pytest.raises(ab.AmtkError, match="th_move must be"):
        pitch_call(ctx, clip, over, clip.pitch_y, params(th_move_y=40000))
    p = ab.default_comb_params()
    assert ctx.L.amtk_scan_comb_frames_pitch(None, ctypes.byref(clip), _arr(over), 1, ctypes.byref(p), clip.pitch_y, 0, 1,
                                             None, None, 0) == 0
    assert b"amtk_scan_comb_frames_pitch: bad argument" in ctx.L.amtk_last_error()


@pytest.mark.parametrize("mem", ["device", "pinned"])
def test_no_override_is_the_fused_call(ctx, mem):
    """8 bits with override 0 or pitch_y, and 10 bits with override 0 or pitch_y / 2: amtk_scan_comb_frames byte for
    byte, launches included (one fused launch with one logo on 8-bit device clips)."""
    for bits in (8, 10):
        fr = make_frames(13, W, H, bits, seed=17 + bits)
        clip = device_clip(fr, W, H, bits)[0] if mem == "device" else host_clip(fr, W, H, bits, True)
        for names in (["tl"], ["tl", "half", None]):
            logos = make_logos(names, W, H)
            want = fused_call(ctx, clip, logos)
            for ov in (0, -3, clip.pitch_y // clip.bytes_per_sample):
                got = pitch_call(ctx, clip, logos, ov)
                assert same(got, want) and got[2] == want[2], (bits, names, ov)
            if mem == "device" and bits == 8 and len(names) == 1:
                assert want[2] == 1


def test_other_override_at_8_bits_runs_the_two_calls(ctx):
    fr = make_frames(9, W, H, 8, seed=19)
    clip, _t = device_clip(fr, W, H, 8)
    logos = make_logos(["tl"], W, H)
    got, want = pitch_call(ctx, clip, logos, 2 * clip.pitch_y), two_calls(ctx, clip, logos, 2 * clip.pitch_y)
    assert same(got, want) and got[2] == want[2]


def test_odd_height_last_half_row(ctx):
    """On an odd height the byte step's last element row starts on the frame's last luma row: a rectangle ending there is
    accepted and reads that row, as the logo scan stream reads it."""
    w, h, bits = 256, 161, 10
    fr = make_frames(6, w, h, bits, seed=23)
    lg = ab.Logo.create(synth.make_logo(48, 40, seed=5)["data"], 48, 40, w, h, w - 48, (h + 1) // 2 - 40).deint().create_mask(0.35)
    clip, _t = device_clip(fr, w, h, bits)
    want = ctx.scan_frames(clip, [lg], out=np.empty((6, 1, 2), np.float32), pitch_elems_override=clip.pitch_y)
    ls = ctx.logo_scan_stream([lg], 4, reference_pitch=True)
    for k in range(6):
        ls.send(Frame(fr[k], w, h, bits).desc)
    ls.finish()
    assert np.array_equal(bits_of(ls.recv(6)), bits_of(want))
    ls.close()


# ---------------------------------------------------------------------------------------------------------------------
# the stream
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 16, 256])
def test_stream_every_length_around_the_batch_size(ctx, B):
    bits = 10
    fr = make_frames(3 * B + 5, W, H, bits, seed=B)
    logos = make_logos(["tl"], W, H)
    es, ec, _ = resident_pitch(ctx, fr, W, H, bits, logos)
    assert (ec != 0).any(axis=0).all() and np.abs(es[:, 0, 0]).max() > 0
    for N in lengths(B):
        sc, cn, (sent, received, h2d, d2h), nhost, launches = run(ctx, logos, fr[:N], W, H, bits, B, mems=("pinned",))
        assert np.array_equal(bits_of(sc), bits_of(es[:N])) and np.array_equal(cn, ec[:N]), (B, N)
        assert (sent, received, d2h) == (N, N, (48 + 8) * N)
        assert h2d == nhost * slot_bytes(W, H, bits) == N * slot_bytes(W, H, bits)
        assert launches == 3 * ((N + B - 1) // B)       # per batch: comb + the logo's two evaluation launches


STREAM_GEOMS = [(1920, 1080, 10), (1920, 1080, 12), (1920, 1080, 16), (202, 142, 10), (718, 478, 12), (3840, 2160, 10)]


@pytest.mark.parametrize("w,h,bits", STREAM_GEOMS)
def test_stream_geometries_sources_and_layouts(ctx, w, h, bits):
    """Every depth and size, all sources and layouts: equal to the resident clip call and to the two streams."""
    B = 4 if w >= 3840 else 7
    N = B + 3 if w >= 3840 else 2 * B + 3
    fr = make_frames(N, w, h, bits, seed=w + bits)
    logos = make_logos(["tl", None, "other", "half"], w, h)
    es, ec, per = resident_pitch(ctx, fr[:B], w, h, bits, logos)
    assert per == 1 + 2 + 1 + 1 + 2
    es, ec, _ = resident_pitch(ctx, fr, w, h, bits, logos)
    sc, cn, (sent, received, h2d, d2h), nhost, launches = run(ctx, logos, fr, w, h, bits, B, layouts=tuple(LAYOUTS), mems=MEMS)
    assert np.array_equal(bits_of(sc), bits_of(es)) and np.array_equal(cn, ec)
    ls, cs = separate_streams(ctx, logos, fr, w, h, bits, B, layouts=tuple(LAYOUTS))
    assert np.array_equal(bits_of(sc), bits_of(ls)) and np.array_equal(cn, cs)
    assert d2h == (48 + 8 * 4) * N and h2d == nhost * slot_bytes(w, h, bits)
    assert launches == ((N + B - 1) // B) * per


@pytest.mark.parametrize("names,per_batch", [
    (["tl"], 3), (["half"], 3), (["tl", "half"], 5), ([None], 2), (["other"], 2), ([None, "tl"], 4),
    (["tl", None, "other", "half"], 7)])
@pytest.mark.parametrize("bits", [10, 16])
def test_stream_logo_sets_and_launches(ctx, names, per_batch, bits):
    """1 to 4 logos, NULL and other-size logos: exact, and per batch exactly the launches of the clip call on a device
    clip of the batch's frames."""
    B = 6
    fr = make_frames(2 * B + 1, W, H, bits, seed=len(names) + bits)
    logos = make_logos(names, W, H)
    es, ec, _ = resident_pitch(ctx, fr, W, H, bits, logos)
    sc, cn, (sent, received, h2d, d2h), nhost, launches = run(ctx, logos, fr, W, H, bits, B, mems=MEMS)
    assert np.array_equal(bits_of(sc), bits_of(es)) and np.array_equal(cn, ec)
    assert d2h == (48 + 8 * len(names)) * fr.shape[0]
    assert resident_pitch(ctx, fr[:B], W, H, bits, logos)[2] == per_batch
    assert launches == 3 * per_batch


def test_stream_device_frames_upload_nothing(ctx):
    B = 4
    fr = make_frames(11, W, H, 12, seed=5)
    logos = make_logos(["tl", "half"], W, H)
    sc, cn, (sent, received, h2d, d2h), nhost, _ = run(ctx, logos, fr, W, H, 12, B, layouts=("vfirst", "odd", "pad8"), mems=("device",))
    es, ec, _ = resident_pitch(ctx, fr, W, H, 12, logos)
    assert np.array_equal(bits_of(sc), bits_of(es)) and np.array_equal(cn, ec)
    assert (nhost, h2d, d2h) == (0, 0, 64 * 11)


@pytest.mark.parametrize("chunk", [1, 3])
def test_stream_partial_reads(ctx, chunk):
    B = 5
    fr = make_frames(4 * B + 2, W, H, 10, seed=7)
    logos = make_logos(["tl", "half"], W, H)
    es, ec, _ = resident_pitch(ctx, fr, W, H, 10, logos)
    sc, cn, _, _, _ = run(ctx, logos, fr, W, H, 10, B, mems=MEMS, chunk=chunk)
    assert np.array_equal(bits_of(sc), bits_of(es)) and np.array_equal(cn, ec)


@pytest.mark.parametrize("B", [1, 16])
def test_stream_at_8_bits_is_the_fused_stream(ctx, B):
    """8-bit frames: reference_pitch = 1 is amtk_scan_comb_stream_create in results, bytes and launches (one fused launch
    per batch with one logo)."""
    fr = make_frames(2 * B + 3, W, H, 8, seed=29)
    for names in (["tl"], ["tl", None, "half"]):
        logos = make_logos(names, W, H)
        a = run(ctx, logos, fr, W, H, 8, B, reference_pitch=True, mems=MEMS)
        b = run(ctx, logos, fr, W, H, 8, B, reference_pitch=False, mems=MEMS)
        assert same(a, b) and a[2:] == b[2:], names
        if len(names) == 1:
            assert a[4] == (fr.shape[0] + B - 1) // B


def test_reference_pitch_0_is_the_stream_create(ctx):
    """reference_pitch = 0 through amtk_scan_comb_stream_create_pitch: amtk_scan_comb_stream_create in results, bytes and
    launches, also on 2-byte frames (no byte step there)."""
    B, bits = 5, 10
    fr = make_frames(2 * B + 2, W, H, bits, seed=31)
    logos = make_logos(["tl", "half"], W, H)
    p = ab.default_comb_params()
    out = ctypes.c_void_p()
    check(ctx.L.amtk_scan_comb_stream_create_pitch(ctx.h, _arr(logos), len(logos), ctypes.byref(p), B, 0, ctypes.byref(out)))
    s = ScanCombStream(ctx, out, len(logos))
    n0 = ctx.launches
    for k in range(fr.shape[0]):
        s.send(Frame(fr[k], W, H, bits, mem=MEMS[k % 3]).desc)
    s.finish()
    got = s.recv(100)
    launches, counts = ctx.launches - n0, s.counts()
    s.close()
    want = run(ctx, logos, fr, W, H, bits, B, reference_pitch=False, mems=MEMS)
    assert same(got, want) and (counts, launches) == (want[2], want[4])
    clip, _t = device_clip(fr, W, H, bits)
    assert same(got, fused_call(ctx, clip, logos))


# ---------------------------------------------------------------------------------------------------------------------
# refusals and lifetime
# ---------------------------------------------------------------------------------------------------------------------
def test_stream_create_refusals(ctx):
    logos = make_logos(["tl"], W, H)
    for B in (0, 257):
        with pytest.raises(ab.AmtkError, match="batch_size"):
            ctx.scan_comb_stream(logos, None, B, reference_pitch=True)
    with pytest.raises(ab.AmtkError, match="thresholds must be >= 1"):
        ctx.scan_comb_stream(logos, params(th_shima_y=0), 4, reference_pitch=True)
    lg = synth.make_logo(64, 64, seed=3)
    with pytest.raises(ab.AmtkError, match="no mask"):
        ctx.scan_comb_stream([ab.Logo.create(lg["data"], 64, 64, W, H, 1, 3).deint()], None, 4, reference_pitch=True)
    p, out = ab.default_comb_params(), ctypes.c_void_p()
    assert ctx.L.amtk_scan_comb_stream_create_pitch(None, _arr(logos), 1, ctypes.byref(p), 4, 1, ctypes.byref(out)) == 0
    assert b"amtk_scan_comb_stream_create_pitch: bad argument" in ctx.L.amtk_last_error()


def test_stream_boundary_refusal_leaves_the_stream_unchanged(ctx):
    """A rectangle that, as addressed, leaves the Y plane is refused at the send, with the logo scan stream's message,
    whatever the frame's layout; the stream stays as it was and then takes frames it can evaluate.  8-bit frames have no
    byte step, so the same logo is evaluated there."""
    bits = 10
    fr = make_frames(9, W, H, bits, seed=37)
    over = make_logos(["over"], W, H)
    ls = ctx.logo_scan_stream(over, 4, reference_pitch=True)
    s = ctx.scan_comb_stream(over, None, 4, reference_pitch=True)
    for layout in LAYOUTS:
        f = Frame(fr[0], W, H, bits, layout)
        for st in (ls, s):
            with pytest.raises(ab.AmtkError, match="logo rectangle lies outside the frame"):
                st.send(f.desc)
    assert s.counts() == (0, 0, 0, 0)
    ls.close(); s.close()
    logos = make_logos(["tl", "half"], W, H)
    s = ctx.scan_comb_stream(logos, None, 4, reference_pitch=True)
    s.send(Frame(fr[0], W, H, bits).desc)
    clip2, _t = device_clip(fr[:2], W, H, bits)
    with pytest.raises(ab.AmtkError, match="exactly one frame"):
        s.send(clip2)
    with pytest.raises(ab.AmtkError, match="format differs"):
        s.send(Frame(make_frames(1, W, H, 12)[0], W, H, 12).desc)
    with pytest.raises(ab.AmtkError, match="format differs"):
        s.send(Frame(make_frames(1, W, H, 8)[0], W, H, 8).desc)
    assert s.counts() == (1, 0, 0, 0)
    for k in range(1, 9):
        s.send(Frame(fr[k], W, H, bits, list(LAYOUTS)[k % 4], MEMS[k % 3]).desc)
    s.finish()
    with pytest.raises(ab.AmtkError, match=r"closed \(finished\)"):
        s.send(Frame(fr[0], W, H, bits).desc)
    with pytest.raises(ab.AmtkError, match=r"closed \(finished\)"):
        s.finish()
    got = s.recv(100)
    s.close()
    assert same(got, resident_pitch(ctx, fr, W, H, bits, logos))
    fr8 = make_frames(5, W, H, 8, seed=38)
    got = run(ctx, over, fr8, W, H, 8, 2)
    assert same(got, fused_call(ctx, device_clip(fr8, W, H, 8)[0], over))


@pytest.mark.parametrize("stage", ["created", "mid_batch", "launched", "finished"])
def test_stream_destroy_at_every_stage(ctx, stage):
    B, bits = 4, 10
    fr = make_frames(2 * B + 2, W, H, bits)
    logos = make_logos(["tl", "half"], W, H)
    s = ctx.scan_comb_stream(logos, None, B, reference_pitch=True)
    n = {"created": 0, "mid_batch": 2, "launched": 2 * B + 1, "finished": 2 * B + 2}[stage]
    for k in range(n):
        s.send(Frame(fr[k], W, H, bits, mem=MEMS[k % 3]).desc)
    if stage == "finished":
        s.finish()
        assert len(s.recv(3)[0]) == 3
    s.close()
    del logos[:]                                     # the stream held its own copies
    logos = make_logos(["tl", "half"], W, H)
    got = run(ctx, logos, fr, W, H, bits, B)
    assert same(got, resident_pitch(ctx, fr, W, H, bits, logos))


def test_stream_interleaved_with_other_calls_and_streams(ctx):
    """comb_frames, scan_frames (with and without the override), the clip calls, a comb stream and a logo scan stream on
    the stream's context between its batches: all exact."""
    B, bits = 5, 10
    fr = make_frames(3 * B + 2, W, H, bits, seed=41)
    other = make_frames(12, W, H, 8, seed=42)
    logos = make_logos(["tl", "half"], W, H)
    es, ec, _ = resident_pitch(ctx, fr, W, H, bits, logos)
    oc, _t = device_clip(other, W, H, 8)
    fc, _t2 = device_clip(fr, W, H, bits)
    one = make_logos(["tl"], W, H)
    os_, ocn, _ = fused_call(ctx, oc, one)
    qs = ctx.scan_frames(fc, logos, out=np.empty((fr.shape[0], 2, 2), np.float32), pitch_elems_override=fc.pitch_y)
    s = ctx.scan_comb_stream(logos, None, B, reference_pitch=True)
    cs, ls = ctx.comb_stream(None, 4), ctx.logo_scan_stream(one, 3)
    gs, gc, gcs, gls = [], [], [], []
    for k in range(fr.shape[0]):
        s.send(Frame(fr[k], W, H, bits, mem=MEMS[k % 3]).desc)
        if k < other.shape[0]:
            f = Frame(other[k], W, H, 8, mem=MEMS[(k + 1) % 3])
            cs.send(f.desc); ls.send(f.desc)
            gcs.append(cs.recv(100)); gls.append(ls.recv(100))
        if k % 3 == 1:
            assert np.array_equal(ctx.comb_frames(oc).cpu().numpy(), ocn)
            assert np.array_equal(bits_of(ctx.scan_frames(fc, logos, pitch_elems_override=fc.pitch_y).cpu().numpy()), bits_of(qs))
        if k % 4 == 2:
            assert same(fused_call(ctx, oc, one), (os_, ocn))
            assert same(pitch_call(ctx, fc, logos, fc.pitch_y), (es, ec))
        sc, cn = s.recv(2)
        gs.append(sc); gc.append(cn)
    s.finish(); cs.finish(); ls.finish()
    sc, cn = s.recv(100)
    gs.append(sc); gc.append(cn); gcs.append(cs.recv(100)); gls.append(ls.recv(100))
    assert np.array_equal(bits_of(np.concatenate(gs)), bits_of(es)) and np.array_equal(np.concatenate(gc), ec)
    assert np.array_equal(bits_of(qs), bits_of(es))
    assert np.array_equal(np.concatenate(gcs), ocn) and np.array_equal(bits_of(np.concatenate(gls)), bits_of(os_))
    s.close(); cs.close(); ls.close()
