"""amtk_erase_logo_clip: AMTEraseLogo(AMTAnalyzeLogo(src, logo), logo, logof, maxfade) over a whole clip in one call
(DESIGN.md section 3.3.4).

Every output and its fades must equal amtk_erase_logo_stream's for the same frames, the host composition
(amtk_logo_analyze_frames records, amtk_calc_fade2_index + amtk_calc_fade2_records, amtk_erase_logo_frames), and the
composition built from the reference's own code (oracle/_ref, else the C port) -- byte for byte and bit for bit."""

import ctypes as C

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200.capi import c_float_p
from test_erase_logo_stream_rule import fade2_index, fade_codes, record_set
from test_gpu_erase_logo_stream import LOGO, LOGOF, H, Reference, W, make_clip, run_stream, write_logof

pytestmark = pytest.mark.gpu

SENT = 0x5A
IMGX, IMGY = 100, 42


def logo_at(imgx=IMGX, imgy=IMGY):
    return ab.Logo.create(LOGO["data"], 64, 64, W, H, imgx, imgy)


def device_clip(frames, bits):
    t = torch.from_numpy(frames.copy()).cuda()
    return t, ab.yv12_clip(t, W, H, frames.shape[0], True, bits)


def clip_erase(ctx, frames, bits, logo, fr, maxfade, frame0=0, nframes=None, out_of_place=False):
    """(outputs, fades) of one call on a device copy of frames; out of place into a packed dst."""
    N = frames.shape[0]
    n = N - frame0 if nframes is None else nframes
    t, src = device_clip(frames, bits)
    if out_of_place:
        d = torch.zeros((n,) + frames.shape[1:], dtype=t.dtype, device="cuda")
        fades = ctx.erase_logo_clip(src, logo, ab.yv12_clip(d, W, H, n, True, bits), fr, maxfade, frame0, n)
        torch.cuda.synchronize()
        assert np.array_equal(t.cpu().numpy(), frames), "an out-of-place call changed src"
        return d.cpu().numpy(), fades
    fades = ctx.erase_logo_clip(src, logo, None, fr, maxfade, frame0, n)
    torch.cuda.synchronize()
    out = t.cpu().numpy()
    assert np.array_equal(out[:frame0], frames[:frame0]) and np.array_equal(out[frame0 + n:], frames[frame0 + n:])
    return out[frame0:frame0 + n], fades


def host_composition(ctx, frames, bits, logo, fr, maxfade):
    """The mirror's previous composition from the C ABI: records, CalcFade on the host, a one-frame erase per output."""
    N = frames.shape[0]
    dl, ft, fb = logo.deint().create_mask(0.35), logo.field(0).create_mask(0.35), logo.field(1).create_mask(0.35)
    rec = ctx.analyze_frames(ab.yv12_clip(frames, W, H, N, False, bits), dl, ft, fb)
    rec = np.ascontiguousarray(rec.cpu().numpy() if isinstance(rec, torch.Tensor) else rec, np.float32).reshape(N, 33)
    L = ab.lib()
    codes = fade_codes(N, fr, maxfade)
    fades = np.zeros((N, 2), np.float32)
    for n in range(N):
        if codes[n] < 2:
            fades[n] = codes[n]
            continue
        rec9 = np.ascontiguousarray(np.stack([rec[L.amtk_calc_fade2_index(N, N, n, i)] for i in range(-4, 5)]), np.float32)
        t, b = C.c_float(), C.c_float()
        L.amtk_calc_fade2_records(rec9.ctypes.data_as(c_float_p), C.byref(t), C.byref(b))
        fades[n] = (t.value, b.value)
    out = frames.copy()
    for n in range(N):
        one = out[n:n + 1]
        ctx.erase_logo(ab.yv12_clip(one, W, H, 1, False, bits), logo, fades[n:n + 1])
    return out, fades


def frame_result_of(kind, N, tmp_path):
    """(frame_result or None, logoframe path or None)"""
    if kind == "none":
        return None, None
    if kind in ("uniform0", "uniform2"):
        return np.full(N, 0 if kind == "uniform0" else 2, np.uint8), None
    path = write_logof(tmp_path / "logof.txt", LOGOF[kind])
    from test_gpu_erase_logo_stream import read_logoframe
    return read_logoframe(path, N).astype(np.uint8), path


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a, np.float32).view(np.uint32), np.ascontiguousarray(b, np.float32).view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------
# parity with the stream, the host composition and the reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [8, 10, 12, 16])
@pytest.mark.parametrize("kind,maxfade", [("none", 16), ("close", 16), ("middle", 5), ("start", 0), ("uniform0", 16),
                                          ("uniform2", 7)])
def test_parity_with_stream_host_and_reference(ctx, oracle, tmp_path, bits, kind, maxfade):
    N = 100
    frames = make_clip(N, bits, IMGX, IMGY, seed=bits)
    fr, path = frame_result_of(kind, N, tmp_path)
    logo = logo_at()
    got, fades = clip_erase(ctx, frames, bits, logo, fr, maxfade)
    oop, fades2 = clip_erase(ctx, frames, bits, logo, fr, maxfade, out_of_place=True)
    assert np.array_equal(got, oop) and same_bits(fades, fades2)
    s_out, s_fades, s, _ = run_stream(ctx, logo, frames, bits, fr, maxfade, 16, src=("device",), check_rule=False)
    s.close()
    assert same_bits(fades, s_fades), "fades differ from the stream's"
    assert np.array_equal(got, s_out), "pixels differ from the stream's"
    h_out, h_fades = host_composition(ctx, frames, bits, logo, fr, maxfade)
    assert same_bits(fades, h_fades), "fades differ from the host composition's"
    assert np.array_equal(got, h_out), "pixels differ from the host composition's"
    if kind in ("none", "close", "middle", "start"):
        ref = Reference(oracle, bits, IMGX, IMGY)
        rf, _ = ref.fades(ref.records(frames), N, path, maxfade)
        assert same_bits(fades, rf), "fades differ from the reference's (%s)" % ref.kind
        assert np.array_equal(got, ref.pixels(frames, rf)), "pixels differ from the reference composition (%s)" % ref.kind


@pytest.mark.parametrize("N", list(range(1, 21)))
def test_short_clips_every_length(ctx, N):
    """Lengths where the (nsrc + i) quirk's negative offsets land in frames 4..7, and clips shorter than one block."""
    frames = make_clip(N, 8, IMGX, IMGY, seed=N)
    logo = logo_at()
    got, fades = clip_erase(ctx, frames, 8, logo, None, 16)
    h_out, h_fades = host_composition(ctx, frames, 8, logo, None, 16)
    assert same_bits(fades, h_fades) and np.array_equal(got, h_out)


def test_long_clip_with_transitions(ctx, tmp_path):
    N = 700
    frames = make_clip(N, 8, IMGX, IMGY, seed=11)
    fr = np.zeros(N, np.uint8)
    fr[100:300] = 2; fr[95:100] = 1; fr[300:305] = 1; fr[500:650] = 2
    logo = logo_at()
    got, fades = clip_erase(ctx, frames, 8, logo, fr, 16, out_of_place=True)
    s_out, s_fades, s, _ = run_stream(ctx, logo, frames, 8, fr, 16, 64, src=("device",), check_rule=False)
    s.close()
    assert same_bits(fades, s_fades) and np.array_equal(got, s_out)


@pytest.mark.parametrize("frame0,nframes", [(1, 1), (5, 10), (37, 20), (80, 20), (99, 1), (0, 100)])
@pytest.mark.parametrize("oop", [False, True])
def test_ranges_read_records_outside_the_range(ctx, frame0, nframes, oop):
    N = 100
    frames = make_clip(N, 8, IMGX, IMGY, seed=5)
    logo = logo_at()
    fr = np.zeros(N, np.uint8); fr[30:60] = 2; fr[28:30] = 1
    got, fades = clip_erase(ctx, frames, 8, logo, fr, 16, frame0, nframes, out_of_place=oop)
    h_out, h_fades = host_composition(ctx, frames, 8, logo, fr, 16)
    assert same_bits(fades, h_fades[frame0:frame0 + nframes])
    assert np.array_equal(got, h_out[frame0:frame0 + nframes])


# ---------------------------------------------------------------------------------------------------------------------
# placement
# ---------------------------------------------------------------------------------------------------------------------
def staged_payload(rx, ry, rw, rh, bps, chroma):
    """Bytes the ROI staging of a host clip moves per frame (for_each_roi_window, 4:2:0)."""
    A = 32
    xb0 = (rx * bps) // A * A
    xb1 = min(W * bps, -(-((rx + rw) * bps) // A) * A)
    dy, y1 = ry & ~1, min(H, (ry + rh + 1) & ~1)
    span, rows = xb1 - xb0, y1 - dy
    spanc = min((W // 2) * bps - (xb0 >> 1), span >> 1)
    return span * rows + (2 * spanc * (rows >> 1) if chroma else 0)


@pytest.mark.parametrize("bits", [8, 16])
@pytest.mark.parametrize("frame0,nframes,kind", [(0, 60, "none"), (20, 10, "none"), (20, 10, "mixed"), (0, 60, "uniform2")])
def test_in_place_on_a_host_clip_moves_only_rectangles(ctx, bits, frame0, nframes, kind):
    N = 60
    frames = make_clip(N, bits, IMGX, IMGY, seed=2)
    fr = None
    if kind == "mixed":
        fr = np.zeros(N, np.uint8); fr[25:40] = 2
    elif kind == "uniform2":
        fr = np.full(N, 2, np.uint8)
    logo = logo_at()
    host = frames.copy()
    fades = ctx.erase_logo_clip(ab.yv12_clip(host, W, H, N, False, bits), logo, None, fr, 16, frame0, nframes)
    h2d = ctx.last_h2d_bytes
    dev, dfades = clip_erase(ctx, frames, bits, logo, fr, 16, frame0, nframes)
    assert same_bits(fades, dfades)
    assert np.array_equal(host[frame0:frame0 + nframes], dev)
    assert np.array_equal(host[:frame0], frames[:frame0]) and np.array_equal(host[frame0 + nframes:], frames[frame0 + nframes:])
    bps = 1 if bits == 8 else 2
    codes = fade_codes(N, fr, 16)
    need = sorted({fade2_index(N, n, i) for n in range(frame0, frame0 + nframes) if codes[n] == 2 for i in range(-4, 5)})
    span = need[-1] - need[0] + 1 if need else 0
    # the analysis stages the luma rectangle of the frames the records span, the erase all three of the outputs
    assert h2d == span * staged_payload(IMGX, IMGY, 64, 64, bps, False) + nframes * staged_payload(IMGX, IMGY, 64, 64, bps, True)
    assert h2d < nframes * W * H * bps


class DstLayout:
    """A device dst of n frames in a padded, V-first or odd-pitch layout, sentinel-filled."""

    def __init__(self, kind, n, bits):
        bps = 1 if bits == 8 else 2
        self.bps, self.n = bps, n
        if kind == "padded":
            py, pc = W * bps + 64, (W // 2) * bps + 32
            offu = py * H + 32; offv = offu + pc * (H // 2) + 32; total = offv + pc * (H // 2) + 96
        elif kind == "vfirst":
            py, pc = W * bps + 16, (W // 2) * bps + 16
            offv = py * H; offu = offv + pc * (H // 2); total = offu + pc * (H // 2) + 16
        else:                                                  # odd pitches and offsets: no 16-byte loads
            py, pc = W * bps + (2 * bps + 1 if bps == 1 else 6), (W // 2) * bps + (3 if bps == 1 else 2)
            offu = py * H + 5 * bps; offv = offu + pc * (H // 2) + 3 * bps; total = offv + pc * (H // 2) + 7 * bps
        self.py, self.pc, self.offu, self.offv, self.total = py, pc, offu, offv, total
        self.buf = torch.full((n * total + 16,), SENT, dtype=torch.uint8, device="cuda")
        d = ab.ClipDesc()
        base = self.buf.data_ptr() + (1 if kind == "odd" and bps == 1 else 0)
        d.base, d.frame_stride, d.off_u, d.off_v = base, total, offu, offv
        d.width, d.height, d.pitch_y, d.pitch_uv = W, H, py, pc
        d.log_uvx = d.log_uvy = 1
        d.bytes_per_sample, d.bits_per_sample, d.num_frames, d.on_device = bps, bits, n, 1
        self.desc, self.shift = d, base - self.buf.data_ptr()

    def frames_and_padding(self):
        raw = self.buf.cpu().numpy()
        bps, mask = self.bps, np.ones(raw.size, bool)
        out = []
        for k in range(self.n):
            rows = []
            for off, pitch, rb, r in ((0, self.py, W * bps, H), (self.offu, self.pc, (W // 2) * bps, H // 2),
                                      (self.offv, self.pc, (W // 2) * bps, H // 2)):
                o = self.shift + k * self.total + off
                blk = raw[o:o + pitch * r].reshape(r, pitch)
                rows.append(blk[:, :rb].reshape(-1))
                mask[o:o + pitch * r].reshape(r, pitch)[:, :rb] = False
            out.append(np.concatenate(rows).view(np.uint8 if bps == 1 else np.uint16))
        return np.stack(out), raw[mask]


@pytest.mark.parametrize("bits", [8, 10, 16])
@pytest.mark.parametrize("layout", ["padded", "vfirst", "odd"])
def test_out_of_place_layouts(ctx, bits, layout):
    N, frame0, n = 40, 6, 30
    frames = make_clip(N, bits, IMGX, IMGY, seed=4)
    logo = logo_at()
    t, src = device_clip(frames, bits)
    dst = DstLayout(layout, n, bits)
    fades = ctx.erase_logo_clip(src, logo, dst.desc, None, 16, frame0, n)
    got, pad = dst.frames_and_padding()
    assert (pad == SENT).all(), "row padding or bytes between planes were written"
    assert np.array_equal(t.cpu().numpy(), frames), "src changed"
    exp, efades = clip_erase(ctx, frames, bits, logo, None, 16, frame0, n)
    assert same_bits(fades, efades)
    assert np.array_equal(got, exp)
    from test_gpu_erase import logo_rect_mask
    outside = ~logo_rect_mask(W, H, 64, 64, IMGX, IMGY)
    assert np.array_equal(got[:, outside], frames[frame0:frame0 + n][:, outside]), "a sample outside the rectangles changed"


# ---------------------------------------------------------------------------------------------------------------------
# launch counts
# ---------------------------------------------------------------------------------------------------------------------
def launches_of(ctx, fn):
    ctx.synchronize()
    l0 = ctx.launches
    fn()
    return ctx.launches - l0


@pytest.mark.parametrize("oop", [False, True])
def test_launch_count_does_not_depend_on_nframes(ctx, oop):
    N = 200
    frames = make_clip(N, 8, IMGX, IMGY, seed=9)
    logo = logo_at()
    counts = set()
    for frame0, n in ((0, 1), (50, 10), (0, 100), (0, N)):
        t, src = device_clip(frames, 8)
        d = torch.zeros((n,) + frames.shape[1:], dtype=t.dtype, device="cuda") if oop else None
        dst = ab.yv12_clip(d, W, H, n, True, 8) if oop else None
        counts.add(launches_of(ctx, lambda: ctx.erase_logo_clip(src, logo, dst, None, 16, frame0, n)))
    assert counts == {8}, counts           # one analysis pass (3 evaluations x 2 kernels), the fade kernel, one erase kernel


@pytest.mark.parametrize("value", [0, 1, 2])
def test_uniform_frame_result_launches_no_evaluation(ctx, value):
    N = 50
    frames = make_clip(N, 8, IMGX, IMGY, seed=9)
    t, src = device_clip(frames, 8)
    fr = np.full(N, value, np.uint8)
    assert launches_of(ctx, lambda: ctx.erase_logo_clip(src, logo_at(), None, fr, 16)) == 2


def test_scattered_need_is_one_analysis_pass(ctx):
    """Transitions far apart: the needed frames form several runs, analysed by one pass over a frame list."""
    N = 400
    frames = make_clip(N, 8, IMGX, IMGY, seed=12)
    fr = np.zeros(N, np.uint8)
    fr[50:120] = 2; fr[200:260] = 2; fr[330:390] = 2
    assert len(record_set(N, fr, 4)) < N // 2
    t, src = device_clip(frames, 8)
    logo = logo_at()
    fades = None

    def run():
        nonlocal fades
        fades = ctx.erase_logo_clip(src, logo, None, fr, 4)
    assert launches_of(ctx, run) == 8
    _, h_fades = host_composition(ctx, frames, 8, logo, fr, 4)
    assert same_bits(fades, h_fades)


# ---------------------------------------------------------------------------------------------------------------------
# refusals: each with its reason, nothing written
# ---------------------------------------------------------------------------------------------------------------------
def test_refusals(ctx):
    N = 20
    frames = make_clip(N, 8, IMGX, IMGY, seed=1)
    t, src = device_clip(frames, 8)
    logo = logo_at()
    good = torch.full((N,) + frames.shape[1:], SENT, dtype=t.dtype, device="cuda")
    gdst = ab.yv12_clip(good, W, H, N, True, 8)

    def refused(match, **kw):
        a = dict(src=src, logo=logo, dst=None, frame_result=None, max_fade_length=16, frame0=0, nframes=N)
        a.update(kw)
        with pytest.raises(ab.AmtkError, match=match):
            ctx.erase_logo_clip(a["src"], a["logo"], a["dst"], a["frame_result"], a["max_fade_length"], a["frame0"],
                                a["nframes"], maskratio=a.get("maskratio", 0.35))
        torch.cuda.synchronize()
        assert np.array_equal(t.cpu().numpy(), frames) and (good.cpu().numpy() == SENT).all(), "written after a refusal"

    refused("frame range outside the clip", frame0=5, nframes=N)
    refused("frame range outside the clip", frame0=-1, nframes=2)
    refused("max_fade_length", max_fade_length=-1)
    refused("maskratio", maskratio=0.0)
    refused("frame_result values", frame_result=np.full(N, 3, np.uint8))
    refused("logo rectangle lies outside the frame", logo=ab.Logo.create(LOGO["data"], 64, 64, W, H, W - 32, IMGY))
    c422 = ab.yv12_clip(t, W, H, N, True, 8); c422.log_uvy = 0; c422.num_frames = N // 2
    refused("chroma subsampling mismatch", src=c422, nframes=N // 2)
    refused("bits_per_sample", src=_with(src, bits_per_sample=7))
    refused("dst must be device resident", dst=_with(gdst, on_device=0, base=frames.ctypes.data))
    refused("format differs", dst=_with(gdst, bits_per_sample=10, bytes_per_sample=2, num_frames=N // 2,
                                         pitch_y=2 * W, pitch_uv=W, off_u=2 * W * H, off_v=2 * W * H + W * H // 2,
                                         frame_stride=3 * W * H), nframes=N // 2)
    refused("fewer than nframes", dst=_with(gdst, num_frames=N - 1))
    refused("overlaps src", dst=src)
    host = frames.copy()
    refused("needs a device-resident src", src=ab.yv12_clip(host, W, H, N, False, 8), dst=gdst)


def _with(desc, **kw):
    d = ab.ClipDesc.from_buffer_copy(desc)
    for k, v in kw.items():
        setattr(d, k, v)
    return d
