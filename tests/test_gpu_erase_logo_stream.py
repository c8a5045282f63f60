"""amtk_erase_logo_stream: AMTEraseLogo(AMTAnalyzeLogo(src, logo), logo, logof, maxfade) fed one decoded frame at a time
(DESIGN.md section 3.3.2).

Every output must equal the composition built from the reference's own code (oracle/_ref, else the C port): the
AMTAnalyzeLogo::GetFrameT records of the clip, AMTEraseLogo's fade selection over them (ReadLogoFrameFile + CalcFade), and
Delogo with those fades -- byte for byte -- and also amtk_erase_logo_frames with those fades.  The fades recv returns equal
the reference's bit for bit.  After every send the outputs that can be received equal the restated receive rule
(tests/test_erase_logo_stream_rule.py, checked there against a port of CalcFade)."""

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth
from test_erase_logo_stream_rule import fade2_index, fade_codes, receivable, record_set
from test_gpu_erase import _expected

pytestmark = pytest.mark.gpu

W, H = 256, 160
LOGO = synth.make_logo(64, 64, seed=3)
SENT = 0xA5


# ---------------------------------------------------------------------------------------------------------------------
# clips: a logo that fades in and out, appears and vanishes abruptly, and shows on one field only at two frames
# ---------------------------------------------------------------------------------------------------------------------
def field_fades(N):
    """(N, 2) logo strength 0..256 for the top and bottom field of every frame."""
    f = np.zeros((N, 2), np.int64)
    a0, a1, b0, b1 = N // 5, N // 2, (3 * N) // 5, (9 * N) // 10
    f[a0:a1] = 256
    f[b0:b1] = 256
    if N >= 10:
        f[a0 - 1] = (0, 256)                           # bottom field only
        f[b1] = (256, 0)                               # top field only
        f[a1] = (128, 128)
    return f


def make_clip(N, bits, imgx, imgy, seed=7, lw=64, lh=64, logo=LOGO):
    bg = synth.make_frames(0, N, W, H, seed=0x5EED0100 + seed, mode="interlaced").numpy().astype(np.int64)
    ff = field_fades(N)
    ysz, csz = W * H, (W // 2) * (H // 2)
    Y = bg[:, :ysz].reshape(N, H, W)
    al = logo["alpha8"].astype(np.int64)
    a = (al[None, :, :] * np.where((np.arange(lh) & 1)[None, :, None] == 1, ff[:, 1, None, None], ff[:, 0, None, None])) >> 8
    roi = Y[:, imgy:imgy + lh, imgx:imgx + lw]
    Y[:, imgy:imgy + lh, imgx:imgx + lw] = (roi * (256 - a) + a * logo["L8"] + 128) >> 8
    alC = logo["alphaC"].astype(np.int64)
    aC = (alC[None] * ff.max(axis=1)[:, None, None]) >> 8
    for o in (ysz, ysz + csz):
        P = bg[:, o:o + csz].reshape(N, H // 2, W // 2)
        r = P[:, imgy // 2:imgy // 2 + lh // 2, imgx // 2:imgx // 2 + lw // 2]
        P[:, imgy // 2:imgy // 2 + lh // 2, imgx // 2:imgx // 2 + lw // 2] = (r * (256 - aC) + aC * 128 + 128) >> 8
    if bits == 8:
        return bg.astype(np.uint8)
    rng = np.random.default_rng(seed)
    low = rng.integers(0, 1 << (bits - 8), bg.shape)
    return ((bg << (bits - 8)) | low).astype(np.uint16)


def write_logof(path, events):
    """events: (start_best, start_lo, start_hi, end_best, end_lo, end_hi) per logo section (LogoScan.hpp:1818-1819)."""
    with open(path, "w") as f:
        for sb, s0, s1, eb, e0, e1 in events:
            f.write("%6d S 0 ALL %6d %6d\n%6d E 0 ALL %6d %6d\n" % (sb, s0, s1, eb, e0, e1))
    return str(path)


LOGOF = {
    "start": [(1, 0, 3, 60, 58, 62)],
    "middle": [(40, 38, 42, 70, 69, 72)],
    "end": [(20, 19, 21, 97, 95, 99)],
    "close": [(30, 29, 31, 36, 35, 37), (44, 43, 45, 80, 78, 82)],       # transitions closer than maxfade
}


# ---------------------------------------------------------------------------------------------------------------------
# the reference composition
# ---------------------------------------------------------------------------------------------------------------------
def read_logoframe(path, N):
    """AMTEraseLogo::ReadLogoFrameFile (LogoScan.hpp:1421-1461) for the C-port fallback."""
    el = []
    for line in open(path):
        t = line.split()
        el.append((t[1].lower() == "s", int(t[4]), int(t[5])))
    fr = np.zeros(N, np.int32)

    def fill(a, b, v):
        fr[min(N, a):min(N, max(a, b))] = v
    for i in range(0, len(el), 2):
        fill(el[i][1], el[i][2] + 1, 1)
        fill(el[i][2], el[i + 1][1] + 1, 2)
        fill(el[i + 1][1] + 1, el[i + 1][2] + 1, 1)
    return fr


class Reference:
    def __init__(self, po, bits, imgx, imgy, logo=LOGO):
        self.po, self.bits, self.imgx, self.imgy, self.logo = po, bits, imgx, imgy, logo
        lw, lh = logo["w"], logo["h"]
        if po.ref_has_drivers():
            raw = po.RefLogo.create(logo["data"], lw, lh, W, H, imgx, imgy)
            self.dl, self.ft, self.fb = raw.deint().create_mask(0.35), raw.field(0).create_mask(0.35), raw.field(1).create_mask(0.35)
            self.kind = "reference"
        else:
            raw = po.OracleLogo.create(logo["data"], lw, lh, W, H, imgx, imgy)
            self.dl, self.ft, self.fb = raw.deint().create_mask(0.35), raw.field(0).create_mask(0.35), raw.field(1).create_mask(0.35)
            self.kind = "port"

    def records(self, frames):
        N = frames.shape[0]
        if self.kind == "reference":
            blocks = [self.po.ref_analyze_getframe(self.dl, self.ft, self.fb, frames, W, H, a, self.bits) for a in range((N + 7) // 8)]
            return np.concatenate(blocks)[:N]
        Y = frames[:, :W * H].reshape(N, H, W)
        return np.stack([self.po.or_analyze_frame(self.dl, self.ft, self.fb, Y[i], float((1 << self.bits) - 1)) for i in range(N)])

    def fades(self, rec, N, logof, maxfade):
        if self.kind == "reference":
            f, fr = self.po.ref_erase_fades(rec, N, logof, maxfade)
            return f, (None if fr is None else fr.astype(np.uint8))
        fr = read_logoframe(logof, N) if logof else None
        codes = fade_codes(N, fr, maxfade)
        out = np.zeros((N, 2), np.float32)
        for n in range(N):
            out[n] = self.po.or_calc_fade2(rec, N, n) if codes[n] == 2 else (codes[n], codes[n])
        return out, (None if fr is None else fr.astype(np.uint8))

    def pixels(self, frames, fades):
        lw, lh = self.logo["w"], self.logo["h"]
        return _expected(self.po, self.logo["data"], lw, lh, self.imgx, self.imgy, frames, W, H, fades, (1 << self.bits) - 1)


# ---------------------------------------------------------------------------------------------------------------------
# frame layouts: packed, or V-first with padded rows and planes (sentinel-filled); pageable, pinned or device memory
# ---------------------------------------------------------------------------------------------------------------------
class Frame:
    def __init__(self, packed, bits, layout, mem):
        bps = 1 if bits == 8 else 2
        self.bits, self.bps, self.layout, self.mem = bits, bps, layout, mem
        if layout == "packed":
            py, pc = W * bps, (W // 2) * bps
            offu, offv = py * H, py * H + pc * (H // 2)
            total = offv + pc * (H // 2)
        else:
            py, pc = W * bps + 48, (W // 2) * bps + 32
            offv = py * H + 16
            offu = offv + pc * (H // 2) + 16
            total = offu + pc * (H // 2) + 64
        self.py, self.pc, self.offu, self.offv, self.total = py, pc, offu, offv, total
        buf = np.full(total, SENT, np.uint8)
        b = packed.view(np.uint8)
        ysz, csz = W * H * bps, (W // 2) * (H // 2) * bps
        self._put(buf, 0, py, b[:ysz], W * bps, H)
        self._put(buf, offu, pc, b[ysz:ysz + csz], (W // 2) * bps, H // 2)
        self._put(buf, offv, pc, b[ysz + csz:], (W // 2) * bps, H // 2)
        if mem == "pageable":
            self.buf = buf
            base = buf.ctypes.data
        elif mem == "pinned":
            self.buf = torch.from_numpy(buf).pin_memory()
            base = self.buf.data_ptr()
        else:
            self.buf = torch.from_numpy(buf).cuda()
            base = self.buf.data_ptr()
        d = ab.ClipDesc()
        d.base, d.frame_stride, d.off_u, d.off_v = base, total, offu, offv
        d.width, d.height, d.pitch_y, d.pitch_uv = W, H, py, pc
        d.log_uvx = d.log_uvy = 1
        d.bytes_per_sample, d.bits_per_sample, d.num_frames, d.on_device = bps, bits, 1, 1 if mem == "device" else 0
        self.desc = d

    @staticmethod
    def _put(buf, off, pitch, src, rb, rows):
        buf[off:off + pitch * rows].reshape(rows, pitch)[:, :rb] = src.reshape(rows, rb)

    def raw(self):
        torch.cuda.synchronize()
        return self.buf.cpu().numpy() if isinstance(self.buf, torch.Tensor) else self.buf.copy()

    def packed(self):
        """(frame as packed samples, padding bytes)"""
        raw, bps = self.raw(), self.bps
        rows = []
        pad = []
        for off, pitch, rb, n in ((0, self.py, W * bps, H), (self.offu, self.pc, (W // 2) * bps, H // 2), (self.offv, self.pc, (W // 2) * bps, H // 2)):
            blk = raw[off:off + pitch * n].reshape(n, pitch)
            rows.append(blk[:, :rb].reshape(-1))
            pad.append(blk[:, rb:].reshape(-1))
        mask = np.ones(self.total, bool)
        for off, pitch, rb, n in ((0, self.py, W * bps, H), (self.offu, self.pc, (W // 2) * bps, H // 2), (self.offv, self.pc, (W // 2) * bps, H // 2)):
            mask[off:off + pitch * n].reshape(n, pitch)[:, :rb] = False
        dt = np.uint8 if bps == 1 else np.uint16
        return np.concatenate(rows).view(dt), raw[mask]


MEMS = ("pageable", "pinned", "device")


def run_stream(ctx, logo, frames, bits, frame_result, maxfade, B, src=("pageable",), src_layout="packed",
               dst_mem="pageable", dst_layout="packed", check_rule=True, stream=None):
    """Sends every frame, receiving whatever can be received after each send.  Returns (outputs (N, ...), fades (N, 2),
    the stream, host frames sent)."""
    N = frames.shape[0]
    s = stream or ctx.erase_logo_stream(logo, N, frame_result, maxfade, B)
    outs = np.zeros_like(frames)
    fades = np.zeros((N, 2), np.float32)
    got = 0
    host_sent = 0
    for S in range(1, N + 1):
        mem = src[(S - 1) % len(src)]
        f = Frame(frames[S - 1], bits, src_layout, mem)
        s.send(f.desc)
        host_sent += mem != "device"
        while True:
            d = Frame(frames[got], bits, dst_layout, dst_mem) if got < N else Frame(frames[0], bits, dst_layout, dst_mem)
            r = s.recv(d.desc)
            if r is None:
                break
            n, fd = r
            assert n == got
            px, pad = d.packed()
            assert (pad == SENT).all(), "bytes outside the frame's samples were written"
            outs[n], fades[n] = px, fd
            got += 1
        if check_rule:
            assert got == receivable(S, N, B), (S, got)
    assert got == N
    return outs, fades, s, host_sent


def check_against_reference(ctx, po, frames, bits, imgx, imgy, logof, maxfade, B, **kw):
    N = frames.shape[0]
    ref = Reference(po, bits, imgx, imgy)
    rec = ref.records(frames)
    rf, fr = ref.fades(rec, N, logof, maxfade)
    logo = ab.Logo.create(LOGO["data"], 64, 64, W, H, imgx, imgy)
    outs, fades, s, host_sent = run_stream(ctx, logo, frames, bits, fr, maxfade, B, **kw)
    assert np.array_equal(fades.view(np.uint32), rf.view(np.uint32)), "fades differ from the reference's"
    exp = ref.pixels(frames, rf)
    assert np.array_equal(outs, exp), "pixels differ from the reference composition (%s)" % ref.kind
    lib_out = frames.copy()
    ctx.erase_logo(ab.yv12_clip(lib_out, W, H, N, False, bits), logo, rf)
    assert np.array_equal(outs, lib_out), "pixels differ from amtk_erase_logo_frames"
    sent, received, analysed, h2d, d2h = s.counts()
    payload = (64 * 64 + 2 * 32 * 32) * (1 if bits == 8 else 2)
    assert (sent, received) == (N, N)
    assert analysed == len(record_set(N, fr, maxfade))
    assert h2d == host_sent * payload
    assert d2h == N * (payload + 8)
    s.close()
    return fades


# ---------------------------------------------------------------------------------------------------------------------
# pixels and fades
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3, 8, 16, 64])
@pytest.mark.parametrize("N", [1, 2, 7, 8, 9, 17, 100])
def test_no_logoframe_file_every_length_and_batch(ctx, oracle, N, B):
    frames = make_clip(N, 8, 100, 40)
    check_against_reference(ctx, oracle, frames, 8, 100, 40, None, 16, B)


@pytest.mark.parametrize("maxfade", [0, 1, 16, 31])
@pytest.mark.parametrize("kind", sorted(LOGOF))
def test_logoframe_files(ctx, oracle, tmp_path, kind, maxfade):
    frames = make_clip(100, 8, 100, 40)
    path = write_logof(tmp_path / "logof.txt", LOGOF[kind])
    check_against_reference(ctx, oracle, frames, 8, 100, 40, path, maxfade, 16)


@pytest.mark.parametrize("B", [1, 8, 64])
@pytest.mark.parametrize("N", [9, 17])
def test_logoframe_short_clips(ctx, oracle, tmp_path, N, B):
    frames = make_clip(N, 8, 100, 40)
    path = write_logof(tmp_path / "logof.txt", [(2, 1, 3, N - 3, N - 4, N - 2)])
    check_against_reference(ctx, oracle, frames, 8, 100, 40, path, 4, B)


def test_coverage_field_mode_and_both_fade_ends(ctx, oracle, tmp_path):
    """The test clip reaches field mode (fadeT != fadeB), fade 0 and fade 1, with and without a logoframe file."""
    frames = make_clip(100, 8, 100, 40)
    a = check_against_reference(ctx, oracle, frames, 8, 100, 40, None, 16, 16)
    b = check_against_reference(ctx, oracle, frames, 8, 100, 40, write_logof(tmp_path / "l.txt", LOGOF["close"]), 16, 16)
    allf = np.concatenate([a, b])
    assert (allf[:, 0] != allf[:, 1]).any(), "no output in field mode"
    assert ((allf[:, 0] == 0) & (allf[:, 1] == 0)).any(), "no output at fade 0"
    assert ((allf[:, 0] == 1) & (allf[:, 1] == 1)).any(), "no output at fade 1"


@pytest.mark.parametrize("bits", [8, 10, 12, 16])
@pytest.mark.parametrize("pos", [(100, 40), (100, 42), (128, 40), (37, 42)])
def test_bits_and_positions(ctx, oracle, bits, pos):
    """imgx 100 and 37 are not 16-byte aligned; (imgy/2) % 2 is 0 at 40 and 1 at 42."""
    frames = make_clip(40, bits, pos[0], pos[1], seed=bits)
    check_against_reference(ctx, oracle, frames, bits, pos[0], pos[1], None, 16, 8)


# ---------------------------------------------------------------------------------------------------------------------
# layouts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [8, 16])
@pytest.mark.parametrize("src_layout,dst_layout,dst_mem", [("packed", "vfirst", "pageable"), ("vfirst", "packed", "pinned"),
                                                           ("vfirst", "vfirst", "device"), ("packed", "packed", "device")])
def test_mixed_memory_and_layouts(ctx, oracle, bits, src_layout, dst_layout, dst_mem):
    """Pinned, pageable and device frames mixed within one stream; V-first padded layouts (padding must stay sentinel);
    a dst whose layout differs from the source's."""
    frames = make_clip(30, bits, 100, 42, seed=3)
    check_against_reference(ctx, oracle, frames, bits, 100, 42, None, 16, 4, src=MEMS, src_layout=src_layout,
                            dst_layout=dst_layout, dst_mem=dst_mem)


def test_device_frames_upload_nothing(ctx, oracle):
    frames = make_clip(20, 8, 100, 40)
    check_against_reference(ctx, oracle, frames, 8, 100, 40, None, 16, 4, src=("device",))


def test_dst_outside_rectangles_untouched(ctx):
    """A dst filled with a sentinel outside the logo rectangles keeps it: only the three rectangles are written."""
    N = 12
    frames = make_clip(N, 8, 100, 40)
    logo = ab.Logo.create(LOGO["data"], 64, 64, W, H, 100, 40)
    s = ctx.erase_logo_stream(logo, N, None, 16, 4)
    for n in range(N):
        s.send(Frame(frames[n], 8, "packed", "pinned").desc)
    from test_gpu_erase import logo_rect_mask
    m = logo_rect_mask(W, H, 64, 64, 100, 40)
    for n in range(N):
        fill = frames[n].copy()
        fill[~m] = 0x5A
        d = Frame(fill, 8, "vfirst", "pageable")
        assert s.recv(d.desc)[0] == n
        px, pad = d.packed()
        assert (px[~m] == 0x5A).all() and (pad == SENT).all()
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# counts and launches
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("value", [0, 1, 2])
def test_uniform_frame_result_analyses_nothing(ctx, oracle, value):
    N, B = 50, 8
    frames = make_clip(N, 8, 100, 40)
    logo = ab.Logo.create(LOGO["data"], 64, 64, W, H, 100, 40)
    fr = np.full(N, value, np.uint8)
    l0 = ctx.launches
    outs, fades, s, _ = run_stream(ctx, logo, frames, 8, fr, 16, B)
    nb = (N + B - 1) // B
    assert ctx.launches - l0 == 2 * nb                    # fade + erase kernel per batch, no evaluation kernel
    assert s.counts()[2] == 0
    f = 1.0 if value == 2 else 0.0
    assert (fades == f).all()
    lib_out = frames.copy()
    ctx.erase_logo(ab.yv12_clip(lib_out, W, H, N, False), logo, fades)
    assert np.array_equal(outs, lib_out)


def test_large_logo_with_uniform_frame_result(ctx):
    """A logo above the evaluation plan's limit is refused only when some frame would be analysed."""
    big = synth.make_logo(256, 128, seed=5)
    logo = ab.Logo.create(big["data"], 256, 128, 320, 192, 16, 16)
    with pytest.raises(ab.AmtkError, match="too large"):
        ctx.erase_logo_stream(logo, 10, None, 16, 4)
    with pytest.raises(ab.AmtkError, match="too large"):
        ctx.erase_logo_stream(logo, 10, np.array([0] * 5 + [2] * 5, np.uint8), 4, 4)
    s = ctx.erase_logo_stream(logo, 10, np.zeros(10, np.uint8), 4, 4)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# rejections and lifetime
# ---------------------------------------------------------------------------------------------------------------------
def _logo(imgx=100, imgy=40):
    return ab.Logo.create(LOGO["data"], 64, 64, W, H, imgx, imgy)


@pytest.mark.parametrize("args,msg", [((0, None, 16, 4), "num_frames"), ((5, None, -1, 4), "max_fade_length"),
                                      ((5, None, 16, 0), "batch_size"), ((5, None, 16, 257), "batch_size"),
                                      ((3, np.array([0, 3, 0], np.uint8), 16, 4), "frame_result")])
def test_create_rejections(ctx, args, msg):
    with pytest.raises(ab.AmtkError, match=msg):
        ctx.erase_logo_stream(_logo(), *args)
    with pytest.raises(ab.AmtkError, match="maskratio"):
        ctx.erase_logo_stream(_logo(), 5, None, 16, 4, maskratio=0.0)


def test_send_rejections_leave_the_stream_as_it_was(ctx):
    """A two-frame clip, another bit depth, another size (sends) and a dst of another format (recv) are refused; the stream
    then runs on and its outputs equal a clean run's.  Sends beyond N are refused."""
    N = 20
    frames = make_clip(N, 8, 100, 40)
    logo = _logo()
    clean, _, s0, _ = run_stream(ctx, logo, frames, 8, None, 16, 4)
    s0.close()
    s = ctx.erase_logo_stream(logo, N, None, 16, 4)
    other = make_clip(1, 10, 100, 40)
    with pytest.raises(ab.AmtkError, match="exactly one frame"):
        s.send(ab.yv12_clip(frames[:2].copy(), W, H, 2, False))
    s.send(Frame(frames[0], 8, "packed", "pageable").desc)
    with pytest.raises(ab.AmtkError, match="format"):
        s.send(Frame(other[0], 10, "packed", "pageable").desc)
    with pytest.raises(ab.AmtkError, match="format"):
        s.send(ab.yv12_clip(np.zeros(128 * 96 * 3 // 2, np.uint8), 128, 96, 1, False))
    with pytest.raises(ab.AmtkError, match="format"):
        s.recv(Frame(other[0], 10, "packed", "pageable").desc)
    for n in range(1, N):
        s.send(Frame(frames[n], 8, "packed", "pageable").desc)
    with pytest.raises(ab.AmtkError, match="all num_frames"):
        s.send(Frame(frames[0], 8, "packed", "pageable").desc)
    outs = np.zeros_like(frames)
    for n in range(N):
        d = Frame(frames[n], 8, "packed", "pageable")
        assert s.recv(d.desc)[0] == n
        outs[n] = d.packed()[0]
    assert s.recv(Frame(frames[0], 8, "packed", "pageable").desc) is None
    assert np.array_equal(outs, clean)
    s.close()


def test_rejected_frames_do_not_change_outputs(ctx, oracle):
    """Rejected sends between valid ones leave every output as the clean run's."""
    N = 20
    frames = make_clip(N, 8, 100, 40)
    logo = _logo()
    clean, cf, s0, _ = run_stream(ctx, logo, frames, 8, None, 16, 4)
    s0.close()
    s = ctx.erase_logo_stream(logo, N, None, 16, 4)
    other = make_clip(1, 12, 100, 40)
    outs = np.zeros_like(frames)
    got = 0
    for n in range(N):
        if n:                                     # the first frame fixes the format
            with pytest.raises(ab.AmtkError, match="format"):
                s.send(Frame(other[0], 12, "packed", "pageable").desc)
        s.send(Frame(frames[n], 8, "packed", "pinned").desc)
        while True:
            d = Frame(frames[min(got, N - 1)], 8, "packed", "pageable")
            r = s.recv(d.desc)
            if r is None:
                break
            outs[r[0]] = d.packed()[0]
            got += 1
    assert got == N and np.array_equal(outs, clean)
    with pytest.raises(ab.AmtkError, match="all num_frames"):
        s.send(Frame(frames[0], 8, "packed", "pageable").desc)
    s.close()


@pytest.mark.parametrize("stage", ["created", "some_sent", "all_sent", "half_received", "all_received"])
def test_destroy_at_every_stage(ctx, stage):
    N = 30
    frames = make_clip(N, 8, 100, 40)
    s = ctx.erase_logo_stream(_logo(), N, None, 16, 4)
    if stage != "created":
        k = 7 if stage == "some_sent" else N
        for n in range(k):
            s.send(Frame(frames[n], 8, "packed", ("pinned", "device")[n % 2]).desc)
        want = {"some_sent": 0, "all_sent": 0, "half_received": N // 2, "all_received": N}[stage]
        for n in range(want):
            assert s.recv(Frame(frames[n], 8, "packed", "pageable").desc)[0] == n
    s.close()
    ctx.synchronize()


def test_two_interleaved_streams_on_one_context(ctx, oracle):
    N = 40
    fa = make_clip(N, 8, 100, 40, seed=1)
    fb = make_clip(N, 8, 37, 42, seed=2)
    ra, rb = Reference(oracle, 8, 100, 40), Reference(oracle, 8, 37, 42)
    fa_ref, _ = ra.fades(ra.records(fa), N, None, 16)
    fb_ref, _ = rb.fades(rb.records(fb), N, None, 16)
    sa = ctx.erase_logo_stream(_logo(100, 40), N, None, 16, 3)
    sb = ctx.erase_logo_stream(_logo(37, 42), N, None, 16, 16)
    outs = {id(sa): np.zeros_like(fa), id(sb): np.zeros_like(fb)}
    got = {id(sa): 0, id(sb): 0}
    for n in range(N):
        for s, fr in ((sa, fa), (sb, fb)):
            s.send(Frame(fr[n], 8, "packed", "pinned").desc)
            while True:
                k = got[id(s)]
                d = Frame(fr[min(k, N - 1)], 8, "packed", "pageable")
                r = s.recv(d.desc)
                if r is None:
                    break
                outs[id(s)][r[0]] = d.packed()[0]
                got[id(s)] += 1
    assert np.array_equal(outs[id(sa)], ra.pixels(fa, fa_ref))
    assert np.array_equal(outs[id(sb)], rb.pixels(fb, fb_ref))
    sa.close()
    sb.close()


def test_record_reads_stay_inside_the_lookahead():
    """The indices the device reads are amtk_calc_fade2_index's, which stay within [n-8, min(N-1, n+8)]."""
    for N in (1, 9, 17, 100):
        for n in range(N):
            for i in range(-4, 5):
                f = ab.lib().amtk_calc_fade2_index(N, N, n, i)
                assert f == fade2_index(N, n, i) and n - 8 <= f <= min(N - 1, n + 8)
