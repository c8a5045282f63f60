"""amtk_comb_stream: the combing counters of the telecine pre-pass fed one decoded frame at a time (DESIGN.md section 3.1d).

With C the clip of all frames sent, the 12 counters of sent frame n must equal row n of amtk_comb_frames(C, 0, N) on a
resident clip of the same frames -- integers, so identical -- and the CPU spec oracle on a few cases.  After every send and
after finish, the rows that can be received equal the restated receive rule."""

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth

pytestmark = pytest.mark.gpu


def params(**kw):
    p = ab.default_comb_params()
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def make_frames(N, w, h, bits, seed=1, mode="telecine"):
    """(N, w*h*3/2) packed 4:2:0 frames, uint8 or uint16 at `bits` (every sample <= maxv): 3:2 pulldown or interlaced
    motion, so that every counter moves."""
    f = synth.make_frames(0, N, w, h, seed=0x5EED0400 + seed, mode=mode).numpy()
    if bits == 8:
        return f
    low = np.random.default_rng(seed).integers(0, 1 << (bits - 8), f.shape)
    return ((f.astype(np.int64) << (bits - 8)) | low).astype(np.uint16)


def resident(ctx, fr, w, h, bits, prm):
    """amtk_comb_frames over the frames as one resident clip: (N, 12)."""
    t = torch.from_numpy(fr.view(np.int16) if bits > 8 else fr).cuda()
    return ctx.comb_frames(ab.yv12_clip(t, w, h, fr.shape[0], True, bits), prm).cpu().numpy()


def slot_bytes(w, h, bits):
    """The frame stride of the stream's own layout: 16-byte aligned pitches and planes, 256-byte aligned frames."""
    bps = 1 if bits == 8 else 2
    py, pc = (w * bps + 15) & ~15, ((w // 2) * bps + 15) & ~15
    return (py * h + 2 * pc * (h // 2) + 255) & ~255


# frame layouts: name -> (extra luma pitch bytes, extra chroma pitch bytes, V plane first)
LAYOUTS = {"packed": (0, 0, False), "vfirst": (32, 16, True), "odd": (1, 3, False), "pad8": (8, 8, True)}
MEMS = ("pageable", "pinned", "device")


class Frame:
    """One packed frame re-laid out in host (pageable or pinned) or device memory, with its one-frame descriptor."""

    def __init__(self, packed, w, h, bits, layout="packed", mem="pageable"):
        bps = 1 if bits == 8 else 2
        ey, ec, vfirst = LAYOUTS[layout]
        if bps == 2:                 # whole samples per row (odd byte pitches would split them)
            ey, ec = ey + (ey & 1), ec + (ec & 1)
        b = np.ascontiguousarray(packed).view(np.uint8)
        ysz, csz = w * h * bps, (w // 2) * (h // 2) * bps
        ry, rc, hc = w * bps, (w // 2) * bps, h // 2
        py, pc = ry + ey, rc + ec
        planes = [(b[:ysz], ry, py, h), (b[ysz:ysz + csz], rc, pc, hc), (b[ysz + csz:], rc, pc, hc)]
        order = [2, 1, 0] if vfirst else [0, 1, 2]
        offs, pos = {}, 0
        for i in order:
            offs[i] = pos
            pos += planes[i][2] * planes[i][3]
        buf = np.full(pos + 64, 0xA5, np.uint8)
        for i, (src, row, pitch, rows) in enumerate(planes):
            dst = buf[offs[i]:offs[i] + pitch * rows].reshape(rows, pitch)
            dst[:, :row] = src.reshape(rows, row)
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
        d.frame_stride = pos
        d.off_u, d.off_v = offs[1] - offs[0], offs[2] - offs[0]
        d.base = base + offs[0]
        d.width, d.height = w, h
        d.pitch_y, d.pitch_uv = py, pc
        d.log_uvx = d.log_uvy = 1
        d.bytes_per_sample, d.bits_per_sample = bps, bits
        d.num_frames = 1
        d.on_device = 1 if mem == "device" else 0
        d.keep = self.buf            # the descriptor keeps the frame's memory alive (send(Frame(...).desc))
        self.desc = d


def receivable(S, B, finished):
    """Rows that can have been received after S sends: batch k once batch k+1 was launched (S >= (k+2)B), all after finish."""
    return S if finished else max(0, S // B - 1) * B


def run(ctx, fr, w, h, bits, B, prm=None, layouts=("packed",), mems=("pageable",), chunk=1 << 20):
    """Sends every frame (layouts and memory kinds cycling), receiving after each send and after finish; checks the
    receive rule throughout.  Returns (rows (N, 12), counts, host frames sent)."""
    s = ctx.comb_stream(prm, B)
    got, nhost = [], 0
    for k in range(fr.shape[0]):
        f = Frame(fr[k], w, h, bits, layouts[k % len(layouts)], mems[k % len(mems)])
        nhost += f.desc.on_device == 0
        s.send(f.desc)
        while True:
            r = s.recv(chunk)
            got.append(r)
            if len(r) < chunk:
                break
        assert sum(len(g) for g in got) == receivable(k + 1, B, False), (k, B)
    s.finish()
    got.append(s.recv(fr.shape[0] + 1))
    assert sum(len(g) for g in got) == fr.shape[0]
    assert len(s.recv(5)) == 0
    counts = s.counts()
    s.close()
    return np.concatenate(got).reshape(-1, 12), counts, nhost


def lengths(B):
    return sorted({n for n in (1, 2, B - 1, B, B + 1, 2 * B, 2 * B + 1, 3 * B + 5) if n >= 1})


# ---------------------------------------------------------------------------------------------------------------------
# the result rule
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 2, 7, 64, 256])
def test_every_length_around_the_batch_size(ctx, B):
    w, h = 256, 160
    fr = make_frames(3 * B + 5, w, h, 8, seed=B)
    exp = resident(ctx, fr, w, h, 8, None)
    assert (exp != 0).any(axis=0).all()              # every counter moves
    for N in lengths(B):
        rows, (sent, received, h2d, d2h), nhost = run(ctx, fr[:N], w, h, 8, B, mems=("pinned",))
        assert np.array_equal(rows, exp[:N]), (B, N)      # a prefix clip's rows are the prefix of the rows
        assert (sent, received, d2h) == (N, N, 48 * N)
        assert h2d == nhost * slot_bytes(w, h, 8) == N * slot_bytes(w, h, 8)


GEOMS = [(1920, 1080, 8), (1440, 1080, 8), (1920, 1080, 10), (720, 480, 12), (720, 480, 16), (202, 94, 8), (202, 94, 10)]


@pytest.mark.parametrize("w,h,bits", GEOMS)
def test_geometries_and_sample_sizes(ctx, w, h, bits):
    B = 7
    fr = make_frames(3 * B + 5, w, h, bits, seed=w + bits, mode="interlaced")
    exp = resident(ctx, fr, w, h, bits, None)
    rows, (sent, received, h2d, d2h), _ = run(ctx, fr, w, h, bits, B, mems=("pinned", "device"))
    assert np.array_equal(rows, exp)
    assert (exp != 0).any()


@pytest.mark.parametrize("bits", [8, 10, 16])
def test_cpu_spec_oracle(ctx, oracle, bits):
    w, h, B = 128, 64, 4
    fr = make_frames(11, w, h, bits, seed=bits)
    prm = ab.default_comb_params()
    rows, _, _ = run(ctx, fr, w, h, bits, B, mems=MEMS)
    ysz, csz = w * h, (w // 2) * (h // 2)
    Y = fr[:, :ysz].reshape(-1, h, w)
    U = fr[:, ysz:ysz + csz].reshape(-1, h // 2, w // 2)
    V = fr[:, ysz + csz:].reshape(-1, h // 2, w // 2)
    assert np.array_equal(rows, oracle.or_comb_clip(Y, U, V, prm.as_list()))


@pytest.mark.parametrize("bits,kw", [(8, dict(th_move_y=1, th_move_c=1)), (8, dict(th_move_y=128, th_move_c=128)),
                                     (8, dict(th_shima_y=2047, th_lshima_y=2047, th_shima_c=2047, th_lshima_c=2047)),
                                     (16, dict(th_move_y=32768, th_move_c=32768))])
def test_threshold_edges(ctx, bits, kw):
    w, h, B = 256, 160, 7
    prm = params(**kw)
    fr = make_frames(2 * B + 1, w, h, bits, seed=3)
    rows, _, _ = run(ctx, fr, w, h, bits, B, prm, mems=MEMS)
    assert np.array_equal(rows, resident(ctx, fr, w, h, bits, prm))


# ---------------------------------------------------------------------------------------------------------------------
# sources and layouts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [8, 10, 16])
def test_mixed_sources_and_layouts_run_the_tma_kernels(ctx, bits):
    """Pinned, pageable and device frames mixed in one stream, in V-first, padded, odd-pitch and 8-mod-16-pitch layouts:
    exact, and every batch is one timed launch of a streaming (TMA) kernel -- the plain-load kernel is not timed."""
    w, h, B = 240, 136, 5
    fr = make_frames(4 * B + 3, w, h, bits, seed=11)
    exp = resident(ctx, fr, w, h, bits, None)
    ctx.set_kernel_timing(True)
    try:
        ctx.kernel_timing(reset=True)
        before = ctx.launches
        rows, (sent, received, h2d, d2h), nhost = run(ctx, fr, w, h, bits, B, layouts=tuple(LAYOUTS), mems=MEMS)
        launches = ctx.launches - before
        ms, timed = ctx.kernel_timing(reset=True)
    finally:
        ctx.set_kernel_timing(False)
    nb = -(-fr.shape[0] // B)
    assert np.array_equal(rows, exp)
    assert launches == nb and timed == nb and ms > 0
    assert h2d == nhost * slot_bytes(w, h, bits) and 0 < nhost < fr.shape[0]
    assert d2h == 48 * fr.shape[0]


def test_device_frames_upload_nothing(ctx):
    w, h, B = 256, 160, 4
    fr = make_frames(10, w, h, 8)
    rows, (sent, received, h2d, d2h), _ = run(ctx, fr, w, h, 8, B, mems=("device",))
    assert np.array_equal(rows, resident(ctx, fr, w, h, 8, None)) and h2d == 0 and d2h == 480


# ---------------------------------------------------------------------------------------------------------------------
# the receive rule with partial reads
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk", [1, 3])
def test_receive_rule_partial_reads(ctx, chunk):
    w, h, B, N = 256, 160, 4, 19
    fr = make_frames(N, w, h, 8, seed=5)
    exp = resident(ctx, fr, w, h, 8, None)
    s = ctx.comb_stream(None, B)
    got = []
    for k in range(N):
        s.send(Frame(fr[k], w, h, 8, mem=MEMS[k % 3]).desc)
        assert len(s.recv(0)) == 0
        r = s.recv(chunk)                        # at most chunk, never beyond the rule
        got.append(r)
        assert len(r) == min(chunk, receivable(k + 1, B, False) - sum(len(g) for g in got[:-1]))
        assert s.counts()[:2] == (k + 1, sum(len(g) for g in got))
    s.finish()
    while True:
        r = s.recv(chunk)
        if len(r) == 0:
            break
        got.append(r)
    assert np.array_equal(np.concatenate(got), exp)
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# rejections
# ---------------------------------------------------------------------------------------------------------------------
def test_create_refusals(ctx):
    for B in (0, 257):
        with pytest.raises(ab.AmtkError, match="batch_size"):
            ctx.comb_stream(None, B)
    with pytest.raises(ab.AmtkError, match="thresholds must be >= 1"):
        ctx.comb_stream(params(th_lshima_c=0), 4)


def test_rejections_leave_the_stream_unchanged(ctx):
    w, h, B = 256, 160, 3
    fr = make_frames(8, w, h, 8, seed=9)
    exp = resident(ctx, fr, w, h, 8, None)
    s = ctx.comb_stream(None, B)
    t = torch.from_numpy(fr[:2]).cuda()
    with pytest.raises(ab.AmtkError, match="exactly one frame"):
        s.send(ab.yv12_clip(t, w, h, 2, True))
    s.send(Frame(fr[0], w, h, 8).desc)
    other = make_frames(1, w + 16, h, 8)
    with pytest.raises(ab.AmtkError, match="format differs"):
        s.send(Frame(other[0], w + 16, h, 8).desc)
    with pytest.raises(ab.AmtkError, match="format differs"):
        s.send(Frame(make_frames(1, w, h, 10)[0], w, h, 10).desc)
    assert s.counts() == (1, 0, 0, 0)               # nothing launched yet: host frames are uploaded at launch
    for k in range(1, 8):
        s.send(Frame(fr[k], w, h, 8, mem=MEMS[k % 3]).desc)
    s.finish()
    with pytest.raises(ab.AmtkError, match=r"closed \(finished\)"):
        s.send(Frame(fr[0], w, h, 8).desc)
    with pytest.raises(ab.AmtkError, match=r"closed \(finished\)"):
        s.finish()
    assert np.array_equal(s.recv(100), exp)
    s.close()


def test_first_frame_thresholds_for_its_sample_size(ctx):
    """th_move 200 is refused for 1-byte samples when the first frame comes (with comb_frames' message) and fixes no
    format; a 2-byte frame then starts the stream, exact."""
    w, h, B = 256, 160, 4
    prm = params(th_move_y=200, th_move_c=300)
    s = ctx.comb_stream(prm, B)
    f8 = make_frames(1, w, h, 8)
    with pytest.raises(ab.AmtkError, match=r"th_move must be in \[1,128\]"):
        s.send(Frame(f8[0], w, h, 8).desc)
    assert s.counts() == (0, 0, 0, 0)
    fr = make_frames(9, w, h, 16, seed=2)
    for k in range(9):
        s.send(Frame(fr[k], w, h, 16, mem=MEMS[k % 3]).desc)
    s.finish()
    assert np.array_equal(s.recv(9), resident(ctx, fr, w, h, 16, prm))
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# lifetime and sharing the context
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stage", ["created", "mid_batch", "launched", "finished"])
def test_destroy_at_every_stage(ctx, stage):
    w, h, B = 256, 160, 4
    fr = make_frames(2 * B + 2, w, h, 8)
    s = ctx.comb_stream(None, B)
    n = {"created": 0, "mid_batch": 2, "launched": 2 * B + 1, "finished": 2 * B + 2}[stage]
    for k in range(n):
        s.send(Frame(fr[k], w, h, 8, mem=MEMS[k % 3]).desc)
    if stage == "finished":
        s.finish()
        assert len(s.recv(3)) == 3             # rows left
    s.close()
    assert np.array_equal(run(ctx, fr, w, h, 8, B)[0], resident(ctx, fr, w, h, 8, None))


def test_two_streams_interleaved(ctx):
    w, h = 256, 160
    a, b = make_frames(23, w, h, 8, seed=21), make_frames(17, w, h, 10, seed=22)
    sa, sb = ctx.comb_stream(None, 4), ctx.comb_stream(params(th_move_y=7), 3)
    ga, gb = [], []
    for k in range(max(len(a), len(b))):
        if k < len(a):
            sa.send(Frame(a[k], w, h, 8, mem=MEMS[k % 3]).desc)
            ga.append(sa.recv(100))
        if k < len(b):
            sb.send(Frame(b[k], w, h, 10, mem=MEMS[(k + 1) % 3]).desc)
            gb.append(sb.recv(100))
    sa.finish(); sb.finish()
    ga.append(sa.recv(100)); gb.append(sb.recv(100))
    assert np.array_equal(np.concatenate(ga), resident(ctx, a, w, h, 8, None))
    assert np.array_equal(np.concatenate(gb), resident(ctx, b, w, h, 10, params(th_move_y=7)))
    sa.close(); sb.close()


@pytest.mark.parametrize("bits", [8, 10])
def test_interleaved_with_other_comb_calls(ctx, bits):
    """comb_frames and scan_comb_frames on the stream's context between its batches share its cached plan and the band
    form's watchdog record: all results stay exact."""
    w, h, B = 256, 160, 5
    fr = make_frames(3 * B + 2, w, h, bits, seed=31)
    other = make_frames(12, w, h, 8, seed=32)
    exp, exp_other = resident(ctx, fr, w, h, bits, None), resident(ctx, other, w, h, 8, None)
    lg = synth.make_logo(64, 64, seed=3)
    logo = ab.Logo.create(lg["data"], 64, 64, w, h, 40, 24).deint().create_mask(0.35)
    t = torch.from_numpy(other).cuda()
    oc = ab.yv12_clip(t, w, h, other.shape[0], True)
    ref_scores = ctx.scan_frames(oc, [logo]).cpu().numpy()
    s = ctx.comb_stream(None, B)
    got = []
    for k in range(fr.shape[0]):
        s.send(Frame(fr[k], w, h, bits, mem=MEMS[k % 3]).desc)
        if k % 3 == 1:
            assert np.array_equal(ctx.comb_frames(oc).cpu().numpy(), exp_other)
        if k % 4 == 2:
            sc, cn = ctx.scan_comb_frames(oc, [logo])
            assert np.array_equal(cn.cpu().numpy(), exp_other) and np.array_equal(sc.cpu().numpy(), ref_scores)
        got.append(s.recv(2))
    s.finish()
    assert np.array_equal(ctx.comb_frames(oc).cpu().numpy(), exp_other)
    got.append(s.recv(100))
    assert np.array_equal(np.concatenate(got), exp)
    s.close()

