"""How host-resident clips are cut into chunks and staged into HBM, pinned call by call.

Every entry point that accepts host frames moves them through the context's two staging buffers in chunks.  The size of
a chunk decides how many bytes cross PCIe and how many kernels run, and `bench.py` reports both.  This module restates
the chunk rules and checks `last_h2d_bytes`, the launch count of every call and the comb kernel's timed launches against
them, at a 1 MB staging budget (many chunks) and at the default one.  Every expected value is computed here from the
rules, never read back from the library:

- whole frames (comb, fused step, full-frame ScanFrame): `per = max(1, min(n, budget // fs))`, one less when a
  previous frame is needed and `per > 1`; chunk [lo, hi) stages frames [lo-1, hi) (or [lo, hi) at frame 0);
- logo rectangle (ScanFrame, AMTAnalyzeLogo, fade sweep, LogoScan, erase): the rectangle's columns widened to multiples
  of 16 << log_uvx bytes and its rows to whole chroma rows; `per = max(1, min(n, budget // roi_fs))` where roi_fs is one
  compact staged frame; `last_h2d_bytes` counts the rectangle's payload bytes;
- temporal noise reduction: `per = max(1, min(n, budget // sfs - 2d))` for host sources, further capped by
  `budget // dfs` for host destinations; chunk [lo, hi) stages frames [lo-d, hi+d) clamped to the clip.

Calls on device clips stage nothing and leave `last_h2d_bytes` as the previous call left it.
"""
import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth

pytestmark = pytest.mark.gpu

DEFAULT_MB = 256
W, H, N = 512, 256, 160                 # 192 KB frames: five per MB
FS = W * H * 3 // 2
BUDGETS = [1, None]                     # AMTK_STAGE_MB (None: the default budget)


def _budget(mb):
    return (DEFAULT_MB if mb is None else mb) << 20


def _chunks(frame0, n, per):
    return [(lo, min(frame0 + n, lo + per)) for lo in range(frame0, frame0 + n, per)]


def full_frame_plan(frame0, n, fs, budget, need_prev):
    """(chunks, staged bytes) of whole-frame staging."""
    per = max(1, min(n, budget // fs))
    if need_prev and per > 1:
        per -= 1
    ch = _chunks(frame0, n, per)
    staged = sum((hi - (lo - 1 if need_prev and lo > 0 else lo)) * fs for lo, hi in ch)
    return ch, staged


def roi_plan(frame0, n, budget, rx, ry, rw, rh, chroma, bps=1, lx=1, ly=1, width=W, height=H):
    """(chunks, payload bytes) of logo-rectangle staging on a packed 4:2:0 clip."""
    pitch_y, pitch_uv = width * bps, (width >> lx) * bps
    A = 16 << lx
    up = lambda v, m: -(-v // m) * m
    xb0 = (rx * bps) // A * A
    xb1 = min(pitch_y, up((rx + rw) * bps, A))
    y0 = ry & ~((1 << ly) - 1)
    y1 = min(height, up(ry + rh, 1 << ly))
    rows_y = y1 - y0
    rows_c = rows_y >> ly if chroma else 0
    span_y = xb1 - xb0
    span_c = min(pitch_uv - (xb0 >> lx), span_y >> lx)
    cp = up(span_y, A)
    rows_c_as_y = up((cp >> lx) * rows_c, cp) // cp
    roi_fs = cp * rows_y + (2 * cp * rows_c_as_y if chroma else 0)
    per = max(1, min(n, budget // roi_fs))
    payload = n * (span_y * rows_y + (2 * span_c * rows_c if chroma else 0))
    return _chunks(frame0, n, per), payload


def tnr_plan(frame0, n, nclip, d, sfs, dfs, src_host, dst_host, budget):
    per = n
    if src_host:
        per = max(1, min(per, budget // sfs - 2 * d))
    if dst_host:
        per = max(1, min(per, budget // dfs))
    ch = _chunks(frame0, n, per)
    staged = sum((min(nclip, hi + d) - max(0, lo - d)) * sfs for lo, hi in ch) if src_host else None
    return ch, staged


def eval_launches(chunks, nfades, logo):
    """Kernels of one logo evaluation: a scores kernel and a sum kernel per batch of frames (96 MB of scores)."""
    count_pad = max(32, (logo.info().count + 31) & ~31)
    batch = max(1, (96 << 20) // (nfades * count_pad * 4))
    return sum(2 * -(-(hi - lo) // batch) for lo, hi in chunks)


@pytest.fixture(scope="module")
def clips():
    lg = synth.make_logo(64, 64)
    dev = synth.make_frames(0, N, W, H, device="cuda", logo=lg, imgx=400, imgy=40, logo_period=20)
    host = dev.cpu().numpy()
    return lg, dev, host


def _measure(ctx, call):
    l0 = ctx.launches
    call()
    torch.cuda.synchronize()
    return ctx.last_h2d_bytes, ctx.launches - l0


def _set_budget(monkeypatch, mb):
    if mb is None:
        monkeypatch.delenv("AMTK_STAGE_MB", raising=False)
    else:
        monkeypatch.setenv("AMTK_STAGE_MB", str(mb))


@pytest.mark.parametrize("mb", BUDGETS)
def test_whole_frame_staging(ctx, clips, monkeypatch, mb):
    """comb_frames, the fused step and full-frame ScanFrame: staged bytes (halo frames included) and launches."""
    _set_budget(monkeypatch, mb)
    lg, dev, host = clips
    hclip, dclip = ab.yv12_clip(host, W, H, N, False), ab.yv12_clip(dev, W, H, N, True)
    logo = ab.Logo.create(lg["data"], 64, 64, W, H, 400, 40).deint().create_mask(0.35)
    for frame0, n in ((0, N), (7, 101), (N - 1, 1)):
        ch, staged = full_frame_plan(frame0, n, FS, _budget(mb), True)
        assert _measure(ctx, lambda: ctx.comb_frames(hclip, frame0=frame0, nframes=n)) == (staged, len(ch))
        # one launch per chunk: the logo is evaluated in work items of the comb kernel
        assert _measure(ctx, lambda: ctx.scan_comb_frames(hclip, [logo], frame0=frame0, nframes=n)) == (staged, len(ch))
        ch, staged = full_frame_plan(frame0, n, FS, _budget(mb), False)
        assert _measure(ctx, lambda: ctx.scan_frames(hclip, [logo], frame0, n, pitch_elems_override=W)) == \
            (staged, eval_launches(ch, 2, logo))
        # device clips stage nothing and leave the count alone
        assert _measure(ctx, lambda: ctx.comb_frames(dclip, frame0=frame0, nframes=n)) == (staged, 1)


@pytest.mark.parametrize("mb", BUDGETS)
def test_roi_staging(ctx, clips, monkeypatch, mb):
    """ScanFrame, AMTAnalyzeLogo, the fade sweep, LogoScan and erase on host frames: rectangle payload bytes and launches."""
    _set_budget(monkeypatch, mb)
    lg, dev, host = clips
    hclip = ab.yv12_clip(host, W, H, N, False)
    budget = _budget(mb)
    # ScanFrame with two logos: the staged rectangle is their bounding box (most of the frame: several chunks at 1 MB)
    lw, lh = 64, 48
    raw_a = ab.Logo.create(synth.make_logo(lw, lh, seed=3)["data"], lw, lh, W, H, 18, 10)
    raw_b = ab.Logo.create(synth.make_logo(lw, lh, seed=4)["data"], lw, lh, W, H, 430, 190)
    la, lb = raw_a.deint().create_mask(0.35), raw_b.deint().create_mask(0.35)
    for frame0, n in ((0, N), (5, 77)):
        ch, payload = roi_plan(frame0, n, budget, 18, 10, 430 + lw - 18, 190 + lh - 10, False)
        assert _measure(ctx, lambda: ctx.scan_frames(hclip, [la, lb], frame0, n)) == \
            (payload, eval_launches(ch, 2, la) + eval_launches(ch, 2, lb))
    # AMTAnalyzeLogo, the fade sweep and erase on one large logo at an odd position
    lw, lh, ix, iy = 128, 96, 37, 23
    data = synth.make_logo(lw, lh, seed=5)["data"]
    raw = ab.Logo.create(data, lw, lh, W, H, ix, iy)
    de, top, bot = raw.deint().create_mask(0.35), raw.field(0).create_mask(0.35), raw.field(1).create_mask(0.35)
    fades = np.arange(20, dtype=np.float32) * np.float32(0.1)
    for frame0, n in ((0, N), (3, 8), (11, 131)):      # 8 frames: the GetFrame-sized call, three evaluations side by side
        ch, payload = roi_plan(frame0, n, budget, ix, iy, lw, lh, False)
        want = eval_launches(ch, 11, de) + eval_launches(ch, 11, top) + eval_launches(ch, 11, bot)
        assert _measure(ctx, lambda: ctx.analyze_frames(hclip, de, top, bot, frame0, n)) == (payload, want)
        assert _measure(ctx, lambda: ctx.eval_fades(hclip, de, fades, frame0, n)) == (payload, eval_launches(ch, 20, de))
        ch, payload = roi_plan(frame0, n, budget, ix, iy, lw, lh, True)
        work = host.copy()
        fd = np.stack([np.linspace(0, 1, n), np.linspace(1, 0, n)], axis=1).astype(np.float32)
        assert _measure(ctx, lambda: ctx.erase_logo(ab.yv12_clip(work, W, H, N, False), raw, fd, frame0, n)) == \
            (payload, len(ch))
        assert not np.array_equal(work[frame0:frame0 + n], host[frame0:frame0 + n])
    # LogoScan::AddFrame on a rectangle at odd coordinates
    sx, sy, sw, sh = 146, 34, 96, 72
    acc = ctx.logo_scan(sw, sh, 12)
    for frame0, n in ((0, N), (9, 40)):
        ch, payload = roi_plan(frame0, n, budget, sx, sy, sw, sh, True)
        assert _measure(ctx, lambda: acc.add_frames(hclip, sx, sy, frame0, n)) == (payload, 2 * len(ch))


@pytest.mark.parametrize("mb", BUDGETS)
def test_tnr_staging(ctx, monkeypatch, mb):
    """tnr_frames in the three pairings that touch host memory: staged bytes (window frames included) and launches."""
    _set_budget(monkeypatch, mb)
    w, h, nclip = 256, 128, 40
    fs = w * h * 3 // 2
    src = synth.noisy_clip(21, nclip, w, h)
    dsrc = torch.from_numpy(src).cuda()
    prm = ab.tnr_params(3, 1)
    budget = _budget(mb)
    for frame0, n in ((0, nclip), (6, 29)):
        for src_host, dst_host in ((True, False), (False, True), (True, True)):
            dst = np.zeros_like(src) if dst_host else torch.zeros_like(dsrc)
            s = ab.yv12_clip(src if src_host else dsrc, w, h, nclip, not src_host)
            dd = ab.yv12_clip(dst, w, h, nclip, not dst_host)
            ch, staged = tnr_plan(frame0, n, nclip, 3, fs, fs, src_host, dst_host, budget)
            before = ctx.last_h2d_bytes
            got = _measure(ctx, lambda: ctx.tnr_frames(s, dd, prm, frame0, n, frame0))
            assert got == (staged if src_host else before, len(ch)), (src_host, dst_host)


@pytest.mark.parametrize("mb", BUDGETS)
def test_comb_kernel_timing(ctx, clips, monkeypatch, mb):
    """With kernel timing on, every comb launch is timed once: one for a device call, one per chunk for a host call."""
    _set_budget(monkeypatch, mb)
    _, dev, host = clips
    ctx.set_kernel_timing(True)
    try:
        ctx.kernel_timing(reset=True)
        ctx.comb_frames(ab.yv12_clip(dev, W, H, N, True))
        assert ctx.kernel_timing(reset=True)[1] == 1
        ch, _ = full_frame_plan(0, N, FS, _budget(mb), True)
        ctx.comb_frames(ab.yv12_clip(host, W, H, N, False))
        ms, launches = ctx.kernel_timing(reset=True)
        assert launches == len(ch) and ms > 0
    finally:
        ctx.set_kernel_timing(False)
