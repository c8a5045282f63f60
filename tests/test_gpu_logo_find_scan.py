"""The logo finder on synthetic recordings (synth.make_frames: interlaced, telecine and flat content with semi-transparent
logos that fade in and out, so each is present in about 60 % of the frames): the rectangles it finds, and the logo that
amtk_scan_logo makes from the best one, which must tell logo-on from logo-off frames under amtk_logo_scan_frames."""

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth

pytestmark = pytest.mark.gpu

W, H = 1920, 1080
LOGO = synth.make_logo(64, 64, seed=1)
CHUNK = 100


def alpha_box(x, y, logo=LOGO):
    """(x, y, w, h) of the logo's non-zero alpha at (x, y)."""
    ys, xs = np.nonzero(logo["alpha8"])
    return x + xs.min(), y + ys.min(), xs.max() - xs.min() + 1, ys.max() - ys.min() + 1


def bounded(rect, box, slack):
    """rect contains box and exceeds it by at most slack on each side."""
    rx, ry, rw, rh = rect
    x, y, w, h = box
    return (rx <= x and ry <= y and rx + rw >= x + w and ry + rh >= y + h and
            x - rx <= slack and y - ry <= slack and rx + rw - (x + w) <= slack and ry + rh - (y + h) <= slack)


def composite_y(fr, n0, spots, logo=LOGO, period=200):
    """Composites logo at every (x, y) of spots into the Y planes of packed frames fr (uint8, device) as make_frames does,
    with the logo_fade256 schedule."""
    cnt = fr.shape[0]
    Y = fr[:, :W * H].view(cnt, H, W)
    n = torch.arange(n0, n0 + cnt, device=fr.device, dtype=torch.int64).view(cnt, 1, 1)
    al = torch.from_numpy(logo["alpha8"].astype(np.int64)).to(fr.device)
    lh, lw = al.shape
    a = (al.view(1, lh, lw) * synth.logo_fade256(n, period)) >> 8
    for x, y in spots:
        roi = Y[:, y:y + lh, x:x + lw].to(torch.int64)
        Y[:, y:y + lh, x:x + lw] = ((roi * (256 - a) + a * logo["L8"] + 128) >> 8).to(torch.uint8)


def find(ctx, mode, nframes=1800, logo_at=None, spots=(), pillar=0):
    fd = ctx.logo_find()
    for n0 in range(0, nframes, CHUNK):
        c = min(CHUNK, nframes - n0)
        kw = dict(logo=LOGO, imgx=logo_at[0], imgy=logo_at[1]) if logo_at else {}
        fr = synth.make_frames(n0, c, W, H, device="cuda", mode=mode, **kw)
        if spots:
            composite_y(fr, n0, spots)
        if pillar:
            Y = fr[:, :W * H].view(c, H, W)
            Y[:, :, :pillar] = 16
            Y[:, :, W - pillar:] = 16
        fd.add_frames(ab.yv12_clip(fr, W, H, c, True))
    rects, scores = fd.rects()
    s1, s2, n = fd.sums()
    assert n == nframes
    p = ab.default_logo_find_params()
    return [tuple(r) for r in rects.tolist()], scores, p.margin + p.block


@pytest.mark.parametrize("mode", ["interlaced", "telecine", "flat"])
def test_one_logo(ctx, mode):
    rects, scores, slack = find(ctx, mode, logo_at=(1700, 60))
    assert rects, "no rectangle found"
    assert bounded(rects[0], alpha_box(1700, 60), slack), (rects, alpha_box(1700, 60))


@pytest.mark.parametrize("mode", ["interlaced", "telecine", "flat"])
def test_no_logo(ctx, mode):
    rects, _, _ = find(ctx, mode)
    assert rects == []


def test_four_corner_logos(ctx):
    spots = [(40, 40), (W - 104, 40), (40, H - 104), (W - 104, H - 104)]
    rects, scores, slack = find(ctx, "interlaced", spots=spots)
    assert len(rects) == 4, rects
    for x, y in spots:
        assert sum(bounded(r, alpha_box(x, y), slack) for r in rects) == 1, (x, y, rects)


def test_pillarbox_bars_are_not_reported(ctx):
    rects, _, slack = find(ctx, "interlaced", logo_at=(1700, 60), pillar=140)
    assert len(rects) == 1 and bounded(rects[0], alpha_box(1700, 60), slack), rects


# ---------------------------------------------------------------------------------------------------------------------
# into ScanLogo: the flat clip of tests/test_gpu_scan_logo_stream.py, with the 64 x 64 logo
# ---------------------------------------------------------------------------------------------------------------------
SW, SH, SX, SY, THY, SEED = 320, 192, 200, 64, 12, 0x5EED0005


def flat_fade(n, seed=SEED):
    """The logo's fade in make_frames' flat mode (256 or 0) per frame index."""
    n = np.asarray(n, np.int64)
    return np.where((synth._hash32(n, n * 0 + 13, n * 0, 6, seed) & 3) != 0, 256, 0)


def test_rectangle_into_scan_logo(ctx, tmp_path):
    N = 450
    fr = synth.make_frames(0, N, SW, SH, seed=SEED, device="cuda", mode="flat", logo=LOGO, imgx=SX, imgy=SY)
    clip = ab.yv12_clip(fr, SW, SH, N, True)
    fd = ctx.logo_find()
    fd.add_frames(clip)
    rects, _ = fd.rects()
    p = ab.default_logo_find_params()
    assert len(rects) >= 1 and bounded(tuple(rects[0]), alpha_box(SX, SY), p.margin + p.block), rects
    x, y, w, h = (int(v) for v in rects[0])
    dst = str(tmp_path / "found.lgd")
    ctx.scan_logo(clip, dst, x, y, w, h, THY, N, service_id=3)
    with open(dst, "rb") as f:
        raw = f.read()
    logo = ab.Logo.load(dst)
    info = logo.info()
    assert (info.imgx, info.imgy, info.w, info.h) == (x, y, w, h)
    assert (info.imgw, info.imgh) == (SW, SH) and len(raw) > 540
    deint = logo.deint().create_mask(0.35)
    scores = ctx.scan_frames(clip, [deint]).cpu().numpy()[:, 0, 0]
    fade = flat_fade(np.arange(N))
    on, off = scores[fade == 256], scores[fade == 0]
    assert len(on) and len(off)
    assert on.min() > off.max(), (on.min(), off.max())
