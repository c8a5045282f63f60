"""The serial logo evaluation (logo_scores_kernel, then logo_sum_bulk_kernel or logo_sum_kernel) and the (0, -1) pairs of
logos that do not match the frame (fill_pairs_kernel), into outputs filled beforehand with a NaN no kernel computes
(0x7FC00001): feature counts at every remainder of the ordered sums' four-wide steps, several logos per call with an absent
and a mismatched one between them, and AMTAnalyzeLogo records, whose sums are taken as absolute values, compared bit for
bit with the reference (the C port where oracle/_ref is absent).  The mutants of tools/mutants.py that a test is there to
kill are named in its docstring."""
import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from test_gpu_fused_item_plans import count_case
from test_gpu_fused_step import MASKRATIO, _logo
from test_gpu_logo_plans import Oracle, _bits_of, make_clip_frames, to_device, y_planes

pytestmark = pytest.mark.gpu

SCORE_POISON = 0x7FC00001


def poisoned(*shape):
    return torch.full(shape, SCORE_POISON, dtype=torch.int32, device="cuda").view(torch.float32)


@pytest.mark.timeout(900)
def test_several_logos_every_count_remainder(ctx, oracle):
    """Logos whose feature counts leave 1, 2 and 3 scores after the four-wide steps, an absent logo and one made for another
    frame size, in one amtk_logo_scan_frames call.  Kills bulk_tail_drop, fill_pairs_swap, scores_pair_bin."""
    W, H, n = 320, 120, 9
    packed = make_clip_frames(n, W, H, 8, seed=31)
    Y = y_planes(packed, W, H)
    logos, want = [], []
    for r, (x, y) in zip((1, 2, 3), ((5, 3), (150, 40), (260, 70))):
        w, h, c = count_case(lambda c, r=r: c % 4 == r)
        data, P = _logo(w, h, W, H, x, y, h)
        assert P.info().count == c
        O = Oracle(oracle, data, w, h, W, H, x, y)
        de = O.deint(MASKRATIO)
        logos.append(P)
        want.append(np.stack([O.scan(de, Y[i], 255.0) for i in range(1, n)]))
    _, other = _logo(32, 16, W + 16, H, 4, 4, 16)               # made for 336 x 120 frames: no match
    filler = np.tile(np.array([0.0, -1.0], np.float32), (n - 1, 1))
    logos = [logos[0], None, logos[1], other, logos[2]]
    want = [want[0], filler, want[1], filler, want[2]]
    buf = to_device(packed)
    clip = ab.yv12_clip(buf, W, H, n, True)
    out = poisoned(n - 1, len(logos), 2)
    ctx.scan_frames(clip, logos, 1, n - 1, out=out)
    got = out.cpu().numpy()
    for k, wk in enumerate(want):
        bad = np.argwhere(_bits_of(got[:, k]) != _bits_of(wk))
        assert bad.size == 0, (k, bad[:6].tolist())


@pytest.mark.timeout(900)
@pytest.mark.parametrize("r", [0, 1, 3])
def test_analyze_records_poisoned(ctx, oracle, r):
    """AMTAnalyzeLogo's 33 values per frame (fade scores as absolute values) for a logo whose feature count leaves r after
    the four-wide steps, from frame 2 on.  Kills bulk_take_abs, bulk_tail_drop, scores_pair_bin."""
    W, H, n = 256, 96, 8
    w, h, c = count_case(lambda c: c % 4 == r and c > 200)
    x, y = 40, 20
    packed = make_clip_frames(n, W, H, 8, seed=40 + r)
    data, _ = _logo(w, h, W, H, x, y, h)
    raw = ab.Logo.create(data, w, h, W, H, x, y)
    de, top, bot = raw.deint().create_mask(MASKRATIO), raw.field(0).create_mask(MASKRATIO), raw.field(1).create_mask(MASKRATIO)
    assert de.info().count == c
    buf = to_device(packed)
    clip = ab.yv12_clip(buf, W, H, n, True)
    out = poisoned(n - 2, 33)
    ctx.analyze_frames(clip, de, top, bot, 2, n - 2, out=out)
    got = out.cpu().numpy()
    O = Oracle(oracle, data, w, h, W, H, x, y)
    ode = O.deint(MASKRATIO)
    ot, ob = O.fields(MASKRATIO)
    Y = y_planes(packed, W, H)
    want = np.stack([O.analyze(ode, ot, ob, Y[i], 255.0) for i in range(2, n)])
    bad = np.argwhere(_bits_of(got) != _bits_of(want))
    assert bad.size == 0, bad[:6].tolist()
