"""Logo items of the fused step sized to the ring that runs, and launches that check the previous launch's watchdog record
after enqueueing their own work.

The tall band form's ring holds many more frames per logo item than the 512 x 4R ring (scan_item in
csrc/logo_kernels.cuh), so frame ranges, logo sizes and call sequences move item boundaries and the shared-memory plan.
Every case compares the scores bit for bit with the reference's ScanFrame and the counters with the combing spec, using
the helpers of test_gpu_fused_step.py."""
import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from test_gpu_fused_step import _check, _logo, _refs, _run, budget_pair
from test_gpu_logo_plans import _bits_of, make_clip_frames, to_device

W, H = 320, 120


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("frame0,n", [(0, 1), (0, 8), (0, 15), (0, 16), (0, 17), (3, 31), (2, 33), (0, 47), (5, 42)])
def test_item_boundaries(ctx, oracle, frame0, n):
    """Frame ranges that end mid-item, one short of an item, on an item and one past it, and ragged tails."""
    packed = make_clip_frames(frame0 + n, W, H, 8, seed=100 + frame0 + n)
    _check(ctx, oracle, packed, W, H, (64, 64, 200, 40, 21), frame0=frame0, n=n)


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("spec", [(61, 45, 64, 20, 22), (37, 29, 3, 5, 23), (63, 63, 250, 50, 24)])
def test_odd_logo_sizes(ctx, oracle, spec):
    """Logo sizes whose pixel and feature counts are not multiples of 4."""
    packed = make_clip_frames(35, W, H, 8, seed=spec[-1])
    _check(ctx, oracle, packed, W, H, spec)


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("band", ["2", "1"])
def test_near_budget(native_lib, oracle, monkeypatch, band):
    """The largest logo that runs fused takes a small item in the tall ring and the smallest plan in the 4R ring."""
    monkeypatch.setenv("AMTK_COMB_WS_BAND", band)
    c = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    try:
        under, _ = budget_pair()
        packed = make_clip_frames(21, W, H, 8, seed=25)
        _check(c, oracle, packed, W, H, (96, under, 8, 2, under), fused=True)
    finally:
        c.close()


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_back_to_back_then_host_outputs(native_lib, oracle):
    """A long run of device-output fused calls, then host-output fused and comb-only calls on the same context: one launch
    per call, exact results throughout."""
    c = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    try:
        n = 40
        packed = make_clip_frames(n, W, H, 8, seed=26)
        buf = to_device(packed)
        clip = ab.yv12_clip(buf, W, H, n, True)
        data, P = _logo(64, 64, W, H, 120, 30, 27)
        rs, rc = _refs(oracle, packed, W, H, data, 64, 64, 120, 30, 0, n)
        prm = ab.default_comb_params()
        outs = []
        l0 = c.launches
        for _ in range(50):
            outs.append(c.scan_comb_frames(clip, [P], prm))
        assert c.launches - l0 == 50
        for s, cnt in outs:
            assert np.array_equal(_bits_of(s.cpu().numpy()[:, 0]), _bits_of(rs))
            assert np.array_equal(cnt.cpu().numpy(), rc)
        hclip = ab.yv12_clip(packed, W, H, n, False)
        for _ in range(3):
            s, cnt = _run(c, hclip, P, 0, n, None)
            assert np.array_equal(_bits_of(s), _bits_of(rs))
            assert np.array_equal(cnt, rc)
            got = c.comb_frames(clip, prm).cpu().numpy()
            assert np.array_equal(got, rc)
    finally:
        c.close()
