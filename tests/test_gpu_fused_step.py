"""The fused step (amtk_scan_comb_frames) with the logo evaluation run as work items of the band-form comb kernel.

On 8-bit clips whose combing pass runs the band form, one logo's LogoFrame::ScanFrame scores are computed by the comb
kernel itself, in logo items spread through its work queue (csrc/comb_stream.cuh, scan_item in csrc/logo_kernels.cuh): one
launch per window instead of three.  Every case here compares the scores bit for bit with the reference's ScanFrame (or
the C port tests/test_oracle.py pins to it) and the counters with the combing spec, on frame sizes, logo shapes and
positions, frame ranges, layouts and call sequences that move the item list, the shared-memory plan and the cached plan.
Calls that are not eligible (logos too large for the ring, several logos, layouts without TMA) take the serial path and
must give the same results."""
import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth
from test_gpu_erase import logo_data
from test_gpu_frame_layouts import Layout
from test_gpu_logo_plans import Oracle, _bits_of, make_clip_frames, to_device, y_planes
from test_gpu_plane_order import VFirst

MASKRATIO = 0.35


def _logo(w, h, W, H, imgx, imgy, seed):
    data = synth.make_logo(w, h, seed=seed)["data"] if w % 2 == 0 and h % 2 == 0 else logo_data(w, h, seed)
    return data, ab.Logo.create(data, w, h, W, H, imgx, imgy).deint().create_mask(MASKRATIO)


def budget_pair(W=320, H=120, w=96):
    """(h_under, h_over): logo heights of a w-wide logo whose item just fits in the ring, and the next that does not
    (the plan restated in test_gpu_fused_item_plans.py)."""
    from test_gpu_fused_item_plans import plan
    prev = None
    for h in range(40, H - 4):
        _, P = _logo(w, h, W, H, 8, 2, seed=h)
        fused = plan(W, H, w, h, P.info().count) != "serial"
        if prev is not None and prev[1] and not fused:
            return prev[0], h
        prev = (h, fused)
    return None


def test_budget_cases_straddle_the_ring(native_lib):
    """The just-under / just-over logos of test_budget really sit on both sides of the ring budget, and the headline
    logo (64x64 on 1080p frames) takes 13 frames per item in the tall ring and two in the 512 x 4R ring."""
    from test_gpu_fused_item_plans import plan
    assert budget_pair() is not None
    _, P = _logo(64, 64, 1920, 1080, 1700, 60, seed=1)
    assert plan(1920, 1080, 64, 64, P.info().count).F == 13
    assert plan(1920, 1080, 64, 64, P.info().count, {"AMTK_COMB_WS_BAND": "1"}).F == 2


# ---- GPU side ------------------------------------------------------------------------------------------------------------
def _refs(oracle, packed, W, H, data, w, h, imgx, imgy, frame0, n):
    Y = y_planes(packed, W, H)
    ysz, csz = W * H, (W // 2) * (H // 2)
    U = packed[:, ysz:ysz + csz].reshape(-1, H // 2, W // 2)
    V = packed[:, ysz + csz:].reshape(-1, H // 2, W // 2)
    O = Oracle(oracle, data, w, h, W, H, imgx, imgy)
    ode = O.deint(MASKRATIO)
    scores = np.stack([O.scan(ode, Y[i], 255.0) for i in range(frame0, frame0 + n)])
    counts = oracle.or_comb_clip(Y, U, V, ab.default_comb_params().as_list())[frame0:frame0 + n]
    return scores, counts


def _run(c, clip, P, frame0, n, fused):
    l0 = c.launches
    s, cnt = c.scan_comb_frames(clip, [P], ab.default_comb_params(), frame0=frame0, nframes=n)
    s = s.cpu().numpy() if isinstance(s, torch.Tensor) else np.asarray(s)
    cnt = cnt.cpu().numpy() if isinstance(cnt, torch.Tensor) else np.asarray(cnt)
    if fused is not None:
        assert (c.launches - l0 == 1) == fused, (c.launches - l0, fused)
    return s[:, 0], cnt


def _check(c, oracle, packed, W, H, spec, frame0=0, n=None, fused=True, clip=None):
    w, h, imgx, imgy, seed = spec
    n = packed.shape[0] - frame0 if n is None else n
    data, P = _logo(w, h, W, H, imgx, imgy, seed)
    if clip is None:
        buf = to_device(packed)
        clip = ab.yv12_clip(buf, W, H, packed.shape[0], True)
    s, cnt = _run(c, clip, P, frame0, n, fused)
    rs, rc = _refs(oracle, packed, W, H, data, w, h, imgx, imgy, frame0, n)
    assert np.array_equal(_bits_of(s), _bits_of(rs)), (W, H, spec, frame0, n)
    assert np.array_equal(cnt, rc), (W, H, spec, frame0, n)


# (W, H, n, (logo w, h, imgx, imgy, seed)): the headline geometry, 1440x1080, ragged widths, non-64 and odd-height logos,
# logos touching every frame edge
CASES = {
    "1080p_1700_60": (1920, 1080, 40, (64, 64, 1700, 60, 1)),
    "1440x1080": (1440, 1080, 24, (64, 64, 1300, 40, 2)),
    "1952x136_right": (1952, 136, 40, (64, 64, 1952 - 64, 30, 3)),
    "320x120_48x40": (320, 120, 40, (48, 40, 101, 30, 4)),
    "320x120_odd": (320, 120, 40, (61, 45, 64, 20, 5)),
    "320x120_topleft": (320, 120, 30, (40, 32, 0, 0, 6)),
    "320x120_bottomright": (320, 120, 30, (40, 32, 280, 88, 7)),
    "320x120_bottomleft": (320, 120, 30, (33, 27, 0, 93, 8)),
    "320x120_topright": (320, 120, 30, (35, 30, 285, 0, 9)),
}


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", sorted(CASES))
def test_shapes(ctx, oracle, name):
    W, H, n, spec = CASES[name]
    packed = make_clip_frames(n, W, H, 8, seed=len(name))
    _check(ctx, oracle, packed, W, H, spec)


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_budget(ctx, oracle):
    """The largest logo whose item fits in the ring runs fused; the next one up takes the serial path."""
    under, over = budget_pair()
    W, H = 320, 120
    packed = make_clip_frames(12, W, H, 8, seed=11)
    _check(ctx, oracle, packed, W, H, (96, under, 8, 2, under), fused=True)
    _check(ctx, oracle, packed, W, H, (96, over, 8, 2, over), fused=False)


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("frame0,n", [(0, 1), (7, 1), (0, 2), (5, 2), (17, 3), (3, 37), (1, 39)])
def test_frame_ranges(ctx, oracle, frame0, n):
    W, H = 320, 120
    packed = make_clip_frames(40, W, H, 8, seed=frame0 + 10 * n)
    _check(ctx, oracle, packed, W, H, (64, 64, 200, 40, 12), frame0=frame0, n=n)


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("kind", ["vfirst_packed", "vfirst_padded", "padded", "row8"])
def test_layouts(ctx, oracle, kind):
    """V-first and padded layouts run fused; rows 8 bytes longer than a 16-byte multiple cannot be described by a tensor
    map and take the serial path (generic comb kernel)."""
    W, H, n = 320, 120, 30
    L = {"vfirst_packed": lambda: VFirst(W, H, 8, packed=True), "vfirst_padded": lambda: VFirst(W, H, 8, gap=32),
         "padded": lambda: Layout(W, H, 8, gap=16), "row8": lambda: Layout(W, H, 8, 328, 168)}[kind]()
    packed = make_clip_frames(n, W, H, 8, seed=21)
    buf = torch.from_numpy(L.pack(packed)).cuda()
    _check(ctx, oracle, packed, W, H, (48, 40, 250, 70, 13), clip=L.desc(buf, True), fused=kind != "row8")


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_host_clip_staged_windows(ctx, oracle, monkeypatch):
    """Host clips through 1 MiB staging buffers: many windows, each one fused launch."""
    monkeypatch.setenv("AMTK_STAGE_MB", "1")
    W, H, n = 320, 120, 60
    packed = make_clip_frames(n, W, H, 8, seed=31)
    clip = ab.yv12_clip(packed, W, H, n, False)
    for frame0, m in ((0, n), (9, 40), (59, 1)):
        _check(ctx, oracle, packed, W, H, (64, 64, 100, 30, 14), frame0=frame0, n=m, clip=clip, fused=None)


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_one_context_alternating_calls(native_lib, oracle):
    """Comb-only calls, fused calls and fused calls with another logo position and frame count on one context: each must
    build its own item list (the cached plan is keyed by the logo-item layout) and give exact results."""
    c = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    try:
        W, H, n = 320, 120, 40
        packed = make_clip_frames(n, W, H, 8, seed=41)
        buf = to_device(packed)
        clip = ab.yv12_clip(buf, W, H, n, True)
        _, rc = _refs(oracle, packed, W, H, *_logo(48, 40, W, H, 10, 10, 15)[:1], 48, 40, 10, 10, 0, n)
        for step in range(2):
            got = c.comb_frames(clip, ab.default_comb_params()).cpu().numpy()
            assert np.array_equal(got, rc), step
            _check(c, oracle, packed, W, H, (48, 40, 10, 10, 15), clip=clip)
            got = c.comb_frames(clip, ab.default_comb_params()).cpu().numpy()
            assert np.array_equal(got, rc), step
            _check(c, oracle, packed, W, H, (64, 64, 230, 50, 16), frame0=3, n=20, clip=clip)
            _check(c, oracle, packed, W, H, (61, 45, 0, 75, 17), frame0=0, n=n, clip=clip)
    finally:
        c.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_several_logos_take_the_serial_path(ctx, oracle):
    W, H, n = 320, 120, 20
    packed = make_clip_frames(n, W, H, 8, seed=51)
    buf = to_device(packed)
    clip = ab.yv12_clip(buf, W, H, n, True)
    specs = [(64, 64, 100, 30, 18), (48, 40, 10, 70, 19)]
    logos = [_logo(w, h, W, H, x, y, sd) for (w, h, x, y, sd) in specs]
    l0 = ctx.launches
    s, cnt = ctx.scan_comb_frames(clip, [P for _, P in logos], ab.default_comb_params())
    assert ctx.launches - l0 > 1
    for k, (w, h, x, y, sd) in enumerate(specs):
        rs, rc = _refs(oracle, packed, W, H, logos[k][0], w, h, x, y, 0, n)
        assert np.array_equal(_bits_of(s.cpu().numpy()[:, k]), _bits_of(rs)), k
        assert np.array_equal(cnt.cpu().numpy(), rc)
