"""The logo finder's 32-bit partial sums over long runs of one tile.  find_walk (csrc/find_kernels.cuh) keeps s1 and s2 of
8-bit samples, and s1 of 16-bit samples, in 32 bits while a CTA stays on one tile, and flushes them to the 64-bit totals
every kFindRunCap frames.  A CTA only stays that long on one tile when the picture is one tile and its share of the frames
is longer than the cap: at least 2^32 / 255^2 + 1 = 66 052 frames for 8-bit s2, 2^32 / 65535 + 1 = 65 538 for 16-bit s1.
The grid is at most four 512-thread CTAs per SM, so the clips below have that many frames per CTA of the largest grid
(about 8.9 GB at 8 bits and 132 SMs), every sample at the largest value, and the sums are known in closed form.  They are
skipped where the GPU has not that much free memory.  The mutants of tools/mutants.py that a test is there to kill are
named in its docstring."""
import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab

pytestmark = pytest.mark.gpu

MAX_CTAS_PER_SM = 2048 // 512                 # threads per SM / threads per finder CTA: the largest possible grid


def _frames_needed(bits):
    """Frames of a one-tile picture that give every CTA of the largest grid a run that wraps a 32-bit partial."""
    maxv = (1 << bits) - 1
    per_cta = (2 ** 32) // (maxv * maxv if bits == 8 else maxv) + 1
    return per_cta * MAX_CTAS_PER_SM * torch.cuda.get_device_properties(0).multi_processor_count


def _y_only_clip(buf, W, H, n, pitch, stride, bits):
    d = ab.ClipDesc()
    d.base = buf.data_ptr()
    d.frame_stride, d.off_u, d.off_v = stride, 0, 0
    d.width, d.height, d.pitch_y, d.pitch_uv = W, H, pitch, pitch // 2
    d.log_uvx = d.log_uvy = 1
    d.bytes_per_sample, d.bits_per_sample, d.num_frames = (1 if bits == 8 else 2), bits, n
    d.on_device = 1
    return d


# (bits, pitch bytes): 16 and 32 are multiples of 16 bytes (the TMA kernel), 17 is not (the plain-load kernel)
CASES = {"8bit_tma": (8, 16), "8bit_plain": (8, 17), "16bit_tma": (16, 32)}     # in this order


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("name", list(CASES))
def test_run_cap_on_one_tile(ctx, name):
    """16 x 16 Y-only clip, every sample at maxv, one amtk_logo_find_add_frames call: s1 = n * maxv and s2 = n * maxv^2 at
    every pixel.  Kills find_no_run_cap."""
    bits, pitch = CASES[name]
    W = H = 16
    maxv = (1 << bits) - 1
    n = _frames_needed(bits)
    stride = pitch * H
    need = n * stride
    free, _ = torch.cuda.mem_get_info()
    if free < need + (1 << 30):
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 1e9, free / 1e9))
    buf = torch.full((need,), 0xFF, dtype=torch.uint8, device="cuda")
    fd = ctx.logo_find()
    fd.add_frames(_y_only_clip(buf, W, H, n, pitch, stride, bits))
    s1, s2, got_n = fd.sums()
    del fd, buf
    torch.cuda.empty_cache()
    assert got_n == n
    assert (s1 == np.uint64(n * maxv)).all(), (int(s1.min()), int(s1.max()), n * maxv)
    assert (s2 == np.uint64(n * maxv * maxv)).all(), (int(s2.min()), int(s2.max()), n * maxv * maxv)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("bits", [8, 16])
def test_shares_split_tiles(ctx, bits):
    """A 300 x 70 picture (two tiles wide at 8 bits, three at 16, three tall) over more frames than CTAs, so most shares
    start and end inside a tile, against numpy in int64.  Kills find_share_begin, find_flush_last_column, find_widen16."""
    W, H = 300, 70
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 4 * sms + 7
    rng = np.random.default_rng(bits)
    maxv = (1 << bits) - 1
    Y = rng.integers(0, maxv + 1, (n, H, W), dtype=np.int64)
    Y[::2, :, -1] = maxv                                       # the last column at its largest value on every other frame
    if bits == 16:
        Y[:8] = maxv                                           # 16-bit s2 partials of eight frames pass 2^32
    dt = np.uint8 if bits == 8 else np.uint16
    buf = torch.from_numpy(Y.astype(dt).reshape(n, -1).view(np.uint8)).cuda()
    bps = 1 if bits == 8 else 2
    fd = ctx.logo_find()
    fd.add_frames(_y_only_clip(buf, W, H, n, W * bps, W * H * bps, bits))
    s1, s2, got_n = fd.sums()
    assert got_n == n
    assert np.array_equal(s1.astype(np.int64), Y.sum(0))
    assert np.array_equal(s2.view(np.int64), (Y * Y).sum(0))
