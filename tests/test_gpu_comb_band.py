"""The band form of the 8-bit warp-stream kernel (comb_stream.cuh, ws_bands): four warps share one ring of 512-byte-wide
slots (the default for 8-bit clips; AMTK_COMB_WS_BAND=0 selects one 128-byte tile per warp instead).  Counters must equal
the spec oracle's bit for bit:
bands that end inside the plane (zero-filled right box, warps wholly right of the plane), planes narrower than one box,
edge rows, extreme thresholds, frame-range calls with a halo frame, 1440x1080, and host clips staged in small chunks."""
import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth

pytestmark = pytest.mark.gpu


def _band_ctx(monkeypatch, mode):
    monkeypatch.setenv("AMTK_COMB_WS_BAND", mode)
    c = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    monkeypatch.delenv("AMTK_COMB_WS_BAND")
    return c


@pytest.mark.timeout(900)
def test_band_form_is_bit_exact(oracle, monkeypatch):
    po = oracle
    c = _band_ctx(monkeypatch, "1")
    try:
        prm = ab.default_comb_params()
        prm.th_move_y, prm.th_shima_y, prm.th_lshima_y = 1, 1, 2047
        prm.th_move_c, prm.th_shima_c, prm.th_lshima_c = 128, 700, 701
        # widths: one partial box (160), exactly one box (256), a right box with one used column (640 -> 512 + 128),
        # 3.75 bands (1920), a 32-byte-wide chroma plane in a 512-byte band (64), 1952 = 3 bands + 416
        for (w, h, n) in ((160, 34, 3), (256, 62, 4), (640, 360, 9), (1920, 64, 2), (64, 1100, 2), (1952, 36, 2), (352, 288, 23)):
            fr = synth.make_frames(3, n, w, h, device="cuda", mode="interlaced")
            clip = ab.yv12_clip(fr, w, h, n, True)
            out = c.comb_frames(clip, prm).cpu().numpy()
            Y, U, V = synth.split_planes(fr, w, h)
            ref = po.or_comb_clip(Y, U, V, prm.as_list())
            assert np.array_equal(out, ref), (w, h, np.argwhere(out != ref)[:5])
            if n > 4:
                part = np.concatenate([c.comb_frames(clip, prm, 0, 3).cpu().numpy(), c.comb_frames(clip, prm, 3, 1).cpu().numpy(),
                                       c.comb_frames(clip, prm, 4, n - 4).cpu().numpy()])
                assert np.array_equal(part, ref), ("ranges", w, h)
        # maximum response everywhere: alternating 0 / 255 rows
        w, h = 512, 128
        fr = torch.zeros((2, w * h * 3 // 2), dtype=torch.uint8, device="cuda")
        fr[:, : w * h].view(2, h, w)[:, 0::2, :] = 255
        p2 = ab.default_comb_params()
        p2.th_shima_y, p2.th_lshima_y = 1530, 1531
        out = c.comb_frames(ab.yv12_clip(fr, w, h, 2, True), p2).cpu().numpy()
        assert out[0, 1] + out[0, 4] == (h - 4) * w and out[0, 2] + out[0, 5] == 0 and out[:, 0].sum() == 0
        # 1440x1080, default thresholds
        w, h, n = 1440, 1080, 6
        fr = synth.make_frames(5, n, w, h, device="cuda", mode="telecine")
        prm = ab.default_comb_params()
        out = c.comb_frames(ab.yv12_clip(fr, w, h, n, True), prm).cpu().numpy()
        Y, U, V = synth.split_planes(fr, w, h)
        assert np.array_equal(out, po.or_comb_clip(Y, U, V, prm.as_list()))
    finally:
        c.close()


@pytest.mark.timeout(900)
def test_band_form_on_staged_host_chunks(oracle, monkeypatch):
    po = oracle
    c = _band_ctx(monkeypatch, "1")
    try:
        w, h, n = 640, 360, 17
        fr = synth.make_frames(0, n, w, h, device="cuda", mode="telecine")
        prm = ab.default_comb_params()
        Y, U, V = synth.split_planes(fr, w, h)
        ref = po.or_comb_clip(Y, U, V, prm.as_list())
        monkeypatch.setenv("AMTK_STAGE_MB", "1")          # 1 MiB staging -> a few frames per chunk, one launch each
        hbuf = fr.cpu().numpy()                            # the clip descriptor holds only its address
        host = ab.yv12_clip(hbuf, w, h, n, False)
        got = c.comb_frames(host, prm)
        got = got.cpu().numpy() if hasattr(got, "cpu") else np.asarray(got)
        assert np.array_equal(got, ref)
    finally:
        c.close()


def test_every_band_setting_agrees(monkeypatch):
    """AMTK_COMB_WS_BAND = 0 (per-warp form, U|V remainder columns of 960-byte chroma rows folded into one tile) and 1 (band
    form) return the same counters."""
    outs = {}
    for mode in ("0", "1"):
        c = _band_ctx(monkeypatch, mode)
        try:
            for (w, h, n) in ((1920, 120, 3), (1440, 120, 3)):
                fr = synth.make_frames(7, n, w, h, device="cuda", mode="interlaced")
                outs[(mode, w)] = c.comb_frames(ab.yv12_clip(fr, w, h, n, True), ab.default_comb_params()).cpu().numpy()
        finally:
            c.close()
    for w in (1920, 1440):
        assert np.array_equal(outs[("0", w)], outs[("1", w)]), w
