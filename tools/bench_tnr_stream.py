"""Measure amtk_tnr_stream (temporal noise reduction fed one frame at a time) against the ways a frame-at-a-time caller
could use amtk_tnr_frames, on 1080p clips, d = 3, t = 1, and print one JSON line.

    python tools/bench_tnr_stream.py [--frames8 1800] [--frames14 900]

Workloads: 8-bit YV12 and 14-bit samples in 16-bit containers, progressive, from pinned host frames to pinned host frames:
  - stream_B<b>: amtk_tnr_stream at batch size b (1, 4, 16, 64): send each frame, receive whatever may be received;
  - gather: what KTemporalNR does for a child that is not device resident: per output frame the 2d+1 clamped frames are
    copied into one pinned buffer, then a one-frame amtk_tnr_frames call (host to host);
  - clip_h2h: one whole-clip host-to-host amtk_tnr_frames call (the ceiling for host clips, which needs the whole clip);
  - device_stream_B<b> / device_clip: frames and outputs resident in HBM, through the stream and one amtk_tnr_frames call.
Timing: wall clock around each pass (the calls return when their copies are done), after a short warm-up.  Reported:
frames/s, and H2D and D2H bytes per output frame (H2D from the library's own count).  Sampled output frames (the first and
last d, and the middle) are checked against the C port of the reference's TemporalNRFilter; any mismatch exits non-zero.
Writes nothing to the tree.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import amatsukaze_b200 as ab  # noqa: E402
from oracle import pytnr as pt  # noqa: E402
from bench_tnr import gpu_info, make_clip  # noqa: E402

W, H, D, T = 1920, 1080, 3, 1


def desc(base, bits, n, on_device):
    d = ab.yv12_clip(base, W, H, n, on_device, bits=16 if bits > 8 else 8)
    d.bits_per_sample = bits
    return d


class Clip:
    """n packed frames at `ptr` (host or device), one descriptor per frame."""

    def __init__(self, ptr, bits, n, on_device):
        self.bits, self.n, self.dev = bits, n, on_device
        self.fs = W * H * 3 // 2 * (1 if bits == 8 else 2)
        self.ptr = ptr
        self.frames = [desc(ptr + k * self.fs, bits, 1, on_device) for k in range(n)]
        self.all = desc(ptr, bits, n, on_device)


def run_stream(ctx, src, dst, B, n=None):
    n = src.n if n is None else n
    prm = ab.tnr_params(D, T, 0)
    st = ctx.tnr_stream(prm, B)
    h2d, got = 0, 0
    t0 = time.perf_counter()
    for k in range(n):
        st.send(src.frames[k], k)
        h2d += ctx.last_h2d_bytes
        while True:
            tag = st.recv(dst.frames[got])
            if tag is None:
                break
            assert tag == got
            got += 1
    st.finish()
    while got < n:
        tag = st.recv(dst.frames[got])
        assert tag == got
        got += 1
    dt = time.perf_counter() - t0
    st.close()
    return dt, h2d


def run_gather(ctx, src_host, dst, stage, n=None):
    """src_host: numpy uint8 view of the pinned source clip; stage: pinned buffer of 2d+1 frames."""
    n = dst.n if n is None else n
    fs, N = dst.fs, dst.n
    prm = ab.tnr_params(D, T, 0)
    sd = desc(stage.ctypes.data, dst.bits, 2 * D + 1, False)
    h2d = 0
    t0 = time.perf_counter()
    for k in range(n):
        for i in range(2 * D + 1):
            f = min(max(k - D + i, 0), N - 1)
            stage[i * fs:(i + 1) * fs] = src_host[f * fs:(f + 1) * fs]
        ctx.tnr_frames(sd, dst.frames[k], prm, D, 1)
        h2d += ctx.last_h2d_bytes
    return time.perf_counter() - t0, h2d


def check(src_np, out_np, bits, n):
    """Sampled frames against the C port; returns the mismatching frame numbers."""
    fs = W * H * 3 // 2
    dt = np.uint8 if bits == 8 else np.uint16
    s, o = src_np.view(dt).reshape(n, fs), out_np.view(dt).reshape(n, fs)
    bad = []
    for k in sorted({0, 1, 2, n // 2, n - 3, n - 2, n - 1}):
        win = [s[min(max(k - D + i, 0), n - 1)] for i in range(2 * D + 1)]
        if not np.array_equal(o[k], pt.or_tnr_frame(win, W, H, bits, T, 0)):
            bad.append(k)
    return bad


def workload(ctx, bits, n):
    bps = 1 if bits == 8 else 2
    fs = W * H * 3 // 2 * bps
    dev_src = make_clip(bits, n)
    host_src = torch.empty(n * fs, dtype=torch.uint8, pin_memory=True)
    host_src.copy_(dev_src)
    host_dst = torch.empty(n * fs, dtype=torch.uint8, pin_memory=True)
    src_np = host_src.numpy()
    hs, hd = Clip(host_src.data_ptr(), bits, n, False), Clip(host_dst.data_ptr(), bits, n, False)
    res, bad = {}, {}

    def record(name, dt, h2d, out_np):
        res[name] = {"s": round(dt, 3), "frames_per_s": round(n / dt, 1), "h2d_bytes_per_frame": round(h2d / n),
                     "d2h_bytes_per_frame": fs if out_np is not None else 0}
        if out_np is not None:
            m = check(src_np, out_np, bits, n)
            if m:
                bad[name] = m

    run_stream(ctx, hs, hd, 4, n=min(n, 40))                 # warm-up: ring and output buffers, pinned pages
    for B in (1, 4, 16, 64):
        host_dst.fill_(0)
        dt, h2d = run_stream(ctx, hs, hd, B)
        record("stream_B%d" % B, dt, h2d, host_dst.numpy())
    stage = torch.empty((2 * D + 1) * fs, dtype=torch.uint8, pin_memory=True).numpy()
    run_gather(ctx, src_np, hd, stage, n=min(n, 20))
    host_dst.fill_(0)
    dt, h2d = run_gather(ctx, src_np, hd, stage)
    record("gather", dt, h2d, host_dst.numpy())
    ctx.tnr_frames(hs.all, hd.all, ab.tnr_params(D, T, 0))
    host_dst.fill_(0)
    t0 = time.perf_counter()
    ctx.tnr_frames(hs.all, hd.all, ab.tnr_params(D, T, 0))
    record("clip_h2h", time.perf_counter() - t0, ctx.last_h2d_bytes, host_dst.numpy())
    dev_dst = torch.empty_like(dev_src)
    ds, dd = Clip(dev_src.data_ptr(), bits, n, True), Clip(dev_dst.data_ptr(), bits, n, True)
    for B in (16, 64):
        torch.cuda.synchronize()
        dt, _ = run_stream(ctx, ds, dd, B)
        record("device_stream_B%d" % B, dt, 0, None)
        out = dev_dst.cpu().numpy()
        m = check(src_np, out, bits, n)
        if m:
            bad["device_stream_B%d" % B] = m
    ctx.tnr_frames(ds.all, dd.all, ab.tnr_params(D, T, 0))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ctx.tnr_frames(ds.all, dd.all, ab.tnr_params(D, T, 0))
    torch.cuda.synchronize()
    record("device_clip", time.perf_counter() - t0, 0, None)
    for r in res.values():
        if r["h2d_bytes_per_frame"] == 0 and r["d2h_bytes_per_frame"] == 0:
            r.pop("h2d_bytes_per_frame"), r.pop("d2h_bytes_per_frame")
    res["stream_B16_over_gather"] = round(res["stream_B16"]["frames_per_s"] / res["gather"]["frames_per_s"], 2)
    res["best_stream_over_gather"] = round(max(res["stream_B%d" % B]["frames_per_s"] for B in (1, 4, 16, 64)) /
                                           res["gather"]["frames_per_s"], 2)
    del dev_src, dev_dst, host_src, host_dst
    torch.cuda.empty_cache()
    return {"bits": bits, "container_bytes": bps, "frames": n, "frame_bytes": fs, "results": res,
            "oracle_mismatch_frames": bad}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames8", type=int, default=1800)
    ap.add_argument("--frames14", type=int, default=900)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tnr_stream.py needs a GPU: there is no CPU fallback")
    torch.cuda.set_device(0)
    ctx = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    info = gpu_info()
    res = [workload(ctx, 8, a.frames8), workload(ctx, 14, a.frames14)]
    print(json.dumps({"metric": "tnr_stream_frames_per_s", "d": D, "t": T, "width": W, "height": H, **info,
                      "workloads": res}))
    ctx.close()
    if any(r["oracle_mismatch_frames"] for r in res):
        sys.exit("output frames differ from the C port of the reference's TemporalNRFilter")


if __name__ == "__main__":
    main()
