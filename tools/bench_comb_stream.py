"""Combing stream (amtk_comb_stream) vs the mirror's old K = 16 path and vs amtk_comb_frames on a whole pinned host clip,
on 1080-line frames from host (pinned, pageable) and device memory.

The old path is what the host mirror's AMTCombAnalyze ran on a source that is not device resident: a 17-frame pinned
buffer whose slot 0 holds the frame before the batch, 16 frames copied into it on the host, one synchronous
amtk_comb_frames call per 16 frames (which stages all 17 frames), then the last slot copied into slot 0.  The whole-clip
call is the PCIe ceiling: amtk_comb_frames on one pinned host clip, staged in chunks.  The stream sends every frame once
and receives after every send, then finishes and drains.  Frames are replayed from --distinct seeded ones.

    python tools/bench_comb_stream.py [--frames 1500] [--distinct 64] [--repeat 3] [--tiny]

Prints one JSON line: frames/s of each format, source and batch size (timed to a device synchronise, the median of
--repeat runs, each after a warm-up stream at the same batch size), H2D / D2H bytes per frame, the host seconds spent in
sends that only copy (copy_s), in sends that also launch a batch (launch_s: the launch waits for the previous batch's
watchdog record, i.e. its kernel) and in receives (recv_s), and the card's name, power limit and SM clock read in the
same command.  Every run's rows are checked against one resident amtk_comb_frames call on the distinct frames.
--tiny rehearses at 320x180 with few frames; without a GPU it builds the inputs and stops there.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import amatsukaze_b200 as ab  # noqa: E402
from amatsukaze_b200 import synth  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smmax = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": pl, "sm_clock": sm, "sm_clock_max": smmax}
    except Exception as e:           # the measurement still stands; say what is missing
        return {"gpu": torch.cuda.get_device_name(0) if torch.cuda.is_available() else None,
                "nvidia_smi": "unavailable (%s)" % type(e).__name__}


def make_distinct(D, W, H, bits, device):
    """D interlaced frames (every counter moves), packed 4:2:0: uint8, or int16 holding 10-bit samples."""
    fsz = W * H * 3 // 2
    f8 = torch.empty((D, fsz), dtype=torch.uint8, device=device)
    for n0 in range(0, D, 16):
        synth.make_frames(n0, min(16, D - n0), W, H, seed=0x5EED0600, device=device, mode="interlaced", out=f8[n0:n0 + 16])
    if bits == 8:
        return f8
    g = torch.Generator(device=device).manual_seed(bits)
    low = torch.randint(0, 1 << (bits - 8), f8.shape, device=device, generator=g, dtype=torch.int32)
    return ((f8.to(torch.int32) << (bits - 8)) | low).to(torch.int16)


def expected(ctx, dev, N, W, H, bits):
    """Rows of frames 0..N-1 replayed from the D distinct ones: row i has distinct frame i % D and, for i > 0, the previous
    replayed frame; a resident call on the distinct frames followed by frame 0 again covers both cases."""
    D = dev.shape[0]
    ext = torch.cat([dev, dev[:1]]).contiguous()
    r = ctx.comb_frames(ab.yv12_clip(ext, W, H, D + 1, True, bits)).cpu().numpy()
    j = np.arange(N) % D
    out = r[j]
    out[(np.arange(N) > 0) & (j == 0)] = r[D]
    return out


def run_stream(ctx, descs, N, B):
    out = np.empty((N, 12), np.int32)
    copy_s = launch_s = recv_s = 0.0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    s = ctx.comb_stream(None, B)
    got = 0
    for i in range(N):
        ta = time.perf_counter()
        s.send(descs[i % len(descs)])
        tb = time.perf_counter()
        r = s.recv(N - got)
        tc = time.perf_counter()
        if (i + 1) % B == 0:
            launch_s += tb - ta
        else:
            copy_s += tb - ta
        recv_s += tc - tb
        out[got:got + len(r)] = r
        got += len(r)
    s.finish()
    r = s.recv(N - got)
    out[got:got + len(r)] = r
    got += len(r)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    c = s.counts()
    s.close()
    assert got == N
    return dt, c, out, {"copy_s": copy_s, "launch_s": launch_s, "recv_s": recv_s}


def old_path(ctx, src, N, W, H, bits):
    """The mirror's old generic branch: K = 16 frames per amtk_comb_frames call through a 17-frame pinned buffer."""
    K = 16
    fb = (src.shape[1] * src.itemsize + 15) & ~15
    buf = torch.empty((K + 1) * fb, dtype=torch.uint8).pin_memory()
    view = buf.numpy()
    hc = ab.yv12_clip(buf, W, H, K + 1, False, bits)
    hc.frame_stride = fb
    raw = src.view(np.uint8)
    fsz = raw.shape[1]
    out = np.empty((N, 12), np.int32)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for n0 in range(0, N, K):
        cnt = min(K, N - n0)
        slot0 = 0 if n0 == 0 else 1
        for k in range(cnt):
            o = (slot0 + k) * fb
            view[o:o + fsz] = raw[(n0 + k) % raw.shape[0]]
        ctx.comb_frames(hc, None, slot0, cnt, out=out[n0:n0 + cnt])
        last = (slot0 + cnt - 1) * fb
        view[:fb] = view[last:last + fb]
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def whole_clip(ctx, pinned_clip, W, H, bits):
    n = pinned_clip.shape[0]
    clip = ab.yv12_clip(pinned_clip, W, H, n, False, bits)
    out = np.empty((n, 12), np.int32)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ctx.comb_frames(clip, None, 0, n, out=out)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out, ctx.last_h2d_bytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1500)
    ap.add_argument("--whole-frames", type=int, default=480, help="frames of the pinned whole-clip call")
    ap.add_argument("--distinct", type=int, default=64, help="distinct seeded frames, replayed")
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--tiny", action="store_true", help="320x180 and few frames; without a GPU, stop after the inputs")
    a = ap.parse_args()
    formats = [("yv12_1920x1080", 1920, 1080, 8), ("yv12_1440x1080", 1440, 1080, 8), ("yuv420p10_1920x1080", 1920, 1080, 10)]
    if a.tiny:
        formats = [(n.split("_")[0] + "_320x180", 320, 180, b) for n, _, _, b in formats[::2]]
        a.frames, a.whole_frames, a.distinct, a.repeat = min(a.frames, 200), min(a.whole_frames, 48), min(a.distinct, 16), 1
    gpu = torch.cuda.is_available()
    res = {"metric": "comb_stream", "frames": a.frames, "distinct": a.distinct, "repeat": a.repeat, "cases": []}
    res.update(gpu_info())
    ctx = None
    if gpu:
        torch.cuda.set_device(0)
        ctx = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    for fname, W, H, bits in formats:
        case = {"format": fname, "bits": bits, "sources": {}}
        res["cases"].append(case)
        if not gpu:
            make_distinct(2, W, H, bits, "cpu")
            case["note"] = "no GPU: inputs built, nothing measured"
            continue
        dev = make_distinct(a.distinct, W, H, bits, "cuda")
        exp = expected(ctx, dev, max(a.frames, a.whole_frames), W, H, bits)
        pinned = dev.cpu().pin_memory()
        pageable = dev.cpu().numpy().copy()
        # baselines, in the same run
        to, oo = old_path(ctx, pageable, a.frames, W, H, bits)
        assert np.array_equal(oo, exp[:a.frames]), (fname, "old path")
        case["old_k16"] = {"fps": a.frames / to, "h2d_per_frame": 17 * ((pageable.shape[1] * pageable.itemsize + 15) & ~15) / 16}
        reps = -(-a.whole_frames // a.distinct)
        whole = torch.cat([dev] * reps)[:a.whole_frames].cpu().pin_memory()
        whole_clip(ctx, whole[:16], W, H, bits)                                  # warm-up
        tw, ow, hw = whole_clip(ctx, whole, W, H, bits)
        assert np.array_equal(ow, exp[:a.whole_frames]), (fname, "whole clip")
        case["whole_pinned_clip"] = {"fps": a.whole_frames / tw, "frames": a.whole_frames, "h2d_per_frame": hw / a.whole_frames}
        del whole
        for sname, src, on_dev in (("pinned", pinned, False), ("pageable", pageable, False), ("device", dev, True)):
            descs = [ab.yv12_clip(src[i], W, H, 1, on_dev, bits) for i in range(a.distinct)]
            rows = []
            for B in (16, 64, 256):
                run_stream(ctx, descs, min(a.frames, 2 * B + 32), B)          # warm-up
                fps, splits = [], []
                for _ in range(a.repeat):
                    dt, c, out, split = run_stream(ctx, descs, a.frames, B)
                    assert np.array_equal(out, exp[:a.frames]), (fname, sname, B)
                    fps.append(a.frames / dt)
                    splits.append(split)
                mid = int(np.argsort(fps)[len(fps) // 2])
                rows.append({"B": B, "fps": float(np.median(fps)), "fps_runs": fps, "h2d_per_frame": c[2] / a.frames,
                             "d2h_per_frame": c[3] / a.frames, "send_split_median_run": splits[mid]})
            case["sources"][sname] = rows
        del dev, pinned, pageable
        torch.cuda.empty_cache()
    if ctx:
        ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
