"""Measure amtk_tnr_frames (temporal noise reduction, d = 3, t = 1) on resident 1080p clips and print one JSON line.

    python tools/bench_tnr.py [--frames8 1800] [--frames14 900] [--reps 20]

Workloads: 8-bit YV12 and 14-bit samples in 16-bit containers (the product runs the filter after ConvertBits(14)), each
progressive and interlaced, source and destination resident in HBM.  Timing: CUDA events on the context's stream around
`reps` calls after two warm-up calls (each call is one kernel launch over the whole clip).  Reported per workload: ms per
call, frames/s, bytes moved (every source byte read once, every destination byte written once) and bytes/s against the
3.35 TB/s data sheet and against the read-only ceiling measured in the same run, and the issue-rate bound from an
operation count of the algorithm (see OPS_*).  Sampled output frames are checked
against the C port of the reference's TemporalNRFilter; any mismatch exits non-zero.  Writes nothing to the tree.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import amatsukaze_b200 as ab  # noqa: E402
from amatsukaze_b200 import synth  # noqa: E402
from oracle import pytnr as pt  # noqa: E402

HBM_TBS = 3.35
W, H, D, T = 1920, 1080, 3, 1
# Issue-rate bound from the algorithm (not from this kernel's instruction stream): the operations the spec needs per luma
# pixel.  Per window frame: |Y-Yi| (1), + the U/V distance (1), <= thresh (1), and the weighted add f*Yi + acc (2) = 5.
# Per window frame and chroma sample, shared by its 2x2 luma pixels (a quarter each): |U-Ui| + |V-Vi| (3) and the U and V
# adds (4) = 7.  Per luma pixel: 1/k (1) and the conversion of the result (1) = 2.  About 49 at d = 3.
OPS_PER_FRAME_PX = 5 + 7 / 4
OPS_FIXED_PX = 2


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": q[0], "power_limit_w": float(q[1]), "sm_clock_max_mhz": float(q[2])}
    except Exception as e:      # the measurement still stands; the card is then named by torch only
        return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_error": str(e)}


def make_clip(bits, n):
    """n resident 1080p frames (packed 4:2:0) as a uint8 CUDA tensor of n * frame_bytes."""
    bps = 1 if bits == 8 else 2
    fs = W * H * 3 // 2
    out = torch.empty(n * fs * bps, dtype=torch.uint8, device="cuda")
    step = 60
    for n0 in range(0, n, step):
        c = min(step, n - n0)
        f8 = synth.make_frames(n0, c, W, H, device="cuda", mode="interlaced")
        if bits == 8:
            out[n0 * fs:(n0 + c) * fs].copy_(f8.reshape(-1))
        else:                   # 14 significant bits: the 8-bit picture << 6 plus a seeded low-order pattern
            idx = torch.arange(fs, device="cuda", dtype=torch.int32).view(1, fs)
            lo = (idx * 40503 + torch.arange(n0, n0 + c, device="cuda", dtype=torch.int32).view(c, 1) * 9973) & 63
            v = ((f8.to(torch.int32) << 6) + lo).clamp(0, (1 << bits) - 1).to(torch.int16)
            out.view(torch.int16)[n0 * fs:(n0 + c) * fs].copy_(v.reshape(-1))
    return out


def run_workload(ctx, stream, bits, n, il, reps, probe_gbs):
    bps = 1 if bits == 8 else 2
    src = make_clip(bits, n)
    dst = torch.empty_like(src)
    sd = ab.yv12_clip(src, W, H, n, True, bits=16 if bits > 8 else 8)
    dd = ab.yv12_clip(dst, W, H, n, True, bits=16 if bits > 8 else 8)
    sd.bits_per_sample = dd.bits_per_sample = bits
    prm = ab.tnr_params(D, T, il)
    for _ in range(2):
        ctx.tnr_frames(sd, dd, prm)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(reps):
        ctx.tnr_frames(sd, dd, prm)
    e1.record(stream)
    e1.synchronize()
    ms = e0.elapsed_time(e1) / reps
    # sampled frames against the C port of the reference's TemporalNRFilter
    fs = W * H * 3 // 2
    dt = np.uint8 if bps == 1 else np.uint16
    bad = []
    for k in sorted({0, 1, 2, n // 2, n - 2, n - 1}):
        win = [src[min(max(k - D + i, 0), n - 1) * fs * bps:(min(max(k - D + i, 0), n - 1) + 1) * fs * bps].cpu().numpy().view(dt)
               for i in range(2 * D + 1)]
        want = pt.or_tnr_frame(win, W, H, bits, T, il)
        got = dst[k * fs * bps:(k + 1) * fs * bps].cpu().numpy().view(dt)
        if not np.array_equal(got, want):
            bad.append(k)
    moved = 2 * n * fs * bps
    px = n * W * H
    nf = 2 * D + 1
    ops = px * (nf * OPS_PER_FRAME_PX + OPS_FIXED_PX)
    props = torch.cuda.get_device_properties(0)
    del src, dst
    torch.cuda.empty_cache()
    return {"bits": bits, "container_bytes": bps, "frames": n, "interlaced": il, "ms_per_call": round(ms, 4),
            "frames_per_s": round(n / (ms * 1e-3)), "bytes_moved": moved, "tb_per_s": round(moved / (ms * 1e-3) / 1e12, 3),
            "frac_of_3_35_tbs": round(moved / (ms * 1e-3) / (HBM_TBS * 1e12), 3),
            "frac_of_read_ceiling": round(moved / (ms * 1e-3) / (probe_gbs * 1e9), 3),
            "hbm_bound_ms": round(moved / (HBM_TBS * 1e12) * 1e3, 4),
            "ops_algorithm": int(ops), "sms": props.multi_processor_count,
            "oracle_mismatch_frames": bad}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames8", type=int, default=1800)
    ap.add_argument("--frames14", type=int, default=900)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tnr.py needs a GPU: there is no CPU fallback")
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream()
    ctx = ab.Context(0, stream.cuda_stream)
    info = gpu_info()
    probe = torch.empty(W * H * 3 // 2 * 1800, dtype=torch.uint8, device="cuda").fill_(1)
    probe_gbs = ctx.probe_read_gbs(probe, reps=10)
    del probe
    clock_mhz = info.get("sm_clock_max_mhz") or torch.cuda.get_device_properties(0).clock_rate / 1e3
    res = []
    for bits, n in ((8, a.frames8), (14, a.frames14)):
        for il in (0, 1):
            r = run_workload(ctx, stream, bits, n, il, a.reps, probe_gbs)
            lanes = r["sms"] * 128 * clock_mhz * 1e6
            r["issue_bound_ms"] = round(r["ops_algorithm"] / lanes * 1e3, 4)
            bound = max(r["issue_bound_ms"], r["hbm_bound_ms"])
            r["bound_by"] = "issue" if r["issue_bound_ms"] > r["hbm_bound_ms"] else "hbm"
            r["frac_of_larger_bound"] = round(bound / r["ms_per_call"], 3)
            res.append(r)
    out = {"metric": "tnr_frames_per_s", "d": D, "t": T, "width": W, "height": H, "read_ceiling_tb_per_s": round(probe_gbs / 1e3, 3),
           **info, "sm_clock_used_for_bound_mhz": clock_mhz, "workloads": res}
    print(json.dumps(out))
    ctx.close()
    if any(r["oracle_mismatch_frames"] for r in res):
        sys.exit("output frames differ from the C port of the reference's TemporalNRFilter")


if __name__ == "__main__":
    main()
