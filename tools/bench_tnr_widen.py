"""Measure the server's `ConvertBits(14)` + `KTemporalNR(3, 1)` on resident 1080p YV12 clips and print one JSON line.

    python tools/bench_tnr_widen.py [--frames 1800] [--reps 10] [--rounds 3]

Workloads, each progressive and interlaced, source and destinations resident in HBM:
  fused      one amtk_tnr_frames call from the 8-bit clip into 14-bit frames (the widening kernels);
  two_pass   a d = 0 widening call into a 14-bit copy of the clip (what ConvertBits materialises), then the 14-bit call;
  tnr8       the 8-bit clip filtered at 8 bits (the existing call; no widening).
Timing: CUDA events on the context's stream around `reps` calls after two warm-up calls, the workloads alternated over
`rounds` rounds; the median round is reported.  Bytes moved = every source byte read once + every destination byte written
once (fused: 8-bit reads + 16-bit writes; two_pass adds the intermediate's write and read), against the read-only ceiling
of the same run and against the issue bound of tools/bench_tnr.py (DESIGN.md section 6.1).  Sampled fused frames are
checked against the C port of the reference's TemporalNRFilter on the shifted frames, the two-pass output against the fused
output, the 8-bit output against the C port at 8 bits; any mismatch exits non-zero.  Writes nothing to the tree.
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_tnr import D, H, HBM_TBS, OPS_FIXED_PX, OPS_PER_FRAME_PX, T, W, gpu_info, make_clip  # noqa: E402

import amatsukaze_b200 as ab  # noqa: E402
from oracle import pytnr as pt  # noqa: E402

FS = W * H * 3 // 2           # samples per frame


def desc(buf, n, bits):
    d = ab.yv12_clip(buf, W, H, n, True, bits=8 if bits == 8 else 16)
    d.bits_per_sample = bits
    return d


def time_calls(stream, reps, calls):
    for _ in range(2):
        calls()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(reps):
        calls()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def check_frames(src8, out, n, il, out_bits):
    """Sampled output frames against the C port on the (shifted) 8-bit source; returns the mismatching indices."""
    k = out_bits - 8
    dt = np.uint8 if out_bits == 8 else np.uint16
    bad = []
    for f in sorted({0, 1, 2, n // 2, n - 2, n - 1}):
        win = []
        for i in range(2 * D + 1):
            w = min(max(f - D + i, 0), n - 1)
            win.append(src8[w * FS:(w + 1) * FS].cpu().numpy().astype(dt) << k)
        want = pt.or_tnr_frame(win, W, H, out_bits, T, il)
        got = out.view(torch.uint8)[f * FS * dt().itemsize:(f + 1) * FS * dt().itemsize].cpu().numpy().view(dt)
        if not np.array_equal(got, want):
            bad.append(f)
    return bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1800)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tnr_widen.py needs a GPU: there is no CPU fallback")
    torch.cuda.set_device(0)
    stream = torch.cuda.current_stream()
    ctx = ab.Context(0, stream.cuda_stream)
    info = gpu_info()
    probe = torch.empty(FS * 1800, dtype=torch.uint8, device="cuda").fill_(1)
    probe_gbs = ctx.probe_read_gbs(probe, reps=10)
    del probe
    clock_mhz = info.get("sm_clock_max_mhz") or torch.cuda.get_device_properties(0).clock_rate / 1e3
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = a.frames
    src8 = make_clip(8, n)
    out14 = torch.empty(n * FS, dtype=torch.int16, device="cuda")
    mid14 = torch.empty(n * FS, dtype=torch.int16, device="cuda")
    two14 = torch.empty(n * FS, dtype=torch.int16, device="cuda")
    out8 = torch.empty_like(src8)
    s8, o14, m14, t14, o8 = desc(src8, n, 8), desc(out14, n, 14), desc(mid14, n, 14), desc(two14, n, 14), desc(out8, n, 8)
    fs8, fs16 = FS, 2 * FS
    moved = {"fused": n * (fs8 + fs16), "two_pass": n * (fs8 + fs16) + n * (fs16 + fs16), "tnr8": n * (fs8 + fs8)}
    launches = {"fused": 1, "two_pass": 2, "tnr8": 1}
    ops = n * W * H * ((2 * D + 1) * OPS_PER_FRAME_PX + OPS_FIXED_PX)
    issue_ms = ops / (sms * 128 * clock_mhz * 1e6) * 1e3
    res = []
    for il in (0, 1):
        prm, copy = ab.tnr_params(D, T, il), ab.tnr_params(0, 0, 0)
        calls = {"fused": lambda: ctx.tnr_frames(s8, o14, prm),
                 "two_pass": lambda: (ctx.tnr_frames(s8, m14, copy), ctx.tnr_frames(m14, t14, prm)),
                 "tnr8": lambda: ctx.tnr_frames(s8, o8, prm)}
        ms = {k: [] for k in calls}
        for _ in range(a.rounds):
            for k, c in calls.items():
                ms[k].append(time_calls(stream, a.reps, c))
        bad = {"fused": check_frames(src8, out14, n, il, 14),
               "two_pass": [] if torch.equal(out14, two14) else ["differs from fused"],
               "tnr8": check_frames(src8, out8, n, il, 8)}
        for k in calls:
            m = statistics.median(ms[k])
            res.append({"workload": k, "interlaced": il, "frames": n, "launches_per_call": launches[k],
                        "ms_per_call": round(m, 4), "ms_rounds": [round(x, 4) for x in ms[k]],
                        "frames_per_s": round(n / (m * 1e-3)), "bytes_moved": moved[k],
                        "tb_per_s": round(moved[k] / (m * 1e-3) / 1e12, 3),
                        "frac_of_read_ceiling": round(moved[k] / (m * 1e-3) / (probe_gbs * 1e9), 3),
                        "hbm_bound_ms": round(moved[k] / (HBM_TBS * 1e12) * 1e3, 4),
                        "issue_bound_ms": round(issue_ms, 4),
                        "frac_of_issue_bound": round(issue_ms / m, 3),
                        "mismatch": bad[k]})
    out = {"metric": "tnr_widen_frames_per_s", "d": D, "t": T, "width": W, "height": H,
           "read_ceiling_tb_per_s": round(probe_gbs / 1e3, 3), **info, "sm_clock_used_for_bound_mhz": clock_mhz,
           "workloads": res}
    print(json.dumps(out))
    ctx.close()
    if any(r["mismatch"] for r in res):
        sys.exit("outputs differ from the C port of the reference's TemporalNRFilter on the shifted frames")


if __name__ == "__main__":
    main()
