"""Measure the frame stream widening as it filters (amtk_tnr_stream_create_widening) and KTemporalNR over a CPU source, on
1080p clips, d = 3, t = 1, and print one JSON line.

    python tools/bench_tnr_filter_stream.py [--frames 1800] [--reverse 300]

(a) C ABI, batch 16, progressive, pinned host frames in and out (send each frame, receive whatever may be received):
  - s8_to_14: 8-bit frames, 14-bit outputs (ConvertBits(14) fused into the stream);
  - s8_to_8: 8-bit frames and outputs;  s14_to_14: 14-bit frames (in 16-bit containers) and outputs.
  1800 frames each; the 8-bit source is 1800 pinned frames, the 14-bit one cycles through 900 (frame k is picture
  k mod 900, which keeps the pinned source at the 8-bit one's size), and outputs land in a pool of 32 pinned frames.
(b) the host-side mirror's KTemporalNR as AMTFilterSource's output pass over a CPU source (tests/cpp/test_tnr_filter_stream
  in its bench mode, frame n = picture n mod 60 of a raw file, every frame pulled once):
  - cb14_tnr_in_order: ConvertBits(14) + KTemporalNR(3, 1), frames 0 .. N-1 (the frame stream, widening on the device);
  - cb14_tnr_reverse: the same, the last `--reverse` frames from the last one down (every read gathered);
  - tnr8_in_order: KTemporalNR(3, 1) alone on the 8-bit clip.
  Each runs twice: with the mirror's frames freshly allocated (every 1080p frame is new memory, faulted in and zeroed by
  the kernel), and with suffix _frame_pool, where malloc reuses freed frames as AviSynth+ reuses frames from its cache.
  source_alone_s is the CPU source producing the same frames on its own.
Timing: wall clock around the pass; every call returns once its copies are done.  Reported: frames/s and H2D/D2H bytes per
frame (the filter's H2D by count: each frame sent once, 2d+1 frames per gathered one).  Sampled output frames are checked against the C port of the reference's TemporalNRFilter on the frames shifted
left by the widening; any mismatch exits non-zero.  Writes nothing to the tree (the raw file goes to a temporary
directory).
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import amatsukaze_b200 as ab  # noqa: E402
from amatsukaze_b200 import _build  # noqa: E402
from oracle import pytnr as pt  # noqa: E402
from bench_tnr import gpu_info, make_clip  # noqa: E402

W, H, D, T, B = 1920, 1080, 3, 1, 16
ELEMS = W * H * 3 // 2


def desc(ptr, bits, n=1):
    d = ab.yv12_clip(ptr, W, H, n, False, bits=16 if bits > 8 else 8)
    d.bits_per_sample = bits
    return d


def expected(pic, n, N, sb, ob):
    """Output frame n of a clip of N frames whose frame f is pic(f), at ob bits, by the C port."""
    win = [pic(min(max(n - D + i, 0), N - 1)).astype(np.uint16 if ob > 8 else np.uint8) << (ob - sb) for i in range(2 * D + 1)]
    return pt.or_tnr_frame(win, W, H, ob, T, 0)


def samples(N):
    return sorted({0, 1, 2, N // 2, N - 3, N - 2, N - 1})


def stream_pass(ctx, pool, P, sb, ob, N):
    """Sends N frames (frame k = pool picture k mod P) through a stream at out_bits ob; returns (seconds, h2d, sampled)."""
    ibps, obps = (1 if sb == 8 else 2), (1 if ob == 8 else 2)
    fs_in, fs_out = ELEMS * ibps, ELEMS * obps
    src = [desc(pool.data_ptr() + k * fs_in, sb) for k in range(P)]
    outpool = torch.empty(32 * fs_out, dtype=torch.uint8, pin_memory=True)
    dst = [desc(outpool.data_ptr() + k * fs_out, ob) for k in range(32)]
    out_np = outpool.numpy()
    keep, kept = set(samples(N)), {}
    st = ctx.tnr_stream(ab.tnr_params(D, T, 0), B, False, out_bits=ob if ob != sb else 0)
    h2d, got = 0, 0

    def take():
        nonlocal got
        tag = st.recv(dst[got % 32])
        if tag is None:
            return False
        assert tag == got
        if got in keep:
            kept[got] = out_np[(got % 32) * fs_out:(got % 32 + 1) * fs_out].copy()
        got += 1
        return True

    t0 = time.perf_counter()
    for k in range(N):
        st.send(src[k % P], k)
        h2d += ctx.last_h2d_bytes
        while take():
            pass
    st.finish()
    while got < N:
        assert take()
    dt = time.perf_counter() - t0
    st.close()
    return dt, h2d, kept


def c_abi(ctx, N, res, bad):
    for sb, P, pairs in ((8, N, ((8, 14), (8, 8))), (14, max(1, N // 2), ((14, 14),))):
        fs = ELEMS * (1 if sb == 8 else 2)
        pool = torch.empty(P * fs, dtype=torch.uint8, pin_memory=True)
        for p0 in range(0, P, 300):          # in slices of 300 generated frames
            c = min(300, P - p0)
            pool[p0 * fs:(p0 + c) * fs].copy_(make_clip(sb, c))
        torch.cuda.empty_cache()
        view = pool.numpy().view(np.uint8 if sb == 8 else np.uint16).reshape(P, ELEMS)
        for _, ob in pairs:
            name = "s%d_to_%d" % (sb, ob)
            stream_pass(ctx, pool, P, sb, ob, min(N, 40))       # warm-up: ring, output buffers, pinned pages
            dt, h2d, kept = stream_pass(ctx, pool, P, sb, ob, N)
            res[name] = {"frames": N, "s": round(dt, 3), "frames_per_s": round(N / dt, 1),
                         "h2d_bytes_per_frame": round(h2d / N), "d2h_bytes_per_frame": ELEMS * (1 if ob == 8 else 2)}
            dt_out = np.uint8 if ob == 8 else np.uint16
            m = [n for n, o in kept.items() if not np.array_equal(o.view(dt_out), expected(lambda f: view[f % P], n, N, sb, ob))]
            if m:
                bad[name] = m
        del pool, view


def filter_pass(exe, tmp, pics, N, widen, rev, count, res, bad, name, pool):
    keep = samples(N) if not rev else sorted({N - 1, N - 2, N - 3, N - count // 2, N - count}, reverse=True)
    out = os.path.join(tmp, "out.bin")
    r = subprocess.run([exe, "bench", tmp, str(N), str(widen), "rev" if rev else "fwd", str(count), out,
                        ",".join(map(str, keep)), "pool" if pool else "fresh"], capture_output=True, text=True, timeout=3600)
    if r.returncode != 0:
        sys.exit("filter bench failed: " + r.stdout + r.stderr)
    line = next(l for l in r.stdout.splitlines() if l.startswith("bench: "))
    s = dict(kv.split("=") for kv in line.split(": ", 1)[1].split())
    ob = 14 if widen else 8
    sent, gathered = int(s["sent"]), int(s["gathered"])
    in_fs = ELEMS                                       # 8-bit source frames
    h2d = sent * in_fs + gathered * (2 * D + 1) * in_fs
    res[name] = {"frames": count, "s": round(float(s["seconds"]), 3), "frames_per_s": round(float(s["fps"]), 1),
                 "source_alone_s": round(float(s["source_seconds"]), 3),
                 "h2d_bytes_per_frame": round(h2d / count), "d2h_bytes_per_frame": ELEMS * (2 if widen else 1),
                 "frames_sent": sent, "frames_gathered": gathered, "host_widened": int(s["host_widened"]),
                 "child_frames_asked": int(s["child_total"])}
    got = np.fromfile(out, np.uint16 if widen else np.uint8).reshape(len(keep), ELEMS)
    m = [n for n, o in zip(keep, got) if not np.array_equal(o, expected(lambda f: pics[f % len(pics)], n, N, 8, ob))]
    if m:
        bad[name] = m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1800)
    ap.add_argument("--reverse", type=int, default=300)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tnr_filter_stream.py needs a GPU: there is no CPU fallback")
    torch.cuda.set_device(0)
    info = gpu_info()
    ctx = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    res, bad = {}, {}
    c_abi(ctx, a.frames, res, bad)
    ctx.close()
    torch.cuda.empty_cache()
    exe = _build.build_tnr_filter_stream_test() if os.path.exists("/usr/bin/g++") else _build.TNR_FILTER_STREAM_TEST
    with tempfile.TemporaryDirectory() as tmp:
        pics = make_clip(8, 60).cpu().numpy().reshape(60, ELEMS)
        with open(os.path.join(tmp, "amts0.dat"), "wb") as f:
            f.write(b"AMTSRAW1" + np.array([W, H, 8, 60, 30000, 1001], "<i4").tobytes())
            f.write(pics.tobytes())
        torch.cuda.empty_cache()
        for pool, sfx in ((False, ""), (True, "_frame_pool")):
            filter_pass(exe, tmp, pics, a.frames, 14, False, a.frames, res, bad, "cb14_tnr_in_order" + sfx, pool)
            filter_pass(exe, tmp, pics, a.frames, 14, True, a.reverse, res, bad, "cb14_tnr_reverse" + sfx, pool)
            filter_pass(exe, tmp, pics, a.frames, 0, False, a.frames, res, bad, "tnr8_in_order" + sfx, pool)
            res["cb14_in_order_over_reverse" + sfx] = round(res["cb14_tnr_in_order" + sfx]["frames_per_s"] /
                                                            res["cb14_tnr_reverse" + sfx]["frames_per_s"], 2)
    print(json.dumps({"metric": "tnr_filter_stream_frames_per_s", "d": D, "t": T, "batch": B, "width": W, "height": H,
                      **info, "results": res, "oracle_mismatch_frames": bad}))
    if bad:
        sys.exit("output frames differ from the C port of the reference's TemporalNRFilter")


if __name__ == "__main__":
    main()
