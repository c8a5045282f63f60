"""Logo scan stream (amtk_logo_scan_stream) vs the per-frame path, on 1080p frames from host (pinned, pageable) and device
memory.

The per-frame path is what the host mirror's logo::LogoFrame::scanFrames ran on a source that is not device resident:
one synchronous amtk_logo_scan_frames call per frame, with the byte-pitch override at 2-byte samples (which stages whole
frames).  The stream sends every frame once and receives after every send, then finishes and drains.  Frames are
replayed from --distinct seeded ones.

    python tools/bench_logo_scan_stream.py [--frames 12000] [--baseline-frames 600] [--tiny]

Prints one JSON line: frames/s of each case, source and batch size (timed to a device synchronise, the median of
--repeat runs, each after a warm-up stream at the same batch size), H2D / D2H bytes per frame, and the card's name,
power limit and SM clock read in the same command.  Every stream's results are checked bit for bit against one resident
amtk_logo_scan_frames call on the distinct frames.
--tiny rehearses at 320x192 with few frames; without a GPU it builds the inputs and logos and stops there.
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


def cases(W, H):
    """name: (bits, reference_pitch, [(w, h, imgx, imgy)]).  The 10-bit logo lies in the upper half, where the byte-pitch
    row step keeps it inside the plane.  Device frames are gathered with the widest copy the rectangle's byte x allows:
    1-byte copies at odd x and 8 bits, 2-byte copies at odd x and 10 bits, 16-byte copies in the aligned case."""
    x = lambda v, w=64: min(W - w - 1, int(round(v * W / 1920.0))) | 1      # odd x positions inside the frame
    xa = lambda v, w=64: min(W - w, int(round(v * W / 1920.0))) & ~15     # 16-byte aligned x
    y = lambda v: int(round(v * H / 1080.0))
    return {
        "yv12_1x64": (8, False, [(64, 64, x(1700), y(60))]),
        "yv12_1x64_aligned": (8, False, [(64, 64, xa(1696), y(60))]),
        "yv12_4x64_corners": (8, False, [(64, 64, x(24), y(20)), (64, 64, W - 64 - x(24), y(20)),
                                         (64, 64, x(24), H - 64 - y(20)), (64, 64, W - 64 - x(24), H - 64 - y(20))]),
        "yv12_1x192x96": (8, False, [(192, 96, x(1680, 192), y(48))]),
        "yuv420p10_quirk_1x64": (10, True, [(64, 64, x(1700), y(60))]),
    }


def make_distinct(D, W, H, bits, logo, ix, iy, device):
    fsz = W * H * 3 // 2
    f8 = torch.empty((D, fsz), dtype=torch.uint8, device=device)
    for n0 in range(0, D, 20):
        synth.make_frames(n0, min(20, D - n0), W, H, seed=0x5EED0400, device=device, logo=logo, imgx=ix, imgy=iy,
                          logo_period=40, out=f8[n0:n0 + 20])
    if bits == 8:
        return f8
    g = torch.Generator(device=device).manual_seed(bits)
    low = torch.randint(0, 1 << (bits - 8), f8.shape, device=device, generator=g, dtype=torch.int32)
    return ((f8.to(torch.int32) << (bits - 8)) | low).to(torch.int16)


def desc(buf, i, W, H, bits, on_device):
    b = buf[i % buf.shape[0]]
    return ab.yv12_clip(b, W, H, 1, on_device, bits)


def run_stream(ctx, logos, src, N, W, H, bits, B, quirk, on_device):
    L = len(logos)
    out = np.empty((N, L, 2), np.float32)
    descs = [desc(src, i, W, H, bits, on_device) for i in range(src.shape[0])]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    s = ctx.logo_scan_stream(logos, B, quirk)
    got = 0
    for i in range(N):
        s.send(descs[i % len(descs)])
        r = s.recv(N - got)
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
    return dt, c, out


def per_frame(ctx, logos, src, N, W, H, bits, quirk):
    """The mirror's old path: one amtk_logo_scan_frames call per host frame."""
    L = len(logos)
    out = np.empty((N, L, 2), np.float32)
    descs = [desc(src, i, W, H, bits, False) for i in range(src.shape[0])]
    override = descs[0].pitch_y if quirk and bits > 8 else 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(N):
        ctx.scan_frames(descs[i % len(descs)], logos, out=out[i:i + 1], pitch_elems_override=override)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=12000)
    ap.add_argument("--baseline-frames", type=int, default=600)
    ap.add_argument("--distinct", type=int, default=200, help="distinct seeded frames, replayed")
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--tiny", action="store_true", help="320x192 and few frames; without a GPU, stop after the inputs")
    a = ap.parse_args()
    W, H = (320, 192) if a.tiny else (1920, 1080)
    if a.tiny:
        a.frames, a.baseline_frames, a.distinct, a.repeat = min(a.frames, 300), min(a.baseline_frames, 60), min(a.distinct, 24), 1
    gpu = torch.cuda.is_available()
    res = {"metric": "logo_scan_stream", "width": W, "height": H, "frames": a.frames, "distinct": a.distinct,
           "repeat": a.repeat, "cases": []}
    res.update(gpu_info())
    ctx = None
    if gpu:
        torch.cuda.set_device(0)
        ctx = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    lg64 = synth.make_logo(64, 64, seed=3)
    for cname, (bits, quirk, rects) in cases(W, H).items():
        logos = [ab.Logo.create(synth.make_logo(w, h, seed=3 + k)["data"], w, h, W, H, x, y).deint().create_mask(0.35)
                 for k, (w, h, x, y) in enumerate(rects)]
        case = {"case": cname, "bits": bits, "reference_pitch": quirk, "logos": rects, "sources": {}}
        res["cases"].append(case)
        if not gpu:
            make_distinct(2, W, H, bits, lg64, rects[0][2], rects[0][3], "cpu")
            case["note"] = "no GPU: inputs and logos built, nothing measured"
            continue
        dev = make_distinct(a.distinct, W, H, bits, lg64, rects[0][2], rects[0][3], "cuda")
        clip = ab.yv12_clip(dev, W, H, a.distinct, True, bits)
        exp = ctx.scan_frames(clip, logos, pitch_elems_override=clip.pitch_y if quirk else 0).cpu().numpy()
        pinned = dev.cpu().pin_memory()
        pageable = dev.cpu().numpy().copy()
        idx = np.arange(a.frames) % a.distinct
        tb, ob = per_frame(ctx, logos, pageable, a.baseline_frames, W, H, bits, quirk)
        assert np.array_equal(ob.view(np.uint32), exp[idx[:a.baseline_frames]].view(np.uint32)), (cname, "per-frame")
        case["per_frame"] = {"fps": a.baseline_frames / tb, "frames": a.baseline_frames, "source": "pageable",
                             "h2d_per_frame": ctx.last_h2d_bytes}
        for sname, src, on_dev in (("pinned", pinned, False), ("pageable", pageable, False), ("device", dev, True)):
            rows = []
            for B in (1, 16, 64, 256):
                run_stream(ctx, logos, src, min(a.frames, 4 * B + 64), W, H, bits, B, quirk, on_dev)     # warm-up
                fps = []
                for _ in range(a.repeat):
                    dt, c, out = run_stream(ctx, logos, src, a.frames, W, H, bits, B, quirk, on_dev)
                    assert np.array_equal(out.view(np.uint32), exp[idx].view(np.uint32)), (cname, sname, B)
                    fps.append(a.frames / dt)
                rows.append({"B": B, "fps": float(np.median(fps)), "fps_runs": fps,
                             "h2d_per_frame": c[2] / a.frames, "d2h_per_frame": c[3] / a.frames})
            case["sources"][sname] = rows
        del dev, pinned, pageable
        torch.cuda.empty_cache()
    if ctx:
        ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
