"""Fused-step stream (amtk_scan_comb_stream) vs the logo scan stream and the comb stream fed the same frames back to back,
and vs one amtk_scan_comb_frames call on a whole pinned host clip, on 1080-line frames from host (pinned, pageable) and
device memory.

The fused stream sends every frame once and receives after every send, then finishes and drains.  The back-to-back pair
runs amtk_logo_scan_stream over all frames, then amtk_comb_stream over all frames (what the mirror's CMAnalyze and
AMTCombAnalyze pass 1 cost today when each pulls the source on its own, without the decode itself).  Frames are replayed
from --distinct seeded ones; logos are one 64x64 logo, or four 64x64 logos in the corners.

    python tools/bench_scan_comb_stream.py [--frames 1200] [--distinct 64] [--repeat 3] [--tiny]
    python tools/bench_scan_comb_stream.py --pitch [--frames 600] [--distinct 32] [--repeat 3] [--tiny]

--pitch measures ScanFrame's byte-pitch row step on 2-byte samples instead: the fused stream with reference_pitch = 1
against the logo scan stream (reference_pitch = 1) and the comb stream each fed every frame as it is sent (the mirror's
former 2-byte path), on pinned 1920x1080 and 3840x2160 YUV420P10 frames at B = 16 with one and four logos, checked
against one resident amtk_scan_comb_frames_pitch call.

Prints one JSON line: frames/s of each format, logo set, source and batch size (timed to a device synchronise, the median
of --repeat runs, each after a warm-up at the same batch size), H2D / D2H bytes per frame, launches per batch, and the
card's name, power limit and SM clocks read in the same command.  Every run's results are checked against one resident
amtk_scan_comb_frames call on the replayed frames.  --tiny rehearses at 320x180 with few frames; without a GPU it builds
the inputs and stops there.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import amatsukaze_b200 as ab  # noqa: E402
from amatsukaze_b200 import synth  # noqa: E402
from bench_comb_stream import gpu_info, make_distinct  # noqa: E402


def make_logos(kind, W, H):
    lg = synth.make_logo(64, 64, seed=3)["data"]
    spots = [(W - 64 - 40, 40)] if kind == "one64" else [(40, 40), (W - 104, 40), (40, H - 104), (W - 104, H - 104)]
    return [ab.Logo.create(lg, 64, 64, W, H, x, y).deint().create_mask(0.35) for x, y in spots]


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def fused(ctx, logos, descs, N, B):
    L = len(logos)
    sc, cn = np.empty((N, L, 2), np.float32), np.empty((N, 12), np.int32)
    s = ctx.scan_comb_stream(logos, None, B)
    n0, got = ctx.launches, 0
    for i in range(N):
        s.send(descs[i % len(descs)])
        a, b = s.recv(N - got)
        sc[got:got + len(a)], cn[got:got + len(a)] = a, b
        got += len(a)
    s.finish()
    a, b = s.recv(N - got)
    sc[got:got + len(a)], cn[got:got + len(a)] = a, b
    got += len(a)
    c, launches = s.counts(), ctx.launches - n0
    s.close()
    assert got == N
    return sc, cn, c, launches


def back_to_back(ctx, logos, descs, N, B):
    out = []
    for s in (ctx.logo_scan_stream(logos, B), ctx.comb_stream(None, B)):
        rows, got = [], 0
        for i in range(N):
            s.send(descs[i % len(descs)])
            r = s.recv(N - got)
            rows.append(r)
            got += len(r)
        s.finish()
        rows.append(s.recv(N - got))
        out.append((np.concatenate(rows), s.counts()))
        s.close()
    return out


def pitch_logos(kind, W, H):
    """One or four 64x64 logos inside the rows the byte-pitch step reads (imgy + h <= H / 2)."""
    lg = synth.make_logo(64, 64, seed=3)["data"]
    y1 = H // 2 - 104
    spots = [(W - 104, 40)] if kind == "one64" else [(40, 40), (W - 104, 40), (40, y1), (W - 104, y1)]
    return [ab.Logo.create(lg, 64, 64, W, H, x, y).deint().create_mask(0.35) for x, y in spots]


def fused_pitch(ctx, logos, descs, N, B):
    L = len(logos)
    sc, cn = np.empty((N, L, 2), np.float32), np.empty((N, 12), np.int32)
    s = ctx.scan_comb_stream(logos, None, B, reference_pitch=True)
    n0, got = ctx.launches, 0
    for i in range(N):
        s.send(descs[i % len(descs)])
        a, b = s.recv(N - got)
        sc[got:got + len(a)], cn[got:got + len(a)] = a, b
        got += len(a)
    s.finish()
    a, b = s.recv(N - got)
    sc[got:got + len(a)], cn[got:got + len(a)] = a, b
    got += len(a)
    c, launches = s.counts(), ctx.launches - n0
    s.close()
    assert got == N
    return sc, cn, c, launches


def two_streams(ctx, logos, descs, N, B):
    """The logo scan stream (reference_pitch = 1) and the comb stream, each fed every frame as it is sent."""
    L = len(logos)
    sc, cn = np.empty((N, L, 2), np.float32), np.empty((N, 12), np.int32)
    ls, cs = ctx.logo_scan_stream(logos, B, reference_pitch=True), ctx.comb_stream(None, B)
    n0, gs, gc = ctx.launches, 0, 0

    def drain():
        nonlocal gs, gc
        a = ls.recv(N - gs)
        sc[gs:gs + len(a)] = a
        gs += len(a)
        b = cs.recv(N - gc)
        cn[gc:gc + len(b)] = b
        gc += len(b)
    for i in range(N):
        ls.send(descs[i % len(descs)]); cs.send(descs[i % len(descs)])
        drain()
    ls.finish(); cs.finish()
    drain()
    c1, c2, launches = ls.counts(), cs.counts(), ctx.launches - n0
    ls.close(); cs.close()
    assert gs == gc == N
    return sc, cn, (c1[2] + c2[2], c1[3] + c2[3]), launches


def pitch_main(a):
    formats = [("yuv420p10_1920x1080", 1920, 1080), ("yuv420p10_3840x2160", 3840, 2160)]
    if a.tiny:
        formats = [("yuv420p10_320x180", 320, 180)]
        a.frames, a.distinct, a.repeat = min(a.frames, 120), min(a.distinct, 16), 1
    gpu = torch.cuda.is_available()
    res = {"metric": "scan_comb_stream_pitch", "frames": a.frames, "distinct": a.distinct, "repeat": a.repeat, "B": 16,
           "source": "pinned", "cases": []}
    res.update(gpu_info())
    ctx = None
    if gpu:
        torch.cuda.set_device(0)
        ctx = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    B, N = 16, a.frames
    for fname, W, H in formats:
        if not gpu:
            make_distinct(2, W, H, 10, "cpu")
            res["cases"].append({"format": fname, "note": "no GPU: inputs built, nothing measured"})
            continue
        dev = make_distinct(a.distinct, W, H, 10, "cuda")
        pinned = dev.cpu().pin_memory()
        descs = [ab.yv12_clip(pinned[i], W, H, 1, False, 10) for i in range(a.distinct)]
        idx = torch.arange(N, device="cuda") % a.distinct
        full = dev[idx].contiguous()
        for lname in ("one64", "corners4"):
            logos = pitch_logos(lname, W, H)
            clip = ab.yv12_clip(full, W, H, N, True, 10)
            es, ec = ctx.scan_comb_frames(clip, logos, pitch_elems_override=clip.pitch_y)
            es, ec = es.cpu().numpy(), ec.cpu().numpy()
            fused_pitch(ctx, logos, descs, 2 * B + 8, B)                                # warm-up
            two_streams(ctx, logos, descs, 2 * B + 8, B)
            f_fps, p_fps = [], []
            for _ in range(a.repeat):                                                # the two forms alternate
                dt, (sc, cn, c, fl) = timed(lambda: fused_pitch(ctx, logos, descs, N, B))
                assert np.array_equal(sc.view(np.uint32), es.view(np.uint32)) and np.array_equal(cn, ec), (fname, lname)
                f_fps.append(N / dt)
                dp, (ps, pc, pb, pl) = timed(lambda: two_streams(ctx, logos, descs, N, B))
                assert np.array_equal(ps.view(np.uint32), es.view(np.uint32)) and np.array_equal(pc, ec), (fname, lname)
                p_fps.append(N / dp)
            res["cases"].append({"format": fname, "logos": lname, "fps": float(np.median(f_fps)), "fps_runs": f_fps,
                                 "two_streams_fps": float(np.median(p_fps)), "two_streams_runs": p_fps,
                                 "h2d_per_frame": c[2] / N, "d2h_per_frame": c[3] / N,
                                 "two_streams_h2d_per_frame": pb[0] / N, "two_streams_d2h_per_frame": pb[1] / N,
                                 "launches_per_batch": fl / -(-N // B), "two_streams_launches_per_batch": pl / -(-N // B)})
            del logos
        del dev, pinned, full, descs
        torch.cuda.empty_cache()
    if ctx:
        res.update({"after": gpu_info()})
        ctx.close()
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1200)
    ap.add_argument("--whole-frames", type=int, default=480, help="frames of the pinned whole-clip call")
    ap.add_argument("--distinct", type=int, default=64, help="distinct seeded frames, replayed")
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--tiny", action="store_true", help="320x180 and few frames; without a GPU, stop after the inputs")
    ap.add_argument("--pitch", action="store_true", help="the byte-pitch row step on YUV420P10 (see above)")
    a = ap.parse_args()
    if a.pitch:
        return pitch_main(a)
    formats = [("yv12_1920x1080", 1920, 1080, 8), ("yuv420p10_1920x1080", 1920, 1080, 10)]
    if a.tiny:
        formats = [(n.split("_")[0] + "_320x180", 320, 180, b) for n, _, _, b in formats]
        a.frames, a.whole_frames, a.distinct, a.repeat = min(a.frames, 120), min(a.whole_frames, 48), min(a.distinct, 16), 1
    gpu = torch.cuda.is_available()
    res = {"metric": "scan_comb_stream", "frames": a.frames, "distinct": a.distinct, "repeat": a.repeat, "cases": []}
    res.update(gpu_info())
    ctx = None
    if gpu:
        torch.cuda.set_device(0)
        ctx = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    for fname, W, H, bits in formats:
        if not gpu:
            make_distinct(2, W, H, bits, "cpu")
            res["cases"].append({"format": fname, "note": "no GPU: inputs built, nothing measured"})
            continue
        dev = make_distinct(a.distinct, W, H, bits, "cuda")
        idx = torch.arange(max(a.frames, a.whole_frames), device="cuda") % a.distinct
        full = dev[idx].contiguous()
        pinned = dev.cpu().pin_memory()
        pageable = dev.cpu().numpy().copy()
        for lname in ("one64", "corners4"):
            logos = make_logos(lname, W, H)
            es, ec = ctx.scan_comb_frames(ab.yv12_clip(full, W, H, full.shape[0], True, bits), logos)
            es, ec = es.cpu().numpy(), ec.cpu().numpy()
            case = {"format": fname, "bits": bits, "logos": lname, "sources": {}}
            res["cases"].append(case)
            whole = full[:a.whole_frames].cpu().pin_memory()
            clip = ab.yv12_clip(whole, W, H, a.whole_frames, False, bits)
            ctx.scan_comb_frames(ab.yv12_clip(whole[:16], W, H, 16, False, bits), logos)          # warm-up
            tw, (ws, wc) = timed(lambda: ctx.scan_comb_frames(clip, logos))
            assert np.array_equal(ws.view(np.uint32), es[:a.whole_frames].view(np.uint32)) and np.array_equal(wc, ec[:a.whole_frames])
            case["whole_pinned_clip"] = {"fps": a.whole_frames / tw, "frames": a.whole_frames, "h2d_per_frame": ctx.last_h2d_bytes / a.whole_frames}
            del whole
            for sname, src, on_dev in (("pinned", pinned, False), ("pageable", pageable, False), ("device", dev, True)):
                descs = [ab.yv12_clip(src[i], W, H, 1, on_dev, bits) for i in range(a.distinct)]
                rows = []
                for B in (16, 64):
                    N = a.frames
                    fused(ctx, logos, descs, min(N, 2 * B + 32), B)                  # warm-up
                    back_to_back(ctx, logos, descs, min(N, 2 * B + 32), B)
                    f_fps, p_fps = [], []
                    for _ in range(a.repeat):                                        # the two forms alternate
                        dt, (sc, cn, c, launches) = timed(lambda: fused(ctx, logos, descs, N, B))
                        assert np.array_equal(sc.view(np.uint32), es[:N].view(np.uint32)) and np.array_equal(cn, ec[:N]), (fname, lname, sname, B)
                        f_fps.append(N / dt)
                        dp, ((ls, lc), (cs, cc)) = timed(lambda: back_to_back(ctx, logos, descs, N, B))
                        assert np.array_equal(ls.view(np.uint32), es[:N].view(np.uint32)) and np.array_equal(cs, ec[:N])
                        p_fps.append(N / dp)
                    rows.append({"B": B, "fps": float(np.median(f_fps)), "fps_runs": f_fps,
                                 "back_to_back_fps": float(np.median(p_fps)), "back_to_back_runs": p_fps,
                                 "h2d_per_frame": c[2] / N, "d2h_per_frame": c[3] / N,
                                 "back_to_back_h2d_per_frame": (lc[2] + cc[2]) / N,
                                 "launches_per_batch": launches / -(-N // B)})
                case["sources"][sname] = rows
            del logos
        del dev, full, pinned, pageable
        torch.cuda.empty_cache()
    if ctx:
        res.update({"after": gpu_info()})
        ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
