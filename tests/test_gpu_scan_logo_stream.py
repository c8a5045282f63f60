"""amtk_scan_logo_stream: the ScanLogo pipeline fed one decoded frame at a time (InitialLogoCreator::onFrame,
LogoScan.hpp:881-914).  Its logo file must equal amtk_scan_logo's on a clip of the same frames byte for byte; its
callbacks, `more` flags and counts must equal what `stream_rule` (the pure-Python restatement of the rule in DESIGN.md
section 3.3.1, checked against a port of onFrame in test_scan_logo_stream_rule.py) predicts."""
import ctypes as C
import os
import struct
import subprocess
import threading

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth

pytestmark = pytest.mark.gpu

W, H, SX, SY, SW, SH, THY = 320, 192, 200, 64, 64, 48, 12
BATCH = 200


# ---------------------------------------------------------------------------------------------------------------------
# the stream rule, restated
# ---------------------------------------------------------------------------------------------------------------------
def stream_rule(valid, max_frames, pos=None, size=None):
    """valid[i]: AddFrame's verdict on the i-th frame sent.  Returns a dict: stored (indices of the stored frames), calls
    (MakeInitialLogo callbacks as (float32 progress, nread, 0, ngather)), more (after every send), nread, ngather."""
    n = len(valid)
    pos = list(range(1, n + 1)) if pos is None else pos
    size = [max(1, n)] * n if size is None else size
    stored, calls, more = [], [], []
    cut = 0 if max_frames == 0 else None          # read count of the cut-off frame
    reads, batch = 0, []

    def resolve():
        nonlocal cut
        for i in batch:
            if valid[i] and len(stored) < max_frames:
                stored.append(i)
                if len(stored) == max_frames:
                    cut = i + 1
        batch.clear()
        if reads % BATCH == 0 and (cut is None or reads <= cut):
            r = reads
            calls.append((np.float32(np.float32(pos[r - 1]) / np.float32(size[r - 1])) * np.float32(50.0), r, 0, len(stored)))

    for i in range(n):
        if cut is not None:
            more.append(False)
            continue
        reads += 1
        batch.append(i)
        if reads % BATCH == 0:
            resolve()
        more.append(cut is None)
    if batch:
        resolve()                                  # finish: reads % 200 != 0 here, no callback
    nread = reads if cut is None else min(reads, cut)
    return {"stored": stored, "calls": calls, "more": more, "nread": nread, "ngather": len(stored)}


def remake_calls(num_frames):
    """ReMakeLogo x2 and the final callback (:977-982, :1071)."""
    out = []
    for base in (50.0, 75.0):
        out += [(np.float32(np.float32(i) / np.float32(num_frames) * np.float32(25.0) + np.float32(base)), i, num_frames, num_frames)
                for i in range(0, num_frames, 100)]
    out.append((np.float32(1.0), num_frames, num_frames, num_frames))
    return out


def _f32(calls):
    return [(np.float32(c[0]),) + tuple(c[1:]) for c in calls]


# ---------------------------------------------------------------------------------------------------------------------
# frames and feeding
# ---------------------------------------------------------------------------------------------------------------------
LOGO = synth.make_logo(SW, SH, seed=4)


@pytest.fixture(scope="module")
def clips():
    return {90: synth.make_frames(0, 90, W, H, seed=0x5EED0004, device="cuda", mode="flat", logo=LOGO, imgx=SX, imgy=SY),
            450: synth.make_frames(0, 450, W, H, seed=0x5EED0005, device="cuda", mode="flat", logo=LOGO, imgx=SX, imgy=SY)}


def _valid(ctx, fr, w=W, h=H, sx=SX, sy=SY, sw=SW, sh=SH, thy=THY):
    acc = ctx.logo_scan(sw, sh, thy)
    return [bool(v) for v in acc.add_frames(ab.yv12_clip(fr, w, h, fr.shape[0], True), sx, sy)]


def _one(frame, w, h, on_device):
    return ab.yv12_clip(frame, w, h, 1, on_device)


class Source:
    """One-frame descriptors of a packed clip: 'device', 'pinned', 'pageable', 'mix' (cycling through the three), or a
    padded V-first host layout with poisoned padding ('layout')."""

    def __init__(self, fr, w, h, kind):
        self.fr, self.w, self.h, self.kind = fr, w, h, kind
        self.host = fr.cpu().numpy()
        self.keep = []

    def clip(self, i):
        i %= self.fr.shape[0]
        kind = self.kind if self.kind != "mix" else ("device", "pinned", "pageable")[i % 3]
        if kind == "device":
            return _one(self.fr[i:i + 1], self.w, self.h, True)
        if kind == "pinned":
            t = torch.from_numpy(self.host[i:i + 1].copy()).pin_memory()
            self.keep = [t]
            return _one(t, self.w, self.h, False)
        if kind == "pageable":
            a = self.host[i:i + 1].copy()
            self.keep = [a]
            return _one(a, self.w, self.h, False)
        return self._layout(i)

    def _layout(self, i):
        w, h = self.w, self.h
        py, pc = w + 48, w // 2 + 40
        Y, U, V = synth.split_planes(self.host[i:i + 1], w, h)
        rng = np.random.default_rng(i)
        buf = rng.integers(0, 256, py * h + 2 * pc * (h // 2) + 4096 + 7, dtype=np.uint8)     # poisoned padding
        offv = py * h + 16
        offu = offv + pc * (h // 2) + 3
        buf[:py * h].reshape(h, py)[:, :w] = Y[0]
        buf[offv:offv + pc * (h // 2)].reshape(h // 2, pc)[:, :w // 2] = V[0]
        buf[offu:offu + pc * (h // 2)].reshape(h // 2, pc)[:, :w // 2] = U[0]
        d = ab.ClipDesc()
        d.base = buf.ctypes.data
        d.frame_stride = len(buf) - 5                       # not a whole number of rows
        d.off_u, d.off_v = offu, offv
        d.width, d.height, d.pitch_y, d.pitch_uv = w, h, py, pc
        d.log_uvx = d.log_uvy = 1
        d.bytes_per_sample, d.bits_per_sample, d.num_frames, d.on_device = 1, 8, 1, 0
        self.keep = [buf]
        return d


def _stream(ctx, tmp_path, fr, max_frames, name, kind="device", pos=None, size=None, w=W, h=H, sx=SX, sy=SY, sid=7, thy=THY):
    """Feeds every frame of fr and finishes.  Returns (calls, mores, counts, file bytes)."""
    calls, mores = [], []
    s = ctx.scan_logo_stream(sx, sy, SW, SH, thy, max_frames, cb=lambda *a: calls.append(a) or True)
    src = Source(fr, w, h, kind)
    n = fr.shape[0]
    pos = list(range(1, n + 1)) if pos is None else pos
    size = [n] * n if size is None else size
    for i in range(n):
        mores.append(s.send(src.clip(i), pos[i], size[i]))
    dst = str(tmp_path / name)
    s.finish(dst, sid)
    counts = s.counts()                                 # finish resolved the open batch
    s.close()
    return calls, mores, counts, open(dst, "rb").read()


def _whole(ctx, tmp_path, fr, max_frames, name, w=W, h=H, sx=SX, sy=SY, sid=7, thy=THY):
    dst = str(tmp_path / name)
    ctx.scan_logo(ab.yv12_clip(fr, w, h, fr.shape[0], True), dst, sx, sy, SW, SH, thy, max_frames, service_id=sid)
    return open(dst, "rb").read()


def _payload(w=SW, h=SH):
    return w * h + 2 * (w >> 1) * (h >> 1)


# ---------------------------------------------------------------------------------------------------------------------
# 1 + 2: equality with amtk_scan_logo, callbacks, more, counts
# ---------------------------------------------------------------------------------------------------------------------
def _cases(valid450):
    nv = np.concatenate([[0], np.cumsum(valid450)])
    mid = next(r for r in range(290, 320) if valid450[r - 1])        # a valid frame inside the second batch
    on200 = next(r for r in (200, 400) if valid450[r - 1])
    return ([(90, 40), (90, 100000), (450, 40), (450, 100000), (450, int(nv[mid])), (450, int(nv[on200])), (90, 1), (450, 1)],
            mid, on200, nv)


def test_stream_equals_whole_clip(ctx, clips, tmp_path):
    v = {n: _valid(ctx, fr) for n, fr in clips.items()}
    cases, mid, on200, nv = _cases(v[450])
    rng = np.random.default_rng(11)
    for n, maxf in cases:
        fr = clips[n]
        pos = list(np.cumsum(rng.integers(1, 5_000_000, n)))           # irregular reader positions and sizes
        size = [int(pos[-1]) + int(x) for x in rng.integers(1, 3_000_000, n)]
        try:
            want = _whole(ctx, tmp_path, fr, maxf, "w.lgd")
        except ab.AmtkError as e:                      # max_frames = 1: GetLogo has too few frames in both
            assert maxf == 1 and "Insufficient logo frames" in str(e)
            with pytest.raises(ab.AmtkError, match="Insufficient logo frames"):
                _stream(ctx, tmp_path, fr, maxf, "s.lgd", pos=pos, size=size)
            continue
        calls, mores, counts, got = _stream(ctx, tmp_path, fr, maxf, "s.lgd", pos=pos, size=size)
        assert got == want, (n, maxf)
        rule = stream_rule(v[n], maxf, pos, size)
        assert mores == rule["more"], (n, maxf)
        assert _f32(calls) == _f32(rule["calls"] + remake_calls(rule["ngather"])), (n, maxf)
        assert counts[:2] == (rule["nread"], rule["ngather"]) and counts[2] == 0, (n, maxf, counts)
    # the cut-off cases really cut where intended
    assert stream_rule(v[450], int(nv[mid]))["nread"] == mid
    assert stream_rule(v[450], int(nv[on200]))["nread"] == on200
    assert stream_rule(v[450], int(nv[on200]))["calls"][-1][1] == on200


def test_frames_after_the_cutoff_change_nothing(ctx, clips, tmp_path):
    fr = clips[450]
    v = _valid(ctx, fr)
    rule = stream_rule(v, 40)
    stop = rule["more"].index(False) + 1               # the send that resolves the batch holding the cut-off (r = 200)
    assert stop == 200 and rule["nread"] < 200
    want = _whole(ctx, tmp_path, fr, 40, "w.lgd")
    for extra in (0, 250):
        calls = []
        s = ctx.scan_logo_stream(SX, SY, SW, SH, THY, 40, cb=lambda *a: calls.append(a) or True)
        src = Source(fr, W, H, "pinned")
        mores = [s.send(src.clip(i), i + 1, 450) for i in range(stop + extra)]
        assert mores == rule["more"][:stop] + [False] * extra
        s.finish(str(tmp_path / "s.lgd"), 7)
        assert open(str(tmp_path / "s.lgd"), "rb").read() == want
        assert _f32(calls) == _f32(rule["calls"] + remake_calls(40))
        assert s.counts() == (rule["nread"], 40, stop * _payload())          # frames after more == 0 are not copied
        s.close()


def test_oracle_rebuild(ctx, oracle, clips, tmp_path):
    """The logo the stream writes equals the pipeline composed from the oracle's pieces (as test_scan_logo_pipeline)."""
    po = oracle
    fr, maxf, n = clips[90], 40, 90
    _, _, _, got = _stream(ctx, tmp_path, fr, maxf, "o.lgd", kind="mix")
    Y, U, V = synth.split_planes(fr, W, H)
    roi = lambda i: (Y[i][SY:SY + SH, SX:SX + SW], U[i][SY // 2:(SY + SH) // 2, SX // 2:(SX + SW) // 2],
                     V[i][SY // 2:(SY + SH) // 2, SX // 2:(SX + SW) // 2])
    sc = po.OracleScan(SW, SH, THY)
    stored = []
    for i in range(n):
        if len(stored) >= maxf:
            break
        if sc.add_frame(*roi(i)):
            stored.append(i)
    data = sc.get_logo(255, False)
    for _ in range(2):
        de = po.OracleLogo.create(data, SW, SH, SW, SH, 0, 0).deint().create_mask(0.1)
        keep = []
        for i in stored:
            ry = np.ascontiguousarray(roi(i)[0])
            dd = np.zeros(SW * SH + 8, np.float32)
            po.oracle_lib().amtk_or_deint_y_u8(dd.ctypes.data_as(po.c_float_p), ry.ctypes.data_as(po.c_u8_p), SW, SW, SH)
            res = [abs(np.float32(de.evaluate(dd, 255.0, np.float32(0.1) * np.float32(fi)))) for fi in range(20)]
            if int(np.argmin(res)) > 8:
                keep.append(i)
        sc2 = po.OracleScan(SW, SH, THY)
        for i in keep:
            sc2.add_frame(*roi(i))
        data = sc2.get_logo(255, True)
    path = str(tmp_path / "o.lgd")
    lg = ab.Logo.load(path)
    assert np.array_equal(lg.tables()["data"].view(np.uint32), data.view(np.uint32))
    gi = lg.info()
    assert (gi.w, gi.h, gi.imgw, gi.imgh, gi.imgx, gi.imgy) == (SW, SH, W, H, SX, SY)


def test_insufficient_frames_fail_alike(ctx, clips, tmp_path):
    fr = clips[90]
    for maxf, thy in ((0, THY), (40, 0)):
        with pytest.raises(ab.AmtkError, match="Insufficient logo frames"):
            _whole(ctx, tmp_path, fr, maxf, "w.lgd", thy=thy)
        s = ctx.scan_logo_stream(SX, SY, SW, SH, thy, maxf)
        mores = [s.send(_one(fr[i:i + 1], W, H, True), i + 1, 90) for i in range(90)]
        if maxf == 0:
            assert not any(mores) and s.counts() == (0, 0, 0)
        with pytest.raises(ab.AmtkError, match="Insufficient logo frames"):
            s.finish(str(tmp_path / "s.lgd"))
        s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3: cancel
# ---------------------------------------------------------------------------------------------------------------------
def test_cancel(ctx, clips, tmp_path):
    fr = clips[450]
    v = _valid(ctx, fr)
    rule = stream_rule(v, 100000)
    want = rule["calls"] + remake_calls(rule["ngather"])
    first = len(rule["calls"])
    n_remake = (rule["ngather"] + 99) // 100
    for stop in (1, first + 1, first + n_remake + 1, len(want)):     # a 200-frame callback, ReMakeLogo 1 and 2, the final one
        seen = []
        s = ctx.scan_logo_stream(SX, SY, SW, SH, THY, 100000, cb=lambda *a: seen.append(a) or len(seen) < stop)
        failed_at = None
        for i in range(450):
            try:
                s.send(_one(fr[i:i + 1], W, H, True), i + 1, 450)
            except ab.AmtkError as e:
                assert "Cancel requested" in str(e)
                failed_at = i
                break
        if stop <= first:
            assert failed_at == 199
        else:
            assert failed_at is None
            with pytest.raises(ab.AmtkError, match="Cancel requested"):
                s.finish(str(tmp_path / "c.lgd"))
        assert _f32(seen) == _f32(want[:stop])
        with pytest.raises(ab.AmtkError, match="closed"):
            s.send(_one(fr[0:1], W, H, True), 1, 450)
        with pytest.raises(ab.AmtkError, match="closed"):
            s.finish(str(tmp_path / "c.lgd"))
        s.counts()
        s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4: sources and layouts
# ---------------------------------------------------------------------------------------------------------------------
def test_sources_and_layouts(ctx, clips, tmp_path):
    fr = clips[450]
    v = _valid(ctx, fr)
    for maxf in (100000, 250):
        rule = stream_rule(v, maxf)
        want = _whole(ctx, tmp_path, fr, maxf, "w.lgd")
        hostframes = next((i + 1 for i, m in enumerate(rule["more"]) if not m), 450)
        for kind in ("device", "pinned", "pageable", "mix", "layout"):
            _, mores, counts, got = _stream(ctx, tmp_path, fr, maxf, "s.lgd", kind=kind)
            assert got == want, (maxf, kind)
            assert mores == rule["more"]
            nhost = {"device": 0, "mix": sum(1 for i in range(hostframes) if i % 3), }.get(kind, hostframes)
            assert counts == (rule["nread"], rule["ngather"], nhost * _payload()), (maxf, kind, counts)


def test_1080p_rectangle_on_the_edges(ctx, tmp_path):
    w, h, n = 1920, 1080, 40
    sx, sy = w - SW, h - SH
    fr = synth.make_frames(0, n, w, h, seed=0x5EED0006, device="cuda", mode="flat", logo=LOGO, imgx=sx, imgy=sy)
    want = _whole(ctx, tmp_path, fr, 100000, "w.lgd", w=w, h=h, sx=sx, sy=sy)
    for kind in ("device", "pageable"):
        _, _, _, got = _stream(ctx, tmp_path, fr, 100000, "s.lgd", kind=kind, w=w, h=h, sx=sx, sy=sy)
        assert got == want, kind


# ---------------------------------------------------------------------------------------------------------------------
# 5: destroy at every stage, later streams unaffected
# ---------------------------------------------------------------------------------------------------------------------
def test_destroy_at_every_stage(ctx, clips, tmp_path):
    fr = clips[450]
    want = _stream(ctx, tmp_path, fr, 100000, "a.lgd")
    ctx.scan_logo_stream(SX, SY, SW, SH, THY, 100).close()                         # before any send
    s = ctx.scan_logo_stream(SX, SY, SW, SH, THY, 100000)
    for i in range(250):                                                             # middle of a batch
        s.send(_one(fr[i:i + 1], W, H, True), i + 1, 450)
    s.close()
    s = ctx.scan_logo_stream(SX, SY, SW, SH, THY, 100000, cb=lambda *a: False)      # after a cancel
    with pytest.raises(ab.AmtkError, match="Cancel"):
        for i in range(250):
            s.send(_one(fr[i:i + 1], W, H, True), i + 1, 450)
    s.close()
    assert _stream(ctx, tmp_path, fr, 100000, "b.lgd") == want                     # after finish (inside _stream)
    fresh = ab.Context(0, torch.cuda.current_stream().cuda_stream)
    try:
        assert _stream(fresh, tmp_path, fr, 100000, "c.lgd") == want
    finally:
        fresh.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6: rejections, refusals, independence
# ---------------------------------------------------------------------------------------------------------------------
def test_rejected_frames_leave_the_stream_unchanged(ctx, clips, tmp_path):
    fr = clips[90]
    want = _stream(ctx, tmp_path, fr, 40, "a.lgd")[3]
    s = ctx.scan_logo_stream(SX, SY, SW, SH, THY, 40)
    small = synth.make_frames(0, 1, 160, 96, device="cuda", mode="flat")
    with pytest.raises(ab.AmtkError, match="outside"):                             # rectangle outside the first frame
        s.send(_one(small, 160, 96, True), 1, 90)
    f16 = torch.zeros((1, W * H * 3), dtype=torch.uint8, device="cuda")
    bad = [ab.yv12_clip(f16, W, H, 1, True, bits=10)]                              # 10-bit
    d = _one(fr[0:1], W, H, True); d.num_frames = 2; bad.append(d)                 # two frames
    d = _one(fr[0:1], W, H, True); d.num_frames = 0; bad.append(d)                 # no frame
    for i in range(90):
        if i == 5:
            for b in bad + [_one(small, 160, 96, True)]:                            # + a size change
                with pytest.raises(ab.AmtkError):
                    s.send(b, 1, 90)
            d = _one(fr[0:1], W, H, True); d.log_uvy = 0                             # subsampling change
            with pytest.raises(ab.AmtkError):
                s.send(d, 1, 90)
            with pytest.raises(ab.AmtkError, match="size"):                          # size < 1
                s.send(_one(fr[0:1], W, H, True), 1, 0)
        s.send(_one(fr[i:i + 1], W, H, True), i + 1, 90)
    s.finish(str(tmp_path / "b.lgd"), 7)
    assert open(str(tmp_path / "b.lgd"), "rb").read() == want


def test_refusals(ctx, clips, tmp_path):
    L = ab.lib()
    out = C.c_void_p()
    for args in ((SX, SY, 3, SH), (SX, SY, SW, 3), (SX, SY, 4097, SH), (SX, SY, SW, 4097), (-2, SY, SW, SH), (SX, -2, SW, SH)):
        assert not L.amtk_scan_logo_stream_create(ctx.h, args[0], args[1], args[2], args[3], THY, 10, None, C.byref(out))
    assert not L.amtk_scan_logo_stream_create(ctx.h, SX, SY, SW, SH, THY, -1, None, C.byref(out))
    assert not L.amtk_scan_logo_stream_create(None, SX, SY, SW, SH, THY, 10, None, C.byref(out))
    assert not L.amtk_scan_logo_stream_create(ctx.h, SX, SY, SW, SH, THY, 10, None, None)
    s = ctx.scan_logo_stream(SX, SY, SW, SH, THY, 10)
    with pytest.raises(ab.AmtkError, match="without any frame"):
        s.finish(str(tmp_path / "x.lgd"))
    with pytest.raises(ab.AmtkError, match="closed"):
        s.send(_one(clips[90][0:1], W, H, True), 1, 90)
    with pytest.raises(ab.AmtkError, match="closed"):
        s.finish(str(tmp_path / "x.lgd"))
    s.close()
    s = ctx.scan_logo_stream(SX, SY, SW, SH, THY, 10)
    for i in range(60):
        s.send(_one(clips[90][i:i + 1], W, H, True), i + 1, 90)
    s.finish(str(tmp_path / "y.lgd"))
    with pytest.raises(ab.AmtkError, match="closed"):
        s.send(_one(clips[90][0:1], W, H, True), 1, 90)
    with pytest.raises(ab.AmtkError, match="closed"):
        s.finish(str(tmp_path / "y.lgd"))
    s.close()


def test_streams_are_independent(ctx, clips, tmp_path):
    a_fr, b_fr = clips[450], clips[90]
    want_a = _stream(ctx, tmp_path, a_fr, 100000, "a.lgd")[3]
    want_b = _stream(ctx, tmp_path, b_fr, 40, "b.lgd")[3]
    sa = ctx.scan_logo_stream(SX, SY, SW, SH, THY, 100000)
    sb = ctx.scan_logo_stream(SX, SY, SW, SH, THY, 40)
    src_b = Source(b_fr, W, H, "mix")
    for i in range(450):                                                              # fed alternately
        sa.send(_one(a_fr[i:i + 1], W, H, True), i + 1, 450)
        if i < 90:
            sb.send(src_b.clip(i), i + 1, 90)
    sb.finish(str(tmp_path / "b2.lgd"), 7)
    sa.finish(str(tmp_path / "a2.lgd"), 7)
    sa.close(); sb.close()
    assert open(str(tmp_path / "a2.lgd"), "rb").read() == want_a
    assert open(str(tmp_path / "b2.lgd"), "rb").read() == want_b
    # two host threads, each driving a stream on the same context
    errors = []

    def run(fr, maxf, name, kind):
        try:
            # the device source's frames live on the current device of this thread
            torch.cuda.set_device(0)
            _stream(ctx, tmp_path, fr, maxf, name, kind=kind)
        except Exception as e:          # noqa: BLE001 -- reported below
            errors.append(e)

    ts = [threading.Thread(target=run, args=(a_fr, 100000, "a3.lgd", "pageable")),
          threading.Thread(target=run, args=(b_fr, 40, "b3.lgd", "device"))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    assert open(str(tmp_path / "a3.lgd"), "rb").read() == want_a
    assert open(str(tmp_path / "b3.lgd"), "rb").read() == want_b


# ---------------------------------------------------------------------------------------------------------------------
# the host-side mirror: logo::LogoAnalyzer (tests/cpp/test_scan_logo_stream.cpp)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("maxf", [100000, 250, 40])
def test_mirror_logo_analyzer(ctx, clips, tmp_path, maxf):
    from amatsukaze_b200 import _build
    exe = _build.build_scan_logo_stream_test() if os.path.exists("/usr/bin/g++") else _build.SCAN_LOGO_STREAM_TEST
    fr = clips[450]
    n = fr.shape[0]
    with open(tmp_path / "src.dat", "wb") as f:
        f.write(b"AMTSRAW1" + struct.pack("<6i", W, H, 8, n, 30000, 1001))
        f.write(fr.cpu().numpy().tobytes())
    args = [tmp_path / "src.dat", SX, SY, SW, SH, THY, maxf, 7, tmp_path / "cpu.lgd", tmp_path / "dev.lgd"]
    r = subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    want = _whole(ctx, tmp_path, fr, maxf, "w.lgd")
    assert open(tmp_path / "cpu.lgd", "rb").read() == want
    assert open(tmp_path / "dev.lgd", "rb").read() == want
    rule = stream_rule(_valid(ctx, fr), maxf)
    asked = next((i + 1 for i, m in enumerate(rule["more"]) if not m), n)     # up to the end of the cut-off's batch
    assert "cpu: asked=%d in_order=1" % asked in r.stdout, r.stdout
    assert "device: frames_asked=0" in r.stdout, r.stdout
