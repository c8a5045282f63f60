"""When a call is done with the caller's host memory.

A call that takes host memory (a host clip or frame, or a host array such as fades, frame_result, frame_select or
top_idx / bottom_idx) returns only when it no longer reads that memory; its host outputs are complete when it returns
(include/amtk_b200.h, beside amtk_clip).  Real callers rely on it: a decoder reuses a small pool of frame buffers,
AviSynth's cache hands the same frame memory back out, and INTEGRATION.md section 5e loops
amtk_logo_find_add_frames over decoded frames in one buffer.  A call that returned with a copy still queued would read
the next picture.

Every case holds the context's stream with a device spin of about 100 ms (`hold`) before the call, so that whatever the
call leaves queued behind that stream is still pending when it returns.  As soon as the call returns it copies the host
outputs, overwrites every input byte the call could still read with a value the data never holds, and only then
synchronises and compares with the same call on a device-resident copy (which the other suites pin to the oracles).
AMTK_STAGE_MB=1 cuts every host clip here into at least three staging chunks; the upload of chunk k >= 2 waits on the
device for the work of chunk k - 2, which is queued behind the hold.  Pinned memory is what shows a late read: the driver
copies pageable memory into its own staging before an asynchronous copy returns, so pageable cases pass either way.

Calls on device clips with device outputs stay asynchronous: under a hold they return with the stream still busy.
"""
import ctypes as C
import functools
import itertools

import numpy as np
import pytest
import torch

import amatsukaze_b200 as ab
from amatsukaze_b200 import capi, synth

pytestmark = pytest.mark.gpu

HOLD_CYCLES = 200_000_000          # about 100 ms at the H100's 1.98 GHz clock; the exact length does not matter
MEMS = ("pinned", "pageable")

BW, BH, BN = 1920, 1080, 6         # whole-frame staging: a 1080p frame is more than 1 MB, so every frame is a chunk
SW, SH, SN = 640, 360, 150         # rectangle staging: 150 frames of a 128 x 96 rectangle are 3 or more 1 MB chunks
LA = (64, 48, 128, 96)             # logo rectangles (x, y, w, h) on the 1080p clip; their bounding box is most of a frame
LB = (1728, 960, 128, 96)
LS = (400, 200, 128, 96)           # the logo and scan rectangle on the 640 x 360 clip
LT = (400, 16, 128, 96)            # a logo high enough in that frame for ScanFrame's byte-pitch row step on 2-byte samples


@pytest.fixture(autouse=True)
def stage_1mb(monkeypatch):
    monkeypatch.setenv("AMTK_STAGE_MB", "1")          # read on every call


def hold():
    """Enqueues a bounded device spin on torch's current stream, the stream the session context runs on."""
    torch.cuda._sleep(HOLD_CYCLES)


# ---------------------------------------------------------------------------------------------------------------------
# data and memory
# ---------------------------------------------------------------------------------------------------------------------
def widen(f, bits):
    return f if bits == 8 else (f.astype(np.uint16) << (bits - 8))


@functools.lru_cache(None)
def big(bits):
    lg = synth.make_logo(LA[2], LA[3], seed=2)
    f = synth.make_frames(0, BN, BW, BH, device="cuda", logo=lg, imgx=LA[0], imgy=LA[1], logo_period=4).cpu().numpy()
    return widen(f, bits)


@functools.lru_cache(None)
def small(bits):
    lg = synth.make_logo(LS[2], LS[3], seed=5)
    f = synth.make_frames(0, SN, SW, SH, device="cuda", mode="flat", logo=lg, imgx=LS[0], imgy=LS[1]).cpu().numpy()
    return widen(f, bits)


@functools.lru_cache(None)
def moving(bits, n=24):
    """Telecined 640 x 360 frames with the LS logo fading in and out, for the frame streams."""
    lg = synth.make_logo(LS[2], LS[3], seed=5)
    f = synth.make_frames(0, n, SW, SH, device="cuda", mode="telecine", logo=lg, imgx=LS[0], imgy=LS[1],
                          logo_period=12).cpu().numpy()
    return widen(f, bits)


_absent = {}


def absent(a):
    """A sample value within the clip's range (8 or 10 bits) that the frames `a` never hold: the poison."""
    if id(a) not in _absent:        # the entry holds `a`, so that its id is not reused
        top = 256 if a.dtype == np.uint8 else 1024
        free = np.flatnonzero(np.bincount(a.ravel(), minlength=top)[:top] == 0)
        assert free.size, "the frames use every sample value"
        _absent[id(a)] = (a, a.dtype.type(free[-1]))
    return _absent[id(a)][1]


def host(a, mem):
    """A copy of the numpy array a in new host memory, page-locked or pageable."""
    if mem == "pinned":
        out = torch.empty(a.nbytes, dtype=torch.uint8, pin_memory=True).numpy().view(a.dtype).reshape(a.shape)
    else:
        out = np.empty_like(a)
    out[...] = a
    return out


def device(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8)).cuda()


def clip(buf, w, h, bits, n=None):
    on_dev = isinstance(buf, torch.Tensor)
    return ab.yv12_clip(buf, w, h, buf.shape[0] if n is None else n, on_dev, bits)


def deint(rect, w, h, seed):
    x, y, lw, lh = rect
    return ab.Logo.create(synth.make_logo(lw, lh, seed=seed)["data"], lw, lh, w, h, x, y).deint().create_mask(0.35)


def raw_logo(rect, w, h, seed):
    x, y, lw, lh = rect
    return ab.Logo.create(synth.make_logo(lw, lh, seed=seed)["data"], lw, lh, w, h, x, y)


def as_np(x):
    if isinstance(x, torch.Tensor):
        return x.cpu().numpy()
    if isinstance(x, (tuple, list)):
        return tuple(as_np(v) for v in x)
    return x


def snapshot(x):
    """Host arrays copied as they are now; device tensors and immutable values as they are."""
    if isinstance(x, np.ndarray):
        return x.copy()
    if isinstance(x, (tuple, list)):
        return tuple(snapshot(v) for v in x)
    return x


def assert_same(got, want, what=""):
    """Bit for bit (float results included)."""
    if isinstance(want, tuple):
        assert isinstance(got, tuple) and len(got) == len(want), what
        for i, (g, w) in enumerate(zip(got, want)):
            assert_same(g, w, "%s[%d]" % (what, i))
        return
    if isinstance(want, np.ndarray):
        g, w = np.ascontiguousarray(got), np.ascontiguousarray(want)
        assert g.shape == w.shape and g.dtype == w.dtype, what
        bad = np.flatnonzero(g.view(np.uint8) != w.view(np.uint8))
        assert bad.size == 0, "%s: %d bytes differ, first at byte %d" % (what, bad.size, bad[0])
        return
    assert got == want, what


def held(ctx, call, *poisons):
    """hold, call(), copy its host outputs, run every poison, then wait for the context.  Returns the copies."""
    hold()
    out = snapshot(call())
    for p in poisons:
        p()
    ctx.synchronize()
    torch.cuda.synchronize()
    return out


def fill(a, v):
    return lambda: a.fill(v)


def run_case(ctx, src, mem, call, extras=()):
    """call(buf, *arrays) with buf the clip's frames: a device tensor for the expectation, host memory (`mem`) for the two
    calls after it.  The first host call runs unheld, so that every buffer the call grows exists before the hold; the
    second is held, and its frames and its copies of `extras` ((array, poison) pairs: poison(copy) overwrites the copy)
    are poisoned as soon as it returns."""
    fresh = lambda: [host(a, mem) for a, _ in extras]
    want = as_np(call(device(src), *fresh()))
    call(host(src, mem), *fresh())
    torch.cuda.synchronize()
    buf, ex = host(src, mem), fresh()
    got = held(ctx, lambda: call(buf, *ex), fill(buf, absent(src)), *[functools.partial(p, e) for (_, p), e in zip(extras, ex)])
    assert_same(as_np(got), want)


def raw_bytes(buf):
    """Frames as bytes, host or device (the device copies of a clip are byte tensors)."""
    return buf.view(np.uint8) if isinstance(buf, np.ndarray) else buf


def out_tensor(out_dev, shape, dtype):
    return torch.empty(shape, dtype=dtype, device="cuda") if out_dev else None


# ---------------------------------------------------------------------------------------------------------------------
# one-shot calls on host clips
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out_dev", [0, 1])
@pytest.mark.parametrize("bits,pitch", [(8, False), (10, False), (10, True)])
@pytest.mark.parametrize("mem", MEMS)
def test_logo_scan_frames(ctx, mem, bits, pitch, out_dev):
    """Two logos in opposite corners stage nearly whole frames; pitch_elems_override stages whole frames."""
    logos = [deint(LA, BW, BH, 2)] if pitch else [deint(LA, BW, BH, 2), deint(LB, BW, BH, 3)]
    out = out_tensor(out_dev, (BN, len(logos), 2), torch.float32)

    def call(buf):
        c = clip(buf, BW, BH, bits)
        return ctx.scan_frames(c, logos, out=out, pitch_elems_override=c.pitch_y if pitch else 0)
    run_case(ctx, big(bits), mem, call)


@pytest.mark.parametrize("out_dev", [0, 1])
@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("mem", MEMS)
def test_logo_analyze_frames(ctx, mem, bits, out_dev):
    raw = raw_logo(LS, SW, SH, 5)
    de, top, bot = raw.deint().create_mask(0.35), raw.field(0).create_mask(0.35), raw.field(1).create_mask(0.35)
    out = out_tensor(out_dev, (SN, 33), torch.float32)
    run_case(ctx, small(bits), mem, lambda buf: ctx.analyze_frames(clip(buf, SW, SH, bits), de, top, bot, out=out))


@pytest.mark.parametrize("out_dev", [0, 1])
@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("mem", MEMS)
def test_logo_eval_fades(ctx, mem, bits, out_dev):
    de = deint(LS, SW, SH, 5)
    fades = np.arange(20, dtype=np.float32) * np.float32(0.1)
    out = out_tensor(out_dev, (SN, 20), torch.float32)
    run_case(ctx, small(bits), mem, lambda buf, f: ctx.eval_fades(clip(buf, SW, SH, bits), de, f, out=out),
             [(fades, lambda a: a.fill(np.nan))])


@pytest.mark.parametrize("out_dev", [0, 1])
@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("mem", MEMS)
def test_comb_frames(ctx, mem, bits, out_dev):
    out = out_tensor(out_dev, (BN, 12), torch.int32)
    run_case(ctx, big(bits), mem, lambda buf: ctx.comb_frames(clip(buf, BW, BH, bits), out=out))


@pytest.mark.parametrize("out_dev", [0, 1])
@pytest.mark.parametrize("pitch", [False, True], ids=["scan_comb_frames", "scan_comb_frames_pitch"])
@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("mem", MEMS)
def test_scan_comb_frames(ctx, mem, bits, pitch, out_dev):
    """The fused step; with `pitch` through amtk_scan_comb_frames_pitch at the clip's byte pitch (ScanFrame's row step)."""
    logos = [deint(LA, BW, BH, 2)]
    scores, counts = out_tensor(out_dev, (BN, 1, 2), torch.float32), out_tensor(out_dev, (BN, 12), torch.int32)

    def call(buf):
        c = clip(buf, BW, BH, bits)
        return ctx.scan_comb_frames(c, logos, scores=scores, counts=counts, pitch_elems_override=c.pitch_y if pitch else 0)
    run_case(ctx, big(bits), mem, call)


@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("mem", MEMS)
def test_scan_add_frames(ctx, mem, bits):
    """LogoScan accumulation with a frame selection: valid_out is complete on return, the sums follow."""
    thy = 12 << (bits - 8)
    accs = [ctx.logo_scan(LS[2], LS[3], thy) for _ in range(3)]      # expectation, unheld, held
    order = iter(accs)
    select = (np.arange(SN) % 5 != 2).astype(np.uint8)
    run_case(ctx, small(bits), mem, lambda buf, sel: next(order).add_frames(clip(buf, SW, SH, bits), LS[0], LS[1], select=sel),
             [(select, lambda a: np.copyto(a, 1 - a))])
    assert accs[2].num_valid == accs[0].num_valid > 0
    assert_same(accs[2].sums(), accs[0].sums())


@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("mem", MEMS)
def test_scan_logo(ctx, mem, bits, tmp_path):
    """The ScanLogo pipeline: the logo file is written when the call returns."""
    names = (str(tmp_path / ("%d.lgd" % k)) for k in itertools.count())

    def call(buf):
        path = next(names)
        ctx.scan_logo(clip(buf, SW, SH, bits), path, LS[0], LS[1], LS[2], LS[3], 12 << (bits - 8), 60)
        with open(path, "rb") as f:
            return f.read()
    run_case(ctx, small(bits), mem, call)


@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("mem", MEMS)
def test_erase_logo_frames(ctx, mem, bits):
    """Erase in place: the rectangles of the host clip are final on return."""
    raw = raw_logo(LS, SW, SH, 5)
    fades = np.stack([np.linspace(0, 1, SN), np.linspace(1, 0, SN)], axis=1).astype(np.float32)

    def call(buf, f):
        ctx.erase_logo(clip(buf, SW, SH, bits), raw, f)
        return raw_bytes(buf)
    run_case(ctx, small(bits), mem, call, [(fades, lambda a: a.fill(np.nan))])


@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("mem", MEMS)
def test_erase_logo_clip(ctx, mem, bits):
    """AMTEraseLogo(AMTAnalyzeLogo(...)) in place on a host clip: frames and fades final on return."""
    raw = raw_logo(LS, SW, SH, 5)
    frame_result = np.repeat(np.array([0, 1, 2, 1, 0], np.uint8), SN // 5)

    def call(buf, fr):
        fades = ctx.erase_logo_clip(clip(buf, SW, SH, bits), raw, None, fr, 16)
        return fades, raw_bytes(buf)
    run_case(ctx, small(bits), mem, call, [(frame_result, lambda a: np.copyto(a, (a + 1) % 3))])


@pytest.mark.parametrize("dst_host", [True, False], ids=["host_dst", "device_dst"])
@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("mem", MEMS)
def test_tnr_frames(ctx, mem, bits, dst_host):
    """A host source staged in windows of 2d + 1 frames, one output frame per chunk at 640 x 360."""
    src = synth.noisy_clip(31, 8, SW, SH, bits)
    prm = ab.tnr_params(3, 1)

    def call(buf):      # the expectation writes a device dst; results compare as bytes
        if dst_host and not isinstance(buf, torch.Tensor):
            dst = np.zeros_like(src)
            ctx.tnr_frames(clip(buf, SW, SH, bits), clip(dst, SW, SH, bits), prm)
            return raw_bytes(dst)
        dst = torch.zeros((src.shape[0], src[0].nbytes), dtype=torch.uint8, device="cuda")
        ctx.tnr_frames(clip(buf, SW, SH, bits), clip(dst, SW, SH, bits), prm)
        return dst
    run_case(ctx, src, mem, call)


@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("mem", MEMS)
def test_logo_find_add_frames_one_reused_frame(ctx, mem, bits):
    """INTEGRATION.md section 5e: every decoded frame in one buffer, one call per frame, the next frame written into
    the buffer as soon as the call returns."""
    src = big(bits)
    want = ctx.logo_find()
    want.add_frames(clip(device(src), BW, BH, bits))
    ws1, ws2, wn = want.sums()
    warm = ctx.logo_find()
    buf = host(src[:1], mem)
    warm.add_frames(clip(buf, BW, BH, bits))
    fd = ctx.logo_find()
    fd.add_frames(clip(buf, BW, BH, bits), 0, 0)          # the finder's sums exist before the hold
    torch.cuda.synchronize()
    hold()
    for n in range(BN):
        buf[0] = src[n]
        fd.add_frames(clip(buf, BW, BH, bits), 0, 1)
    buf.fill(absent(src))
    ctx.synchronize()
    s1, s2, got_n = fd.sums()
    assert got_n == wn == BN
    assert_same((s1, s2), (ws1, ws2))


@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("mem", MEMS)
def test_weave_frames(ctx, mem, bits):
    """Device clips, host index arrays: the indices are read before the call returns."""
    n = 8
    src = device(synth.noisy_clip(32, n, SW, SH, bits))
    top = np.array([0, 1, 2, 2, 4, 5], np.int32)
    bot = np.array([1, 2, 2, 3, 5, 6], np.int32)
    dsts = [torch.zeros((len(top), src.shape[1]), dtype=torch.uint8, device="cuda") for _ in range(2)]
    ctx.weave_frames(clip(src, SW, SH, bits), clip(dsts[0], SW, SH, bits), top, bot)
    want = dsts[0].cpu().numpy()
    t, b = host(top, mem), host(bot, mem)
    held(ctx, lambda: ctx.weave_frames(clip(src, SW, SH, bits), clip(dsts[1], SW, SH, bits), t, b),
         lambda: np.copyto(t, (t + 1) % n), lambda: np.copyto(b, (b + 3) % n))
    assert_same(dsts[1].cpu().numpy(), want)


# ---------------------------------------------------------------------------------------------------------------------
# the group: a one-member amtk_group (no NCCL) whose context runs on its own stream
# ---------------------------------------------------------------------------------------------------------------------
GN = 48         # 1080p frames: 48 one-frame chunks, so the uploads outlast the enqueue by far


@pytest.fixture(scope="module")
def group1(native_lib):
    g = ab.Group(1)
    yield g
    g.close()


@pytest.mark.parametrize("bits", [8, 10])
def test_group_scan_comb_streams_host_clip(ctx, group1, bits):
    """bench.py's group host-clip path.  At 8 bits each band-form launch first waits for the previous launch's watchdog
    record, which paces the uploads; at 10 bits nothing does."""
    g = group1
    lg = synth.make_logo(LA[2], LA[3], seed=2)
    src = widen(synth.make_frames(0, GN, BW, BH, device="cuda", logo=lg, imgx=LA[0], imgy=LA[1], logo_period=16).cpu().numpy(), bits)
    logo = deint(LA, BW, BH, 2)
    prm = ab.default_comb_params()
    ws, wc = as_np(ctx.scan_comb_frames(clip(device(src), BW, BH, bits), [logo], prm))
    pv = absent(src)
    buf = g.host_alloc(0, src.nbytes).view(src.dtype).reshape(src.shape)
    buf[...] = src
    g.scan_comb_streams([clip(buf, BW, BH, bits)], [logo], prm, GN)      # unheld: every buffer exists
    g.synchronize()
    g.scan_comb_streams([clip(buf, BW, BH, bits)], [logo], prm, GN)
    for f in range(GN - 1, -1, -1):            # the last frames first: their uploads are queued the longest
        buf[f].fill(pv)
    g.synchronize()
    s, c = g.fetch_results(GN, 0)
    assert_same((s[0], c[0]), (ws[:, 0], wc))


def test_group_scan_add_frames_host_clip(ctx, group1):
    g = group1
    src = small(8)
    dacc = ctx.logo_scan(LS[2], LS[3], 12)
    dacc.add_frames(clip(device(src), SW, SH, 8), LS[0], LS[1])
    buf = g.host_alloc(0, src.nbytes).reshape(src.shape)
    buf[...] = src
    acc = g.ctx(0).logo_scan(LS[2], LS[3], 12)
    g.scan_add_frames([acc], [clip(buf, SW, SH, 8)], LS[0], LS[1], [0], [SN])
    buf.fill(absent(src))
    g.synchronize()
    assert acc.num_valid == dacc.num_valid > 0
    assert_same(acc.sums(), dacc.sums())


# ---------------------------------------------------------------------------------------------------------------------
# frame streams, fed as a decoder feeds them
# ---------------------------------------------------------------------------------------------------------------------
STREAM_MEMS = ("pinned", "pageable", "device")


def feed(ctx, frames, w, h, bits, mem, send, drain, launches):
    """Sends frames[0..N) one at a time, then poisons what was sent from.  Host frames: each frame decoded into one
    reused host buffer, the next frame written into it as soon as send returns.  Device frames: a pool of two device
    buffers, each overwritten with poison by torch on the context's stream right after its send.  launches(n): whether
    send n launches work (the context's stream is held before it).  drain() runs after every send."""
    pv = absent(frames)
    if mem == "device":
        src = device(frames)
        pool = [torch.empty(src.shape[1], dtype=torch.uint8, device="cuda") for _ in range(2)]
    else:
        buf = host(frames[:1], mem)
    for n in range(frames.shape[0]):
        if mem == "device":
            b = pool[n % 2]
            b.copy_(src[n])
        else:
            buf[0] = frames[n]
            b = buf
        if launches(n):
            hold()
        send(clip(b, w, h, bits, 1))
        if mem == "device":
            (b if bits == 8 else b.view(torch.int16)).fill_(int(pv))
        drain()
    if mem != "device":
        buf.fill(pv)


def every(B, first=0):
    return lambda n: n + 1 >= first + B and (n + 1 - first) % B == 0


class RowReceiver:
    """Receives a row stream's results into one reused host buffer (per output array) and copies them out as soon as
    recv returns."""

    def __init__(self, s, shapes, mem, N):
        self.s, self.N, self.got = s, N, 0
        self.bufs = [host(np.zeros((N,) + sh, dt), mem) for sh, dt in shapes]
        self.rows = [np.zeros_like(b) for b in self.bufs]

    def __call__(self):
        got = C.c_int()
        ptrs = [b.ctypes.data_as(capi.c_float_p if b.dtype == np.float32 else capi.c_i32_p) for b in self.bufs]
        self.s._call("recv", *ptrs, self.N, C.byref(got))
        k = got.value
        for b, r in zip(self.bufs, self.rows):
            r[self.got:self.got + k] = b[:k]
            b.fill(0x7F)
        self.got += k

    def result(self):
        assert self.got == self.N
        return tuple(self.rows)


@pytest.mark.parametrize("mem", STREAM_MEMS)
def test_comb_stream(ctx, mem):
    fr, B = moving(8), 4
    want = as_np(ctx.comb_frames(clip(device(fr), SW, SH, 8)))
    s = ctx.comb_stream(None, B)
    rx = RowReceiver(s, [((12,), np.int32)], "pageable" if mem == "device" else mem, fr.shape[0])
    feed(ctx, fr, SW, SH, 8, mem, s.send, rx, every(B))
    s.finish()
    rx()
    assert_same(rx.result(), (want,))


@pytest.mark.parametrize("bits,pitch", [(8, False), (10, True)])
@pytest.mark.parametrize("mem", STREAM_MEMS)
def test_logo_scan_stream(ctx, mem, bits, pitch):
    fr, B = moving(bits), 4
    logos = [deint(LT, SW, SH, 5)]
    c = clip(device(fr), SW, SH, bits)
    want = as_np(ctx.scan_frames(c, logos, pitch_elems_override=c.pitch_y if pitch else 0))
    s = ctx.logo_scan_stream(logos, B, reference_pitch=pitch)
    rx = RowReceiver(s, [((1, 2), np.float32)], "pageable" if mem == "device" else mem, fr.shape[0])
    feed(ctx, fr, SW, SH, bits, mem, s.send, rx, every(B))
    s.finish()
    rx()
    assert_same(rx.result(), (want,))


@pytest.mark.parametrize("bits,pitch", [(8, False), (10, True)], ids=["scan_comb_stream", "scan_comb_stream_pitch"])
@pytest.mark.parametrize("mem", STREAM_MEMS)
def test_scan_comb_stream(ctx, mem, bits, pitch):
    fr, B = moving(bits), 4
    logos = [deint(LT, SW, SH, 5)]
    c = clip(device(fr), SW, SH, bits)
    want = as_np(ctx.scan_comb_frames(c, logos, pitch_elems_override=c.pitch_y if pitch else 0))
    s = ctx.scan_comb_stream(logos, None, B, reference_pitch=pitch)
    rx = RowReceiver(s, [((1, 2), np.float32), ((12,), np.int32)], "pageable" if mem == "device" else mem, fr.shape[0])
    feed(ctx, fr, SW, SH, bits, mem, s.send, rx, every(B))
    s.finish()
    rx()
    assert_same(rx.result(), want)


@pytest.mark.parametrize("out_bits", [0, 14], ids=["plain", "widening"])
@pytest.mark.parametrize("mem", STREAM_MEMS)
def test_tnr_stream(ctx, mem, out_bits):
    fr, B, d = moving(8, 20), 4, 3
    N = fr.shape[0]
    ob = out_bits or 8
    out_dtype = np.uint8 if ob == 8 else np.uint16
    dst = torch.zeros((N, SW * SH * 3 // 2), dtype=torch.uint8 if ob == 8 else torch.int16, device="cuda")
    ctx.tnr_frames(clip(device(fr), SW, SH, 8), clip(dst, SW, SH, ob), ab.tnr_params(d, 1))
    want = dst.cpu().numpy().view(out_dtype)
    st = ctx.tnr_stream(ab.tnr_params(d, 1), B, out_bits=out_bits)
    out = host(np.zeros((1, SW * SH * 3 // 2), out_dtype), "pageable" if mem == "device" else mem)
    got = np.zeros((N, SW * SH * 3 // 2), out_dtype)
    seen = []

    def drain():
        while True:
            tag = st.recv(clip(out, SW, SH, ob, 1))
            if tag is None:
                return
            got[len(seen)] = out[0]
            out.fill(1)
            seen.append(tag)
    sent = itertools.count()
    feed(ctx, fr, SW, SH, 8, mem, lambda c: st.send(c, next(sent)), drain, every(B, d))
    st.finish()
    drain()
    assert seen == list(range(N))
    assert_same(got, want)


@pytest.mark.parametrize("mem", STREAM_MEMS)
def test_erase_logo_stream(ctx, mem):
    """dst is one reused host frame holding source frame n when recv writes output n's rectangles into it."""
    fr, B = moving(8), 4
    N = fr.shape[0]
    raw = raw_logo(LS, SW, SH, 5)
    dev = device(fr)
    want_fades = ctx.erase_logo_clip(clip(dev, SW, SH, 8), raw, None, None, 16)
    want = dev.cpu().numpy()
    s = ctx.erase_logo_stream(raw, N, None, 16, B)
    dst = host(fr[:1], "pageable" if mem == "device" else mem)
    got, fades = np.zeros_like(fr), np.zeros((N, 2), np.float32)
    k = [0]

    def drain():
        while k[0] < N:
            dst[0] = fr[k[0]]
            r = s.recv(clip(dst, SW, SH, 8, 1))
            if r is None:
                return
            n, fd = r
            assert n == k[0]
            got[n], fades[n] = dst[0], fd
            k[0] += 1
    feed(ctx, fr, SW, SH, 8, mem, s.send, drain, every(B))
    drain()
    assert k[0] == N
    assert_same((got, fades), (want, want_fades))


@pytest.mark.parametrize("mem", STREAM_MEMS)
def test_scan_logo_stream(ctx, mem, tmp_path):
    """210 frames: the batch of 200 rectangles is resolved by a send, the rest by finish."""
    n, w, h, rect = 210, 320, 192, (200, 64, 64, 48)
    fr = synth.make_frames(0, n, w, h, seed=0x5EED0005, device="cuda", mode="flat",
                           logo=synth.make_logo(64, 48, seed=4), imgx=rect[0], imgy=rect[1]).cpu().numpy()
    ctx.scan_logo(clip(device(fr), w, h, 8), str(tmp_path / "w.lgd"), *rect, 12, 150)
    s = ctx.scan_logo_stream(*rect, 12, 150)
    pos = itertools.count(1)
    feed(ctx, fr, w, h, 8, mem, lambda c: s.send(c, next(pos), n), lambda: None, lambda k: k == 199)
    s.finish(str(tmp_path / "s.lgd"))
    assert (tmp_path / "s.lgd").read_bytes() == (tmp_path / "w.lgd").read_bytes()


# ---------------------------------------------------------------------------------------------------------------------
# device clips with device outputs stay asynchronous
# ---------------------------------------------------------------------------------------------------------------------
def _returns_before_the_hold_ends(ctx, call):
    call()                                   # unheld: every buffer and table the call needs exists
    torch.cuda.synchronize()
    hold()
    call()
    busy = not torch.cuda.current_stream().query()
    ctx.synchronize()
    return busy


def test_device_clip_calls_stay_asynchronous(ctx):
    d = device(big(8))
    c = clip(d, BW, BH, 8)
    logos = [deint(LA, BW, BH, 2)]
    scores = torch.empty((BN, 1, 2), dtype=torch.float32, device="cuda")
    counts = torch.empty((BN, 12), dtype=torch.int32, device="cuda")
    fd = ctx.logo_find()
    calls = {
        "logo_scan_frames": lambda: ctx.scan_frames(c, logos, out=scores),
        "comb_frames": lambda: ctx.comb_frames(c, out=counts),
        "scan_comb_frames": lambda: ctx.scan_comb_frames(c, logos, scores=scores, counts=counts),
        "logo_find_add_frames": lambda: fd.add_frames(c),
    }
    for name, call in calls.items():
        assert _returns_before_the_hold_ends(ctx, call), name
