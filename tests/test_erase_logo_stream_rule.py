"""CPU checks of the erase logo stream's rule (DESIGN.md section 3.3.2): the restated receive rule and analysed-frame set
against a line-by-line port of the reference's AMTEraseLogo::CalcFade / CalcFade2 (LogoScan.hpp:1263-1341) that records
which analyze records it reads, and the lookahead bound exhaustively for N <= 40."""
import numpy as np
import pytest

import amatsukaze_b200 as ab


# ---- the restatement the GPU tests use (kept in step with tests/test_gpu_erase_logo_stream.py) ----------------------
def fade2_index(N, n, i):
    nblk = (N + 7) // 8
    nsrc = max(0, min(N - 1, n + i))
    r = nsrc + i
    blk = max(0, min(nblk - 1, r >> 3))
    return max(0, min(N - 1, blk * 8 + (r & 7)))


def fade_codes(N, frame_result, maxfade):
    """Per output: 0 / 1 = the uniform logoframe window's fade, 2 = CalcFade2."""
    if frame_result is None:
        return [2] * N
    half = maxfade >> 1
    out = []
    for n in range(N):
        win = [frame_result[max(0, min(N - 1, n + i))] for i in range(-half, half + 1)]
        out.append((1 if frame_result[n] == 2 else 0) if all(v == win[0] for v in win) else 2)
    return out


def record_set(N, frame_result, maxfade):
    codes = fade_codes(N, frame_result, maxfade)
    return sorted({fade2_index(N, n, i) for n in range(N) if codes[n] == 2 for i in range(-4, 5)})


def receivable(S, N, B):
    """Outputs that can have been received after S sends (the receive rule)."""
    launched = sum(1 for k in range((N + B - 1) // B) if S >= min(N, (k + 1) * B + 8))
    return N if S == N else min(N, max(0, launched - 1) * B)


# ---- line-by-line port of the reference, recording what it reads ------------------------------------------------------
class PortEraseLogo:
    """AMTEraseLogo::CalcFade / CalcFade2 over an AMTAnalyzeLogo clip of N source frames; `reads` collects the source
    frames whose records CalcFade2 takes."""

    def __init__(self, N, frame_result, max_fade_length):
        self.num_frames = N
        self.frameResult = [] if frame_result is None else list(frame_result)
        self.maxFadeLength = max_fade_length
        self.reads = set()
        self.nblocks = (N + 7) // 8                                  # AMTAnalyzeLogo's vi.num_frames

    def analyze_getframe(self, a):                                  # AviSynth clamps GetFrame to the clip
        a = max(0, min(self.nblocks - 1, a))
        return [min(self.num_frames - 1, a * 8 + j) for j in range(8)]   # nsrc clamps to the last source frame (:1133)

    def CalcFade2(self, n):
        DIST = 4
        prev_n = None
        frame = None
        for i in range(-DIST, DIST + 1):
            nsrc = max(0, min(self.num_frames - 1, n + i))
            analyze_n = (nsrc + i) >> 3
            idx = (nsrc + i) & 7
            if analyze_n != prev_n:
                frame = self.analyze_getframe(analyze_n)
                prev_n = analyze_n
            self.reads.add(frame[idx])
            self.last_reads.append(frame[idx])

    def CalcFade(self, n):
        self.last_reads = []
        if len(self.frameResult) == 0:
            self.CalcFade2(n)
            return 2
        halfWidth = self.maxFadeLength >> 1
        frames = [self.frameResult[max(0, min(self.num_frames - 1, n + i))] for i in range(-halfWidth, halfWidth + 1)]
        if all(p == frames[0] for p in frames):
            return 1 if frames[halfWidth] == 2 else 0
        self.CalcFade2(n)
        return 2


def logoframe_results(N, rng, kind):
    if kind == "none":
        return None
    if kind == "uniform0":
        return np.zeros(N, np.uint8)
    if kind == "uniform2":
        return np.full(N, 2, np.uint8)
    fr = np.zeros(N, np.uint8)
    marks = sorted(rng.choice(np.arange(N + 1), size=min(N + 1, int(rng.integers(1, 5))), replace=False).tolist())
    v = int(rng.integers(0, 3))
    pos = 0
    for m in marks + [N]:
        fr[pos:m] = v
        v = (v + 1 + int(rng.integers(0, 2))) % 3
        pos = m
    return fr


@pytest.mark.parametrize("N", [1, 2, 7, 8, 9, 15, 16, 17, 23, 24, 25, 40, 100])
@pytest.mark.parametrize("kind", ["none", "uniform0", "uniform2", "random"])
@pytest.mark.parametrize("maxfade", [0, 1, 16, 31])
def test_record_set_and_codes_match_the_reference_port(N, kind, maxfade):
    rng = np.random.default_rng(N * 1000 + maxfade)
    for _ in range(3 if kind == "random" else 1):
        fr = logoframe_results(N, rng, kind)
        port = PortEraseLogo(N, fr, maxfade)
        codes = fade_codes(N, fr, maxfade)
        for n in range(N):
            code = port.CalcFade(n)
            assert code == codes[n]
            if code == 2:
                assert port.last_reads == [fade2_index(N, n, i) for i in range(-4, 5)]
                assert port.last_reads == [ab.lib().amtk_calc_fade2_index(N, N, n, i) for i in range(-4, 5)]
        assert sorted(port.reads) == record_set(N, fr, maxfade)
        if kind.startswith("uniform"):
            assert record_set(N, fr, maxfade) == []


def test_lookahead_bound_exhaustive():
    """Output n reads records of frames in [n - 8, min(N - 1, n + 8)] only, including the (nsrc + i) quirk's negative
    offsets: so batch k's fades need frames below min(N, (k+1)B + 8), all sent by the send that launches it, and a ring
    of B + 16 records holds every record a batch reads."""
    for N in range(1, 41):
        port = PortEraseLogo(N, None, 16)
        for n in range(N):
            port.CalcFade(n)
            for f in port.last_reads:
                assert n - 8 <= f <= min(N - 1, n + 8), (N, n, f)


@pytest.mark.parametrize("B", [1, 3, 8, 16, 64, 256])
@pytest.mark.parametrize("N", [1, 2, 7, 8, 9, 17, 100, 300])
def test_receive_rule_launches_cover_their_records(N, B):
    """Every batch is launched by a send at which all records its outputs read were sent; the outputs receivable grow
    monotonically in frame order and reach N exactly at the N-th send; the records a batch reads span < B + 16 frames."""
    prev = 0
    for S in range(1, N + 1):
        r = receivable(S, N, B)
        assert prev <= r <= S
        prev = r
        launched = [k for k in range((N + B - 1) // B) if S >= min(N, (k + 1) * B + 8)]
        for k in launched:
            lo, hi = k * B, min(N, (k + 1) * B)
            reads = [fade2_index(N, n, i) for n in range(lo, hi) for i in range(-4, 5)]
            assert max(reads) < S
            assert max(reads) - min(f for f in reads if f >= lo - 8) < B + 16
    assert receivable(N, N, B) == N
    if N > B + 8:
        assert receivable(N - 1, N, B) < N


def test_python_binding_is_bound():
    names = [s[0] for s in ab.SIGNATURES]
    for fn in ("create", "destroy", "send", "recv", "counts"):
        assert "amtk_erase_logo_stream_" + fn in names
        assert hasattr(ab.lib(), "amtk_erase_logo_stream_" + fn)
    assert hasattr(ab.Context, "erase_logo_stream")


def test_create_refuses_a_null_context_without_a_device():
    import ctypes as C
    L = ab.lib()
    lg = ab.Logo.create(np.zeros((64 * 64 + 2 * 32 * 32) * 2, np.float32), 64, 64, 1920, 1080, 100, 100)
    out = C.c_void_p()
    fake_ctx = C.c_void_p(0)
    assert L.amtk_erase_logo_stream_create(fake_ctx, lg.h, C.c_float(0.35), 10, None, 16, 16, C.byref(out)) == 0
    assert b"null" in L.amtk_last_error()
