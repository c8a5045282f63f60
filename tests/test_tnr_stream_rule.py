"""The Python restatement of amtk_tnr_stream's receive rule and emission sets (oracle/pytnr_stream.py), which the GPU tests
hold the library to, checked here without a GPU: the reference emission set against the CPU TemporalNRFilter's own queue
order (pytnr.sequence_windows), and the receive rule against the properties it promises."""
from oracle import pytnr as pt
from oracle import pytnr_stream as ps


def _clamped(n, d, N):
    return [min(max(n - d + i, 0), N - 1) for i in range(2 * d + 1)]


def test_emission_sets_match_the_reference_queue():
    for d in range(8):
        for B in range(1, 9):
            for N in range(1, 3 * (2 * d + B) + 1):
                seq = pt.sequence_windows(N, d)
                assert ps.emitted(N, d, True) == [i for i, _ in seq], (d, B, N)
                for i, win in seq:                  # the queue's windows are the clamped windows of the library
                    assert win == _clamped(i, d, N)
                assert ps.emitted(N, d, False) == list(range(N))


def test_short_clip_drops():
    assert ps.emitted(5, 3, True) == [0, 1, 3, 4]
    assert ps.emitted(4, 3, True) == [0, 3]
    assert all(ps.emitted(N, 3, True) == [] for N in range(4))
    assert ps.emitted(6, 3, True) == list(range(6))


def test_receive_rule():
    for d in range(8):
        for B in range(1, 9):
            Nmax = 3 * (2 * d + B)
            prev = 0
            for S in range(Nmax + 1):
                r = ps.receivable(S, d, B, False)
                assert r >= prev                     # never takes back an output
                prev = r
                assert r % B == 0 and r <= S
                assert r == 0 or r - 1 + d < S       # every receivable output had its whole window sent
                L = ps.launched_batches(S, d, B, False)
                assert all((k + 1) * B + d <= S for k in range(L)) and (L + 1) * B + d > S
                assert r == max(0, L - 1) * B        # the newest launched batch is held back
                if S >= 2 * B + d:                   # ...so a batch is in flight while the one before it is received
                    assert r + B <= L * B
                assert ps.receivable(S, d, B, True) == S
                assert ps.launched_batches(S, d, B, True) * B >= S
