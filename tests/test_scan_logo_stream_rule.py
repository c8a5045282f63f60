"""The restatement of amtk_scan_logo_stream's rule (stream_rule in test_gpu_scan_logo_stream.py, which the GPU tests hold
the library to), checked here without a GPU against a line-by-line port of the reference's InitialLogoCreator::onFrame
(LogoScan.hpp:881-914) driven as SimpleVideoReader::readAll drives it: frames are read until onFrame returns false."""
import numpy as np

from test_gpu_scan_logo_stream import stream_rule


def on_frame_port(valid, num_max_frames, pos, size):
    """readAll + onFrame.  Returns (stored, callbacks, number of frames the reader delivered)."""
    read_count = 0
    num_frames = 0
    stored, calls = [], []
    delivered = 0
    for i in range(len(valid)):
        delivered += 1
        # onFrame(frame)
        read_count += 1
        if num_frames >= num_max_frames:
            break                                                   # return false: the reader stops
        if valid[i]:                                                # logoscan->AddFrame(...)
            num_frames += 1
            stored.append(i)
        if read_count % 200 == 0:
            progress = np.float32(np.float32(pos[i]) / np.float32(size[i])) * np.float32(50)
            calls.append((progress, read_count, 0, num_frames))
    return stored, calls, delivered


def test_rule_matches_on_frame():
    rng = np.random.default_rng(5)
    checked_on, checked_off = 0, 0
    for trial in range(400):
        n = int(rng.integers(1, 1300))
        p = rng.uniform(0.0, 1.0)
        valid = list(rng.random(n) < p)
        nv = np.concatenate([[0], np.cumsum(valid)])
        pick = trial % 4
        if pick == 0:                                   # cut-off on a multiple of 200 when one is valid
            rs = [r for r in range(200, n + 1, 200) if valid[r - 1]]
            maxf = int(nv[rs[0]]) if rs else int(rng.integers(0, 50))
        elif pick == 1:
            maxf = int(rng.integers(0, max(1, int(nv[-1]) + 5)))
        elif pick == 2:
            maxf = 100000
        else:
            maxf = int(rng.integers(0, 3))
        pos = list(np.cumsum(rng.integers(1, 10_000_000, n)))
        size = [int(pos[-1]) + int(x) for x in rng.integers(1, 1_000_000, n)]
        stored, calls, delivered = on_frame_port(valid, maxf, pos, size)
        rule = stream_rule(valid, maxf, pos, size)
        assert rule["stored"] == stored, (trial, maxf)
        assert [(np.float32(c[0]),) + c[1:] for c in rule["calls"]] == calls, (trial, maxf)
        assert rule["ngather"] == len(stored)
        # the reference reads the cut-off frame and one more (whose onFrame returns false), or the whole source
        assert delivered == min(n, rule["nread"] + 1)
        # *more is 0 from the send that resolves the batch holding the cut-off (max_frames = 0: the first send)
        if False in rule["more"]:
            first_stop = rule["more"].index(False) + 1
            assert first_stop == (1 if maxf == 0 else -(-rule["nread"] // 200) * 200)
            assert not any(rule["more"][first_stop - 1:])
            if rule["nread"] % 200 == 0 and rule["nread"]:
                checked_on += 1
            else:
                checked_off += 1
        else:
            assert n < -(-rule["nread"] // 200) * 200 or (rule["nread"] == n and len(stored) < maxf)
        # the result does not depend on frames sent after the cut-off
        extra = stream_rule(valid + list(rng.random(250) < 0.5), maxf, pos + [1] * 250, size + [1] * 250)
        if False in rule["more"]:
            assert (extra["stored"], extra["calls"], extra["nread"]) == (rule["stored"], rule["calls"], rule["nread"])
    assert checked_on > 5 and checked_off > 20
