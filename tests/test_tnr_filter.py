"""KTemporalNR of the host-side filter mirror, driven through tests/cpp/test_tnr_filter.cpp: the server's
`KTemporalNR(3, 1)` line as the output pass of AMTFilterSource on a device-resident source and on a CPU source (every
output frame equals the C port of the reference's TemporalNRFilter), and AMTEraseLogo run in place on the filter's
device clip."""
import os
import struct
import subprocess

import numpy as np
import pytest

import amatsukaze_b200 as ab
from amatsukaze_b200 import synth, _build
from oracle import pytnr as pt

pytestmark = pytest.mark.gpu
W, H, IMGX, IMGY = 256, 128, 160, 32


@pytest.fixture(scope="module")
def exe():
    return _build.build_tnr_filter_test() if os.path.exists("/usr/bin/g++") else _build.TNR_FILTER_TEST


def _write_raw1(path, frames):
    with open(path, "wb") as f:
        f.write(b"AMTSRAW1" + struct.pack("<6i", W, H, 8, frames.shape[0], 30000, 1001))
        f.write(frames.tobytes())


@pytest.mark.parametrize("source", ["dev", "cpu"])
def test_ktemporalnr_output_pass(exe, tmp_path, source):
    n = 17
    frames = synth.noisy_clip(4242, n, W, H, 8)
    _write_raw1(tmp_path / "amts0.dat", frames)
    r = subprocess.run([exe, "pass", str(tmp_path), source, str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "preproc=0 frames=%d" % n in r.stdout
    assert "params=c[dist]i[thresh]i[interlaced]b" in r.stdout
    if source == "dev":        # filtered once into HBM, served as device views, an IDeviceClip itself
        assert "resident=1 device_frames=%d" % n in r.stdout
    else:                      # gathered windows, CPU frames
        assert "resident=0 device_frames=0" in r.stdout
    assert "typed=%d" % n in r.stdout                    # frame properties carried over from the source frame
    got = np.fromfile(tmp_path / "out.bin", np.uint8).reshape(n, -1)
    assert np.array_equal(got, pt.or_tnr_clip(frames, W, H, 8, 3, 1, 0))


def test_erase_in_place_on_the_filters_device_clip(exe, tmp_path):
    n = 24
    lg = synth.make_logo(64, 64, seed=1)
    frames = synth.make_frames(35, n, W, H, logo=lg, imgx=IMGX, imgy=IMGY, logo_period=16).numpy()
    _write_raw1(tmp_path / "amts0.dat", frames)
    logo_path = str(tmp_path / "logo.lgd")
    ab.Logo.create(lg["data"], 64, 64, W, H, IMGX, IMGY).save(logo_path)
    r = subprocess.run([exe, "erase", str(tmp_path), logo_path, str(tmp_path / "per_frame.bin"), str(tmp_path / "in_place.bin")],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "identical=1" in r.stdout
    per_frame = np.fromfile(tmp_path / "per_frame.bin", np.uint8).reshape(n, -1)
    tnr = pt.or_tnr_clip(frames, W, H, 8, 3, 1, 0)
    assert not np.array_equal(per_frame, tnr)                 # the logo was erased from the filtered frames ...
    ysz = W * H
    Y = per_frame[:, :ysz].reshape(n, H, W)
    T = tnr[:, :ysz].reshape(n, H, W)
    outside = np.ones((H, W), bool)
    outside[IMGY:IMGY + 64, IMGX:IMGX + 64] = False
    assert np.array_equal(Y[:, outside], T[:, outside])       # ... and nothing outside its rectangle changed
