"""Build recipe for the in-tree native library (explicit nvcc/g++ commands, sm_90a only).

    python -m amatsukaze_b200._build          # builds amatsukaze_b200/lib/libamtk_b200.so

The .so is a build product (git-ignored).
"""
import functools
import hashlib
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
LIB = os.path.join(LIBDIR, "libamtk_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

HOST_FLAGS = ["-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-fvisibility=hidden", "-Wno-unknown-pragmas"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
              "--expt-relaxed-constexpr", "--extended-lambda",
              "-Xcompiler", ",".join(["-fPIC", "-ffp-contract=off", "-fno-fast-math", "-fvisibility=hidden"])]


def _sources():
    out = []
    for root, _, files in os.walk(CSRC):
        for f in files:
            out.append(os.path.join(root, f))
    out.append(os.path.join(PKG, "..", "include", "amtk_b200.h"))
    return out


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(s) > t for s in _sources())


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    os.makedirs(LIBDIR, exist_ok=True)
    obj = os.path.join(LIBDIR, "logo_host.o")
    cmd1 = ["g++", "-std=c++17", *HOST_FLAGS, "-c", os.path.join(CSRC, "logo_host.cpp"), "-o", obj]
    cmd2 = [NVCC, *NVCC_FLAGS, *(["-Xptxas", "-v"] if verbose else []), "-shared", "-o", LIB,
            os.path.join(CSRC, "amtk_b200.cu"), obj, "-ldl", "-lpthread"]
    for cmd in (cmd1, cmd2):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or r.returncode != 0:
            sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError("native build failed: " + " ".join(cmd))
    os.remove(obj)
    return LIB


# The C++ test drivers tests/cpp/<name>.cpp: what each drives, and its extra link flags.
CPP_TESTS = {
    "test_filters": ("the C++ driver of the host-side filter mirror (amatsukaze_b200/host/*.h*)", []),
    "test_pipeline": ("multi-pass driver, ingest semantics and device frames on a real device", []),
    "test_host_only": ("driver of the host-side logic that needs no device (CPU test suite)", []),
    "test_tnr_filter": ("KTemporalNR of the host-side mirror as the output pass of AMTFilterSource", []),
    "test_tnr_widen": ("ConvertBits(14) then KTemporalNR(3, 1) of the host-side mirror, fused on the device", []),
    "test_tnr_filter_stream": ("KTemporalNR of the host-side mirror over a host clip (frame stream and gather)", ["-ldl"]),
    "test_scan_logo_stream": ("logo::LogoAnalyzer of the host-side mirror over a CPU and a device-resident source", []),
    "test_scan_logo_stream_deep": ("logo::LogoAnalyzer of the host-side mirror over 10- and 12-bit CPU and AMTSource sources", []),
    "test_erase_logo_stream": ("logo::AMTEraseLogo of the host-side mirror over a CPU source (frame stream and "
                               "per-frame path)", []),
    "test_erase_logo_clip": ("logo::AMTEraseLogo of the host-side mirror over a device-resident source (one "
                             "amtk_erase_logo_clip call), against the per-frame path and the frame stream", []),
    "test_logo_scan_stream": ("logo::LogoFrame and CMAnalyze of the host-side mirror over a CPU source (frame stream) "
                              "and a device-resident source", []),
    "test_comb_stream": ("AMTCombAnalyze of the host-side mirror over a CPU source (frame stream) and a "
                         "device-resident source, alone and as KFM pass 1 under AMTFilterSource", []),
    "test_scan_comb_stream": ("CMAnalyze of the host-side mirror with its combing-stats path over a CPU source (fused "
                              "frame stream) and a device-resident source, against AMTCombAnalyze", []),
    "test_scan_comb_pitch": ("CMAnalyze of the host-side mirror with its combing-stats path over 8- and 10-bit CPU and "
                             "device-resident sources, counting the streams and whole-clip calls it makes", ["-ldl"]),
}


CPP_TEST_SRC = os.path.join(PKG, "..", "tests", "cpp")
CPP_TEST_BIN = os.path.join(LIBDIR, "cpp_tests")     # build products stay out of tests/, next to the library


def cpp_test_path(name):
    """The built driver of tests/cpp/<name>.cpp."""
    return os.path.join(CPP_TEST_BIN, name)


def _stamp(paths):
    h = hashlib.sha256()
    for p in paths:
        with open(p, "rb") as f:
            h.update(hashlib.sha256(f.read()).digest())
    return h.hexdigest()


def build_cpp_test(name, force=False):
    """Builds the driver of tests/cpp/<name>.cpp against the native library, unless the one there was built from the same
    source, headers and library.  Up to date is decided on the files' contents, not their times, so that a copy of the
    tree with fresh timestamps (a checkout of the same sources) uses the drivers build() made."""
    what, link = CPP_TESTS[name]
    exe, src = cpp_test_path(name), os.path.join(CPP_TEST_SRC, name + ".cpp")
    deps = [src, os.path.join(PKG, "host", "filters.hpp"), os.path.join(PKG, "host", "avs_compat.h"), LIB]
    stamp = _stamp(deps)
    if not force and os.path.exists(exe) and os.path.exists(exe + ".stamp"):
        with open(exe + ".stamp") as f:
            if f.read() == stamp:
                return exe
    os.makedirs(CPP_TEST_BIN, exist_ok=True)
    cmd = ["g++", "-std=c++17", "-O2", "-o", exe, src, "-L" + LIBDIR, "-lamtk_b200", *link, "-Wl,-rpath,$ORIGIN/.."]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("build of tests/cpp/%s (%s) failed" % (name, what))
    with open(exe + ".stamp", "w") as f:
        f.write(stamp)
    return exe


def _driver(name):
    return cpp_test_path(name), functools.partial(build_cpp_test, name)


# <X>_TEST: the driver's path; build_<x>_test(force=False) builds it and returns that path
HOST_TEST, build_host_test = _driver("test_filters")
PIPELINE_TEST, build_pipeline_test = _driver("test_pipeline")
HOST_ONLY_TEST, build_host_only_test = _driver("test_host_only")
TNR_FILTER_TEST, build_tnr_filter_test = _driver("test_tnr_filter")
TNR_WIDEN_TEST, build_tnr_widen_test = _driver("test_tnr_widen")
TNR_FILTER_STREAM_TEST, build_tnr_filter_stream_test = _driver("test_tnr_filter_stream")
SCAN_LOGO_STREAM_TEST, build_scan_logo_stream_test = _driver("test_scan_logo_stream")
SCAN_LOGO_STREAM_DEEP_TEST, build_scan_logo_stream_deep_test = _driver("test_scan_logo_stream_deep")
ERASE_LOGO_STREAM_TEST, build_erase_logo_stream_test = _driver("test_erase_logo_stream")
ERASE_LOGO_CLIP_TEST, build_erase_logo_clip_test = _driver("test_erase_logo_clip")
LOGO_SCAN_STREAM_TEST, build_logo_scan_stream_test = _driver("test_logo_scan_stream")
COMB_STREAM_TEST, build_comb_stream_test = _driver("test_comb_stream")
SCAN_COMB_STREAM_TEST, build_scan_comb_stream_test = _driver("test_scan_comb_stream")
SCAN_COMB_PITCH_TEST, build_scan_comb_pitch_test = _driver("test_scan_comb_pitch")


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
