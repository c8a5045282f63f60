"""Build recipe for the in-tree native library (explicit nvcc/g++ commands, sm_90a only).

    python -m amatsukaze_b200._build          # builds amatsukaze_b200/lib/libamtk_b200.so

The .so is a build product (git-ignored).
"""
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


HOST_TEST = os.path.join(PKG, "..", "tests", "cpp", "test_filters")


def build_host_test(force=False):
    """tests/cpp/test_filters: the C++ driver of the host-side filter mirror (amatsukaze_b200/host/*.h*)."""
    src = os.path.join(PKG, "..", "tests", "cpp", "test_filters.cpp")
    deps = [src, os.path.join(PKG, "host", "filters.hpp"), os.path.join(PKG, "host", "avs_compat.h"), LIB]
    if (not force and os.path.exists(HOST_TEST) and all(os.path.getmtime(HOST_TEST) >= os.path.getmtime(d) for d in deps)):
        return HOST_TEST
    cmd = ["g++", "-std=c++17", "-O2", "-o", HOST_TEST, src, "-L" + LIBDIR, "-lamtk_b200",
           "-Wl,-rpath,$ORIGIN/../../amatsukaze_b200/lib"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("host test build failed")
    return HOST_TEST


PIPELINE_TEST = os.path.join(PKG, "..", "tests", "cpp", "test_pipeline")


def build_pipeline_test(force=False):
    """tests/cpp/test_pipeline: multi-pass driver, ingest semantics and device frames on a real device."""
    src = os.path.join(PKG, "..", "tests", "cpp", "test_pipeline.cpp")
    deps = [src, os.path.join(PKG, "host", "filters.hpp"), os.path.join(PKG, "host", "avs_compat.h"), LIB]
    if (not force and os.path.exists(PIPELINE_TEST) and all(os.path.getmtime(PIPELINE_TEST) >= os.path.getmtime(d) for d in deps)):
        return PIPELINE_TEST
    cmd = ["g++", "-std=c++17", "-O2", "-o", PIPELINE_TEST, src, "-L" + LIBDIR, "-lamtk_b200",
           "-Wl,-rpath,$ORIGIN/../../amatsukaze_b200/lib"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("pipeline test build failed")
    return PIPELINE_TEST


HOST_ONLY_TEST = os.path.join(PKG, "..", "tests", "cpp", "test_host_only")


def build_host_only_test(force=False):
    """tests/cpp/test_host_only: driver of the host-side logic that needs no device (CPU test suite)."""
    src = os.path.join(PKG, "..", "tests", "cpp", "test_host_only.cpp")
    deps = [src, os.path.join(PKG, "host", "filters.hpp"), os.path.join(PKG, "host", "avs_compat.h"), LIB]
    if (not force and os.path.exists(HOST_ONLY_TEST) and all(os.path.getmtime(HOST_ONLY_TEST) >= os.path.getmtime(d) for d in deps)):
        return HOST_ONLY_TEST
    cmd = ["g++", "-std=c++17", "-O2", "-o", HOST_ONLY_TEST, src, "-L" + LIBDIR, "-lamtk_b200",
           "-Wl,-rpath,$ORIGIN/../../amatsukaze_b200/lib"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("host-only test build failed")
    return HOST_ONLY_TEST


TNR_FILTER_TEST = os.path.join(PKG, "..", "tests", "cpp", "test_tnr_filter")


def build_tnr_filter_test(force=False):
    """tests/cpp/test_tnr_filter: KTemporalNR of the host-side mirror as the output pass of AMTFilterSource."""
    src = os.path.join(PKG, "..", "tests", "cpp", "test_tnr_filter.cpp")
    deps = [src, os.path.join(PKG, "host", "filters.hpp"), os.path.join(PKG, "host", "avs_compat.h"), LIB]
    if (not force and os.path.exists(TNR_FILTER_TEST) and all(os.path.getmtime(TNR_FILTER_TEST) >= os.path.getmtime(d) for d in deps)):
        return TNR_FILTER_TEST
    cmd = ["g++", "-std=c++17", "-O2", "-o", TNR_FILTER_TEST, src, "-L" + LIBDIR, "-lamtk_b200",
           "-Wl,-rpath,$ORIGIN/../../amatsukaze_b200/lib"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("KTemporalNR filter test build failed")
    return TNR_FILTER_TEST


TNR_WIDEN_TEST = os.path.join(PKG, "..", "tests", "cpp", "test_tnr_widen")


def build_tnr_widen_test(force=False):
    """tests/cpp/test_tnr_widen: ConvertBits(14) then KTemporalNR(3, 1) of the host-side mirror, fused on the device."""
    src = os.path.join(PKG, "..", "tests", "cpp", "test_tnr_widen.cpp")
    deps = [src, os.path.join(PKG, "host", "filters.hpp"), os.path.join(PKG, "host", "avs_compat.h"), LIB]
    if (not force and os.path.exists(TNR_WIDEN_TEST) and all(os.path.getmtime(TNR_WIDEN_TEST) >= os.path.getmtime(d) for d in deps)):
        return TNR_WIDEN_TEST
    cmd = ["g++", "-std=c++17", "-O2", "-o", TNR_WIDEN_TEST, src, "-L" + LIBDIR, "-lamtk_b200",
           "-Wl,-rpath,$ORIGIN/../../amatsukaze_b200/lib"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("ConvertBits + KTemporalNR filter test build failed")
    return TNR_WIDEN_TEST


TNR_FILTER_STREAM_TEST = os.path.join(PKG, "..", "tests", "cpp", "test_tnr_filter_stream")


def build_tnr_filter_stream_test(force=False):
    """tests/cpp/test_tnr_filter_stream: KTemporalNR of the host-side mirror over a host clip (frame stream and gather)."""
    src = os.path.join(PKG, "..", "tests", "cpp", "test_tnr_filter_stream.cpp")
    deps = [src, os.path.join(PKG, "host", "filters.hpp"), os.path.join(PKG, "host", "avs_compat.h"), LIB]
    if (not force and os.path.exists(TNR_FILTER_STREAM_TEST) and
            all(os.path.getmtime(TNR_FILTER_STREAM_TEST) >= os.path.getmtime(d) for d in deps)):
        return TNR_FILTER_STREAM_TEST
    cmd = ["g++", "-std=c++17", "-O2", "-o", TNR_FILTER_STREAM_TEST, src, "-L" + LIBDIR, "-lamtk_b200", "-ldl",
           "-Wl,-rpath,$ORIGIN/../../amatsukaze_b200/lib"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("KTemporalNR frame-stream filter test build failed")
    return TNR_FILTER_STREAM_TEST


SCAN_LOGO_STREAM_TEST = os.path.join(PKG, "..", "tests", "cpp", "test_scan_logo_stream")


def build_scan_logo_stream_test(force=False):
    """tests/cpp/test_scan_logo_stream: logo::LogoAnalyzer of the host-side mirror over a CPU and a device-resident source."""
    src = os.path.join(PKG, "..", "tests", "cpp", "test_scan_logo_stream.cpp")
    deps = [src, os.path.join(PKG, "host", "filters.hpp"), os.path.join(PKG, "host", "avs_compat.h"), LIB]
    if (not force and os.path.exists(SCAN_LOGO_STREAM_TEST) and
            all(os.path.getmtime(SCAN_LOGO_STREAM_TEST) >= os.path.getmtime(d) for d in deps)):
        return SCAN_LOGO_STREAM_TEST
    cmd = ["g++", "-std=c++17", "-O2", "-o", SCAN_LOGO_STREAM_TEST, src, "-L" + LIBDIR, "-lamtk_b200",
           "-Wl,-rpath,$ORIGIN/../../amatsukaze_b200/lib"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("LogoAnalyzer frame-stream test build failed")
    return SCAN_LOGO_STREAM_TEST


ERASE_LOGO_STREAM_TEST = os.path.join(PKG, "..", "tests", "cpp", "test_erase_logo_stream")


def build_erase_logo_stream_test(force=False):
    """tests/cpp/test_erase_logo_stream: logo::AMTEraseLogo of the host-side mirror over a CPU source (frame stream and
    per-frame path)."""
    src = os.path.join(PKG, "..", "tests", "cpp", "test_erase_logo_stream.cpp")
    deps = [src, os.path.join(PKG, "host", "filters.hpp"), os.path.join(PKG, "host", "avs_compat.h"), LIB]
    if (not force and os.path.exists(ERASE_LOGO_STREAM_TEST) and
            all(os.path.getmtime(ERASE_LOGO_STREAM_TEST) >= os.path.getmtime(d) for d in deps)):
        return ERASE_LOGO_STREAM_TEST
    cmd = ["g++", "-std=c++17", "-O2", "-o", ERASE_LOGO_STREAM_TEST, src, "-L" + LIBDIR, "-lamtk_b200",
           "-Wl,-rpath,$ORIGIN/../../amatsukaze_b200/lib"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("AMTEraseLogo frame-stream test build failed")
    return ERASE_LOGO_STREAM_TEST


LOGO_SCAN_STREAM_TEST = os.path.join(PKG, "..", "tests", "cpp", "test_logo_scan_stream")


def build_logo_scan_stream_test(force=False):
    """tests/cpp/test_logo_scan_stream: logo::LogoFrame and CMAnalyze of the host-side mirror over a CPU source (frame
    stream) and a device-resident source."""
    src = os.path.join(PKG, "..", "tests", "cpp", "test_logo_scan_stream.cpp")
    deps = [src, os.path.join(PKG, "host", "filters.hpp"), os.path.join(PKG, "host", "avs_compat.h"), LIB]
    if (not force and os.path.exists(LOGO_SCAN_STREAM_TEST) and
            all(os.path.getmtime(LOGO_SCAN_STREAM_TEST) >= os.path.getmtime(d) for d in deps)):
        return LOGO_SCAN_STREAM_TEST
    cmd = ["g++", "-std=c++17", "-O2", "-o", LOGO_SCAN_STREAM_TEST, src, "-L" + LIBDIR, "-lamtk_b200",
           "-Wl,-rpath,$ORIGIN/../../amatsukaze_b200/lib"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("LogoFrame frame-stream test build failed")
    return LOGO_SCAN_STREAM_TEST


COMB_STREAM_TEST = os.path.join(PKG, "..", "tests", "cpp", "test_comb_stream")


def build_comb_stream_test(force=False):
    """tests/cpp/test_comb_stream: AMTCombAnalyze of the host-side mirror over a CPU source (frame stream) and a
    device-resident source, alone and as KFM pass 1 under AMTFilterSource."""
    src = os.path.join(PKG, "..", "tests", "cpp", "test_comb_stream.cpp")
    deps = [src, os.path.join(PKG, "host", "filters.hpp"), os.path.join(PKG, "host", "avs_compat.h"), LIB]
    if (not force and os.path.exists(COMB_STREAM_TEST) and
            all(os.path.getmtime(COMB_STREAM_TEST) >= os.path.getmtime(d) for d in deps)):
        return COMB_STREAM_TEST
    cmd = ["g++", "-std=c++17", "-O2", "-o", COMB_STREAM_TEST, src, "-L" + LIBDIR, "-lamtk_b200",
           "-Wl,-rpath,$ORIGIN/../../amatsukaze_b200/lib"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("AMTCombAnalyze frame-stream test build failed")
    return COMB_STREAM_TEST


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
