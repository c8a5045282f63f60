"""amtk_scan_comb_frames_pitch and amtk_scan_comb_stream_create_pitch at the C ABI, without a device: the header declares
them in C99, the library exports them, the ctypes binding and the Context keywords exist, and calls without a context
are refused with their reason."""
import ctypes as C
import inspect
import os
import subprocess

import amatsukaze_b200 as ab

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUNCS = ["amtk_scan_comb_frames_pitch", "amtk_scan_comb_stream_create_pitch"]


def test_header_compiles_as_c99_with_the_new_symbols(tmp_path):
    src = tmp_path / "use.c"
    src.write_text('#include "amtk_b200.h"\n'
                   "int (*frames)(amtk_ctx*, const amtk_clip*, amtk_logo* const*, int, const amtk_comb_params*, int, int, int,\n"
                   "              float*, int32_t*, int) = amtk_scan_comb_frames_pitch;\n"
                   "int (*create)(amtk_ctx*, amtk_logo* const*, int, const amtk_comb_params*, int, int, amtk_scan_comb_stream**) =\n"
                   "    amtk_scan_comb_stream_create_pitch;\n")
    r = subprocess.run(["cc", "-std=c99", "-pedantic", "-Werror", "-c", str(src), "-I", os.path.join(ROOT, "include"),
                        "-o", str(tmp_path / "use.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_ctypes_sees_the_symbols():
    names = [s[0] for s in ab.SIGNATURES]
    L = ab.lib()
    for f in FUNCS:
        assert f in names and hasattr(L, f), f
    assert inspect.signature(ab.Context.scan_comb_frames).parameters["pitch_elems_override"].default == 0
    assert inspect.signature(ab.Context.scan_comb_stream).parameters["reference_pitch"].default is False


def test_null_arguments_are_refused():
    L = ab.lib()
    out, p = C.c_void_p(), ab.default_comb_params()
    assert L.amtk_scan_comb_stream_create_pitch(None, None, 1, C.byref(p), 16, 1, C.byref(out)) == 0
    assert b"amtk_scan_comb_stream_create_pitch: bad argument" in L.amtk_last_error()
    assert L.amtk_scan_comb_frames_pitch(None, None, None, 1, C.byref(p), 0, 0, 1, None, None, 0) == 0
    assert b"amtk_scan_comb_frames_pitch: bad argument" in L.amtk_last_error()
    assert L.amtk_scan_comb_frames_pitch(None, None, None, 1, C.byref(p), 0, 0, 0, None, None, 0) == 0   # no context
