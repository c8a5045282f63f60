"""amtk_scan_comb_stream at the C ABI, without a device: the header declares it in C99, the library exports every function,
the ctypes binding and the Context method exist, and calls without a context or stream are refused with their reason."""
import ctypes as C
import os
import subprocess

import amatsukaze_b200 as ab

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUNCS = ["amtk_scan_comb_stream_" + f for f in ("create", "destroy", "send", "finish", "recv", "counts")]


def test_header_compiles_as_c99_with_the_new_symbols(tmp_path):
    src = tmp_path / "use.c"
    src.write_text('#include "amtk_b200.h"\n'
                   "int (*create)(amtk_ctx*, amtk_logo* const*, int, const amtk_comb_params*, int, amtk_scan_comb_stream**) =\n"
                   "    amtk_scan_comb_stream_create;\n"
                   "void (*destroy)(amtk_scan_comb_stream*) = amtk_scan_comb_stream_destroy;\n"
                   "int (*send)(amtk_scan_comb_stream*, const amtk_clip*) = amtk_scan_comb_stream_send;\n"
                   "int (*finish)(amtk_scan_comb_stream*) = amtk_scan_comb_stream_finish;\n"
                   "int (*recv)(amtk_scan_comb_stream*, float*, int32_t*, int, int*) = amtk_scan_comb_stream_recv;\n"
                   "int (*counts)(const amtk_scan_comb_stream*, int*, int*, int64_t*, int64_t*) = amtk_scan_comb_stream_counts;\n")
    r = subprocess.run(["cc", "-std=c99", "-pedantic", "-Werror", "-c", str(src), "-I", os.path.join(ROOT, "include"),
                        "-o", str(tmp_path / "use.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_ctypes_sees_the_symbols():
    names = [s[0] for s in ab.SIGNATURES]
    L = ab.lib()
    for f in FUNCS:
        assert f in names and hasattr(L, f), f
    assert hasattr(ab.Context, "scan_comb_stream")


def test_null_arguments_are_refused():
    L = ab.lib()
    out, p = C.c_void_p(), ab.default_comb_params()
    assert L.amtk_scan_comb_stream_create(None, None, 1, C.byref(p), 16, C.byref(out)) == 0
    assert b"bad argument" in L.amtk_last_error()
    assert L.amtk_scan_comb_stream_send(None, None) == 0
    assert b"null argument" in L.amtk_last_error()
    assert L.amtk_scan_comb_stream_finish(None) == 0
    assert b"null stream" in L.amtk_last_error()
    got = C.c_int()
    assert L.amtk_scan_comb_stream_recv(None, None, None, 1, C.byref(got)) == 0
    assert b"bad argument" in L.amtk_last_error()
    assert L.amtk_scan_comb_stream_counts(None, None, None, None, None) == 0
    assert b"null stream" in L.amtk_last_error()
    L.amtk_scan_comb_stream_destroy(None)
