"""amtk_erase_logo_clip at the C ABI, without a device: the header declares it in C99, the library exports it, the ctypes
binding and the Context method exist, and a call without a context is refused with its reason."""
import ctypes as C
import os
import subprocess

import amatsukaze_b200 as ab

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_compiles_as_c99_with_the_new_symbol(tmp_path):
    src = tmp_path / "use.c"
    src.write_text('#include "amtk_b200.h"\n'
                   "int (*fn)(amtk_ctx*, const amtk_clip*, const amtk_clip*, const amtk_logo*, float, const uint8_t*, int, int,\n"
                   "          int, float*) = amtk_erase_logo_clip;\n")
    r = subprocess.run(["cc", "-std=c99", "-pedantic", "-Werror", "-c", str(src), "-I", os.path.join(ROOT, "include"),
                        "-o", str(tmp_path / "use.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_ctypes_sees_the_symbol():
    assert "amtk_erase_logo_clip" in [s[0] for s in ab.SIGNATURES]
    assert hasattr(ab.lib(), "amtk_erase_logo_clip")
    assert hasattr(ab.Context, "erase_logo_clip")


def test_null_context_is_refused():
    L = ab.lib()
    assert L.amtk_erase_logo_clip(None, None, None, None, C.c_float(0.35), None, 16, 0, 1, None) == 0
    assert b"null argument" in L.amtk_last_error()
