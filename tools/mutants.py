"""Mutation check of the fused step's kernels and the logo finder: does the suite notice a counter or a score that is
slightly wrong?

Each entry of MUTANTS changes one value in one source file: a comparison, a constant, a rounding, a parity, which frame or
row inside a buffer is read or written, or a host work-list boundary that keeps every item inside the call's frames.  A
mutant is built in a copy of the repository with the flags of amatsukaze_b200/_build.py and its pytest selection is run
there with -x; it is killed when a test fails, survives when all pass.  An equivalent mutant computes what the library
computes on every input; its entry carries the one-line argument.  The working tree is never changed.

Safety rule (part of the table's contract, checked by tests/test_mutant_table.py): no entry touches address or offset
arithmetic that could leave a buffer, loop trip counts that index memory, block barriers, mbarriers, TMA or bulk copies,
atomics, the work-queue counter, the watchdog, or grid, block and shared-memory sizes.  A mutant that faults or hangs
anyway is a finding: its run is recorded as such and never repeated automatically.

    python tools/mutants.py --list
    python tools/mutants.py --build [-j 6] [NAME ...]       # cross-compiles; needs nvcc, no GPU
    python tools/mutants.py --all [-j 4] [--out FILE]       # runs every mutant's selection (needs the H100)
    python tools/mutants.py NAME ...                        # runs the named mutants
    python tools/mutants.py NAME --only-new --keep-going    # every new test that fails on the named mutant
Built libraries go to tools/_bin/mutants/<name>.so.gz; a mutant without one is built before it runs.
"""
import argparse
import concurrent.futures as cf
import gzip
import json
import os
import re
import shutil
import signal
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tools", "_bin", "mutants")
FORBIDDEN = ("__syncthreads", "mbar_", "tma_", "bulk_", "atomic", "queue", "watch")

CS = "amatsukaze_b200/csrc/comb_stream.cuh"
CU = "amatsukaze_b200/csrc/amtk_b200.cu"
LK = "amatsukaze_b200/csrc/logo_kernels.cuh"
CK = "amatsukaze_b200/csrc/comb_kernels.cuh"
FK = "amatsukaze_b200/csrc/find_kernels.cuh"

# pytest selections: the existing tests of the code first, then the tests written to kill what they miss
E_TALL = "tests/test_gpu_comb_tall.py"
E_FUSED = "tests/test_gpu_fused_step.py"
E_LOGO = "tests/test_gpu_logo_plans.py"
E_CTA = "tests/test_gpu_comb_values.py"
E_FIND = "tests/test_gpu_logo_find.py"
N_EDGE = "tests/test_gpu_fused_step_edges.py"
N_LOGO = "tests/test_gpu_logo_scores_edges.py"
N_FIND = "tests/test_gpu_logo_find_runs.py"
NEW = (N_EDGE, N_LOGO, N_FIND)

# the band form's lines repeat those of the per-warp streams; these prefixes make them unique
_BAND_FIX = ("issue_at(j, (int)((gload + (uint32_t)j) % S));\n    }\n    // rows of this lane's run the spec excludes (bit j = row "
             "y_first + j)\n    uint32_t fix_mine = 0u;\n")
_BAND_SLOTS = "__syncwarp();\n      }\n      const uint32_t s0 = flip ? c.S[1] : c.S[0], s1 = flip ? c.S[0] : c.S[1];\n"


def M(name, file, before, after, what, tests, equivalent=None):
    return {"name": name, "file": file, "before": before, "after": after, "what": what, "tests": list(tests),
            "equivalent": equivalent}


MUTANTS = [
    # ---- comb_stream.cuh: the band form (ws_bands; the tall band is the same code with three row groups) ----
    M("band_top_rows", CS, _BAND_FIX + "    if (y_first < 2)", _BAND_FIX + "    if (y_first < 1)",
      "band form: a run that starts on row 1 no longer excludes it", [E_TALL, N_EDGE],
      equivalent="a run starts on a multiple of R (band heights, row groups and runs are all multiples of R >= 15), so "
                 "y_first < 2 and y_first < 1 both mean y_first == 0"),
    M("band_top_mask", CS, _BAND_FIX + "    if (y_first < 2) fix_mine |= (1u << (2 - y_first)) - 1u;",
      _BAND_FIX + "    if (y_first < 2) fix_mine |= (1u << (1 - y_first)) - 1u;",
      "band form: row 1 is no longer excluded from the comb response", [E_TALL, N_EDGE]),
    M("band_lo_j", CS, _BAND_FIX + "    if (y_first < 2) fix_mine |= (1u << (2 - y_first)) - 1u;\n    {\n      const int lo_j = max(C.H - 2 - y_first, 0)",
      _BAND_FIX + "    if (y_first < 2) fix_mine |= (1u << (2 - y_first)) - 1u;\n    {\n      const int lo_j = max(C.H - 1 - y_first, 0)",
      "band form: row H-2 is no longer excluded", [E_TALL, N_EDGE]),
    M("band_hi_j", CS, "lo_j = max(C.H - 2 - y_first, 0), hi_j = min(C.H + 2 - y_first, R);     // rows H-2 .. H+1\n      if (hi_j > lo_j) fix_mine |= ((1u << hi_j) - 1u) & ~((1u << lo_j) - 1u);\n    }\n    const uint32_t fix_rows = __reduce_or_sync(0xFFFFFFFFu, fix_mine);\n    const int flip = y_first & 1;                            // slot 0 of this lane's run holds rows of this parity\n    const uint32_t kM = C.thM, tS = C.thS, tL = C.thL;\n    int* const crow = a.counts + C.cls * 6 + lane + ((long long)seg.fbegin - 1 - a.out_frame0) * 12;\n\n    int st = (int)(gload % S);\n    uint32_t ph = (gload / S) & 1u;\n    mm_wait",
      "lo_j = max(C.H - 2 - y_first, 0), hi_j = min(C.H + 1 - y_first, R);     // rows H-2 .. H+1\n      if (hi_j > lo_j) fix_mine |= ((1u << hi_j) - 1u) & ~((1u << lo_j) - 1u);\n    }\n    const uint32_t fix_rows = __reduce_or_sync(0xFFFFFFFFu, fix_mine);\n    const int flip = y_first & 1;                            // slot 0 of this lane's run holds rows of this parity\n    const uint32_t kM = C.thM, tS = C.thS, tL = C.thL;\n    int* const crow = a.counts + C.cls * 6 + lane + ((long long)seg.fbegin - 1 - a.out_frame0) * 12;\n\n    int st = (int)(gload % S);\n    uint32_t ph = (gload / S) & 1u;\n    mm_wait",
      "band form: the zero-filled row H+1 below the plane is no longer excluded", [E_TALL, N_EDGE]),
    M("band_flip_off", CS, "const int flip = y_first & 1;                            // slot 0 of this lane's run holds rows of this parity\n    const uint32_t kM = C.thM, tS = C.thS, tL = C.thL;\n    int* const crow = a.counts + C.cls * 6 + lane + ((long long)seg.fbegin - 1 - a.out_frame0) * 12;\n\n    int st = (int)(gload % S);\n    uint32_t ph = (gload / S) & 1u;\n    mm_wait",
      "const int flip = 0;                            // slot 0 of this lane's run holds rows of this parity\n    const uint32_t kM = C.thM, tS = C.thS, tL = C.thL;\n    int* const crow = a.counts + C.cls * 6 + lane + ((long long)seg.fbegin - 1 - a.out_frame0) * 12;\n\n    int st = (int)(gload % S);\n    uint32_t ph = (gload / S) & 1u;\n    mm_wait",
      "band form: runs that start on an odd row keep their slots as fields (no parity flip)", [E_TALL, N_EDGE]),
    M("band_flip_move_only", CS, _BAND_SLOTS + "      const uint32_t l0 = flip ? c.L[1] : c.L[0], l1 = flip ? c.L[0] : c.L[1];\n      const uint32_t m0 = flip ? c.M[1] : c.M[0], m1 = flip ? c.M[0] : c.M[1];",
      _BAND_SLOTS + "      const uint32_t l0 = flip ? c.L[1] : c.L[0], l1 = flip ? c.L[0] : c.L[1];\n      const uint32_t m0 = c.M[0], m1 = c.M[1];",
      "band form: the move counter of a run that starts on an odd row goes to the wrong field", [E_TALL, N_EDGE]),
    M("band_prev_window_frame1", CS, "fprev = seg.fbegin > 0 ? seg.fbegin - 1 : seg.fbegin;\n    const CUtensorMap* map",
      "fprev = seg.fbegin > 1 ? seg.fbegin - 1 : seg.fbegin;\n    const CUtensorMap* map",
      "band form: an item that starts at window frame 1 takes frame 1 as its previous frame", [E_TALL, N_EDGE]),
    M("band_prev_first_next", CS, "fprev = seg.fbegin > 0 ? seg.fbegin - 1 : seg.fbegin;\n    const CUtensorMap* map",
      "fprev = seg.fbegin > 0 ? seg.fbegin - 1 : seg.fbegin + (seg.fend - seg.fbegin > 1);\n    const CUtensorMap* map",
      "band form: the first frame of the window is compared with the next frame, not with itself", [E_TALL, N_EDGE]),
    M("band_move_round", CS, "v = met == 0 ? (v >> 7) : (met == 2 && kWsLviaIdp)", "v = met == 0 ? ((v + 64u) >> 7) : (met == 2 && kWsLviaIdp)",
      "band form: the move counter is rounded to the nearest 128 before the shift", [E_TALL, N_EDGE],
      equivalent="every move hit adds exactly 128 (bytes_ge leaves bit 7 per byte), so the warp sum is a multiple of 128 "
                 "and adding 64 before the shift never changes the quotient"),
    M("decode_pair_15bit", CK, "return ((a >> 16) + 2u * (a & 0xFFFFu)) & 0xFFFFu;", "return ((a >> 16) + 2u * (a & 0xFFFFu)) & 0x7FFFu;",
      "pair-coded S/L sums decoded modulo 2^15 instead of 2^16", [E_TALL, N_EDGE],
      equivalent="a decoded sum is one field's hits in one tile-frame of a warp or CTA: at most 128 columns x 68 rows "
                 "< 2^15, so the two masks agree on every value that can occur"),
    M("active_group_h", CS, "const bool active = x0 + col < C.W && y0 + grow < C.H + 2;", "const bool active = x0 + col < C.W && y0 + grow < C.H;",
      "band form: row groups that start on rows H and H+1 skip their arithmetic", [E_TALL, N_EDGE],
      equivalent="such a group's rows are all at or below row H: their comb response is removed again by the fix-up, and "
                 "their move difference compares zero-filled rows, so they count nothing either way"),
    # ---- logo items of the band form (scan_item) ----
    M("item_fade_order", LK, "j.scores[(size_t)(fbegin + (tid >> 1) - out_frame0) * 2 + (tid & 1)]",
      "j.scores[(size_t)(fbegin + (tid >> 1) - out_frame0) * 2 + ((tid & 1) ^ (fend - fbegin == 1))]",
      "logo items of one frame write fade 1 into the fade 0 column and back", [E_FUSED, N_EDGE]),
    M("item_last_row_unwritten", LK, "if (tid < 2 * (fend - fbegin)) {", "if (tid < 2 * (fend - fbegin) - 2 * (fend - fbegin < j.frames)) {",
      "logo items: the last frame of a short (final) item gets no score row", [E_FUSED, N_EDGE]),
    M("item_row_behind", LK, "j.scores[(size_t)(fbegin + (tid >> 1) - out_frame0) * 2 + (tid & 1)]",
      "j.scores[(size_t)(fbegin + (tid >> 1) - ((tid >> 1) > 0 && (tid >> 1) + 1 == fend - fbegin) - out_frame0) * 2 + (tid & 1)]",
      "logo items: the last frame of an item writes the row of the frame before it", [E_FUSED, N_EDGE]),
    M("item_black_mul", LK, "j.scores[(size_t)(fbegin + (tid >> 1) - out_frame0) * 2 + (tid & 1)] = AMTK_FDIV(r, lg.blackScore);",
      "j.scores[(size_t)(fbegin + (tid >> 1) - out_frame0) * 2 + (tid & 1)] = AMTK_FMUL(r, AMTK_FDIV(1.0f, lg.blackScore));",
      "logo items: multiply by 1/blackScore instead of dividing", [E_FUSED, N_EDGE]),
    M("item_sum_tail", LK, "if (c + 4 <= count) {\n          r = AMTK_FADD", "if (c + 4 < count) {\n          r = AMTK_FADD",
      "logo items: the ordered sum drops the last score when the feature count is a multiple of 4", [E_FUSED, N_EDGE]),
    # ---- launch_comb_ws: threshold encodings and the work list ----
    M("ws_move_encoding", CU, "C.thM = (unsigned)(0x80 - tM) * 0x01010101u;", "C.thM = (unsigned)(0x81 - tM) * 0x01010101u;",
      "8-bit move threshold encoded one lower (|d| >= th - 1)", [E_TALL, N_EDGE]),
    M("ws_shima_gt", CU, "C.thS = (unsigned)tS * 0x00010001u;     // integer k", "C.thS = (unsigned)(tS + 1) * 0x00010001u;     // integer k",
      "8-bit small-threshold compare becomes >", [E_TALL, N_EDGE]),
    M("ws10_lshima_clamp", CU, "C.thL = (unsigned)(8192 + std::min(tL, 8191)) * 0x00010001u;", "C.thL = (unsigned)(8192 + std::min(tL, 6138)) * 0x00010001u;",
      "10-bit warp streams: large thresholds above the largest response clamped onto it", ["tests/test_gpu_comb_plans.py::test_every_compiled_variant", N_EDGE]),
    M("ws10_lshima_clamp_equiv", CU, "C.thL = (unsigned)(8192 + std::min(tL, 8191)) * 0x00010001u;", "C.thL = (unsigned)(8192 + std::min(tL, 6139)) * 0x00010001u;",
      "10-bit warp streams: large thresholds clamped just above the largest response", ["tests/test_gpu_comb_plans.py::test_every_compiled_variant", N_EDGE],
      equivalent="a 10-bit response is at most 6 x 1023 = 6138, so any threshold from 6139 up counts nothing, clamped or not"),
    M("tier_mid_skip", CU, "tier(head_frames, mid_end, small);", "tier(head_frames + 1, mid_end, small);",
      "work list: the first frame of the second tier is in no item", [E_TALL, N_EDGE]),
    M("tier_mid_twice", CU, "tier(head_frames, mid_end, small);", "tier(std::max(0, head_frames - 1), mid_end, small);",
      "work list: the last head frame is counted twice", [E_TALL, N_EDGE]),
    M("tier_end_skip", CU, "if (tiny > 0) tier(mid_end, nf, tiny);", "if (tiny > 0) tier(mid_end + 1, nf, tiny);",
      "work list: the first frame of the third tier is in no item", [E_TALL, N_EDGE]),
    M("tier_split_moved", CU, "const int tail_frames = std::min(nf, std::max(small, (int)(nf * 0.15)));\n    const int head_frames = nf - tail_frames;\n    // third tier",
      "const int tail_frames = std::min(nf, std::max(small, (int)(nf * 0.25)));\n    const int head_frames = nf - tail_frames;\n    // third tier",
      "work list: the head tier ends at 75 % of the frames instead of 85 %", [E_TALL, N_EDGE],
      equivalent="head_frames only moves where the long items stop and the short ones start: every frame of every tile is "
                 "still in exactly one item, and the counters are integer sums"),
    M("logo_item_end", CU, "f0 + std::min(nf, (k + 1) * logoF) }", "f0 + std::min(nf, (k + 1) * logoF - 1) }",
      "work list: every logo item ends one frame early", [E_FUSED, N_EDGE]),
    M("logo_item_last_frame", CU, "f0 + std::min(nf, (k + 1) * logoF) }", "f0 + std::min(nf - 1, (k + 1) * logoF) }",
      "work list: the call's last frame is in no logo item", [E_FUSED, N_EDGE]),
    # ---- logo_kernels.cuh: the serial evaluation and its sums ----
    M("sum_kernel_lt", LK, "if (c + 32 <= count) {", "if (c + 32 < count) {",
      "logo_sum_kernel: a full last line of scores takes the per-element path", [E_LOGO, N_LOGO],
      equivalent="the per-element path adds the same scores in the same order, so the sum is the same float"),
    M("bulk_tail_drop", LK, "for (int c = n4 << 2; c < count; ++c) r = AMTK_FADD(r, tail[c]);",
      "for (int c = n4 << 2; c < count; ++c) r = AMTK_FADD(r, c + 1 < count ? tail[c] : 0.0f);",
      "logo_sum_bulk_kernel: the last score of a count that is not a multiple of 4 is dropped", [E_LOGO, N_LOGO]),
    M("bulk_take_abs", LK, "if (take_abs) v = fabsf(v);\n  const int t = t0 + lane;", "if (take_abs) v = fmaxf(v, 0.0f);\n  const int t = t0 + lane;",
      "logo_sum_bulk_kernel: AMTAnalyzeLogo's absolute value clamps negative scores to 0", [E_LOGO, N_LOGO]),
    M("fill_pairs_swap", LK, "out[(size_t)f * stride + off] = v0; out[(size_t)f * stride + off + 1] = v1;",
      "out[(size_t)f * stride + off] = v1; out[(size_t)f * stride + off + 1] = v0;",
      "fill_pairs_kernel: the (0, -1) pair of a logo that does not match the frame is written reversed", [E_LOGO, N_LOGO]),
    M("scores_pair_bin", LK, "const float2 s1 = __ldg(sc + bin[1][p]);", "const float2 s1 = __ldg(sc + bin[0][p]);",
      "logo_scores_kernel: the second fade of a pair takes the first fade's score-scale bin", [E_LOGO, N_LOGO]),
    # ---- comb_kernels.cuh: 2-byte samples and the generic kernel ----
    M("u16_exact_float", CK, "r.v[1] = __uint_as_float(__byte_perm(raw.x, 0x4B000000u, 0x7432)) - 8388608.0f;",
      "r.v[1] = __uint_as_float(__byte_perm(raw.x, 0x4A000000u, 0x7432)) - 8388608.0f;",
      "2-byte stencil: the second sample of each group is read as 2^21 + x/4 (exponent one step low)", [E_CTA, N_EDGE]),
    M("u16_exact_offset", CK, "r.v[0] = __uint_as_float(__byte_perm(raw.x, 0x4B000000u, 0x7410)) - 8388608.0f;",
      "r.v[0] = __uint_as_float(__byte_perm(raw.x, 0x4B000001u, 0x7410)) - 8388608.0f;",
      "2-byte stencil: the first sample of each group is read 65536 too high", [E_CTA, N_EDGE],
      equivalent="the stencil's taps sum to 0 (1 + 4 + 1 - 3 - 3) and the same lane of all five rows shifts by 65536, "
                 "exactly in fp32 (below 2^24), so every response is unchanged"),
    M("u16_shima_gt", CK, "fS[f] += (r >= tS) ? 1.0f : 0.0f;", "fS[f] += (r > tS) ? 1.0f : 0.0f;",
      "2-byte stencil: the small-threshold compare becomes >", [E_CTA, N_EDGE]),
    M("generic_rows", CK, "if (y >= 2 && y < H - 2) {", "if (y >= 2 && y < H - 1) {",
      "generic kernel: row H-2 gets a comb response", [E_CTA, N_EDGE]),
    M("generic_prev_self", CK, "prev_f = f == 0 ? a.prev_of_first : cur_f - 1;", "prev_f = f == 0 ? cur_f : cur_f - 1;",
      "generic kernel: the first frame of a launch is its own previous frame", [E_CTA, N_EDGE]),
    M("generic_split_prev", CU, "gg.prev_of_first = f0 ? gg.first_frame - 1 : g.prev_of_first;", "gg.prev_of_first = f0 ? gg.first_frame : g.prev_of_first;",
      "generic kernel: the first frame after each 16384-frame split is its own previous frame",
      ["tests/test_gpu_comb_plans.py::test_generic_kernel_past_16384_frames", N_EDGE]),
    # ---- find_kernels.cuh: the logo finder's sums ----
    M("find_no_run_cap", FK, "if (tile_ends || p + 1 == end || run == kFindRunCap) {", "if (tile_ends || p + 1 == end) {",
      "finder: 32-bit partials are no longer flushed every kFindRunCap frames of one tile", [E_FIND, N_FIND]),
    M("find_share_begin", FK, "*begin = total * blockIdx.x / gridDim.x;", "*begin = total * blockIdx.x / gridDim.x + (blockIdx.x > 0);",
      "finder: every share but the first skips its first tile frame", [E_FIND, N_FIND]),
    M("find_widen16", FK, "s2[2 * i + h] += (unsigned long long)(v * v);", "s2[2 * i + h] = (uint32_t)(s2[2 * i + h] + v * v);",
      "finder: 16-bit s2 partials wrap at 2^32", [E_FIND, N_FIND]),
    M("find_flush_last_column", FK, "const int x = xb + j;\n      if (x < a.width && s2[j])", "const int x = xb + j;\n      if (x < a.width - 1 && s2[j])",
      "finder: 8-bit partials of the last column are never flushed", [E_FIND, N_FIND]),
    M("find_flush_s1", FK, "const int x = xb + j;\n      if (x < a.width && s2[j])", "const int x = xb + j;\n      if (x < a.width && s1[j])",
      "finder: 8-bit partials are flushed when s1, not s2, is non-zero", [E_FIND, N_FIND],
      equivalent="s2 is a sum of squares of the same samples s1 sums, so one is 0 exactly when the other is"),
]

BY_NAME = {m["name"]: m for m in MUTANTS}


def apply(src, m):
    """The source with mutant m applied; m's before snippet must occur exactly once."""
    n = src.count(m["before"])
    if n != 1:
        raise ValueError("%s: before snippet occurs %d times in %s" % (m["name"], n, m["file"]))
    return src.replace(m["before"], m["after"])


def _copy_tree(dst, with_lib):
    """The working tree without .git, caches and the built libraries of the mutants."""
    skip = {".git", ".pytest_cache", "__pycache__"}

    def ignore(d, names):
        out = [n for n in names if n in skip]
        if os.path.abspath(d) == os.path.join(ROOT, "tools") and "_bin" in names:
            out.append("_bin")
        if not with_lib and os.path.abspath(d) == os.path.join(ROOT, "amatsukaze_b200"):
            out.append("lib")
        return out
    shutil.copytree(ROOT, dst, ignore=ignore, symlinks=True)


def _mutated_copy(m, tmp, with_lib):
    work = os.path.join(tmp, "repo")
    _copy_tree(work, with_lib)
    path = os.path.join(work, m["file"])
    with open(path) as f:
        src = f.read()
    with open(path, "w") as f:
        f.write(apply(src, m))
    return work


def lib_path(name):
    return os.path.join(BIN, name + ".so.gz")


def build(m):
    """Builds mutant m's library with _build.py's recipe in a mutated copy; returns (name, seconds, error or None)."""
    t0 = time.time()
    with tempfile.TemporaryDirectory(prefix="amtk_mut_") as tmp:
        work = _mutated_copy(m, tmp, with_lib=False)
        r = subprocess.run([sys.executable, "-m", "amatsukaze_b200._build", "--force"], cwd=work, capture_output=True, text=True)
        if r.returncode != 0:
            return m["name"], time.time() - t0, (r.stdout + r.stderr)[-2000:]
        os.makedirs(BIN, exist_ok=True)
        with open(os.path.join(work, "amatsukaze_b200", "lib", "libamtk_b200.so"), "rb") as f, \
                gzip.open(lib_path(m["name"]) + ".part", "wb", compresslevel=6) as g:
            shutil.copyfileobj(f, g)
        os.replace(lib_path(m["name"]) + ".part", lib_path(m["name"]))
    return m["name"], time.time() - t0, None


_FAIL = re.compile(r"^(?:FAILED|ERROR) (\S+)", re.M)


def run(m, timeout, only_new=False, keep_going=False):
    """Runs mutant m's selection (only_new: its new tests only; keep_going: without -x) in a mutated copy holding its
    prebuilt library.  Returns the result record."""
    rec = {"name": m["name"], "file": m["file"], "what": m["what"]}
    if not os.path.exists(lib_path(m["name"])):
        _, _, err = build(m)
        if err:
            rec.update(result="build failed", detail=err)
            return rec
    t0 = time.time()
    with tempfile.TemporaryDirectory(prefix="amtk_mut_") as tmp:
        work = _mutated_copy(m, tmp, with_lib=True)
        lib = os.path.join(work, "amatsukaze_b200", "lib", "libamtk_b200.so")
        with gzip.open(lib_path(m["name"]), "rb") as g, open(lib + ".part", "wb") as f:
            shutil.copyfileobj(g, f)
        os.replace(lib + ".part", lib)
        os.chmod(lib, 0o755)
        os.utime(lib)                                          # newer than the mutated source: no rebuild in the copy
        tests = [t for t in m["tests"] if t.split("::")[0] in NEW] if only_new else m["tests"]
        cmd = [sys.executable, "-m", "pytest", *([] if keep_going else ["-x"]), "-q", "-p", "no:cacheprovider", "-o", "addopts=", *tests]
        p = subprocess.Popen(cmd, cwd=work, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, start_new_session=True)
        try:
            out, _ = p.communicate(timeout=timeout)
        except subprocess.TimeoutExpired:
            os.killpg(p.pid, signal.SIGKILL)
            out, _ = p.communicate()
            rec.update(result="timed out (finding: do not rerun)", seconds=round(time.time() - t0, 1), detail=out[-3000:])
            return rec
    rec["seconds"] = round(time.time() - t0, 1)
    failed = _FAIL.findall(out)
    if p.returncode == 0:
        rec["result"] = "equivalent" if m["equivalent"] else "survived"
    elif p.returncode == 1 and failed:
        rec["result"] = "killed"
        rec["killed_by"] = failed[0]
        rec["by_new_test"] = failed[0].split("::")[0] in NEW
        if keep_going:
            rec["failed"] = failed
        if m["equivalent"]:
            rec["result"] = "killed, but marked equivalent"
    else:
        rec["result"] = "error (exit %d)" % p.returncode
    if rec["result"] != "killed":
        rec["detail"] = out[-3000:]
    return rec


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("names", nargs="*")
    ap.add_argument("--list", action="store_true")
    ap.add_argument("--build", action="store_true", help="build the libraries only (no GPU needed)")
    ap.add_argument("--all", action="store_true")
    ap.add_argument("-j", type=int, default=1, help="mutants built or run at once (finder mutants always run alone)")
    ap.add_argument("--timeout", type=float, default=1200.0, help="seconds per mutant run")
    ap.add_argument("--out", default=None, help="JSON lines file for the results")
    ap.add_argument("--only-new", action="store_true", help="run only the tests written for the table (the new-test files)")
    ap.add_argument("--keep-going", action="store_true", help="run the whole selection (no -x) and list every failing test")
    a = ap.parse_args()
    todo = MUTANTS if a.all or (a.build and not a.names) else [BY_NAME[n] for n in a.names]
    if a.list:
        for m in MUTANTS:
            print("%-26s %-40s %s%s" % (m["name"], m["file"], m["what"], "  [equivalent]" if m["equivalent"] else ""))
        return 0
    if a.build:
        bad = 0
        with cf.ThreadPoolExecutor(max(1, a.j)) as ex:
            for name, sec, err in ex.map(build, todo):
                print("%-26s %6.0f s %s" % (name, sec, "ok" if not err else "FAILED\n" + err), flush=True)
                bad += err is not None
        return 1 if bad else 0
    out = open(a.out, "a") if a.out else None
    alone = [m for m in todo if m["file"] == FK]
    shared = [m for m in todo if m["file"] != FK]
    results = []

    def report(rec):
        results.append(rec)
        line = json.dumps(rec)
        print("%-26s %-36s %s" % (rec["name"], rec["result"], rec.get("killed_by", "")), flush=True)
        if out:
            out.write(line + "\n"); out.flush()
    with cf.ThreadPoolExecutor(max(1, a.j)) as ex:
        for rec in ex.map(lambda m: run(m, a.timeout, a.only_new, a.keep_going), shared):
            report(rec)
    for m in alone:                      # the finder's long cases need up to ~18 GB of free HBM: never two at once
        report(run(m, a.timeout, a.only_new, a.keep_going))
    bad = [r for r in results if r["result"] not in ("killed", "equivalent")]
    print("killed %d (new tests %d), equivalent %d, other %d" % (
        sum(r["result"] == "killed" for r in results), sum(bool(r.get("by_new_test")) for r in results),
        sum(r["result"] == "equivalent" for r in results), len(bad)))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
