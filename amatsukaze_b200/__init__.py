"""amatsukaze_b200 -- H100-native (sm_90a) implementation of Amatsukaze's per-frame pixel-analysis hot path.

The product is the CUDA library amatsukaze_b200/lib/libamtk_b200.so behind the C ABI of include/amtk_b200.h;
this package is the thin Python plumbing used by tests/, bench.py and multi-GPU launches.
"""
from .capi import (AmtkError, ClipDesc, CombParams, Context, Group, Logo, LogoFind, LogoFindParams, LogoScanAcc, TnrParams, TnrStream, calc_fade2,
                   default_comb_params, default_logo_find_params, default_tnr_params, lib, logo_find_rects, tnr_params, yv12_clip, LIB_PATH, SIGNATURES)

__all__ = ["AmtkError", "ClipDesc", "CombParams", "Context", "Group", "Logo", "LogoScanAcc", "calc_fade2",
           "default_comb_params", "lib", "yv12_clip", "LIB_PATH", "SIGNATURES", "TnrParams", "TnrStream", "default_tnr_params", "tnr_params",
           "LogoFind", "LogoFindParams", "default_logo_find_params", "logo_find_rects"]
