"""ctypes binding of libdsmil_b200.so (include/dsmil_b200.h).

There is no CPU fallback and no alternative backend: if the library is missing or a call
fails, a RuntimeError carrying dsmil_last_error() is raised.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
# DSMIL_B200_LIBPATH: load another build of the SAME sources (kernel tuning experiments, tools/); never a fallback
LIB_PATH = os.environ.get("DSMIL_B200_LIBPATH") or os.path.join(_HERE, "lib", "libdsmil_b200.so")

c_float_p = C.c_void_p  # device pointers travel as integers
c_i64 = C.c_int64


class DsmilParams(C.Structure):
    _fields_ = [("D", C.c_int32), ("C", C.c_int32), ("nonlinear", C.c_int32), ("passing_v", C.c_int32),
                ("Wi", C.c_void_p), ("bi", C.c_void_p), ("W1", C.c_void_p), ("b1", C.c_void_p),
                ("W2", C.c_void_p), ("b2", C.c_void_p), ("Wv", C.c_void_p), ("bv", C.c_void_p),
                ("Wf", C.c_void_p), ("bf", C.c_void_p)]


class DsmilGrads(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in
                ("gWi", "gbi", "gW1", "gb1", "gW2", "gb2", "gWv", "gbv", "gWf", "gbf", "gX")]


# name -> (restype, argtypes); every symbol include/dsmil_b200.h declares
SIGNATURES = {
    "dsmil_abi_version": (C.c_int, []),
    "dsmil_last_error": (C.c_char_p, []),
    "dsmil_launch_count": (C.c_uint64, []),
    "dsmil_gather_rows": (C.c_int, [C.c_void_p, c_i64, C.c_int32, C.c_void_p, c_i64, C.c_void_p, C.c_void_p]),
    "dsmil_patches_u8_to_f32": (C.c_int, [C.c_void_p, c_i64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "dsmil_instnorm_act": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, c_i64, C.c_int32, C.c_float, C.c_int32, C.c_void_p]),
    "dsmil_instnorm_act_nhwc": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, c_i64, C.c_int32, C.c_int32, C.c_float, C.c_int32,
                                          C.c_void_p]),
    "dsmil_jpeg_header_bytes_dev": (C.c_int32, []),
    "dsmil_jpeg_workspace_bytes": (c_i64, [C.c_int32, C.c_int32, C.c_int32, c_i64]),
    "dsmil_jpeg_decode_batch": (C.c_int, [C.c_void_p, c_i64, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                          C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, c_i64, C.c_void_p]),
    "dsmil_profile_enable": (C.c_int, [C.c_int]),
    "dsmil_profile_read": (C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_uint64)]),
    "dsmil_forward_path": (C.c_int, [C.POINTER(DsmilParams), c_i64]),
    "dsmil_forward_workspace_bytes": (C.c_size_t, [C.POINTER(DsmilParams), c_i64]),
    "dsmil_forward": (C.c_int, [C.POINTER(DsmilParams), C.c_void_p, C.c_void_p, c_i64,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_forward_bags_workspace_bytes": (C.c_size_t, [C.POINTER(DsmilParams), C.POINTER(c_i64), C.c_int32]),
    "dsmil_forward_bags": (C.c_int, [C.POINTER(DsmilParams), C.POINTER(C.c_void_p), C.POINTER(c_i64), C.c_int32,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_instance_scores": (C.c_int, [C.POINTER(DsmilParams), C.c_void_p, c_i64, C.c_void_p, C.c_void_p]),
    "dsmil_instance_scores_backward": (C.c_int, [C.POINTER(DsmilParams), C.c_void_p, c_i64, C.c_void_p,
                                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                                 C.c_void_p]),
    "dsmil_bag_forward": (C.c_int, [C.POINTER(DsmilParams), C.c_void_p, C.c_void_p, C.c_void_p, c_i64,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_backward_workspace_bytes": (C.c_size_t, [C.POINTER(DsmilParams), c_i64, C.c_int]),
    "dsmil_backward": (C.c_int, [C.POINTER(DsmilParams), C.c_void_p, C.c_void_p, c_i64,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.POINTER(DsmilGrads), C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_cand_floats": (C.c_size_t, [C.c_int32]),
    "dsmil_rec_floats": (C.c_size_t, [C.c_int32, C.c_int32]),
    "dsmil_shard_workspace_bytes": (C.c_size_t, [C.POINTER(DsmilParams), c_i64]),
    "dsmil_shard_phase1": (C.c_int, [C.POINTER(DsmilParams), C.c_void_p, C.c_void_p, C.c_void_p, c_i64, c_i64,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_shard_merge_candidates": (C.c_int, [C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dsmil_shard_phase2": (C.c_int, [C.POINTER(DsmilParams), C.c_void_p, C.c_void_p, c_i64, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_shard_merge_partials": (C.c_int, [C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "dsmil_shard_phase3": (C.c_int, [C.POINTER(DsmilParams), c_i64, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p]),
    "dsmil_shard_backward_phase1": (C.c_int, [C.POINTER(DsmilParams), C.c_void_p, c_i64, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_shard_backward_phase2": (C.c_int, [C.POINTER(DsmilParams), c_i64, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_shard_backward_phase3": (C.c_int, [C.POINTER(DsmilParams), C.c_void_p, c_i64, c_i64, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_forward_bags_train_workspace_bytes": (C.c_size_t, [C.POINTER(DsmilParams), C.POINTER(c_i64), C.c_int32]),
    "dsmil_forward_bags_train": (C.c_int, [C.POINTER(DsmilParams), C.POINTER(C.c_void_p), C.POINTER(c_i64), C.c_int32,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_backward_bags_workspace_bytes": (C.c_size_t, [C.POINTER(DsmilParams), C.POINTER(c_i64), C.c_int32, C.c_int]),
    "dsmil_backward_bags": (C.c_int, [C.POINTER(DsmilParams), C.POINTER(C.c_void_p), C.POINTER(c_i64), C.c_int32,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.POINTER(DsmilGrads), C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_forward_bags_train_dev_workspace_bytes": (C.c_size_t, [C.POINTER(DsmilParams), C.c_int32, c_i64]),
    "dsmil_forward_bags_train_dev": (C.c_int, [C.POINTER(DsmilParams), C.c_void_p, C.c_void_p, C.c_int32, c_i64,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                               C.c_void_p]),
    "dsmil_backward_bags_dev_workspace_bytes": (C.c_size_t, [C.POINTER(DsmilParams), C.c_int32, c_i64]),
    "dsmil_backward_bags_dev": (C.c_int, [C.POINTER(DsmilParams), C.c_void_p, C.c_void_p, C.c_int32, c_i64,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.POINTER(DsmilGrads), C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_shard_bags_supported": (C.c_int, [C.POINTER(DsmilParams)]),
    "dsmil_shard_bags_workspace_bytes": (C.c_size_t, [C.POINTER(DsmilParams), C.POINTER(c_i64), C.c_int32]),
    "dsmil_shard_bags_phase1": (C.c_int, [C.POINTER(DsmilParams), C.POINTER(C.c_void_p), C.POINTER(c_i64), C.c_int32,
                                          C.POINTER(c_i64), C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_shard_bags_phase2": (C.c_int, [C.POINTER(DsmilParams), C.POINTER(C.c_void_p), C.POINTER(c_i64), C.c_int32,
                                          C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_shard_bags_phase3": (C.c_int, [C.POINTER(DsmilParams), C.POINTER(C.c_void_p), C.POINTER(c_i64), C.c_int32,
                                          C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_shard_bags_phase1_train": (C.c_int, [C.POINTER(DsmilParams), C.POINTER(C.c_void_p), C.POINTER(c_i64),
                                                C.c_int32, C.POINTER(c_i64), C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_shard_bags_phase2_train": (C.c_int, [C.POINTER(DsmilParams), C.POINTER(C.c_void_p), C.POINTER(c_i64),
                                                C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_shard_backward_bags_workspace_bytes": (C.c_size_t, [C.POINTER(DsmilParams), C.POINTER(c_i64), C.c_int32]),
    "dsmil_shard_backward_bags_phase1": (C.c_int, [C.POINTER(DsmilParams), C.POINTER(C.c_void_p), C.POINTER(c_i64),
                                                   C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_shard_backward_bags_phase2": (C.c_int, [C.POINTER(DsmilParams), C.POINTER(c_i64), C.c_int32, C.c_void_p,
                                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_void_p, C.c_size_t, C.c_void_p]),
    "dsmil_shard_backward_bags_phase3": (C.c_int, [C.POINTER(DsmilParams), C.POINTER(C.c_void_p), C.POINTER(c_i64),
                                                   C.c_int32, C.POINTER(c_i64), C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
}

_lib: Optional[C.CDLL] = None


def load() -> C.CDLL:
    """Loads the library (once).  Raises if it has not been built: the product has no other path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"libdsmil_b200.so not found at {LIB_PATH}. Build it with `python -m dsmil_wsi_b200.build` "
            "(nvcc, sm_90a). There is no CPU or PyTorch fallback for the DSMIL hot path.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the header and the library disagree
        fn.restype = res
        fn.argtypes = args
    if lib.dsmil_abi_version() != 1:
        raise RuntimeError("libdsmil_b200.so ABI version mismatch")
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().dsmil_last_error()
        raise RuntimeError(f"{what} failed (status {rc}): {msg.decode() if msg else '?'}")


def launch_count() -> int:
    return int(load().dsmil_launch_count())
