"""ctypes binding of libdcr_b200.so (include/dcr_b200.h).  The product path has no CPU fallback: if the library is
missing or a call fails, a DcrError is raised."""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
LIB_PATH = Path(os.environ.get("DCR_B200_LIB", PKG_DIR / "libdcr_b200.so"))


class DcrError(RuntimeError):
    pass


ERR_CAPACITY = -3   # DCR_ERR_CAPACITY: dcr_sim_range(_split|_cross)(_sharded) found more candidate pairs than its capacities


# name -> (restype, argtypes); mirrors include/dcr_b200.h one to one (tests check the header against this table)
SIGNATURES = {
    "dcr_version": (C.c_int, []),
    "dcr_last_error": (C.c_char_p, []),
    "dcr_device_sm_count": (C.c_int, []),
    "dcr_l2_normalize": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "dcr_sim_topk_workspace_size": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "dcr_sim_topk": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int64,
                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dcr_sim_topk_split_workspace_size": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "dcr_sim_topk_split": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64,
                                     C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dcr_sim_topk_cross_workspace_size": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "dcr_sim_topk_cross": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64,
                                     C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dcr_sim_topk_host": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                    C.c_void_p]),
    "dcr_sim_topk_sharded_workspace_size": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "dcr_sim_topk_sharded": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dcr_sim_range_workspace_size": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int64]),
    "dcr_sim_range": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int64, C.c_int64,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_void_p,
                                C.c_size_t, C.c_void_p]),
    "dcr_sim_range_sharded_workspace_size": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64]),
    "dcr_sim_range_sharded": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int64,
                                        C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_int64, C.c_int64, C.POINTER(C.c_int64), C.c_void_p, C.c_size_t,
                                        C.c_void_p]),
    "dcr_sim_range_split_workspace_size": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64]),
    "dcr_sim_range_split": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int64,
                                      C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64),
                                      C.c_void_p, C.c_size_t, C.c_void_p]),
    "dcr_sim_range_cross_workspace_size": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64]),
    "dcr_sim_range_cross": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int64,
                                      C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64),
                                      C.c_void_p, C.c_size_t, C.c_void_p]),
    "dcr_sim_range_split_sharded_workspace_size": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64]),
    "dcr_sim_range_split_sharded": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float,
                                              C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.POINTER(C.c_int64),
                                              C.c_void_p, C.c_size_t, C.c_void_p]),
    "dcr_sim_range_cross_sharded_workspace_size": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64]),
    "dcr_sim_range_cross_sharded": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float,
                                              C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.POINTER(C.c_int64),
                                              C.c_void_p, C.c_size_t, C.c_void_p]),
    "dcr_sim_topk_last_stats": (C.c_int, [C.POINTER(C.c_int)]),
    "dcr_sim_topk_last_kernel_ms": (C.c_float, []),
    "dcr_sim_topk_last_sm_mhz": (C.c_float, []),
    "dcr_sim_topk_last_epilogue_sets": (C.c_int, []),
    "dcr_sim_topk_last_second_pass": (C.c_int, []),
    "dcr_kernel_launch_count": (C.c_longlong, []),
    "dcr_conv2d_bf16": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int,
                                  C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                  C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int,
                                  C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "dcr_net_create": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "dcr_net_set_exact": (C.c_int, [C.c_void_p, C.c_int]),
    "dcr_net_destroy": (None, [C.c_void_p]),
    "dcr_net_fork": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "dcr_net_add_tensor": (C.c_int, [C.c_void_p, C.c_int64, C.c_int]),
    "dcr_net_alias_tensor": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int]),
    "dcr_net_add_param": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "dcr_net_set_output": (C.c_int, [C.c_void_p, C.c_int]),
    "dcr_net_add_op": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_float), C.c_int]),
    "dcr_net_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "dcr_net_tensor": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]),
    "dcr_stem_plane_units": (C.c_int64, [C.c_int, C.c_int]),
    "dcr_net_forward_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "dcr_fid_create": (C.c_int, [C.c_int, C.POINTER(C.c_void_p)]),
    "dcr_fid_destroy": (None, [C.c_void_p]),
    "dcr_fid_accumulate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "dcr_fid_finalize": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p]),
    "dcr_fid_packed_size": (C.c_size_t, [C.c_int]),
    "dcr_fid_export": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "dcr_fid_merge": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "dcr_split_rescore": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                    C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dcr_topk_merge": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                 C.c_void_p]),
    "dcr_image_stats": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dcr_jpeg_workspace_size": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "dcr_jpeg_max_bytes": (C.c_int64, [C.c_int, C.c_int]),
    "dcr_jpeg_encode": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_size_t, C.c_void_p]),
}

# the all-gather callback of dcr_sim_topk_sharded / dcr_sim_range_sharded: int (*)(const void* send, void* recv, size_t bytes_per_rank, void* ctx, void* stream)
ALLGATHER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p)

_lib = None


def load() -> C.CDLL:
    """Load the shared library (once).  Raises DcrError with a build hint when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise DcrError(
            f"{LIB_PATH} not found: build it with `python -m dcr_b200.build` (needs nvcc). "
            "dcr_b200 has no CPU fallback for its compute path.")
    lib = C.CDLL(str(LIB_PATH))
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:  # pragma: no cover
            raise DcrError(f"{LIB_PATH} does not export {name}; rebuild (python -m dcr_b200.build --force)") from e
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error() -> str:
    return load().dcr_last_error().decode("utf-8", "replace")


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise DcrError(f"{what} failed (rc={rc}): {last_error()}")
