"""ctypes binding of libcfmm_b200.so (the C ABI in include/cfmm_b200.h).

There is no CPU fallback: if the library cannot be built or loaded, every entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

KIND_PRODUCT, KIND_SUM, KIND_GEOMEAN, KIND_BOUNDED, KIND_STABLESWAP, KIND_STABLESWAP_N, KIND_CONCENTRATED = 0, 1, 2, 3, 4, 5, 6
KIND_CRYPTOSWAP, KIND_CRYPTOSWAP_3 = 8, 9
KIND_BINS = 10
KIND_ECLP = 11
KIND_PMM = 12

_ERRORS = {
    -1: "CFMM_E_NULL (required pointer is NULL)",
    -2: "CFMM_E_KIND (unknown kind / unsupported arity)",
    -3: "CFMM_E_SIZE (bad size)",
    -4: "CFMM_E_CUDA (CUDA runtime error)",
    -5: "CFMM_E_NODEVICE (no sm_90 device)",
    -6: "CFMM_E_STATE (handle used in the wrong state)",
}


class CfmmError(RuntimeError):
    pass


class Bucket(C.Structure):
    _fields_ = [
        ("kind", C.c_int32), ("arity", C.c_int32), ("n_pools", C.c_int64), ("stride", C.c_int64),
        ("reserves", C.c_void_p), ("tok_idx", C.c_void_p), ("gamma", C.c_void_p),
        ("weights", C.c_void_p), ("logrw", C.c_void_p), ("theta_bar", C.c_void_p),
    ]


class BlockedPairs(C.Structure):
    _fields_ = [
        ("n_pools", C.c_int64), ("n_tiles", C.c_int64), ("pools_per_tile", C.c_int32), ("reserved", C.c_int32),
        ("r0", C.c_void_p), ("r1", C.c_void_p), ("gamma_inv", C.c_void_p), ("pw", C.c_void_p),
        ("fee", C.c_void_p), ("rows", C.c_void_p), ("tok", C.c_void_p), ("desc", C.c_void_p),
    ]


class SolveParams(C.Structure):
    _fields_ = [("tol", C.c_double), ("nu_floor", C.c_double), ("max_iter", C.c_int32), ("cg_max", C.c_int32)]


class MarketParams(C.Structure):
    _fields_ = [("tol", C.c_double), ("nu_floor", C.c_double), ("eps0", C.c_double), ("eps_min", C.c_double),
                ("eps_shrink", C.c_double), ("max_iter", C.c_int32), ("cg_max", C.c_int32), ("max_outer", C.c_int32),
                ("linear_solver", C.c_int32)]


class SolveResult(C.Structure):
    _fields_ = [("dual_value", C.c_double), ("primal_value", C.c_double), ("gap", C.c_double),
                ("primal_infeas", C.c_double), ("err", C.c_double), ("iters", C.c_int32), ("evals", C.c_int32),
                ("hvps", C.c_int32), ("status", C.c_int32)]


class PeerCtx(C.Structure):
    _fields_ = [("recv_acc_dev", C.c_void_p), ("recv_vec_dev", C.c_void_p), ("rank", C.c_int32), ("world", C.c_int32),
                ("seq_acc", C.c_uint64), ("seq_vec", C.c_uint64)]


class CsrPools(C.Structure):
    _fields_ = [("n_tokens", C.c_int32), ("n_pools", C.c_int64), ("nnz", C.c_int64), ("pool_ptr", C.c_void_p),
                ("tok_idx", C.c_void_p), ("reserves", C.c_void_p), ("weights", C.c_void_p), ("logrw", C.c_void_p),
                ("gamma", C.c_void_p), ("kind", C.c_void_p)]


class Batch(C.Structure):
    _fields_ = [("n_problems", C.c_int32), ("pool_range", C.c_void_p), ("c", C.c_void_p), ("a", C.c_void_p),
                ("flags", C.c_void_p), ("nu", C.c_void_p), ("psi", C.c_void_p), ("stats", C.c_void_p),
                ("delta", C.c_void_p), ("lambda_", C.c_void_p), ("trade_stride", C.c_int64)]


class BatchParams(C.Structure):
    _fields_ = [("tol", C.c_double), ("eps0", C.c_double), ("eps_min", C.c_double), ("eps_shrink", C.c_double),
                ("floor_rel", C.c_double), ("max_outer", C.c_int32), ("max_inner", C.c_int32)]


class EvalOut(C.Structure):
    _fields_ = [("delta", C.c_void_p), ("lambda_", C.c_void_p), ("hcoef", C.c_void_p), ("hmask", C.c_void_p)]


_lib = None


def lib_path() -> str:
    return _build.LIB


def load(build_if_missing: bool = True):
    """Load (building first if the .so is absent or stale and nvcc is present)."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    if build_if_missing and _build.needs_build():
        try:
            _build.build_library()
        except Exception as e:  # stale .so + no nvcc (GPU box): use what travelled
            if not os.path.exists(path):
                raise CfmmError(f"libcfmm_b200.so is missing and could not be built: {e}") from e
    if not os.path.exists(path):
        raise CfmmError("libcfmm_b200.so is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
    lib = C.CDLL(path)
    vp, i32, i64, dbl = C.c_void_p, C.c_int32, C.c_int64, C.c_double
    lib.cfmm_arb_eval.argtypes = [C.POINTER(Bucket), i32, vp, vp, dbl, vp, vp, C.POINTER(EvalOut), vp]
    lib.cfmm_arb_eval.restype = C.c_int
    for name in ("cfmm_hvp", "cfmm_hess_diag", "cfmm_hess_dense"):
        fn = getattr(lib, name)
        fn.restype = C.c_int
    lib.cfmm_hvp.argtypes = [C.POINTER(Bucket), i32, vp, vp, vp, vp, vp]
    lib.cfmm_hess_diag.argtypes = [C.POINTER(Bucket), i32, vp, vp, vp, vp]
    lib.cfmm_hess_dense.argtypes = [C.POINTER(Bucket), i32, vp, vp, vp, vp]
    lib.cfmm_blocked_layout_info.argtypes = [C.POINTER(i32)] * 4
    lib.cfmm_blocked_layout_info.restype = C.c_int
    lib.cfmm_blocked_fee_words.argtypes = []
    lib.cfmm_blocked_fee_words.restype = i32
    lib.cfmm_set_blocked_config.argtypes = [i32]
    lib.cfmm_set_blocked_config.restype = C.c_int
    lib.cfmm_blocked_build_work_bytes.argtypes = [i64]
    lib.cfmm_blocked_build_work_bytes.restype = i64
    lib.cfmm_blocked_build.argtypes = [i64, i32, vp, vp, vp, C.POINTER(BlockedPairs), vp, vp, vp, i64, vp]
    lib.cfmm_blocked_build.restype = C.c_int
    lib.cfmm_blocked_update_work_bytes.argtypes = [C.POINTER(BlockedPairs)]
    lib.cfmm_blocked_update_work_bytes.restype = i64
    lib.cfmm_blocked_update.argtypes = [C.POINTER(BlockedPairs), i64, vp, vp, vp, C.POINTER(i32), vp, i64, vp]
    lib.cfmm_blocked_update.restype = C.c_int
    lib.cfmm_ladder_splice_work_bytes.argtypes = [i64, i64]
    lib.cfmm_ladder_splice_work_bytes.restype = i64
    lib.cfmm_ladder_splice.argtypes = [C.POINTER(Bucket), i64, vp, vp, vp, i64, vp, vp, i64, C.POINTER(i64), vp, i64, vp]
    lib.cfmm_ladder_splice.restype = C.c_int
    lib.cfmm_bins_splice.argtypes = [C.POINTER(Bucket), i64, vp, vp, vp, i64, vp, vp, i64, C.POINTER(i64), vp, i64, vp]
    lib.cfmm_bins_splice.restype = C.c_int
    lib.cfmm_blocked_eval.argtypes = [C.POINTER(BlockedPairs), i32, vp, vp, vp, C.POINTER(EvalOut), vp, i64, vp]
    lib.cfmm_blocked_eval.restype = C.c_int
    lib.cfmm_blocked_hvp.argtypes = [C.POINTER(BlockedPairs), i32, vp, vp, vp, vp, vp]
    lib.cfmm_blocked_hvp.restype = C.c_int
    lib.cfmm_blocked_diag.argtypes = [C.POINTER(BlockedPairs), i32, vp, vp, vp]
    lib.cfmm_blocked_diag.restype = C.c_int
    lib.cfmm_blocked_dense.argtypes = [C.POINTER(BlockedPairs), i32, vp, vp, vp]
    lib.cfmm_blocked_dense.restype = C.c_int
    lib.cfmm_blocked_solve_work_bytes.argtypes = [C.POINTER(BlockedPairs), i32]
    lib.cfmm_blocked_solve_work_bytes.restype = i64
    lib.cfmm_blocked_solve.argtypes = [C.POINTER(BlockedPairs), i32, vp, vp, vp, vp, vp, vp, vp,
                                       C.POINTER(SolveParams), C.POINTER(SolveResult), vp]
    lib.cfmm_blocked_solve.restype = C.c_int
    lib.cfmm_blocked_solve_peer.argtypes = [C.POINTER(BlockedPairs), i32, vp, vp, vp, vp, vp, vp, vp,
                                            C.POINTER(SolveParams), C.POINTER(SolveResult), C.POINTER(PeerCtx), vp]
    lib.cfmm_blocked_solve_peer.restype = C.c_int
    lib.cfmm_market_solve_work_bytes.argtypes = [C.POINTER(Bucket), i32, C.POINTER(BlockedPairs), i32, i32]
    lib.cfmm_market_solve_work_bytes.restype = i64
    lib.cfmm_market_solve.argtypes = [C.POINTER(Bucket), C.POINTER(EvalOut), i32, C.POINTER(BlockedPairs),
                                      C.POINTER(EvalOut), i32, vp, vp, vp, vp, vp, vp, vp, C.POINTER(MarketParams),
                                      C.POINTER(SolveResult), vp]
    lib.cfmm_market_solve.restype = C.c_int
    lib.cfmm_dense_cholesky.argtypes = [i32, vp, vp, vp]
    lib.cfmm_dense_cholesky.restype = C.c_int
    lib.cfmm_persist_solve_work_bytes.argtypes = [C.POINTER(BlockedPairs), i32]
    lib.cfmm_persist_solve_work_bytes.restype = i64
    lib.cfmm_persist_solve.argtypes = lib.cfmm_blocked_solve_peer.argtypes
    lib.cfmm_persist_solve.restype = C.c_int
    lib.cfmm_set_persist_cooperative.argtypes = [i32]
    lib.cfmm_set_persist_cooperative.restype = C.c_int
    lib.cfmm_persist_last_profile.argtypes = [vp]
    lib.cfmm_persist_last_profile.restype = C.c_int
    lib.cfmm_batch_solve_work_bytes.argtypes = [C.POINTER(CsrPools), i32, i64]
    lib.cfmm_batch_solve_work_bytes.restype = i64
    lib.cfmm_set_batch_lanes.argtypes = [i32]
    lib.cfmm_set_batch_lanes.restype = C.c_int
    lib.cfmm_batch_solve.argtypes = [C.POINTER(CsrPools), C.POINTER(Batch), C.POINTER(BatchParams), vp, vp]
    lib.cfmm_batch_solve.restype = C.c_int
    lib.cfmm_batch_solve_stableswap.argtypes = lib.cfmm_batch_solve.argtypes
    lib.cfmm_batch_solve_stableswap.restype = C.c_int
    lib.cfmm_batch_solve_stableswap_n.argtypes = lib.cfmm_batch_solve.argtypes
    lib.cfmm_batch_solve_stableswap_n.restype = C.c_int
    lib.cfmm_batch_solve_concentrated.argtypes = [C.POINTER(CsrPools), vp, C.POINTER(Batch), C.POINTER(BatchParams), vp, vp]
    lib.cfmm_batch_solve_concentrated.restype = C.c_int
    lib.cfmm_batch_solve_cryptoswap.argtypes = lib.cfmm_batch_solve_concentrated.argtypes
    lib.cfmm_batch_solve_cryptoswap.restype = C.c_int
    lib.cfmm_batch_solve_tricrypto.argtypes = lib.cfmm_batch_solve_concentrated.argtypes
    lib.cfmm_batch_solve_tricrypto.restype = C.c_int
    lib.cfmm_batch_solve_bins.argtypes = lib.cfmm_batch_solve_concentrated.argtypes
    lib.cfmm_batch_solve_bins.restype = C.c_int
    lib.cfmm_batch_solve_eclp.argtypes = lib.cfmm_batch_solve_concentrated.argtypes
    lib.cfmm_batch_solve_eclp.restype = C.c_int
    lib.cfmm_batch_solve_pmm.argtypes = lib.cfmm_batch_solve_concentrated.argtypes
    lib.cfmm_batch_solve_pmm.restype = C.c_int
    lib.cfmm_allreduce_ll.argtypes = [vp, vp, i32, i32, i32, i64, i64, vp, C.c_uint64, vp]
    lib.cfmm_allreduce_ll.restype = C.c_int
    lib.cfmm_sum_update_multipliers.argtypes = [C.POINTER(Bucket), vp, vp, vp, vp]
    lib.cfmm_sum_update_multipliers.restype = C.c_int
    lib.cfmm_bins_update_multipliers.argtypes = [C.POINTER(Bucket), vp, vp, vp, vp, vp]
    lib.cfmm_bins_update_multipliers.restype = C.c_int
    lib.cfmm_zero.argtypes = [vp, i64, vp]
    lib.cfmm_zero.restype = C.c_int
    lib.cfmm_set_scatter_mode.argtypes = [i32]
    lib.cfmm_set_scatter_mode.restype = C.c_int
    lib.cfmm_launch_count.restype = i64
    lib.cfmm_reset_launch_count.restype = None
    lib.cfmm_last_cuda_error.restype = C.c_char_p
    lib.cfmm_version.restype = C.c_char_p
    if os.environ.get("CFMM_BATCH_LANES"):          # 1 | 32 threads per problem in cfmm_batch_solve (experiments)
        lib.cfmm_set_batch_lanes(int(os.environ["CFMM_BATCH_LANES"]))
    if os.environ.get("CFMM_BLOCKED_CFG"):          # experiment knobs, e.g. "200" = no programmatic dependent launch
        for c in os.environ["CFMM_BLOCKED_CFG"].split(","):
            lib.cfmm_set_blocked_config(int(c))
    _lib = lib
    return lib


def check(rc: int, what: str = "cfmm call"):
    if rc != 0:
        extra = ""
        if rc == -4 and _lib is not None:
            extra = ": " + _lib.cfmm_last_cuda_error().decode()
        raise CfmmError(f"{what} failed: {_ERRORS.get(rc, rc)}{extra}")
