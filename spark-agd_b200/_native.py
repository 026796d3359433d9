"""ctypes binding of libagd_b200.so (include/agd_b200.h).  No fallback: if the CUDA extension is
missing or cannot be built, importing a compute entry point raises."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libagd_b200.so")
CSRC = os.path.join(_HERE, "csrc")
HEADER = os.path.join(os.path.dirname(_HERE), "include", "agd_b200.h")

GRAD_LOGISTIC, GRAD_LEAST_SQUARES, GRAD_HINGE, GRAD_LEAST_SQUARES_HALF = 0, 1, 2, 3
UPD_SIMPLE, UPD_SQUARED_L2, UPD_L1 = 0, 1, 2
F64, F32, BF16 = 0, 1, 2
FLAG_MEMOIZE_FX = 1
FLAG_NO_FUSE = 2
ABI_VERSION = 2
XCHG_HANDLE_BYTES = 192
# agd_evaluate: indices of the sums it returns (AGD_EVAL_*), EVAL_N of them
(EVAL_COUNT, EVAL_LOSS, EVAL_TP, EVAL_FP, EVAL_TN, EVAL_FN, EVAL_SUM_ERR, EVAL_SUM_ERR2, EVAL_SUM_ABS_ERR, EVAL_SUM_Y,
 EVAL_SUM_Y2, EVAL_N) = range(12)
# agd_binary_curve: the summary it returns (AGD_BIN_*), BIN_N doubles
BIN_POS, BIN_NEG, BIN_NAN, BIN_AUROC, BIN_AUPR, BIN_N = range(6)
# agd_col_stats: rows of the statistic-major block it returns (AGD_COLSTAT_*), COLSTAT_N of them
(COLSTAT_SUM, COLSTAT_SUM_SQ, COLSTAT_SUM_ABS, COLSTAT_NNZ, COLSTAT_DEV, COLSTAT_DEV2, COLSTAT_MAX, COLSTAT_MIN,
 COLSTAT_N) = range(9)
# agd_gramian: the largest agd_dim(h) it takes (AGD_GRAMIAN_MAX_DIM; beyond it the call fails and allocates nothing)
GRAMIAN_MAX_DIM = 8192
# agd_class_sums / agd_linear_confusion: the most class labels they take (AGD_MAX_CLASSES)
MAX_CLASSES = 1024


class Params(C.Structure):
    _fields_ = [("convergence_tol", C.c_double), ("num_iterations", C.c_int32), ("reg_param", C.c_double),
                ("L0", C.c_double), ("Lexact", C.c_double), ("beta", C.c_double), ("alpha", C.c_double),
                ("may_restart", C.c_int32), ("gradient", C.c_int32), ("updater", C.c_int32), ("flags", C.c_int32)]


class Stats(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("passes", C.c_int32), ("backtracks", C.c_int32),
                ("restarts", C.c_int32), ("converged", C.c_int32), ("stopped_nan", C.c_int32),
                ("nonterminating", C.c_int32), ("collective_kind", C.c_int32), ("final_L", C.c_double),
                ("final_theta", C.c_double), ("seconds_total", C.c_double), ("k1_ms_total", C.c_double),
                ("k1_launches", C.c_int64), ("gpu_launches", C.c_int64), ("allreduce_ms_total", C.c_double),
                ("device_ms_total", C.c_double), ("collective_calls", C.c_int64), ("wasted_passes", C.c_int32),
                ("fused_passes", C.c_int32)]


def _sources():
    out = [HEADER, os.path.join(CSRC, "Makefile")]
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh")):
            out.append(os.path.join(CSRC, f))
    return out


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every CUDA source for sm_90a into spark-agd_b200/libagd_b200.so (nvcc cross-compiles
    without a GPU).  Rebuilds only when a source is newer than the library."""
    stale = (not os.path.exists(LIB_PATH)) or any(
        os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in _sources())
    if force or stale:
        cmd = ["make", "-C", CSRC, "-j4"] + (["-B"] if force else [])
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if verbose or res.returncode != 0:
            print(res.stdout)
        if res.returncode != 0:
            raise RuntimeError("building libagd_b200.so failed (nvcc for sm_90a is required; there is no fallback)")
    return LIB_PATH


_lib = None

_SIGNATURES = {
    "agd_abi_version": (C.c_int, []),
    "agd_sizeof_params": (C.c_int, []),
    "agd_sizeof_stats": (C.c_int, []),
    "agd_default_params": (None, [C.POINTER(Params)]),
    "agd_create": (C.c_int, [C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_void_p)]),
    "agd_destroy": (C.c_int, [C.c_void_p]),
    "agd_last_error": (C.c_char_p, [C.c_void_p]),
    "agd_comm_unique_id": (C.c_int, [C.c_void_p]),
    "agd_comm_init": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]),
    "agd_comm_init_ipc": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32]),
    "agd_xchg_export": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]),
    "agd_xchg_import": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64]),
    "agd_kernel_name": (C.c_char_p, [C.c_void_p, C.c_int32]),
    "agd_reserve": (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.c_int32, C.c_int32]),
    "agd_load_dense": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64,
                                 C.c_int32, C.c_int64, C.c_int32]),
    "agd_load_csr": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                               C.c_void_p, C.c_int64, C.c_int32, C.c_int32]),
    "agd_libsvm_read": (C.c_int, [C.c_char_p, C.c_int32, C.POINTER(C.c_void_p)]),
    "agd_libsvm_rows": (C.c_int64, [C.c_void_p]),
    "agd_libsvm_dim": (C.c_int32, [C.c_void_p]),
    "agd_libsvm_nnz": (C.c_int64, [C.c_void_p]),
    "agd_libsvm_rowptr": (C.c_void_p, [C.c_void_p]),
    "agd_libsvm_indices": (C.c_void_p, [C.c_void_p]),
    "agd_libsvm_values": (C.c_void_p, [C.c_void_p]),
    "agd_libsvm_labels": (C.c_void_p, [C.c_void_p]),
    "agd_libsvm_error": (C.c_char_p, [C.c_void_p]),
    "agd_libsvm_free": (None, [C.c_void_p]),
    "agd_load_libsvm": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int32, C.c_int32]),
    "agd_clear": (C.c_int, [C.c_void_p]),
    "agd_rows": (C.c_int64, [C.c_void_p, C.c_int32]),
    "agd_dim": (C.c_int32, [C.c_void_p]),
    "agd_generate": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_uint64, C.c_int32]),
    "agd_get_rows": (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "agd_synth_wtrue": (C.c_int, [C.c_void_p, C.c_uint64, C.c_int32, C.c_void_p]),
    "agd_generate_csr": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_uint64, C.c_int32]),
    "agd_get_csr_rows": (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_int64, C.c_void_p]),
    "agd_smooth": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(C.c_double), C.c_void_p,
                             C.POINTER(C.c_int64)]),
    "agd_smooth_pair": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(C.c_double), C.c_void_p,
                                  C.POINTER(C.c_int64), C.POINTER(C.c_double)]),
    "agd_smooth_two": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(C.c_double), C.c_void_p,
                                 C.POINTER(C.c_int64), C.POINTER(C.c_double), C.c_void_p]),
    "agd_margins": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_double, C.c_int64, C.c_int64, C.c_void_p]),
    "agd_evaluate": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_double, C.c_double, C.c_void_p]),
    "agd_col_stats": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.c_void_p]),
    "agd_gramian": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_double), C.c_void_p]),
    "agd_project": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32]),
    "agd_binary_curve": (C.c_int, [C.c_void_p, C.c_void_p, C.c_double, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.POINTER(C.c_int64), C.c_void_p]),
    "agd_kmeans_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(C.c_double)]),
    "agd_kmeans_assign": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "agd_kmeans_costs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_double)]),
    "agd_kmeans_sample": (C.c_int, [C.c_void_p, C.c_uint64, C.c_double, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p,
                                    C.POINTER(C.c_int64)]),
    "agd_label_classes": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64),
                                    C.POINTER(C.c_int64)]),
    "agd_class_sums": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(C.c_double)]),
    "agd_linear_argmax": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_int64,
                                    C.c_void_p]),
    "agd_linear_confusion": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "agd_set_row_filter": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "agd_row_filter_mask": (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.c_int64, C.c_void_p]),
    "agd_set_feature_transform": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32]),
    "agd_prox": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_int32,
                           C.c_void_p, C.POINTER(C.c_double)]),
    "agd_run": (C.c_int, [C.c_void_p, C.POINTER(Params), C.c_void_p, C.c_void_p, C.c_void_p,
                          C.POINTER(C.c_int32), C.POINTER(Stats)]),
    "agd_gd_run": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_double, C.c_int32, C.c_double, C.c_void_p,
                             C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(Stats)]),
    "agd_gd_run_minibatch": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_double, C.c_int32, C.c_double, C.c_double,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(Stats)]),
    "agd_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_char_p]),
}


def lib():
    """dlopen the C-ABI library (building it first if needed) and attach prototypes."""
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError here means the .so does not export the ABI
            fn.restype = res
            fn.argtypes = args
        if L.agd_abi_version() != ABI_VERSION:
            raise RuntimeError("libagd_b200.so ABI version mismatch")
        if L.agd_sizeof_params() != C.sizeof(Params) or L.agd_sizeof_stats() != C.sizeof(Stats):
            raise RuntimeError("agd_params / agd_stats layout differs between the binding and the library")
        _lib = L
    return _lib


def exported_symbols():
    return sorted(_SIGNATURES)


class NativeError(RuntimeError):
    pass


def check(rc: int, handle=None):
    if rc != 0:
        msg = lib().agd_last_error(handle)
        raise NativeError((msg or b"unknown error").decode())
