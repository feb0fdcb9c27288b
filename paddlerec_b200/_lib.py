"""ctypes binding of libb200rec.so (the C ABI declared in include/b200rec.h).

The product path has NO fallback: if the shared library is missing or a call returns an error
code, we raise.  Nothing here imports `oracle/`.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import sys
from ctypes import c_char_p, c_double, c_float, c_int, c_int64, c_size_t, c_void_p, POINTER, c_uint64

_HERE = os.path.dirname(os.path.abspath(__file__))
REPO_ROOT = os.path.dirname(_HERE)
CSRC = os.path.join(_HERE, "csrc")
LIB_DIR = os.path.join(_HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libb200rec.so")
INCLUDE_DIR = os.path.join(REPO_ROOT, "include")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-shared", "-Xcompiler", "-fPIC",
]


class B200RecError(RuntimeError):
    pass


def _sources():
    out = [os.path.join(INCLUDE_DIR, "b200rec.h")]
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh", ".inc", ".h")):
            out.append(os.path.join(CSRC, f))
    return out


def needs_build() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(s) > t for s in _sources())


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/b200rec.cu for sm_90a (H100) into paddlerec_b200/lib/libb200rec.so (in-tree)."""
    if not force and not needs_build():
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "nvcc")
    os.makedirs(LIB_DIR, exist_ok=True)
    tmp = LIB_PATH + ".tmp.%d" % os.getpid()
    cmd = [nvcc, *NVCC_FLAGS, "-I", INCLUDE_DIR, os.path.join(CSRC, "b200rec.cu"), "-o", tmp]
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
        print(" ".join(cmd), file=sys.stderr)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise B200RecError("nvcc failed:\n" + res.stdout + res.stderr)
    os.replace(tmp, LIB_PATH)
    if verbose:
        print(res.stderr, file=sys.stderr)
    return LIB_PATH


ABI_VERSION = 7
_P = c_void_p
_SIG = {
    "b200rec_abi_version": (c_int, []),
    "b200rec_last_error": (c_char_p, []),
    "b200rec_oob_count": (c_int, [POINTER(c_uint64), c_int, _P]),
    "b200rec_embed_fm_fwd": (c_int, [_P, c_int64, _P, c_int64, _P, _P, _P, _P, _P, _P, _P, _P,
                                     c_int64, c_int, c_int, c_int, c_int64, c_int64, _P]),
    "b200rec_group_ids_workspace_bytes": (c_int, [c_int64, c_int64, POINTER(c_size_t)]),
    "b200rec_group_ids": (c_int, [_P, c_int64, c_int64, c_int64, _P, _P, _P, _P, _P, c_size_t, _P]),
    "b200rec_embed_fm_bwd_workspace_bytes": (c_int, [c_int64, c_int, c_int, c_int,
                                                     POINTER(c_size_t)]),
    "b200rec_embed_fm_bwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int64, _P, c_int64,
                                     c_int, _P, _P, c_int64, c_int, c_int, c_int, _P, c_size_t,
                                     _P]),
    "b200rec_ffm_fwd": (c_int, [_P, c_int64, _P, _P, _P, _P, _P, _P, _P, c_int64, c_int, c_int,
                                c_int, c_int64, c_int64, _P]),
    "b200rec_ffm_bwd_workspace_bytes": (c_int, [c_int64, c_int, c_int, c_int, POINTER(c_size_t)]),
    "b200rec_ffm_bwd": (c_int, [_P, c_int64, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int64, _P, _P,
                                _P, c_int64, c_int, c_int, c_int, c_int64, c_int64, _P, c_size_t,
                                _P]),
    "b200rec_fat_ffm_pool_fwd": (c_int, [_P, c_int64, _P, _P, _P, _P, c_int64, c_int, c_int, c_int,
                                         c_int64, c_int64, _P]),
    "b200rec_fat_ffm_fwd": (c_int, [_P, c_int64, _P, _P, _P, _P, _P, _P, _P, c_int64, c_int, c_int,
                                    c_int, c_int64, c_int64, _P]),
    "b200rec_fat_ffm_bwd_attn": (c_int, [_P, c_int64, _P, _P, _P, _P, _P, _P, _P, c_int64, c_int,
                                         c_int, c_int, c_int64, c_int64, _P]),
    "b200rec_fat_ffm_bwd_workspace_bytes": (c_int, [c_int64, c_int, c_int, c_int,
                                                    POINTER(c_size_t)]),
    "b200rec_fat_ffm_bwd": (c_int, [_P, c_int64, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int64,
                                    _P, _P, c_int64, c_int, c_int, c_int, c_int64, c_int64, _P,
                                    c_size_t, _P]),
    "b200rec_gather": (c_int, [_P, c_int64, _P, _P, c_int64, c_int, c_int64, c_int64, _P]),
    "b200rec_gate_embed_fwd": (c_int, [_P, c_int64, _P, _P, _P, _P, c_int64, c_int64, c_int, c_int,
                                       c_int, c_int64, _P]),
    "b200rec_gate_embed_bwd_workspace_bytes": (c_int, [c_int64, c_int, POINTER(c_size_t)]),
    "b200rec_gate_embed_bwd": (c_int, [_P, c_int64, _P, _P, _P, c_int64, _P, _P, c_int64, c_int, c_int,
                                       c_int64, _P, c_size_t, _P]),
    "b200rec_segment_reduce_workspace_bytes": (c_int, [c_int64, c_int, POINTER(c_size_t)]),
    "b200rec_segment_reduce": (c_int, [_P, _P, _P, _P, _P, _P, c_int64, c_int, _P, c_size_t, _P]),
    "b200rec_gather_pool_sum": (c_int, [_P, c_int64, _P, _P, _P, _P, c_int64, c_int, c_int64,
                                        c_int64, _P]),
    "b200rec_rows_to_dense": (c_int, [_P, _P, c_int64, _P, _P, c_int64, c_int64, c_int, c_int64,
                                      _P]),
    "b200rec_sparse_sgd": (c_int, [_P, c_int64, _P, _P, c_int64, _P, c_int64, c_int, c_int64,
                                   c_double, _P]),
    "b200rec_sparse_adam": (c_int, [_P, _P, _P, c_int64, _P, _P, c_int64, _P, c_int64, c_int,
                                    c_int64, c_double, c_double, c_double, c_double, c_double,
                                    c_double, _P]),
    "b200rec_sparse_adagrad": (c_int, [_P, _P, c_int64, _P, _P, c_int64, _P, c_int64, c_int,
                                       c_int64, c_double, c_double, c_double, c_double, _P]),
    "b200rec_cross_v2_fwd": (c_int, [_P, _P, _P, _P, _P, c_int64, c_int, _P]),
    "b200rec_cross_bwd_workspace_bytes": (c_int, [c_int64, c_int, POINTER(c_size_t)]),
    "b200rec_cross_v2_bwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, c_int64, c_int, _P, c_size_t, _P]),
    "b200rec_din_attn_fwd": (c_int, [_P] * 13 + [c_int64, c_int, c_int, c_float, _P]),
    "b200rec_din_attn_bwd_workspace_bytes": (c_int, [c_int64, c_int, c_int, POINTER(c_size_t)]),
    "b200rec_din_attn_bwd": (c_int, [_P] * 19 + [c_int64, c_int, c_int, c_float, _P, c_size_t,
                                                  _P]),
    "b200rec_cvm_fwd": (c_int, [_P, _P, c_int64, c_int, c_int, _P]),
    "b200rec_cvm_bwd": (c_int, [_P, _P, _P, c_int64, c_int, c_int, _P]),
    "b200rec_tower_split": (c_int, [_P, _P, c_int, _P, c_int64, c_int, _P]),
    "b200rec_tower_bwd_workspace_bytes": (c_int, [c_int64, c_int, POINTER(c_size_t)]),
    "b200rec_tower_relu_bwd_split": (c_int, [_P, _P, _P, _P, c_int64, c_int, _P, c_size_t, _P]),
    "b200rec_tower_prep_weight": (c_int, [_P, _P, _P, _P, c_int, c_int, _P]),
    "b200rec_tower_fold_dw": (c_int, [_P, _P, c_int, c_int, _P]),
    "b200rec_shard_gather_push": (c_int, [_P, c_int64, c_int, c_int64, c_int64, _P, _P, _P,
                                          POINTER(c_uint64), c_int64, c_int, c_int64, _P]),
    "b200rec_shard_fm_grads_push": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, POINTER(c_uint64), c_int64,
                                            c_int, c_int64, c_int, c_int, c_int, c_int, _P]),
    "b200rec_shard_push_rows": (c_int, [_P, c_int64, c_int, _P, _P, POINTER(c_uint64), c_int64,
                                        c_int, c_int64, _P]),
    "b200rec_tc_split": (c_int, [_P, c_int64, _P, c_int, _P, c_int64, c_int64, c_int, c_int, _P]),
    "b200rec_tc_split_bwd": (c_int, [_P, _P, c_int64, _P, c_int64, _P, c_int64, c_int, _P, c_size_t,
                                     _P]),
    "b200rec_tc_prep_weight": (c_int, [_P, c_int, c_int, _P, c_int64, _P, c_int64, _P]),
    "b200rec_tc_linear_fwd": (c_int, [_P, c_int64, _P, c_int64, _P, c_int, _P, c_int64, _P, c_int64,
                                      c_int, c_int64, c_int, c_int, _P]),
    "b200rec_tc_cross_fwd": (c_int, [_P, c_int64, _P, c_int64, _P, _P, _P, c_int64, _P, _P, c_int64,
                                     _P, c_int64, c_int, c_int64, c_int, _P]),
    "b200rec_tc_gate_fwd": (c_int, [_P, c_int64, _P, c_int64, _P, _P, c_int64, _P, c_int64, c_int,
                                    c_int64, c_int, _P]),
    "b200rec_tc_gate_bwd": (c_int, [_P, _P, c_int64, _P, _P, c_int64, _P, c_int64, c_int, _P]),
    "b200rec_tc_linear_bwd_workspace_bytes": (c_int, [c_int64, c_int, c_int, POINTER(c_size_t)]),
    "b200rec_tc_linear_bwd_dx": (c_int, [_P, c_int64, _P, c_int64, _P, c_int64, _P, _P, c_int64, _P,
                                         c_int64, _P, c_int64, c_int, c_int, _P, c_size_t, _P]),
    "b200rec_tc_linear_bwd_dw": (c_int, [_P, c_int64, _P, c_int64, _P, c_int64, c_int, c_int, _P,
                                         c_size_t, _P]),
    "b200rec_tc_head_fwd": (c_int, [_P, c_int64, c_int, _P, _P, _P, c_int64, _P]),
    "b200rec_esmm_head_fwd": (c_int, [_P, _P, c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int64,
                                      _P]),
    "b200rec_esmm_head_bwd_workspace_bytes": (c_int, [c_int64, c_int, POINTER(c_size_t)]),
    "b200rec_esmm_head_bwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int, _P, _P, _P, _P,
                                      _P, _P, _P, _P, c_int64, _P, c_size_t, _P]),
    "b200rec_tc_head_bwd_workspace_bytes": (c_int, [c_int, POINTER(c_size_t)]),
    "b200rec_tc_head_bwd": (c_int, [_P, c_int64, c_int, _P, _P, _P, c_int64, _P, _P, c_int64, _P,
                                    c_size_t, _P]),
    "b200rec_sum_sigmoid_fwd": (c_int, [_P, _P, _P, _P, c_int64, _P]),
    "b200rec_sum_sigmoid_bwd": (c_int, [_P, _P, _P, c_int64, _P]),
    "b200rec_log_loss_workspace_bytes": (c_int, [POINTER(c_size_t)]),
    "b200rec_log_loss_mean_fwd": (c_int, [_P, _P, c_int, c_double, _P, c_int64, _P, c_size_t, _P]),
    "b200rec_log_loss_mean_bwd": (c_int, [_P, _P, c_int, c_double, _P, _P, c_int64, _P]),
    "b200rec_auc_update": (c_int, [_P, _P, c_int, _P, _P, c_int, c_int64, _P]),
    "b200rec_tc_debug": (c_int, [c_int, c_int]),
    "b200rec_tc_timeout_word": (c_int, [POINTER(ctypes.c_uint)]),
    "b200rec_dot_interact_fwd": (c_int, [_P, _P, c_int64, c_int, c_int, c_int, _P]),
    "b200rec_dot_interact_bwd": (c_int, [_P, _P, _P, c_int64, c_int, c_int, c_int, _P]),
    "b200rec_hash_keys": (c_int, [_P, _P, c_int64, c_int64, c_int, _P, _P]),
    "b200rec_shard_bucketize_workspace_bytes": (c_int, [c_int64, c_int, POINTER(c_size_t)]),
    "b200rec_shard_bucketize": (c_int, [_P, c_int64, c_int, c_int64, _P, _P, _P, _P, _P, c_size_t,
                                        _P]),
}

_lib = None


def declared_symbols():
    """Every entry point include/b200rec.h declares (parsed from the header)."""
    import re

    text = open(os.path.join(INCLUDE_DIR, "b200rec.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200rec_[a-z0-9_]+)\s*\(", text)))


def load() -> ctypes.CDLL:
    """Load the library (building it first if nvcc is available and sources are newer)."""
    global _lib
    if _lib is not None:
        return _lib
    if needs_build():
        try:
            build()
        except (B200RecError, FileNotFoundError) as e:  # no nvcc on this box
            if not os.path.exists(LIB_PATH):
                raise B200RecError(
                    "libb200rec.so is missing and could not be built (%s). The b200rec hot path "
                    "has no CPU fallback: run `python -c 'import __graft_entry__ as g; g.build()'`."
                    % e)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in _SIG.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    got = lib.b200rec_abi_version()
    if got != ABI_VERSION:
        raise B200RecError("libb200rec ABI version %d, expected %d" % (got, ABI_VERSION))
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().b200rec_last_error().decode("utf-8", "replace")
        raise B200RecError("%s failed (rc=%d): %s" % (what or "b200rec call", rc, msg))


def ptr(t):
    """Device pointer of a torch tensor (None -> NULL)."""
    if t is None:
        return None
    return c_void_p(t.data_ptr())
