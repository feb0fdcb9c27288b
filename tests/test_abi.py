"""The drop-in boundary: libb200rec.so builds for sm_90a, loads, and exports every symbol that
include/b200rec.h declares.  No compute calls (runs without a GPU)."""
import ctypes
import os
import subprocess

import pytest

from paddlerec_b200 import _lib


def test_build_and_load():
    path = _lib.build()
    assert os.path.exists(path)
    lib = _lib.load()
    assert lib.b200rec_abi_version() == _lib.ABI_VERSION


def test_every_declared_symbol_is_exported_and_bound():
    lib = ctypes.CDLL(_lib.LIB_PATH)
    declared = _lib.declared_symbols()
    assert len(declared) >= 19
    for name in declared:
        assert hasattr(lib, name), "missing export: " + name
        assert name in _lib._SIG, "no ctypes signature for " + name
    assert set(_lib._SIG) == set(declared)


def test_binary_targets_sm_90a_only():
    out = subprocess.run(["cuobjdump", "-lelf", _lib.LIB_PATH], capture_output=True, text=True)
    if out.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    assert "sm_90a" in out.stdout
    assert "sm_100" not in out.stdout and "sm_80" not in out.stdout


def test_no_cpu_fallback_on_cpu_tensors():
    import torch

    from paddlerec_b200 import ops
    with pytest.raises(_lib.B200RecError):
        ops.raw_gather(torch.zeros(4, 4), torch.zeros(3, dtype=torch.int64), -1)


def test_argument_errors_are_reported_not_thrown():
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    rc = lib.b200rec_group_ids_workspace_bytes(-5, 100, ctypes.byref(n))
    assert rc == -1 and b"n=" in lib.b200rec_last_error()
    rc = lib.b200rec_gather(None, 16, None, None, 10, 16, 100, -1, None)
    assert rc == -1 and b"NULL" in lib.b200rec_last_error()


def test_product_never_imports_oracle():
    root = os.path.join(_lib.REPO_ROOT, "paddlerec_b200")
    for dp, _, files in os.walk(root):
        for f in files:
            if f.endswith(".py"):
                text = open(os.path.join(dp, f)).read()
                assert "import oracle" not in text and "from oracle" not in text, f


def test_every_entry_point_has_a_torch_wrapper():
    """Guards the binding layer: every C entry point must be called from paddlerec_b200/ops.py (a
    refactor once dropped the DIN/CVM wrappers silently — only the GPU tests noticed)."""
    from paddlerec_b200 import ops
    src = open(os.path.join(_lib.REPO_ROOT, "paddlerec_b200", "ops.py")).read()
    for name in _lib.declared_symbols():
        if name in ("b200rec_abi_version", "b200rec_last_error"):
            continue
        assert "lib." + name + "(" in src, "no wrapper calls " + name
    for attr in ("embed_fm", "gather", "gather_pool_sum", "cross_v2", "cross_combine", "split_mm",
                 "din_attention", "continuous_value_model", "raw_shard_bucketize", "SelectedRows",
                 "raw_sparse_adam", "raw_sparse_sgd", "raw_sparse_adagrad", "raw_tower_split"):
        assert hasattr(ops, attr), attr


def _prototypes(header):
    """{name: [category per parameter]} parsed from a C header; category in ptr / i64 / i32 / f64 / f32."""
    import re

    text = open(os.path.join(_lib.INCLUDE_DIR, header)).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"//[^\n]*", "", text)
    protos = {}
    for m in re.finditer(r"\b(?:int|uint64_t|uint32_t|const char\s*\*)\s+(b200rec_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;",
                         text, flags=re.S):
        name, args = m.group(1), m.group(2).strip()
        cats = []
        if args and args != "void":
            for a in args.split(","):
                a = " ".join(a.split())
                if "*" in a:
                    cats.append("ptr")
                elif re.search(r"\b(int64_t|uint64_t|size_t)\b", a):
                    cats.append("i64")
                elif re.search(r"\bdouble\b", a):
                    cats.append("f64")
                elif re.search(r"\bfloat\b", a):
                    cats.append("f32")
                elif re.search(r"\b(int|uint32_t|int32_t)\b", a):
                    cats.append("i32")
                else:
                    raise AssertionError("unparsed parameter %r of %s" % (a, name))
        protos[name] = cats
    return protos


def _ctype_category(t):
    if t in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(t, ctypes._Pointer):
        return "ptr"
    return {ctypes.c_int64: "i64", ctypes.c_size_t: "i64", ctypes.c_uint64: "i64", ctypes.c_int: "i32",
            ctypes.c_uint32: "i32", ctypes.c_double: "f64", ctypes.c_float: "f32"}[t]


@pytest.mark.parametrize("header,module", [("b200rec.h", "_lib"), ("b200rec_io.h", "dataio")])
def test_ctypes_signatures_match_the_header_prototypes(header, module):
    """Arity and the width/kind of every parameter of every bound function — a wrong ctypes
    signature corrupts arguments silently (an int64 passed as int loses its upper half)."""
    import importlib

    mod = importlib.import_module("paddlerec_b200." + module)
    protos = _prototypes(header)
    assert set(protos) == set(mod._SIG)
    for name, (_res, argtypes) in mod._SIG.items():
        got = [_ctype_category(t) for t in argtypes]
        assert got == protos[name], "%s: header %s, ctypes %s" % (name, protos[name], got)
