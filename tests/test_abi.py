"""The C-ABI library loads on a CPU-only box and exports every symbol include/b2hist.h declares;
compute entry points fail loudly without a GPU (no CPU fallback)."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    from xgboost_ray_b200 import build
    return build.build()


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "b2hist.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(B2_\w+)\s*\(", text)))


def test_header_symbols_exported(built):
    lib = ctypes.CDLL(built)
    syms = declared_symbols()
    assert len(syms) >= 30
    for s in syms:
        assert hasattr(lib, s), "missing export %s" % s


def test_python_binding_covers_header(built):
    from xgboost_ray_b200 import engine
    assert sorted(engine.ABI) == declared_symbols()
    assert engine.lib().B2_GetVersion() >= 100


def test_no_cpu_fallback(built):
    from xgboost_ray_b200 import engine
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    with pytest.raises(engine.XGBoostError, match="no CUDA device|CUDA"):
        engine.DMatrix(np.zeros((4, 2), np.float32), label=np.zeros(4, np.float32))
    with pytest.raises(engine.XGBoostError):
        engine.hist_build_raw(np.zeros((4, 2), np.uint8), np.zeros(4, np.int32), np.zeros(4, np.int32))


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "xgboost_ray_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, fn)).read()
                assert "import oracle" not in src and "from oracle" not in src and "liboracle" not in src, fn


def test_python_binding_argument_types_match_header(built):
    """Every ctypes prototype in engine.ABI has the argument types the header declares (a wrong handle / pointer type
    only shows up when the call is made, which for the multi-GPU entry points means on a GPU box)."""
    from xgboost_ray_b200 import engine
    C = ctypes
    H = engine._H
    tmap = {"B2Handle": H, "B2Handle*": C.POINTER(H), "char*": C.c_char_p, "const char*": C.c_char_p,
            "const double*": C.POINTER(C.c_double), "double*": C.POINTER(C.c_double),
            "const float*": C.POINTER(C.c_float), "float*": C.POINTER(C.c_float),
            "const int32_t*": C.POINTER(C.c_int32), "int32_t*": C.POINTER(C.c_int32),
            "const uint32_t*": C.POINTER(C.c_uint32), "uint32_t*": C.POINTER(C.c_uint32),
            "const uint8_t*": C.POINTER(C.c_uint8), "uint8_t*": C.POINTER(C.c_uint8),
            "int64_t*": C.POINTER(C.c_int64), "int*": C.POINTER(C.c_int),
            "float": C.c_float, "double": C.c_double, "int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "uint64_t": C.c_uint64,
            "const B2Tree*": C.POINTER(engine.B2Tree), "B2Tree*": C.POINTER(engine.B2Tree)}
    text = open(os.path.join(ROOT, "include", "b2hist.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    checked = 0
    for m in re.finditer(r"\b(B2_\w+)\s*\(([^)]*)\)\s*;", text):
        name, args = m.groups()
        want = []
        for a in [x.strip() for x in args.split(",")]:
            if not a or a == "void":
                continue
            if a.endswith("]"):                                   # uint8_t uid[128]
                a = re.sub(r"\s*\w+\[\d+\]$", "*", a)
            elif not a.endswith("*"):
                a = re.sub(r"\s*\w+$", "", a).strip() if " " in a else a
            a = re.sub(r"\s*\*\s*\w*$", "*", a) if "*" in a else a
            want.append(tmap[a])
        got = engine.ABI[name][1]
        assert len(got) == len(want), (name, len(got), len(want))
        for i, (g, w) in enumerate(zip(got, want)):
            # pointer classes from POINTER() are cached, so identity works; c_void_p is accepted for any pointer argument
            ok = g is w or (g is C.c_void_p and issubclass(w, C._Pointer)) or (g is C.c_char_p and w in (C.POINTER(C.c_uint8),))
            assert ok, "%s argument %d: binding %s, header %s" % (name, i + 1, g, w)
        checked += 1
    assert checked == len(declared_symbols())


def test_tree_record_matches_header():
    """engine.B2Tree has the fields of the header's B2Tree, in its order, and each array's element type: ctypes lays the
    record out from this list alone, so a field out of place would hand the engine one array for another."""
    from xgboost_ray_b200 import engine
    C = ctypes
    scalar = {"int32_t": C.c_int32, "int64_t": C.c_int64}
    element = {"int32_t": np.int32, "float": np.float32, "double": np.float64, "uint8_t": np.uint8, "uint32_t": np.uint32}
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b2hist.h")).read(), flags=re.S)
    body = re.search(r"typedef struct B2Tree \{(.*?)\} B2Tree;", text, flags=re.S).group(1)
    fields = re.findall(r"(\w+)\s*(\*?)\s*(\w+);", body)
    assert len(fields) == 16
    assert [name for name, _ in engine.B2Tree._fields_] == [name for _, _, name in fields]
    for (name, got), (typ, star, _) in zip(engine.B2Tree._fields_, fields):
        if star:
            assert got is C.c_void_p and engine.B2Tree.DTYPES[name] is element[typ], name
        else:
            assert got is scalar[typ], name
