"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol include/gorse_b200.h
declares, and fails loudly (no CPU fallback) when there is no CUDA device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "gorse_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(gorse_b200_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol(gb):
    from gorse_b200 import _lib

    syms = header_symbols()
    assert len(syms) >= 30
    raw = C.CDLL(_lib.LIB_PATH)
    for s in syms:
        assert hasattr(raw, s), f"{s} declared in include/gorse_b200.h but not exported"
    assert set(syms) == set(_lib.PROTOTYPES), set(syms) ^ set(_lib.PROTOTYPES)
    assert _lib.lib.gorse_b200_version() == 1


def test_only_sm90a_code_in_library(gb):
    import shutil
    import subprocess

    from gorse_b200 import _lib

    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not on PATH")
    out = subprocess.run(["cuobjdump", "-lelf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_product_never_touches_the_oracle():
    # the oracle is test infrastructure: nothing under gorse_b200/ may import, link or dlopen it
    bad = []
    for dp, _, files in os.walk(os.path.join(ROOT, "gorse_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h", ".hpp", "Makefile")):
                txt = open(os.path.join(dp, f), errors="replace").read()
                if re.search(r"import oracle|from oracle|gbo_|libgorse_oracle|oracle/", txt):
                    bad.append(os.path.join(dp, f))
    assert not bad, bad


def test_no_cpu_fallback_without_a_device(gb):
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the loud-failure path is exercised on the CPU box")
    with pytest.raises(gb.GorseB200Error) as ei:
        gb.Context(0)
    assert ei.value.status == -2  # GORSE_B200_ERR_CUDA
    assert ei.value.message


def test_argument_errors_do_not_need_a_device(gb):
    from gorse_b200 import _lib

    h = C.c_void_p()
    assert _lib.lib.gorse_b200_cf_create(None, 1, 1, 8, None, None, None, None, C.byref(h)) == _lib.ERR_ARG
    assert b"NULL" in _lib.lib.gorse_b200_last_error()
    assert _lib.lib.gorse_b200_index_create(None, 8, 1, C.byref(h)) == _lib.ERR_ARG
    assert _lib.lib.gorse_b200_ctx_sync(None) == _lib.ERR_ARG
    # the similarity host functions and the sparse index validate before they touch anything
    n = C.c_int32(0)
    assert _lib.lib.gorse_b200_similar_scores(7, 1.0, 0, 1, None, None, 0, None, None, C.byref(n)) == _lib.ERR_ARG
    assert b"metric" in _lib.lib.gorse_b200_last_error()
    assert _lib.lib.gorse_b200_index_query_similar(None, 0, 1, 5, 1.0, None, None, None) == _lib.ERR_ARG
    assert _lib.lib.gorse_b200_bf16_truncate(None, 4, None) == _lib.ERR_ARG
    assert _lib.lib.gorse_b200_sparse_index_create(None, C.byref(h)) == _lib.ERR_ARG
    assert _lib.lib.gorse_b200_sparse_index_add(None, None, None, None, 0, None) == _lib.ERR_ARG
    assert _lib.lib.gorse_b200_sparse_index_search_range(None, 0, 1, 5, None, None, None) == _lib.ERR_ARG
    assert _lib.lib.gorse_b200_als_epoch(None, 0.06, 0.001) == _lib.ERR_ARG


def test_synth_shapes(gb):
    from gorse_b200 import synth

    off, items = synth.make_feedback(500, 200, 5000, seed=1)
    assert off[0] == 0 and off[-1] == items.size and np.all(np.diff(off) >= 1)
    for u in range(0, 500, 37):
        row = items[off[u]:off[u + 1]]
        assert np.all(np.diff(row) > 0) and row.min() >= 0 and row.max() < 200
    (tro, tri), (teo, tei) = synth.leave_one_out(off, items, seed=2)
    assert tro[-1] + teo[-1] == off[-1] and teo[-1] == 500
    no, ni = synth.sample_negatives(200, (tro, tri), (teo, tei), 20, seed=3)
    assert no[-1] == 500 * 20
    t = synth.conflict_free_triples(off, items, 200, 40, seed=4)
    assert len(set(t[:, 0])) == len(t) and len(set(t[:, 1]) | set(t[:, 2])) == 2 * len(t)


def test_go_shim_only_calls_declared_entry_points():
    """The cgo shim cannot be compiled here (no Go toolchain); at least every C.gorse_b200_* / C.GORSE_B200_* it names must be
    declared in include/gorse_b200.h."""
    header = open(os.path.join(ROOT, "include", "gorse_b200.h")).read()
    declared = set(re.findall(r"\b(gorse_b200_[a-z0-9_]+)\s*\(", header)) | set(re.findall(r"\b(GORSE_B200_[A-Z0-9_]+)\b", header))
    declared |= set(re.findall(r"typedef struct (gorse_b200_[a-z0-9_]+)", header)) | set(re.findall(r"}\s*(gorse_b200_[a-z0-9_]+);", header))
    used = set()
    for dp, _, files in os.walk(os.path.join(ROOT, "go")):
        for f in files:
            if f.endswith(".go"):
                txt = open(os.path.join(dp, f)).read()
                used |= set(re.findall(r"\bC\.((?:gorse_b200|GORSE_B200)_[A-Za-z0-9_]+)", txt))
                declared |= set(re.findall(r"static\s+[\w\s\*]+?\b(gorse_b200_[a-z0-9_]+)\s*\(", txt))   # helpers of the cgo preamble
    assert used, "no cgo calls found under go/"
    missing = sorted(u for u in used if u not in declared)
    assert not missing, missing


def test_go_shim_memory_rules():
    """Lint by inspection (the shim cannot be compiled here).  (1) No C allocation may be turned into a Go slice
    (unsafe.Slice / (*[n]T)(ptr)[:]) in a file that also frees it from a finalizer: round 1 stored rows of a cudaHostAlloc
    buffer in the model while a finalizer could free it.  (2) A cgo.Handle travels as unsafe.Pointer(&h), never
    unsafe.Pointer(h) (go vet / cgocheck).  (3) C functions are called directly, not through Go function values.
    (4) every method of a finalizer-owning type keeps the receiver alive across its C calls."""
    for dp, _, files in os.walk(os.path.join(ROOT, "go")):
        for f in files:
            if not f.endswith(".go"):
                continue
            txt = open(os.path.join(dp, f)).read()
            code = re.sub(r"//[^\n]*", "", txt)
            if "SetFinalizer" in code:
                assert "unsafe.Slice(" not in code and not re.search(r"\(\*\[[^\]]*\][^)]*\)\(", code), f"{f}: C memory escapes as a slice next to a finalizer"
                recv = re.search(r"SetFinalizer\((\w+), func\(\w+ \*(\w+)\)", code)
                assert recv, f
                for m in re.finditer(r"func \((\w+) \*%s\) (\w+)\([^\n]*\{\n([^\n]*)" % recv.group(2), code):
                    assert "runtime.KeepAlive(%s)" % m.group(1) in m.group(3), f"{f}: method {m.group(2)} does not keep the receiver alive"
            assert not re.search(r"unsafe\.Pointer\(h\)", code), f"{f}: cgo.Handle passed by value as a pointer"
            assert not re.search(r":?=\s*C\.gorse_b200_\w+\s*$", code, flags=re.M), f"{f}: C function used as a Go value"


def test_public_header_is_plain_c(tmp_path):
    """The boundary is a C ABI: the header must compile as C99 (what cgo feeds it to) and as C++11, warnings as errors."""
    import shutil
    import subprocess

    src = tmp_path / "hdr.c"
    src.write_text('#include "gorse_b200.h"\nint main(void) { return 0; }\n')
    inc = os.path.join(ROOT, "include")
    for cc, args in (("gcc", ["-std=c99", "-pedantic"]), ("g++", ["-std=c++11", "-x", "c++"])):
        if shutil.which(cc) is None:
            pytest.skip(f"{cc} not found")
        r = subprocess.run([cc, *args, "-Wall", "-Wextra", "-Werror", "-I", inc, "-fsyntax-only", str(src)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
