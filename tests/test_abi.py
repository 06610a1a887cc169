"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol include/lmod.h declares,
and the ctypes table covers them (no compute calls -- there is no GPU here)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "lmod.h")).read()
    src = re.sub(r"/\*LMOD_PLANNED_BEGIN.*?LMOD_PLANNED_END\*/", "", src, flags=re.S)   # planned, not yet exported
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(lmod_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from llavamod import _C
    assert os.path.exists(_C.LIB_PATH), "build with python llava-mod_b200/build_ext.py"
    lib = ctypes.CDLL(_C.LIB_PATH)
    syms = declared_symbols()
    assert len(syms) >= 30
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, missing


def test_ctypes_table_matches_header():
    from llavamod import _C
    syms = set(declared_symbols())
    table = set(_C.SIGNATURES) | {"lmod_last_error", "lmod_launch_count"}
    assert syms <= table, sorted(syms - table)
    assert _C.lib().lmod_version() >= 100
    assert _C.lib().lmod_last_error() is not None


def test_ctypes_signatures_have_the_arity_of_the_header_prototypes():
    """An argument ctypes has no declared type for is passed as a 32-bit int -- a truncated pointer (e.g. the stream) that crashes on the GPU
    box only.  Every ctypes signature must list exactly as many parameters as the prototype in include/lmod.h."""
    from llavamod import _C
    src = open(os.path.join(ROOT, "include", "lmod.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    seen = 0
    for m in re.finditer(r"\b(?:int|int64_t|const char\*|void)\s+(lmod_\w+)\s*\(([^;]*?)\)\s*;", src, flags=re.S):
        name, params = m.group(1), m.group(2).strip()
        if name not in _C.SIGNATURES:
            continue
        n = 0 if params in ("", "void") else params.count(",") + 1
        assert len(_C.SIGNATURES[name]) == n, (name, len(_C.SIGNATURES[name]), n)
        seen += 1
    assert seen >= 40


def test_missing_library_fails_loudly(monkeypatch):
    from llavamod import _C
    monkeypatch.setattr(_C, "_lib", None)
    monkeypatch.setattr(_C, "LIB_PATH", "/nonexistent/liblmod_b200.so")
    import pytest
    with pytest.raises(_C.LmodError):
        _C.lib()


def test_cpu_tensor_is_rejected_not_silently_computed():
    import pytest
    import torch
    from llavamod import _C, kernels as K
    with pytest.raises(_C.LmodError):
        K.kl_fused(torch.zeros(4, 8, dtype=torch.bfloat16), torch.zeros(4, 8, dtype=torch.bfloat16), torch.zeros(4, dtype=torch.int64), 4, 8, 1.0, 1.0)


def test_fused_swiglu_refuses_h1():
    """lmod_gemm_swiglu / lmod_grouped_gemm_swiglu are forward-only: a non-NULL h1 (the retired pre-activation output) is refused before
    any operand is read or anything is launched."""
    from llavamod import _C
    L = _C.lib()
    p = 1 << 20                                # never dereferenced: the call must return before
    assert L.lmod_gemm_swiglu(p, 64, p, 64, p, 128, p, 256, 128, 128, 64, None) == -1
    assert b"h1" in L.lmod_last_error()
    assert L.lmod_grouped_gemm_swiglu(p, 64, p, 64, p, 128, p, 256, p, 1, 128, 128, 64, None) == -1
    assert b"h1" in L.lmod_last_error()
