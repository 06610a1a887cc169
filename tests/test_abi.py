"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol include/lmod.h declares,
and the ctypes types taken from that header are the right ones (no compute calls -- there is no GPU here)."""
import ctypes
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    from llavamod import _C
    with open(os.path.join(ROOT, "include", "lmod.h")) as f:
        return sorted(_C.parse_header(f.read()))


def test_library_exports_every_declared_symbol():
    from llavamod import _C
    assert os.path.exists(_C.LIB_PATH), "build with python llava-mod_b200/build_ext.py"
    lib = ctypes.CDLL(_C.LIB_PATH)
    syms = declared_symbols()
    assert len(syms) >= 30
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, missing


def test_every_declared_symbol_is_typed_on_load():
    """lib() gives every prototype of include/lmod.h its ctypes argument and return types; none is left to ctypes' int default."""
    from llavamod import _C
    L = _C.lib()
    untyped = [s for s in declared_symbols() if getattr(L, s).argtypes is None]
    assert not untyped, untyped
    assert L.lmod_version() >= 100
    assert L.lmod_last_error() is not None


def test_header_parser():
    """The parser behind the ctypes types: multi-line prototypes, inline comments, const pointers, (void), every return type, and a
    type it does not know refused rather than guessed (ctypes would pass an untyped argument as a 32-bit int)."""
    from llavamod import _C
    P, I, L, F, D = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_double
    src = """
    #include <stdint.h>
    /* lmod_commented_out(int x); */
    typedef enum { LMOD_OK = 0, LMOD_ERR_ARG = -1 } lmod_status;
    const char* lmod_name(void);
    void lmod_reset(void);
    int64_t lmod_elems(int64_t n, int k /* heads */, double cf);
    int lmod_op(const void* x, int64_t ld /* row stride */, const int32_t *perm,
                float eps, uint8_t* codes,
                void* stream);
    float lmod_scale(float* out);
    double lmod_ratio(const char* tag, double d);
    """
    got = _C.parse_header(src)
    assert got == {
        "lmod_name": ([], ctypes.c_char_p),
        "lmod_reset": ([], None),
        "lmod_elems": ([L, I, D], L),
        "lmod_op": ([P, L, P, F, P, P], I),
        "lmod_scale": ([P], F),
        "lmod_ratio": ([ctypes.c_char_p, D], D),
    }
    for bad in ("int lmod_bad(size_t n, void* stream);", "unsigned lmod_bad(void* stream);", "int lmod_bad(long long n);"):
        with pytest.raises(_C.LmodError, match="lmod_bad"):
            _C.parse_header(bad)


def test_loaded_library_types():
    from llavamod import _C
    L = _C.lib()
    assert len(declared_symbols()) >= 60
    assert L.lmod_moe_capacity.argtypes == [ctypes.c_int64, ctypes.c_int, ctypes.c_double, ctypes.c_int64]
    assert L.lmod_moe_capacity.restype is ctypes.c_int
    assert L.lmod_attn_decode_ws_elems.restype is ctypes.c_int64
    assert L.lmod_last_error.argtypes == [] and L.lmod_last_error.restype is ctypes.c_char_p
    assert L.lmod_launch_count_reset.argtypes == [] and L.lmod_launch_count_reset.restype is None


def test_missing_header_fails_loudly(monkeypatch):
    from llavamod import _C
    monkeypatch.setattr(_C, "_lib", None)
    monkeypatch.setattr(_C, "HEADER_PATH", "/nonexistent/lmod.h")
    with pytest.raises(_C.LmodError, match="lmod.h"):
        _C.lib()


def test_missing_library_fails_loudly(monkeypatch):
    from llavamod import _C
    monkeypatch.setattr(_C, "_lib", None)
    monkeypatch.setattr(_C, "LIB_PATH", "/nonexistent/liblmod_b200.so")
    with pytest.raises(_C.LmodError):
        _C.lib()


def test_cpu_tensor_is_rejected_not_silently_computed():
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
