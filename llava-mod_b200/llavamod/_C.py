"""ctypes binding of liblmod_b200.so (the C ABI declared in include/lmod.h).

There is no CPU fallback: if the shared library is missing, or a call fails, an exception is raised.
PyTorch is used only for device memory and streams; every entry point receives raw ``data_ptr()``s and the
current CUDA stream handle.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblmod_b200.so")

_lib = None

c_void_p, c_int, c_int64, c_float, c_double = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_double

# name -> argtypes (all return int unless listed in _RESTYPES)
_P, _I, _L, _F, _D = c_void_p, c_int, c_int64, c_float, c_double
SIGNATURES = {
    "lmod_kl_counts": [_P, _L, _L, _I, _P, _P],
    "lmod_kl_fwd_bwd": [_P, _L, _P, _L, _P, _L, _L, _L, _I, _F, _F, _P, _P, _P, _L, _P],
    "lmod_kl_fwd_bwd_rows": [_P, _L, _P, _L, _P, _L, _L, _L, _I, _F, _F, _P, _P, _P, _L, _P, _P, _P],
    "lmod_active_rows": [_P, _L, _L, _I, _P, _P, _P],
    "lmod_gather_rows": [_P, _L, _P, _P, _L, _L, _L, _P, _L, _P],
    "lmod_scatter_rows": [_P, _L, _P, _P, _L, _L, _P, _L, _P],
    "lmod_kl_finalize": [_P, _P, _L, _L, _I, _P, _P],
    "lmod_logp_gather_fwd": [_P, _L, _P, _L, _L, _L, _P, _P, _P, _I, _P],
    "lmod_logp_gather_bwd": [_P, _L, _P, _L, _L, _L, _P, _P, _I, _P, _L, _P],
    "lmod_softmax_rows": [_P, _L, _L, _L, _I, _P, _L, _P],
    "lmod_align_loss_dense": [_P, _P, _L, _P, _L, _L, _I, _P, _P, _P],
    "lmod_moe_capacity": [_L, _I, _D, _L],
    "lmod_moe_route_ws_elems": [_L, _I],
    "lmod_moe_route_scatter": [_P, _P, _P, _L, _L, _I, _D, _L, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P],
    "lmod_moe_gather_combine": [_P, _P, _P, _P, _L, _L, _P, _P],
    "lmod_moe_combine_bwd": [_P, _P, _P, _P, _L, _L, _P, _P, _P],
    "lmod_moe_gate_bwd": [_P, _P, _P, _P, _P, _P, _L, _I, _P, _P],
    "lmod_moe_scatter_bwd": [_P, _P, _P, _P, _P, _L, _L, _I, _P, _P],
    "lmod_moe_wg_grad": [_P, _P, _L, _L, _I, _P, _P, _P],
    "lmod_rmsnorm_fwd": [_P, _P, _P, _L, _L, _F, _P, _P, _P, _P],
    "lmod_rmsnorm_bwd": [_P, _P, _P, _P, _P, _L, _L, _P, _P],
    "lmod_rmsnorm_wgrad": [_P, _P, _P, _L, _L, _P, _P, _P],
    "lmod_embed_grad": [_P, _P, _L, _L, _P, _P],
    "lmod_layernorm_fwd": [_P, _P, _P, _L, _L, _F, _P, _P],
    "lmod_rope": [_P, _L, _I, _P, _L, _I, _I, _P, _P, _P, _L, _I, _P],
    "lmod_silu_mul_fwd": [_P, _L, _L, _L, _P, _P],
    "lmod_silu_mul_bwd": [_P, _P, _L, _L, _L, _P, _P],
    "lmod_bias_act_fwd": [_P, _P, _L, _L, _I, _P, _P],
    "lmod_gelu_bwd": [_P, _P, _L, _P, _P],
    "lmod_add": [_P, _P, _L, _P, _P],
    "lmod_splice_embed": [_P, _P, _P, _P, _L, _L, _L, _P, _P],
    "lmod_splice_embed_bwd": [_P, _P, _P, _L, _L, _L, _P, _P],
    "lmod_sumsq": [_P, _I, _L, _P, _P],
    "lmod_adamw": [_P, _P, _P, _P, _I, _P, _L, _F, _F, _F, _F, _F, _L, _P, _F, _F, _P],
    "lmod_gemm_bf16": [_P, _L, _I, _P, _L, _I, _P, _L, _L, _L, _L, _P, _I, _P, _P],
    "lmod_gemm_bf16_dyn": [_P, _L, _I, _P, _L, _I, _P, _L, _L, _L, _L, _P, _I, _P, _P, _P, _P],
    "lmod_gemm_qkv_rope": [_P, _L, _P, _L, _P, _P, _L, _L, _L, _I, _I, _I, _P, _P, _P, _P],
    "lmod_gemm_swiglu": [_P, _L, _P, _L, _P, _L, _P, _L, _L, _L, _L, _P],
    "lmod_grouped_gemm_swiglu": [_P, _L, _P, _L, _P, _L, _P, _L, _P, _I, _L, _L, _L, _P],
    "lmod_gemm_silu_bwd": [_P, _L, _P, _L, _P, _L, _P, _L, _L, _L, _L, _P],
    "lmod_grouped_gemm_silu_bwd": [_P, _L, _P, _L, _P, _L, _P, _L, _P, _I, _L, _L, _L, _P],
    "lmod_grouped_gemm_bf16": [_P, _L, _P, _L, _P, _L, _P, _I, _L, _L, _L, _L, _I, _I, _P],
    "lmod_gemm_residual": [_P, _L, _P, _L, _P, _P, _L, _P, _L, _L, _L, _L, _P],
    "lmod_attn_fwd": [_P, _L, _L, _L, _I, _I, _I, _I, _F, _P, _L, _P, _P, _P, _P],
    "lmod_attn_bwd": [_P, _L, _P, _L, _P, _L, _P, _L, _L, _I, _I, _I, _I, _F, _P, _L, _P, _P, _P, _P, _P],
    "lmod_kv_append": [_P, _L, _L, _L, _I, _I, _I, _P, _P, _P, _L, _P],
    "lmod_attn_decode_ws_elems": [_L, _I, _I, _I, _L],
    "lmod_attn_decode": [_P, _L, _P, _P, _P, _L, _I, _I, _I, _L, _F, _P, _L, _P, _P, _L, _P],
    "lmod_version": [],
    "lmod_launch_count_reset": [],
}
_RESTYPES = {"lmod_last_error": ctypes.c_char_p, "lmod_launch_count": c_int64, "lmod_launch_count_reset": None,
             "lmod_moe_route_ws_elems": c_int64, "lmod_attn_decode_ws_elems": c_int64}


class LmodError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise LmodError(
                "liblmod_b200.so not found at %s -- build it with `python llava-mod_b200/build_ext.py` "
                "(there is no CPU / PyTorch fallback for the hot path)" % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        for name, args in SIGNATURES.items():
            fn = getattr(L, name)
            fn.argtypes = args
            fn.restype = _RESTYPES.get(name, c_int)
        L.lmod_last_error.argtypes = []
        L.lmod_last_error.restype = ctypes.c_char_p
        L.lmod_launch_count.argtypes = []
        L.lmod_launch_count.restype = c_int64
        _lib = L
    return _lib


def stream_ptr():
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    if t is None:
        return None
    return t.data_ptr()


def call(name, *args):
    """Invoke an entry point; append the current stream; raise on a non-zero status."""
    L = lib()
    fn = getattr(L, name)
    if len(args) + 1 != len(fn.argtypes):      # an argument ctypes has no type for would be passed as a 32-bit int (a truncated pointer)
        raise LmodError("%s takes %d arguments + stream, got %d" % (name, len(fn.argtypes) - 1, len(args)))
    rc = fn(*args, stream_ptr())
    if rc != 0:
        raise LmodError("%s failed (%d): %s" % (name, rc, L.lmod_last_error().decode()))


def launch_count():
    return int(lib().lmod_launch_count())


def launch_count_reset():
    lib().lmod_launch_count_reset()
