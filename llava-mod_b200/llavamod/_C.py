"""ctypes binding of liblmod_b200.so (the C ABI declared in include/lmod.h).

There is no CPU fallback: if the shared library is missing, or a call fails, an exception is raised.
PyTorch is used only for device memory and streams; every entry point receives raw ``data_ptr()``s and the
current CUDA stream handle.
"""
import ctypes
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblmod_b200.so")
HEADER_PATH = os.path.normpath(os.path.join(_HERE, "..", "..", "include", "lmod.h"))

_lib = None

# The C types the ABI uses; any pointer other than const char* is passed as void*.
_CTYPES = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "float": ctypes.c_float, "double": ctypes.c_double, "void": None,
           "const char*": ctypes.c_char_p}


class LmodError(RuntimeError):
    pass


def _ctype(decl, proto):
    t = re.sub(r"\s*\*\s*", "*", " ".join(decl.split()))
    if t in _CTYPES:
        return _CTYPES[t]
    if t.endswith("*"):
        return ctypes.c_void_p
    raise LmodError("%s: C type %r has no ctypes mapping (int, int64_t, float, double, void, pointers)" % (proto, t))


def parse_header(src):
    """{name: (argtypes, restype)} of every lmod_* prototype in the C header text src.  Any type other than int, int64_t, float, double,
    void, const char* and pointers raises LmodError: an argument ctypes had no type for would be passed as a 32-bit int."""
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    src = re.sub(r"^\s*#.*$", "", src, flags=re.M)
    protos = {}
    for stmt in re.split(r"[;{}]", src):
        m = re.fullmatch(r"(.*?)\b(lmod_\w+)\s*\((.*)\)", stmt.strip(), flags=re.S)
        if m is None:
            continue
        ret, name, params = m.group(1), m.group(2), m.group(3).strip()
        args = []
        if params != "void":
            for p in filter(None, (p.strip() for p in params.split(","))):
                typ = re.fullmatch(r"(.*[\s*])\w+", p, flags=re.S)          # drop the parameter name
                args.append(_ctype(typ.group(1) if typ else p, name))
        protos[name] = (args, _ctype(ret, name))
    return protos


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise LmodError(
                "liblmod_b200.so not found at %s -- build it with `python llava-mod_b200/build_ext.py` "
                "(there is no CPU / PyTorch fallback for the hot path)" % LIB_PATH)
        try:
            with open(HEADER_PATH) as f:
                protos = parse_header(f.read())
        except OSError as e:
            raise LmodError("cannot read the C ABI header the ctypes types come from: %s" % e) from e
        L = ctypes.CDLL(LIB_PATH)
        for name, (args, res) in protos.items():
            fn = getattr(L, name)
            fn.argtypes, fn.restype = args, res
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
