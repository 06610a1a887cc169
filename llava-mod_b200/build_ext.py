"""Builds liblmod_b200.so (all CUDA kernels + the C ABI) for sm_90a (H100) with nvcc, in-tree.

    python llava-mod_b200/build_ext.py [--force]

Output: llava-mod_b200/llavamod/liblmod_b200.so  (git-ignored build product).
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "llavamod", "liblmod_b200.so")
OBJ = os.path.join(HERE, "build")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-diag-suppress", "177", "-Xptxas", "-v"]
# ptxas messages that mean it serialized the wgmma pipeline of a kernel (every MMA waited on before the next issues): a function call
# in the kernel (C7510) or accumulator registers read on a path without a wgmma.wait_group (C7517).  A build that has one fails.
WGMMA_SERIALIZED = ("C7510", "C7517", "wgmma.mma_async instructions are serialized", "warpgroup.wait is injected")


def wgmma_serialization_messages(ptxas_output):
    return [ln for ln in ptxas_output.splitlines() if any(m in ln for m in WGMMA_SERIALIZED)]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest():
    h = hashlib.sha256()
    for f in sorted(os.listdir(CSRC)) + ["../../include/lmod.h"]:
        p = os.path.join(CSRC, f)
        if os.path.isfile(p):
            h.update(open(p, "rb").read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    stamp = os.path.join(OBJ, "stamp")
    dig = _digest()
    if not force and os.path.exists(OUT) and os.path.exists(stamp) and open(stamp).read() == dig:
        return OUT

    def cc(f):
        o = os.path.join(OBJ, f[:-3] + ".o")
        cmd = [NVCC] + FLAGS + ["-c", os.path.join(CSRC, f), "-o", o]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (f, r.stdout, r.stderr))
        bad = wgmma_serialization_messages(r.stdout + r.stderr)
        if bad:
            os.remove(o)
            raise RuntimeError("ptxas serialized the wgmma pipeline in %s (keep calls such as printf out of wgmma kernels, and wait on "
                               "every path before reading an accumulator):\n%s" % (f, "\n".join(bad)))
        if verbose:
            sys.stderr.write(r.stderr)
        return o

    with ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(cc, sources()))
    cmd = [NVCC, "-shared", "-o", OUT] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    open(stamp, "w").write(dig)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
