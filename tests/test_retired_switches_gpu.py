"""The teacher forward has one set of GEMM epilogue forms: the environment variables that used to select other ones
(LLAVAMOD_FUSE_SWIGLU, LLAVAMOD_FUSE_ROPE, LLAVAMOD_FUSE_RESIDUAL, LMOD_GEMM_NOSTORE) change neither its launches nor its bytes.

Each run is a fresh interpreter, so that the variables are read the way a user's process would read them: one decoder layer at
H 2048 (the fused SwiGLU's reduction length), I 5632, 16 heads of 128 (the fused q|k|v + RoPE), T 256, no grad."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "llava-mod_b200")
RETIRED = {"LLAVAMOD_FUSE_SWIGLU": "1", "LLAVAMOD_FUSE_ROPE": "0", "LLAVAMOD_FUSE_RESIDUAL": "1", "LMOD_GEMM_NOSTORE": "1"}
CHILD = """
import hashlib
import torch
from llavamod import _C
from tests.test_layers_cfg2_gpu import build_lm
m, _, _ = build_lm(2048, 5632, 16, seed=3)
x = torch.randn(1, 256, 2048, generator=torch.Generator().manual_seed(5)).to(torch.bfloat16).cuda()
with torch.no_grad():
    m(x)                                       # first call: allocations and module loads
    n0 = _C.launch_count()
    out, _, _ = m(x)
    n = _C.launch_count() - n0
print(n, hashlib.sha256(out.view(torch.int16).cpu().numpy().tobytes()).hexdigest())
"""


def _run(env):
    r = subprocess.run([sys.executable, "-c", f"import sys; sys.path[:0] = [{ROOT!r}, {PKG!r}]\n" + CHILD], env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    launches, digest = r.stdout.split()[-2:]
    return int(launches), digest


def test_retired_epilogue_switches_change_nothing():
    clean = {k: v for k, v in os.environ.items() if k not in RETIRED}
    want = _run(clean)
    got = _run(dict(clean, **RETIRED))
    assert got == want, f"with {RETIRED}: (launches, output SHA-256) {got}, without: {want}"
