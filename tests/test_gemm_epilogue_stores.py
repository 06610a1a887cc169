"""The plain bf16 epilogue of the GEMM stores whole 16-byte blocks of 8 columns (the four lanes of a quad trade their column pairs first).

CPU: compiled for sm_90a with the build's flags (no GPU needed), every gemm_wgmma_kernel instantiation contains 128-bit global stores.
GPU: the blocks land where they belong -- ragged M and N, a row stride wider than N, bias, every operand layout -- and nothing outside
the output rectangle is written."""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "llava-mod_b200")


def test_gemm_kernels_store_16_byte_blocks(tmp_path):
    spec = importlib.util.spec_from_file_location("lmod_build_ext", os.path.join(PKG, "build_ext.py"))
    be = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(be)
    if not (os.path.isfile(be.NVCC) or shutil.which(be.NVCC)):
        pytest.skip("nvcc not found at %s (set NVCC): the SASS check compiles gemm.cu for sm_90a" % be.NVCC)
    obj = str(tmp_path / "gemm.o")
    r = subprocess.run([be.NVCC] + be.FLAGS + ["-c", os.path.join(be.CSRC, "gemm.cu"), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([os.path.join(os.path.dirname(be.NVCC), "cuobjdump"), "-sass", obj], capture_output=True, text=True,
                          check=True).stdout
    kernels, name = {}, None
    for ln in sass.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            name = m.group(1)
            kernels[name] = []
        elif name:
            kernels[name].append(ln)
    gemm = {k: v for k, v in kernels.items() if "gemm_wgmma_kernel" in k}
    assert len(gemm) == 8, sorted(gemm)
    without = [k for k, v in gemm.items() if not any(re.search(r"\bSTG\.E\.128\b", ln) for ln in v)]
    assert not without, "no 16-byte global store in: %s" % without


@pytest.mark.gpu
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K", [(130, 520, 192), (300, 8, 64), (1282, 1048, 320), (2048, 4096, 256)])
def test_plain_epilogue_writes_exactly_its_rectangle(M, N, K, a_mn, b_mn):
    import torch
    from llavamod import kernels as Kk
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    pad = lambda n: (n + 7) // 8 * 8          # noqa: E731  row strides must be multiples of 8
    a = torch.randn((K, pad(M)) if a_mn else (M, pad(K)), device="cuda", generator=g).to(torch.bfloat16)
    b = torch.randn((K, pad(N)) if b_mn else (N, pad(K)), device="cuda", generator=g).to(torch.bfloat16)
    a = a[:, :M] if a_mn else a[:, :K]
    b = b[:, :N] if b_mn else b[:, :K]
    bias = torch.randn(N, device="cuda", generator=g).to(torch.bfloat16)
    buf = torch.full((M + 3, N + 40), 3.0, dtype=torch.bfloat16, device="cuda")
    Kk.gemm(a, b, a_mn=a_mn, b_mn=b_mn, bias=bias, out=buf[:M, :N])
    torch.cuda.synchronize()
    A = a.float().t() if a_mn else a.float()
    B = b.float() if b_mn else b.float().t()
    ref = A @ B + bias.float()
    err = (buf[:M, :N].float() - ref).abs()
    tol = 2.0 ** -8 * ref.abs() + 2.0 ** -8 * (K ** 0.5) * 2e-2
    assert bool((err <= tol).all()), f"max err {err.max().item():.4e}, bad {(err > tol).sum().item()} / {err.numel()}"
    assert bool((buf[M:] == 3.0).all()) and bool((buf[:M, N:] == 3.0).all())
