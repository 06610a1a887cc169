"""The wgmma kernels (GEMM, flash-attention forward and backward) keep their tensor-core MMAs asynchronous.

ptxas silently serializes every wgmma.mma_async of a kernel -- each MMA waited on before the next one issues -- when the kernel contains a
function call (a device printf is one) or reads accumulator registers on a path without a wgmma.wait_group.  It says so only in a
warning.  These tests compile the three sources for sm_90a with the build's flags (no GPU needed) and check both the warnings and the
machine code: within a k-block the MMAs are chained, so only the last one of a group carries the gsb0 scoreboard that is waited on."""
import importlib.util
import os
import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "llava-mod_b200")
SOURCES = ("gemm.cu", "attn.cu", "attn_bwd.cu")


def _build_ext():
    spec = importlib.util.spec_from_file_location("lmod_build_ext", os.path.join(PKG, "build_ext.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """{source: (ptxas output, {kernel name: [SASS lines]})}"""
    be = _build_ext()
    if not (os.path.isfile(be.NVCC) or shutil.which(be.NVCC)):
        pytest.skip("nvcc not found at %s (set NVCC): the wgmma pipeline checks compile the kernels for sm_90a" % be.NVCC)
    cuobjdump = os.path.join(os.path.dirname(be.NVCC), "cuobjdump")
    out = tmp_path_factory.mktemp("wgmma")

    def one(src):
        obj = str(out / (src[:-3] + ".o"))
        r = subprocess.run([be.NVCC] + be.FLAGS + ["-c", os.path.join(be.CSRC, src), "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
        kernels, name = {}, None
        for ln in sass.splitlines():
            m = re.search(r"Function : (\S+)", ln)
            if m:
                name = m.group(1)
                kernels[name] = []
            elif name:
                kernels[name].append(ln)
        return r.stdout + r.stderr, kernels

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        return dict(zip(SOURCES, ex.map(one, SOURCES)))


def test_build_flags_show_ptxas_diagnostics():
    be = _build_ext()
    assert "-v" in be.FLAGS[be.FLAGS.index("-Xptxas") + 1:]
    assert be.wgmma_serialization_messages("ptxas warning : (C7510) Potential Performance Loss: wgmma.mma_async instructions are serialized")
    assert not be.wgmma_serialization_messages("ptxas info    : Used 168 registers, used 1 barriers")


@pytest.mark.parametrize("src", SOURCES)
def test_ptxas_does_not_serialize_wgmma(compiled, src):
    be = _build_ext()
    log, kernels = compiled[src]
    assert "ptxas info" in log, "no ptxas report in the compiler output: -Xptxas -v is missing from the build flags"
    assert not be.wgmma_serialization_messages(log), "\n".join(be.wgmma_serialization_messages(log))
    assert any("HGMMA" in ln for k in kernels.values() for ln in k), "no wgmma in %s" % src


@pytest.mark.parametrize("src", SOURCES)
def test_mmas_are_chained_in_sass(compiled, src):
    """Every kernel with wgmma has MMAs that do not carry gsb0, i.e. that issue behind another MMA without a drain in between."""
    _, kernels = compiled[src]
    with_mma = {k: [ln for ln in v if "HGMMA" in ln] for k, v in kernels.items()}
    with_mma = {k: v for k, v in with_mma.items() if v}
    if src == "gemm.cu":
        assert len([k for k in with_mma if "gemm_wgmma_kernel" in k]) == 8, sorted(with_mma)
    serialized = [k for k, v in with_mma.items() if all("gsb0" in ln for ln in v)]
    assert not serialized, "every HGMMA carries gsb0 (waited on one by one) in: %s" % serialized
