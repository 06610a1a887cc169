"""The e4m3 GEMM (csrc/gemm_fp8.cu) keeps its tensor-core MMAs asynchronous, as tests/test_wgmma_pipeline.py checks for the bf16 kernels.

Compiled for sm_90a with the build's flags (no GPU needed): ptxas reports no spills and none of the messages that mean it serialized the
wgmma pipeline, and in the machine code the four QGMMA of a k-block are chained -- only the last one carries the gsb0 scoreboard that is
waited on.  The plain epilogue stores 16-byte blocks."""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "llava-mod_b200")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """(ptxas output, {kernel name: [SASS lines]}) of gemm_fp8.cu"""
    spec = importlib.util.spec_from_file_location("lmod_build_ext", os.path.join(PKG, "build_ext.py"))
    be = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(be)
    if not (os.path.isfile(be.NVCC) or shutil.which(be.NVCC)):
        pytest.skip("nvcc not found at %s (set NVCC): the check compiles gemm_fp8.cu for sm_90a" % be.NVCC)
    obj = str(tmp_path_factory.mktemp("fp8") / "gemm_fp8.o")
    r = subprocess.run([be.NVCC] + be.FLAGS + ["-c", os.path.join(be.CSRC, "gemm_fp8.cu"), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([os.path.join(os.path.dirname(be.NVCC), "cuobjdump"), "-sass", obj], capture_output=True, text=True, check=True).stdout
    kernels, name = {}, None
    for ln in sass.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            name = m.group(1)
            kernels[name] = []
        elif name:
            kernels[name].append(ln)
    return be, r.stdout + r.stderr, {k: v for k, v in kernels.items() if "gemm_e4m3_kernel" in k}


def test_ptxas_reports_no_spills_and_no_serialized_wgmma(compiled):
    be, log, kernels = compiled
    assert len(kernels) == 1, sorted(kernels)                   # one tile shape: 128 x 128
    assert "gemm_fp8.cu" in be.sources()                        # so the build fails on C7510 / C7517 in this file too
    assert not be.wgmma_serialization_messages(log), "\n".join(be.wgmma_serialization_messages(log))
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) >= 1 and all(s == ("0", "0") for s in spills), spills


def test_qgmma_are_chained_within_a_k_block(compiled):
    _, _, kernels = compiled
    for name, lines in kernels.items():
        mma = [ln for ln in lines if "QGMMA" in ln]
        assert mma and all("E4M3.E4M3" in ln for ln in mma), name
        assert len(mma) % 4 == 0, (name, len(mma))              # four m64nNk32 per 128-element k-block
        for i in range(0, len(mma), 4):
            assert ["gsb0" in ln for ln in mma[i:i + 4]] == [False, False, False, True], (name, mma[i:i + 4])
        assert not any("HGMMA" in ln for ln in lines), name


def test_plain_epilogue_stores_16_byte_blocks(compiled):
    _, _, kernels = compiled
    without = [k for k, v in kernels.items() if not any(re.search(r"\bSTG\.E\.128\b", ln) for ln in v)]
    assert not without, without
