"""The fused GEMM epilogues (RoPE, SwiGLU, D = bf16(D + acc), fp32 D32 += acc) store whole 16-byte blocks.

The four lanes of a quad trade their column pairs after the first bf16 rounding (or, for the fp32 forms, before any), so that each lane
finishes the element-wise work on 8 consecutive columns and loads and stores them 16 bytes at a time.
CPU: compiled for sm_90a with the build's flags (no GPU needed), no gemm_wgmma_kernel or gemm_e4m3_kernel instantiation keeps a 32-bit
global store, and none spills.
GPU: every fused form is bit for bit the unfused composition (GEMM + lmod_rope / lmod_silu_mul_fwd, or the fp32 arithmetic of the accumulating forms), written into a sentinel-filled buffer taller and wider than the output -- ragged M with a last
128-row tile of one row, a row stride wider than N, grouped rows with empty groups, device row counts -- and nothing outside the output
rectangle changes."""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "llava-mod_b200")
KERNELS = ("gemm_wgmma_kernel", "gemm_e4m3_kernel")


def _build_ext():
    spec = importlib.util.spec_from_file_location("lmod_build_ext", os.path.join(PKG, "build_ext.py"))
    be = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(be)
    if not (os.path.isfile(be.NVCC) or shutil.which(be.NVCC)):
        pytest.skip("nvcc not found at %s (set NVCC): the SASS check compiles the GEMMs for sm_90a" % be.NVCC)
    return be


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """{source: (ptxas -v output, {kernel: SASS lines})} of gemm.cu and gemm_fp8.cu built with the build's flags."""
    be = _build_ext()
    out = {}
    for src in ("gemm.cu", "gemm_fp8.cu"):
        obj = str(tmp_path_factory.mktemp("sass") / (src + ".o"))
        r = subprocess.run([be.NVCC] + be.FLAGS + ["-c", os.path.join(be.CSRC, src), "-o", obj], capture_output=True, text=True)
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
        out[src] = (r.stdout + r.stderr, {k: v for k, v in kernels.items() if any(n in k for n in KERNELS)})
    return out


def test_gemm_kernels_have_no_32_bit_global_store(compiled):
    count = {src: len(k) for src, (_, k) in compiled.items()}
    assert count == {"gemm.cu": 8, "gemm_fp8.cu": 1}, count
    bad = {}
    for _, kernels in compiled.values():
        for name, lines in kernels.items():
            stores = [m.group(0) for ln in lines for m in re.finditer(r"\bSTG\.E[\w.]*", ln)]
            narrow = sorted({s for s in stores if ".64" not in s and ".128" not in s})
            if narrow:
                bad[name] = narrow
    assert not bad, "32-bit (or narrower) global stores in: %s" % bad


def test_gemm_kernels_do_not_spill(compiled):
    seen = 0
    for src, (ptxas, _) in compiled.items():
        name = None
        for ln in ptxas.splitlines():
            m = re.search(r"Compiling entry function '(\S+)'", ln)
            if m:
                name = m.group(1)
                continue
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
            if m and name and any(n in name for n in KERNELS):
                assert (int(m.group(1)), int(m.group(2))) == (0, 0), (src, name, ln.strip())
                seen += 1
                name = None
    assert seen == 9, seen


# ---- GPU: bit for bit against the unfused composition, sentinels everywhere else -----------------------------------------------------
SENT16 = 0x7FB3                 # a bf16 NaN payload no kernel computes
SENT32 = 0x7FC0ABCD             # likewise in fp32


def _gen(seed):
    import torch
    return torch.Generator(device="cuda").manual_seed(seed)


def _rnd(gen, *shape, scale=1.0):
    import torch
    return (torch.randn(*shape, device="cuda", generator=gen) * scale).to(torch.bfloat16)


def _buf(rows, cols, fp32=False):
    """A sentinel-filled buffer 130 rows taller and 40 columns wider than [rows, cols]: the row stride is wider than the output, and rows up
    to the end of the last 128-row tile exist."""
    import torch
    if fp32:
        return torch.full((rows + 130, cols + 40), SENT32, dtype=torch.int32, device="cuda").view(torch.float32)
    return torch.full((rows + 130, cols + 40), SENT16, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def _bits(t):
    import torch
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _check(name, buf, rects):
    """rects: [(row0, row1, col0, col1, want)]: each rectangle of buf holds want bit for bit; every other element is still the sentinel."""
    import torch
    torch.cuda.synchronize()
    keep = torch.ones(buf.shape, dtype=torch.bool, device="cuda")
    for r0, r1, c0, c1, want in rects:
        got = buf[r0:r1, c0:c1]
        assert got.shape == want.shape, (name, got.shape, want.shape)
        diff = _bits(got) != _bits(want.contiguous())
        n = int(diff.sum())
        assert n == 0, f"{name}: {n} / {got.numel()} elements differ in bits; first at {tuple(int(t) for t in torch.nonzero(diff)[0])}"
        keep[r0:r1, c0:c1] = False
    sent = SENT32 if buf.dtype == torch.float32 else SENT16
    changed = int((_bits(buf)[keep] != sent).sum())
    assert changed == 0, f"{name}: {changed} elements outside the output were written"


def _offsets(sizes):
    o = [0]
    for s in sizes:
        o.append(o[-1] + s)
    return o


ROPE = [(129, 200, 4, 2, 64), (129, 200, 2, 1, 128), (300, 136, 3, 1, 64), (2561, 136, 16, 16, 64), (2561, 136, 8, 8, 128),
        (2561, 136, 12, 4, 128)]


def _rope_inputs(M, H, nh, nkv, hd, seed):
    import torch
    from llavamod.model.language_model.qwen2_core import rope_tables
    N, max_pos = (nh + 2 * nkv) * hd, 4096
    g = _gen(seed)
    x, w, b = _rnd(g, M, H), _rnd(g, N, H, scale=0.1), _rnd(g, N)
    pos = torch.randint(0, max_pos, (M,), device="cuda", generator=g)
    pos[::3] = max_pos - 1
    cos, sin = rope_tables(hd, max_pos, 1e6, torch.bfloat16, "cuda")
    return N, x, w, b, pos, cos, sin


@pytest.mark.gpu
@pytest.mark.parametrize("M,H,nh,nkv,hd", ROPE)
def test_qkv_rope_stores(M, H, nh, nkv, hd):
    """(2561, .., 16|8|12, ..) run 256-wide tiles, the others 128-wide; (3, 1, 64) ends in a partial tile with the q|k / v boundary inside it;
    (12, 4, 128) is GQA at the teacher's head size."""
    from llavamod import kernels as Kk
    N, x, w, b, pos, cos, sin = _rope_inputs(M, H, nh, nkv, hd, M + nh + hd)
    buf = _buf(M, N)
    out = buf[:M, :N]
    Kk.call("lmod_gemm_qkv_rope", Kk.ptr(x), x.stride(0), Kk.ptr(w), w.stride(0), Kk.ptr(b), Kk.ptr(out), out.stride(0), M, H, nh, nkv, hd,
            Kk.ptr(cos), Kk.ptr(sin), Kk.ptr(pos))
    import torch
    with torch.no_grad():
        want = Kk.rope_(Kk.gemm(x, w, bias=b), cos, sin, pos, nh, nkv, hd)
    _check("qkv", buf, [(0, M, 0, N, want)])


@pytest.mark.gpu
@pytest.mark.parametrize("M,I", [(1, 128), (128, 128), (129, 384), (257, 512), (2561, 256), (5000, 384)])
def test_swiglu_stores(M, I):
    import torch
    from llavamod import kernels as Kk
    H = 200
    g = _gen(M + I)
    x, w = _rnd(g, M, H), _rnd(g, 2 * I, H, scale=0.1)
    abuf = _buf(M, I)
    act = abuf[:M, :I]
    Kk.call("lmod_gemm_swiglu", Kk.ptr(x), x.stride(0), Kk.ptr(w), w.stride(0), Kk.ptr(act), act.stride(0), None, 0, M, I, H)
    with torch.no_grad():
        act_ref = Kk.silu_mul(Kk.gemm(x, w))
    _check("act", abuf, [(0, M, 0, I, act_ref)])


@pytest.mark.gpu
@pytest.mark.parametrize("sizes,I", [([128, 0, 256], 128), ([0, 384, 128, 0], 256)])
def test_grouped_swiglu_forms_store_only_their_rows(sizes, I):
    import torch
    from llavamod import kernels as Kk
    G, H = len(sizes), 200
    offs = _offsets(sizes)
    R, n = offs[-1] + 128, offs[-1]
    g = _gen(G + I + R)
    xp, w_gu = _rnd(g, R, H), _rnd(g, G, 2 * I, H, scale=0.1)
    offsets = torch.tensor(offs, dtype=torch.int32, device="cuda")
    abuf = _buf(R, I)
    act = abuf[:R, :I]
    Kk.call("lmod_grouped_gemm_swiglu", Kk.ptr(xp), xp.stride(0), Kk.ptr(w_gu), w_gu.stride(1), Kk.ptr(act), act.stride(0), None, 0,
            Kk.ptr(offsets), G, R, I, H)
    h_ref = torch.zeros(R, 2 * I, dtype=torch.bfloat16, device="cuda")
    Kk.grouped_gemm(xp, w_gu, h_ref, offsets, 0)
    with torch.no_grad():
        _check("grouped act", abuf, [(0, n, 0, I, Kk.silu_mul(h_ref[:n]))])


# (300, 8) runs a 256-wide tile of which 8 columns exist; (3073, 2056) 256-wide ones ending in a partial transpose group
ACC = [(129, 520, 136), (300, 8, 64), (3073, 2056, 64)]


def _acc_operands(M, N, K):
    g = _gen(M + N + K)
    return _rnd(g, M, K), _rnd(g, N, K, scale=0.1), _rnd(g, N), g


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", ACC)
def test_fp32_accumulate_stores(M, N, K):
    """D32 += acc (not split): from zeros it is the accumulator itself, whose bf16 rounding is the plain GEMM's output; from random values
    it is their fp32 sum with that accumulator."""
    import torch
    from llavamod import kernels as Kk
    x, w, _, g = _acc_operands(M, N, K)
    zbuf = _buf(M, N, fp32=True)
    zbuf[:M, :N] = 0.0
    Kk.gemm(x, w, out_f32=zbuf[:M, :N])
    acc = zbuf[:M, :N].clone()
    _check("D32 from zero", zbuf, [(0, M, 0, N, acc)])
    plain = Kk.gemm(x, w)
    torch.cuda.synchronize()
    assert bool((_bits(acc.to(torch.bfloat16)) == _bits(plain)).all()), "D32 accumulator rounds differently from the plain output"
    old = torch.randn(M, N, device="cuda", generator=g)
    buf = _buf(M, N, fp32=True)
    buf[:M, :N] = old
    Kk.gemm(x, w, out_f32=buf[:M, :N])
    _check("D32", buf, [(0, M, 0, N, old + acc)])


@pytest.mark.gpu
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("M,N,K", ACC)
def test_beta_stores(M, N, K, bias):
    """D = bf16(D + (acc + bias)), with acc the fp32 accumulator (D32 from zeros)."""
    import torch
    from llavamod import kernels as Kk
    x, w, b, g = _acc_operands(M, N, K)
    acc = torch.zeros(M, N, device="cuda")
    Kk.gemm(x, w, out_f32=acc)
    old = _rnd(g, M, N)
    buf = _buf(M, N)
    buf[:M, :N] = old
    Kk.gemm(x, w, bias=b if bias else None, out=buf[:M, :N], accumulate=True)
    f = acc + b.float() if bias else acc
    _check("beta", buf, [(0, M, 0, N, (f + old.float()).to(torch.bfloat16))])


@pytest.mark.gpu
@pytest.mark.parametrize("m_eff", [0, 1, 129, 300])
def test_device_row_count_stores(m_eff):
    """m_dev: the tiles holding rows below the device count store their whole 128-row tile, within M, and nothing else -- bf16 (+bias) and
    fp32 D32 += acc."""
    import torch
    from llavamod import kernels as Kk
    M, N, K = 300, 264, 136
    x, w, b, _ = _acc_operands(M, N, K)
    cnt = torch.tensor([m_eff], dtype=torch.int32, device="cuda")
    rows = min(M, -(-m_eff // 128) * 128)
    full = Kk.gemm(x, w, bias=b)
    buf = _buf(M, N)
    Kk.gemm(x, w, bias=b, out=buf[:M, :N], m_dev=cnt)
    _check("m_dev bf16", buf, [(0, rows, 0, N, full[:rows])])
    acc = torch.zeros(M, N, device="cuda")
    Kk.gemm(x, w, out_f32=acc)
    fbuf = _buf(M, N, fp32=True)
    fbuf[:M, :N] = 0.0
    Kk.gemm(x, w, out_f32=fbuf[:M, :N], m_dev=cnt)
    _check("m_dev D32", fbuf, [(0, rows, 0, N, acc[:rows]), (rows, M, 0, N, torch.zeros(M - rows, N, device="cuda"))])


# ---- e4m3: the same epilogue functions on the scaled accumulators ---------------------------------------------------------------------
def _q(t):
    from llavamod import kernels as Kk
    return Kk.quant_rows(t)


def _gemm8(a, w, bias, D):
    from llavamod import kernels as Kk
    Kk.call("lmod_gemm_e4m3", Kk.ptr(a.q), a.q.stride(0), Kk.ptr(a.scale), Kk.ptr(w.q), w.q.stride(0), Kk.ptr(w.scale),
            Kk.ptr(bias) if bias is not None else None, Kk.ptr(D), D.stride(0), a.shape[0], w.shape[0], a.shape[1])


@pytest.mark.gpu
@pytest.mark.parametrize("M,H,nh,nkv,hd", [(129, 144, 4, 2, 64), (300, 144, 3, 1, 64), (257, 144, 2, 1, 128), (2561, 144, 12, 4, 128)])
def test_e4m3_qkv_rope_stores(M, H, nh, nkv, hd):
    import torch
    from llavamod import kernels as Kk
    N, x, w, b, pos, cos, sin = _rope_inputs(M, H, nh, nkv, hd, 7 * M + nh + hd)
    a, wq = _q(x), _q(w)
    buf = _buf(M, N)
    out = buf[:M, :N]
    Kk.call("lmod_gemm_e4m3_qkv_rope", Kk.ptr(a.q), a.q.stride(0), Kk.ptr(a.scale), Kk.ptr(wq.q), wq.q.stride(0), Kk.ptr(wq.scale), Kk.ptr(b),
            Kk.ptr(out), out.stride(0), M, H, nh, nkv, hd, Kk.ptr(cos), Kk.ptr(sin), Kk.ptr(pos))
    want = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    _gemm8(a, wq, b, want)
    with torch.no_grad():
        Kk.rope_(want, cos, sin, pos, nh, nkv, hd)
    _check("e4m3 qkv", buf, [(0, M, 0, N, want)])


@pytest.mark.gpu
@pytest.mark.parametrize("M,I", [(1, 128), (129, 384), (2561, 256)])
def test_e4m3_swiglu_stores(M, I):
    import torch
    from llavamod import kernels as Kk
    H = 144
    g = _gen(M + I + 1)
    a, wq = _q(_rnd(g, M, H)), _q(_rnd(g, 2 * I, H, scale=0.1))
    buf = _buf(M, I)
    act = buf[:M, :I]
    Kk.call("lmod_gemm_e4m3_swiglu", Kk.ptr(a.q), a.q.stride(0), Kk.ptr(a.scale), Kk.ptr(wq.q), wq.q.stride(0), Kk.ptr(wq.scale), Kk.ptr(act),
            act.stride(0), M, I, H)
    h = torch.empty(M, 2 * I, dtype=torch.bfloat16, device="cuda")
    _gemm8(a, wq, None, h)
    with torch.no_grad():
        want = Kk.silu_mul(h)
    _check("e4m3 act", buf, [(0, M, 0, I, want)])


@pytest.mark.gpu
def test_cos_sin_must_be_16_byte_aligned():
    """The RoPE epilogue reads cos and sin 8 bf16 at a time: a table 4 bytes into its allocation is refused before any launch."""
    import torch
    from llavamod import _C, kernels as Kk
    M, K, hd = 8, 128, 128
    N = 3 * hd
    x, w = torch.zeros(M, K, dtype=torch.bfloat16, device="cuda"), torch.zeros(N, K, dtype=torch.bfloat16, device="cuda")
    tab = torch.zeros(64 * hd + 2, dtype=torch.bfloat16, device="cuda")
    good, off = tab[:64 * hd], tab[2:]
    pos = torch.zeros(M, dtype=torch.int64, device="cuda")
    D = torch.zeros(M, N, dtype=torch.bfloat16, device="cuda")
    for cos, sin in ((off, good), (good, off)):
        with pytest.raises(_C.LmodError, match="16-byte aligned"):
            Kk.call("lmod_gemm_qkv_rope", Kk.ptr(x), K, Kk.ptr(w), K, None, Kk.ptr(D), N, M, K, 1, 1, hd, Kk.ptr(cos), Kk.ptr(sin), Kk.ptr(pos))
    a, wq = _q(x), _q(w)
    with pytest.raises(_C.LmodError, match="16-byte aligned"):
        Kk.call("lmod_gemm_e4m3_qkv_rope", Kk.ptr(a.q), K, Kk.ptr(a.scale), Kk.ptr(wq.q), K, Kk.ptr(wq.scale), None, Kk.ptr(D), N, M, K, 1, 1, hd,
                Kk.ptr(off), Kk.ptr(good), Kk.ptr(pos))
