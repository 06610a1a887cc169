"""Norm, rotary, activation, splice, embedding-gradient and optimizer kernels (csrc/elementwise.cu, csrc/optim.cu) element by element
against the float64 references of tests/helpers.py, at the shapes the models run, on both sides of every dispatch boundary and on the
edges where such kernels go wrong (tails, strides, saturation, duplicates, multi-block reductions).  Every stage is checked from the
kernel's own previous stage (y from the kernel's rstd), so the copies and the stages with the reference's roundings are compared by bits."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import restated as R  # noqa: E402
from tests.helpers import (FP32_U, accumulate_tol, adamw_reference_fp64, bias_act_reference_fp64, check_bound,  # noqa: E402
                           embed_grad_reference_fp64, gelu_bwd_reference_fp64, layernorm_reference_fp64, rmsnorm_bwd_reference_fp64,
                           rmsnorm_reference_fp64, rmsnorm_wgrad_reference_fp64, rope_bwd_reference_fp64, silu_mul_reference_fp64,
                           splice_bwd_reference, splice_reference, sumsq_blocks, sumsq_chain, sumsq_reference_fp64)

bf16 = torch.bfloat16
DEV = "cuda"


def K():
    from llavamod import kernels
    return kernels


def randn(*shape, seed, scale=1.0, dtype=bf16):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(dtype)


def n_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------------
# RMSNorm: register kernels VPT = 1, 2, 4, 8 (H <= 1024, 2048, 4096, 8192) and the streaming kernel above
# ---------------------------------------------------------------------------------------------------------------------
RMS_H = [8, 64, 896, 1024, 1032, 1536, 2048, 2056, 3584, 4096, 4104, 8192, 8200, 16384]


def rms_inputs(rows, H, seed):
    x = randn(rows, H, seed=seed)
    if rows >= 3:
        x[0] = 0                                                  # rstd = eps^-1/2
        x[1] *= 1000
        x[2] *= 1e-3
    res = randn(rows, H, seed=seed + 1)
    if rows >= 3:
        res[0] = 0
    w = (1 + 0.1 * randn(H, seed=seed + 2).float()).to(bf16)
    return x, res, w


@pytest.mark.parametrize("H", RMS_H)
def test_rmsnorm_fwd_bwd_element_wise(H):
    k, eps = K(), 1e-6
    for rows in (1, 37, 2049):
        x, res, w = rms_inputs(rows, H, seed=H + rows)
        dy, dres = randn(rows, H, seed=H + rows + 7), randn(rows, H, seed=H + rows + 8)
        for with_res in (True, False):
            y = torch.empty_like(x)
            s = torch.empty_like(x) if with_res else x
            rstd = torch.empty(rows, dtype=torch.float32, device=DEV)
            k.call("lmod_rmsnorm_fwd", k.ptr(x), k.ptr(res) if with_res else None, k.ptr(w), rows, H, eps, k.ptr(y),
                   k.ptr(s) if with_res else None, k.ptr(rstd))
            ref = rmsnorm_reference_fp64(x, w, eps, res=res if with_res else None, rstd_k=rstd)
            tag = f"H={H} rows={rows} res={with_res}"
            check_bound(f"s {tag}", s, ref["s"])
            check_bound(f"rstd {tag}", rstd, ref["rstd"], ref["rstd_tol"])
            check_bound(f"y {tag}", y, ref["y"])
            # x_out / rstd NULL: the same y
            y2 = torch.empty_like(x)
            k.call("lmod_rmsnorm_fwd", k.ptr(x), k.ptr(res) if with_res else None, k.ptr(w), rows, H, eps, k.ptr(y2), None, None)
            assert torch.equal(y2, y), tag
            # backward from the kernel's s and rstd, with and without the residual stream's gradient
            for dr in ((dres, None) if with_res else (None,)):
                dx = torch.empty_like(x)
                k.call("lmod_rmsnorm_bwd", k.ptr(dy), k.ptr(s), k.ptr(w), k.ptr(rstd), k.ptr(dr), rows, H, k.ptr(dx))
                b = rmsnorm_bwd_reference_fp64(dy, s, w, rstd, dr)
                check_bound(f"dx {tag} dres={dr is not None}", dx, b["dx"], b["tol"])


@pytest.mark.parametrize("H", [8, 264, 896, 3584])
def test_rmsnorm_wgrad_element_wise(H):
    k = K()
    ws = torch.zeros(H + 64, dtype=torch.float32, device=DEV)
    for rows in (1, 7, 255, 256, 257, 4099, 16384):
        s, dy = randn(rows, H, seed=rows + H), randn(rows, H, seed=rows + H + 1)
        rstd = torch.rsqrt(s.float().pow(2).mean(-1) + 1e-6) * (1 + 0.01 * randn(rows, seed=rows, dtype=torch.float32))
        old = randn(H, seed=H, scale=0.5)
        wg = old.clone()
        k.call("lmod_rmsnorm_wgrad", k.ptr(dy), k.ptr(s), k.ptr(rstd), rows, H, k.ptr(ws), k.ptr(wg))
        ref = rmsnorm_wgrad_reference_fp64(dy, s, rstd, old)
        check_bound(f"wgrad H={H} rows={rows}", wg, ref["want"], ref["tol"])
        assert int(ws.ne(0).sum()) == 0, "the workspace is handed back zeroed"
        first = wg.clone()
        k.call("lmod_rmsnorm_wgrad", k.ptr(dy), k.ptr(s), k.ptr(rstd), rows, H, k.ptr(ws), k.ptr(wg))   # a second call adds again
        ref2 = rmsnorm_wgrad_reference_fp64(dy, s, rstd, first)
        check_bound(f"wgrad twice H={H} rows={rows}", wg, ref2["want"], ref2["tol"])
        assert int(ws.ne(0).sum()) == 0


# ---------------------------------------------------------------------------------------------------------------------
# LayerNorm (CLIP-L/336: 577 tokens per image)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [64, 1024])
def test_layernorm_element_wise(H):
    rows = 577 * 3
    x = randn(rows, H, seed=H)
    x[0] = (100 + randn(H, seed=1, scale=0.01, dtype=torch.float32)).to(bf16)      # large mean, spread below the bf16 spacing
    x[1] = (100 + randn(H, seed=2, scale=2.0, dtype=torch.float32)).to(bf16)       # large mean, small spread
    x[2] = (-300 + randn(H, seed=3, scale=0.5, dtype=torch.float32)).to(bf16)
    x[3] = 0
    w, b = randn(H, seed=4), randn(H, seed=5)
    y = K().layernorm(x, w, b, 1e-5)
    ref = layernorm_reference_fp64(x, w, b, 1e-5)
    check_bound(f"layernorm H={H}", y, ref["y"], ref["tol"])


# ---------------------------------------------------------------------------------------------------------------------
# RoPE: forward bit exact against the oracle, backward against the float64 transpose rotation
# ---------------------------------------------------------------------------------------------------------------------
def rope_buffers(rows, nh, nkv, hd, ld, seed, P=32768):
    buf = randn(rows * ld + 64, seed=seed)                      # 64 guard elements past the last row
    pos = torch.randint(0, P, (rows,), generator=torch.Generator().manual_seed(seed)).to(DEV)
    pos[0], pos[-1] = 0, P - 1
    return buf, pos


def rope_call(buf, ld, nh, nkv, hd, cos, sin, pos, rows, backward):
    k = K()
    k.call("lmod_rope", k.ptr(buf), ld, nh, buf.data_ptr() + nh * hd * 2, ld, nkv, hd, k.ptr(cos), k.ptr(sin), k.ptr(pos), rows, backward)


def rows_view(buf, rows, ld, width):
    return buf[: rows * ld].view(rows, ld)[:, :width]


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("nh,nkv", [(16, 16), (14, 2), (28, 4), (32, 32)])
def test_rope_element_wise(nh, nkv, hd):
    from llavamod.model.language_model.qwen2_core import rope_tables
    rows, P = 257, 32768
    ld = (nh + 2 * nkv) * hd
    cos, sin = rope_tables(hd, P, 1e6, bf16, DEV)
    buf, pos = rope_buffers(rows, nh, nkv, hd, ld, seed=nh + hd)
    orig = buf.clone()
    rope_call(buf, ld, nh, nkv, hd, cos, sin, pos, rows, 0)
    x = rows_view(orig, rows, ld, ld)
    q = x[:, : nh * hd].reshape(1, rows, nh, hd).transpose(1, 2)
    kk = x[:, nh * hd:(nh + nkv) * hd].reshape(1, rows, nkv, hd).transpose(1, 2)
    qr, kr = R.apply_rope(q, kk, cos, sin, pos.view(1, rows))
    got = rows_view(buf, rows, ld, ld)
    check_bound("rope q", got[:, : nh * hd], qr.transpose(1, 2).reshape(rows, -1))
    check_bound("rope k", got[:, nh * hd:(nh + nkv) * hd], kr.transpose(1, 2).reshape(rows, -1))
    check_bound("v untouched", got[:, (nh + nkv) * hd:], x[:, (nh + nkv) * hd:])
    check_bound("guard untouched", buf[rows * ld:], orig[rows * ld:])
    # the scalar kernel (row stride not a multiple of 8) gives the same bytes
    lds = ld + 2
    sbuf = torch.zeros(rows * lds + 64, dtype=bf16, device=DEV)
    rows_view(sbuf, rows, lds, ld).copy_(x)
    guard = sbuf.clone()
    rope_call(sbuf, lds, nh, nkv, hd, cos, sin, pos, rows, 0)
    check_bound("rope scalar kernel", rows_view(sbuf, rows, lds, ld), got)
    check_bound("scalar kernel: row padding untouched", sbuf[: rows * lds].view(rows, lds)[:, ld:], guard[: rows * lds].view(rows, lds)[:, ld:])
    # backward: transpose rotation, element-wise against float64 and within one ulp of bf16 autograd of the oracle
    dbuf = randn(rows * ld + 64, seed=nh + hd + 1)
    dorig = dbuf.clone()
    rope_call(dbuf, ld, nh, nkv, hd, cos, sin, pos, rows, 1)
    dy = rows_view(dorig, rows, ld, (nh + nkv) * hd)
    ref = rope_bwd_reference_fp64(dy, cos, sin, pos, hd)
    dgot = rows_view(dbuf, rows, ld, (nh + nkv) * hd)
    check_bound("rope bwd", dgot, ref["d"], ref["tol"])
    check_bound("rope bwd: v untouched", rows_view(dbuf, rows, ld, ld)[:, (nh + nkv) * hd:], rows_view(dorig, rows, ld, ld)[:, (nh + nkv) * hd:])
    qa, ka = q.detach().clone().requires_grad_(True), kk.detach().clone().requires_grad_(True)
    qo, ko = R.apply_rope(qa, ka, cos, sin, pos.view(1, rows))
    torch.autograd.backward([qo, ko], [dy[:, : nh * hd].reshape(1, rows, nh, hd).transpose(1, 2),
                                       dy[:, nh * hd:].reshape(1, rows, nkv, hd).transpose(1, 2)])
    ag = torch.cat([qa.grad.transpose(1, 2).reshape(rows, -1), ka.grad.transpose(1, 2).reshape(rows, -1)], 1)
    check_bound("rope bwd vs bf16 autograd", dgot, ag.double(), ref["tol_ag"])
    sd = torch.zeros_like(sbuf)
    rows_view(sd, rows, lds, ld).copy_(rows_view(dorig, rows, ld, ld))
    rope_call(sd, lds, nh, nkv, hd, cos, sin, pos, rows, 1)
    check_bound("rope bwd scalar kernel", rows_view(sd, rows, lds, (nh + nkv) * hd), ref["d"], ref["tol"])


def test_rope_scalar_kernel_head_dim_24():
    from llavamod.model.language_model.qwen2_core import rope_tables
    nh, nkv, hd, rows, P = 6, 2, 24, 33, 4096                 # hd % 16 != 0: the scalar kernel
    ld = (nh + 2 * nkv) * hd
    cos, sin = rope_tables(hd, P, 1e6, bf16, DEV)
    buf, pos = rope_buffers(rows, nh, nkv, hd, ld, seed=24, P=P)
    orig = buf.clone()
    rope_call(buf, ld, nh, nkv, hd, cos, sin, pos, rows, 0)
    x = rows_view(orig, rows, ld, ld)
    qr, kr = R.apply_rope(x[:, : nh * hd].reshape(1, rows, nh, hd).transpose(1, 2),
                          x[:, nh * hd:(nh + nkv) * hd].reshape(1, rows, nkv, hd).transpose(1, 2), cos, sin, pos.view(1, rows))
    got = rows_view(buf, rows, ld, ld)
    check_bound("rope hd=24 q", got[:, : nh * hd], qr.transpose(1, 2).reshape(rows, -1))
    check_bound("rope hd=24 k", got[:, nh * hd:(nh + nkv) * hd], kr.transpose(1, 2).reshape(rows, -1))
    check_bound("rope hd=24 v", got[:, (nh + nkv) * hd:], x[:, (nh + nkv) * hd:])
    check_bound("rope hd=24 guard", buf[rows * ld:], orig[rows * ld:])


# ---------------------------------------------------------------------------------------------------------------------
# activations
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("I", [8, 2816, 4864, 5504, 11008])
def test_silu_mul_element_wise(I):
    k = K()
    rows = 64
    ld = 2 * I + 24                                             # a row stride wider than 2I
    gu = randn(rows, ld, seed=I, scale=3.0)
    gu[:, :I][0] = torch.linspace(-100, 100, I, device=DEV).to(bf16)            # saturating gates
    gu[1, :min(I, 8)] = torch.tensor([100, -100, 90, -90, -88.5, 30, -30, 0.0], device=DEV)[:min(I, 8)].to(bf16)
    out = torch.empty(rows, I, dtype=bf16, device=DEV)
    k.call("lmod_silu_mul_fwd", k.ptr(gu), ld, rows, I, k.ptr(out))
    ref = silu_mul_reference_fp64(gu, I)
    check_bound(f"silu_mul I={I}", out, ref["out"], ref["out_tol"])
    d = randn(rows, I, seed=I + 1)
    dgu = torch.full((rows, ld), 7.0, dtype=bf16, device=DEV)
    k.call("lmod_silu_mul_bwd", k.ptr(d), k.ptr(gu), ld, rows, I, k.ptr(dgu))
    b = ref["bwd"](d)
    check_bound(f"silu_mul dgate I={I}", dgu[:, :I], b["dg"], b["dg_tol"])
    check_bound(f"silu_mul dup I={I}", dgu[:, I:2 * I], b["du"], b["du_tol"])
    assert bool((dgu[:, 2 * I:] == 7).all()), "bytes past 2I of a row untouched"


@pytest.mark.parametrize("n", [8, 1024, 4096, 5504])
def test_bias_act_and_gelu_bwd_element_wise(n):
    k = K()
    rows = 77
    x = randn(rows, n, seed=n, scale=3.0)
    x[0, : min(n, 8)] = torch.tensor([-9.0, -5.0, -3.0, -0.75, 0.0, 3.0, 9.0, 40.0], device=DEV)[: min(n, 8)].to(bf16)
    bias = randn(n, seed=n + 1)
    for act in (k.ACT_GELU, k.ACT_QUICK_GELU, k.ACT_NONE):
        for b in (None, bias):
            y = k.bias_act(x, b, act)
            ref = bias_act_reference_fp64(x, b, act)
            check_bound(f"act={act} bias={b is not None} n={n}", y, ref["y"], ref["tol"])
    for count in (8 * 33, n * rows - 8 * 7):                   # counts not multiples of 256
        xx, dy = x.reshape(-1)[:count], randn(count, seed=count)
        dx = torch.empty(count, dtype=bf16, device=DEV)
        k.call("lmod_gelu_bwd", k.ptr(dy), k.ptr(xx), count, k.ptr(dx))
        ref = gelu_bwd_reference_fp64(dy, xx)
        check_bound(f"gelu_bwd count={count}", dx, ref["dx"], ref["tol"])


# ---------------------------------------------------------------------------------------------------------------------
# add, splice forward / backward at production size, the token-embedding gradient
# ---------------------------------------------------------------------------------------------------------------------
def production_splice(side):
    """4 samples of T' <= 2048 with 576-patch images: two images in samples 0 and 2, one in 1, none in 3; padding in samples 1 and 3."""
    from llavamod.model.llava_arch import splice_plan
    B, P, V = 4, 576, 151936
    Tt = 2048 - 2 * (P - 1)
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(0, V, (B, Tt), generator=g)
    ids[:, :40] = torch.randint(0, 64, (B, 40), generator=g)               # a chat template: few tokens, many repeats
    ids[0, 3] = ids[0, 400] = ids[1, 10] = ids[2, 0] = ids[2, Tt - 1] = -200
    mask = torch.ones(B, Tt, dtype=torch.bool)
    mask[1, Tt - 100:] = False
    mask[3, Tt - 333:] = False
    return [torch.from_numpy(a) for a in splice_plan(ids.numpy(), mask.numpy(), None, P, side)], P, V


def test_add_bit_exact():
    n = 2048 * 1024
    a, b = randn(n, seed=1, scale=100.0), randn(n, seed=2, scale=0.01)
    out = torch.empty_like(a)
    k = K()
    k.call("lmod_add", k.ptr(a), k.ptr(b), n, k.ptr(out))
    check_bound("add", out, a + b)


@pytest.mark.parametrize("side", ["right", "left"])
def test_splice_forward_backward_bit_exact(side):
    from llavamod.model.llava_arch import embed_grad_order
    (src, _, _, _, img), P, V = production_splice(side)
    H = 1024
    n_img = 6                                                   # 5 image tokens + the entry sample 3 consumes without one
    emb, feats = randn(V, H, seed=3), randn(n_img, P, H, seed=4)
    src_d, img_d = src.to(DEV), img.to(DEV)
    order = torch.from_numpy(embed_grad_order(src.numpy())).to(DEV)
    fd = feats.clone().requires_grad_(True)
    gbuf = randn(V, H, seed=6, scale=0.1)
    old = gbuf.clone()
    out = K().splice_embed(fd, emb, src_d, img_d, P, embed_grad=gbuf, order=order)
    check_bound(f"splice {side}", out.view(-1, H), splice_reference(emb, feats, src_d, img_d, P))
    d = randn(*out.shape, seed=7)
    out.backward(d)
    check_bound(f"splice bwd {side}", fd.grad, splice_bwd_reference(d, src_d, img_d, n_img, P))
    ref = embed_grad_reference_fp64(d, src_d, old)
    check_bound(f"embed grad through the splice {side}", gbuf[ref["toks"]], ref["want"], ref["tol"])


@pytest.mark.parametrize("H", [896, 1024])
def test_embed_grad_element_wise_and_deterministic(H):
    from llavamod.model.llava_arch import PAD_SRC, embed_grad_order
    k = K()
    V = 151936
    g = torch.Generator().manual_seed(H)
    toks = torch.randperm(V, generator=g)[:300]
    reps = {8: int(toks[200]), 64: int(toks[201]), 512: int(toks[202]), 4096: int(toks[203])}
    parts = [toks[:200], torch.tensor([V - 1, 0])] + [torch.full((n,), t) for n, t in reps.items()]
    parts += [-1 - torch.arange(576), torch.full((78,), PAD_SRC)]                 # image rows and padding skipped
    src = torch.cat(parts)
    src = src[torch.randperm(src.numel(), generator=g)].view(2, -1)
    d = randn(src.numel(), H, seed=H + 1).view(2, -1, H)
    old = randn(V, H, seed=H + 2, scale=0.1)
    src_d = src.to(DEV)
    order = torch.from_numpy(embed_grad_order(src.numpy())).to(DEV)
    runs = []
    for _ in range(2):
        gr = old.clone()
        k.embed_grad_(d, src_d, order, gr)
        runs.append(gr)
    assert torch.equal(runs[0], runs[1]), "two runs from the same gradient differ"
    ref = embed_grad_reference_fp64(d, src_d, old)
    report = {}
    check_bound(f"embed grad H={H}", runs[0][ref["toks"]], ref["want"], ref["tol"], report)
    for n, t in reps.items():
        i = int((ref["toks"] == t).nonzero())
        assert int(ref["counts"][i]) == n
        check_bound(f"embed grad x{n}", runs[0][t], ref["want"][i], ref["tol"][i])
    untouched = torch.ones(V, dtype=torch.bool, device=DEV)
    untouched[ref["toks"]] = False
    assert torch.equal(runs[0][untouched], old[untouched]), "an untouched vocabulary row changed"


# ---------------------------------------------------------------------------------------------------------------------
# gradient sum of squares (multi-block partials + last-block ticket) and AdamW
# ---------------------------------------------------------------------------------------------------------------------
def sumsq_check(buf, name):
    k = K()
    n = buf.numel()
    outs = []
    for _ in range(2):
        out = torch.full((1,), 3.5, dtype=torch.float32, device=DEV)             # accumulates into a non-zero out
        k.sumsq_(buf, out)
        outs.append(out)
    assert torch.equal(outs[0], outs[1]), f"{name}: two runs differ"
    S = sumsq_reference_fp64(buf)
    chain = sumsq_chain(n, sumsq_blocks(n, n_sms()))
    tol = chain * FP32_U * S + FP32_U * (S + 3.5)
    got = float(outs[0])
    assert abs(got - (3.5 + S)) <= tol, (name, n, got, 3.5 + S, tol)


@pytest.mark.parametrize("dtype", [bf16, torch.float32])
def test_sumsq_sizes_element_wise(dtype):
    cap = 2048 * n_sms() * 8                                    # the element count at which the grid reaches its cap
    for n in (1000, 2048 + 3, cap - 8, cap, cap + 1, 5 * cap + 7):
        sumsq_check(randn(n, seed=n, scale=0.3, dtype=dtype), f"{dtype} n={n}")


def test_sumsq_1e9_bf16_elements():
    n = 10 ** 9 + 3
    buf = torch.empty(n, dtype=bf16, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(9)
    for i in range(0, n, 1 << 27):
        buf[i:i + (1 << 27)].normal_(generator=g)
    sumsq_check(buf, "1e9")
    del buf


@pytest.mark.parametrize("gdtype", [bf16, torch.float32])
@pytest.mark.parametrize("with_model", [True, False])
@pytest.mark.parametrize("clip", ["active", "inactive", "off"])
@pytest.mark.parametrize("step,wd", [(1, 0.0), (1, 0.01), (10000, 0.0), (10000, 0.01)])
def test_adamw_element_wise(gdtype, with_model, clip, step, wd):
    k = K()
    n = n_sms() * 16 * 256 * 2 + 5                              # past the grid cap: the grid-stride loop
    seed = step + int(wd * 100) + (clip == "active")
    p = randn(n, seed=seed, dtype=torch.float32)
    m = randn(n, seed=seed + 1, scale=0.01, dtype=torch.float32)
    v = randn(n, seed=seed + 2, scale=1e-2, dtype=torch.float32).square()
    grad = randn(n, seed=seed + 3, scale=3.0, dtype=gdtype)
    nsq = torch.zeros(1, device=DEV)
    k.sumsq_(grad, nsq)
    gs = 0.125
    total = float(nsq.sqrt()) * gs
    max_norm = {"active": total / 4, "inactive": total * 4, "off": 0.0}[clip]
    model = torch.empty(n, dtype=bf16, device=DEV) if with_model else None
    pk, mk, vk = p.clone(), m.clone(), v.clone()
    k.adamw_(pk, mk, vk, grad, model, 1e-3, 0.9, 0.999, 1e-8, wd, step, nsq, max_norm, gs)
    ref = adamw_reference_fp64(p, m, v, grad, step, 1e-3, 0.9, 0.999, 1e-8, wd, float(nsq), max_norm, gs)
    tag = f"{gdtype} model={with_model} clip={clip} step={step} wd={wd}"
    check_bound(f"m {tag}", mk, ref["m"], ref["m_tol"])
    check_bound(f"v {tag}", vk, ref["v"], ref["v_tol"])
    check_bound(f"master {tag}", pk, ref["master"], ref["master_tol"])
    if with_model:
        check_bound(f"model {tag}", model, pk.to(bf16))
