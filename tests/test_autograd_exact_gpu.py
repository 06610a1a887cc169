"""The student's autograd Functions (llavamod/kernels.py: LinearFn, QKVRopeFn, RopeFn, RMSNormFn, SiluMulFn, GeluFn, SpliceFn) element by
element against float64: which kernel gets which operand, and where each gradient lands.

Every case
  - carves every gradient view it writes out of ONE flat bf16 buffer in the gradient arena's layout (train/engine.py _pack: each unit
    starts on a multiple of ALIGN elements, 256 bytes), prefilled with seeded values, with a sentinel in every other element;
  - runs three micro-batches with different inputs into the same views, each under helpers.poisoned_uninitialised_memory, and after each
    one checks the outputs, the gradients and every view against float64, every sentinel unchanged and no NaN in any output;
  - builds each reference stage by stage from the kernels' own previous stage (the tensors the Functions saved, or the gradient a node
    received), so each bound covers one stage: _gemm_tol for a GEMM (with the old view value for an accumulated wgrad), the element-wise
    references of tests/helpers.py for the rest;
  - checks every accumulated view from the value the kernels left in it after the micro-batch before: g <- bf16(g + contribution), so a
    lost, doubled or overwritten micro-batch fails at the step where it happens;
  - runs twice and requires the same bytes from both runs.  No shape here reaches the split-K dgrad of mm_nn (the lm_head's: see
    test_distill_head_exact_gpu.py); the one
    fp32-atomic path that is reached, lmod_rmsnorm_wgrad from 257 rows on, is left out of the byte comparison (see test_rmsnorm_fn);
  - prints its worst err / bound."""
import types

import pytest
import torch

from tests.helpers import (BF16_U, DEV, Arena, _gemm_tol, bias_act_reference_fp64, bias_grad_reference_fp64, check_bound,  # noqa: E402
                           embed_grad_reference_fp64, gelu_bwd_reference_fp64, no_nan, poisoned_uninitialised_memory,
                           qkv_rope_reference_fp64, randn, rmsnorm_bwd_reference_fp64, rmsnorm_reference_fp64, rmsnorm_wgrad_reference_fp64,
                           rope_bwd_reference_fp64, silu_mul_reference_fp64, splice_bwd_reference, splice_reference, twice)

pytestmark = pytest.mark.gpu

bf16 = torch.bfloat16
MICRO_BATCHES = 3
# (B, T) of the 3-D inputs: row counts 1, 127, 129, 333 and 2047 leave a tail tile in every GEMM and wgrad, 2048 is the step's T'
ROWS = [(1, 1), (1, 127), (3, 43), (3, 111), (23, 89), (2, 1024)]
ROW_IDS = [f"rows{b * t}" for b, t in ROWS]


def K():
    from llavamod import kernels
    return kernels


def gemm_check(name, got, A, B, k_red, report, bias=None, old=None):
    """got = bf16(A B^T (+ bias) (+ old)) from the wgmma GEMM: A [M, k_red], B [N, k_red] (any float tensors, views allowed)."""
    A64, B64 = A.double(), B.double()
    ref, maj = A64 @ B64.t(), A64.abs() @ B64.abs().t()
    extra = 0.0
    if bias is not None:
        ref, maj = ref + bias.double(), maj + bias.double().abs()
    if old is not None:
        ref, maj = ref + old.double(), maj + old.double().abs()
        extra = 2.0 ** -23 * ref.abs()                  # D = bf16(fp32(D_old) + acc): the fp32 add
    return check_bound(name, got.reshape(ref.shape), ref, _gemm_tol(ref, maj, k_red) + extra, report)


def bias_check(name, got, dy2, old, report):
    r = bias_grad_reference_fp64(dy2, old)
    return check_bound(name, got, r["want"], r["tol"], report)


def rope_bwd_kernel(d, cos, sin, pos, nh, nkv, hd):
    """The transpose rotation of lmod_rope on a copy of the contiguous [rows, (nh + 2 nkv) hd] gradient."""
    k = K()
    d = d.clone()
    ld = d.shape[-1]
    k.call("lmod_rope", k.ptr(d), ld, nh, d.data_ptr() + nh * hd * 2, ld, nkv, hd, k.ptr(cos), k.ptr(sin), k.ptr(pos), d.numel() // ld, 1)
    return d


def strided_dy(rows, n, seed, shape):
    """A gradient that is a column slice of a wider buffer (not contiguous), viewed as `shape`."""
    return randn(rows, n + 8, seed=seed)[:, :n].view(*shape, n)


# ---------------------------------------------------------------------------------------------------------------------
# LinearFn / K.linear: dx, the wgrad accumulated into the arena, the bias gradient; every combination of x.requires_grad x a wgrad view
# ---------------------------------------------------------------------------------------------------------------------
# (K, N): config 2's o_proj and down_proj, the 1.8B student's down_proj
LINEAR_SHAPES = [(1024, 1024), (2816, 1024), (5504, 2048)]


@pytest.mark.parametrize("bt", ROWS, ids=ROW_IDS)
@pytest.mark.parametrize("kn", LINEAR_SHAPES, ids=[f"{k}to{n}" for k, n in LINEAR_SHAPES])
@pytest.mark.parametrize("x_grad,train_w", [(True, True), (False, True), (True, False), (False, False)])
def test_linear_fn(bt, kn, x_grad, train_w):
    B, T = bt
    Kin, N = kn
    rows = B * T
    k = K()
    seed = rows * 7 + Kin + N + 2 * x_grad + train_w
    w = randn(N, Kin, seed=seed, scale=Kin ** -0.5).requires_grad_(train_w)
    b = randn(N, seed=seed + 1)
    tag = f"linear rows={rows} {Kin}->{N} x_grad={x_grad} wgrad={train_w}"

    def run(report):
        arena = Arena([(N, Kin), (N,)], seed=seed + 2)
        gw, gb = arena.views if train_w else (None, None)
        outs = []
        for mb in range(MICRO_BATCHES):
            x = randn(B, T, Kin, seed=seed + 10 * mb + 3).requires_grad_(x_grad)
            dy = strided_dy(rows, N, seed + 10 * mb + 4, (B, T))
            old = arena.snapshot()
            before = arena.buf.clone()
            with poisoned_uninitialised_memory():
                y = k.linear(x, w, b, gw, gb)
                if x_grad or train_w:
                    assert y.grad_fn is not None and type(y.grad_fn).__name__.startswith("LinearFn")
                    y.backward(dy)
                else:
                    assert not y.requires_grad
            torch.cuda.synchronize()
            t = f"{tag} mb={mb}"
            arena.check_sentinels(t)
            dx = x.grad
            assert (dx is not None) == x_grad, f"{t}: dx is {'missing' if x_grad else 'not None'}"
            assert w.grad is None, f"{t}: the weight gradient must land in the arena view only"
            no_nan(t, y=y, dx=dx)
            if not train_w:
                assert torch.equal(arena.buf.view(torch.int16), before.view(torch.int16)), f"{t}: no wgrad view, but the arena changed"
            if report is not None:
                x2, dy2 = x.detach().reshape(rows, Kin), dy.reshape(rows, N)
                assert y.shape == (B, T, N)
                gemm_check(f"y mb={mb}", y.detach(), x2, w.detach(), Kin, report, bias=b)
                if x_grad:
                    assert dx.shape == x.shape
                    gemm_check(f"dx mb={mb}", dx, dy2, w.detach().t(), N, report)
                if train_w:
                    gemm_check(f"wgrad mb={mb}", gw, dy2.t(), x2.t(), rows, report, old=old[0])
                    bias_check(f"bgrad mb={mb}", gb, dy2, old[1], report)
            outs += [y.detach().clone()] + ([dx.clone()] if x_grad else [])
        return outs + [arena.buf.clone()]

    twice(tag, run)


# ---------------------------------------------------------------------------------------------------------------------
# QKVRopeFn (hd 64 / 128, MHA and GQA) and RopeFn behind LinearFn (hd 32, the unfused path K.qkv_rope takes)
# ---------------------------------------------------------------------------------------------------------------------
# (H, nh, nkv, hd): config 2, Qwen2-0.5B's GQA, the 1.8B student, a GQA form at hd 128, and hd 32
QKV_SHAPES = [(1024, 16, 16, 64), (896, 14, 2, 64), (2048, 16, 16, 128), (2048, 16, 4, 128), (256, 8, 2, 32)]
MAX_POS = 4096


@pytest.mark.parametrize("bt", ROWS, ids=ROW_IDS)
@pytest.mark.parametrize("shape", QKV_SHAPES, ids=[f"H{h}_{a}x{c}_hd{d}" for h, a, c, d in QKV_SHAPES])
def test_qkv_rope_fn(bt, shape):
    from llavamod.model.language_model.qwen2_core import rope_tables
    B, T = bt
    H, nh, nkv, hd = shape
    rows, N = B * T, (nh + 2 * nkv) * hd
    nr = (nh + nkv) * hd
    k = K()
    fused = hd in k.ATTN_HEAD_DIMS
    seed = rows * 5 + H + hd
    cos, sin = rope_tables(hd, MAX_POS, 1e6, bf16, DEV)
    w = randn(N, H, seed=seed, scale=H ** -0.5).requires_grad_(True)
    b = randn(N, seed=seed + 1)
    tag = f"{'QKVRopeFn' if fused else 'LinearFn+RopeFn'} rows={rows} H={H} {nh}x{nkv} hd={hd}"

    def run(report):
        arena = Arena([(N, H), (N,)], seed=seed + 2)
        gw, gb = arena.views
        outs = []
        for mb in range(MICRO_BATCHES):
            x = randn(B, T, H, seed=seed + 10 * mb + 3).requires_grad_(True)
            pos = torch.randint(0, MAX_POS, (rows,), device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed + mb))
            pos[0] = MAX_POS - 1
            d = randn(rows, N, seed=seed + 10 * mb + 4)          # the fused dq|dk|dv of the attention backward
            d_keep = d.clone()
            seen, into_linear = [], []
            old = arena.snapshot()
            with poisoned_uninitialised_memory():
                out = k.qkv_rope(x, w, b, cos, sin, pos, nh, nkv, hd, gw, gb)
                name = type(out.grad_fn).__name__
                assert name.startswith("QKVRopeFn" if fused else "RopeFn"), name
                assert out.shape == (rows, N), "both paths return the fused q|k|v rows"
                if not fused:                                 # the rotated-back gradient LinearFn receives
                    out.grad_fn.next_functions[0][0].register_prehook(lambda g: into_linear.append(g[0].clone()))
                out.register_hook(lambda g: seen.append(g))  # a second reader of the incoming gradient
                out.backward(d.view(out.shape))
            torch.cuda.synchronize()
            t = f"{tag} mb={mb}"
            arena.check_sentinels(t)
            no_nan(t, out=out, dx=x.grad)
            # the incoming gradient is read, never written: by the caller and by the hook, it is the tensor it was
            assert torch.equal(d.view(torch.int16), d_keep.view(torch.int16)), f"{t}: backward changed the caller's gradient tensor"
            assert torch.equal(seen[0].reshape(rows, N).view(torch.int16), d_keep.view(torch.int16)), \
                f"{t}: backward changed the gradient a hook received"
            assert w.grad is None
            if report is not None:
                x2 = x.detach().reshape(rows, H)
                want, tol = qkv_rope_reference_fp64(x2, w.detach(), b, cos, sin, pos, nh, nkv, hd, H)
                check_bound(f"out mb={mb}", out.detach().reshape(rows, N), want, tol, report)
                dr = rope_bwd_kernel(d_keep, cos, sin, pos, nh, nkv, hd)
                rb = rope_bwd_reference_fp64(d_keep[:, :nr], cos, sin, pos, hd)
                check_bound(f"rotated-back dq|dk mb={mb}", dr[:, :nr], rb["d"], rb["tol"], report)
                check_bound(f"dv passes unrotated mb={mb}", dr[:, nr:], d_keep[:, nr:], None, report)
                if not fused:
                    check_bound(f"gradient into LinearFn mb={mb}", into_linear[0].reshape(rows, N), dr, None, report)
                gemm_check(f"dx mb={mb}", x.grad, dr, w.detach().t(), N, report)
                gemm_check(f"wgrad mb={mb}", gw, dr.t(), x2.t(), rows, report, old=old[0])
                bias_check(f"q|k|v bgrad mb={mb}", gb, dr, old[1], report)
            outs += [out.detach().clone(), x.grad.clone()]
        return outs + [arena.buf.clone()]

    twice(tag, run)


# ---------------------------------------------------------------------------------------------------------------------
# RMSNormFn / K.rmsnorm: with the fused residual (ds given or not) and without it; the weight gradient from s into the arena
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bt", ROWS, ids=ROW_IDS)
@pytest.mark.parametrize("H", [1024, 2048])
@pytest.mark.parametrize("mode", ["res+ds", "res", "nores"])
def test_rmsnorm_fn(bt, H, mode):
    B, T = bt
    rows = B * T
    k, eps = K(), 1e-6
    seed = rows * 3 + H + len(mode)
    w = (1 + 0.1 * randn(H, seed=seed).float()).to(bf16)
    with_res = mode != "nores"
    tag = f"RMSNormFn rows={rows} H={H} {mode}"

    def run(report):
        arena = Arena([(H,)], seed=seed + 1)
        (gw,) = arena.views
        outs = []
        for mb in range(MICRO_BATCHES):
            x = randn(B, T, H, seed=seed + 10 * mb + 2, scale=2.0).requires_grad_(True)
            res = randn(B, T, H, seed=seed + 10 * mb + 3).requires_grad_(True) if with_res else None
            dy = randn(B, T, H, seed=seed + 10 * mb + 4)
            ds = randn(B, T, H, seed=seed + 10 * mb + 5) if mode != "res" else None
            old = arena.snapshot()
            with poisoned_uninitialised_memory():
                if not with_res:                              # the Function's own second output is the empty tensor
                    assert k.RMSNormFn.apply(x, None, w, eps, None)[1].numel() == 0
                y, s = k.rmsnorm(x, w, eps, res=res, wgrad=gw)
                s_saved, _, rstd = y.grad_fn.saved_tensors
                if not with_res:
                    assert s is x, "without a residual the stream is x itself"
                torch.autograd.backward([y, s] if ds is not None else [y], [dy, ds] if ds is not None else [dy])
            torch.cuda.synchronize()
            t = f"{tag} mb={mb}"
            arena.check_sentinels(t)
            ws = [v for v in k._ZERO_WS.values()]
            assert all(int(v.ne(0).sum()) == 0 for v in ws), f"{t}: the shared workspace came back dirty"
            no_nan(t, y=y, s=s, dx=x.grad, dres=res.grad if with_res else None)
            if report is not None:
                x2, dy2 = x.detach().reshape(rows, H), dy.reshape(rows, H)
                res2 = res.detach().reshape(rows, H) if with_res else None
                ref = rmsnorm_reference_fp64(x2, w, eps, res=res2, rstd_k=rstd)
                check_bound(f"s mb={mb}", s.detach().reshape(rows, H), ref["s"], None, report)
                check_bound(f"saved s mb={mb}", s_saved.reshape(rows, H), ref["s"], None, report)
                check_bound(f"rstd mb={mb}", rstd, ref["rstd"], ref["rstd_tol"], report)
                check_bound(f"y mb={mb}", y.detach().reshape(rows, H), ref["y"], None, report)
                sk = ref["s"]
                ds2 = ds.reshape(rows, H) if ds is not None else None
                if with_res:
                    bw = rmsnorm_bwd_reference_fp64(dy2, sk, w, rstd, ds2)
                    check_bound(f"dx mb={mb}", x.grad.reshape(rows, H), bw["dx"], bw["tol"], report)
                    check_bound(f"dres mb={mb}", res.grad.reshape(rows, H), bw["dx"], bw["tol"], report)
                else:                                         # autograd adds the stream's gradient to the norm's dx in bf16
                    bw = rmsnorm_bwd_reference_fp64(dy2, sk, w, rstd)
                    want = bw["dx"] + ds2.double()
                    check_bound(f"dx + ds mb={mb}", x.grad.reshape(rows, H), want, BF16_U * want.abs() + (1 + BF16_U) * bw["tol"], report)
                wr = rmsnorm_wgrad_reference_fp64(dy2, sk, rstd, old[0])
                check_bound(f"wgrad mb={mb}", gw, wr["want"], wr["tol"], report)
            outs += [y.detach().clone(), s.detach().clone(), x.grad.clone()] + ([res.grad.clone()] if with_res else [])
        # lmod_rmsnorm_wgrad adds the partial sums of its 256-row chunks with fp32 atomics in any order: from 257 rows on, two runs may
        # differ in the last bit of a weight-gradient element (rmsnorm_wgrad_reference_fp64 bounds every order)
        return outs + ([arena.buf.clone()] if rows <= 256 else [])

    twice(tag, run)


# ---------------------------------------------------------------------------------------------------------------------
# K.mlp on its training path: LinearFn -> SiluMulFn -> LinearFn, every stage from the previous one
# ---------------------------------------------------------------------------------------------------------------------
MLP_SHAPES = [(1024, 2816), (2048, 5504)]


@pytest.mark.parametrize("bt", ROWS, ids=ROW_IDS)
@pytest.mark.parametrize("hi", MLP_SHAPES, ids=[f"H{h}_I{i}" for h, i in MLP_SHAPES])
def test_mlp_training_path(bt, hi):
    B, T = bt
    H, I = hi
    rows = B * T
    k = K()
    seed = rows * 11 + H
    w_gu = randn(2 * I, H, seed=seed, scale=H ** -0.5)
    w_dn = randn(H, I, seed=seed + 1, scale=I ** -0.5)
    tag = f"K.mlp rows={rows} H={H} I={I}"

    def run(report):
        arena = Arena([(2 * I, H), (H, I)], seed=seed + 2)
        g_gu, g_dn = arena.views
        outs = []
        for mb in range(MICRO_BATCHES):
            x = randn(B, T, H, seed=seed + 10 * mb + 3).requires_grad_(True)
            dy = strided_dy(rows, H, seed + 10 * mb + 4, (B, T))
            got = {}
            old = arena.snapshot()
            with poisoned_uninitialised_memory():
                y = k.mlp(x, w_gu, w_dn, g_gu, g_dn)
                dn_node = y.grad_fn
                act = dn_node.saved_tensors[0]
                silu_node = dn_node.next_functions[0][0]
                gu = silu_node.saved_tensors[0]
                gu_node = silu_node.next_functions[0][0]
                names = [type(n).__name__ for n in (dn_node, silu_node, gu_node)]
                assert [n[:n.index("Fn") + 2] for n in names] == ["LinearFn", "SiluMulFn", "LinearFn"], names
                silu_node.register_prehook(lambda g: got.__setitem__("dact", g[0].clone()))
                gu_node.register_prehook(lambda g: got.__setitem__("dgu", g[0].clone()))
                y.backward(dy)
            torch.cuda.synchronize()
            t = f"{tag} mb={mb}"
            arena.check_sentinels(t)
            no_nan(t, y=y, dx=x.grad, act=act, gu=gu, dact=got["dact"], dgu=got["dgu"])
            if report is not None:
                x2, dy2 = x.detach().reshape(rows, H), dy.reshape(rows, H)
                gu2, act2 = gu.detach().reshape(rows, 2 * I), act.detach().reshape(rows, I)
                dact, dgu = got["dact"].reshape(rows, I), got["dgu"].reshape(rows, 2 * I)
                gemm_check(f"gate|up mb={mb}", gu2, x2, w_gu, H, report)
                sm = silu_mul_reference_fp64(gu2, I)
                check_bound(f"act mb={mb}", act2, sm["out"], sm["out_tol"], report)
                gemm_check(f"y mb={mb}", y.detach(), act2, w_dn, I, report)
                gemm_check(f"dact mb={mb}", dact, dy2, w_dn.t(), H, report)
                gemm_check(f"g_dn mb={mb}", g_dn, dy2.t(), act2.t(), rows, report, old=old[1])
                bw = sm["bwd"](dact)
                check_bound(f"dgate mb={mb}", dgu[:, :I], bw["dg"], bw["dg_tol"], report)
                check_bound(f"dup mb={mb}", dgu[:, I:], bw["du"], bw["du_tol"], report)
                gemm_check(f"dx mb={mb}", x.grad, dgu, w_gu.t(), 2 * I, report)
                gemm_check(f"g_gu mb={mb}", g_gu, dgu.t(), x2.t(), rows, report, old=old[0])
            outs += [y.detach().clone(), x.grad.clone()]
        return outs + [arena.buf.clone()]

    twice(tag, run)


# ---------------------------------------------------------------------------------------------------------------------
# the mlp2x_gelu projector as multimodal_projector/builder.py runs it: K.linear (+bias) -> K.gelu -> K.linear (+bias)
# ---------------------------------------------------------------------------------------------------------------------
PATCHES = 576                                     # CLIP-L/14 at 336 px


@pytest.mark.parametrize("n_img", [1, 3])
@pytest.mark.parametrize("Hs", [1024, 2048])
def test_projector_chain(n_img, Hs):
    from llavamod.model.multimodal_projector.builder import build_projector
    Hc = 1024
    rows = n_img * PATCHES
    seed = Hs + n_img
    cfg = types.SimpleNamespace(mm_image_tower="clip-l-336", image_projector_type="mlp2x_gelu", mm_hidden_size=Hc, hidden_size=Hs,
                                initializer_range=0.02)
    proj = build_projector(cfg)
    l1, l2 = proj.image_spatial_proj.linears()
    with torch.no_grad():
        l1.weight.copy_(randn(Hs, Hc, seed=seed, scale=2 * Hc ** -0.5))
        l1.bias.copy_(randn(Hs, seed=seed + 1))
        l2.weight.copy_(randn(Hs, Hs, seed=seed + 2, scale=Hs ** -0.5))
        l2.bias.copy_(randn(Hs, seed=seed + 3))
    W1, b1, W2, b2 = (p.detach() for p in (l1.weight, l1.bias, l2.weight, l2.bias))
    tag = f"projector {n_img}x{PATCHES} {Hc}->{Hs}"

    def run(report):
        arena = Arena([(Hs, Hc), (Hs,), (Hs, Hs), (Hs,)], seed=seed + 4)
        gW1, gb1, gW2, gb2 = arena.views
        proj.grad_views = {id(l1.weight): gW1, id(l1.bias): gb1, id(l2.weight): gW2, id(l2.bias): gb2}
        outs = []
        for mb in range(MICRO_BATCHES):
            feats = randn(n_img, PATCHES, Hc, seed=seed + 10 * mb + 5).requires_grad_(True)
            dy = randn(n_img, PATCHES, Hs, seed=seed + 10 * mb + 6)
            got = {}
            old = arena.snapshot()
            with poisoned_uninitialised_memory():
                y = proj.forward_image(feats)
                n2 = y.grad_fn
                a = n2.saved_tensors[0]
                ng = n2.next_functions[0][0]
                h = ng.saved_tensors[0]
                n1 = ng.next_functions[0][0]
                names = [type(n).__name__ for n in (n2, ng, n1)]
                assert [n[:n.index("Fn") + 2] for n in names] == ["LinearFn", "GeluFn", "LinearFn"], names
                ng.register_prehook(lambda g: got.__setitem__("da", g[0].clone()))
                n1.register_prehook(lambda g: got.__setitem__("dh", g[0].clone()))
                y.backward(dy)
            torch.cuda.synchronize()
            t = f"{tag} mb={mb}"
            arena.check_sentinels(t)
            for p in (l1.weight, l1.bias, l2.weight, l2.bias):
                assert p.grad is None, f"{t}: a projector gradient must land in the arena view only"
            no_nan(t, y=y, dfeats=feats.grad, h=h, a=a, da=got["da"], dh=got["dh"])
            if report is not None:
                f2, dy2 = feats.detach().reshape(rows, Hc), dy.reshape(rows, Hs)
                h2, a2 = h.detach().reshape(rows, Hs), a.detach().reshape(rows, Hs)
                da, dh = got["da"].reshape(rows, Hs), got["dh"].reshape(rows, Hs)
                gemm_check(f"fc1 mb={mb}", h2, f2, W1, Hc, report, bias=b1)
                ga = bias_act_reference_fp64(h2, None, 0)
                check_bound(f"gelu mb={mb}", a2, ga["y"], ga["tol"], report)
                gemm_check(f"fc2 mb={mb}", y.detach(), a2, W2, Hs, report, bias=b2)
                gemm_check(f"da mb={mb}", da, dy2, W2.t(), Hs, report)
                gemm_check(f"gW2 mb={mb}", gW2, dy2.t(), a2.t(), rows, report, old=old[2])
                bias_check(f"gb2 mb={mb}", gb2, dy2, old[3], report)
                gb = gelu_bwd_reference_fp64(da, h2)
                check_bound(f"gelu bwd mb={mb}", dh, gb["dx"], gb["tol"], report)
                gemm_check(f"dfeats mb={mb}", feats.grad, dh, W1.t(), Hs, report)
                gemm_check(f"gW1 mb={mb}", gW1, dh.t(), f2.t(), rows, report, old=old[0])
                bias_check(f"gb1 mb={mb}", gb1, dh, old[1], report)
            outs += [y.detach().clone(), feats.grad.clone()]
        return outs + [arena.buf.clone()]

    twice(tag, run)


# ---------------------------------------------------------------------------------------------------------------------
# SpliceFn / K.splice_embed: dfeats a scatter of the image rows, the embedding gradient into the arena through `order`
# ---------------------------------------------------------------------------------------------------------------------
def splice_batch(seed, side, V):
    """Four samples: two images in sample 0, one in samples 1 and 2, none in sample 3 (which still consumes a feature entry, whose
    gradient must stay zero); padding in samples 1 and 3; a chat-template-like prefix whose tokens repeat within and across samples,
    one token 200 times across every sample, and ids 0 and V - 1."""
    from llavamod.model.llava_arch import IMAGE_TOKEN_INDEX, splice_plan
    B, Tt = 4, 480
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, V, (B, Tt), generator=g)
    ids[:, :40] = torch.randint(0, 16, (B, 40), generator=g)
    hot = torch.randperm(B * Tt, generator=g)[:200]
    ids.view(-1)[hot] = 7
    ids[0, 0], ids[2, 5] = 0, V - 1
    for b, c in ((0, 3), (0, 300), (1, 10), (2, 0)):
        ids[b, c] = IMAGE_TOKEN_INDEX
    mask = torch.ones(B, Tt, dtype=torch.bool)
    mask[1, Tt - 100:] = False
    mask[3, Tt - 333:] = False
    src, _, _, _, img = splice_plan(ids.numpy(), mask.numpy(), None, PATCHES, side)
    return torch.from_numpy(src), torch.from_numpy(img), 5


@pytest.mark.parametrize("side", ["right", "left"])
def test_splice_fn(side):
    from llavamod.model.llava_arch import embed_grad_order
    k = K()
    H, V = 1024, 4096
    emb = randn(V, H, seed=1)
    tag = f"SpliceFn {side}"
    src0, img0, n_img = splice_batch(0, side, V)
    feats0 = randn(n_img, PATCHES, H, seed=2).requires_grad_(True)
    with pytest.raises(ValueError):                       # an embedding gradient without the plan's row order is refused
        k.splice_embed(feats0, emb, src0.to(DEV), img0.to(DEV), PATCHES, embed_grad=torch.zeros(V, H, dtype=bf16, device=DEV))

    def run(report):
        arena = Arena([(V, H)], seed=3)
        (ge,) = arena.views
        outs = []
        for mb in range(MICRO_BATCHES):
            src, img, n_img = splice_batch(10 + mb, side, V)
            order = torch.from_numpy(embed_grad_order(src.numpy())).to(DEV)
            src_d, img_d = src.to(DEV), img.to(DEV)
            feats = randn(n_img, PATCHES, H, seed=20 + mb).requires_grad_(True)
            d = randn(*src.shape, H, seed=30 + mb)
            old = arena.snapshot()
            with poisoned_uninitialised_memory():
                out = k.splice_embed(feats, emb, src_d, img_d, PATCHES, embed_grad=ge, order=order)
                assert type(out.grad_fn).__name__.startswith("SpliceFn")
                out.backward(d)
            torch.cuda.synchronize()
            t = f"{tag} mb={mb}"
            arena.check_sentinels(t)
            no_nan(t, out=out, dfeats=feats.grad)
            if report is not None:
                check_bound(f"out mb={mb}", out.detach().view(-1, H), splice_reference(emb, feats.detach(), src_d, img_d, PATCHES), None, report)
                check_bound(f"dfeats mb={mb}", feats.grad, splice_bwd_reference(d, src_d, img_d, n_img, PATCHES), None, report)
                er = embed_grad_reference_fp64(d, src_d, old[0])
                assert int(er["counts"].max()) >= 100              # the hot token, less what the padding masks
                check_bound(f"embed grad mb={mb}", ge[er["toks"]], er["want"], er["tol"], report)
                untouched = torch.ones(V, dtype=torch.bool, device=DEV)
                untouched[er["toks"]] = False
                check_bound(f"untouched embedding rows mb={mb}", ge[untouched], old[0][untouched], None, report)
            outs += [out.detach().clone(), feats.grad.clone()]
        return outs + [arena.buf.clone()]

    twice(tag, run)
