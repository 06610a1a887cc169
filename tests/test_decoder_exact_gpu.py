"""The Qwen2 decoder stack (Qwen2Model._layers in llavamod/model/language_model/qwen2_core.py) element by element against float64 at the
teacher and student shapes, bf16 and e4m3, and the production forward bit for bit against a stage replica.

The replica calls the llavamod.kernels functions of _layers in their order, with the same arguments, through every layer of the case.
After every call the stage is checked against the float64 reference of tests/decoder_oracle.py computed from the kernel's own output of
the stage before:
  input norm (residual add fused from layer 1 on), post-attention norm, final norm   rmsnorm bound; the stream bit for bit against torch's
                                                                                       bf16 add
  q|k|v + bias + RoPE (bf16 or e4m3 GEMM)                                              GEMM bound, then the rotation's
  causal attention with the pad ranges and GQA                                         attention bound
  o_proj                                                                               GEMM bound
  MLP                                                                                  its parts: gate|up GEMM, SwiGLU, (e4m3: the
                                                                                       quantised rows), down GEMM
  the MoE layer of the sparse student                                                  tests/test_moe_exact_gpu.py's forward stages
The calls that launch several kernels (mlp, mlp_fp8, linear_fp8, rmsnorm_quant) are also run as their parts, each part checked, and the
composite call must return the parts' bytes.

Qwen2Model.forward then runs under a spy on the same function names.  Each call's arguments and output must match the replica's entry of
the same index bit for bit, so a difference is reported at the first stage it reaches.  Three entry points: the no-grad forward, the
training forward (input that requires grad, gradient views attached; the autograd functions must give the no-grad bytes) and a prefill
into a KVCache, whose rows must be the k|v columns of the replica's q|k|v output, packed per sequence for padded prompts.

Weights are N(0, 1/K), norm weights 1 + 0.1 N, biases N(0, 0.1^2), rope_theta 1e6 (tests/decoder_oracle.py init_decoder_).  The inputs
carry an outlier channel at +-2000, a near-zero row (eps sets its rstd), for e4m3 an all-zero row (scale 1), and padded samples down to
length 1."""
import time
import types

import pytest
import torch

from tests import decoder_oracle as O
from tests.helpers import check_attn, check_bound, check_moe_stages, moe_reference_fp64, poisoned_uninitialised_memory, \
    qkv_rope_reference_fp64, rmsnorm_reference_fp64, silu_mul_reference_fp64

pytestmark = pytest.mark.gpu

BF16, DEV = torch.bfloat16, "cuda"
KERNEL_FNS = ("rmsnorm", "qkv_rope", "attention", "linear", "mlp", "rmsnorm_quant", "qkv_rope_fp8", "linear_fp8", "mlp_fp8", "kv_append",
              "kv_append_rows", "moe_forward_nograd", "MoEFn")
KV_FNS = ("kv_append", "kv_append_rows")
# the gradient-view arguments of the training forward (None in the no-grad forward): keyword names or positions
GRAD_VIEW_ARGS = {"rmsnorm": ("wgrad",), "qkv_rope": (9, 10), "linear": (3,), "mlp": (3, 4)}
E_MOE, TOP_K, CF, MIN_CAP = 4, 2, 1.5, 0        # the sparse student of the distillation recipes


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t0 = time.perf_counter()
    yield
    print(f"\nDECODER wall time {time.perf_counter() - t0:.1f} s")


def bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32) if t.element_size() == 4 else t


def same_bits(a, b):
    from llavamod.kernels import Fp8Rows
    if isinstance(a, (tuple, list)):
        return isinstance(b, (tuple, list)) and len(a) == len(b) and all(same_bits(x, y) for x, y in zip(a, b))
    if isinstance(a, Fp8Rows):
        return isinstance(b, Fp8Rows) and same_bits(a.q, b.q) and same_bits(a.scale, b.scale)
    if not torch.is_tensor(a):
        return not torch.is_tensor(b) and a == b
    return torch.is_tensor(b) and a.dtype == b.dtype and a.shape == b.shape and torch.equal(bits(a), bits(b))


def clone(v):
    from llavamod.kernels import Fp8Rows
    if isinstance(v, (tuple, list)):
        return type(v)(clone(x) for x in v)
    if isinstance(v, Fp8Rows):
        return Fp8Rows(v.q.clone(), v.scale.clone())
    return v.detach().clone() if torch.is_tensor(v) else v


def canon(name, args, out):
    """The MoE layer is moe_forward_nograd without autograd and MoEFn.apply with it: one entry 'moe' with the arguments they share (all
    but MoEFn's gradient views) and the outputs (stream, l_aux)."""
    if name == "MoEFn":
        return "moe", args[:8] + args[9:], out[:2]
    if name == "moe_forward_nograd":
        return "moe", args, out[:2]
    return name, args, out


class KernelCalls:
    """Spies on the llavamod.kernels functions _layers calls.  Each top-level call (calls a spied function makes inside another are not
    entries) is an entry {fn, args, kw, out, stage}, the tensor arguments cloned before the call (kv_append writes into its arguments).
    With `expect` (the log of another run), every call is compared with the entry of the same index, bit for bit, instead of being kept:
    its arguments before it runs, its output after; grad_views: the gradient-view arguments must be given (the replica's are None) and
    are not compared."""

    def __init__(self, expect=None, grad_views=False):
        from llavamod import kernels
        self.K, self.expect, self.grad_views, self.log, self.count, self.depth = kernels, expect, grad_views, [], 0, 0

    def __enter__(self):
        self.orig = {name: getattr(self.K, name) for name in KERNEL_FNS}
        for name, fn in self.orig.items():
            spy = self._spy(name, fn.apply if name == "MoEFn" else fn)
            setattr(self.K, name, types.SimpleNamespace(apply=spy) if name == "MoEFn" else spy)
        return self

    def __exit__(self, *exc):
        for name, fn in self.orig.items():
            setattr(self.K, name, fn)

    def name(self, stage):
        self.log[-1]["stage"] = stage

    def _spy(self, name, fn):
        def call(*args, **kw):
            if self.depth:
                return fn(*args, **kw)
            fname, snap, _ = canon(name, [clone(a) for a in args], ())
            e = dict(fn=fname, args=snap, kw={k: clone(v) for k, v in kw.items()}, stage="(inside kernels.%s)" % name)
            if self.expect is not None:
                self._compare_args(e)                       # before the call: a call with other arguments than the replica's never runs
            self.depth += 1
            try:
                out = fn(*args, **kw)
            finally:
                self.depth -= 1
            e["out"] = clone(canon(name, (), out)[2])
            if self.expect is None:
                self.log.append(e)
            else:
                r = self.expect[self.count]
                assert same_bits(e["out"], r["out"]), f"kernel call {self.count} ({r['stage']}): the output differs from the replica's"
            self.count += 1
            return out
        return call

    def _compare_args(self, e):
        i = self.count
        assert i < len(self.expect), f"the forward makes more kernel calls than the replica ({len(self.expect)}); call {i} is {e['fn']}"
        r = self.expect[i]
        where = f"kernel call {i} ({r['stage']})"
        assert e["fn"] == r["fn"], f"{where}: function mismatch: the forward calls kernels.{e['fn']}, the replica kernels.{r['fn']}"
        assert len(e["args"]) == len(r["args"]) and e["kw"].keys() == r["kw"].keys(), f"{where}: different arguments"
        views = GRAD_VIEW_ARGS.get(e["fn"], ()) if self.grad_views else ()
        pairs = [(j, a, b) for j, (a, b) in enumerate(zip(e["args"], r["args"]))] + [(k, e["kw"][k], r["kw"][k]) for k in r["kw"]]
        for j, a, b in pairs:
            if j in views:
                assert a is not None, f"{where}: argument {j}: no gradient view attached"
                continue
            assert same_bits(a, b), f"{where}: argument {j} differs from the replica's" + ("" if torch.is_tensor(a) else f" ({a!r} != {b!r})")


# ---------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------
# name: (H, I, layers, nh, nkv, B, T, lengths or None, padding side, path, entry points)
#   path: bf16, e4m3 (quantize_fp8_) or moe (MoE layers where initialize_moe_modules' default "sparse" mode puts them: every other layer
#   from 0); entry points: f = no-grad forward, t = training forward, c = prefill into a KVCache
CASES = {
    "qwen1.5-7b-bf16": (4096, 11008, 2, 32, 32, 1, 2048, None, None, "bf16", "fc"),
    "qwen1.5-7b-e4m3": (4096, 11008, 2, 32, 32, 1, 2048, None, None, "e4m3", "fc"),
    "qwen2-7b-bf16": (3584, 18944, 2, 28, 4, 2, 1100, [1100, 577], "right", "bf16", "fc"),
    "qwen2-7b-e4m3": (3584, 18944, 2, 28, 4, 2, 1100, [1100, 577], "right", "e4m3", "fc"),
    "qwen1.5-0.5b-dense": (1024, 2816, 3, 16, 16, 2, 2048, None, None, "bf16", "ftc"),
    "qwen1.5-0.5b-moe": (1024, 2816, 3, 16, 16, 2, 2048, None, None, "moe", "ftc"),
    "qwen1.5-1.8b": (2048, 5504, 2, 16, 16, 1, 4096, None, None, "bf16", "ftc"),
    "qwen2-0.5b": (896, 4864, 2, 14, 2, 3, 600, [600, 129, 1], "left", "bf16", "ftc"),
    "tiny-hd64-gqa": (256, 384, 2, 4, 2, 2, 100, [100, 37], "right", "bf16", "ftc"),
    "tiny-hd64-e4m3": (256, 384, 2, 4, 2, 2, 100, [100, 37], "right", "e4m3", "fc"),
    "tiny-hd32-moe": (128, 320, 3, 4, 4, 2, 70, [70, 1], "left", "moe", "ftc"),
}


def build(name, seed):
    from llavamod.model.language_model.qwen2_core import MoE, Qwen2Config, Qwen2Model
    H, I, L, nh, nkv, _, _, _, _, path, _ = CASES[name]
    cfg = Qwen2Config(vocab_size=64, hidden_size=H, intermediate_size=I, num_hidden_layers=L, num_attention_heads=nh,
                      num_key_value_heads=nkv, rope_theta=O.THETA, rms_norm_eps=O.EPS)
    m = Qwen2Model(cfg, DEV, BF16)
    if path == "moe":
        for li in range(L)[::2]:
            m.layers[li].mlp = MoE(cfg, m.layers[li].mlp, num_experts=E_MOE, k=TOP_K, capacity_factor=CF, eval_capacity_factor=2.0,
                                   min_capacity=MIN_CAP)
    O.init_decoder_(m, seed)
    if path == "e4m3":
        m.quantize_fp8_()
    return m


def inputs(name, seed):
    """(embeds [B, T, H], mask [B, T] bool or None, real [B, T], lo, hi int32 [B], pos [B, T] int64, planted rows)."""
    H, _, _, _, _, B, T, lengths, side, path, _ = CASES[name]
    real = torch.ones(B, T, dtype=torch.bool, device=DEV)
    lo = torch.zeros(B, dtype=torch.int32, device=DEV)
    hi = torch.full((B,), T, dtype=torch.int32, device=DEV)
    if lengths is not None:
        real.zero_()
        for b, n in enumerate(lengths):
            lo[b], hi[b] = (T - n, T) if side == "left" else (0, n)
            real[b, int(lo[b]):int(hi[b])] = True
    x, rows = O.planted_embeds(B, T, H, real, seed, zero_row=path == "e4m3")
    m = real.to(torch.int64)
    pos = (m.cumsum(1) - 1) * m                         # compact positions over the real rows (the splice plan's)
    return x, (real if lengths is not None else None), real, lo, hi, pos, rows


def moe_noise(model, S, seed):
    from llavamod.model.language_model.qwen2_core import MoE
    g = torch.Generator(device=DEV).manual_seed(seed)
    n = sum(isinstance(l.mlp, MoE) for l in model.layers)
    u = torch.rand(n, S, E_MOE, generator=g, device=DEV).clamp_(min=1e-20, max=1.0 - 1e-7)
    return list((-torch.log(-torch.log(u))).unbind(0))


# ---------------------------------------------------------------------------------------------------
# the replica
# ---------------------------------------------------------------------------------------------------
def check_cache_rows(tag, kc, vc, qkv, B, T, nh, nkv, hd, lo, hi):
    """Cache rows [0, n_b) of every sequence are the k / v columns of its real q|k|v rows [lo_b, hi_b), bit for bit; the head padding
    columns are zero, the rows past n_b untouched (zero)."""
    hp = kc.shape[-1]
    for b in range(B):
        l0, n = int(lo[b]), int(hi[b]) - int(lo[b])
        rows = qkv[b * T + l0:b * T + l0 + n].view(n, nh + 2 * nkv, hd)
        for c, part in ((kc, rows[:, nh:nh + nkv]), (vc, rows[:, nh + nkv:])):
            check_bound(f"{tag} cache rows of sequence {b}", c[b, :, :n, :hd], part.transpose(0, 1))
            assert int(c[b, :, :n, hd:].ne(0).sum()) == 0 and int(c[b, :, n:].ne(0).sum()) == 0, f"{tag}: sequence {b} wrote outside its rows"


def replica(model, x, keep, lo, hi, pos, noise, path, report, cache):
    """_layers' kernel calls for every layer, each stage checked against float64 from the kernel's own previous stage.  cache: also the
    prefill's k / v appends (into the replica's own zeroed caches).  Returns (out [B*T, H], l_aux per MoE layer, q|k|v per layer, log)."""
    from llavamod import kernels as K
    c = model.config
    B, T, H = x.shape
    nh, nkv = c.num_attention_heads, c.num_key_value_heads
    hd, I = H // nh, c.intermediate_size
    n_tab = max(T, min(c.max_position_embeddings, 8192))                        # the table length Qwen2Model.rope keeps
    cos, sin = (t.to(DEV).contiguous() for t in O.R.rope_cache(hd, n_tab, O.THETA, BF16))
    p = pos.reshape(-1).contiguous()
    padded = keep is not None
    pad = (lo, hi) if padded else None
    calls = KernelCalls()
    qkvs, l_auxes = [], []

    def chk(stage, li, got, want, tol=None):
        name = stage if li is None else f"layer {li} {stage}"
        worst = check_bound(name, got, want, tol)
        report[stage] = max(report.get(stage, 0.0), worst)

    def norm(stage, li, xin, w, res, quant):
        """rmsnorm / rmsnorm_quant on (xin, res): the stream against torch's add, rstd against float64, y bit for bit from the kernel's rstd,
        (e4m3) the rows quantised bit for bit, and the composite's bytes."""
        rstd = torch.empty(xin.shape[0], dtype=torch.float32, device=DEV)
        y, s = K._rmsnorm_fwd(xin, res, w, O.EPS, rstd)
        if quant:
            a, s2 = K.rmsnorm_quant(xin, w, O.EPS, res=res)
        else:
            a, s2 = K.rmsnorm(xin, w, O.EPS, res=res, wgrad=None)
        calls.name(f"layer {li} {stage}" if li is not None else stage)
        ref = rmsnorm_reference_fp64(xin, w, O.EPS, res=res, rstd_k=rstd)
        chk(stage + " rstd", li, rstd, ref["rstd"], ref["rstd_tol"])
        chk(stage, li, y, ref["y"])
        chk(stage + " stream", li, s, xin if res is None else xin + res)
        assert same_bits(s2, s), f"{stage}: the stream differs from lmod_rmsnorm_fwd's"
        if not quant:
            assert same_bits(a, y), f"layer {li} {stage}: kernels.rmsnorm differs from lmod_rmsnorm_fwd"
            return a, s2
        q = K.quant_rows(y)
        qr, sr = O.quant_rows_reference(y)
        chk(stage + " quantised rows", li, q.q, qr)
        chk(stage + " quantised rows scale", li, q.scale, sr)
        assert same_bits(a, q), f"layer {li} {stage}: rmsnorm_quant differs from quant_rows(rmsnorm)"
        return a, s2

    def gemm_part(stage, li, got, a, w, bias=None):
        if isinstance(w, K.Fp8Rows):
            chk(stage, li, got, *O.gemm_e4m3_reference_fp64(a, w, bias))
        else:
            chk(stage, li, got, *O.linear_reference_fp64(a, w, bias))

    def silu_part(stage, li, gu):
        act = K.silu_mul(gu)
        r = silu_mul_reference_fp64(gu, I)
        chk(stage, li, act, r["out"], r["out_tol"])
        return act

    with calls:
        kcs = [torch.zeros(B, nkv, T, O.attn_width(hd), dtype=BF16, device=DEV) for _ in model.layers] if cache else None
        vcs = [torch.zeros_like(t) for t in kcs] if cache else None
        lens = torch.zeros(B, dtype=torch.int32, device=DEV)
        stream, branch, moe_i = x.reshape(B * T, H), None, 0
        for li, layer in enumerate(model.layers):
            at, mlp = layer.self_attn, layer.mlp
            fp8 = path == "e4m3"
            xin, res = (stream, None) if branch is None else (branch, stream)
            y, stream = norm("input norm", li, xin, layer.input_layernorm.weight, res, fp8)
            if fp8:
                qkv = K.qkv_rope_fp8(y, at.qkv_weight, at.qkv_bias, cos, sin, p, nh, nkv, hd)
                calls.name(f"layer {li} q|k|v+RoPE")
                chk("q|k|v+RoPE", li, qkv, *O.qkv_rope_e4m3_reference_fp64(y, at.qkv_weight, at.qkv_bias, cos, sin, p, nh, nkv, hd))
            else:
                qkv = K.qkv_rope(y, at.qkv_weight, at.qkv_bias, cos, sin, p, nh, nkv, hd, None, None)
                calls.name(f"layer {li} q|k|v+RoPE")
                chk("q|k|v+RoPE", li, qkv, *qkv_rope_reference_fp64(y, at.qkv_weight, at.qkv_bias, cos, sin, p, nh, nkv, hd, H))
            qkvs.append(qkv)
            if cache:
                if padded:
                    K.kv_append_rows(qkv, B, T, nh, nkv, hd, kcs[li], vcs[li], lo, hi, lens)
                else:
                    K.kv_append(qkv, B, T, nh, nkv, hd, kcs[li], vcs[li], lens)
                calls.name(f"layer {li} cache append")
                check_cache_rows(f"layer {li} replica", kcs[li], vcs[li], qkv, B, T, nh, nkv, hd, lo, hi)
            attn = K.attention(qkv, B, T, nh, nkv, hd, True, None, pad)
            calls.name(f"layer {li} attention")
            want, tol = O.attention_reference_fp64(qkv, B, T, nh, nkv, hd, keep)
            worst = check_attn(f"layer {li} attention", attn, want, tol, T, hd)
            report["attention"] = max(report.get("attention", 0.0), worst)
            del want, tol
            if fp8:
                branch = K.linear_fp8(attn, at.o_fp8)
                calls.name(f"layer {li} o_proj")
                aq = K.quant_rows(attn)
                qr, sr = O.quant_rows_reference(attn)
                chk("o_proj quantised rows", li, aq.q, qr)
                chk("o_proj quantised rows scale", li, aq.scale, sr)
                o = K.gemm_fp8(aq, at.o_fp8)
                gemm_part("o_proj", li, o, aq, at.o_fp8)
                assert same_bits(branch, o), f"layer {li}: linear_fp8 differs from its parts"
            else:
                branch = K.linear(attn, at.o_proj.weight, None, None, None)
                calls.name(f"layer {li} o_proj")
                gemm_part("o_proj", li, branch, attn, at.o_proj.weight)
            y, stream = norm("post-attention norm", li, branch, layer.post_attention_layernorm.weight, stream, fp8)
            if hasattr(mlp, "deepspeed_moe"):
                ds = mlp.deepspeed_moe
                wg, gu, dn = ds.gate.wg.weight, ds.experts.gu_weight, ds.experts.dn_weight
                nz = noise[moe_i]
                moe_i += 1
                out, l_aux, _ = K.moe_forward_nograd(y, stream, wg, gu, dn, nz, CF, MIN_CAP, TOP_K)
                calls.name(f"layer {li} MoE")
                st = K.moe_forward_stages(y, stream, wg, gu, dn, nz, CF, MIN_CAP, TOP_K)
                ref = moe_reference_fp64(y, stream, wg, gu, dn, nz, CF, MIN_CAP, k=st, store=torch.float32)
                moe_report = {}
                check_moe_stages(st, ref, E_MOE, None, moe_report, backward=False)
                for k_, v in moe_report.items():
                    report["MoE " + k_] = max(report.get("MoE " + k_, 0.0), v)
                del ref
                assert same_bits(out, st["out"]) and same_bits(l_aux, st["meta"][0]), f"layer {li}: moe_forward_nograd differs from its stages"
                stream, branch = out, None
                l_auxes.append(l_aux)
            elif fp8:
                branch = K.mlp_fp8(y, mlp.gu_weight, mlp.down_fp8)
                calls.name(f"layer {li} MLP")
                g = K.gemm_fp8(y, mlp.gu_weight)
                gemm_part("gate|up", li, g, y, mlp.gu_weight)
                act = silu_part("SwiGLU", li, g)
                aq = K.quant_rows(act)
                qr, sr = O.quant_rows_reference(act)
                chk("SwiGLU quantised rows", li, aq.q, qr)
                chk("SwiGLU quantised rows scale", li, aq.scale, sr)
                d = K.gemm_fp8(aq, mlp.down_fp8)
                gemm_part("down", li, d, aq, mlp.down_fp8)
                assert same_bits(branch, d), f"layer {li}: mlp_fp8 differs from its parts"
            else:
                branch = K.mlp(y, mlp.gu_weight, mlp.down_proj.weight, None, None)
                calls.name(f"layer {li} MLP")
                g = K.mm_nt(y, mlp.gu_weight)
                gemm_part("gate|up", li, g, y, mlp.gu_weight)
                act = silu_part("SwiGLU", li, g)
                d = K.mm_nt(act, mlp.down_proj.weight)
                gemm_part("down", li, d, act, mlp.down_proj.weight)
                assert same_bits(branch, d), f"layer {li}: mlp differs from its parts"
        xin, res = (stream, None) if branch is None else (branch, stream)
        out, _ = norm("final norm", None, xin, model.norm.weight, res, False)
    return out, l_auxes, qkvs, calls.log


def attach_grad_views(model):
    """A zero gradient view for every decoder tensor _layers looks one up for (what TrainState hands out for trainable parameters)."""
    views = {}
    for layer in model.layers:
        at, mlp = layer.self_attn, layer.mlp
        ts = [layer.input_layernorm.weight, layer.post_attention_layernorm.weight, at.qkv_weight, at.qkv_bias, at.o_proj.weight]
        if hasattr(mlp, "deepspeed_moe"):
            ds = mlp.deepspeed_moe
            ts += [ds.gate.wg.weight, ds.experts.gu_weight, ds.experts.dn_weight]
        else:
            ts += [mlp.gu_weight, mlp.down_proj.weight]
        for t in ts:
            views[id(t)] = torch.zeros_like(t.detach())
    views[id(model.norm.weight)] = torch.zeros_like(model.norm.weight.detach())
    model.grad_views = views


@pytest.mark.parametrize("name", list(CASES))
def test_decoder_stage_by_stage(name):
    from llavamod.model.language_model.qwen2_core import KVCache
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    H, I, L, nh, nkv, B, T, lengths, side, path, entries = CASES[name]
    model = build(name, seed=H + L)
    x, mask, real, lo, hi, pos, rows = inputs(name, seed=T + B)
    noise = moe_noise(model, B * T, seed=7) if path == "moe" else None
    hd = H // nh
    position_ids = pos if mask is not None else None
    report = {}
    with poisoned_uninitialised_memory():
        with torch.no_grad():
            out, l_auxes, qkvs, log = replica(model, x, mask, lo, hi, pos, noise, path, report, cache="c" in entries)
        assert torch.isfinite(out.float()).all()
        no_kv = [e for e in log if e["fn"] not in KV_FNS]
        want = out.view(B, T, H)

        def run(expect, grad_views=False, **kw):
            with KernelCalls(expect=expect, grad_views=grad_views) as prod:
                got, la, _ = model(xin, mask, position_ids, moe_noise=noise, **kw)
            assert prod.count == len(expect), f"the forward makes {prod.count} kernel calls, the replica {len(expect)}"
            assert same_bits(got.detach(), want), "the forward's output differs from the replica's"
            assert len(la) == len(l_auxes) and all(same_bits(a.detach(), b) for a, b in zip(la, l_auxes)), "l_aux"

        xin = x
        if "f" in entries:
            with torch.no_grad():
                run(no_kv)
        if "t" in entries:
            attach_grad_views(model)
            xin = x.clone().requires_grad_(True)
            run(no_kv, grad_views=True)
            model.grad_views = {}
            xin = x
        if "c" in entries:
            cache = KVCache(model, B, T)
            for t in cache.k + cache.v:
                t.zero_()
            with torch.no_grad():
                run(log, cache=cache)
            want_len = (hi - lo).tolist()
            assert cache.lengths == want_len and cache.len.tolist() == want_len
            for li in range(L):
                check_cache_rows(f"layer {li} prefill", cache.k[li], cache.v[li], qkvs[li], B, T, nh, nkv, hd, lo, hi)
    planted = ", ".join(f"{k} row {v}" for k, v in rows.items())
    print(f"\nDECODER {name} ({path}, entry points {entries}; {planted}): max err/bound " +
          ", ".join(f"{k} {v:.3g}" for k, v in report.items()) +
          f"; {time.perf_counter() - t0:.1f} s, peak allocated {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")
