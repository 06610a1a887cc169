"""Float64 restatement of the Qwen2 decoder stack (Qwen2Model._layers in llavamod/model/language_model/qwen2_core.py) stage by stage,
with the element-wise bound of each stage's kernel, and the weights and planted inputs the exact decoder tests run with.

Each stage reference takes its input as given (on the GPU: the kernel's own output of the stage before), so its bound covers the
arithmetic of one stage.  Every bound is one of tests/helpers.py or tests/test_gemm_fp8_gpu.py:
  input / post-attention / final norm   helpers.rmsnorm_reference_fp64: s = bf16(x + res) and y bit for bit from the kernel's rstd
  q|k|v + bias + RoPE                   helpers.qkv_rope_reference_fp64 (bf16 GEMM, reduction length H)
  e4m3 q|k|v + bias + RoPE              helpers.rope_of_product_fp64 on the e4m3 GEMM bound below
  causal attention with key padding     helpers.attn_reference_fp64 (GQA by index, heads zero-padded to the kernel's width)
  o_proj, gate|up, down                 the bf16 GEMM bound helpers._gemm_tol (clip_oracle.linear_reference_fp64)
  SwiGLU                                helpers.silu_mul_reference_fp64
  e4m3 row quantiser                    bit for bit against fp8_oracle.quant_rows
  e4m3 GEMMs                            2^-8 |ref| + ACC_EPS sum |a||w| of the dequantised operands (test_gemm_fp8_gpu.py)
The MoE layer is checked with helpers.moe_reference_fp64 / check_moe_stages from the kernels' own routing record.

lm_chain_fp64 runs the same stage references on their own float64 outputs; tests/test_decoder_reference.py pins that chain against
oracle.restated.lm_forward, so a stage reference that computes the wrong thing cannot pass unnoticed."""
import math

import torch
import torch.nn.functional as F

from oracle import restated as R
from tests import fp8_oracle as Q
from tests.clip_oracle import linear_reference_fp64
from tests.helpers import ELEM_ABS_FLOOR, attn_reference_fp64, qkv_rope_reference_fp64, rmsnorm_reference_fp64, rope_of_product_fp64
from tests.test_gemm_fp8_gpu import ACC_EPS

F64 = torch.float64
EPS = 1e-6                # rms_norm_eps of every Qwen1.5 / Qwen2 config.json
THETA = 1e6               # rope_theta of the same configs


def attn_width(hd):
    """The head width the attention kernels run (kernels.attn_head_dim, stated here so the reference does not lean on it)."""
    return hd if hd in (64, 128) else (64 if hd < 64 else 128)


def attention_reference_fp64(qkv, B, T, nh, nkv, hd, keep=None):
    """Causal attention of the fused [B*T, (nh + 2 nkv) hd] q|k|v rows with key padding keep [B, T] bool (None: every key), scale hd^-0.5
    -> (o [B*T, nh hd], bound).  The heads are zero-padded to the kernel's width, at which the bound is taken (the extra score terms are
    exact zeros)."""
    hp = attn_width(hd)
    rows = qkv.shape[0]
    x = qkv.to(F64)
    if hp != hd:
        x = F.pad(x.view(rows, nh + 2 * nkv, hd), (0, hp - hd)).reshape(rows, (nh + 2 * nkv) * hp)
    ref = attn_reference_fp64(x, B, T, nh, nkv, hp, True, hd ** -0.5, keep=keep)

    def unpad(t):
        return t if hp == hd else t.view(rows, nh, hp)[:, :, :hd].reshape(rows, nh * hd)
    return unpad(ref["o"]), unpad(ref["o_tol"])


def gemm_e4m3_reference_fp64(a, w, bias=None):
    """a (Fp8Rows [M, K]) x w (Fp8Rows [N, K])^T (+ bias) from the dequantised operands -> (want, tol), tol = 2^-8 |want| + ACC_EPS
    (|a| |w|^T + |bias|): the bf16 store and the e4m3 accumulator with its promotion (tests/test_gemm_fp8_gpu.py)."""
    A, W = Q.dequant(a.q, a.scale), Q.dequant(w.q, w.scale)
    want, maj = A @ W.t(), A.abs() @ W.abs().t()
    if bias is not None:
        want, maj = want + bias.to(F64), maj + bias.to(F64).abs()
    return want, 2.0 ** -8 * want.abs() + ACC_EPS * maj + ELEM_ABS_FLOOR


def qkv_rope_e4m3_reference_fp64(a, w, bias, cos, sin, pos, nh, nkv, hd):
    """lmod_gemm_e4m3_qkv_rope (bit-identical to lmod_gemm_e4m3 + lmod_rope): the e4m3 GEMM bound, then the rotation of
    helpers.qkv_rope_reference_fp64."""
    P, E = gemm_e4m3_reference_fp64(a, w, bias)
    return rope_of_product_fp64(P, E, cos, sin, pos, nh, nkv, hd)


def quant_rows_reference(x):
    """fp8_oracle.quant_rows of bf16 rows x on the CPU -> (q, scale) on x's device."""
    q, s = Q.quant_rows(x)
    return q.to(x.device), s.to(x.device)


def rmsnorm_fp64(x, w, eps):
    """Qwen2RMSNorm in float64: x rstd w, rstd from helpers.rmsnorm_reference_fp64."""
    return x * rmsnorm_reference_fp64(x, w, eps)["rstd"][:, None] * w.to(F64)


def rope_tables_fp64(hd, n, theta):
    """The RoPE tables in float64 (oracle.restated.rope_cache, as lm_forward builds them for float64 inputs)."""
    return R.rope_cache(hd, n, theta, F64)


def lm_chain_fp64(sd, c, x, keep, pos, pre="model."):
    """The stage references above, each on the previous one's float64 output, for a dense decoder: the final-normed hidden [B, T, H].
    sd: a Qwen2Model state dict with the checkpoint's per-projection keys (prefixed by `pre`), c: an oracle.restated.LMCfg, x [B, T, H]
    inputs_embeds, keep [B, T] bool or None, pos [B, T] int64 RoPE positions."""
    def g(k):
        return sd[pre + k].to(F64)
    B, T, H = x.shape
    nh, nkv, hd, I = c.heads, c.kv_heads, c.head_dim, c.inter
    cos, sin = rope_tables_fp64(hd, int(pos.max()) + 1, c.rope_theta)
    p = pos.reshape(-1)
    h = x.reshape(B * T, H).to(F64)
    for i in range(c.layers):
        def lw(k):
            return g(f"layers.{i}.{k}")
        y = rmsnorm_fp64(h, lw("input_layernorm.weight"), c.eps)
        a = "self_attn."
        w = torch.cat([lw(a + f"{m}_proj.weight") for m in "qkv"])
        b = torch.cat([lw(a + f"{m}_proj.bias") for m in "qkv"])
        qkv, _ = qkv_rope_reference_fp64(y, w, b, cos, sin, p, nh, nkv, hd, H)
        o, _ = attention_reference_fp64(qkv, B, T, nh, nkv, hd, keep)
        h = h + linear_reference_fp64(o, lw(a + "o_proj.weight"))[0]
        y = rmsnorm_fp64(h, lw("post_attention_layernorm.weight"), c.eps)
        gu, _ = linear_reference_fp64(y, torch.cat([lw("mlp.gate_proj.weight"), lw("mlp.up_proj.weight")]))
        act = F.silu(gu[:, :I]) * gu[:, I:]
        h = h + linear_reference_fp64(act, lw("mlp.down_proj.weight"))[0]
    return rmsnorm_fp64(h, g("norm.weight"), c.eps).view(B, T, H)


# ---------------------------------------------------------------------------------------------------
# weights and planted inputs
# ---------------------------------------------------------------------------------------------------
OUTLIER_CH = 5            # the "massive activation" channel of the residual stream: +-1500..2500 in every real row
OUTLIER = 2000.0
TINY_ROW = 1e-4           # a row of |x| ~ 1e-4: mean(x^2) ~ 1e-8, so eps = 1e-6 sets its rstd


def init_decoder_(model, seed):
    """Fill a Qwen2Model's decoder weights in place: linears N(0, 1/K), biases N(0, 0.1^2), norm weights 1 + 0.1 N(0, 1); every expert of
    an MoE layer its own N(0, 1/K) draw (up-cycled copies would make a misrouted token invisible).  Seeded, on the model's device."""
    dev = model.embed_tokens.weight.device
    gen = torch.Generator(device=dev).manual_seed(seed)

    def rn(*shape, scale=1.0):
        return torch.randn(*shape, generator=gen, device=dev, dtype=torch.float32) * scale

    H = model.config.hidden_size
    with torch.no_grad():
        model.norm.weight.copy_(1 + 0.1 * rn(H))
        for layer in model.layers:
            at, mlp = layer.self_attn, layer.mlp
            at.qkv_weight.copy_(rn(*at.qkv_weight.shape, scale=1 / math.sqrt(H)))
            at.qkv_bias.copy_(rn(*at.qkv_bias.shape, scale=0.1))
            at.o_proj.weight.copy_(rn(*at.o_proj.weight.shape, scale=1 / math.sqrt(at.o_proj.weight.shape[1])))
            layer.input_layernorm.weight.copy_(1 + 0.1 * rn(H))
            layer.post_attention_layernorm.weight.copy_(1 + 0.1 * rn(H))
            if hasattr(mlp, "deepspeed_moe"):
                ex = mlp.deepspeed_moe.experts
                ex.gu_weight.copy_(rn(*ex.gu_weight.shape, scale=1 / math.sqrt(H)))
                ex.dn_weight.copy_(rn(*ex.dn_weight.shape, scale=1 / math.sqrt(ex.dn_weight.shape[2])))
            else:
                mlp.gu_weight.copy_(rn(*mlp.gu_weight.shape, scale=1 / math.sqrt(H)))
                mlp.down_proj.weight.copy_(rn(*mlp.down_proj.weight.shape, scale=1 / math.sqrt(mlp.down_proj.weight.shape[1])))
    return model


def planted_embeds(B, T, H, real, seed, zero_row=False, device="cuda"):
    """inputs_embeds [B, T, H] bf16: N(0, 1) rows with the outlier channel OUTLIER_CH at +-(0.75..1.25) OUTLIER, one near-zero row (sample
    0, its second real row; |x| ~ TINY_ROW, no outlier) and with zero_row an all-zero row (sample B - 1, its last real row).  real: [B, T]
    bool, the real tokens.  Returns (embeds, {name: (b, t)} of the planted rows)."""
    gen = torch.Generator(device=device).manual_seed(seed)
    x = torch.randn(B, T, H, generator=gen, device=device)
    sign = torch.randint(0, 2, (B, T), generator=gen, device=device) * 2 - 1
    x[:, :, OUTLIER_CH] = OUTLIER * sign * (0.75 + 0.5 * torch.rand(B, T, generator=gen, device=device))
    rows = {}
    idx0 = real[0].nonzero()[:, 0].tolist()
    t = idx0[min(1, len(idx0) - 1)]
    x[0, t] = TINY_ROW * torch.randn(H, generator=gen, device=device)
    rows["near-zero"] = (0, t)
    if zero_row:
        t = real[B - 1].nonzero()[-1, 0].item()
        x[B - 1, t] = 0
        rows["all-zero"] = (B - 1, t)
    return x.to(torch.bfloat16), rows
