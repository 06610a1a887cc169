"""TEST INFRASTRUCTURE ONLY -- restatement of DeepSpeed 0.9.5's MoE(use_residual=True) (Residual-MoE, SURVEY.md Appendix A "Residual"),
on top of oracle/restated.py's routed layer and tests/moe_top1_oracle.py's top-1 dispatch.

    out     = deepspeed_moe(x)                     # the routed layer, unchanged
    out_mlp = mlp(x)                               # the dense Qwen2MLP the experts were up-cycled from, on every token
    coef    = softmax(coefficient(x), dim=-1)      # Linear(H, 2) with a bias, [S, 2]
    out     = out * coef[..., 0:1] + out_mlp * coef[..., 1:]

In bf16 every line rounds once: z = bf16(x Wc^T + b), c = bf16(softmax_fp32(z)), out = bf16(bf16(moe c0) + bf16(mlp c1)); the layer then
adds bf16(residual + out).  A layer is residual when the state dict holds ``<layer>.mlp.coefficient.weight``."""
import contextlib
import math

import torch
import torch.nn.functional as F

from oracle import restated as R
from tests import moe_top1_oracle as O1

u24 = 2.0 ** -24


def residual_mix(moe, mlp_out, x, wc, bc):
    """The last two DeepSpeed lines, literally (torch rounds each op to the tensors' dtype).  Returns (out, coef)."""
    coef = F.softmax(F.linear(x, wc, bc), dim=-1)
    return moe * coef[..., 0:1] + mlp_out * coef[..., 1:], coef


def moe_layer(sd, pre, cfg, x, noise, record=None):
    """O1.moe_layer (top-1 / top-2 by cfg.top_k), plus the residual MLP and the mix when the layer has a coefficient."""
    out, l_aux, counts = O1.moe_layer(sd, pre, cfg, x, noise, record)
    base = pre[:-len("deepspeed_moe.")]
    if base + "coefficient.weight" not in sd:
        return out, l_aux, counts
    mixed, coef = residual_mix(out, R.mlp(sd, base + "mlp.", x), x, sd[base + "coefficient.weight"], sd[base + "coefficient.bias"])
    if record is not None:
        record[-1]["coef"] = coef.reshape(-1, 2)
    return mixed, l_aux, counts


@contextlib.contextmanager
def dispatching_moe_layer():
    old = R.moe_layer
    R.moe_layer = moe_layer
    try:
        yield
    finally:
        R.moe_layer = old


def llava_forward(sd, cfg, clip_cfg, input_ids, attention_mask, labels, images, moe_noise=None, record=None):
    with dispatching_moe_layer():
        return R.llava_forward(sd, cfg, clip_cfg, input_ids, attention_mask, labels, images, moe_noise, record)


# ---- float64 references of the two mix kernels, each stage from the kernel's own inputs, with element-wise bounds --------------------
def _acc_terms(H):
    """fp32 roundings on the way of one warp's dot product over H: 8 FMAs per 16-byte vector per lane, five shuffle levels, the bias."""
    return 8 * math.ceil(H / 256) + 7


def mix_reference_fp64(x, moe, mlp_out, res, wc, bc, coef):
    """-> dict name -> (want, tol) for 'coef' (float64 bound) and 'out' (bit exact, tol None, from the kernel's coef)."""
    S, H = x.shape
    xd, wd = x.double(), wc.double()
    z = xd @ wd.t() + (bc.double() if bc is not None else 0.0)
    maj = xd.abs() @ wd.abs().t() + (bc.double().abs() if bc is not None else 0.0)
    dz = 2.0 ** -8 * z.abs() + (1 + 2.0 ** -8) * _acc_terms(H) * u24 * maj         # |bf16(z_kernel) - z|
    c = torch.softmax(z, dim=-1)
    c_tol = 2.0 ** -8 * c + (1 + 2.0 ** -8) * (c[:, :1] * c[:, 1:] * (dz[:, :1] + dz[:, 1:]) + 8 * u24 * c)
    k0, k1 = coef[:, :1].float(), coef[:, 1:].float()
    bf = torch.bfloat16
    out = (res.float() + ((moe.float() * k0).to(bf).float() + (mlp_out.float() * k1).to(bf).float()).to(bf).float()).to(bf)
    return dict(coef=(c, c_tol), out=(out, None))


def mix_bwd_reference_fp64(g, x, moe, mlp_out, coef, wc, dz_k, old_w=None, old_b=None):
    """Backward stages from the kernel's inputs: d_moe / d_mlp bit exact; dz in float64; the dx term, dWc and db from the kernel's dz."""
    S, H = g.shape
    bf = torch.bfloat16
    k0, k1 = coef[:, :1].float(), coef[:, 1:].float()
    ref = dict(d_moe=((g.float() * k0).to(bf), None), d_mlp=((g.float() * k1).to(bf), None))
    gd, c = g.double(), coef.double()
    dc = torch.stack([(gd * moe.double()).sum(1), (gd * mlp_out.double()).sum(1)], 1)
    e = _acc_terms(H) * u24 * torch.stack([(gd.abs() * moe.double().abs()).sum(1), (gd.abs() * mlp_out.double().abs()).sum(1)], 1)
    dot = (c * dc).sum(1, keepdim=True)
    dz = c * (dc - dot)
    ce = (c * e).sum(1, keepdim=True)
    mag = c * (dc.abs() + (c * dc.abs()).sum(1, keepdim=True))
    ref["dz"] = (dz, c * (e + ce) + 6 * u24 * mag + 2.0 ** -140)
    zk, wd = dz_k.double(), wc.double()
    dx = zk @ wd
    ref["dx"] = (dx, 2.0 ** -8 * dx.abs() + (1 + 2.0 ** -8) * 2 * u24 * (zk.abs() @ wd.abs()))
    per = -(-S // 128)
    xd = x.double()
    for name, a, a_abs, old in (("dwc", zk.t() @ xd, zk.abs().t() @ xd.abs(), old_w), ("dbc", zk.sum(0), zk.abs().sum(0), old_b)):
        o = old.double() if old is not None else torch.zeros_like(a)
        want = a + o
        ref[name] = (want, 2.0 ** -8 * want.abs() + (1 + 2.0 ** -8) * (per + 128 + 2) * u24 * (a_abs + o.abs()))
    return ref
