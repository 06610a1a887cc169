"""Residual-MoE (DeepSpeed MoE(use_residual=True), --use_residual True) on the CPU: the oracle of tests/moe_residual_oracle.py against a
literal transcription of DeepSpeed's forward in torch bf16 (forward and autograd, top-2 and top-1, a token whose choices were all dropped),
a DeepSpeed pin that skips while DeepSpeed is absent, the flag and config round trip, the state-dict layout, the requires_grad rules of
the two initialize_moe_modules paths and the optimizer groups."""
import importlib
import math
import os
import sys
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import restated as R
from tests import moe_residual_oracle as O
from tests import moe_top1_oracle as O1

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
bf = torch.bfloat16
H, I, E = 32, 48, 4


class _MLP(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.gate_proj = torch.nn.Linear(H, I, bias=False)
        self.up_proj = torch.nn.Linear(H, I, bias=False)
        self.down_proj = torch.nn.Linear(I, H, bias=False)

    def forward(self, x):
        return self.down_proj(F.silu(self.gate_proj(x)) * self.up_proj(x))


class _Routed(torch.nn.Module):
    """The routed layer (deepspeed_moe) over its own parameters, through the restated gating (already pinned on its own)."""

    def __init__(self, k, noise, cf):
        super().__init__()
        self.wg = torch.nn.Parameter(torch.randn(E, H) * 0.5)
        self.experts = torch.nn.ModuleList([_MLP() for _ in range(E)])
        self.k, self.noise, self.cf = k, noise, cf

    def sd(self, pre):
        d = {pre + "gate.wg.weight": self.wg}
        for e, m in enumerate(self.experts):
            for n in ("gate_proj", "up_proj", "down_proj"):
                d[pre + "experts.deepspeed_experts.%d.%s.weight" % (e, n)] = getattr(m, n).weight
        return d

    def forward(self, x):
        cfg = types.SimpleNamespace(capacity_factor=self.cf, min_capacity=0, num_experts=E, top_k=self.k)
        return O1.moe_layer(self.sd("p."), "p.", cfg, x, self.noise)


class LiteralResidualMoE(torch.nn.Module):
    """deepspeed.moe.layer.MoE.forward with use_residual=True, line by line."""

    def __init__(self, k, noise, cf):
        super().__init__()
        self.deepspeed_moe = _Routed(k, noise, cf)
        self.mlp = _MLP()
        self.coefficient = torch.nn.Linear(H, 2)

    def forward(self, hidden_states):
        output, l_aux, exp_counts = self.deepspeed_moe(hidden_states)
        output_mlp = self.mlp(hidden_states)
        coef = self.coefficient(hidden_states)
        coef = torch.nn.functional.softmax(coef, dim=-1)
        output = output * coef[..., 0:1] + output_mlp * coef[..., 1:]
        return output, l_aux, exp_counts


def _sd_of(m):
    d = m.deepspeed_moe.sd("L.mlp.deepspeed_moe.")
    for n in ("gate_proj", "up_proj", "down_proj"):
        d["L.mlp.mlp.%s.weight" % n] = getattr(m.mlp, n).weight
    d["L.mlp.coefficient.weight"], d["L.mlp.coefficient.bias"] = m.coefficient.weight, m.coefficient.bias
    return d


@pytest.mark.parametrize("k", [2, 1])
def test_oracle_equals_literal_deepspeed_forward_and_autograd(k):
    S = 96
    torch.manual_seed(k)
    g = torch.Generator().manual_seed(10 + k)
    noise = torch.rand(S, E, generator=g) if k == 1 else R.gumbel_noise((S, E), g)
    cf = 0.5
    m = LiteralResidualMoE(k, noise, cf)
    m.deepspeed_moe.wg.data[:, 0] = torch.tensor([4.0, 3.0, -4.0, -4.0])          # experts 0 and 1 overflow: some tokens lose every choice
    m.to(bf)
    m.deepspeed_moe.wg.data = m.deepspeed_moe.wg.data.float()                        # TopKGate keeps wg in fp32
    x = torch.randn(S, H, generator=g)
    x[:, 0] = 2.0 + x[:, 0].abs()
    x = x.to(bf)
    x1, x2 = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    out, l_aux, _ = m(x1)
    cfg = types.SimpleNamespace(capacity_factor=cf, min_capacity=0, num_experts=E, top_k=k)
    sd = {n: t.detach().clone().requires_grad_(True) for n, t in _sd_of(m).items()}
    rec = []
    out2, l_aux2, _ = O.moe_layer(sd, "L.mlp.deepspeed_moe.", cfg, x2, noise, rec)
    assert out.dtype == bf and torch.equal(out, out2) and torch.equal(l_aux, l_aux2)
    # tokens whose choices were all dropped: only c1 * mlp passes
    lost = ~rec[0]["keep1"] & ~rec[0]["keep2"]
    assert bool(lost.any())
    coef = rec[0]["coef"]
    mlp = m.mlp(x)
    want = (mlp[lost] * coef[lost][:, 1:]).to(bf)
    assert torch.equal(out2[lost].detach(), (torch.zeros_like(want) + want).detach())
    # the bf16 rounding chain: z, c, the two products and their sum each round once
    z = F.linear(x, m.coefficient.weight, m.coefficient.bias)
    c = torch.softmax(z.float(), -1).to(bf)
    assert torch.equal(coef.detach(), c)
    moe_out, _, _ = m.deepspeed_moe(x)
    chain = ((moe_out.float() * c[:, :1].float()).to(bf).float() + (mlp.float() * c[:, 1:].float()).to(bf).float()).to(bf)
    assert torch.equal(out.detach(), chain)
    # autograd: the same gradient for every parameter and for x
    dout = torch.randn(S, H, generator=g).to(bf)
    ((out.float() * dout.float()).sum() + 0.3 * l_aux.float()).backward()
    ((out2.float() * dout.float()).sum() + 0.3 * l_aux2.float()).backward()
    assert torch.equal(x1.grad, x2.grad)
    for n, p in _sd_of(m).items():
        assert p.grad is not None and torch.equal(p.grad, sd[n].grad), n


def _import_deepspeed_moe():
    ref = os.path.join(ROOT, "baseline", "_ref")
    if os.path.isdir(ref) and ref not in sys.path:
        sys.path.append(ref)
    try:
        sm = importlib.import_module("deepspeed.moe.sharded_moe")
        from deepspeed.moe.layer import MoE
        return sm, MoE
    except Exception as e:                                  # noqa: BLE001 -- any import failure means "no usable DeepSpeed here"
        pytest.skip("deepspeed is not importable here (%s: %s): the Residual-MoE oracle stays 'parity unpinned'" % (type(e).__name__, e))


def test_residual_oracle_equals_deepspeed_moe_module():
    """deepspeed.moe.layer.MoE(use_residual=True) on CPU, ep_size 1, same weights and noise, against the oracle's residual layer."""
    sm, MoE = _import_deepspeed_moe()
    S = 96
    torch.manual_seed(0)
    try:
        moe = MoE(H, expert=_MLP(), num_experts=E, ep_size=1, k=2, capacity_factor=1.5, eval_capacity_factor=2.0, min_capacity=0,
                  use_residual=True)
    except Exception as e:                                  # noqa: BLE001 -- needs an initialised process group in some versions
        pytest.skip("deepspeed MoE could not be constructed without a distributed backend: %s" % e)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, S, H, generator=g)
    noise = R.gumbel_noise((S, E), g)
    orig = sm.gumbel_rsample
    sm.gumbel_rsample = lambda shape, device=None: noise
    try:
        out, l_aux, counts = moe(x)
    finally:
        sm.gumbel_rsample = orig
    sd = {"m." + k: v.detach() for k, v in moe.state_dict().items()}
    cfg = types.SimpleNamespace(capacity_factor=1.5, min_capacity=0, num_experts=E, top_k=2)
    y, la, _ = O.moe_layer(sd, "m.deepspeed_moe.", cfg, x, noise)
    torch.testing.assert_close(out, y, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(l_aux, la, rtol=1e-6, atol=1e-7)


# ---------------------------------------------------------------------------------------------------------------------------------
# host side: flags, config, layout, requires_grad, optimizer groups (the model builds on the CPU; nothing here launches a kernel)
# ---------------------------------------------------------------------------------------------------------------------------------
def test_flag_parses_and_round_trips_through_config_moe(tmp_path):
    from llavamod.config.args import AlignArguments, DataArguments, ModelArguments, TrainingArguments, parse_args_into_dataclasses
    from llavamod.model.language_model.llava_qwen1_5_moe import LLaVAMoDQwen1_5Config
    argv = "--use_residual True --moe_enable True --num_experts 4 --output_dir /tmp/o".split()
    m, _, _, _ = parse_args_into_dataclasses((ModelArguments, DataArguments, TrainingArguments, AlignArguments), argv)
    assert m.use_residual is True
    m2, _, _, _ = parse_args_into_dataclasses((ModelArguments, DataArguments, TrainingArguments, AlignArguments),
                                              "--moe_enable True --output_dir /tmp/o".split())
    assert m2.use_residual is False
    student = _student(use_residual=True)
    assert student.config.moe["use_residual"] is True
    student.config.save_pretrained(str(tmp_path))
    cfg = LLaVAMoDQwen1_5Config.from_pretrained(str(tmp_path))
    assert cfg.moe["use_residual"] is True


def _student(use_residual=True, train_modules=None, top_k=2):
    from llavamod.model import synthetic as S
    from llavamod.model.language_model.llava_qwen1_5_moe import LLaVAMoDQwen1_5Config, LLaVAMoDQwen1_5ForCausalLM
    d, _ = S._common_cfg(dict(S.ARCH["tiny"], vocab_size=512), "tiny")
    torch.manual_seed(0)
    m = LLaVAMoDQwen1_5ForCausalLM(LLaVAMoDQwen1_5Config(**d), device="cpu", dtype=bf)
    kw = {} if train_modules is None else dict(train_modules=train_modules)
    m.initialize_moe_modules(S.moe_args(use_residual=use_residual, top_k=top_k, **kw))
    return m


def test_state_dict_layout_and_the_dense_module_is_kept():
    m = _student()
    p = "model.layers.0.mlp."
    keys = [n for n in m.state_dict() if n.startswith(p)]
    want = ([p + "deepspeed_moe.gate.wg.weight"] + [p + "deepspeed_moe.experts.deepspeed_experts.%d.%s.weight" % (e, w)
                                                    for e in range(4) for w in ("gate_proj", "up_proj", "down_proj")]
            + [p + "mlp.%s.weight" % w for w in ("gate_proj", "up_proj", "down_proj")] + [p + "coefficient.weight", p + "coefficient.bias"])
    assert keys == want
    sd = m.state_dict()
    assert sd[p + "coefficient.weight"].shape == (2, 128) and sd[p + "coefficient.bias"].shape == (2,)
    assert sd[p + "coefficient.weight"].dtype == bf and sd[p + "coefficient.bias"].dtype == bf
    assert sd[p + "mlp.gate_proj.weight"].shape == (256, 128) and sd[p + "mlp.down_proj.weight"].shape == (128, 256)
    layer = m.model.layers[0].mlp
    assert layer.use_residual and isinstance(layer.mlp, type(m.model.layers[1].mlp))
    for e in range(4):                                       # the experts are copies of the kept dense module
        ex = layer.deepspeed_moe.experts.deepspeed_experts[e]
        assert torch.equal(ex.gate_proj.weight, layer.mlp.gate_proj.weight) and torch.equal(ex.down_proj.weight, layer.mlp.down_proj.weight)
    # nn.Linear's default init: |W| <= 1/sqrt(H) (kaiming-uniform, a = sqrt 5), |b| <= 1/sqrt(H)
    lim = 1 / math.sqrt(128) * (1 + 2 ** -8)
    assert float(layer.coefficient.weight.float().abs().max()) <= lim and float(layer.coefficient.bias.float().abs().max()) <= lim
    plain = _student(use_residual=False)
    kp = list(plain.state_dict())
    assert not any(".mlp.mlp." in n or "coefficient" in n for n in kp)
    assert [n for n in sd if n in kp] == kp


def test_requires_grad_of_the_two_initialize_paths():
    from llavamod.model import synthetic as S
    from llavamod.model.language_model.llava_qwen1_5_moe import LLaVAMoDQwen1_5ForCausalLMFineTune
    p = "model.layers.0.mlp."
    # dense -> sparse (align_train): frozen by name BEFORE wrapping, so the new coefficient trains and mlp.mlp.* keeps its dense name's rule
    m = _student(train_modules=S.TRAIN_MODULES)
    rg = {n: q.requires_grad for n, q in m.named_parameters()}
    assert rg[p + "coefficient.weight"] and rg[p + "coefficient.bias"]
    assert rg[p + "mlp.gate_proj.weight"] and rg[p + "mlp.down_proj.weight"]
    assert not rg["model.layers.0.self_attn.q_proj.weight"]
    m_att = _student(train_modules=["self_attn"])
    rg = {n: q.requires_grad for n, q in m_att.named_parameters()}
    # modules created by the wrap (the router, the coefficient) train whatever the names say; the dense module keeps its frozen state
    assert rg[p + "coefficient.weight"] and rg[p + "deepspeed_moe.gate.wg.weight"] and not rg[p + "mlp.gate_proj.weight"]
    # the preference stage (FineTune): re-decided by name over the wrapped names, and "mlp.coefficient.*" matches none of the shell's
    ft = LLaVAMoDQwen1_5ForCausalLMFineTune(m.config, device="cpu", dtype=bf)
    assert ft.model.layers[0].mlp.use_residual
    ft.initialize_moe_modules(types.SimpleNamespace(train_modules=list(S.TRAIN_MODULES)))
    rg = {n: q.requires_grad for n, q in ft.named_parameters()}
    assert not rg[p + "coefficient.weight"] and not rg[p + "coefficient.bias"]
    assert rg[p + "mlp.gate_proj.weight"] and rg[p + "deepspeed_moe.gate.wg.weight"]
    ft.initialize_moe_modules(types.SimpleNamespace(train_modules=list(S.TRAIN_MODULES) + ["coefficient"]))
    rg = {n: q.requires_grad for n, q in ft.named_parameters()}
    assert rg[p + "coefficient.weight"] and rg[p + "coefficient.bias"]


def test_optimizer_groups_and_arena_membership():
    from llavamod.model import synthetic as S
    from llavamod.train.engine import TrainState, param_group_of
    m = _student(train_modules=S.TRAIN_MODULES)
    p = "model.layers.0.mlp."
    assert param_group_of(p + "coefficient.bias", False, False) == (False, True)
    assert param_group_of(p + "coefficient.weight", False, False) == (False, False)
    assert param_group_of(p + "mlp.gate_proj.weight", False, False) == (False, False)
    ts = TrainState(m)
    named = dict(m.named_parameters())
    segs = dict(((k, (a, b)) for k, a, b in ts.segments["16"]))
    base = ts.w16.data_ptr()

    def seg_of(n):
        off = (named[n].data_ptr() - base) // 2
        return [k for k, (a, b) in segs.items() if a <= off < b]

    assert seg_of(p + "coefficient.bias") == [(False, True)]
    for n in (p + "coefficient.weight", p + "mlp.gate_proj.weight", p + "mlp.up_proj.weight", p + "mlp.down_proj.weight"):
        assert seg_of(n) == [(False, False)], n
    gv = m.get_model().grad_views
    layer = m.model.layers[0].mlp
    for t in (layer.mlp.gu_weight, layer.mlp.down_proj.weight, layer.coefficient.weight, layer.coefficient.bias):
        assert id(t) in gv
    assert named[p + "coefficient.weight"].grad is not None and named[p + "coefficient.weight"].grad.data_ptr() >= ts.g16.data_ptr()
