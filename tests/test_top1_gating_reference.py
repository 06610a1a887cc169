"""Top-1 MoE routing on the CPU: the restated top1gating (tests/moe_top1_oracle.py) against an independent token-by-token simulation of
random token selection, its pin against a real DeepSpeed (skipped while DeepSpeed is absent), and the host side of --top_k_experts 1."""
import importlib
import os
import sys

import pytest
import torch

from oracle import restated as R
from tests import moe_top1_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def planted_logits(idx1, E, seed):
    """fp32 logits whose softmax argmax is idx1[s] (margin 3 over random values in [0, 1))."""
    g = torch.Generator().manual_seed(seed)
    lg = torch.rand(len(idx1), E, generator=g)
    lg[torch.arange(len(idx1)), torch.as_tensor(idx1)] += 3.0
    return lg


def skewed_idx(S, E, counts, seed):
    idx = torch.cat([torch.full((n,), e, dtype=torch.long) for e, n in enumerate(counts)])
    assert idx.numel() == S
    return idx[torch.randperm(S, generator=torch.Generator().manual_seed(seed))]


def assert_matches_simulation(logits, u, cf, mc):
    o = O.top1gating(logits, u, cf, mc)
    idx1, keep, slot, w, l_aux, counts, C = O.simulate_top1(logits, u, cf, mc)
    assert o["capacity"] == C
    assert o["idx1"].tolist() == idx1
    assert o["keep1"].tolist() == keep
    assert o["slot1"][o["keep1"]].tolist() == [slot[s] for s in range(len(keep)) if keep[s]]
    assert o["exp_counts"].tolist() == counts
    torch.testing.assert_close(o["g1"], torch.tensor(w), rtol=0, atol=0)
    torch.testing.assert_close(o["l_aux"].double(), torch.tensor(l_aux, dtype=torch.float64), rtol=2e-6, atol=1e-9)
    # the combine tensor holds exactly the kept tokens' raw gates at their seats
    S, E = logits.shape
    assert int(o["dispatch"].sum()) == sum(keep)
    for s in range(S):
        if keep[s]:
            assert float(o["combine"][s, idx1[s], slot[s]]) == w[s]
    # per expert: at most C seats, 0 .. kept-1 in token order
    for e in range(E):
        seats = [slot[s] for s in range(S) if keep[s] and idx1[s] == e]
        assert seats == list(range(min(counts[e], C)))
    return o


@pytest.mark.parametrize("S,E,cf,mc,counts", [
    (64, 2, 1.0, 0, [40, 24]),                    # expert 0 over-full, expert 1 under-full
    (333, 4, 1.5, 0, [200, 60, 40, 33]),
    (2048, 4, 1.5, 0, [1600, 200, 120, 128]),     # config 2: C = 768
    (500, 8, 1.0, 0, [200, 100, 60, 50, 40, 30, 20, 0]),
    (100, 8, 0.5, 30, [60, 20, 10, 5, 3, 2, 0, 0]),   # min_capacity 30 above ceil(100/8 * 0.5) = 7
    (17, 4, 2.0, 0, [17, 0, 0, 0]),
])
def test_top1gating_equals_token_by_token_simulation(S, E, cf, mc, counts):
    idx = skewed_idx(S, E, counts, S + E)
    logits = planted_logits(idx, E, S)
    u = torch.rand(S, E, generator=torch.Generator().manual_seed(S * 7 + E))
    o = assert_matches_simulation(logits, u, cf, mc)
    assert torch.equal(o["idx1"], idx)


def test_ties_straddling_the_cut_keep_the_lower_index():
    S, E, cf = 40, 2, 1.0                          # C = 20
    idx = torch.tensor([0] * 30 + [1] * 10)
    logits = planted_logits(idx, E, 1)
    u = torch.rand(S, E, generator=torch.Generator().manual_seed(2)) * 0.5
    tied = [3, 11, 17, 25, 29]                    # five equal keys; 17 larger keys above them, so 3 of the 5 are kept
    big = [s for s in range(30) if s not in tied][:17]
    for s in big:
        u[s, 0] = 0.9
    for s in tied:
        u[s, 0] = 0.625
    o = assert_matches_simulation(logits, u, cf, 0)
    kept = o["keep1"].tolist()
    assert [kept[s] for s in tied] == [True, True, True, False, False]


def test_a_zero_uniform_in_an_under_full_expert_is_kept():
    S, E = 32, 4
    idx = skewed_idx(S, E, [20, 6, 3, 3], 5)
    logits = planted_logits(idx, E, 3)
    u = torch.rand(S, E, generator=torch.Generator().manual_seed(4))
    s0 = int((idx == 1).nonzero()[0])
    u[s0, 1] = 0.0
    o = assert_matches_simulation(logits, u, 1.0, 0)     # C = 8 > 6 routed to expert 1
    assert bool(o["keep1"][s0])


def test_selection_is_not_by_position():
    """A skewed expert drops an early token and keeps a later one: the selection follows the uniform, not the token order."""
    S, E = 64, 4
    idx = skewed_idx(S, E, [40, 8, 8, 8], 9)
    logits = planted_logits(idx, E, 9)
    u = torch.rand(S, E, generator=torch.Generator().manual_seed(10))
    toks = (idx == 0).nonzero()[:, 0].tolist()
    u[toks[0], 0] = 0.001                          # the first token of expert 0 has the smallest key, the last the largest
    u[toks[-1], 0] = 0.999
    o = assert_matches_simulation(logits, u, 1.0, 0)     # C = 16 of 40
    assert not bool(o["keep1"][toks[0]]) and bool(o["keep1"][toks[-1]])
    dropped_before_kept = any(not o["keep1"][a] and o["keep1"][b] for a in toks for b in toks if a < b)
    assert dropped_before_kept


def test_top1gating_failure_cases_raise():
    lg = torch.randn(8, 4)
    u = torch.rand(8, 4)
    with pytest.raises(ValueError, match="min_capacity"):
        O.top1gating(lg, u, 1.0, 9)
    with pytest.raises(ValueError, match="capacity"):
        O.top1gating(lg, u, 8.0, 0)                # C = ceil(8/4 * 8) = 16 > 8


# ---------------------------------------------------------------------------------------------------------------------------------
# pin against deepspeed.moe.sharded_moe.top1gating (deepspeed==0.9.5)
# ---------------------------------------------------------------------------------------------------------------------------------
def _import_deepspeed_gating():
    ref = os.path.join(ROOT, "baseline", "_ref")
    if os.path.isdir(ref) and ref not in sys.path:
        sys.path.append(ref)
    try:
        return importlib.import_module("deepspeed.moe.sharded_moe")
    except Exception as e:                                  # noqa: BLE001 -- any import failure means "no usable DeepSpeed here"
        pytest.skip("deepspeed is not importable here (%s: %s): the top-1 gate oracle stays 'parity unpinned'" % (type(e).__name__, e))


@pytest.mark.parametrize("S,E,cf,min_cap", [(64, 4, 1.0, 0), (333, 4, 1.5, 4), (2048, 4, 1.5, 0), (500, 8, 0.5, 0), (16, 2, 2.0, 8)])
def test_restated_top1gating_equals_deepspeed(S, E, cf, min_cap):
    sm = _import_deepspeed_gating()
    g = torch.Generator().manual_seed(S * 13 + E)
    logits = torch.randn(S, E, generator=g) * 2.0
    u = torch.rand(S, E, generator=g)                      # continuous: no two keys tie
    # top1gating: `uniform = exp_selection_uniform_map.get(logits.device)`, then `mask1_rand = mask1 * uniform(mask1.shape)`
    dev = logits.device
    saved = sm.exp_selection_uniform_map.get(dev)
    sm.exp_selection_uniform_map[dev] = lambda shape: u.reshape(shape).clone()
    try:
        out = sm.top1gating(logits.clone(), cf, min_cap)
    finally:
        if saved is None:
            sm.exp_selection_uniform_map.pop(dev, None)
        else:
            sm.exp_selection_uniform_map[dev] = saved
    l_aux, combine, dispatch, exp_counts = out[0], out[1], out[2], out[3]
    mine = O.top1gating(logits, u, cf, min_cap)
    assert combine.shape == mine["combine"].shape, (combine.shape, mine["combine"].shape)
    assert torch.equal(dispatch.bool(), mine["dispatch"])
    torch.testing.assert_close(combine.float(), mine["combine"], rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(l_aux.float(), mine["l_aux"], rtol=1e-6, atol=1e-7)
    assert torch.equal(torch.as_tensor(exp_counts).long().cpu(), mine["exp_counts"].long())


# ---------------------------------------------------------------------------------------------------------------------------------
# host side: MoE(k=1), the flag, the saved config
# ---------------------------------------------------------------------------------------------------------------------------------
def _tiny_cfg():
    from llavamod.model import LLaVAMoDQwen1_5Config
    from llavamod.model import synthetic as S
    clip = S.CLIP["tiny"]
    return LLaVAMoDQwen1_5Config(**dict(S.ARCH["tiny"], num_hidden_layers=4), mm_image_tower=dict(clip), image_projector_type="mlp2x_gelu",
                                 mm_hidden_size=64, mm_vision_select_layer=-2), clip


def test_moe_accepts_top1_and_refuses_other_widths():
    from llavamod.model.language_model.qwen2_core import MoE, Qwen2MLP
    cfg, _ = _tiny_cfg()
    dense = Qwen2MLP(cfg, "cpu", torch.float32)
    m = MoE(cfg, dense, num_experts=4, k=1)
    assert m.k == 1 and m.deepspeed_moe.gate.wg.weight.shape == (4, cfg.hidden_size)
    for k in (0, 3, 4):
        with pytest.raises(ValueError, match="top-1 and top-2"):
            MoE(cfg, dense, num_experts=4, k=k)


def test_top_k_experts_flag_parses():
    from llavamod.config.args import AlignArguments, DataArguments, ModelArguments, TrainingArguments, parse_args_into_dataclasses
    argv = ("--moe_enable True --num_experts 4 --top_k_experts 1 --capacity_factor 1.5 --moe_mode sparse --output_dir /tmp/o "
            "--policy_model_type sparse --ref_model_type dense").split()
    m, _, _, _ = parse_args_into_dataclasses((ModelArguments, DataArguments, TrainingArguments, AlignArguments), argv)
    assert m.top_k_experts == 1


def test_top1_config_round_trips(tmp_path):
    from llavamod.model import LLaVAMoDQwen1_5ForCausalLM, LLaVAMoDQwen1_5ForCausalLMFineTune, EvalLLaVAMoDQwen1_5ForCausalLM
    from llavamod.model import synthetic as S
    cfg, clip = _tiny_cfg()
    m = LLaVAMoDQwen1_5ForCausalLM(cfg, device="cpu", dtype=torch.float32)
    m.initialize_moe_modules(S.moe_args(top_k=1))
    m.get_model().initialize_vision_modules(S.vision_args(clip))
    assert m.config.moe["top_k_experts"] == 1
    assert all(l.mlp.k == 1 for l in m.model.layers if hasattr(l.mlp, "deepspeed_moe"))
    m.save_pretrained(str(tmp_path))
    for cls in (LLaVAMoDQwen1_5ForCausalLMFineTune, EvalLLaVAMoDQwen1_5ForCausalLM):
        m2 = cls.from_pretrained(str(tmp_path), device="cpu", torch_dtype=torch.float32)
        assert m2.config.moe["top_k_experts"] == 1
        moes = [l.mlp for l in m2.model.layers if hasattr(l.mlp, "deepspeed_moe")]
        assert moes and all(x.k == 1 for x in moes)
        for k, v in m.state_dict().items():
            assert torch.equal(v, m2.state_dict()[k]), k
