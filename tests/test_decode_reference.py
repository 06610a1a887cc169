"""CPU checks of the cached-decoding oracle (tests/decode_oracle.py), the reference the GPU decode tests compare against:
it reproduces the reference's own cached decoding (tests/golden/decode_*.pt, made by tests/golden/make_decode_golden.py, and the live
reference where its tree is present), a dense decoder decoded through the cache equals a full recompute in float64, and the MoE layers
of a cached step route the step's B tokens alone, with capacity ceil(B/E * ecf * 2) raised to min_capacity, dropping tokens when that
capacity is exceeded."""
import math
import warnings

import pytest
import torch

from oracle import ref_shim
from oracle import restated as R
from tests import decode_oracle as D
from tests.golden import make_decode_golden as MG
from tests.golden import shards


def cfgs_from_kw(kw):
    cc = R.ClipCfg(hidden=64, inter=128, layers=3, heads=kw.get("clip_heads", 4), image=32, patch=8)
    lc = R.LMCfg(hidden=kw["hidden"], inter=kw["inter"], layers=kw["layers"], heads=kw["heads"], kv_heads=kw["kv_heads"], vocab=kw["vocab"],
                 kd_vocab=kw["vocab"])
    return cc, lc


def check_against_reference(fx):
    cc, lc = cfgs_from_kw(fx["kw"])
    logits, past = D.llava_decode(fx["state_dict"], lc, cc, fx["input_ids"], fx["images"], fx["tokens"])
    torch.testing.assert_close(logits, fx["logits"], rtol=2e-4, atol=2e-5)          # the tolerance of test_oracle_pin
    for i, (k, v) in enumerate(past):
        torch.testing.assert_close(k, fx["k"][str(i)], rtol=2e-4, atol=2e-5)
        torch.testing.assert_close(v, fx["v"][str(i)], rtol=2e-4, atol=2e-5)


@pytest.mark.parametrize("name", list(MG.CASES))
def test_restated_cached_decoder_matches_reference_golden(name, golden_dir):
    fx = shards.load(golden_dir, name)
    assert fx["logits"].shape[0] == MG.STEPS + 1
    check_against_reference(fx)


@pytest.mark.parametrize("name", ["decode_gqa_4_2", "decode_text_only"])
def test_restated_cached_decoder_matches_live_reference(name):
    if not ref_shim.available():
        msg = "reference tree not present at %s: the live cached-decoding leg did not run" % ref_shim.REF_ROOT
        warnings.warn(msg)
        pytest.skip(msg)
    check_against_reference(MG.run_live(name))


def _model(heads, kv_heads, hidden=64, layers=2, moe_layers=(), seed=0, **kw):
    cfg = R.LMCfg(hidden=hidden, inter=96, layers=layers, heads=heads, kv_heads=kv_heads, vocab=97, moe_layers=list(moe_layers), **kw)
    g = torch.Generator().manual_seed(seed)
    sd = R.init_lm(cfg, 32, g, std=0.3, dtype=torch.float64)
    return cfg, sd, g


@pytest.mark.parametrize("heads,kv_heads,hidden", [(4, 4, 64), (4, 2, 128), (2, 1, 128)])
def test_dense_cached_decode_equals_full_recompute_fp64(heads, kv_heads, hidden):
    cfg, sd, g = _model(heads, kv_heads, hidden)
    B, T0, N = 2, 9, 6
    x = torch.randn(B, T0 + N, hidden, generator=g, dtype=torch.float64)
    full, _ = R.lm_forward(sd, cfg, x, None, None)
    h, past, _ = D.lm_forward_cached(sd, cfg, x[:, :T0])
    steps = [h]
    for t in range(T0, T0 + N):
        h, past, _ = D.lm_forward_cached(sd, cfg, x[:, t:t + 1], past)
        steps.append(h)
    got = torch.cat(steps, 1)
    assert (got - full).abs().max().item() < 1e-12
    # the cache holds every position's rotated k / v, [B, nkv, T, hd] per layer (HF's legacy layout)
    assert past[0][0].shape == (B, kv_heads, T0 + N, hidden // heads)


def _step_capacity(S, E, ecf, min_cap):
    return max(int(math.ceil(S / E * ecf * 2)), min_cap)


@pytest.mark.parametrize("B,ecf,min_cap", [(8, 0.5, 1), (8, 2.0, 4), (1, 2.0, 0), (5, 0.3, 0)])
def test_moe_cached_step_routes_the_step_tokens_only(B, ecf, min_cap):
    E = 4
    cfg, sd, g = _model(2, 2, 64, layers=2, moe_layers=(0, 1), num_experts=E, min_capacity=min_cap, capacity_factor=1.5)
    T0 = 7
    x = torch.randn(B, T0, 64, generator=g, dtype=torch.float64)
    noise = [R.gumbel_noise((B * T0, E), g).double() for _ in range(2)]
    rec = []
    _, past, _ = D.lm_forward_cached(sd, cfg, x, None, noise, rec, capacity_factor=ecf)
    assert [r["capacity"] for r in rec] == [_step_capacity(B * T0, E, ecf, min_cap)] * 2
    dropped = 0
    for _ in range(3):
        rec = []
        noise = [R.gumbel_noise((B, E), g).double() for _ in range(2)]
        step = torch.randn(B, 1, 64, generator=g, dtype=torch.float64)
        _, past, _ = D.lm_forward_cached(sd, cfg, step, past, noise, rec, capacity_factor=ecf)
        for r in rec:
            C = _step_capacity(B, E, ecf, min_cap)
            assert r["capacity"] == C and r["gates"].shape == (B, E)
            # first choices take the first C slots of an expert in token order, second choices queue behind every first choice
            for e in range(E):
                n1 = int((r["idx1"] == e).sum())
                assert int((r["keep1"] & (r["idx1"] == e)).sum()) == min(n1, C)
                n2 = int((r["idx2"] == e).sum())
                assert int((r["keep2"] & (r["idx2"] == e)).sum()) == max(0, min(n2, C - n1))
            dropped += int((~r["keep1"]).sum() + (~r["keep2"]).sum())
    if (B, ecf, min_cap) == (8, 0.5, 1):
        assert dropped > 0                                  # capacity 2 for 16 choices over 4 experts: tokens are dropped
