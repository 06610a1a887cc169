"""The float64 stage chain of tests/decoder_oracle.py (which the exact decoder test checks every kernel stage with) against
oracle.restated.lm_forward in float64: dense and GQA, head dims 16 / 32 / 64, unpadded and padded on either side (compact RoPE positions,
a sample of length 1), with the planted outlier channel and near-zero row.  CPU only."""
import pytest
import torch

from oracle import restated as R
from tests import decoder_oracle as O

F64 = torch.float64

# (name, H, I, layers, nh, nkv, B, T, lengths, side)
CASES = [
    ("mha-hd16", 64, 96, 2, 4, 4, 2, 13, None, None),
    ("gqa-hd32-right", 128, 160, 2, 4, 2, 2, 17, [17, 9], "right"),
    ("gqa-hd64-left", 256, 320, 2, 4, 1, 3, 11, [11, 4, 1], "left"),
    ("mha-hd32-left", 128, 64, 3, 4, 4, 2, 9, [5, 9], "left"),
]


def build(H, I, L, nh, nkv, seed):
    from llavamod.model.language_model.qwen2_core import Qwen2Config, Qwen2Model
    cfg = Qwen2Config(vocab_size=32, hidden_size=H, intermediate_size=I, num_hidden_layers=L, num_attention_heads=nh,
                      num_key_value_heads=nkv, rope_theta=O.THETA, rms_norm_eps=O.EPS)
    m = O.init_decoder_(Qwen2Model(cfg, device="cpu", dtype=torch.bfloat16), seed)
    sd = {"model." + k: v.to(F64) for k, v in m.state_dict().items()}
    lc = R.LMCfg(hidden=H, inter=I, layers=L, heads=nh, kv_heads=nkv, vocab=32, rope_theta=O.THETA, eps=O.EPS)
    return sd, lc


def mask_of(B, T, lengths, side):
    if lengths is None:
        return None
    m = torch.zeros(B, T, dtype=torch.bool)
    for b, n in enumerate(lengths):
        if side == "left":
            m[b, T - n:] = True
        else:
            m[b, :n] = True
    return m


def positions(mask, B, T):
    if mask is None:
        return torch.arange(T).unsqueeze(0).expand(B, T)
    m = mask.to(torch.int64)
    return (m.cumsum(1) - 1) * m


def assert_close64(name, got, want, rtol=1e-5):
    """restated.rmsnorm takes its input to float32 first (Qwen2RMSNorm's .to(torch.float32)), so in float64 the two agree to about the
    float32 rounding of each norm's input, 1e-7 relative; a wrong weight, eps, position or mask moves the output by far more."""
    err = (got - want).abs().max().item()
    scale = want.abs().max().item()
    assert err <= rtol * scale, f"{name}: max |diff| {err:.3g} against max |ref| {scale:.3g}"


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_chain_matches_oracle(case):
    name, H, I, L, nh, nkv, B, T, lengths, side = case
    sd, lc = build(H, I, L, nh, nkv, seed=len(name))
    mask = mask_of(B, T, lengths, side)
    real = mask if mask is not None else torch.ones(B, T, dtype=torch.bool)
    x, _ = O.planted_embeds(B, T, H, real, seed=H + T, device="cpu")
    pos = positions(mask, B, T)
    got = O.lm_chain_fp64(sd, lc, x.to(F64), mask, pos)
    want, _ = R.lm_forward(sd, lc, x.to(F64), mask, pos)
    assert_close64(name, got, want)


def test_planted_rows_reach_the_norm():
    """The near-zero row's mean square is far below eps, so eps sets its rstd (1e-5 moves it by a factor ~3); the outlier channel carries
    almost all of a real row's mean square."""
    x, rows = O.planted_embeds(2, 8, 256, torch.ones(2, 8, dtype=torch.bool), seed=1, zero_row=True, device="cpu")
    b, t = rows["near-zero"]
    ms = x[b, t].double().pow(2).mean().item()
    assert ms < 0.05 * O.EPS
    assert abs(x[b, t]).max() < 1e-3 and bool((x[1, 7] == 0).all()) and rows["all-zero"] == (1, 7)
    big = x[0, 0].double().pow(2)
    assert big[O.OUTLIER_CH] > 0.9 * big.sum()


@pytest.mark.parametrize("lengths,side", [([17, 9], "right"), ([11, 4, 1], "left")])
def test_mask_helpers(lengths, side):
    T = max(lengths)
    m = mask_of(len(lengths), T, lengths, side)
    assert m.sum(1).tolist() == lengths
    pos = positions(m, len(lengths), T)
    for b, n in enumerate(lengths):
        assert pos[b][m[b]].tolist() == list(range(n))
