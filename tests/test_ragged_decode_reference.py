"""CPU checks of the padded-batch decoding oracle (tests/ragged_oracle.py), the reference the GPU ragged-decode tests compare against:
each sequence of a padded batch reproduces the reference's own cached decoding of that prompt alone (tests/golden/ragged_*.pt, made by
tests/golden/make_ragged_decode_golden.py, and the live reference where its tree is present), and the reference's left-padded text batch;
in float64 a dense padded batch equals each prompt alone for left, right and mixed padding; and the host plan of a padded prefill
(lengths, source ranges, positions) is what the cache and the kernels need."""
import types
import warnings

import pytest
import torch

from oracle import ref_shim
from oracle import restated as R
from tests import ragged_oracle as RO
from tests.golden import make_ragged_decode_golden as MG
from tests.golden import shards
from tests.test_decode_reference import cfgs_from_kw

TOL = dict(rtol=2e-4, atol=2e-5)          # the tolerance of test_oracle_pin


def _relayout(ids, mask, side):
    """The same prompts padded on `side` ("left", "right", or "mixed": even rows left, odd rows right)."""
    B, T = ids.shape
    out, m = torch.zeros_like(ids), torch.zeros_like(mask)
    for b in range(B):
        n = int(mask[b].sum())
        left = side == "left" or (side == "mixed" and b % 2 == 0)
        sl = slice(T - n, T) if left else slice(0, n)
        out[b, sl] = ids[b][mask[b]]
        m[b, sl] = True
    return out, m


def check_against_reference(fx, side="left", padding_side="right"):
    cc, lc = cfgs_from_kw(fx["kw"])
    ids, mask = _relayout(fx["input_ids"], fx["mask"], side)
    logits, state = RO.llava_decode(fx["state_dict"], lc, cc, ids, mask, fx["images"], fx["tokens"], padding_side)
    for b in range(ids.shape[0]):
        torch.testing.assert_close(logits[:, b], fx["logits"][str(b)], **TOL)
        for i, (k, v) in enumerate(RO.packed_cache(state, b)):
            torch.testing.assert_close(k, fx["k"]["%d.%d" % (b, i)], **TOL)
            torch.testing.assert_close(v, fx["v"]["%d.%d" % (b, i)], **TOL)
    if fx["batch_logits"] is not None:         # the reference's own left-padded text batch: every sequence as alone
        torch.testing.assert_close(fx["batch_logits"], logits, **TOL)


@pytest.mark.parametrize("side,padding_side", [("left", "right"), ("right", "right"), ("mixed", "left")])
@pytest.mark.parametrize("name", list(MG.CASES))
def test_ragged_oracle_matches_reference_golden(name, side, padding_side, golden_dir):
    fx = shards.load(golden_dir, name)
    assert fx["logits"]["0"].shape[0] == MG.STEPS + 1
    check_against_reference(fx, side, padding_side)


@pytest.mark.parametrize("name", ["ragged_gqa_4_2", "ragged_text_only"])
def test_ragged_oracle_matches_live_reference(name):
    if not ref_shim.available():
        msg = "reference tree not present at %s: the live ragged-decoding leg did not run" % ref_shim.REF_ROOT
        warnings.warn(msg)
        pytest.skip(msg)
    check_against_reference(MG.run_live(name))


def _model(heads, kv_heads, hidden, moe_layers=(), seed=0, **kw):
    cfg = R.LMCfg(hidden=hidden, inter=96, layers=2, heads=heads, kv_heads=kv_heads, vocab=97, moe_layers=list(moe_layers), **kw)
    g = torch.Generator().manual_seed(seed)
    return cfg, R.init_lm(cfg, 32, g, std=0.3, dtype=torch.float64), g


@pytest.mark.parametrize("side", ["left", "right", "mixed"])
@pytest.mark.parametrize("heads,kv_heads,hidden", [(4, 4, 64), (4, 2, 128)])
def test_dense_padded_batch_equals_each_prompt_alone_fp64(heads, kv_heads, hidden, side):
    cfg, sd, g = _model(heads, kv_heads, hidden)
    lens, N = [9, 4, 13], 5
    T = max(lens)
    x = torch.randn(len(lens), T, hidden, generator=g, dtype=torch.float64)
    mask = torch.zeros(len(lens), T, dtype=torch.bool)
    for b, n in enumerate(lens):
        mask[b, :n] = True
    _, mask = _relayout(torch.zeros(len(lens), T, dtype=torch.long), mask, side)
    steps = torch.randn(len(lens), N, hidden, generator=g, dtype=torch.float64)
    h, state = RO.prefill(sd, cfg, x, mask)
    got = [RO.last_real(h, mask)]
    for t in range(N):
        got.append(RO.step(sd, cfg, steps[:, t:t + 1], state)[:, 0])
    for b, n in enumerate(lens):
        xb = x[b:b + 1][:, mask[b]]
        one = torch.ones(1, n, dtype=torch.bool)
        hb, sb = RO.prefill(sd, cfg, xb, one)
        alone = [hb[:, -1]]
        for t in range(N):
            alone.append(RO.step(sd, cfg, steps[b:b + 1, t:t + 1], sb)[:, 0])
        for t in range(N + 1):
            assert (got[t][b] - alone[t][0]).abs().max().item() < 1e-12, (b, t)
        for (k, v), (k1, v1) in zip(RO.packed_cache(state, b), RO.packed_cache(sb, 0)):
            assert (k - k1).abs().max().item() < 1e-12 and (v - v1).abs().max().item() < 1e-12
        # the restated cached decoder of an unpadded prompt (tests/decode_oracle.py) is the same function
        full, _ = R.lm_forward(sd, cfg, torch.cat([xb, steps[b:b + 1]], 1), None, None)
        assert (full[0, n - 1:] - torch.stack([a[0] for a in alone])).abs().max().item() < 1e-12


def test_sparse_prefill_routes_pad_rows_and_steps_route_the_batch():
    """Sparse student: the padded prefill routes every row (S = B * T, pads included); a cached step routes its B tokens (S = B)."""
    E = 4
    cfg, sd, g = _model(2, 2, 64, moe_layers=(0, 1), num_experts=E, min_capacity=0, capacity_factor=1.0)
    mask = torch.tensor([[0, 0, 1, 1, 1, 1], [1, 1, 1, 0, 0, 0]], dtype=torch.bool)
    x = torch.randn(2, 6, 64, generator=g, dtype=torch.float64)
    noise = [R.gumbel_noise((12, E), g).double() for _ in range(2)]
    rec = []
    _, state = RO.prefill(sd, cfg, x, mask, noise, rec)
    assert [r["gates"].shape[0] for r in rec] == [12, 12] and all(r["capacity"] == R.moe_capacity(12, E, 1.0, 0) for r in rec)
    rec = []
    RO.step(sd, cfg, torch.randn(2, 1, 64, generator=g, dtype=torch.float64), state, [R.gumbel_noise((2, E), g).double()] * 2, rec)
    assert [r["gates"].shape[0] for r in rec] == [2, 2] and state["lens"].tolist() == [5, 4]


@pytest.mark.parametrize("images", [False, True])
@pytest.mark.parametrize("side", ["left", "right", "mixed"])
def test_host_plan_of_a_padded_prefill(side, images):
    """Per sequence: the cache length n_b (spliced_length, the splice plan's mask, MaskInfo.lengths), the source range [lo, hi) of its
    real rows (K.pad_ranges, what lmod_kv_append_rows reads) and positions 0 .. n_b - 1 on those rows, for either splice padding side."""
    from llavamod import kernels as K
    from llavamod.model import llava_arch as A
    from llavamod.model.language_model.llava_qwen_common import LlavaQwenForCausalLMBase
    P = 5
    g = torch.Generator().manual_seed(7)
    lens = [7, 3, 10, 5]
    T = max(lens)
    ids = torch.zeros(len(lens), T, dtype=torch.long)
    mask = torch.zeros(len(lens), T, dtype=torch.bool)
    for b, n in enumerate(lens):
        ids[b, :n] = torch.randint(1, 90, (n,), generator=g)
        if images:
            ids[b, b % n] = -200
        mask[b, :n] = True
    ids, mask = _relayout(ids, mask, side)
    fake = types.SimpleNamespace(get_image_tower=lambda: types.SimpleNamespace(num_patches=P), config=types.SimpleNamespace())
    n_b = LlavaQwenForCausalLMBase.spliced_length(fake, ids, [None] * len(lens) if images else None, mask)
    assert n_b == [n + (P - 1) * images for n in lens]
    for splice_side in ("left", "right"):
        if images:
            _, _, nm, pos, _ = A.splice_plan(ids.numpy(), mask.numpy(), None, P, splice_side)
            nm, pos = torch.from_numpy(nm), torch.from_numpy(pos)
        else:              # text-only prompts are not re-laid out; the cached prefill computes compact positions from the mask
            nm, pos = mask, RO.compact_positions(mask)
        assert nm.sum(1).tolist() == n_b
        lo, hi = K.pad_ranges(nm)
        assert (hi - lo).tolist() == n_b
        for b, n in enumerate(n_b):
            assert bool(nm[b, lo[b]:hi[b]].all())
            assert pos[b, lo[b]:hi[b]].tolist() == list(range(n)) and int(pos[b][~nm[b]].abs().sum()) == 0
