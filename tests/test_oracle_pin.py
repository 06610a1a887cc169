"""Pins oracle/restated.py against the reference's own dense path.

* golden leg (runs everywhere): tests/golden/dense_*.<i>.pt (shards, tests/golden/shards.py) were produced by the reference's
  LlavaQwen1_5ForCausalLM (tests/golden/make_golden.py); the restatement must reproduce logits,
  post-splice labels, loss and parameter gradients.
* live leg: fresh seeds / GQA / left padding, against the reference's answers stored by tests/golden/make_ref_golden.py
  (tests/golden/ref_live_*.pt).
"""
import os

import pytest
import torch

from oracle import restated as R
from tests.golden.make_ref_golden import LIVE_CASES, live_key, live_request
from tests.golden import shards

CASES = ["dense_mha", "dense_gqa", "dense_nopad", "dense_hd64"]


def cfgs_from_kw(kw):
    cc = R.ClipCfg(hidden=64, inter=128, layers=3, heads=kw.get("clip_heads", 4), image=32, patch=8)
    lc = R.LMCfg(hidden=kw["hidden"], inter=kw["inter"], layers=kw["layers"], heads=kw["heads"],
                 kv_heads=kw["kv_heads"], vocab=kw["vocab"], kd_vocab=kw["vocab"])
    return cc, lc


def run_restated(fx, with_grad=True):
    cc, lc = cfgs_from_kw(fx["kw"])
    sd = {k: v.clone().requires_grad_(with_grad and v.is_floating_point()) for k, v in fx["state_dict"].items()}
    out = R.llava_forward(sd, lc, cc, fx["input_ids"], fx["attention_mask"], fx["labels"], fx["images"])
    if with_grad:
        out["loss"].backward()
    return sd, out


@pytest.mark.parametrize("name", CASES)
def test_restated_matches_reference_golden(name, golden_dir):
    fx = shards.load(golden_dir, name)
    sd, out = run_restated(fx)
    assert torch.equal(out["labels"], fx["out_labels"])           # integer splice logic: bit exact
    valid = out["attention_mask"]
    torch.testing.assert_close(out["logits"][valid], fx["logits"][valid], rtol=2e-4, atol=2e-5)
    torch.testing.assert_close(out["loss"], fx["loss"], rtol=1e-5, atol=1e-6)
    assert len(fx["grads"]) > 5
    for k, g in fx["grads"].items():
        torch.testing.assert_close(sd[k].grad, g, rtol=2e-3, atol=2e-6, msg=lambda m: f"{k}: {m}")


@pytest.mark.parametrize("seed,heads,kv,side", LIVE_CASES)
def test_restated_matches_reference_live(seed, heads, kv, side, golden_dir):
    """Fresh seeds / GQA / left padding: the reference's own outputs on these inputs (stored; see tests/golden/make_ref_golden.py)."""
    req = live_request(seed, heads, kv, side)
    ids, labels, mask, images = req["input_ids"], req["labels"], req["attention_mask"], req["images"]
    ref = torch.load(os.path.join(golden_dir, "ref_live_%s.pt" % live_key(seed, heads, kv, side)), weights_only=False)
    cc = R.ClipCfg(hidden=64, inter=128, layers=3, heads=4, image=32, patch=8)
    lc = R.LMCfg(hidden=64, inter=96, layers=1, heads=heads, kv_heads=kv, vocab=97, kd_vocab=97)
    sd = ref["state_dict"]
    out = R.llava_forward(sd, lc, cc, ids, mask, labels, images, padding_side=side)
    assert torch.equal(out["labels"], ref["labels"])
    valid = out["attention_mask"]
    torch.testing.assert_close(out["logits"][valid], ref["logits"][valid], rtol=2e-4, atol=2e-5)
    torch.testing.assert_close(out["loss"], ref["loss"], rtol=1e-5, atol=1e-6)
    # CLIP arithmetic is third-party (transformers.CLIPVisionModel, call site clip_encoder.py:30,54)
    torch.testing.assert_close(R.clip_tower(sd, cc, torch.stack(images[:2])), ref["clip_features"], rtol=1e-4, atol=1e-5)
