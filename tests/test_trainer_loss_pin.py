"""Pins the oracle's loss code (oracle/restated.py: get_p / get_logp / compute_align_loss / mimic_compute_loss, dpo_get_logp / dpo_loss /
dpo_compute_loss) against outputs of the REFERENCE's own AlignTrainer / DPOTrainer method bodies, executed at golden-generation time on
fake model outputs (tests/golden/make_loss_golden.py -> trainer_losses.<i>.pt).  fp32 CPU on both sides: exact up to summation order."""
import math
import os

import pytest
import torch

from oracle import restated as R
from tests.golden import shards


@pytest.fixture(scope="module")
def gold(golden_dir):
    return shards.load(golden_dir, "trainer_losses")


def _close(a, b, what):
    a, b = torch.as_tensor(a, dtype=torch.float32), torch.as_tensor(b, dtype=torch.float32)
    if bool(torch.isnan(b).all()):
        assert bool(torch.isnan(a).all()), what                     # 0/0 stays NaN (align_trainer.py:526)
        return
    assert torch.allclose(a, b, rtol=1e-5, atol=1e-6), (what, a, b)


def test_mimic_compute_loss_matches_reference_method_bodies(gold):
    seen = set()
    for c in gold["mimic"]:
        kw = c["kw"]
        V = c["s_logits"].shape[-1]
        student = dict(logits=c["s_logits"], labels=c["labels"], loss=c["sft"], moe_loss=c["moe"])
        loss, m = R.mimic_compute_loss(student, c["t_logits"], kw.get("loss_type", "kd_lm"), kw.get("moe_loss_enable", True),
                                       kw.get("distill_all", False), V)
        _close(loss, c["loss"], c["name"])
        for k, v in c["metrics"].items():
            _close(m[k], v, (c["name"], k))
        seen.add(c["name"])
        if "all_masked" in c["name"]:
            assert math.isnan(float(c["loss"]))
        if "moe_off" in c["name"] or "dense" in c["name"]:
            assert float(c["metrics"]["loss/moe_balance"]) == -1.0  # the sentinel (align_trainer.py:579)
    assert len(seen) == 6


def test_align_pieces_match(gold):
    c = gold["mimic"][3]                                            # the -inf student logits case
    V = c["s_logits"].shape[-1]
    p = R.get_p(c["t_logits"], V)
    lp = R.get_logp(c["s_logits"], V)
    assert bool(torch.isinf(lp).any())
    align = R.compute_align_loss(lp, p, c["labels"], False)
    _close(align, c["metrics"]["loss/align"], "align with -inf terms dropped")


def test_dpo_compute_loss_matches_reference_method_bodies(gold):
    for c in gold["dpo"]:
        lg = c["logits"]
        pol_c = dict(logits=lg[0], labels=c["lab_c"], loss=c["sft"][0], moe_loss=c["moe"][0])
        pol_r = dict(logits=lg[1], labels=c["lab_r"], loss=c["sft"][1], moe_loss=c["moe"][1])
        loss, m = R.dpo_compute_loss(pol_c, pol_r, lg[2], c["lab_c"], lg[3], c["lab_r"], 0.1, c["loss_type"], c["moe_loss_enable"])
        what = (c["loss_type"], c["moe_loss_enable"])
        _close(loss, c["loss"], what)
        for k, v in c["metrics"].items():
            _close(m[k], v, what + (k,))
    lp = gold["dpo_smoothed"]["logps"]
    got = R.dpo_loss(*lp, beta=0.1, loss_type="sigmoid", label_smoothing=0.1)
    for a, b in zip(got, gold["dpo_smoothed"]["out"]):
        _close(a, b, "label-smoothed sigmoid")


def test_optimizer_schedule_and_clipping_match_the_installed_libraries():
    """The reference takes these from third-party code (HF Trainer's cosine-with-warmup schedule and max_grad_norm clipping, torch.optim.AdamW;
    call sites align_trainer.py:409-417 and the shells' --lr_scheduler_type cosine --warmup_ratio 0.03).  torch and transformers ARE installed
    here, so the restated arithmetic is pinned against the libraries themselves (the formulas have not changed since the pinned 4.37)."""
    import transformers
    g = torch.Generator().manual_seed(0)
    shapes = [(7, 5), (11,), (3, 4, 2)]
    params = [torch.randn(*s, generator=g) for s in shapes]
    ref_params = [p.clone().requires_grad_(True) for p in params]
    total, base_lr, warm_ratio = 40, 2e-3, 0.03
    opt = torch.optim.AdamW(ref_params, lr=base_lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
    sched = transformers.get_cosine_schedule_with_warmup(opt, num_warmup_steps=math.ceil(warm_ratio * total), num_training_steps=total)
    m = [torch.zeros_like(p) for p in params]
    v = [torch.zeros_like(p) for p in params]
    for step in range(total):
        grads = [torch.randn(*s, generator=g) * (3.0 if step % 5 == 0 else 0.1) for s in shapes]
        for p, gr in zip(ref_params, grads):
            p.grad = gr.clone()
        ref_norm = torch.nn.utils.clip_grad_norm_(ref_params, 1.0)
        mine = [gr.clone() for gr in grads]
        my_norm = R.clip_grad_norm(mine, 1.0)
        assert abs(float(my_norm) - float(ref_norm)) < 1e-5 * max(1.0, float(ref_norm))
        lr = R.cosine_lr(step, total, base_lr, warm_ratio)
        assert abs(lr - sched.get_last_lr()[0]) < 1e-12 + 1e-9 * base_lr, (step, lr, sched.get_last_lr())
        R.adamw_step(params, mine, m, v, step + 1, lr, wd=0.01)
        opt.step()
        sched.step()
        for a, b in zip(params, ref_params):
            assert torch.allclose(a, b.detach(), rtol=1e-5, atol=1e-7), step
