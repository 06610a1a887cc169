"""Generates tests/golden/trainer_losses.<i>.pt (shards, see shards.py) by running the REFERENCE's own trainer methods on seeded fake model outputs:
    python tests/golden/make_loss_golden.py

llavamod/train/align_trainer.py and dpo_trainer.py cannot be imported here (accelerate, transformers 4.37 internals), but the loss code in
them is plain torch.  The method bodies are therefore taken verbatim from the read-only reference tree AT GENERATION TIME (ast ->
source segment -> exec into a bare class), bound to a stand-in `self` that carries only the attributes they read (args.distill_all_tokens,
args.moe_enable, moe_loss_enable, loss_type, beta, label_smoothing, label_pad_token_id, ref_model), and called with a fake `model`
whose call returns the (logits, labels, loss, moe_loss) we hand it:
    AlignTrainer.get_p / get_logp / compute_align_loss / compute_loss      (align_trainer.py:455-594)
    DPOTrainer.get_logp / dpo_loss / compute_loss                          (dpo_trainer.py:462-641)
The vocabulary is 256 (so the hard-coded [:151936] slice is a no-op here, as in the tiny parity configs); inputs include -inf student
logits, all-masked labels (0/0 -> NaN), distill_all_tokens, every DPO loss type and both moe-loss branches (incl. the -1.0 sentinel)."""
import ast
import os
import sys
import types

import torch
import torch.nn as nn
import torch.nn.functional as F
from typing import Any, Dict, List, Literal, Optional, Tuple, Union

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests.golden import shards  # noqa: E402
REF = os.environ.get("LLAVAMOD_REFERENCE", "/root/reference")


def load_methods(path, cls_name, names):
    src = open(path).read()
    tree = ast.parse(src)
    cls = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls_name][0]
    body = "\n".join(ast.get_source_segment(src, f, padded=True) for f in cls.body if isinstance(f, ast.FunctionDef) and f.name in names)
    ns = dict(torch=torch, nn=nn, F=F, Any=Any, Dict=Dict, List=List, Literal=Literal, Optional=Optional, Tuple=Tuple, Union=Union,
              PreTrainedModel=nn.Module)
    exec("class Ref:\n" + body, ns)
    return ns["Ref"]


class FakeModel:
    """Callable like the reference's model: returns an object with .logits/.labels/.loss (+ .moe_loss for the sparse student)."""

    def __init__(self, outs):
        self.outs, self.i = outs, 0

    def __call__(self, **kw):
        o = self.outs[self.i % len(self.outs)]
        self.i += 1
        return o


def out(logits, labels, loss, moe=None):
    o = types.SimpleNamespace(logits=logits, labels=labels, loss=loss)
    if moe is not None:
        o.moe_loss = moe
    return o


def make_self(cls, **kw):
    s = cls.__new__(cls)
    s.args = types.SimpleNamespace(distill_all_tokens=kw.get("distill_all", False), moe_enable=kw.get("moe_enable", True))
    s.moe_loss_enable = kw.get("moe_loss_enable", True)
    s.loss_type = kw.get("loss_type", "kd_lm")
    s.beta, s.label_smoothing, s.label_pad_token_id = kw.get("beta", 0.1), kw.get("label_smoothing", 0.0), -100
    s._stored_metrics = {"train": {}}
    s.store_metrics = lambda metrics, train_eval="train": None
    return s


def main():
    A = load_methods(os.path.join(REF, "llavamod/train/align_trainer.py"), "AlignTrainer", {"get_p", "get_logp", "compute_align_loss", "compute_loss"})
    D = load_methods(os.path.join(REF, "llavamod/train/dpo_trainer.py"), "DPOTrainer", {"get_logp", "dpo_loss", "compute_loss"})
    g = torch.Generator().manual_seed(0)
    B, T, V = 2, 12, 256
    cases = {"mimic": [], "dpo": []}
    for name, kw in [("kd_lm+moe", dict(loss_type="kd_lm")), ("only_kd+moe_off", dict(loss_type="only_kd", moe_loss_enable=False)),
                     ("kd_lm+distill_all", dict(loss_type="kd_lm", distill_all=True)), ("kd_lm+neg_inf", dict(loss_type="kd_lm", neg_inf=True)),
                     ("kd_lm+all_masked", dict(loss_type="kd_lm", all_masked=True)), ("kd_lm+dense_student", dict(loss_type="kd_lm", dense=True))]:
        s_logits = torch.randn(B, T, V, generator=g) * 2
        t_logits = torch.randn(B, T, V, generator=g) * 2
        if kw.get("neg_inf"):
            s_logits[0, 3, 5:9] = float("-inf")
        labels = torch.randint(0, V, (B, T), generator=g)
        labels[:, :5] = -100
        if kw.get("all_masked"):
            labels[:] = -100
        sft = torch.rand((), generator=g) + 5.0
        moe = None if kw.get("dense") else torch.rand((), generator=g) * 0.1 + 0.01
        me = make_self(A, **kw)
        me.ref_model = FakeModel([out(t_logits, labels, torch.tensor(0.0))])
        student = FakeModel([out(s_logits, labels, sft, moe)])
        loss, metrics = A.compute_loss(me, student, dict(input_ids=None), return_outputs=True)
        cases["mimic"].append(dict(name=name, kw=kw, s_logits=s_logits, t_logits=t_logits, labels=labels, sft=sft, moe=moe, loss=loss,
                                   metrics={k: (v if torch.is_tensor(v) else torch.tensor(float(v))) for k, v in metrics.items()}))
    for lt in ("sigmoid", "hinge", "ipo", "kto_pair"):
        for moe_on in (True, False):
            lg = [torch.randn(B, T, V, generator=g) * 2 for _ in range(4)]           # policy chosen / rejected, ref chosen / rejected
            lab_c = torch.randint(0, V, (B, T), generator=g)
            lab_r = torch.randint(0, V, (B, T), generator=g)
            lab_c[:, :5] = -100
            lab_r[:, :5] = -100
            sft = [torch.rand((), generator=g) + 5.0 for _ in range(2)]
            moe = [torch.rand((), generator=g) * 0.1 + 0.01 for _ in range(2)]
            me = make_self(D, loss_type=lt, moe_loss_enable=moe_on, label_smoothing=0.0)
            me.ref_model = FakeModel([out(lg[2], lab_c, torch.tensor(0.0)), out(lg[3], lab_r, torch.tensor(0.0))])
            policy = FakeModel([out(lg[0], lab_c, sft[0], moe[0]), out(lg[1], lab_r, sft[1], moe[1])])
            inputs = dict(chosen_input_ids=None, chosen_labels=lab_c, chosen_attention_mask=None, rejected_input_ids=None, rejected_labels=lab_r,
                          rejected_attention_mask=None)
            loss, metrics = D.compute_loss(me, policy, inputs, return_outputs=True)
            cases["dpo"].append(dict(loss_type=lt, moe_loss_enable=moe_on, logits=lg, lab_c=lab_c, lab_r=lab_r, sft=sft, moe=moe, loss=loss,
                                     metrics={k: (v if torch.is_tensor(v) else torch.tensor(float(v))) for k, v in metrics.items()}))
    # label-smoothed sigmoid loss on bare log-probs
    me = make_self(D, loss_type="sigmoid", label_smoothing=0.1)
    lp = [torch.randn(5, generator=g) for _ in range(4)]
    cases["dpo_smoothed"] = dict(logps=lp, out=D.dpo_loss(me, *lp))
    shards.save(cases, HERE, "trainer_losses")
    print("wrote trainer_losses.<i>.pt:", {k: (len(v) if isinstance(v, list) else 1) for k, v in cases.items()})


if __name__ == "__main__":
    main()
