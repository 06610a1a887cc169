"""One training micro-batch with every uninitialised allocation NaN-filled (helpers.poisoned_uninitialised_memory) against the same step
without: a kernel that reads memory nobody wrote -- an output tail, padding rows, a workspace -- turns a loss or a gradient into NaN or
changes it.  Covers the mimic step (kd_lm) eager and CUDA-graph captured, the preference (DPO) step, and the sparse student with top-2 and
top-1 routing.  The fill runs at allocation, so inside a captured graph it is part of the graph and every replay sees it.

Comparison: losses and both gradient arenas must be finite; then equal to the unpoisoned step within the spread that fp32 atomics (split-K
GEMMs, the attention dQ accumulation, the router weight gradient) give two runs of the same step: the loss to 1e-4 relative, each arena
to 1e-2 in relative norm (test_model_gpu.py compares gradients to 8e-2 against the oracle).  Each case prints whether the runs were
bit-identical."""
import contextlib

import pytest
import torch

from tests import helpers as Hh

pytestmark = pytest.mark.gpu


def _pair(top_k):
    from llavamod.model import synthetic as S
    if top_k == 2:
        return Hh.tiny_pair()
    arch = dict(S.ARCH["tiny"], vocab_size=512)
    teacher = S.make_teacher(dict(arch, intermediate_size=320), "tiny", seed=0)
    student = S.make_student(arch, "tiny", seed=1, margs=S.moe_args(top_k=1), share_tower_with=teacher)
    return student, teacher


def _noise(student, top_k, batch_noise, seed):
    if top_k == 2:
        return [n.cuda() for n in batch_noise]
    g = torch.Generator().manual_seed(seed)
    n_moe = sum(1 for l in student.model.layers if hasattr(l.mlp, "deepspeed_moe"))
    return [torch.rand(2 * 55, 4, generator=g).cuda() for _ in range(n_moe)]


def _inputs(student, kind, top_k, graphs):
    if kind == "align":                                              # padded batches run eagerly (masked attention): the graph case is not
        batch, noise = Hh.tiny_batch(student, seed=11, pad=(0, 0) if graphs else (0, 5))
        return dict(batch, moe_noise=_noise(student, top_k, noise, 21))
    bc, nc = Hh.tiny_batch(student, seed=12)
    br, nr = Hh.tiny_batch(student, seed=13)
    br["images"] = bc["images"]
    br["input_ids"][:, :16] = bc["input_ids"][:, :16]
    br["labels"][:, :16] = bc["labels"][:, :16]
    return dict(chosen_input_ids=bc["input_ids"], chosen_labels=bc["labels"], chosen_attention_mask=bc["attention_mask"],
                rejected_input_ids=br["input_ids"], rejected_labels=br["labels"], rejected_attention_mask=br["attention_mask"],
                images=bc["images"], moe_noise=(_noise(student, top_k, nc, 22), _noise(student, top_k, nr, 23)))


def _step(kind, loss_type, top_k, graphs, poisoned):
    """Losses of `steps` identical micro-batches (lr = 0: the weights do not move) and the gradient arenas of the last one."""
    student, teacher = _pair(top_k)
    tr = Hh.make_trainer(student, teacher, loss_type, accum=1, lr=0.0, kind=kind)
    tr.use_cuda_graphs = graphs
    inputs = _inputs(student, kind, top_k, graphs)
    steps = 4 if graphs else 1                                       # two eager warm-ups, the capture, one replay
    losses = []
    with Hh.poisoned_uninitialised_memory() if poisoned else contextlib.nullcontext():
        for _ in range(steps):
            losses.append(tr.training_step(student, dict(inputs)))
        torch.cuda.synchronize()
    if graphs:
        assert any("graph" in v for v in tr._graphs.values()), "no graph was captured"
    opt = tr.optimizer
    grads = {name: t.detach().float().clone() for name, t in (("g16", opt.g16 if opt.n16 else None), ("g32", opt.g32 if opt.n32 else None))
             if t is not None}
    return [float(l) for l in losses], grads


@pytest.mark.parametrize("kind,loss_type,top_k,graphs", [("align", "kd_lm", 2, False), ("align", "kd_lm", 2, True), ("dpo", "sigmoid", 2, False),
                                                         ("align", "kd_lm", 1, False), ("dpo", "sigmoid", 1, False)])
def test_step_is_the_same_with_poisoned_allocations(kind, loss_type, top_k, graphs):
    clean_l, clean_g = _step(kind, loss_type, top_k, graphs, False)
    pois_l, pois_g = _step(kind, loss_type, top_k, graphs, True)
    for i, (a, b) in enumerate(zip(clean_l, pois_l)):
        assert b == b and abs(b) != float("inf"), f"step {i}: non-finite loss {b} with poisoned allocations (clean {a})"
        assert abs(a - b) <= 1e-4 * abs(a), (i, a, b)
    identical = clean_l == pois_l
    for name in clean_g:
        a, b = clean_g[name], pois_g[name]
        nonfinite = int((~torch.isfinite(b)).sum())
        assert nonfinite == 0, f"{name}: {nonfinite} / {b.numel()} non-finite gradient elements with poisoned allocations"
        assert bool(torch.isfinite(a).all())
        rel = (a - b).norm().item() / max(a.norm().item(), 1e-30)
        assert rel <= 1e-2, (name, rel)
        identical = identical and torch.equal(a, b)
    print(f"\nPOISON {kind} {loss_type} top{top_k} graphs={graphs}: losses {pois_l}, bit-identical to the clean step: {identical}")
