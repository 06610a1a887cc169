"""Host replay of generate's beam search: generation.BeamScorer (the restatement of transformers 4.37's scorer) driven by a logits function,
with the step's scoring written out in torch on the host.  Used by test_beam_search_host.py (logits of a stub LM, pinned against the
installed transformers) and test_beam_search_gpu.py (the per-step logits of a GPU run)."""
import torch

from llavamod.model.generation import BeamScorer


def replay(logits_fn, B, nb, n_ret, max_new, eos, pad, length_penalty=1.0, early_stopping=False, n_vocab=None, stop_fn=None):
    """logits_fn(step, new) -> fp32 logits [B*nb, V] of the running beams whose new tokens so far are `new` (B*nb lists).  stop_fn(new) ->
    True to stop after a step (a stopping criterion).  -> (rows of new tokens [B*n_ret][width], the scorer, per step a dict of the top
    candidates (scores [B][k], tokens, beams), the chosen local parents [B*nb], done per prompt, and the running beams' new tokens after it)."""
    scorer = BeamScorer(B, nb, n_ret, length_penalty, early_stopping, max_new, eos, pad)
    scores = torch.zeros(B, nb, dtype=torch.float32)
    scores[:, 1:] = -1e9
    scores = scores.view(-1)
    seqs = [[] for _ in range(B * nb)]
    k = max(2, 1 + len(eos)) * nb
    steps = []
    nxt_s = None
    for step in range(max_new):
        logits = logits_fn(step, seqs).float()           # on the device the run scored on: the same log-softmax and top-k bytes
        V = n_vocab if n_vocab is not None and n_vocab < logits.shape[-1] else logits.shape[-1]
        lp = torch.log_softmax(logits[:, :V], dim=-1) + scores.to(logits.device)[:, None]
        top_s, top_i = torch.topk(lp.view(B, nb * V), k, dim=1, largest=True, sorted=True)
        cand = dict(scores=top_s.double().tolist(), tokens=(top_i % V).tolist(), beams=torch.div(top_i, V, rounding_mode="floor").tolist())
        nxt_s, nxt_t, parents = scorer.process(step + 1, cand["scores"], cand["tokens"], cand["beams"], seqs)
        seqs = [seqs[b * nb + p] + [t] for b in range(B) for p, t in zip(parents[b * nb:(b + 1) * nb], nxt_t[b * nb:(b + 1) * nb])]
        scores = torch.tensor(nxt_s, dtype=torch.float32)
        steps.append(dict(cand, parents=parents, done=list(scorer.done), seqs=seqs))
        if scorer.is_done or (stop_fn is not None and stop_fn(seqs)):
            break
    return scorer.finalize(seqs, nxt_s), scorer, steps
