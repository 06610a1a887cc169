"""Host-side pieces of the eval path (no GPU): nucleus filtering against transformers' TopPLogitsWarper, and KeywordsStoppingCriteria
against the reference's own class (llavamod/mm_utils.py:73-105), whose answers are stored in tests/golden/keywords_stopping.json
(tests/golden/make_ref_golden.py)."""
import json
import os

import torch

from tests.golden.make_data_golden import load_tokenizer


def test_top_p_filter_matches_transformers_warper():
    from transformers.generation.logits_process import TopPLogitsWarper
    from llavamod.model.generation import _top_p_filter
    g = torch.Generator().manual_seed(0)
    for top_p in (0.1, 0.5, 0.9, 0.999):
        logits = torch.randn(3, 200, generator=g) * 3
        want = TopPLogitsWarper(top_p=top_p)(None, logits.clone())
        assert torch.equal(_top_p_filter(logits.clone(), top_p), want)


CASES = [("USER: hi ASSISTANT: There are two birds.<|endoftext|>", ["<|endoftext|>"]),
         ("USER: hi ASSISTANT: There are two birds", ["<|endoftext|>"]),
         ("USER: hi ASSISTANT: A small red square", ["red square", "zzz"]),
         ("USER: hi ASSISTANT: A", ["red square"])]


def _mine(tok):
    from llavamod.mm_utils import KeywordsStoppingCriteria
    out = []
    for text, kws in CASES:
        ids = torch.tensor([tok(text).input_ids])
        start = ids[:, :5]
        crit = KeywordsStoppingCriteria(kws, tok, start)
        out.append([bool(crit(ids[:, :n], None)) for n in range(6, ids.shape[1] + 1)])
    return out


def test_keywords_stopping_criteria_matches_reference_class(golden_dir):
    tok_path = os.path.join(golden_dir, "tiny_tokenizer.json")
    with open(os.path.join(golden_dir, "keywords_stopping.json")) as f:
        stored = json.load(f)
    assert [[t, k] for t, k in CASES] == stored["cases"]
    want = stored["want"]
    got = _mine(load_tokenizer(tok_path))
    assert got == want
    assert any(any(row) for row in want) and not all(all(row) for row in want)      # the cases exercise both outcomes
