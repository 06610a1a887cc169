"""Generates tests/golden/ragged_*.<i>.pt (shards, see shards.py) by running the REFERENCE's own cached decoding on prompts of different
lengths: LlavaQwen1_5ForCausalLM (imported in place through oracle/ref_shim.py, cache classes pointed at the reference's own
cache_utils.py as in make_decode_golden.py) with use_cache=True, a prefill and then STEPS teacher-forced one-token cached steps.

Every prompt is decoded ALONE (B = 1, no padding): that is the function a padded batch has to compute for each of its sequences.  For the
text-only case the left-padded batch is also decoded as ONE call, the way HF's generate drives a Qwen2 model: position_ids
cumsum(mask) - 1 (pads at 1) for the prefill, then mask.sum - 1 at every step with the mask grown by one column per step.  The reference
has no batched form that matches the alone runs for padded image batches or right padding (DESIGN section 8), so none is recorded.

    python tests/golden/make_ragged_decode_golden.py                     # all cases (needs the reference tree)
    python tests/golden/make_ragged_decode_golden.py --case NAME --out F  # one case, written to F as one file (the live leg of the tests)

Each fixture holds: kw (model numbers), state_dict (reference key names), input_ids [B, T] left-padded with 0, mask [B, T] bool,
images (one per prompt, or None), tokens [B, N] (fed at the steps), logits {str(b): [N + 1, V] fp32} of prompt b alone (the prefill's last
position, then every step), k / v {"b.i": [nkv, n_b + N, hd] fp32} (prompt b's cache of layer i after the last step), batch_logits
[N + 1, B, V] fp32 of the left-padded batch call (text-only case) or None."""
import argparse
import importlib
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402
from tests.golden import shards  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
STEPS = 4

CASES = {
    # name: model kwargs (ref_shim.build_tiny_dense), prompt lengths (tokens), image position per prompt (None: text-only prompts)
    "ragged_mha_hd32": dict(kw=dict(hidden=128, inter=256, layers=2, heads=4, kv_heads=4, vocab=512, seed=30), T=[12, 7, 9], img=[3, 0, 6]),
    "ragged_gqa_4_2": dict(kw=dict(hidden=128, inter=192, layers=2, heads=4, kv_heads=2, vocab=384, seed=31), T=[6, 13, 9, 10],
                           img=[5, 2, 0, 4]),
    "ragged_text_only": dict(kw=dict(hidden=128, inter=256, layers=2, heads=4, kv_heads=2, vocab=512, seed=32), T=[12, 7, 10], img=None),
}


def inputs(name):
    """Seeded prompts, left-padded with 0 into one [B, T] batch, their mask, one image per prompt (or None) and the step tokens."""
    c = CASES[name]
    g = torch.Generator().manual_seed(300 + c["kw"]["seed"])
    V, lens = c["kw"]["vocab"], c["T"]
    B, T = len(lens), max(lens)
    ids = torch.zeros(B, T, dtype=torch.long)
    mask = torch.zeros(B, T, dtype=torch.bool)
    for b, n in enumerate(lens):
        p = torch.randint(1, V, (n,), generator=g)
        if c["img"] is not None:
            p[c["img"][b]] = -200
        ids[b, T - n:] = p
        mask[b, T - n:] = True
    images = [torch.randn(3, 32, 32, generator=g) for _ in lens] if c["img"] is not None else None
    toks = torch.randint(0, V, (B, STEPS), generator=g)
    return ids, mask, images, toks


def _alone(m, ids, image, toks):
    """One prompt [1, n] at B = 1: the prefill, then STEPS cached steps (eval/model_vqa.py-style loop, as make_decode_golden.py)."""
    images = [image] if image is not None else None
    mask = torch.ones(1, ids.shape[1], dtype=torch.long)
    logits = []
    o = m(input_ids=ids, images=images, attention_mask=mask, use_cache=True, return_dict=True)
    logits.append(o.logits[0, -1].float())
    pkv = o.past_key_values
    for t in range(toks.shape[1]):
        o = m(input_ids=toks[:, t:t + 1], past_key_values=pkv, attention_mask=mask, images=images, use_cache=True, return_dict=True)
        logits.append(o.logits[0, -1].float())
        pkv = o.past_key_values
    return torch.stack(logits), pkv


def _batch_text(m, ids, mask, toks):
    """The left-padded text-only batch as one call, positions and mask as HF's generate passes them to a Qwen2 model."""
    am = mask.long()
    pos = (am.cumsum(1) - 1).masked_fill(am == 0, 1)
    logits = []
    o = m(input_ids=ids, attention_mask=am, position_ids=pos, use_cache=True, return_dict=True)
    logits.append(o.logits[:, -1].float())
    pkv = o.past_key_values
    for t in range(toks.shape[1]):
        am = torch.cat([am, torch.ones(am.shape[0], 1, dtype=am.dtype)], 1)
        o = m(input_ids=toks[:, t:t + 1], attention_mask=am, position_ids=am.sum(1, keepdim=True) - 1, past_key_values=pkv, use_cache=True,
              return_dict=True)
        logits.append(o.logits[:, -1].float())
        pkv = o.past_key_values
    return torch.stack(logits)


def run_reference(name, tmp):
    """The reference's cached decoding of every prompt alone (+ the left-padded text batch); call in a process where the reference owns
    the `llavamod` name."""
    ref = ref_shim.load()
    cu = importlib.import_module("llavamod.model.cache_utils")
    ref.modeling_qwen2.Cache = cu.Cache
    ref.modeling_qwen2.DynamicCache = cu.DynamicCache
    c = CASES[name]
    m = ref_shim.build_tiny_dense(os.path.join(tmp, name), **c["kw"])
    m.config.use_cache = True
    ids, mask, images, toks = inputs(name)
    logits, k, v = {}, {}, {}
    with torch.no_grad():
        for b in range(ids.shape[0]):
            lg, pkv = _alone(m, ids[b:b + 1, mask[b]], images[b] if images is not None else None, toks[b:b + 1])
            logits[str(b)] = lg
            for i, kv in enumerate(pkv):
                k["%d.%d" % (b, i)] = kv[0][0].float().clone()
                v["%d.%d" % (b, i)] = kv[1][0].float().clone()
        batch = _batch_text(m, ids, mask, toks) if images is None else None
    return dict(kw=c["kw"], state_dict={n: t.detach().clone() for n, t in m.state_dict().items()}, input_ids=ids, mask=mask, images=images,
                tokens=toks, logits=logits, k=k, v=v, batch_logits=batch)


def run_live(name, timeout=600):
    """One case from the live reference, in a subprocess of its own (the reference and this project both own the `llavamod` name)."""
    import subprocess
    d = tempfile.mkdtemp()
    out = os.path.join(d, "resp.pt")
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--case", name, "--out", out], capture_output=True, text=True,
                       timeout=timeout, env=env)
    if r.returncode != 0:
        raise RuntimeError("reference decode failed:\n" + r.stdout[-2000:] + r.stderr[-4000:])
    return torch.load(out, weights_only=False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    tmp = tempfile.mkdtemp()
    if a.case:
        torch.save(run_reference(a.case, tmp), a.out)
        return
    for name in CASES:
        shards.save(run_reference(name, tmp), OUT, name)
        print("wrote", name)


if __name__ == "__main__":
    main()
