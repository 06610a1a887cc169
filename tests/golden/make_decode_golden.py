"""Generates tests/golden/decode_*.<i>.pt (shards, see shards.py) by running the REFERENCE's own cached decoding: LlavaQwen1_5ForCausalLM
(imported in place through oracle/ref_shim.py) with use_cache=True, a prefill and then N cached one-token steps through its multimodal
past_key_values branch (llava_arch.py:162-172).  The steps are teacher-forced: they feed GIVEN tokens, so a bf16 near-tie cannot make
a decoder under test take another path.

    python tests/golden/make_decode_golden.py                     # all cases (needs the reference tree)
    python tests/golden/make_decode_golden.py --case NAME --out F  # one case, written to F as one file (the live leg of the tests)

The reference's vendored modeling_qwen2.py imports Cache / DynamicCache from the installed transformers, whose DynamicCache has no
from_legacy_cache any more; the cache classes are pointed at the reference's own llavamod/model/cache_utils.py before the model runs
(the only change on top of the shims in oracle/ref_shim.py).

Each fixture holds: kw (model numbers), state_dict (reference key names), input_ids [B, T], images (list or None), tokens [B, N] (fed at
the steps), logits [N + 1, B, V] fp32 (the prefill's last position, then every step), k / v: per layer [B, nkv, T' + N, hd] fp32 (the
reference's cache after the last step)."""
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
STEPS = 6

CASES = {
    # name: model kwargs (ref_shim.build_tiny_dense), prompt length, image position (None: text-only prompt)
    "decode_mha_hd32": dict(kw=dict(hidden=128, inter=256, layers=2, heads=4, kv_heads=4, vocab=512, seed=10), T=14, img=3),
    "decode_gqa_4_2": dict(kw=dict(hidden=128, inter=192, layers=2, heads=4, kv_heads=2, vocab=384, seed=11), T=17, img=5),
    "decode_hd64_kv1": dict(kw=dict(hidden=128, inter=256, layers=2, heads=2, kv_heads=1, vocab=512, seed=12, clip_heads=1), T=15, img=0),
    "decode_text_only": dict(kw=dict(hidden=128, inter=256, layers=2, heads=4, kv_heads=2, vocab=512, seed=13), T=19, img=None),
}


def inputs(name):
    """Seeded prompt (B = 2, one image per sample, equal lengths, no padding) and the teacher-forced step tokens."""
    c = CASES[name]
    g = torch.Generator().manual_seed(200 + c["kw"]["seed"])
    B, V = 2, c["kw"]["vocab"]
    ids = torch.randint(0, V, (B, c["T"]), generator=g)
    images = None
    if c["img"] is not None:
        ids[:, c["img"]] = -200
        images = [torch.randn(3, 32, 32, generator=g) for _ in range(B)]
    toks = torch.randint(0, V, (B, STEPS), generator=g)
    return ids, images, toks


def run_reference(name, tmp):
    """The reference's prefill + STEPS cached steps (call in a process where the reference owns the `llavamod` name)."""
    ref = ref_shim.load()
    cu = importlib.import_module("llavamod.model.cache_utils")
    ref.modeling_qwen2.Cache = cu.Cache                   # the reference's own cache classes (see the module docstring)
    ref.modeling_qwen2.DynamicCache = cu.DynamicCache
    c = CASES[name]
    m = ref_shim.build_tiny_dense(os.path.join(tmp, name), **c["kw"])
    m.config.use_cache = True
    ids, images, toks = inputs(name)
    B = ids.shape[0]
    mask = torch.ones(B, ids.shape[1], dtype=torch.long)
    logits = []
    with torch.no_grad():
        o = m(input_ids=ids, images=images, attention_mask=mask, use_cache=True, return_dict=True)
        logits.append(o.logits[:, -1].float())
        pkv = o.past_key_values
        for t in range(STEPS):
            # eval/model_vqa.py-style loop: the prompt's mask, extended by the multimodal branch to the cache length + 1
            o = m(input_ids=toks[:, t:t + 1], past_key_values=pkv, attention_mask=mask, images=images, use_cache=True, return_dict=True)
            logits.append(o.logits[:, -1].float())
            pkv = o.past_key_values
    return dict(kw=c["kw"], state_dict={k: v.detach().clone() for k, v in m.state_dict().items()}, input_ids=ids, images=images, tokens=toks,
                logits=torch.stack(logits), k={str(i): kv[0].float().clone() for i, kv in enumerate(pkv)},
                v={str(i): kv[1].float().clone() for i, kv in enumerate(pkv)})


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
