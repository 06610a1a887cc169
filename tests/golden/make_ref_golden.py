"""Regenerates the stored answers of the original LLaVA-MoD code that tests compare against, so that the suite needs nothing outside the
repository:

  ref_live_<case>.pt      the reference's dense model (LlavaQwen1_5ForCausalLM, via oracle/ref_shim.py) on the fresh seeds / GQA / left-padding
                          cases of tests/test_oracle_pin.py: its random weights, logits, post-splice labels, loss and CLIP features
  shell_argv.json         the command line of each of the reference's six Qwen training shells (shells/train/qwen/*.sh), as parsed flags
  keywords_stopping.json  the reference's KeywordsStoppingCriteria (llavamod/mm_utils.py:73-105) on tests/test_eval_host.py's cases

    LLAVAMOD_REFERENCE=<checkout of the original project> python tests/golden/make_ref_golden.py
"""
import json
import os
import re
import shlex
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

LIVE_CASES = [(11, 4, 4, "right"), (12, 4, 1, "right"), (13, 2, 2, "left")]
SHELLS = ["dense2dense_distillation.sh", "dense2sparse_distillation.sh", "finetune.sh", "finetune_moe.sh", "preference_distillation.sh",
          "pretrain.sh"]
KEYWORD_CASES = [("USER: hi ASSISTANT: There are two birds.<|endoftext|>", ["<|endoftext|>"]),
                 ("USER: hi ASSISTANT: There are two birds", ["<|endoftext|>"]),
                 ("USER: hi ASSISTANT: A small red square", ["red square", "zzz"]),
                 ("USER: hi ASSISTANT: A", ["red square"])]


def live_request(seed, heads, kv, side):
    """Inputs of one live case: 3 ragged samples with 0, 1 and 2 images, one padded row."""
    g = torch.Generator().manual_seed(seed)
    B, T = 3, 12
    ids = torch.randint(0, 97, (B, T), generator=g)
    ids[0, 1] = -200; ids[2, 4] = -200; ids[2, 9] = -200
    mask = torch.ones(B, T, dtype=torch.bool); mask[1, 8:] = False
    labels = ids.clone(); labels[:, :3] = -100
    images = [torch.randn(3, 32, 32, generator=g) for _ in range(4)]
    kw = dict(hidden=64, inter=96, layers=1, heads=heads, kv_heads=kv, vocab=97, seed=seed)
    return dict(kw=kw, input_ids=ids, labels=labels, attention_mask=mask, images=images, padding_side=side, clip_images=torch.stack(images[:2]))


def live_key(seed, heads, kv, side):
    return "%d-%d-%d-%s" % (seed, heads, kv, side)


def shell_argv(path):
    """(flags, script) of the deepspeed launch line of a training shell, shell variables substituted."""
    text = open(path).read()
    env = {}
    for m in re.finditer(r"^([A-Z_][A-Z0-9_]*)=(.*)$", text, re.M):
        if "deepspeed" in m.group(2):                             # the launch line itself starts with VAR=1 VAR=1 deepspeed ...
            continue
        val = shlex.split(m.group(2).split("#")[0])
        env[m.group(1)] = val[0] if val else ""
    cmd = re.sub(r"\\[ \t]*\n", " ", text[text.index("deepspeed llavamod/train/"):])
    cmd = re.sub(r"\$\{(\w+)\}", lambda m: env.get(m.group(1), "x"), cmd)
    toks = shlex.split(cmd)
    return toks[2:], toks[1]                                      # drop "deepspeed <script>"


def keywords_reference(ref_root):
    code = r'''
import json, os, sys, types, torch
sys.path.insert(0, %r)
from tests.golden.make_data_golden import load_tokenizer
base = os.path.join(%r, "llavamod")
m = types.ModuleType("llavamod"); m.__path__ = [base]; sys.modules["llavamod"] = m
from llavamod.mm_utils import KeywordsStoppingCriteria
tok = load_tokenizer(%r)
out = []
for text, kws in %r:
    ids = torch.tensor([tok(text).input_ids])
    crit = KeywordsStoppingCriteria(kws, tok, ids[:, :5])
    out.append([bool(crit(ids[:, :n], None)) for n in range(6, ids.shape[1] + 1)])
print("RESULT" + json.dumps(out))
''' % (ROOT, ref_root, os.path.join(HERE, "tiny_tokenizer.json"), KEYWORD_CASES)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, check=True)
    return json.loads([line for line in r.stdout.splitlines() if line.startswith("RESULT")][0][6:])


def main():
    sys.path.insert(0, ROOT)
    from oracle import ref_shim
    if not ref_shim.available():
        raise SystemExit("set LLAVAMOD_REFERENCE to a checkout of the original project")
    for c in LIVE_CASES:
        torch.save(ref_shim.run_child(live_request(*c)), os.path.join(HERE, "ref_live_%s.pt" % live_key(*c)))
    shells = {}
    for s in SHELLS:
        argv, script = shell_argv(os.path.join(ref_shim.REF_ROOT, "shells", "train", "qwen", s))
        shells[s] = {"argv": argv, "script": script}
    with open(os.path.join(HERE, "shell_argv.json"), "w") as f:
        json.dump(shells, f, indent=1)
    with open(os.path.join(HERE, "keywords_stopping.json"), "w") as f:
        json.dump({"cases": KEYWORD_CASES, "want": keywords_reference(ref_shim.REF_ROOT)}, f)


if __name__ == "__main__":
    main()
