"""Generates tests/golden/dense_*.<i>.pt (shards, see shards.py) by running the REFERENCE's own dense path
(LlavaQwen1_5ForCausalLM, imported in place through oracle/ref_shim.py) on seeded tiny inputs.
Run in the build container only (needs /root/reference):  python tests/golden/make_golden.py

Each fixture holds: the reference model's state_dict (reference key names), config numbers, the
inputs, and the reference outputs (logits fp32, post-splice labels, loss, a few parameter grads).
"""
import glob
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402
from tests.golden import shards  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))

CASES = {
    # name: (model kwargs, batch builder)
    "dense_mha": dict(kw=dict(hidden=128, inter=256, layers=2, heads=4, kv_heads=4, vocab=512, seed=0),
                      B=2, T=20, img_pos=[[3], [7]], pad=[0, 3]),
    "dense_gqa": dict(kw=dict(hidden=128, inter=192, layers=2, heads=4, kv_heads=2, vocab=384, seed=1),
                      B=3, T=24, img_pos=[[2, 11], [], [0]], pad=[0, 5, 9]),
    # head_dim 64 (2 heads x 64, CLIP 1 head x 64): the shapes our wgmma attention kernel is built for
    "dense_hd64": dict(kw=dict(hidden=128, inter=256, layers=2, heads=2, kv_heads=1, vocab=512, seed=3, clip_heads=1),
                       B=2, T=30, img_pos=[[4], [9]], pad=[0, 0]),
    "dense_nopad": dict(kw=dict(hidden=128, inter=256, layers=2, heads=4, kv_heads=4, vocab=512, seed=2),
                        B=2, T=16, img_pos=[[5], [5]], pad=[0, 0]),
}


def build_batch(case, vocab, gen):
    B, T = case["B"], case["T"]
    ids = torch.randint(0, vocab, (B, T), generator=gen)
    mask = torch.ones(B, T, dtype=torch.bool)
    n_img = 0
    for b in range(B):
        for p in case["img_pos"][b]:
            ids[b, p] = -200
        n_img += max(1, len(case["img_pos"][b]))     # a sample without <image> still owns one entry
        if case["pad"][b]:
            mask[b, T - case["pad"][b]:] = False
    labels = ids.clone()
    labels[:, : T // 3] = -100
    labels[~mask] = -100
    images = [torch.randn(3, 32, 32, generator=gen) for _ in range(n_img)]
    return ids, labels, mask, images


def main():
    tmp = tempfile.mkdtemp()
    for name, case in CASES.items():
        model = ref_shim.build_tiny_dense(os.path.join(tmp, name), **case["kw"])
        os.makedirs(os.path.join(tmp, name), exist_ok=True)
        gen = torch.Generator().manual_seed(100 + case["kw"]["seed"])
        ids, labels, mask, images = build_batch(case, case["kw"]["vocab"], gen)
        for p in model.parameters():
            p.requires_grad_(True)
        out = model(input_ids=ids, labels=labels, attention_mask=mask, images=images, return_dict=True)
        out.loss.backward()
        sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
        grads = {}
        for k, p in model.named_parameters():
            if p.grad is not None and any(s in k for s in ("mm_projector", "layers.0.mlp", "layers.1.self_attn.q_proj",
                                                           "model.norm", "lm_head")):
                grads[k] = p.grad.detach().clone()
        fx = dict(kw=case["kw"], input_ids=ids, labels=labels, attention_mask=mask, images=images,
                  state_dict=sd, logits=out.logits.detach(), out_labels=out.labels, loss=out.loss.detach(),
                  grads=grads)
        shards.save(fx, OUT, name)
        size = sum(os.path.getsize(p) for p in glob.glob(os.path.join(OUT, name + ".*.pt")))
        print(name, "logits", tuple(out.logits.shape), "loss", float(out.loss), "size", size // 1024, "KiB")


if __name__ == "__main__":
    main()
