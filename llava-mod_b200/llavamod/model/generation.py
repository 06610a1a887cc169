"""Autoregressive decoding for the eval path (SURVEY section 8f row N4).

The reference's evaluation scripts call HF `generate` with `use_cache=False` (llavamod/eval/model_vqa_loader.py:119-130; the
DeepSpeed-MoE eval classes do not carry a KV cache through `MoEQwen1_5Model_forward`), i.e. every new token re-runs the multimodal
splice and the whole decoder on the sequence so far.  This module does the same thing on the CUDA path -- the prefill kernels
(wgmma GEMMs, flash attention, fused router) are the hot path here -- with two savings that do not change the result: the CLIP tower
+ projector run once per call instead of once per token, and lm_head is applied to the last position only.  Routing uses
`eval_capacity_factor` (model.eval()), and, as in the reference, fresh Gumbel noise for the second expert at every step
(DeepSpeed top2gating adds it regardless of train / eval).

Supported: greedy, temperature / top-p sampling, num_beams == 1, EOS and `stopping_criteria` callables, batch of equal-length prompts.
`use_cache=True` is accepted and ignored with a note (same tokens, the cache would only change speed)."""
import torch

from .. import kernels as K


@torch.no_grad()
def next_token_logits(model, input_ids, images=None, tower_features=None, attention_mask=None):
    """fp32 logits of the position after the last one: [B, V]."""
    r = model.forward_hidden(input_ids=input_ids, attention_mask=attention_mask, labels=None, images=images, tower_features=tower_features)
    last = r["hidden"][:, -1, :].contiguous()
    return K.mm_nt(last, model.lm_head.weight).float()


def _top_p_filter(logits, top_p):
    """HF TopPLogitsWarper: keep the smallest set of tokens whose probability mass reaches top_p (at least one)."""
    sorted_logits, idx = torch.sort(logits, descending=False, dim=-1)
    cum = sorted_logits.softmax(dim=-1).cumsum(dim=-1)
    remove = cum <= (1.0 - top_p)
    remove[..., -1:] = False
    return logits.masked_fill(remove.scatter(-1, idx, remove), float("-inf"))


@torch.no_grad()
def generate(model, inputs=None, images=None, attention_mask=None, max_new_tokens=20, do_sample=False, temperature=1.0, top_p=None,
             num_beams=1, use_cache=False, stopping_criteria=None, eos_token_id=None, pad_token_id=None, generator=None, **unused):
    """-> [B, T_in + n_new] int64: the prompt ids (image placeholders -200 included, as HF returns them) followed by the new tokens."""
    if num_beams != 1:
        raise NotImplementedError("beam search is not built (the reference's eval shells run num_beams=1)")
    if attention_mask is not None and not bool(attention_mask.all()):
        raise NotImplementedError("padded prompt batches: decode one prompt (or equal-length prompts) per call, as the reference's eval loaders do")
    was_training = model.training
    model.eval()
    dev = model.device
    ids = inputs.to(dev)
    eos = eos_token_id if eos_token_id is not None else getattr(model.config, "eos_token_id", None)
    eos = [eos] if isinstance(eos, int) else (list(eos) if eos is not None else [])
    pad = pad_token_id if pad_token_id is not None else (eos[0] if eos else 0)
    n_vocab = getattr(model, "_active_vocab", None)                     # resize_token_embeddings(len(tokenizer)) narrows the usable vocabulary
    feats = None
    if images is not None and model.get_image_tower() is not None:       # tower + projector once; the splice still runs every step
        imgs = torch.stack([im.to(dev) for im in images]) if not torch.is_tensor(images) else images.to(dev)
        feats = model.get_image_tower()(imgs.to(model.dtype))
        images = imgs
    B = ids.shape[0]
    done = torch.zeros(B, dtype=torch.bool, device=dev)
    for _ in range(int(max_new_tokens)):
        logits = next_token_logits(model, ids, images=images, tower_features=feats)
        if n_vocab is not None and n_vocab < logits.shape[-1]:
            logits[:, n_vocab:] = float("-inf")
        if do_sample:
            if temperature is not None and temperature != 1.0:
                logits = logits / float(temperature)
            if top_p is not None and top_p < 1.0:
                logits = _top_p_filter(logits, float(top_p))
            nxt = torch.multinomial(logits.softmax(dim=-1), 1, generator=generator).squeeze(1)
        else:
            nxt = logits.argmax(dim=-1)
        nxt = torch.where(done, torch.full_like(nxt, pad), nxt)
        ids = torch.cat([ids, nxt[:, None]], dim=1)
        for e in eos:
            done |= nxt == e
        stop = bool(done.all())
        if not stop and stopping_criteria:
            stop = any(bool(c(ids, logits)) for c in stopping_criteria)      # transformers.StoppingCriteriaList.__call__: any criterion stops
        if stop:
            break
    if was_training:
        model.train()
    return ids
