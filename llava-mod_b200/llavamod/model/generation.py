"""Autoregressive decoding for the eval path (SURVEY section 8f row N4).

use_cache=False (the default, and what eval/model_vqa_loader.py:119-130 passes): every new token re-runs the multimodal splice and the
whole decoder on the sequence so far, with two savings that do not change the result: the CLIP tower + projector run once per call
instead of once per token, and lm_head is applied to the last position only.  Routing uses `eval_capacity_factor` (model.eval()), and,
as in the reference, fresh Gumbel noise for the second expert at every step (DeepSpeed top2gating adds it regardless of train / eval),
so the prefix tokens of the sparse student are re-routed at every step.

use_cache=True (what the reference's other eval entry points pass, e.g. eval/model_vqa.py:85, serve/cli.py:109): the prompt is routed
and attended once (prefill into a KVCache), then each step runs the B new tokens through the decoder against the cached K / V
(csrc/decode.cu).  For the dense models this gives the tokens of the no-cache loop up to bf16 rounding; for the sparse student it is a
different function, the one the reference computes with a cache: each step routes only its B tokens (top2gating with S = B, capacity
ceil(B/E * eval_cf * 2) raised to min_capacity, fresh noise), and the prefix keeps the routing of the prefill.
The decode step (embedding, layers, final norm, lm_head over B rows) is captured as a CUDA graph after one eager step and replayed
(LLAVAMOD_CUDA_GRAPHS=0: eager).  Caches are sized to a multiple of CACHE_BUCKET positions, so an eval loop over prompts of different
lengths reuses a few graphs; at most LLAVAMOD_MAX_GRAPHS (cache, graph) pairs are kept, least recently used dropped first.

Supported: greedy, temperature / top-p sampling, num_beams == 1, EOS and `stopping_criteria` callables, batch of equal-length prompts."""
import collections
import os
import weakref

import torch

from .. import kernels as K

CACHE_BUCKET = 512
_STEP_GRAPHS = collections.OrderedDict()     # (model id, B, max_len, weight pointers) -> dict(model, cache, graph, ids, logits)
_GRAPH_POOL = None


@torch.no_grad()
def next_token_logits(model, input_ids, images=None, tower_features=None, attention_mask=None, cache=None):
    """fp32 logits of the position after the last one: [B, V].  cache: prefill into it (empty) or decode one step (input_ids [B,1])."""
    r = model.forward_hidden(input_ids=input_ids, attention_mask=attention_mask, labels=None, images=images, tower_features=tower_features,
                             cache=cache)
    last = r["hidden"][:, -1, :].contiguous()
    return K.mm_nt(last, model.lm_head.weight).float()


def _top_p_filter(logits, top_p):
    """HF TopPLogitsWarper: keep the smallest set of tokens whose probability mass reaches top_p (at least one)."""
    sorted_logits, idx = torch.sort(logits, descending=False, dim=-1)
    cum = sorted_logits.softmax(dim=-1).cumsum(dim=-1)
    remove = cum <= (1.0 - top_p)
    remove[..., -1:] = False
    return logits.masked_fill(remove.scatter(-1, idx, remove), float("-inf"))


def _graphs_enabled():
    return bool(int(os.environ.get("LLAVAMOD_CUDA_GRAPHS", "1")))


def _decoder_entry(model, B, max_len):
    """(cache, graph slot) for B sequences of up to max_len positions, reused across calls while graphs are on.  A captured step holds
    the addresses of the cache buffers and of the weights, and the host decisions made while it was captured: the MoE capacity rule of
    every sparse layer and the epilogue-fusion switches.  All of them are part of the key."""
    if not _graphs_enabled():
        return dict(cache=model.new_kv_cache(B, max_len), graph=None)
    for k in [k for k, v in _STEP_GRAPHS.items() if v["model"]() is None]:       # the model is gone: free its cache and graph
        del _STEP_GRAPHS[k]
    moe = tuple((l.mlp.num_experts, l.mlp.capacity_factor, l.mlp.eval_capacity_factor, l.mlp.min_capacity)
                for l in model.model.layers if hasattr(l.mlp, "deepspeed_moe"))
    key = (id(model), B, max_len, model.training, moe, K.FUSE_SWIGLU, K.FUSE_ROPE, K.FUSE_RESIDUAL,
           tuple(p.data_ptr() for p in model.parameters()))
    ent = _STEP_GRAPHS.pop(key, None)
    if ent is None or ent["model"]() is not model:
        ent = dict(model=weakref.ref(model), cache=model.new_kv_cache(B, max_len), graph=None)
    _STEP_GRAPHS[key] = ent
    while len(_STEP_GRAPHS) > max(1, int(os.environ.get("LLAVAMOD_MAX_GRAPHS", "6"))):
        _STEP_GRAPHS.popitem(last=False)
    ent["cache"].len.zero_()
    ent["cache"].length = 0
    return ent


def _decode_step(model, ent, tok, eager):
    """fp32 logits [B, V] of the next position after feeding tok [B] at the cache's current length."""
    global _GRAPH_POOL
    cache = ent["cache"]
    if eager:
        return next_token_logits(model, tok[:, None], cache=cache)
    if ent["graph"] is None:
        ent["ids"] = tok.clone()
        n0 = cache.length
        g = torch.cuda.CUDAGraph()
        if _GRAPH_POOL is None:
            _GRAPH_POOL = torch.cuda.graph_pool_handle()
        with torch.cuda.graph(g, pool=_GRAPH_POOL):
            ent["logits"] = next_token_logits(model, ent["ids"][:, None], cache=cache)
        cache.length = n0                       # the capture ran the host code of a step; nothing ran on the device
        ent["graph"] = g
    cache.check(tok.shape[0], 1)
    ent["ids"].copy_(tok)
    ent["graph"].replay()
    cache.length += 1
    return ent["logits"].clone()


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
    ent = None
    if use_cache and int(max_new_tokens) > 0:
        need = model.spliced_length(ids, images) + int(max_new_tokens)
        ent = _decoder_entry(model, B, (need + CACHE_BUCKET - 1) // CACHE_BUCKET * CACHE_BUCKET)
        logits = next_token_logits(model, ids, images=images, tower_features=feats, cache=ent["cache"])
    for step in range(int(max_new_tokens)):
        if ent is None:
            logits = next_token_logits(model, ids, images=images, tower_features=feats)
        elif step > 0:
            eager = not _graphs_enabled() or (step == 1 and ent["graph"] is None)      # one eager step before the capture
            logits = _decode_step(model, ent, nxt, eager)
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
