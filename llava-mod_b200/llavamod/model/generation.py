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

Padded prompt batches (attention_mask with zeros; each row's real tokens contiguous, on either side): every sequence is decoded as if
it were alone.  Any input padding side and any config.tokenizer_padding_side give the same tokens.  Positions run 0 .. n_b - 1 over
sequence b's n_b real spliced rows and cached steps continue at n_b + s; every step reads the next-token logits from each sequence's last
real row; a sequence attends to its own real keys only.  So for the dense models a sequence's result does not depend on the other
prompts.  The sparse student's prefill is the padded forward: pad rows are routed and count toward S and the capacity, as DeepSpeed
routes every row of a batch, and each cached step routes its B tokens; prompts are coupled only through routing, as in any batch.
The result is HF's layout: the input ids as given, pads included, followed by the new tokens.  Prompts without padding take the
unpadded path unchanged.  (The reference's own batched decoding differs from this for padded image batches and right-padded batches,
DESIGN section 8.)

Assisted (speculative) decoding, generate(..., assistant_model=draft, num_assistant_tokens=k), HF's names with k fixed per call: the
draft (dense or sparse, e.g. the distilled student) proposes k tokens with k + 1 of its own one-token cached steps, the target (dense)
scores all of them in one cached step of k + 1 tokens per sequence, and lmod_spec_accept (csrc/spec.cu) decides on the device how many
are kept, picks the next token and rolls both caches back; the host reads (n_acc, next) once per round.  Greedy: the target's argmax
is kept wherever it differs from the draft, and the verify step gives each row the bytes of a one-token step, so the tokens are exactly
those of generate(use_cache=True) on the target.  Sampling follows Leviathan et al. (HF _speculative_sampling): the tokens have the
target's distribution.  Both models prefill the prompt with their own tower; padded batches work as in plain cached decoding and
sequences accept different counts.  EOS and max_new_tokens are applied to each round's tokens and stopping_criteria is called once per
round, as HF does.  The per-call counts are kept in `last_assisted_stats`.

num_return_sequences = n (sampling only, as in transformers 4.37): n sampled answers per prompt, returned as [B*n, T_in + new] with row
b*n + j copy j of prompt b, and EOS, padding, max_new_tokens and stopping_criteria applied per row, as for the expanded batch.  A dense
model with use_cache=True runs the tower, projector and prefill once per prompt into a shared KVCache (the prompt's K / V held once,
each copy's new rows apart, lmod_attn_decode_shared reading the prompt's rows once for several copies), repeats the B prefill logits to
B*n rows before the logits processors and the draw, and then decodes B*n rows per cached step.  Every kernel of that path gives each row
the bytes it has in the expanded call, so the tokens are exactly those of generate on the inputs expanded with repeat_interleave(n, 0) and
a generator in the same state.  The sparse student (whose router draws fresh noise for every row, so the copies' K / V differ after its
first MoE layer) and use_cache=False run that expanded call itself.

Beam search, num_beams = nb > 1 with do_sample=False (transformers 4.37 beam_search + BeamSearchScorer, length_penalty, early_stopping
True / False / "never", num_return_sequences <= nb): each step's fp32 log-softmax over the active vocabulary plus the beam scores, the top
max(2, 1 + n_eos) * nb candidates of [B, nb * V] read to the host once, 4.37's process / is_done / finalize in BeamScorer, output
[B*n, T_in + new] with row b*n + j the j-th best hypothesis of prompt b.  A dense model with use_cache=True prefills each prompt once
into the shared cache of num_return_sequences (same graph key as num_return_sequences = nb) and lmod_kv_beam_reorder moves only the
beams' rows past the prompt after each step; the sparse student decodes the inputs expanded nb times in a plain cache whose every row the
same kernel reorders (HF's whole-cache reorder); use_cache=False re-runs each beam's sequence and reorders the ids.  Beam search needs
an EOS id (the call's eos_token_id or the model config's): without one it raises NotImplementedError.

Supported: greedy, temperature / top-p sampling, beam search, num_return_sequences with sampling or beams, EOS and `stopping_criteria`
callables, padded or unpadded batches, assisted decoding with a dense target.  Not built: beam-sample, beams with an assistant."""
import collections
import os
import weakref

import torch

from .. import kernels as K

CACHE_BUCKET = 512
SUFFIX_BUCKET = 64                           # rows per copy past its prompt in a shared cache, rounded up to this
_STEP_GRAPHS = collections.OrderedDict()     # (model id, B, max_len, T, weight pointers[, share]) -> dict(model, cache, graph, ids, logits)
_GRAPH_POOL = None
last_assisted_stats = None                   # counts of the last assisted generate call: rounds, drafted and accepted per sequence


@torch.no_grad()
def next_token_logits(model, input_ids, images=None, tower_features=None, attention_mask=None, cache=None, ragged=False):
    """fp32 logits of the position after the last one: [B, V].  cache: prefill into it (empty) or decode one step (input_ids [B,1]).
    ragged: attention_mask has padding -- the logits of each sequence's last real row (of the spliced mask), gathered on the device."""
    r = model.forward_hidden(input_ids=input_ids, attention_mask=attention_mask, labels=None, images=images, tower_features=tower_features,
                             cache=cache)
    h = r["hidden"]
    if ragged:
        B, T, H = h.shape
        rows = ((K.pad_ranges(r["attention_mask"])[1] - 1) + torch.arange(B, device=h.device, dtype=torch.int32) * T).to(torch.int32)
        last = K.gather_rows(h.reshape(B * T, H), rows, torch.full((1,), B, dtype=torch.int32, device=h.device),
                             out=torch.empty(B, H, dtype=h.dtype, device=h.device))
    else:
        last = h[:, -1, :].contiguous()
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


def _decoder_entry(model, B, max_len, T=1, share=1, suffix=None):
    """(cache, graph slot) for B sequences of up to max_len positions and steps of T tokens per sequence, reused across calls while graphs
    are on (T > 1: the verify step of assisted decoding; a model that is its own assistant gets one entry per width).  A captured step holds
    the addresses of the cache buffers and of the weights, and the host decisions made while it was captured: the MoE capacity rule of
    every sparse layer and the epilogue-fusion switches.  All of them are part of the key; the e4m3 buffers of a quantize_fp8_ model are not
    Parameters, so they are listed beside them (a step captured before the quantisation is never replayed after it).
    share = n > 1: a shared cache of B prompts with n sequences each and `suffix` rows per sequence past its prompt (num_return_sequences);
    n and suffix are part of the key, which is unchanged for n = 1."""
    if not _graphs_enabled():
        return dict(cache=model.new_kv_cache(B, max_len, share=share, suffix=suffix), graph=None)
    for k in [k for k, v in _STEP_GRAPHS.items() if v["model"]() is None]:       # the model is gone: free its cache and graph
        del _STEP_GRAPHS[k]
    moe = tuple((l.mlp.num_experts, l.mlp.k, l.mlp.use_residual, l.mlp.capacity_factor, l.mlp.eval_capacity_factor, l.mlp.min_capacity)
                for l in model.model.layers if hasattr(l.mlp, "deepspeed_moe"))
    fp8 = tuple(t.data_ptr() for l in model.model.layers if isinstance(l.self_attn.qkv_weight, K.Fp8Rows)
                for w in (l.self_attn.qkv_weight, l.self_attn.o_fp8, l.mlp.gu_weight, l.mlp.down_fp8) for t in (w.q, w.scale))
    key = (id(model), B, max_len, T, model.training, moe, tuple(p.data_ptr() for p in model.parameters()), fp8)
    if share > 1:
        key += (("share", share, suffix),)
    ent = _STEP_GRAPHS.pop(key, None)
    if ent is None or ent["model"]() is not model:
        ent = dict(model=weakref.ref(model), cache=model.new_kv_cache(B, max_len, share=share, suffix=suffix), graph=None)
    _STEP_GRAPHS[key] = ent
    while len(_STEP_GRAPHS) > max(1, int(os.environ.get("LLAVAMOD_MAX_GRAPHS", "6"))):
        _STEP_GRAPHS.popitem(last=False)
    ent["cache"].reset()
    return ent


@torch.no_grad()
def chunk_logits(model, input_ids, cache):
    """fp32 logits [B, T, V] of every position of a cached step of input_ids [B, T]."""
    h = model.forward_hidden(input_ids=input_ids, cache=cache)["hidden"]
    B, T, H = h.shape
    return K.mm_nt(h.reshape(B * T, H), model.lm_head.weight).float().view(B, T, -1)


def _decode_step(model, ent, tok, eager):
    """fp32 logits [B, V] of the next position after feeding tok [B] at the cache's current length; tok [B, T]: logits [B, T, V] of
    the T positions (one cached step of T tokens per sequence)."""
    global _GRAPH_POOL
    cache = ent["cache"]
    step = (lambda ids: next_token_logits(model, ids[:, None], cache=cache)) if tok.dim() == 1 else (lambda ids: chunk_logits(model, ids, cache))
    if eager:
        return step(tok)
    if ent["graph"] is None:
        ent["ids"] = tok.clone()
        n0 = list(cache.lengths)
        g = torch.cuda.CUDAGraph()
        if _GRAPH_POOL is None:
            _GRAPH_POOL = torch.cuda.graph_pool_handle()
        with torch.cuda.graph(g, pool=_GRAPH_POOL):
            ent["logits"] = step(ent["ids"])
        cache.lengths = n0                      # the capture ran the host code of a step; nothing ran on the device
        ent["graph"] = g
    T = 1 if tok.dim() == 1 else tok.shape[1]
    cache.check(tok.shape[0], T)
    ent["ids"].copy_(tok)
    ent["graph"].replay()
    cache.advance(T)
    return ent["logits"].clone()


def _process(logits, n_vocab, do_sample, temperature, top_p):
    """The logits processors of a step: the narrowed vocabulary, then (sampling) temperature and top-p.  In place where possible."""
    if n_vocab is not None and n_vocab < logits.shape[-1]:
        logits[..., n_vocab:] = float("-inf")
    if do_sample:
        if temperature is not None and temperature != 1.0:
            logits = logits / float(temperature)
        if top_p is not None and top_p < 1.0:
            logits = _top_p_filter(logits, float(top_p))
    return logits


def _pick(logits, do_sample, generator):
    if do_sample:
        return torch.multinomial(logits.softmax(dim=-1), 1, generator=generator).squeeze(1)
    return logits.argmax(dim=-1)


class BeamsWithAssistantError(ValueError, NotImplementedError):
    """num_beams > 1 with an assistant model: a ValueError, as transformers raises, and a NotImplementedError, as beams with an assistant
    are not built here (callers written against either keep working)."""


@torch.no_grad()
def generate(model, inputs=None, images=None, attention_mask=None, max_new_tokens=20, do_sample=False, temperature=1.0, top_p=None,
             num_beams=1, use_cache=False, stopping_criteria=None, eos_token_id=None, pad_token_id=None, generator=None,
             assistant_model=None, num_assistant_tokens=5, num_return_sequences=1, length_penalty=1.0, early_stopping=False, **unused):
    """-> [B*n, T_in + n_new] int64 (n = num_return_sequences): the prompt ids (image placeholders -200 included, pads included, as HF
    returns them) followed by the new tokens; row b*n + j is copy j of prompt b.  assistant_model: a draft model for assisted decoding
    (use_cache=True, dense target), num_assistant_tokens = k drafted tokens per round.  num_return_sequences: n sampled sequences per
    prompt (do_sample=True); a dense model with use_cache=True prefills each prompt once into a shared cache, the sparse student and
    use_cache=False decode the inputs expanded with repeat_interleave(n, 0) (module docstring)."""
    n_ret = int(num_return_sequences) if num_return_sequences is not None else 1
    if n_ret < 1:
        raise ValueError("generate: num_return_sequences must be >= 1, got %r" % (num_return_sequences,))
    nb = int(num_beams) if num_beams is not None else 1
    if nb < 1:
        raise ValueError("generate: num_beams must be >= 1, got %r" % (num_beams,))
    if nb > 1:
        if do_sample:
            raise NotImplementedError("beam-sample (num_beams > 1 with do_sample=True) is not built; beam search runs with do_sample=False")
        if assistant_model is not None:
            raise BeamsWithAssistantError("assisted generate is only supported with num_beams = 1, got num_beams = %d" % nb)
        if n_ret > nb:
            raise ValueError("num_return_sequences (%d) has to be smaller or equal to num_beams (%d)" % (n_ret, nb))
        return _beam_search(model, inputs, images=images, attention_mask=attention_mask, max_new_tokens=max_new_tokens, num_beams=nb,
                            num_return_sequences=n_ret, length_penalty=length_penalty, early_stopping=early_stopping, use_cache=use_cache,
                            stopping_criteria=stopping_criteria, eos_token_id=eos_token_id, pad_token_id=pad_token_id)
    if n_ret > 1 and not do_sample:
        raise ValueError("num_return_sequences has to be 1 when doing greedy search, but is %d." % n_ret)
    if n_ret > 1 and assistant_model is not None:
        raise ValueError("num_return_sequences has to be 1 when doing assisted generate, but is %d." % n_ret)
    if assistant_model is not None:
        if not use_cache:
            raise ValueError("generate: assisted decoding needs use_cache=True (the draft and the verify step decode against KV caches)")
        if getattr(model, "is_moe", False):
            raise ValueError("generate: assisted decoding needs a dense target; a sparse model cannot verify k + 1 tokens in one step "
                             "(it would route them together)")
        if int(num_assistant_tokens) < 1:
            raise ValueError("generate: num_assistant_tokens must be >= 1, got %r" % (num_assistant_tokens,))
    dev = model.device
    share = n_ret > 1 and use_cache and int(max_new_tokens) > 0 and not getattr(model, "is_moe", False)
    if n_ret > 1 and not share:                 # the sparse student, use_cache=False: the expanded call itself
        inputs, attention_mask, images = _expand(n_ret, inputs, attention_mask, images)
        n_ret = 1
    ids, mask, images, feats, eos, pad, n_vocab, was_training = _prepare(model, inputs, images, attention_mask, eos_token_id, pad_token_id)
    B = ids.shape[0]
    done = torch.zeros(B, dtype=torch.bool, device=dev)
    ent = None
    ragged = mask is not None
    if assistant_model is not None and int(max_new_tokens) > 0:
        ids = _assisted(model, assistant_model, ids, images, feats, mask, int(max_new_tokens), int(num_assistant_tokens), do_sample,
                        temperature, top_p, stopping_criteria, eos, pad, generator, n_vocab)
        if was_training:
            model.train()
        return ids
    if use_cache and int(max_new_tokens) > 0:
        need = max(model.spliced_length(ids, images, mask)) + int(max_new_tokens)
        max_len = (need + CACHE_BUCKET - 1) // CACHE_BUCKET * CACHE_BUCKET
        if n_ret > 1:          # each copy appends at most max_new_tokens - 1 rows past its prompt
            suffix = (int(max_new_tokens) + SUFFIX_BUCKET - 1) // SUFFIX_BUCKET * SUFFIX_BUCKET
            ent = _decoder_entry(model, B, max_len, share=n_ret, suffix=suffix)
        else:
            ent = _decoder_entry(model, B, max_len)
        logits = next_token_logits(model, ids, images=images, tower_features=feats, attention_mask=mask.to(dev) if ragged else None,
                                   cache=ent["cache"], ragged=ragged)
        if n_ret > 1:          # from here on B*n rows, the expanded call's layout; the draws see the expanded call's logits
            logits = logits.repeat_interleave(n_ret, 0)
            ids = ids.repeat_interleave(n_ret, 0)
            B = B * n_ret
            done = torch.zeros(B, dtype=torch.bool, device=dev)
    elif ragged:
        # the no-cache loop re-reads every prompt with its new tokens appended: each row holds its real tokens first, then the new ones,
        # then padding, so a row stays one run of real tokens and the unspliced text rows sit at positions 0 .. n_b - 1
        work = ids.gather(1, torch.argsort((~mask).to(torch.int8), dim=1, stable=True).to(dev))
        wlen = mask.sum(1).to(dev)
    for step in range(int(max_new_tokens)):
        if ent is None and ragged:
            wmask = torch.arange(work.shape[1], device=dev)[None, :] < wlen[:, None]
            logits = next_token_logits(model, work, images=images, tower_features=feats, attention_mask=wmask, ragged=True)
        elif ent is None:
            logits = next_token_logits(model, ids, images=images, tower_features=feats)
        elif step > 0:
            eager = not _graphs_enabled() or (step == 1 and ent["graph"] is None)      # one eager step before the capture
            logits = _decode_step(model, ent, nxt, eager)
        logits = _process(logits, n_vocab, do_sample, temperature, top_p)
        nxt = _pick(logits, do_sample, generator)
        nxt = torch.where(done, torch.full_like(nxt, pad), nxt)
        ids = torch.cat([ids, nxt[:, None]], dim=1)
        if ent is None and ragged:
            work = torch.cat([work, torch.full_like(nxt[:, None], pad)], dim=1).scatter_(1, wlen[:, None], nxt[:, None])
            wlen = wlen + 1
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


def _prepare(model, inputs, images, attention_mask, eos_token_id, pad_token_id):
    """What every decoding loop starts from: the prompt ids on the device; the prompt mask (bool, host) when some prompt is padded, else None
    (every prompt's real tokens must be one contiguous run); the images on the device with the tower + projector run once (the splice still
    runs every step); the EOS ids, the pad id, the active vocabulary and whether the model was training (it is left in eval mode)."""
    dev = model.device
    ids = inputs.to(dev)
    mask = None
    if attention_mask is not None:
        m = attention_mask.cpu().bool()
        if not bool(m.all()):
            n_real = m.sum(1)
            if bool((n_real == 0).any()):
                raise ValueError("generate: prompt %d has no real token" % int((n_real == 0).nonzero()[0]))
            first = m.int().argmax(1)
            if not bool((m.int().cumsum(1).gather(1, (first + n_real - 1)[:, None]).squeeze(1) == n_real).all()):
                raise ValueError("generate: every prompt's real tokens must be contiguous (left or right padding)")
            mask = m
    was_training = model.training
    model.eval()
    eos = eos_token_id if eos_token_id is not None else getattr(model.config, "eos_token_id", None)
    eos = [eos] if isinstance(eos, int) else (list(eos) if eos is not None else [])
    pad = pad_token_id if pad_token_id is not None else (eos[0] if eos else 0)
    n_vocab = getattr(model, "_active_vocab", None)                     # resize_token_embeddings(len(tokenizer)) narrows the usable vocabulary
    feats = None
    if images is not None and model.get_image_tower() is not None:
        imgs = torch.stack([im.to(dev) for im in images]) if not torch.is_tensor(images) else images.to(dev)
        feats = model.get_image_tower()(imgs.to(model.dtype))
        images = imgs
    return ids, mask, images, feats, eos, pad, n_vocab, was_training


def _expand(n, inputs, attention_mask, images):
    """HF's _expand_inputs_for_generation: input_ids, attention_mask and images repeated n times along the batch (repeat_interleave)."""
    if attention_mask is not None:
        attention_mask = attention_mask.repeat_interleave(n, 0)
    if images is not None:
        images = images.repeat_interleave(n, 0) if torch.is_tensor(images) else [im for im in images for _ in range(n)]
    return inputs.repeat_interleave(n, 0), attention_mask, images


def _bucket(n):
    return (n + CACHE_BUCKET - 1) // CACHE_BUCKET * CACHE_BUCKET


def _assisted(model, draft, ids, images, feats, mask, max_new, k, do_sample, temperature, top_p, stopping_criteria, eos, pad, generator,
              n_vocab):
    """Assisted decoding (module docstring).  Each round ends with both caches at base + n_acc + 1 rows: the draft's k + 1 steps and the
    verify step add k + 1, lmod_spec_accept takes back the k - n_acc rejected ones.  A sequence that is finished (EOS or max_new tokens)
    keeps running with the batch, but its cache rows are taken back after every round, so no cache grows past what it was sized for."""
    global last_assisted_stats
    dev = model.device
    B = ids.shape[0]
    ragged = mask is not None
    dmask = mask.to(dev) if ragged else None
    was_training = draft.training
    draft.eval()
    dfeats = None
    if images is not None and draft.get_image_tower() is not None:
        dfeats = draft.get_image_tower()(images.to(draft.dtype))
    d_vocab = [v for v in (getattr(draft, "_active_vocab", None), n_vocab) if v is not None]
    d_vocab = min(d_vocab) if d_vocab else None
    ent_t = _decoder_entry(model, B, _bucket(max(model.spliced_length(ids, images, mask)) + max_new + k + 1), T=k + 1)
    ent_d = _decoder_entry(draft, B, _bucket(max(draft.spliced_length(ids, images, mask)) + max_new + k + 1))
    ct, cd = ent_t["cache"], ent_d["cache"]
    logits = next_token_logits(model, ids, images=images, tower_features=feats, attention_mask=dmask, cache=ct, ragged=ragged)
    draft.forward_hidden(input_ids=ids, attention_mask=dmask, images=images, tower_features=dfeats, cache=cd)
    logits = _process(logits, n_vocab, do_sample, temperature, top_p)
    first = _pick(logits, do_sample, generator)
    out = [[t] for t in first.tolist()]
    done = [bool(eos) and row[0] in eos for row in out]
    last = first
    rounds, drafted, accepted = 0, [0] * B, [0] * B
    graphs = _graphs_enabled()
    warm = set()

    def step(ent, tok):
        eager = not graphs or (ent["graph"] is None and id(ent) not in warm)       # one eager step of each entry before its capture
        warm.add(id(ent))
        return _decode_step(draft if ent is ent_d else model, ent, tok, eager)

    def complete(b):
        return done[b] or len(out[b]) >= max_new

    stop = all(complete(b) for b in range(B))
    if not stop and stopping_criteria:
        stop = any(bool(c(_assemble(ids, out, pad, max_new), logits)) for c in stopping_criteria)
    while not stop:
        active = [not complete(b) for b in range(B)]
        base_t, base_d = list(ct.lengths), list(cd.lengths)
        tok, dtoks, dlogits = last, [], []
        for j in range(k + 1):
            lg = step(ent_d, tok)
            if j == k:
                break                                # the last draft step only puts d_k into the draft's cache
            lg = _process(lg, d_vocab, do_sample, temperature, top_p)
            tok = _pick(lg, do_sample, generator)
            dtoks.append(tok)
            if do_sample:
                dlogits.append(lg)
        dtoks = torch.stack(dtoks, 1)
        vlogits = step(ent_t, torch.cat([last[:, None], dtoks], 1))
        vlogits = _process(vlogits, n_vocab, do_sample, temperature, top_p)
        if do_sample:
            u = torch.rand(B, k + 1, device=dev, dtype=torch.float32, generator=generator)
            n_acc, nxt = K.spec_accept(vlogits, dtoks, torch.stack(dlogits, 1), u, ct.len, cd.len)
        else:
            n_acc, nxt = K.spec_accept(vlogits, dtoks, None, None, ct.len, cd.len)
        host = torch.cat([n_acc.to(torch.int64), nxt, dtoks.reshape(-1)]).tolist()      # the round's one device-to-host read
        n_acc, nxt, dt = host[:B], host[B:2 * B], host[2 * B:]
        ct.rollback([k - n for n in n_acc])
        cd.rollback([k - n for n in n_acc])
        rounds += 1
        for b in range(B):
            if not active[b]:
                continue
            drafted[b] += k
            accepted[b] += n_acc[b]
            for t in dt[b * k:b * k + n_acc[b]] + [nxt[b]]:
                out[b].append(t)
                if t in eos:
                    done[b] = True
                    break
        # finished sequences: back to where they were, so their caches stay within their size
        drop = [0 if active[b] and not complete(b) else ct.lengths[b] - base_t[b] for b in range(B)]
        if any(drop):
            dd = torch.tensor(drop, dtype=torch.int32, device=dev)
            ct.len.sub_(dd)
            ct.rollback(drop)
            dd = torch.tensor([cd.lengths[b] - base_d[b] if drop[b] else 0 for b in range(B)], dtype=torch.int32, device=dev)
            cd.len.sub_(dd)
            cd.rollback(dd.tolist())
        last = torch.tensor([pad if done[b] else out[b][-1] for b in range(B)], dtype=torch.int64, device=dev)
        stop = all(complete(b) for b in range(B))
        if not stop and stopping_criteria:
            rows = torch.tensor(n_acc, dtype=torch.int64, device=dev)
            stop = any(bool(c(_assemble(ids, out, pad, max_new), vlogits[torch.arange(B, device=dev), rows])) for c in stopping_criteria)
    last_assisted_stats = dict(rounds=rounds, drafted=drafted, accepted=accepted)
    if was_training:
        draft.train()
    return _assemble(ids, out, pad, max_new)


def _assemble(ids, out, pad, max_new):
    """The prompt ids followed by each sequence's new tokens, as many columns as the longest (at most max_new), finished rows padded."""
    W = min(max_new, max(len(r) for r in out))
    new = torch.full((len(out), W), pad, dtype=torch.int64)
    for b, r in enumerate(out):
        r = r[:W]
        new[b, :len(r)] = torch.tensor(r, dtype=torch.int64)
    return torch.cat([ids, new.to(ids.device)], dim=1)


class BeamScorer:
    """transformers 4.37 BeamSearchScorer with BeamHypotheses (one beam group), on host numbers.  Lengths count new tokens only (the
    decoder prompt length is 0, as for HF's generate from inputs_embeds), so a hypothesis that ends in EOS at step s has length s + 1.
    hyps[b]: at most num_beams (score, new tokens without the EOS) of prompt b; done[b]: 4.37's _done."""

    def __init__(self, batch, num_beams, num_return_sequences, length_penalty, early_stopping, max_new_tokens, eos, pad):
        if early_stopping not in (True, False, "never"):
            raise ValueError("early_stopping must be True, False or 'never', got %r" % (early_stopping,))
        self.nb, self.n_ret, self.lp, self.es = int(num_beams), int(num_return_sequences), float(length_penalty), early_stopping
        self.max_new, self.eos, self.pad = int(max_new_tokens), list(eos), pad
        self.hyps = [[] for _ in range(batch)]
        self.worst = [1e9] * batch
        self.done = [False] * batch

    @property
    def is_done(self):
        return all(self.done)

    def _add(self, b, tokens, sum_logprobs, generated_len):
        """BeamHypotheses.add: keep the num_beams best by sum_logprobs / generated_len ** length_penalty."""
        score = sum_logprobs / (generated_len ** self.lp)
        hyps = self.hyps[b]
        if len(hyps) < self.nb or score > self.worst[b]:
            hyps.append((score, tokens))
            if len(hyps) > self.nb:
                ranked = sorted((s, i) for i, (s, _) in enumerate(hyps))
                del hyps[ranked[0][1]]
                self.worst[b] = ranked[1][0]
            else:
                self.worst[b] = min(score, self.worst[b])

    def _is_done(self, b, best_sum_logprobs, cur_len):
        """BeamHypotheses.is_done with the three early_stopping modes."""
        if len(self.hyps[b]) < self.nb:
            return False
        if self.es is True:
            return True
        length = self.max_new if self.es == "never" and self.lp > 0.0 else cur_len
        return self.worst[b] >= best_sum_logprobs / length ** self.lp

    def process(self, cur_len, scores, tokens, beams, seqs):
        """BeamSearchScorer.process for the step that makes the new sequences cur_len tokens long.  scores / tokens / beams: per prompt, the
        top max(2, 1 + n_eos) * num_beams candidates, best first (summed log-prob, token, local beam); seqs: each running beam's new tokens.
        -> (next beam scores, next tokens, next local parents), num_beams per prompt; a done prompt takes pad tokens from beam 0 at 0."""
        nb = self.nb
        out_s, out_t, out_p = [], [], []
        for b in range(len(self.done)):
            if self.done[b]:
                out_s += [0.0] * nb
                out_t += [self.pad] * nb
                out_p += [0] * nb
                continue
            n = 0
            for rank, (s, t, j) in enumerate(zip(scores[b], tokens[b], beams[b])):
                if t in self.eos:
                    if rank < nb:                   # an EOS ranked below num_beams is not a hypothesis
                        self._add(b, seqs[b * nb + j], s, cur_len)
                else:
                    out_s.append(s)
                    out_t.append(t)
                    out_p.append(j)
                    n += 1
                if n == nb:
                    break
            if n < nb:
                raise ValueError("beam search: prompt %d has %d non-EOS candidates for %d beams" % (b, n, nb))
            self.done[b] = self.done[b] or self._is_done(b, max(scores[b]), cur_len)
        return out_s, out_t, out_p

    def finalize(self, seqs, scores):
        """BeamSearchScorer.finalize: the running beams of every prompt not done become hypotheses; -> num_return_sequences rows of new
        tokens per prompt, best first, as wide as the longest hypothesis + 1 (at most max_new_tokens); each row gets eos[0] after its tokens
        where it fits (4.37 inserts the first EOS id, also after a beam that stopped without one) and pad after that."""
        nb = self.nb
        for b in range(len(self.done)):
            if not self.done[b]:
                for j in range(nb):
                    self._add(b, seqs[b * nb + j], scores[b * nb + j], len(seqs[b * nb + j]))
        best = []
        for hyps in self.hyps:
            ranked = sorted(hyps, key=lambda h: h[0])
            best += [ranked.pop()[1] for _ in range(self.n_ret)]
        width = min(max(len(r) for r in best) + 1, self.max_new)
        rows = []
        for r in best:
            r = list(r) + ([self.eos[0]] if self.eos and len(r) < width else [])
            rows.append(r + [self.pad] * (width - len(r)))
        return rows


@torch.no_grad()
def _beam_search(model, inputs, images=None, attention_mask=None, max_new_tokens=20, num_beams=2, num_return_sequences=1, length_penalty=1.0,
                 early_stopping=False, use_cache=False, stopping_criteria=None, eos_token_id=None, pad_token_id=None, expand=False,
                 trace=None):
    """Beam search (transformers 4.37 beam_search + BeamSearchScorer; module docstring) -> [B*n, T_in + new], row b*n + j the j-th best
    hypothesis of prompt b.  Each step: fp32 log-softmax over the active vocabulary, plus each beam's score, the top max(2, 1 + n_eos) * nb
    candidates of [B, nb * V] read to the host once, BeamScorer.process, then the running ids and the cache follow the chosen parents.
    A dense model with use_cache=True prefills each prompt once into a shared cache and lmod_kv_beam_reorder moves the beams' rows past
    the prompt; the sparse student, or expand=True, decodes the inputs expanded nb times in a plain cache whose every row is reordered.
    trace: a list that receives every step's fp32 logits [B*nb, V] (the tests replay the scorer on them)."""
    nb, n_ret, max_new = int(num_beams), int(num_return_sequences), int(max_new_tokens)
    eos = eos_token_id if eos_token_id is not None else getattr(model.config, "eos_token_id", None)
    if eos is None or (not isinstance(eos, int) and len(list(eos)) == 0):
        # 4.37's scorer ends a hypothesis only at an EOS and its finalize writes eos_token_id[0] after every hypothesis shorter than the
        # output; without one, a search a stopping criterion ends early has no defined output.  A model config or the call gives one.
        raise NotImplementedError("beam search without an eos_token_id is not built: pass eos_token_id (the model config has none)")
    ids, mask, images, feats, eos, pad, n_vocab, was_training = _prepare(model, inputs, images, attention_mask, eos_token_id, pad_token_id)
    dev = model.device
    B = ids.shape[0]
    R = B * nb
    ragged = mask is not None
    if max_new <= 0:
        return ids.repeat_interleave(n_ret, 0)
    scorer = BeamScorer(B, nb, n_ret, length_penalty, early_stopping, max_new, eos, pad)
    shared = use_cache and not expand and not getattr(model, "is_moe", False)
    x_ids, x_mask, x_images = (ids, mask, images) if shared else _expand(nb, ids, mask, images)
    x_feats = feats if shared or feats is None else feats.repeat_interleave(nb, 0)
    ent = None
    if use_cache:
        max_len = _bucket(max(model.spliced_length(ids, images, mask)) + max_new)
        if shared:
            ent = _decoder_entry(model, B, max_len, share=nb, suffix=(max_new + SUFFIX_BUCKET - 1) // SUFFIX_BUCKET * SUFFIX_BUCKET)
        else:
            ent = _decoder_entry(model, R, max_len)
        logits = next_token_logits(model, x_ids, images=x_images, tower_features=x_feats, attention_mask=x_mask.to(dev) if ragged else None,
                                   cache=ent["cache"], ragged=ragged)
        if shared:
            logits = logits.repeat_interleave(nb, 0)
    elif ragged:        # as in generate's no-cache loop: each row's real tokens first, then its new ones, then padding
        work = x_ids.gather(1, torch.argsort((~x_mask).to(torch.int8), dim=1, stable=True).to(dev))
        wlen = x_mask.sum(1).to(dev)
    run = ids.repeat_interleave(nb, 0)                  # the running beams' ids, as stopping_criteria sees them
    beam_scores = torch.zeros(B, nb, dtype=torch.float32, device=dev)
    beam_scores[:, 1:] = -1e9
    beam_scores = beam_scores.view(-1)
    seqs = [[] for _ in range(R)]
    top = max(2, 1 + len(eos)) * nb
    for step in range(max_new):
        if ent is not None and step > 0:
            ent["cache"].reorder_beams(parents, nb)
            eager = not _graphs_enabled() or (step == 1 and ent["graph"] is None)      # one eager step before the capture
            logits = _decode_step(model, ent, tok, eager)
        elif ent is None and ragged:
            wmask = torch.arange(work.shape[1], device=dev)[None, :] < wlen[:, None]
            logits = next_token_logits(model, work, images=x_images, tower_features=x_feats, attention_mask=wmask, ragged=True)
        elif ent is None:
            logits = next_token_logits(model, run, images=x_images, tower_features=x_feats)
        if trace is not None:
            trace.append(logits.clone())
        V = n_vocab if n_vocab is not None and n_vocab < logits.shape[-1] else logits.shape[-1]
        lp = torch.log_softmax(logits[:, :V], dim=-1) + beam_scores[:, None]
        top_s, top_i = torch.topk(lp.view(B, nb * V), top, dim=1, largest=True, sorted=True)
        host = torch.stack([top_s.double(), top_i.double()]).tolist()      # the step's one device-to-host read
        idx = [[int(i) for i in row] for row in host[1]]
        nxt_s, nxt_t, parents = scorer.process(step + 1, host[0], [[i % V for i in row] for row in idx],
                                               [[i // V for i in row] for row in idx], seqs)
        src = [b * nb + p for b in range(B) for p in parents[b * nb:(b + 1) * nb]]
        seqs = [seqs[g] + [t] for g, t in zip(src, nxt_t)]
        src_d = torch.tensor(src, dtype=torch.int64).to(dev)
        tok = torch.tensor(nxt_t, dtype=torch.int64).to(dev)
        beam_scores = torch.tensor(nxt_s, dtype=torch.float32).to(dev)
        run = torch.cat([run.index_select(0, src_d), tok[:, None]], dim=1)
        if ent is None and ragged:
            work, wlen = work.index_select(0, src_d), wlen.index_select(0, src_d)
            work = torch.cat([work, torch.full_like(tok[:, None], pad)], dim=1).scatter_(1, wlen[:, None], tok[:, None])
            wlen = wlen + 1
        stop = scorer.is_done
        if not stop and stopping_criteria:
            stop = any(bool(c(run, lp)) for c in stopping_criteria)        # transformers.StoppingCriteriaList.__call__: any criterion stops
        if stop:
            break
    rows = scorer.finalize(seqs, nxt_s)
    if was_training:
        model.train()
    return torch.cat([ids.repeat_interleave(n_ret, 0), torch.tensor(rows, dtype=torch.int64, device=dev)], dim=1)
