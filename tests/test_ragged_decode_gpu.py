"""Decoding padded batches of prompts of different lengths through the KV cache (and without it): lmod_kv_append_rows against a torch
copy, every sequence of a padded batch against the same prompt alone at B = 1, the reference's own per-prompt cached decoding
(tests/golden/ragged_*.pt), the sparse student against the ragged oracle (tests/ragged_oracle.py), and generate()."""
import math
import warnings

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import restated as R  # noqa: E402
from tests import helpers as Hh  # noqa: E402
from tests import ragged_oracle as RO  # noqa: E402


def _teacher(heads=2, kv_heads=2, seed=21):
    from llavamod.model import synthetic as S
    return S.make_teacher(dict(S.ARCH["tiny"], num_attention_heads=heads, num_key_value_heads=kv_heads), "tiny", seed=seed).eval()


def _logit_tol(ref):
    return 3e-2 * ref.abs().max().item() + 3e-2          # the stated bf16-vs-fp32 logits tolerance of test_dense_model_matches_reference_golden


def _prompts(V, lens, side, seed, images=True):
    """Prompts of the given token lengths (one image each, or text-only), padded on `side` ("left", "right" or "mixed") with token 0."""
    g = torch.Generator().manual_seed(seed)
    B, T = len(lens), max(lens)
    ids = torch.zeros(B, T, dtype=torch.long)
    mask = torch.zeros(B, T, dtype=torch.bool)
    for b, n in enumerate(lens):
        p = torch.randint(1, V, (n,), generator=g)
        if images:
            p[(3 * b + 1) % n] = -200
        left = side == "left" or (side == "mixed" and b % 2 == 0)
        sl = slice(T - n, T) if left else slice(0, n)
        ids[b, sl], mask[b, sl] = p, True
    imgs = [torch.randn(3, 32, 32, generator=g).to(torch.bfloat16) for _ in lens] if images else None
    return ids, mask, imgs


# ---------------------------------------------------------------------------------------------------------------------------------
# the kernel
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nh,nkv,hd", [(4, 2, 64), (2, 2, 128), (4, 4, 32)])
def test_kv_append_rows_matches_torch_copy(nh, nkv, hd):
    from llavamod import kernels as K
    g = torch.Generator(device="cuda").manual_seed(1)
    B, T, L = 4, 37, 96
    hp = K.attn_head_dim(hd)
    qkv = torch.randn(B * T, (nh + 2 * nkv) * hd, device="cuda", generator=g).to(torch.bfloat16)
    lo = torch.tensor([0, 5, 30, 0], dtype=torch.int32, device="cuda")
    hi = torch.tensor([37, 20, 37, 1], dtype=torch.int32, device="cuda")
    off = torch.tensor([0, 3, 60, 95], dtype=torch.int32, device="cuda")
    kc = torch.full((B, nkv, L, hp), float("nan"), dtype=torch.bfloat16, device="cuda")
    vc = torch.full((B, nkv, L, hp), -7.0, dtype=torch.bfloat16, device="cuda")
    K.kv_append_rows(qkv, B, T, nh, nkv, hd, kc, vc, lo, hi, off)
    torch.cuda.synchronize()
    x = torch.nn.functional.pad(qkv.view(B, T, nh + 2 * nkv, hd), (0, hp - hd))
    ek = torch.full_like(kc, float("nan"))
    ev = torch.full_like(vc, -7.0)
    for b in range(B):
        l, h, o = int(lo[b]), int(hi[b]), int(off[b])
        ek[b, :, o:o + h - l] = x[b, l:h, nh:nh + nkv].transpose(0, 1)
        ev[b, :, o:o + h - l] = x[b, l:h, nh + nkv:].transpose(0, 1)
    # byte-equal, NaN rows included: every row outside the ranges is untouched
    assert torch.equal(kc.view(torch.int16), ek.view(torch.int16)) and torch.equal(vc.view(torch.int16), ev.view(torch.int16))
    # the full range at offset 0 writes exactly the bytes of lmod_kv_append
    kc2, vc2 = torch.zeros_like(kc), torch.zeros_like(vc)
    kc3, vc3 = torch.zeros_like(kc), torch.zeros_like(vc)
    z = torch.zeros(B, dtype=torch.int32, device="cuda")
    K.kv_append_rows(qkv, B, T, nh, nkv, hd, kc2, vc2, z, torch.full_like(z, T), z)
    K.kv_append(qkv, B, T, nh, nkv, hd, kc3, vc3, z)
    assert torch.equal(kc2.view(torch.int16), kc3.view(torch.int16)) and torch.equal(vc2.view(torch.int16), vc3.view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------------------------
# a padded batch against each prompt alone
# ---------------------------------------------------------------------------------------------------------------------------------
def _decode(model, ids, mask, images, toks, max_len):
    """Prefill + teacher-forced cached steps -> (logits [N + 1, B, V], cache)."""
    from llavamod.model.generation import next_token_logits
    cache = model.new_kv_cache(ids.shape[0], max_len)
    ragged = mask is not None and not bool(mask.all())
    with torch.no_grad():
        out = [next_token_logits(model, ids.cuda(), images=images, attention_mask=mask.cuda() if ragged else None, cache=cache,
                                 ragged=ragged)]
        for t in range(toks.shape[1]):
            out.append(next_token_logits(model, toks[:, t:t + 1].cuda(), cache=cache))
    return torch.stack(out), cache


@pytest.mark.parametrize("images", [True, False])
@pytest.mark.parametrize("side,padding_side", [("left", "right"), ("right", "right"), ("right", "left"), ("mixed", "left")])
@pytest.mark.parametrize("heads,kv_heads", [(4, 4), (2, 1)])          # hd 32 (zero-padded heads) and hd 64 GQA
def test_padded_batch_equals_each_prompt_alone(heads, kv_heads, side, padding_side, images):
    """Every sequence's per-step logits and cache rows [0, n_b + N) against the same prompt alone at B = 1 with the same cache bucket.
    Bit-identical when the prefill holds the real rows first (right layout); a left layout shifts the real rows inside the attention
    tiles and is held to the bf16 logits tolerance (and reported when it is not bit-identical)."""
    model = _teacher(heads, kv_heads)
    model.config.tokenizer_padding_side = padding_side
    cfg = model.config
    lens, N = [21, 6, 13], 5
    ids, mask, imgs = _prompts(cfg.vocab_size, lens, side, seed=50, images=images)
    toks = torch.randint(0, cfg.vocab_size, (3, N), generator=torch.Generator().manual_seed(51))
    got, cache = _decode(model, ids, mask, imgs, toks, 512)
    n_b = model.spliced_length(ids, imgs, mask)
    assert cache.lengths == [n + N for n in n_b] and cache.len.tolist() == cache.lengths and cache.length == max(n_b) + N
    real_first = (padding_side == "right") if images else (side == "right")
    for b in range(3):
        one, c1 = _decode(model, ids[b:b + 1, mask[b]], torch.ones(1, lens[b], dtype=torch.bool), imgs[b:b + 1] if images else None,
                          toks[b:b + 1], 512)
        rows = [(cache[i][j][b, :, :n_b[b] + N], c1[i][j][0]) for i in range(cfg.num_hidden_layers) for j in range(2)]
        same = torch.equal(got[:, b], one[:, 0]) and all(torch.equal(x, y) for x, y in rows)
        if real_first:
            assert same, (b, (got[:, b] - one[:, 0]).abs().max().item())
        elif not same:
            err = (got[:, b] - one[:, 0]).abs().max().item()
            warnings.warn("left-laid-out prefill is not bit-identical to the prompt alone (sequence %d, max |d logit| %.3g)" % (b, err))
            assert err < _logit_tol(one[:, 0]), (b, err)


def test_forward_api_continues_a_padded_cache_and_rejects_bad_batches():
    """forward(attention_mask=padded, use_cache=True) returns the cache; forward(input_ids=[B,1], past_key_values=cache) continues it,
    and its attention_mask is not read.  A row without a real token and an overflowing cache are refused before anything runs."""
    from llavamod.model.generation import next_token_logits
    model = _teacher(2, 1)
    ids, mask, imgs = _prompts(model.config.vocab_size, [9, 4, 12], "left", seed=60, images=False)
    toks = torch.randint(0, model.config.vocab_size, (3, 3), generator=torch.Generator().manual_seed(61))
    ref, _ = _decode(model, ids, mask, None, toks, 512)
    with torch.no_grad():
        out = model(input_ids=ids.cuda(), attention_mask=mask.cuda(), use_cache=True, return_dict=True)
        cache = out.past_key_values
        assert cache.lengths == [9, 4, 12] and out.logits.shape[:2] == ids.shape
        # left padding: the last row is every sequence's last real row (lm_head over all B*T rows here, over the B gathered rows there)
        torch.testing.assert_close(out.logits[:, -1], ref[0], rtol=0, atol=1e-2)
        for t in range(3):
            o = model(input_ids=toks[:, t:t + 1].cuda(), past_key_values=cache, attention_mask=torch.zeros(3, 1), use_cache=True,
                      return_dict=True)
            assert torch.equal(o.logits[:, -1], ref[t + 1])
        bad = mask.clone()
        bad[1] = False
        c = model.new_kv_cache(3, 512)
        with pytest.raises(ValueError):
            next_token_logits(model, ids.cuda(), attention_mask=bad.cuda(), cache=c, ragged=True)
        assert c.lengths == [0, 0, 0] and c.len.tolist() == [0, 0, 0]
        c = model.new_kv_cache(3, 11)
        with pytest.raises(ValueError):
            next_token_logits(model, ids.cuda(), attention_mask=mask.cuda(), cache=c, ragged=True)
        assert c.lengths == [0, 0, 0]
    with pytest.raises(ValueError):
        model.generate(ids, attention_mask=bad, max_new_tokens=2, use_cache=True)


# ---------------------------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("side", ["left", "right"])
@pytest.mark.parametrize("name", ["ragged_mha_hd32", "ragged_gqa_4_2", "ragged_text_only"])
def test_padded_batch_matches_reference_golden(name, side, golden_dir):
    """The reference's cached decoding of every prompt alone (tests/golden/make_ragged_decode_golden.py) against one padded-batch call of
    our bf16 CUDA model loaded with the same weights: every step's logits within the stated logits tolerance, the cache within bf16
    rounding of the reference's K / V."""
    from llavamod.model import LlavaQwen1_5Config, LlavaQwen1_5ForCausalLM
    from llavamod.model.builder_io import load_into
    from tests.golden import shards
    from tests.test_ragged_decode_reference import _relayout
    fx = shards.load(golden_dir, name)
    kw = fx["kw"]
    clip = dict(hidden_size=64, intermediate_size=128, num_hidden_layers=3, num_attention_heads=kw.get("clip_heads", 4), image_size=32, patch_size=8)
    cfg = LlavaQwen1_5Config(vocab_size=kw["vocab"], hidden_size=kw["hidden"], intermediate_size=kw["inter"], num_hidden_layers=kw["layers"],
                             num_attention_heads=kw["heads"], num_key_value_heads=kw["kv_heads"], rope_theta=1e6, mm_image_tower=clip,
                             image_projector_type="mlp2x_gelu", mm_hidden_size=64, mm_vision_select_layer=-2)
    m = LlavaQwen1_5ForCausalLM(cfg, device="cuda", dtype=torch.bfloat16)
    m.get_model().get_image_tower().load_model()
    load_into(m, {k: v for k, v in fx["state_dict"].items() if "position_ids" not in k}, strict=True)
    m.eval()
    ids, mask = _relayout(fx["input_ids"], fx["mask"], side)
    images = [im.to(torch.bfloat16) for im in fx["images"]] if fx["images"] is not None else None
    got, cache = _decode(m, ids, mask, images, fx["tokens"], 512)
    for b in range(ids.shape[0]):
        ref = fx["logits"][str(b)]
        err = (got[:, b].float().cpu() - ref).abs().max().item()
        assert err < _logit_tol(ref), (name, b, err)
        for i in range(kw["layers"]):
            for j, key in enumerate("kv"):
                r = fx[key]["%d.%d" % (b, i)]
                mine = cache[i][j][b, :, :r.shape[1]].float().cpu()
                assert (mine - r).abs().max().item() <= 3e-2 * r.abs().max().item(), (name, b, i, key)


# ---------------------------------------------------------------------------------------------------------------------------------
# the sparse student
# ---------------------------------------------------------------------------------------------------------------------------------
def _routing_agrees(gr, o, noise):
    """Our routing record against the oracle's: True if equal; a difference is allowed only on an fp32 near-tie (then False: stop)."""
    E = o["gates"].shape[1]
    idx = gr["idx"].long().cpu()
    diff = (idx[:, 0] != o["idx1"]) | (idx[:, 1] != o["idx2"])
    if bool(diff.any()):
        top = o["gates"].topk(2, dim=1).values
        lw = (o["logits"] + noise).masked_fill(torch.nn.functional.one_hot(o["idx1"], E).bool(), -float("inf")).topk(2, dim=1).values
        tied = ((top[:, 0] - top[:, 1]) < 1e-3) | ((lw[:, 0] - lw[:, 1]) < 1e-3)
        assert bool(tied[diff].all()), diff.nonzero().flatten().tolist()
        return False
    assert gr["capacity"] == o["capacity"]
    keep = gr["row"].cpu() >= 0
    assert torch.equal(keep[:, 0], o["keep1"]) and torch.equal(keep[:, 1], o["keep2"])
    return True


def test_sparse_student_padded_batch_matches_ragged_oracle():
    """Injected noise: the padded prefill routes every row (pads included, S = B * T'), each step routes the B step tokens; routing
    records equal the ragged oracle's (up to fp32 near-ties), logits within the bf16 tolerance."""
    student, _ = Hh.tiny_pair()
    student.eval()
    ecf, min_cap = 0.5, 1
    moes = [l.mlp for l in student.model.layers if hasattr(l.mlp, "deepspeed_moe")]
    for mo in moes:
        mo.eval_capacity_factor, mo.min_capacity = ecf, min_cap
    lc, cc = Hh.cfgs_of(student)
    lc.min_capacity = min_cap
    E = lc.num_experts
    sd = Hh.oracle_state(student)
    ids, mask, imgs = _prompts(lc.vocab, [14, 5, 9, 11], "mixed", seed=70)
    emb, m = RO.prompt_embeds(sd, lc, cc, ids, mask, [im.float() for im in imgs], "right")
    B, T = m.shape
    g = torch.Generator().manual_seed(71)
    noise = [R.gumbel_noise((B * T, E), g) for _ in moes]
    cache = student.new_kv_cache(B, 512)
    with torch.no_grad():
        r = student.forward_hidden(input_ids=ids.cuda(), images=imgs, attention_mask=mask.cuda(), moe_noise=[n.cuda() for n in noise],
                                   cache=cache)
    orec = []
    h, state = RO.prefill(sd, lc, emb, m, noise, orec, capacity_factor=ecf)
    for li, (gr, o) in enumerate(zip(r["records"], orec)):
        assert gr["capacity"] == o["capacity"] == R.moe_capacity(B * T, E, ecf, min_cap)
        if not _routing_agrees(gr, o, noise[li]):
            return
    ref = RO.lm_head(sd, lc, RO.last_real(h, m))
    last = RO.last_real(r["hidden"].float().cpu(), m)
    assert (RO.lm_head(sd, lc, last) - ref).abs().max().item() < _logit_tol(ref)
    toks = torch.randint(0, lc.vocab, (B, 5), generator=g)
    w = sd[R.P_LM + "embed_tokens.weight"]
    for t in range(toks.shape[1]):
        noise = [R.gumbel_noise((B, E), g) for _ in moes]
        with torch.no_grad():
            r = student.forward_hidden(input_ids=toks[:, t:t + 1].cuda(), moe_noise=[n.cuda() for n in noise], cache=cache)
        orec = []
        h = RO.step(sd, lc, w[toks[:, t:t + 1]], state, noise, orec, capacity_factor=ecf)
        for li, (gr, o) in enumerate(zip(r["records"], orec)):
            assert gr["capacity"] == o["capacity"] == max(int(math.ceil(B / E * ecf * 2)), min_cap)
            if not _routing_agrees(gr, o, noise[li]):
                return
        ref = RO.lm_head(sd, lc, h[:, 0])
        got = RO.lm_head(sd, lc, r["hidden"][:, 0].float().cpu())
        assert (got - ref).abs().max().item() < _logit_tol(ref), t


# ---------------------------------------------------------------------------------------------------------------------------------
# generate
# ---------------------------------------------------------------------------------------------------------------------------------
def _alone(model, ids, imgs, b, mask, **kw):
    scores = []
    crit = lambda i, s: (scores.append(s.clone()) or False)       # noqa: E731
    out = model.generate(ids[b:b + 1, mask[b]], images=imgs[b:b + 1], stopping_criteria=[crit], **kw)
    return out[0, int(mask[b].sum()):].cpu(), scores


@pytest.mark.parametrize("use_cache,graphs", [(True, "1"), (True, "0"), (False, "1")])
def test_generate_padded_batch_equals_per_prompt_calls(monkeypatch, use_cache, graphs):
    monkeypatch.setenv("LLAVAMOD_CUDA_GRAPHS", graphs)
    model = _teacher(2, 2, seed=80)
    lens, steps = [17, 6, 11], 7
    ids, mask, imgs = _prompts(model.config.vocab_size, lens, "left", seed=81)
    out = model.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=steps, use_cache=use_cache)
    T = ids.shape[1]
    assert out.shape == (3, T + steps) and torch.equal(out[:, :T].cpu(), ids)          # HF's layout: the input as given, then the new tokens
    for b in range(3):
        want, scores = _alone(model, ids, imgs, b, mask, max_new_tokens=steps, use_cache=use_cache)
        got = out[b, T:].cpu()
        for s in range(steps):
            if got[s] != want[s]:                                    # only where the prompt alone is at a near-tie
                top = scores[s][0].float().topk(2).values
                assert float(top[0] - top[1]) < 5e-2, (b, s)
                break
    # EOS in one sequence: it is padded from there on while the others continue as they would alone
    first0 = int(_alone(model, ids, imgs, 0, mask, max_new_tokens=1, use_cache=use_cache)[0][0])
    out = model.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=steps, use_cache=use_cache, eos_token_id=first0,
                         pad_token_id=3)
    assert int(out[0, T]) == first0 and bool((out[0, T + 1:] == 3).all())
    for b in (1, 2):
        want, _ = _alone(model, ids, imgs, b, mask, max_new_tokens=steps, use_cache=use_cache, eos_token_id=first0, pad_token_id=3)
        assert torch.equal(out[b, T:T + want.shape[0]].cpu(), want)
    # sampling and the narrowed vocabulary on a padded batch
    g = torch.Generator(device="cuda").manual_seed(0)
    a = model.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=4, do_sample=True, temperature=0.7, top_p=0.9, generator=g,
                       use_cache=use_cache)
    g = torch.Generator(device="cuda").manual_seed(0)
    a2 = model.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=4, do_sample=True, temperature=0.7, top_p=0.9, generator=g,
                        use_cache=use_cache)
    assert torch.equal(a, a2)
    model.resize_token_embeddings(100)
    assert int(model.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=4, use_cache=use_cache)[:, T:].max()) < 100
