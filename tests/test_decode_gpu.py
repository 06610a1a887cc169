"""KV-cache decoding through the model: the prefill cache, the decode positions, teacher-forced step logits against the float32 oracle,
the MoE student's per-step routing against the cached oracle (tests/decode_oracle.py), generate(use_cache=True), and graph replay."""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import restated as R  # noqa: E402
from tests import decode_oracle as D  # noqa: E402
from tests import helpers as Hh  # noqa: E402


def _record_qkv(monkeypatch):
    """Every layer's fused, RoPE'd q|k|v output, in call order."""
    from llavamod import kernels as Kk
    out = []
    orig = Kk.qkv_rope

    def rec(*a, **kw):
        y = orig(*a, **kw)
        out.append(y.clone())
        return y
    monkeypatch.setattr(Kk, "qkv_rope", rec)
    return out


def _kv_of(qkv, B, T, nh, nkv, hd):
    x = qkv.view(B, T, nh + 2 * nkv, hd)
    return x[:, :, nh:nh + nkv].transpose(1, 2), x[:, :, nh + nkv:].transpose(1, 2)


def _teacher(heads=2, kv_heads=2, seed=21):
    from llavamod.model import synthetic as S
    return S.make_teacher(dict(S.ARCH["tiny"], num_attention_heads=heads, num_key_value_heads=kv_heads), "tiny", seed=seed)


def _logit_tol(ref):
    return 3e-2 * ref.abs().max().item() + 3e-2          # the stated bf16-vs-fp32 logits tolerance of test_dense_model_matches_reference_golden


@pytest.mark.parametrize("heads,kv_heads", [(2, 2), (4, 2)])          # hd 64 (built) and hd 32 (zero-padded heads), GQA
def test_prefill_and_decode_cache_bit_identical_to_recompute(monkeypatch, heads, kv_heads):
    from llavamod.model.generation import next_token_logits
    model = _teacher(heads, kv_heads)
    cfg = model.config
    nh, nkv, hd = heads, kv_heads, cfg.hidden_size // heads
    batch, _ = Hh.tiny_batch(model, B=2, Tt=24, seed=22)
    ids, images = batch["input_ids"].cuda(), batch["images"]
    B, N = 2, 7
    with torch.no_grad():
        rec = _record_qkv(monkeypatch)
        plain = model.forward_hidden(input_ids=ids, images=images)["hidden"]
        ref_qkv = list(rec)
        rec.clear()
        cache = model.new_kv_cache(B, 128)
        pre = model.forward_hidden(input_ids=ids, images=images, cache=cache)["hidden"]
        T = pre.shape[1]
        assert torch.equal(pre, plain) and cache.length == T and cache.len.tolist() == [T, T]
        for i in range(cfg.num_hidden_layers):                 # prefill cache == K / V of the no-cache forward, every layer
            k, v = _kv_of(ref_qkv[i], B, T, nh, nkv, hd)
            assert torch.equal(cache[i][0], k) and torch.equal(cache[i][1], v), i
        toks = torch.randint(0, cfg.vocab_size, (B, N), generator=torch.Generator().manual_seed(5)).cuda()
        steps = [next_token_logits(model, toks[:, t:t + 1], cache=cache) for t in range(N)]
        full_ids = torch.cat([ids, toks], 1)
        rec.clear()
        model.forward_hidden(input_ids=full_ids, images=images)
        k, v = _kv_of(rec[0], B, T + N, nh, nkv, hd)          # layer 0 of every decoded token: positions and RoPE of the cached step
        assert torch.equal(cache[0][0], k) and torch.equal(cache[0][1], v)
    # teacher-forced step logits against the float32 oracle over the full sequence
    b = dict(batch, input_ids=full_ids.cpu(), attention_mask=torch.ones_like(full_ids.cpu(), dtype=torch.bool),
             labels=torch.full_like(full_ids.cpu(), -100))
    out, _ = Hh.oracle_forward(model, b)
    for t in range(N):
        ref = out["logits"][:, T + t]                          # the token fed at step t sits at position T + t
        err = (steps[t].cpu() - ref).abs().max().item()
        assert err < _logit_tol(ref), (t, err)
    with pytest.raises(ValueError):
        full = model.new_kv_cache(B, T)
        model.forward_hidden(input_ids=ids, images=images, cache=full)
        next_token_logits(model, toks[:, :1], cache=full)         # one position past max_len: refused before anything is written


@pytest.mark.parametrize("name", ["decode_mha_hd32", "decode_gqa_4_2", "decode_hd64_kv1", "decode_text_only"])
def test_cached_forward_matches_reference_golden(name, golden_dir):
    """The reference's own cached decoding (tests/golden/make_decode_golden.py: prefill + teacher-forced cached steps) against
    forward(past_key_values=..., use_cache=True) of our bf16 CUDA model loaded with the same weights: every step's logits within the
    stated logits tolerance of test_dense_model_matches_reference_golden, and the final cache within bf16 rounding of the reference's K / V."""
    from llavamod.model import LlavaQwen1_5Config, LlavaQwen1_5ForCausalLM
    from llavamod.model.builder_io import load_into
    from llavamod.model.language_model.qwen2_core import KVCache
    from tests.golden import shards
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
    ids, toks = fx["input_ids"], fx["tokens"]
    images = [im.to(torch.bfloat16) for im in fx["images"]] if fx["images"] is not None else None
    mask = torch.ones_like(ids)
    with torch.no_grad():
        out = m(input_ids=ids, images=images, attention_mask=mask, use_cache=True, return_dict=True)
        cache = out.past_key_values
        assert isinstance(cache, KVCache) and cache.length == fx["k"]["0"].shape[2] - toks.shape[1]
        got = [out.logits[:, -1]]
        for t in range(toks.shape[1]):
            out = m(input_ids=toks[:, t:t + 1], past_key_values=cache, attention_mask=mask, images=images, use_cache=True, return_dict=True)
            assert out.past_key_values is cache and out.logits.shape[1] == 1
            got.append(out.logits[:, -1])
    for t, (g, ref) in enumerate(zip(got, fx["logits"])):
        err = (g.float().cpu() - ref).abs().max().item()
        assert err < _logit_tol(ref), (name, t, err)
    for i in range(kw["layers"]):
        for j, key in enumerate("kv"):
            ref = fx[key][str(i)]
            mine = cache[i][j].float().cpu()
            assert mine.shape == ref.shape
            err = (mine - ref).abs().max().item()
            assert err <= 3e-2 * ref.abs().max().item(), (name, i, key, err)


def _oracle_prompt(model, sd, ids, images):
    lc, cc = Hh.cfgs_of(model)
    feats = R.encode_images(sd, cc, lc.proj_depth, torch.stack([im.float() for im in images]))
    src, _, _, _, img = R.splice_plan(ids, None, None, feats.shape[1])
    return R.splice_embed(sd[R.P_LM + "embed_tokens.weight"], feats, src, img)


@pytest.mark.parametrize("B", [8, 1])
def test_moe_student_step_routing_matches_cached_oracle(B):
    student, _ = Hh.tiny_pair()
    student.eval()
    ecf, min_cap = 0.5, 1                                     # step capacity max(ceil(B/4 * 0.5 * 2), 1): B = 8 -> 2, drops tokens
    moes = [l.mlp for l in student.model.layers if hasattr(l.mlp, "deepspeed_moe")]
    for m in moes:
        m.eval_capacity_factor, m.min_capacity = ecf, min_cap
    batch, _ = Hh.tiny_batch(student, B=B, Tt=20, seed=40)
    ids, images = batch["input_ids"], batch["images"]
    sd = Hh.oracle_state(student)
    lc, _ = Hh.cfgs_of(student)
    lc.min_capacity = min_cap
    E = lc.num_experts
    g = torch.Generator().manual_seed(41)
    emb = _oracle_prompt(student, sd, ids, images)
    T = emb.shape[1]
    noise = [R.gumbel_noise((B * T, E), g) for _ in moes]
    cache = student.new_kv_cache(B, 64)
    with torch.no_grad():
        student.forward_hidden(input_ids=ids.cuda(), images=images, moe_noise=[n.cuda() for n in noise], cache=cache)
    _, past, _ = D.lm_forward_cached(sd, lc, emb, None, noise, [], capacity_factor=ecf)
    toks = torch.randint(0, lc.vocab, (B, 6), generator=g)
    drops = 0
    for t in range(toks.shape[1]):
        noise = [R.gumbel_noise((B, E), g) for _ in moes]
        with torch.no_grad():
            r = student.forward_hidden(input_ids=toks[:, t:t + 1].cuda(), moe_noise=[n.cuda() for n in noise], cache=cache)
            got = D.lm_head(sd, lc, r["hidden"].float().cpu())
        orec = []
        h, past, _ = D.lm_forward_cached(sd, lc, sd[R.P_LM + "embed_tokens.weight"][toks[:, t:t + 1]], past, noise, orec, capacity_factor=ecf)
        ref = D.lm_head(sd, lc, h)
        for li, (gr, o) in enumerate(zip(r["records"], orec)):
            C = max(int(math.ceil(B / E * ecf * 2)), min_cap)
            assert gr["capacity"] == o["capacity"] == C
            idx = gr["idx"].long().cpu()
            diff = (idx[:, 0] != o["idx1"]) | (idx[:, 1] != o["idx2"])
            if bool(diff.any()):
                # only a token on which the fp32 oracle is near a tie may route differently; the states part from there on, so the
                # comparison stops -- after the capacity-dropping steps of B = 8 have been compared
                top = o["gates"].topk(2, dim=1).values
                lw = (o["logits"] + noise[li]).masked_fill(torch.nn.functional.one_hot(o["idx1"], E).bool(), -float("inf")).topk(2, dim=1).values
                tied = ((top[:, 0] - top[:, 1]) < 1e-3) | ((lw[:, 0] - lw[:, 1]) < 1e-3)
                assert bool(tied[diff].all()), (t, li, diff.nonzero().flatten().tolist())
                assert B != 8 or drops > 0, "routing parted at step %d before a capacity drop was compared" % t
                return
            keep = gr["row"].cpu() >= 0
            assert torch.equal(keep[:, 0], o["keep1"]) and torch.equal(keep[:, 1], o["keep2"]), (t, li)
            drops += int((~keep).sum())
        err = (got - ref).abs().max().item()
        assert err < _logit_tol(ref), (t, err)
    if B == 8:
        assert drops > 0


def test_generate_with_cache_greedy_sampling_eos_stopping_vocab():
    model = _teacher(seed=23)
    batch, _ = Hh.tiny_batch(model, B=2, Tt=24, seed=24)
    steps = 6
    ids = batch["input_ids"].clone()
    toks, margins = [], []
    sd = Hh.oracle_state(model)
    for _ in range(steps):                                    # dense model: the cached oracle is the full recompute (test_decode_reference)
        b = dict(batch, input_ids=ids, attention_mask=torch.ones_like(ids, dtype=torch.bool), labels=torch.full_like(ids, -100))
        out, _ = Hh.oracle_forward(model, b, None, sd=sd)
        top = out["logits"][:, -1, :].float().topk(2, dim=-1)
        toks.append(top.indices[:, 0])
        margins.append(top.values[:, 0] - top.values[:, 1])
        ids = torch.cat([ids, top.indices[:, :1]], dim=1)
    ref_tok, margin = torch.stack(toks, 1), torch.stack(margins, 1)
    out = model.generate(batch["input_ids"], images=batch["images"], max_new_tokens=steps, use_cache=True)
    assert out.shape == (2, 24 + steps) and torch.equal(out[:, :24].cpu(), batch["input_ids"])
    got = out[:, 24:].cpu()
    for b in range(2):
        for s in range(steps):
            if got[b, s] != ref_tok[b, s]:
                assert margin[b, s] < 5e-2, (b, s, float(margin[b, s]))
                break
    one = dict(input_ids=batch["input_ids"][:1], images=batch["images"][:1])
    g = torch.Generator(device="cuda").manual_seed(0)
    a = model.generate(one["input_ids"], images=one["images"], max_new_tokens=5, do_sample=True, temperature=0.7, top_p=0.9, generator=g, use_cache=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    b2 = model.generate(one["input_ids"], images=one["images"], max_new_tokens=5, do_sample=True, temperature=0.7, top_p=0.9, generator=g, use_cache=True)
    assert torch.equal(a, b2) and a.shape[1] == 29
    first = int(model.generate(one["input_ids"], images=one["images"], max_new_tokens=1, use_cache=True)[0, -1])
    assert model.generate(one["input_ids"], images=one["images"], max_new_tokens=8, eos_token_id=first, use_cache=True).shape[1] == 25
    calls = []
    crit = lambda ids, scores: (calls.append(ids.shape[1]) or ids.shape[1] >= 27)      # noqa: E731
    assert model.generate(one["input_ids"], images=one["images"], max_new_tokens=8, stopping_criteria=[crit], use_cache=True).shape[1] == 27
    assert calls == [25, 26, 27]
    model.resize_token_embeddings(100)
    assert int(model.generate(one["input_ids"], images=one["images"], max_new_tokens=6, use_cache=True)[0, 24:].max()) < 100


def test_graph_replay_equals_eager(monkeypatch):
    from llavamod.model import generation as Gm
    model = _teacher(seed=25)
    batch, _ = Hh.tiny_batch(model, B=2, Tt=24, seed=26)
    runs = {}
    for mode in ("0", "1", "1"):
        monkeypatch.setenv("LLAVAMOD_CUDA_GRAPHS", mode)
        scores = []
        crit = lambda ids, s: (scores.append(s.clone()) or False)     # noqa: E731
        ids = model.generate(batch["input_ids"], images=batch["images"], max_new_tokens=12, use_cache=True, stopping_criteria=[crit])
        runs.setdefault(mode, []).append((ids, scores))
    (e_ids, e_sc), = runs["0"]
    for ids, sc in runs["1"]:                                 # first call captures, second replays the kept graph
        assert torch.equal(ids, e_ids) and all(torch.equal(x, y) for x, y in zip(sc, e_sc))
    graphs = [v for v in Gm._STEP_GRAPHS.values() if v["graph"] is not None]
    assert len(graphs) >= 1
    # another prompt length in the same 512-position bucket reuses the graph
    n = len(Gm._STEP_GRAPHS)
    model.generate(batch["input_ids"][:, :20], images=batch["images"], max_new_tokens=3, use_cache=True)
    assert len(Gm._STEP_GRAPHS) == n
    monkeypatch.setenv("LLAVAMOD_MAX_GRAPHS", "1")
    model.generate(batch["input_ids"][:1], images=batch["images"][:1], max_new_tokens=3, use_cache=True)
    assert len(Gm._STEP_GRAPHS) == 1


def test_config_scale_student_decode(monkeypatch):
    """0.5B-4E student with CLIP-L/336 at T' = 650 and 64 new tokens: the decoded layer-0 K / V equal a full recompute bit for bit."""
    from llavamod.model import synthetic as S
    from llavamod.model import generation as Gm
    student = S.make_student("qwen1.5-0.5b", "clip-l-336", seed=3).eval()
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(0, 150000, (1, 75), generator=g)
    ids[0, 3] = -200
    img = [torch.randn(3, 336, 336, generator=g).to(torch.bfloat16)]
    out = student.generate(ids, images=img, max_new_tokens=64, use_cache=True)
    assert out.shape == (1, 75 + 64)
    cache = next(reversed(Gm._STEP_GRAPHS.values()))["cache"]
    assert cache.length == 650 + 63
    cfg = student.config
    rec = _record_qkv(monkeypatch)
    with torch.no_grad():
        student.forward_hidden(input_ids=out[:, :-1], images=img)
    k, v = _kv_of(rec[0], 1, 650 + 63, cfg.num_attention_heads, cfg.num_key_value_heads, cfg.hidden_size // cfg.num_attention_heads)
    assert torch.equal(cache[0][0], k) and torch.equal(cache[0][1], v)
