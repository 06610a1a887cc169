"""Assisted decoding through the model: a cached step of T tokens equals T one-token steps bit for bit (logits and K / V), the reference's
cached decoding fed in chunks, the sparse model's refusal, and generate(assistant_model=...) token for token against generate(use_cache=True)
of the target."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests import helpers as Hh  # noqa: E402
from tests.test_decode_gpu import _logit_tol, _teacher  # noqa: E402
from tests.test_ragged_decode_gpu import _prompts  # noqa: E402


def _prefill(model, ids, mask, imgs, max_len=256):
    cache = model.new_kv_cache(ids.shape[0], max_len)
    with torch.no_grad():
        model(input_ids=ids.cuda(), attention_mask=None if mask is None else mask.cuda(), images=imgs, past_key_values=cache, use_cache=True)
    return cache


@pytest.mark.parametrize("heads,kv_heads", [(2, 2), (4, 2)])
@pytest.mark.parametrize("side", [None, "left", "right"])
def test_chunked_step_equals_single_steps_bitwise(heads, kv_heads, side):
    model = _teacher(heads, kv_heads, seed=31).eval()
    V = model.config.vocab_size
    if side is None:
        batch, _ = Hh.tiny_batch(model, B=3, Tt=20, seed=32)
        ids, mask, imgs = batch["input_ids"], None, batch["images"]
    else:
        ids, mask, imgs = _prompts(V, [17, 6, 11], side, seed=33)
    toks = torch.randint(0, V, (ids.shape[0], 7), generator=torch.Generator().manual_seed(34)).cuda()
    a, b = _prefill(model, ids, mask, imgs), _prefill(model, ids, mask, imgs)
    with torch.no_grad():
        one = [model(input_ids=toks[:, t:t + 1], past_key_values=a, use_cache=True).logits for t in range(7)]
        two = [model(input_ids=toks[:, :3], past_key_values=b, use_cache=True).logits,
               model(input_ids=toks[:, 3:4], past_key_values=b, use_cache=True).logits,
               model(input_ids=toks[:, 4:], past_key_values=b, use_cache=True).logits]
    assert torch.equal(torch.cat(one, 1), torch.cat(two, 1))
    assert a.lengths == b.lengths and torch.equal(a.len, b.len)
    for i in range(len(a)):
        for s, n in enumerate(a.lengths):
            assert torch.equal(a.k[i][s, :, :n], b.k[i][s, :, :n]) and torch.equal(a.v[i][s, :, :n], b.v[i][s, :, :n]), (i, s)


@pytest.mark.parametrize("name", ["decode_mha_hd32", "decode_gqa_4_2", "decode_hd64_kv1", "decode_text_only"])
def test_chunked_cached_forward_matches_reference_golden(name, golden_dir):
    """The reference's teacher-forced cached steps (tests/golden/decode_*.pt) fed as chunks of 2 and 4 tokens: every position's logits
    and the final cache within the tolerances of test_cached_forward_matches_reference_golden (for a dense model the reference's chunked
    cached forward is the same function as its single steps)."""
    from llavamod.model import LlavaQwen1_5Config, LlavaQwen1_5ForCausalLM
    from llavamod.model.builder_io import load_into
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
    assert toks.shape[1] == 6
    images = [im.to(torch.bfloat16) for im in fx["images"]] if fx["images"] is not None else None
    with torch.no_grad():
        out = m(input_ids=ids, images=images, attention_mask=torch.ones_like(ids), use_cache=True, return_dict=True)
        cache = out.past_key_values
        got = [out.logits[:, -1]]
        for lo, hi in ((0, 2), (2, 6)):
            out = m(input_ids=toks[:, lo:hi], past_key_values=cache, use_cache=True, return_dict=True)
            assert out.logits.shape[1] == hi - lo
            got += list(out.logits.unbind(1))
    assert len(got) == len(fx["logits"])
    for t, (g, ref) in enumerate(zip(got, fx["logits"])):
        err = (g.float().cpu() - ref).abs().max().item()
        assert err < _logit_tol(ref), (name, t, err)
    for i in range(kw["layers"]):
        for j, key in enumerate("kv"):
            ref = fx[key][str(i)]
            mine = cache[i][j].float().cpu()
            assert mine.shape == ref.shape
            assert (mine - ref).abs().max().item() <= 3e-2 * ref.abs().max().item(), (name, i, key)


def test_sparse_model_refuses_a_multi_token_step():
    student, _ = Hh.tiny_pair()
    student.eval()
    batch, _ = Hh.tiny_batch(student, B=2, Tt=20, seed=35)
    cache = _prefill(student, batch["input_ids"], None, batch["images"])
    with torch.no_grad(), pytest.raises(NotImplementedError, match="route"):
        student(input_ids=torch.ones(2, 2, dtype=torch.long).cuda(), past_key_values=cache, use_cache=True)


# ---------------------------------------------------------------------------------------------------------------------------------
# generate(assistant_model=...)
# ---------------------------------------------------------------------------------------------------------------------------------
def _stats():
    from llavamod.model import generation as Gm
    return Gm.last_assisted_stats


def _perturbed(seed, scale):
    m = _teacher(seed=seed).eval()
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    w = m.lm_head.weight.data
    w.add_(torch.randn(w.shape, device="cuda", generator=g).to(w.dtype) * (scale * float(w.float().std())))
    return m


@pytest.mark.parametrize("graphs", ["1", "0"])
@pytest.mark.parametrize("k", [1, 4, 7])
def test_assisted_greedy_equals_target(monkeypatch, graphs, k):
    monkeypatch.setenv("LLAVAMOD_CUDA_GRAPHS", graphs)
    model = _teacher(seed=41).eval()
    batch, _ = Hh.tiny_batch(model, B=1, Tt=24, seed=42)
    ids, imgs = batch["input_ids"], batch["images"]
    want = model.generate(ids, images=imgs, max_new_tokens=20, use_cache=True)
    # the target as its own assistant: every draft is kept, which holds only if the verify step equals the one-token step bit for bit
    got = model.generate(ids, images=imgs, max_new_tokens=20, use_cache=True, assistant_model=model, num_assistant_tokens=k)
    assert torch.equal(got, want)
    st = _stats()
    assert st["accepted"] == st["drafted"] and st["drafted"][0] > 0
    # a perturbed copy: both the accept and the reject branch run
    other = _perturbed(41, 1.0)
    got = model.generate(ids, images=imgs, max_new_tokens=20, use_cache=True, assistant_model=other, num_assistant_tokens=k)
    assert torch.equal(got, want)
    st = _stats()
    assert 0 < st["accepted"][0] < st["drafted"][0], st


@pytest.mark.parametrize("graphs", ["1", "0"])
def test_assisted_padded_batch_with_eos_and_sparse_draft(monkeypatch, graphs):
    monkeypatch.setenv("LLAVAMOD_CUDA_GRAPHS", graphs)
    student, teacher = Hh.tiny_pair(seed=5)
    teacher.eval()
    ids, mask, imgs = _prompts(teacher.config.vocab_size, [17, 6, 11, 9], "left", seed=43)
    T = ids.shape[1]
    want = teacher.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=16, use_cache=True)
    for k in (1, 4):
        got = teacher.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=16, use_cache=True, assistant_model=student,
                               num_assistant_tokens=k)
        assert torch.equal(got, want), k
        got = teacher.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=16, use_cache=True, assistant_model=teacher,
                               num_assistant_tokens=k)
        assert torch.equal(got, want), k
    eos = int(want[1, T + 3])                                    # sequence 1 ends mid-run; the others continue and are padded if they end
    want = teacher.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=16, use_cache=True, eos_token_id=eos, pad_token_id=7)
    for draft in (student, teacher, _perturbed(5, 1.0)):
        got = teacher.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=16, use_cache=True, eos_token_id=eos, pad_token_id=7,
                               assistant_model=draft, num_assistant_tokens=4)
        assert torch.equal(got, want)
    # right padding too
    ids, mask, imgs = _prompts(teacher.config.vocab_size, [5, 12, 8, 10], "right", seed=44)
    want = teacher.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=9, use_cache=True)
    got = teacher.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=9, use_cache=True, assistant_model=student,
                           num_assistant_tokens=3)
    assert torch.equal(got, want)


def test_assisted_sampling_and_bad_arguments():
    model = _teacher(seed=45).eval()
    batch, _ = Hh.tiny_batch(model, B=2, Tt=24, seed=46)
    ids, imgs = batch["input_ids"], batch["images"]
    g = torch.Generator(device="cuda").manual_seed(0)
    a = model.generate(ids, images=imgs, max_new_tokens=12, use_cache=True, do_sample=True, temperature=0.7, generator=g,
                       assistant_model=model, num_assistant_tokens=4)
    st = _stats()
    assert a.shape == (2, 36) and st["accepted"] == st["drafted"]            # q == p: every draft is kept
    g = torch.Generator(device="cuda").manual_seed(0)
    a2 = model.generate(ids, images=imgs, max_new_tokens=12, use_cache=True, do_sample=True, temperature=0.7, generator=g,
                        assistant_model=model, num_assistant_tokens=4)
    assert torch.equal(a, a2)
    other = _perturbed(45, 1.0)
    model.resize_token_embeddings(100)
    out = model.generate(ids, images=imgs, max_new_tokens=12, use_cache=True, do_sample=True, temperature=0.9, top_p=0.8,
                         generator=g, assistant_model=other, num_assistant_tokens=3)
    assert out.shape[1] == 36 and int(out[:, 24:].max()) < 100
    with pytest.raises(ValueError):
        model.generate(ids, images=imgs, max_new_tokens=4, use_cache=False, assistant_model=other)
    student, _ = Hh.tiny_pair()
    with pytest.raises(ValueError):
        student.generate(ids, images=imgs, max_new_tokens=4, use_cache=True, assistant_model=model)
    with pytest.raises(NotImplementedError):
        model.generate(ids, images=imgs, max_new_tokens=4, use_cache=True, num_beams=2, assistant_model=other)


def test_config_scale_teacher_with_student_draft():
    """The 7B teacher assisted by the 0.5B-4E student at T' = 650, B = 1, 32 new tokens: the teacher's own cached tokens."""
    from llavamod.model import synthetic as S
    teacher = S.make_teacher("qwen1.5-7b", "clip-l-336", seed=7)
    student = S.make_student("qwen1.5-0.5b", "clip-l-336", seed=8, share_tower_with=teacher).eval()
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(0, 150000, (1, 75), generator=g)
    ids[0, 3] = -200
    img = [torch.randn(3, 336, 336, generator=g).to(torch.bfloat16)]
    want = teacher.generate(ids, images=img, max_new_tokens=32, use_cache=True)
    got = teacher.generate(ids, images=img, max_new_tokens=32, use_cache=True, assistant_model=student, num_assistant_tokens=4)
    assert torch.equal(got, want)
    st = _stats()
    assert st["rounds"] >= 1 and sum(st["drafted"]) > 0
