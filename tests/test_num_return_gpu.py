"""generate(..., do_sample=True, num_return_sequences=n): the dense shared-cache path returns, byte for byte, the tokens of generate on the
inputs expanded with repeat_interleave(n, 0) and a generator in the same state; the sparse student and use_cache=False run that expanded
call; n = 1 is today's path; the shared cache is smaller than the expanded one."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests import helpers as Hh  # noqa: E402
from tests.test_ragged_decode_gpu import _prompts, _teacher  # noqa: E402

MODELS = [(1, 1), (2, 1)]          # hidden 128: one head of 128 (MHA, hd 128), two query heads on one KV head (GQA, hd 64)


def _inputs(model, kind, images):
    V = model.config.vocab_size
    if kind == "unpadded":
        ids, _, imgs = _prompts(V, [19, 19, 19], "left", seed=71, images=images)
        return ids, None, imgs
    return _prompts(V, [17, 6, 11], kind, seed=72, images=images)


def _expanded(n, ids, mask, imgs):
    return (ids.repeat_interleave(n, 0), None if mask is None else mask.repeat_interleave(n, 0),
            None if imgs is None else [im for im in imgs for _ in range(n)])


def _pair(model, n, ids, mask, imgs, seed=5, **kw):
    """(shared call, expanded call) with generators in the same state; the router's noise (sparse model) is reseeded too."""
    kw = dict(dict(max_new_tokens=12, use_cache=True, do_sample=True, temperature=0.8), **kw)
    torch.cuda.manual_seed(seed + 1)
    got = model.generate(ids, images=imgs, attention_mask=mask, num_return_sequences=n,
                         generator=torch.Generator(device="cuda").manual_seed(seed), **kw)
    eids, emask, eimgs = _expanded(n, ids, mask, imgs)
    torch.cuda.manual_seed(seed + 1)
    want = model.generate(eids, images=eimgs, attention_mask=emask, generator=torch.Generator(device="cuda").manual_seed(seed), **kw)
    return got, want


def _shared_entries():
    from llavamod.model import generation as Gm
    return [e for e in Gm._STEP_GRAPHS.values() if e["cache"].shared]


@pytest.mark.parametrize("graphs", ["1", "0"])
@pytest.mark.parametrize("kind", ["unpadded", "left", "right"])
@pytest.mark.parametrize("images", [True, False])
@pytest.mark.parametrize("heads,kv_heads", MODELS)
def test_shared_path_equals_expanded_call_bytewise(monkeypatch, heads, kv_heads, images, kind, graphs):
    monkeypatch.setenv("LLAVAMOD_CUDA_GRAPHS", graphs)
    model = _teacher(heads, kv_heads, seed=70)
    ids, mask, imgs = _inputs(model, kind, images)
    T = ids.shape[1]
    for n in (2, 3):
        got, want = _pair(model, n, ids, mask, imgs)
        assert got.shape == (3 * n, T + 12) and torch.equal(got, want), (n, kind)
        assert torch.equal(got[:, :T].cpu(), ids.repeat_interleave(n, 0))      # row b*n + j: prompt b as given, then copy j's tokens
        assert len({tuple(r) for r in got[:, T:].tolist()}) > 1                  # the copies draw different tokens
    if graphs == "1":
        assert _shared_entries(), "the cached path did not take the shared cache"


@pytest.mark.parametrize("graphs", ["1", "0"])
def test_shared_path_eos_and_stopping_criteria(monkeypatch, graphs):
    monkeypatch.setenv("LLAVAMOD_CUDA_GRAPHS", graphs)
    model = _teacher(2, 1, seed=73)
    ids, mask, imgs = _inputs(model, "left", True)
    T, n = ids.shape[1], 4
    got, want = _pair(model, n, ids, mask, imgs, max_new_tokens=16)
    assert torch.equal(got, want)
    eos = int(want[5, T + 2])                        # row 5 ends early, the others run on and are padded where they end
    got, want = _pair(model, n, ids, mask, imgs, max_new_tokens=16, eos_token_id=eos, pad_token_id=7)
    assert torch.equal(got, want) and int(got[5, T + 3:].ne(7).sum()) == 0

    seen = []

    def crit(tok, scores):
        seen.append((tuple(tok.shape), tuple(scores.shape)))
        return tok.shape[1] >= T + 6

    got, want = _pair(model, n, ids, mask, imgs, max_new_tokens=16, stopping_criteria=[crit])
    assert torch.equal(got, want) and got.shape == (3 * n, T + 6)
    assert seen and all(s[0][0] == 3 * n and s[1][0] == 3 * n for s in seen)


def test_sparse_student_and_no_cache_take_the_expanded_call():
    student, teacher = Hh.tiny_pair(seed=9)
    student.eval()
    ids, mask, imgs = _inputs(teacher, "left", True)
    for model, use_cache in ((student, True), (student, False), (teacher, False)):
        got, want = _pair(model, 3, ids, mask, imgs, max_new_tokens=8, use_cache=use_cache)
        assert got.shape[0] == 9 and torch.equal(got, want), (model.is_moe, use_cache)
    from llavamod.model import generation as Gm
    assert not any(e["cache"].shared for e in Gm._STEP_GRAPHS.values() if e["model"]() is student)


def test_one_return_sequence_is_todays_path(monkeypatch):
    from llavamod.model import generation as Gm
    monkeypatch.setenv("LLAVAMOD_CUDA_GRAPHS", "1")
    model = _teacher(2, 1, seed=74)
    ids, mask, imgs = _inputs(model, "right", True)
    outs, keys = [], []
    for kw in ({}, dict(num_return_sequences=1)):
        Gm._STEP_GRAPHS.clear()
        outs.append(model.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=10, use_cache=True, do_sample=True,
                                   generator=torch.Generator(device="cuda").manual_seed(3), **kw))
        keys.append([k[1:] for k in Gm._STEP_GRAPHS])
        assert not _shared_entries()
    assert torch.equal(outs[0], outs[1]) and keys[0] == keys[1] and len(keys[0]) == 1
    Gm._STEP_GRAPHS.clear()
    model.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=10, use_cache=True, do_sample=True, num_return_sequences=2)
    (key,) = list(Gm._STEP_GRAPHS)
    assert key[-1][:2] == ("share", 2) and key[:-1][1:] == keys[0][0]


def test_bad_arguments_raise():
    model = _teacher(2, 1, seed=75)
    ids, mask, imgs = _inputs(model, "unpadded", True)
    with pytest.raises(ValueError, match="greedy"):
        model.generate(ids, images=imgs, max_new_tokens=4, use_cache=True, num_return_sequences=2)
    with pytest.raises(ValueError, match="assisted"):
        model.generate(ids, images=imgs, max_new_tokens=4, use_cache=True, do_sample=True, num_return_sequences=2, assistant_model=model)
    with pytest.raises(ValueError):
        model.generate(ids, images=imgs, max_new_tokens=4, do_sample=True, num_return_sequences=0)


def test_shared_cache_is_smaller_and_has_no_legacy_view():
    model = _teacher(2, 1, seed=76)
    ids, mask, imgs = _inputs(model, "unpadded", True)
    for n in (2, 4, 8):
        shared = model.new_kv_cache(3, 512, share=n, suffix=64)
        assert shared.batch == 3 * n and shared.nbytes < model.new_kv_cache(3 * n, 512).nbytes, n
    model.generate(ids, images=imgs, max_new_tokens=8, use_cache=True, do_sample=True, num_return_sequences=4)
    ent = _shared_entries()[-1]
    cache = ent["cache"]
    assert cache.share == 4 and cache.prompts == 3 and cache.nbytes < model.new_kv_cache(12, cache.max_len).nbytes
    with pytest.raises(TypeError):
        cache[0]
    with pytest.raises(NotImplementedError):
        model(input_ids=ids[:, :1].repeat_interleave(4, 0).cuda(), past_key_values=cache, use_cache=True)


def test_config_scale_teacher_shares_the_prompt():
    """The 7B teacher at T' = 650, B = 2 prompts, n = 4, 16 sampled tokens: the expanded call's bytes."""
    from llavamod.model import synthetic as S
    teacher = S.make_teacher("qwen1.5-7b", "clip-l-336", seed=7).eval()
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(0, 150000, (2, 75), generator=g)
    ids[:, 3] = -200
    imgs = [torch.randn(3, 336, 336, generator=g).to(torch.bfloat16) for _ in range(2)]
    got, want = _pair(teacher, 4, ids, None, imgs, max_new_tokens=16)
    assert torch.equal(got, want)
