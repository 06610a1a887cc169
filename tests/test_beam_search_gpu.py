"""generate(..., num_beams=nb): transformers 4.37 beam search.  A dense model with use_cache=True decodes the beams on the shared cache
(the prompt's K / V once, lmod_kv_beam_reorder moving the rows past it) and returns, byte for byte, the tokens of the expanded form (the
inputs expanded nb times into a plain cache whose every row is reordered); the decisions are those of the host restatement
(tests/beam_oracle.py) replayed on the run's own per-step logits, and those logits are the ones a full forward of the running beams gives
(so the cache followed the beams).  The sparse student runs the expanded form; num_beams=1 is today's path."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests import helpers as Hh  # noqa: E402
from tests.beam_oracle import replay  # noqa: E402
from tests.test_num_return_gpu import MODELS, _inputs  # noqa: E402
from tests.test_ragged_decode_gpu import _logit_tol, _teacher  # noqa: E402


NO_EOS = 10 ** 6                   # an EOS id outside every vocabulary here: no hypothesis ends early


def _beam(model, ids, mask, imgs, nb, n, expand=False, trace=None, **kw):
    from llavamod.model import generation as Gm
    kw = dict(dict(max_new_tokens=10, use_cache=True, eos_token_id=[NO_EOS]), **kw)
    return Gm._beam_search(model, ids, images=imgs, attention_mask=mask, num_beams=nb, num_return_sequences=n, expand=expand, trace=trace,
                           **kw)


def _replayed(trace, B, nb, n, max_new, eos, pad, **kw):
    rows, _, _ = replay(lambda step, new: trace[step], B, nb, n, max_new, eos, pad, **kw)
    return rows


def _shared_entries(model):
    from llavamod.model import generation as Gm
    return [e for e in Gm._STEP_GRAPHS.values() if e["model"]() is model and e["cache"].shared]


@pytest.mark.parametrize("graphs", ["1", "0"])
@pytest.mark.parametrize("kind", ["unpadded", "left", "right"])
@pytest.mark.parametrize("images", [True, False])
@pytest.mark.parametrize("heads,kv_heads", MODELS)
def test_shared_path_equals_expanded_path_bytewise(monkeypatch, heads, kv_heads, images, kind, graphs):
    monkeypatch.setenv("LLAVAMOD_CUDA_GRAPHS", graphs)
    model = _teacher(heads, kv_heads, seed=80)
    ids, mask, imgs = _inputs(model, kind, images)
    T = ids.shape[1]
    for nb, n in ((2, 2), (3, 1), (4, 3)):
        trace = []
        got = model.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=10, use_cache=True, num_beams=nb, num_return_sequences=n,
                             eos_token_id=NO_EOS)
        want = _beam(model, ids, mask, imgs, nb, n, expand=True, trace=trace)
        assert got.shape[0] == 3 * n and torch.equal(got, want), (nb, n, kind)
        assert torch.equal(got[:, :T].cpu(), ids.repeat_interleave(n, 0))
        rows = _replayed(trace, 3, nb, n, 10, [NO_EOS], NO_EOS)
        assert got[:, T:].tolist() == rows, (nb, n)
    if graphs == "1":
        assert _shared_entries(model), "the cached path did not take the shared cache"


@pytest.mark.parametrize("heads,kv_heads", MODELS)
def test_cached_logits_follow_the_beams(heads, kv_heads):
    """Each step's logits of the shared-cache run equal (bf16 tolerance) a full forward, without a cache, of the running beams' ids that
    the host replay of the run's decisions holds at that step: the reorder moved the right rows."""
    from llavamod.model import generation as Gm
    model = _teacher(heads, kv_heads, seed=81)
    ids, _, imgs = _inputs(model, "unpadded", True)
    T, nb = ids.shape[1], 4
    trace = []
    got = _beam(model, ids, None, imgs, nb, nb, trace=trace, max_new_tokens=12, eos_token_id=[NO_EOS], pad_token_id=0)
    rows, _, steps = replay(lambda step, new: trace[step], 3, nb, nb, 12, [NO_EOS], 0)
    assert got[:, T:].tolist() == rows and len(steps) == 12
    x_imgs = [im for im in imgs for _ in range(nb)]
    moved = 0
    for s in range(1, 12):
        new = torch.tensor(steps[s - 1]["seqs"], dtype=torch.long)
        ref = Gm.next_token_logits(model, torch.cat([ids.repeat_interleave(nb, 0), new], 1).cuda(), images=x_imgs)
        assert (trace[s] - ref).abs().max().item() <= _logit_tol(ref), s
        moved += sum(p != j % nb for j, p in enumerate(steps[s - 1]["parents"]))
    assert moved > 0                                    # some beam took another's rows


def test_sparse_student_cached_and_uncached():
    from llavamod.model import generation as Gm
    student, teacher = Hh.tiny_pair(seed=9)
    student.eval()
    ids, mask, imgs = _inputs(teacher, "left", True)
    T = ids.shape[1]
    for use_cache in (True, False):
        trace = []
        torch.cuda.manual_seed(4)
        got = _beam(student, ids, mask, imgs, 3, 2, trace=trace, use_cache=use_cache, max_new_tokens=8, eos_token_id=[NO_EOS], pad_token_id=0)
        assert got.shape == (6, T + 8)
        assert got[:, T:].tolist() == _replayed(trace, 3, 3, 2, 8, [NO_EOS], 0), use_cache
    assert not _shared_entries(student)
    # a plain cache after a reorder equals index_select of the cache before it (rows below the length, the model's head columns)
    ent = Gm._decoder_entry(student, 6, 512)
    cache = ent["cache"]
    eids, emask, eimgs = Gm._expand(2, ids, mask, imgs)
    Gm.next_token_logits(student, eids.cuda(), images=torch.stack([im.cuda() for im in eimgs]), attention_mask=emask.cuda(), cache=cache,
                         ragged=True)
    before = [t.clone() for t in cache.k + cache.v]
    lens = cache.lengths[::2]
    parent = [1, 1, 0, 1, 1, 0]
    cache.reorder_beams(parent, 2)
    src = torch.tensor([b * 2 + p for b in range(3) for p in parent[b * 2:b * 2 + 2]], device="cuda")
    hd = cache.head_dim
    for t, t0 in zip(cache.k + cache.v, before):
        want = t0.clone()
        for b in range(3):
            want[2 * b:2 * b + 2, :, :lens[b], :hd] = t0.index_select(0, src)[2 * b:2 * b + 2, :, :lens[b], :hd]
        assert torch.equal(t.view(torch.int16), want.view(torch.int16))


class _Tok:
    """Every id decodes to 'x'; keyword 'xxxxx' is five ids, so KeywordsStoppingCriteria stops once every beam has 5 new tokens."""

    bos_token_id = None

    def __call__(self, text):
        return type("E", (), dict(input_ids=[7] * len(text)))()

    def batch_decode(self, ids, skip_special_tokens=True):
        return ["x" * ids.shape[1] for _ in range(ids.shape[0])]


@pytest.mark.parametrize("graphs", ["1", "0"])
def test_eos_and_keywords_stop(monkeypatch, graphs):
    from llavamod.mm_utils import KeywordsStoppingCriteria
    monkeypatch.setenv("LLAVAMOD_CUDA_GRAPHS", graphs)
    model = _teacher(2, 1, seed=83)
    ids, mask, imgs = _inputs(model, "left", True)
    T = ids.shape[1]
    trace = []
    first = _beam(model, ids, mask, imgs, 3, 3, trace=trace, max_new_tokens=16, eos_token_id=[NO_EOS], pad_token_id=0)
    eos = int(first[4, T + 2])                         # a token some beam emits early
    trace = []
    got = _beam(model, ids, mask, imgs, 3, 3, trace=trace, max_new_tokens=16, eos_token_id=[eos], pad_token_id=5)
    want = _beam(model, ids, mask, imgs, 3, 3, expand=True, max_new_tokens=16, eos_token_id=[eos], pad_token_id=5)
    assert torch.equal(got, want)
    assert got[:, T:].tolist() == _replayed(trace, 3, 3, 3, 16, [eos], 5)
    ended = 0
    for r in got[:, T:].tolist():
        if eos in r:
            ended += 1
            assert all(t == 5 for t in r[r.index(eos) + 1:])
    assert ended > 0
    crit = KeywordsStoppingCriteria(["xxxxx"], _Tok(), ids)
    gen = model.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=16, use_cache=True, num_beams=3, num_return_sequences=2,
                         stopping_criteria=[crit], eos_token_id=[eos], pad_token_id=5)
    trace = []
    got = _beam(model, ids, mask, imgs, 3, 2, trace=trace, max_new_tokens=16, stopping_criteria=[crit], eos_token_id=[eos], pad_token_id=5)
    assert torch.equal(gen, got) and len(trace) == 5 and got.shape[1] <= T + 6
    assert got[:, T:].tolist() == _replayed(trace, 3, 3, 2, 16, [eos], 5, stop_fn=lambda new: len(new[0]) >= 5)


def test_one_beam_is_todays_path(monkeypatch):
    from llavamod import kernels as K
    from llavamod.model import generation as Gm
    monkeypatch.setenv("LLAVAMOD_CUDA_GRAPHS", "1")
    model = _teacher(2, 1, seed=84)
    ids, mask, imgs = _inputs(model, "right", True)

    def no_reorder(*a, **kw):
        raise AssertionError("num_beams=1 launched the beam reorder")

    monkeypatch.setattr(K, "kv_beam_reorder", no_reorder)
    outs, keys = [], []
    for kw in ({}, dict(num_beams=1)):
        Gm._STEP_GRAPHS.clear()
        outs.append(model.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=10, use_cache=True, **kw))
        keys.append(list(Gm._STEP_GRAPHS))
    assert torch.equal(outs[0], outs[1]) and [k[1:] for k in keys[0]] == [k[1:] for k in keys[1]] and len(keys[0]) == 1
    monkeypatch.undo()
    # beams take the key num_return_sequences = nb takes
    Gm._STEP_GRAPHS.clear()
    model.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=10, use_cache=True, num_beams=3, eos_token_id=NO_EOS)
    k_beam = list(Gm._STEP_GRAPHS)
    Gm._STEP_GRAPHS.clear()
    model.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=10, use_cache=True, do_sample=True, num_return_sequences=3)
    assert [k[1:] for k in k_beam] == [k[1:] for k in Gm._STEP_GRAPHS] and k_beam[0][-1][:2] == ("share", 3)


def test_bad_arguments_raise():
    model = _teacher(2, 1, seed=85)
    ids, _, imgs = _inputs(model, "unpadded", True)
    with pytest.raises(NotImplementedError, match="beam-sample"):
        model.generate(ids, images=imgs, max_new_tokens=4, num_beams=2, do_sample=True)
    with pytest.raises(ValueError, match="assisted"):
        model.generate(ids, images=imgs, max_new_tokens=4, use_cache=True, num_beams=2, assistant_model=model)
    with pytest.raises(ValueError, match="num_beams"):
        model.generate(ids, images=imgs, max_new_tokens=4, num_beams=2, num_return_sequences=3)
    for use_cache in (True, False):                    # the tiny model's config has no EOS id
        with pytest.raises(NotImplementedError, match="eos_token_id"):
            model.generate(ids, images=imgs, max_new_tokens=4, num_beams=2, use_cache=use_cache)
        with pytest.raises(NotImplementedError, match="eos_token_id"):
            model.generate(ids, images=imgs, max_new_tokens=4, num_beams=2, use_cache=use_cache, eos_token_id=[])
    assert not model.training


def test_config_scale_teacher_beams_share_the_prompt():
    """The 7B teacher at T' = 650, 2 prompts, nb = 3, 12 new tokens: shared equals expanded, and the shared cache is smaller."""
    from llavamod.model import synthetic as S
    teacher = S.make_teacher("qwen1.5-7b", "clip-l-336", seed=7).eval()
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(0, 150000, (2, 75), generator=g)
    ids[:, 3] = -200
    imgs = [torch.randn(3, 336, 336, generator=g).to(torch.bfloat16) for _ in range(2)]
    got = teacher.generate(ids, images=imgs, max_new_tokens=12, use_cache=True, num_beams=3, eos_token_id=NO_EOS)
    cache = _shared_entries(teacher)[-1]["cache"]
    assert cache.share == 3 and cache.nbytes < teacher.new_kv_cache(6, cache.max_len).nbytes
    want = _beam(teacher, ids, None, imgs, 3, 1, expand=True, max_new_tokens=12)
    assert torch.equal(got, want)
