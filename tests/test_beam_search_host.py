"""generate's beam search without a GPU: the restatement of transformers 4.37's BeamSearchScorer (generation.BeamScorer) pinned against
the installed transformers' beam search on a stub causal LM whose logits are a fixed function of the ids, its 4.37 output layout, and the
argument checks.

The installed transformers (5.x) rewrote beam search as tensor ops; where it is known to differ from 4.37, the comparison says so:
- it fills the columns after a hypothesis with `pad_token_id or eos[0]` and keeps the EOS that ended it, where 4.37 appends eos[0] (also
  after a running beam that stopped short of max_new_tokens) and then pads: hypotheses are compared up to their first EOS;
- at the step that reaches max_new_tokens it finishes the top num_beams candidates together.  With early_stopping=True, when that step
  also brings a prompt's num_beams-th hypothesis, 4.37 marks the prompt done and finalize leaves its running beams out, while the
  installed version ranks them with the others (`_last_step_done`; those prompts are left out of the comparison, and
  `test_cases_cover_eos_and_a_prompt_finishing_first` bounds how many are);
- its early-stop test takes the best *running* beam's score, where 4.37's is_done takes the best candidate of the step, which may be an
  EOS.  No case of the grid reaches a different result through it."""
import functools

import pytest
import torch

from llavamod.model import generation as Gm
from tests.beam_oracle import replay

V = 13


@functools.lru_cache(maxsize=None)
def _row_logits(prefix):
    """fp32 [V]: the stub's next-token logits after the ids `prefix` (a tuple), seeded by a hash of the whole prefix."""
    h = 1469598103
    for t in prefix:
        h = (h * 1099511628211 + int(t) + 7) % (1 << 61)
    return torch.randn(V, generator=torch.Generator().manual_seed(h)) * 2.5


def _stub_logits(ids):
    return torch.stack([torch.stack([_row_logits(tuple(r[:t + 1])) for t in range(len(r))]) for r in ids.tolist()])


def _hf_model():
    transformers = pytest.importorskip("transformers")
    from transformers.modeling_outputs import CausalLMOutput

    class Cfg(transformers.PretrainedConfig):
        model_type = "lmod_beam_stub"

    class Stub(transformers.PreTrainedModel, transformers.GenerationMixin):
        config_class = Cfg

        def __init__(self, cfg):
            super().__init__(cfg)
            self.w = torch.nn.Parameter(torch.zeros(1))

        def forward(self, input_ids=None, **kw):
            return CausalLMOutput(logits=_stub_logits(input_ids))

        def prepare_inputs_for_generation(self, input_ids, **kw):
            return dict(input_ids=input_ids)

    return Stub(Cfg(vocab_size=V))


PROMPTS = torch.tensor([[1, 2, 4], [6, 5, 7], [9, 8, 11]])


def _ours(prompts, nb, n, max_new, eos, pad, lp, es, stop_fn=None):
    nbp = prompts.repeat_interleave(nb, 0).tolist()

    def logits(step, new):
        return torch.stack([_row_logits(tuple(p + s)) for p, s in zip(nbp, new)])

    return replay(logits, prompts.shape[0], nb, n, max_new, eos, pad, lp, es, stop_fn=stop_fn)


def _upto_eos(row, eos):
    out = []
    for t in row:
        if t in eos:
            break
        out.append(t)
    return out


CASES = [(nb, n, lp, es, eos)
         for nb in (2, 3, 4) for n in sorted({1, nb}) for lp in (1.0, 0.0, 2.0) for es in (False, True, "never")
         for eos in ([3], [3, 10])]


@pytest.mark.parametrize("nb,n,lp,es,eos", CASES)
def test_scorer_matches_installed_beam_search(nb, n, lp, es, eos):
    model = _hf_model()
    max_new = 7
    want = model.generate(PROMPTS, num_beams=nb, num_return_sequences=n, max_new_tokens=max_new, do_sample=False, use_cache=False,
                          eos_token_id=eos, pad_token_id=99, length_penalty=lp, early_stopping=es)
    rows, scorer, steps = _ours(PROMPTS, nb, n, max_new, eos, 99, lp, es)
    got = [_upto_eos(r, eos) for r in rows]
    ref = [_upto_eos(r, eos) for r in want[:, PROMPTS.shape[1]:].tolist()]
    for b in range(PROMPTS.shape[0]):
        if _last_step_done(steps, b, max_new, es):
            continue                                # the 4.37 corner of the module docstring
        assert got[b * n:(b + 1) * n] == ref[b * n:(b + 1) * n], (b, got, ref)


def _last_step_done(steps, b, max_new, es):
    """early_stopping=True and prompt b's num_beams-th hypothesis arrived at the step that reached max_new_tokens: 4.37 marks the prompt
    done, so finalize leaves its running beams out; the installed version finishes the top num_beams candidates of that step with it."""
    return es is True and len(steps) == max_new and steps[-1]["done"][b] and not (len(steps) > 1 and steps[-2]["done"][b])


def test_cases_cover_eos_and_a_prompt_finishing_first():
    """The grid above is not vacuous: hypotheses end in EOS, with one or two EOS ids, and some prompt is done while another runs on."""
    ended, mixed, second = 0, 0, 0
    for nb, n, lp, es, eos in CASES:
        rows, scorer, steps = _ours(PROMPTS, nb, n, 7, eos, 12, lp, es)
        ended += sum(any(t in eos for t in r) for r in rows)
        second += sum(10 in s["tokens"][b][:nb] for s in steps for b in range(3)) if 10 in eos else 0
        mixed += any(0 < sum(s["done"]) < 3 for s in steps)
    skipped = sum(_last_step_done(_ours(PROMPTS, nb, n, 7, eos, 99, lp, es)[2], b, 7, es) for nb, n, lp, es, eos in CASES for b in range(3))
    assert ended > 0 and mixed > 0 and second > 0, (ended, mixed, second)
    assert skipped <= len(CASES) * 3 // 10, skipped


def test_finalize_layout_is_437s():
    """Rows as wide as the longest hypothesis + 1 (at most max_new_tokens), eos[0] after each hypothesis where it fits (also after a
    running beam), then pad; best first; a hypothesis's score is sum_logprobs / len ** length_penalty."""
    s = Gm.BeamScorer(1, 2, 2, 1.0, False, 10, [3, 10], 12)
    s._add(0, [5, 6], -1.0, 3)                      # ended with an EOS at its third token: -1/3
    s.done[0] = False
    rows = s.finalize([[7, 8, 9, 1], [7, 8, 9, 2]], [-0.4, -3.0])     # running beams: -0.1 and -0.75
    assert rows == [[7, 8, 9, 1, 3], [5, 6, 3, 12, 12]]
    s = Gm.BeamScorer(1, 2, 1, 1.0, False, 4, [3], 12)
    assert s.finalize([[1, 2, 4, 5], [1, 2, 4, 6]], [-0.1, -0.2]) == [[1, 2, 4, 5]]   # max_new_tokens wide: no EOS fits


@pytest.mark.parametrize("es,lp,worst,best,cur,done", [
    (True, 1.0, -9.0, -0.1, 3, True),               # True: done once num_beams hypotheses exist
    (False, 1.0, -1.0, -2.0, 2, True),              # False: worst >= best / cur_len ** lp
    (False, 1.0, -1.0, -1.0, 2, False),
    ("never", 1.0, -1.0, -11.0, 2, True),           # "never", lp > 0: from max_new_tokens, -11 / 10 = -1.1
    ("never", 1.0, -1.0, -9.0, 2, False),           # -0.9 > -1
    ("never", -1.0, -1.0, -0.6, 2, True),           # "never", lp <= 0: from cur_len, -0.6 * 2 = -1.2
    ("never", -1.0, -1.0, -0.4, 2, False),          # -0.8 > -1
])
def test_is_done_modes(es, lp, worst, best, cur, done):
    s = Gm.BeamScorer(1, 1, 1, lp, es, 10, [3], 12)
    assert not s._is_done(0, best, cur)             # fewer than num_beams hypotheses: never done
    s.hyps[0], s.worst[0] = [(worst, [1])], worst
    assert s._is_done(0, best, cur) == done


class _NoModel:
    def __getattr__(self, name):
        raise AttributeError(name)


@pytest.mark.parametrize("kw,exc,match", [
    (dict(num_beams=0), ValueError, "num_beams"),
    (dict(num_beams=2, num_return_sequences=3), ValueError, "smaller or equal to num_beams"),
    (dict(num_beams=2, do_sample=True), NotImplementedError, "beam-sample"),
    (dict(num_beams=2, assistant_model=object(), use_cache=True), ValueError, "assisted"),
    (dict(num_beams=2, assistant_model=object(), use_cache=True), NotImplementedError, "assisted"),
])
def test_argument_checks(kw, exc, match):
    with pytest.raises(exc, match=match):
        Gm.generate(_NoModel(), torch.zeros(2, 3, dtype=torch.long), max_new_tokens=4, **kw)


@pytest.mark.parametrize("config_eos,eos", [(None, None), (None, []), (2, [])])
def test_beam_search_needs_an_eos_id(config_eos, eos):
    """Without an EOS id (neither the call's nor the config's) beam search is refused before the model runs."""
    import types

    class _Model:
        config = types.SimpleNamespace(eos_token_id=config_eos)

        def __getattr__(self, name):
            raise AttributeError(name)

    with pytest.raises(NotImplementedError, match="eos_token_id"):
        Gm.generate(_Model(), torch.zeros(1, 3, dtype=torch.long), max_new_tokens=4, num_beams=2, eos_token_id=eos)


def test_early_stopping_value_is_checked():
    with pytest.raises(ValueError, match="early_stopping"):
        Gm.BeamScorer(1, 2, 1, 1.0, "sometimes", 4, [3], 0)


def test_beam_arguments_are_not_swallowed():
    import inspect
    params = inspect.signature(Gm.generate).parameters
    assert params["num_beams"].default == 1 and params["length_penalty"].default == 1.0 and params["early_stopping"].default is False
