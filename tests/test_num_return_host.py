"""generate's num_return_sequences without a GPU: the argument checks, which run before anything touches the model, and the row layout
of the expanded inputs (HF's repeat_interleave(n, 0))."""
import pytest
import torch

from llavamod.model import generation as Gm


class _NoModel:
    """Stands in for a model: any attribute access fails, so a check that passes would show up as an AttributeError."""

    def __getattr__(self, name):
        raise AttributeError(name)


@pytest.mark.parametrize("kw,match", [
    (dict(num_return_sequences=2), "greedy search"),
    (dict(num_return_sequences=2, do_sample=True, assistant_model=object(), use_cache=True), "assisted generate"),
    (dict(num_return_sequences=0, do_sample=True), ">= 1"),
])
def test_argument_checks(kw, match):
    with pytest.raises(ValueError, match=match):
        Gm.generate(_NoModel(), torch.zeros(2, 3, dtype=torch.long), max_new_tokens=4, **kw)


def test_num_return_sequences_is_not_swallowed():
    import inspect
    assert "num_return_sequences" in inspect.signature(Gm.generate).parameters


def test_expanded_row_layout():
    ids = torch.tensor([[1, 2, 3], [4, 5, 6]])
    mask = torch.tensor([[0, 1, 1], [1, 1, 1]], dtype=torch.bool)
    imgs = [torch.full((3, 2, 2), 1.0), torch.full((3, 2, 2), 2.0)]
    e_ids, e_mask, e_imgs = Gm._expand(3, ids, mask, imgs)
    assert e_ids.tolist() == [[1, 2, 3]] * 3 + [[4, 5, 6]] * 3                 # row b*n + j is copy j of prompt b
    assert torch.equal(e_mask, mask.repeat_interleave(3, 0))
    assert [float(im[0, 0, 0]) for im in e_imgs] == [1.0] * 3 + [2.0] * 3
    _, none_mask, t_imgs = Gm._expand(2, ids, None, torch.stack(imgs))
    assert none_mask is None and t_imgs.shape[0] == 4 and t_imgs[:, 0, 0, 0].tolist() == [1.0, 1.0, 2.0, 2.0]
