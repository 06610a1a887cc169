"""The float64 stage chain of tests/clip_oracle.py (which the exact CLIP tower test checks every kernel stage with) against
oracle.restated.clip_tower in float64, and the im2col + GEMM formulation of the patch embedding against F.conv2d.  CPU only."""
import pytest
import torch
import torch.nn.functional as F

from oracle import restated as R
from tests import clip_oracle as O

F64 = torch.float64

# (name, config, images): the tiny golden tower (head dim 16, K = 192 needs no padding) and a 2-layer tower of CLIP-L width at patch 14
# (K = 588 padded to 592, head dim 64)
TOWERS = [
    ("tiny", dict(hidden_size=64, intermediate_size=128, num_hidden_layers=3, num_attention_heads=4, image_size=32, patch_size=8), 2),
    ("clip-l-width-56px", dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=2, num_attention_heads=16, image_size=56,
                               patch_size=14), 2),
]


def build(cfg, seed):
    from llavamod.model.multimodal_encoder.clip_encoder import CLIPVisionConfig, CLIPVisionModel
    m = CLIPVisionModel(CLIPVisionConfig(**cfg), device="cpu", dtype=torch.bfloat16)
    return O.init_tower_(m, seed)


def images_of(n, S, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 3, S, S, generator=g).to(torch.bfloat16)


def assert_close64(name, got, want, rtol=1e-10):
    err = (got - want).abs().max().item()
    scale = want.abs().max().item()
    assert err <= rtol * scale, f"{name}: max |diff| {err:.3g} against max |ref| {scale:.3g}"


@pytest.mark.parametrize("name,cfg,n", TOWERS, ids=[t[0] for t in TOWERS])
def test_chain_matches_oracle(name, cfg, n):
    m = build(cfg, seed=len(name))
    c = m.config
    sd = {k: v.to(F64) for k, v in m.state_dict().items()}
    x = images_of(n, c.image_size, seed=1)
    hs = O.tower_chain_fp64(sd, c, x, c.num_hidden_layers)
    assert len(hs) == c.num_hidden_layers + 1
    for sel in range(-c.num_hidden_layers - 1, c.num_hidden_layers + 1):
        cc = R.ClipCfg(hidden=c.hidden_size, inter=c.intermediate_size, layers=c.num_hidden_layers, heads=c.num_attention_heads,
                       image=c.image_size, patch=c.patch_size, eps=c.layer_norm_eps, select_layer=sel)
        want = R.clip_tower(sd, cc, x.to(F64), pre="vision_model.")
        k = c.num_hidden_layers + 1 + sel if sel < 0 else sel
        assert_close64(f"{name} select_layer={sel}", hs[k][:, 1:], want)


def test_planted_features_reach_the_stages():
    """The init's outlier channel dominates the residual stream's variance and fc1 pre-activations reach |z| ~ 100, in the chain."""
    name, cfg, n = TOWERS[1]
    m = build(cfg, seed=3)
    c = m.config
    sd = {k: v.to(F64) for k, v in m.state_dict().items()}
    x = images_of(n, c.image_size, seed=4)
    h = O.tower_chain_fp64(sd, c, x, 1)
    pos = sd["vision_model.embeddings.position_embedding.weight"]
    assert pos[:, O.OUTLIER_CH].abs().min() >= 0.75 * O.OUTLIER
    from tests.helpers import layernorm_reference_fp64
    y = layernorm_reference_fp64(h[0].reshape(-1, c.hidden_size), sd["vision_model.encoder.layers.0.layer_norm2.weight"],
                                 sd["vision_model.encoder.layers.0.layer_norm2.bias"], c.layer_norm_eps)["y"]
    z = y @ sd["vision_model.encoder.layers.0.mlp.fc1.weight"].t() + sd["vision_model.encoder.layers.0.mlp.fc1.bias"]
    assert z.max() > 40 and z.min() < -40, (z.min().item(), z.max().item())


@pytest.mark.parametrize("sel", [-5, 4, 100, -100])
def test_select_layer_out_of_range_raises(sel):
    """hidden_states has num_hidden_layers + 1 entries (-4..3 for the 3-layer tower); outside that there is no layer to return (the layer
    slice used to clamp: -5 ran 2 layers, 4 ran 3).  Raised before any kernel runs."""
    m = build(TOWERS[0][1], seed=0)
    with pytest.raises(IndexError, match="select_layer"):
        m.hidden_state(images_of(1, 32, seed=0), select_layer=sel)


@pytest.mark.parametrize("n,S,p", [(2, 32, 8), (2, 56, 14), (1, 336, 14), (2, 224, 14)])
def test_im2col_gemm_matches_conv2d(n, S, p):
    g = torch.Generator().manual_seed(S + p)
    x = torch.randn(n, 3, S, S, generator=g, dtype=F64)
    w = torch.randn(64, 3, p, p, generator=g, dtype=F64)
    k = 3 * p * p
    kp = O.kpad(k)
    assert kp % 8 == 0 and kp - k < 8 and (kp == k) == (p == 8)
    cols = O.im2col(x, p, kp)
    assert cols.shape == (n * (S // p) ** 2, kp) and bool((cols[:, k:] == 0).all())
    got = cols @ F.pad(w.reshape(64, k), (0, kp - k)).t()
    want, tol = O.patch_embed_reference_fp64(x, w, kp)
    assert_close64(f"im2col {S}/{p}", got, want, rtol=1e-13)
    assert bool(((got - want).abs() <= tol).all())
    # the orders a kernel gets wrong are seen: patch rows transposed within an image, channel-last columns
    g_ = S // p
    swapped = x.reshape(n, 3, g_, p, g_, p).permute(0, 4, 2, 1, 3, 5).reshape(n * g_ * g_, k)
    chlast = x.reshape(n, 3, g_, p, g_, p).permute(0, 2, 4, 3, 5, 1).reshape(n * g_ * g_, k)
    for bad in (swapped, chlast):
        assert (bad @ w.reshape(64, k).t() - want).abs().max() > 1.0


@pytest.mark.parametrize("S,p", [(32, 8), (224, 14), (336, 14)])
def test_planted_pixels_select_one_column(S, p):
    imgs, where = O.planted_images(S, p)
    cols = O.im2col(imgs, p)
    g = S // p
    assert any(O.im2col_column(c, y, x, p) == 3 * p * p - 1 for _, c, y, x, _ in where)
    for i, c, y, x, v in where:
        r = i * g * g + (y // p) * g + x // p
        kcol = O.im2col_column(c, y, x, p)
        assert cols[r, kcol] == v
        assert int(cols[r].ne(0).sum()) == 1
    assert int(cols.ne(0).sum()) == len(where)
