"""Float64 restatement of the frozen CLIP tower (CLIPVisionModel.hidden_state in llavamod/model/multimodal_encoder/clip_encoder.py) stage
by stage, with the element-wise bound of each stage's kernel, and the weights the exact tower tests run with.

Each stage reference takes its input as given (on the GPU: the kernel's own output of the stage before), so its bound covers the
arithmetic of one stage.  tower_chain_fp64 runs the same stage references on their own float64 outputs; tests/test_clip_tower_reference.py
pins that chain against oracle.restated.clip_tower, so a stage reference that computes the wrong thing cannot pass unnoticed.
  patch     conv2d(images, W, stride p) as [n*g*g, H] rows, the GEMM bound at the padded reduction length Kpad (helpers._gemm_tol)
  linear    x W^T (+ b), the GEMM bound with |b| in the majorant (as tests/test_gemm_exact_gpu.py)
  attention non-causal softmax attention of all heads (helpers.attn_reference_fp64) on the heads zero-padded to the kernel's width
The layernorm and quick-GELU stages use helpers.layernorm_reference_fp64 and helpers.bias_act_reference_fp64; the embedding and residual
adds are bf16 adds (fp32 sum rounded once), compared by bits against torch's."""
import math

import torch
import torch.nn.functional as F

from tests.helpers import _gemm_tol, attn_reference_fp64, layernorm_reference_fp64

F64 = torch.float64


def kpad(k):
    """The patch GEMM's reduction length: C*p*p rounded up to a multiple of 8 (16-byte rows)."""
    return (k + 7) // 8 * 8


def im2col(x, p, kp=None):
    """[n, C, S, S] images -> [n*g*g, C*p*p] patch rows, g = S / p: row (i, gy, gx) holds patch (gy, gx) of image i channel-major (the
    conv weight's [H, C, p, p] layout), so pixel (c, y, x) lands in column c*p*p + (y mod p)*p + x mod p.  Zero columns on the right up
    to kp."""
    n, C, S, _ = x.shape
    g = S // p
    cols = x.reshape(n, C, g, p, g, p).permute(0, 2, 4, 1, 3, 5).reshape(n * g * g, C * p * p)
    return cols if kp is None or kp == cols.shape[1] else F.pad(cols, (0, kp - cols.shape[1]))


def im2col_column(c, y, x, p):
    return c * p * p + (y % p) * p + x % p


def patch_embed_reference_fp64(images, w, kp):
    """conv2d(images, w, stride p), no bias, as [n*g*g, H] rows (row i*g*g + gy*g + gx), and its bound at reduction length kp."""
    p = w.shape[-1]
    x64, w64 = images.to(F64), w.to(F64)

    def conv(a, b):
        return F.conv2d(a, b, stride=p).flatten(2).transpose(1, 2).reshape(-1, w.shape[0])
    want = conv(x64, w64)
    return want, _gemm_tol(want, conv(x64.abs(), w64.abs()), kp)


def linear_reference_fp64(x, w, b=None):
    """x [M, K] W [N, K]^T (+ b [N]) and its bound (reduction length K)."""
    x64, w64 = x.to(F64), w.to(F64)
    want, maj = x64 @ w64.t(), x64.abs() @ w64.abs().t()
    if b is not None:
        want, maj = want + b.to(F64), maj + b.to(F64).abs()
    return want, _gemm_tol(want, maj, x.shape[-1])


def attention_reference_fp64(qkv, n, T, nh, hd, hd_kernel=None):
    """Non-causal attention of the fused [n*T, 3 nh hd] q|k|v rows, scale hd^-0.5 -> (o [n*T, nh hd], bound).  hd_kernel: the head width
    the kernel runs (hd zero-padded to it, as kernels.attention does); the bound is taken at that width, whose extra score terms are
    exact zeros."""
    hp = hd_kernel or hd
    rows = qkv.shape[0]
    x = qkv.to(F64)
    if hp != hd:
        x = F.pad(x.view(rows, 3 * nh, hd), (0, hp - hd)).reshape(rows, 3 * nh * hp)
    ref = attn_reference_fp64(x, n, T, nh, nh, hp, False, hd ** -0.5)

    def unpad(t):
        return t if hp == hd else t.view(rows, nh, hp)[:, :, :hd].reshape(rows, nh * hd)
    return unpad(ref["o"]), unpad(ref["o_tol"])


def embed_reference(pe, cls, pos, n):
    """[class row | patch rows] + position embedding, [n, T, H], in pe's dtype (for bf16: torch's add, the fp32 sum rounded once)."""
    H = pe.shape[-1]
    seq = torch.cat([cls.to(pe.dtype).expand(n, 1, H), pe.reshape(n, -1, H)], 1)
    return seq + pos.to(pe.dtype)[None]


def tower_chain_fp64(sd, c, images, n_layers, pre="vision_model."):
    """The stage references above, each on the previous one's float64 output: the residual stream [n, T, H] after 0..n_layers encoder
    layers (entry 0 is the pre_layrnorm output), hidden_states[k] of transformers' CLIPVisionModel.  sd: the tower's state dict (keys of
    CLIPVisionModel.state_dict()), c: its CLIPVisionConfig."""
    def g(k):
        return sd[pre + k].to(F64)
    x = images.to(F64)
    n, H, nh = x.shape[0], c.hidden_size, c.num_attention_heads
    hd = H // nh
    w = g("embeddings.patch_embedding.weight")
    pe, _ = patch_embed_reference_fp64(x, w, kpad(w[0].numel()))
    seq = embed_reference(pe, g("embeddings.class_embedding"), g("embeddings.position_embedding.weight"), n)
    T = seq.shape[1]
    h = layernorm_reference_fp64(seq.reshape(n * T, H), g("pre_layrnorm.weight"), g("pre_layrnorm.bias"), c.layer_norm_eps)["y"]
    out = [h]
    for i in range(n_layers):
        def lw(k):
            return g(f"encoder.layers.{i}.{k}")
        y = layernorm_reference_fp64(h, lw("layer_norm1.weight"), lw("layer_norm1.bias"), c.layer_norm_eps)["y"]
        qkv, _ = linear_reference_fp64(y, torch.cat([lw(f"self_attn.{m}_proj.weight") for m in "qkv"]),
                                       torch.cat([lw(f"self_attn.{m}_proj.bias") for m in "qkv"]))
        o, _ = attention_reference_fp64(qkv, n, T, nh, hd)
        o, _ = linear_reference_fp64(o, lw("self_attn.out_proj.weight"), lw("self_attn.out_proj.bias"))
        h = h + o
        y = layernorm_reference_fp64(h, lw("layer_norm2.weight"), lw("layer_norm2.bias"), c.layer_norm_eps)["y"]
        z, _ = linear_reference_fp64(y, lw("mlp.fc1.weight"), lw("mlp.fc1.bias"))
        f, _ = linear_reference_fp64(z * torch.sigmoid(1.702 * z), lw("mlp.fc2.weight"), lw("mlp.fc2.bias"))
        h = h + f
        out.append(h)
    return [t.view(n, T, H) for t in out]


# ---------------------------------------------------------------------------------------------------
# weights: N(0, 1/K) so that activations stay O(1) through 24 layers, plus the two features of a real CLIP tower that the 0.02 randn
# init lacks
# ---------------------------------------------------------------------------------------------------
OUTLIER_CH = 7            # a channel of +-150..250 in the position embedding: the residual stream's large-channel structure, which
OUTLIER = 200.0           # every layernorm then normalises (its mean and variance dominated by one channel)
FC1_BIG = 16              # fc1 rows scaled so that |z| reaches ~100: quick-GELU's sigmoid saturates at both ends
FC1_BIG_STD = 30.0


def init_tower_(model, seed):
    """Fill a CLIPVisionModel's weights in place (seeded, on the model's device, rounded to its dtype)."""
    c, vm = model.config, model.vision_model
    H, I, C, p = c.hidden_size, c.intermediate_size, c.num_channels, c.patch_size
    dev = model.device
    gen = torch.Generator(device=dev).manual_seed(seed)

    def rn(*shape, scale=1.0):
        return torch.randn(*shape, generator=gen, device=dev, dtype=torch.float32) * scale

    def norm_(m):
        m.weight.copy_(1 + 0.1 * rn(H))
        m.bias.copy_(0.1 * rn(H))

    with torch.no_grad():
        e = vm.embeddings
        e.patch_embedding.weight.copy_(rn(H, C, p, p, scale=1 / math.sqrt(C * p * p)))
        e.class_embedding.copy_(rn(H))
        pos = rn(*e.position_embedding.weight.shape, scale=0.5)
        n_pos = pos.shape[0]
        pos[:, OUTLIER_CH] = OUTLIER * rn(n_pos).sign() * (0.75 + 0.5 * torch.rand(n_pos, generator=gen, device=dev))
        e.position_embedding.weight.copy_(pos)
        norm_(vm.pre_layrnorm)
        norm_(vm.post_layernorm)
        for layer in vm.encoder.layers:
            a, m = layer.self_attn, layer.mlp
            a.qkv_weight.copy_(rn(3 * H, H, scale=1 / math.sqrt(H)))      # q|k|v_proj are views of this buffer
            a.qkv_bias.copy_(rn(3 * H, scale=0.1))
            a.out_proj.weight.copy_(rn(H, H, scale=1 / math.sqrt(H)))
            a.out_proj.bias.copy_(rn(H, scale=0.1))
            w1 = rn(I, H, scale=1 / math.sqrt(H))
            big = torch.randperm(I, generator=gen, device=dev)[:min(FC1_BIG, I // 4)]
            w1[big] *= FC1_BIG_STD
            m.fc1.weight.copy_(w1)
            m.fc1.bias.copy_(rn(I, scale=0.1))
            m.fc2.weight.copy_(rn(H, I, scale=1 / math.sqrt(I)))
            m.fc2.bias.copy_(rn(H, scale=0.1))
            norm_(layer.layer_norm1)
            norm_(layer.layer_norm2)
    return model


# ---------------------------------------------------------------------------------------------------
# planted single-pixel images for the im2col layout
# ---------------------------------------------------------------------------------------------------
PIXEL_VALUES = (1.0, -2.0, 0.5, 4.0, -0.25)       # powers of two: w * v is exact in bf16


def planted_pixels(S, p):
    """Per image, the (channel, y, x) pixels that are non-zero: the four corners, the last row and column, channels 0 and 2, the last pixel
    of the first patch, the first pixel of patch (1, 1), and (2, S-1, S-1), the last real im2col column (k = 3 p p - 1).  No two pixels of
    one image share a patch."""
    L, h = S - 1, S // 2
    return [[(0, 0, 0), (1, 0, L), (2, L, 0), (0, L, L), (1, p + 3, 2 * p + 5)],
            [(2, L, L), (1, L, h), (0, h + 1, L), (2, p - 1, p - 1)],
            [(0, p, p), (2, 0, 0), (1, L, L)]]


def planted_images(S, p, C=3):
    """[3, C, S, S] float32 images, zero except planted_pixels (values cycling through PIXEL_VALUES); returns (images, [(image, c, y, x,
    value)])."""
    imgs = torch.zeros(3, C, S, S)
    where = []
    j = 0
    for i, px in enumerate(planted_pixels(S, p)):
        for (c, y, x) in px:
            v = PIXEL_VALUES[j % len(PIXEL_VALUES)]
            j += 1
            imgs[i, c, y, x] = v
            where.append((i, c, y, x, v))
        patches = [(y // p, x // p) for (_, y, x) in px]
        assert len(set(patches)) == len(patches), "two planted pixels share a patch"
    return imgs, where
