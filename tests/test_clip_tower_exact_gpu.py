"""The frozen CLIP tower (CLIPVisionModel.hidden_state in llavamod/model/multimodal_encoder/clip_encoder.py) element by element against
float64 at the CLIP-L/14 shapes every workload runs, and the production path bit for bit against a stage replica.

The replica calls the llavamod.kernels functions of hidden_state in its order, with the same glue (im2col, padding, the class row, the
position rows).  After every call the stage is checked against the float64 reference of tests/clip_oracle.py computed from the kernel's
own output of the stage before:
  im2col + patch GEMM (K = 3 p p zero-padded to 592 at patch 14)   GEMM bound against conv2d in float64
  class row + position add, both residual adds                      bit for bit against torch's bf16 add
  pre_layrnorm, LN1, LN2                                            layernorm bound
  q|k|v GEMM + bias, out_proj + bias, fc1, fc2 + bias               GEMM bound (with |bias| in the majorant)
  non-causal attention (T = 577 / 257 / 17, head dim 64 / 16)       attention bound
  bias_act quick-GELU                                               bias_act bound
in every encoder layer, all of them (so that every select_layer has a reference).  hidden_state then runs under a spy that compares each of
its kernel calls with the replica's, arguments and output, bit for bit, so a difference is reported at the first stage it reaches.

Weights are N(0, 1/K) with a +-200 outlier channel in the position embedding and fc1 rows with |z| up to ~100 (tests/clip_oracle.py
init_tower_).  Shapes: clip-l-336 with 1 and 3 images (with 3 the last, ragged tiles of image i reach into image i+1's rows), clip-l-224
with 2 images (T = 257 = 2 * 128 + 1) and the tiny golden tower (head dim 16: the attention's head padding).

The list-of-images path of CLIPVisionTower.forward is compared with the batched call bit for bit: every stage is row- or image-independent
and mm_nt never splits K, so the bytes of an image do not depend on the batch it runs in.  That includes the GEMM's tile width: on a
132-SM H100, fc1 (N = 4096) runs 256-wide tiles for 3 images at 336 px (14 row tiles) and 128-wide ones for one image (5 row tiles),
and the bytes of every image are still the same."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from tests import clip_oracle as O
from tests.helpers import (ACT_QUICK_GELU_REF, bias_act_reference_fp64, check_attn, check_bound, layernorm_reference_fp64,
                           poisoned_uninitialised_memory)

pytestmark = pytest.mark.gpu

BF16, DEV = torch.bfloat16, "cuda"
CLIP_EPS = 1e-5            # nn.LayerNorm eps of every CLIP-L tower (layer_norm_eps in its config.json)
KERNEL_FNS = ("mm_nt", "add_", "layernorm", "attention", "bias_act")


def tower_config(name):
    from llavamod.model import synthetic as S
    from llavamod.model.multimodal_encoder.clip_encoder import CLIPVisionConfig
    d = {"clip-l-336": S.CLIP["clip-l-336"], "clip-l-224": dict(S.CLIP["clip-l-336"], image_size=224),
         "tiny": dict(hidden_size=64, intermediate_size=128, num_hidden_layers=3, num_attention_heads=4, image_size=32, patch_size=8)}[name]
    c = CLIPVisionConfig(**d)
    assert c.layer_norm_eps == CLIP_EPS
    return c


def make_tower(cfg, seed):
    from llavamod.model.multimodal_encoder.clip_encoder import CLIPVisionConfig, CLIPVisionModel
    c = cfg if isinstance(cfg, CLIPVisionConfig) else tower_config(cfg)
    return O.init_tower_(CLIPVisionModel(c, DEV, BF16), seed)


def images_of(n, S, seed):
    """fp32 images (CLIP-normalised pixels are about N(0, 1))."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(n, 3, S, S, generator=g, device=DEV)


def bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32) if t.element_size() == 4 else t


def same_bits(a, b):
    if not torch.is_tensor(a):
        return a == b
    return torch.is_tensor(b) and a.dtype == b.dtype and a.shape == b.shape and torch.equal(bits(a), bits(b))


class KernelCalls:
    """Spies on the llavamod.kernels functions hidden_state calls.  Each finished call is an entry {fn, args, kw, out, stage}, with the
    tensor arguments cloned before the call (add_ writes in place).  With `expect` (the log of another run), every call is compared with
    the entry of the same index, bit for bit, instead of being kept."""

    def __init__(self, expect=None):
        from llavamod import kernels
        self.K, self.expect, self.log, self.count = kernels, expect, [], 0

    def __enter__(self):
        self.orig = {name: getattr(self.K, name) for name in KERNEL_FNS}
        for name, fn in self.orig.items():
            setattr(self.K, name, self._spy(name, fn))
        return self

    def __exit__(self, *exc):
        for name, fn in self.orig.items():
            setattr(self.K, name, fn)

    def _spy(self, name, fn):
        def clone(v):
            return v.clone() if torch.is_tensor(v) else v

        def call(*args, **kw):
            snap = [clone(a) for a in args], {k: clone(v) for k, v in kw.items()}
            out = fn(*args, **kw)
            e = dict(fn=name, args=snap[0], kw=snap[1], out=out.clone(), stage="(inside kernels.%s)" % name)
            if self.expect is None:
                self.log.append(e)
            else:
                self._compare(e)
            self.count += 1
            return out
        return call

    def _compare(self, e):
        i = self.count
        assert i < len(self.expect), f"hidden_state makes more kernel calls than the replica ({len(self.expect)}); call {i} is {e['fn']}"
        r = self.expect[i]
        where = f"kernel call {i} ({r['stage']})"
        assert e["fn"] == r["fn"], f"{where}: hidden_state calls kernels.{e['fn']}, the replica kernels.{r['fn']}"
        assert len(e["args"]) == len(r["args"]) and e["kw"].keys() == r["kw"].keys(), f"{where}: different arguments"
        for j, (a, b) in enumerate(list(zip(e["args"], r["args"])) + [(e["kw"][k], r["kw"][k]) for k in r["kw"]]):
            assert same_bits(a, b), f"{where}: argument {j} differs from the replica's" + ("" if torch.is_tensor(a) else f" ({a!r} != {b!r})")
        assert same_bits(e["out"], r["out"]), f"{where}: the output differs from the replica's"


def replica(tower, images, report):
    """hidden_state's kernel calls for every encoder layer, each stage checked against float64 from the kernel's own previous stage.
    Returns (the residual stream [n, T, H] after 0..num_hidden_layers layers, the KernelCalls log with each entry's stage named)."""
    c, vm = tower.config, tower.vision_model
    from llavamod import kernels as K
    x = images.to(DEV, BF16)
    n, C = x.shape[0], c.num_channels
    p, g = c.patch_size, c.image_size // c.patch_size
    H, nh = c.hidden_size, c.num_attention_heads
    hd, T, eps = H // nh, g * g + 1, c.layer_norm_eps
    hp = K.attn_head_dim(hd)
    calls = KernelCalls()

    def chk(stage, layer, got, want, tol=None, attn=False):
        name = stage if layer is None else f"layer {layer} {stage}"
        calls.log[-1]["stage"] = name
        worst = check_attn(name, got, want, tol, T, hd) if attn else check_bound(name, got, want, tol)
        report[stage] = max(report.get(stage, 0.0), worst)

    def ln_ref(m, t):
        r = layernorm_reference_fp64(t, m.weight, m.bias, CLIP_EPS)
        return r["y"], r["tol"]

    with calls:
        w = vm.embeddings.patch_embedding.weight
        k = C * p * p
        kp = O.kpad(k)
        w2 = F.pad(w.detach().reshape(H, k), (0, kp - k))
        pe = K.mm_nt(O.im2col(x, p, kp).contiguous(), w2)
        chk("patch GEMM", None, pe, *O.patch_embed_reference_fp64(x, w, kp))
        seq = torch.empty(n, T, H, device=DEV, dtype=BF16)
        seq[:, 0] = vm.embeddings.class_embedding
        seq[:, 1:] = pe.view(n, g * g, H)
        pos = vm.embeddings.position_embedding.weight[None].expand(n, T, H).contiguous()
        K.add_(seq, pos)
        chk("class row + position add", None, seq, O.embed_reference(pe, vm.embeddings.class_embedding,
                                                                     vm.embeddings.position_embedding.weight, n))
        h = K.layernorm(seq.view(n * T, H), vm.pre_layrnorm.weight, vm.pre_layrnorm.bias, eps)
        chk("pre_layrnorm", None, h, *ln_ref(vm.pre_layrnorm, seq.view(n * T, H)))
        hs = [h.clone()]
        for i, layer in enumerate(vm.encoder.layers):
            a, m = layer.self_attn, layer.mlp
            y = K.layernorm(h, layer.layer_norm1.weight, layer.layer_norm1.bias, eps)
            chk("LN1", i, y, *ln_ref(layer.layer_norm1, h))
            qkv = K.mm_nt(y, a.qkv_weight, a.qkv_bias)
            chk("q|k|v GEMM + bias", i, qkv, *O.linear_reference_fp64(y, a.qkv_weight, a.qkv_bias))
            o = K.attention(qkv, n, T, nh, nh, hd, causal=False, scale=hd ** -0.5)
            chk("attention", i, o, *O.attention_reference_fp64(qkv, n, T, nh, hd, hp), attn=True)
            o2 = K.mm_nt(o, a.out_proj.weight, a.out_proj.bias)
            chk("out_proj + bias", i, o2, *O.linear_reference_fp64(o, a.out_proj.weight, a.out_proj.bias))
            h0 = h.clone()
            K.add_(h, o2)
            chk("residual add 1", i, h, h0 + o2)
            y = K.layernorm(h, layer.layer_norm2.weight, layer.layer_norm2.bias, eps)
            chk("LN2", i, y, *ln_ref(layer.layer_norm2, h))
            f = K.mm_nt(y, m.fc1.weight)
            chk("fc1 GEMM", i, f, *O.linear_reference_fp64(y, m.fc1.weight))
            f2 = K.bias_act(f, m.fc1.bias, K.ACT_QUICK_GELU)
            r = bias_act_reference_fp64(f, m.fc1.bias, ACT_QUICK_GELU_REF)
            chk("bias_act quick-GELU", i, f2, r["y"], r["tol"])
            f3 = K.mm_nt(f2, m.fc2.weight, m.fc2.bias)
            chk("fc2 GEMM + bias", i, f3, *O.linear_reference_fp64(f2, m.fc2.weight, m.fc2.bias))
            h0 = h.clone()
            K.add_(h, f3)
            chk("residual add 2", i, h, h0 + f3)
            hs.append(h.clone())
    return [t.view(n, T, H) for t in hs], calls


def tower_wrapper(model, select_feature):
    """CLIPVisionTower (the module the models call) around an existing CLIPVisionModel."""
    import types
    from llavamod.model.multimodal_encoder.clip_encoder import CLIPVisionTower
    args = types.SimpleNamespace(mm_vision_select_layer=-2, mm_vision_select_feature=select_feature)
    t = CLIPVisionTower(model.config, args, delay_load=True, device=DEV)
    t.image_tower, t.is_loaded = model, True
    return t


CASES = [("clip-l-336", 1), ("clip-l-336", 3), ("clip-l-224", 2), ("tiny", 2)]


@pytest.mark.parametrize("name,n", CASES, ids=[f"{c}-x{n}" for c, n in CASES])
def test_tower_stage_by_stage(name, n):
    torch.cuda.reset_peak_memory_stats()
    tower = make_tower(name, seed=n)
    c = tower.config
    L, S = c.num_hidden_layers, c.image_size
    x32 = images_of(n, S, seed=100 + n)
    x = x32.to(BF16)
    report = {}
    with poisoned_uninitialised_memory():
        hs, calls = replica(tower, x, report)
        assert torch.isfinite(hs[-1].float()).all()
        # hidden_state at select_layer -1 runs every layer: each kernel call against the replica's, arguments and output
        with KernelCalls(expect=calls.log) as prod:
            out = tower.hidden_state(x, select_layer=-1)
        assert prod.count == len(calls.log), f"hidden_state makes {prod.count} kernel calls, the replica {len(calls.log)}"
    del calls
    assert same_bits(out, hs[L])
    # every select_layer, both forms: -1 = L, -2 = L - 1, ..., -(L + 1) = 0
    for k in list(range(L + 1)) + list(range(-1, -L - 2, -1)):
        assert same_bits(tower.hidden_state(x, select_layer=k), hs[k if k >= 0 else L + 1 + k]), f"select_layer={k}"
    # fp32 images: the bytes of the same images rounded to bf16
    assert same_bits(tower.hidden_state(x32, select_layer=-2), hs[L - 1])
    # CLIPVisionTower.forward: select_feature, the output dtype, and the list-of-images path
    for feat in ("patch", "cls_patch"):
        vt = tower_wrapper(tower, feat)
        want = hs[L - 1][:, 1:] if feat == "patch" else hs[L - 1]
        assert same_bits(vt(x), want), feat
        assert same_bits(vt(x32), want.float()), feat
        feats = vt([im for im in x])
        assert len(feats) == n
        for i, f in enumerate(feats):
            assert same_bits(f, want[i:i + 1]), f"{feat}: image {i} alone differs from the batched call"
    print(f"\nCLIPTOWER {name} x{n}: max err/bound " + ", ".join(f"{k} {v:.3g}" for k, v in report.items()) +
          f"; peak allocated {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


@pytest.mark.parametrize("name", ["clip-l-336", "clip-l-224", "tiny"])
def test_planted_pixels_select_one_weight_column(name):
    """Images that are zero except single pixels (tests/clip_oracle.py planted_pixels: corners, the last row and column, channels 0 and 2,
    the last real im2col column k = 3 p p - 1).  A patch holding pixel (c, y, x) of value v (a power of two) must come out of the patch
    GEMM as W2[:, c p p + (y mod p) p + x mod p] v exactly, and out of the position add as that plus its position row; every other patch
    as zeros and its position row; the class row as class_embedding + position row 0.  A transposed or channel-last im2col, or padding on
    the wrong side, moves these by O(1)."""
    tower = make_tower(name, seed=7)
    c, e = tower.config, tower.vision_model.embeddings
    p, S, H = c.patch_size, c.image_size, c.hidden_size
    g = S // p
    k = 3 * p * p
    imgs, where = O.planted_images(S, p)
    imgs = imgs.to(DEV)
    n = imgs.shape[0]
    with KernelCalls() as calls:
        tower.hidden_state(imgs, select_layer=0)
    gemm, add = calls.log[0], calls.log[1]
    assert gemm["fn"] == "mm_nt" and add["fn"] == "add_"
    w2 = gemm["args"][1]
    assert w2.shape == (H, O.kpad(k))
    check_bound("padded patch weight", w2[:, :k], e.patch_embedding.weight.reshape(H, k))
    assert int(w2[:, k:].ne(0).sum()) == 0, "the padding columns of the patch weight are not zero"
    pos = e.position_embedding.weight
    pe_want = torch.zeros(n * g * g, H, device=DEV, dtype=BF16)
    seq_want = pos[None].expand(n, g * g + 1, H).clone()
    seq_want[:, 0] = e.class_embedding + pos[0]
    for i, ch, y, xx, v in where:
        r = (y // p) * g + xx // p
        col = (w2[:, O.im2col_column(ch, y, xx, p)].float() * v).to(BF16)
        pe_want[i * g * g + r] = col
        seq_want[i, 1 + r] = col + pos[1 + r]
    check_bound("patch GEMM of planted pixels", gemm["out"], pe_want.double(), torch.zeros(pe_want.shape, dtype=torch.float64, device=DEV))
    check_bound("class row + position add of planted pixels", add["out"], seq_want)


CACHE_CFG = dict(hidden_size=64, intermediate_size=128, num_hidden_layers=1, num_attention_heads=1, image_size=56, patch_size=14)


@pytest.mark.parametrize("how", ["copy_", "load_state_dict_assign", "new_parameter", "data_repoint"])
def test_patch_weight_follows_every_way_of_replacing_it(how):
    """After the patch weight is written in place, loaded with assign=True, replaced by a new Parameter or re-pointed with `.data =`,
    hidden_state gives the output of a tower built fresh with those weights (K = 588 padded to 592).  The tower is used as built, as a
    checkpoint loader finds it: its weights were never written in place, so the replacement has the same version counter (0) as the weight
    it replaces, and a padded copy keyed on the version alone would be taken for current."""
    from llavamod.model.multimodal_encoder.clip_encoder import CLIPVisionConfig, CLIPVisionModel
    cfg = CLIPVisionConfig(**CACHE_CFG)
    torch.manual_seed(11)
    tower = CLIPVisionModel(cfg, DEV, BF16)
    x = images_of(2, cfg.image_size, seed=12).to(BF16)
    before = tower.hidden_state(x)                       # the padded weight of the old kernel was made here
    mod = tower.vision_model.embeddings.patch_embedding
    g = torch.Generator(device=DEV).manual_seed(13)
    new = (torch.randn(mod.weight.shape, generator=g, device=DEV) / 24).to(BF16)
    if how == "copy_":
        with torch.no_grad():
            mod.weight.copy_(new)
    elif how == "load_state_dict_assign":
        mod.load_state_dict({"weight": new.clone()}, assign=True)
    elif how == "new_parameter":
        mod.weight = nn.Parameter(new.clone(), requires_grad=False)
    else:
        mod.weight.data = new.clone()
    assert same_bits(mod.weight.detach(), new)
    got = tower.hidden_state(x)
    fresh = CLIPVisionModel(cfg, DEV, BF16)
    fresh.load_state_dict(tower.state_dict())            # copies into a tower that has never run
    assert same_bits(got, fresh.hidden_state(x)), f"{how}: hidden_state still uses the replaced patch weight"
    assert not same_bits(got, before)
