"""CLIP ViT vision tower, forward only (the tower is frozen in every LLaVA-MoD stage).

Stands in for ``llavamod/model/multimodal_encoder/clip_encoder.py:7-84`` + ``transformers.CLIPVisionModel``:
patch conv (no bias) + CLS + learned position embedding + pre-LN, pre-LN encoder layers with quick_gelu, feature
taken from ``hidden_states[select_layer]`` (select_layer=-2 -> the last encoder layer is never run, the reference
computes and discards it, clip_encoder.py:36,54), CLS dropped for ``select_feature == 'patch'``.

Parameter names follow HF CLIP (``vision_model.embeddings.patch_embedding.weight`` ... incl. the ``pre_layrnorm`` typo) so
the reference's checkpoints load.  q|k|v are one fused buffer; the patch conv runs as im2col + GEMM.
"""
import json
import os

import torch
import torch.nn as nn

from ... import kernels as K
from ..language_model.qwen2_core import ParamLinear, ParamNorm

KNOWN_TOWERS = {
    "clip-vit-large-patch14-336": dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24,
                                       num_attention_heads=16, image_size=336, patch_size=14, layer_norm_eps=1e-5,
                                       hidden_act="quick_gelu"),
    "clip-vit-large-patch14": dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24,
                                   num_attention_heads=16, image_size=224, patch_size=14, layer_norm_eps=1e-5,
                                   hidden_act="quick_gelu"),
}


class CLIPVisionConfig:
    model_type = "clip_vision_model"

    def __init__(self, hidden_size=768, intermediate_size=3072, num_hidden_layers=12, num_attention_heads=12,
                 num_channels=3, image_size=224, patch_size=32, hidden_act="quick_gelu", layer_norm_eps=1e-5, **kw):
        self.hidden_size, self.intermediate_size = hidden_size, intermediate_size
        self.num_hidden_layers, self.num_attention_heads = num_hidden_layers, num_attention_heads
        self.num_channels, self.image_size, self.patch_size = num_channels, image_size, patch_size
        self.hidden_act, self.layer_norm_eps = hidden_act, layer_norm_eps
        if hidden_act != "quick_gelu":
            raise NotImplementedError("CLIP hidden_act %r (only quick_gelu towers are on the path)" % hidden_act)

    @classmethod
    def from_pretrained(cls, path, **kw):
        with open(os.path.join(path, "config.json")) as f:
            d = json.load(f)
        if "vision_config" in d:
            d = d["vision_config"]
        return cls(**d)

    def to_dict(self):
        d = dict(self.__dict__)
        d["model_type"] = self.model_type
        return d


class _Embeddings(nn.Module):
    def __init__(self, c, device, dtype, std=0.02):
        super().__init__()
        n_pos = (c.image_size // c.patch_size) ** 2 + 1
        self.class_embedding = nn.Parameter(torch.randn(c.hidden_size, device=device, dtype=dtype) * std)
        self.patch_embedding = ParamLinear(torch.randn(c.hidden_size, c.num_channels, c.patch_size, c.patch_size, device=device, dtype=dtype) * std)
        self.position_embedding = ParamLinear(torch.randn(n_pos, c.hidden_size, device=device, dtype=dtype) * std)
        self._wcache = None

    def patch_weight_2d(self):
        """[hidden, Kpad] copy of the conv kernel, K = C*p*p zero-padded on the right to a multiple of 8 (16-byte rows for the GEMM).
        Kept until the weight changes.  The version counter alone only sees writes in place: a weight loaded with assign=True, a new
        Parameter or `.data =` brings its own counter, which can equal the old one.  So the key is the storage too (address, device,
        dtype, shape, strides), and the cache holds the tensor it was made from, so that its address cannot be handed to a new weight."""
        w = self.patch_embedding.weight.detach()
        key = (w.data_ptr(), w._version, w.device, w.dtype, w.shape, w.stride())
        if self._wcache is None or self._wcache[0] != key:
            k = w[0].numel()
            kp = (k + 7) // 8 * 8
            self._wcache = (key, w, torch.nn.functional.pad(w.reshape(w.shape[0], k), (0, kp - k)), kp)
        return self._wcache[2], self._wcache[3]


class _Attn(nn.Module):
    def __init__(self, c, device, dtype, std=0.02):
        super().__init__()
        H = c.hidden_size
        self.qkv_weight = torch.randn(3 * H, H, device=device, dtype=dtype) * std
        self.qkv_bias = torch.zeros(3 * H, device=device, dtype=dtype)
        self.k_proj = ParamLinear(self.qkv_weight[H:2 * H], self.qkv_bias[H:2 * H])
        self.v_proj = ParamLinear(self.qkv_weight[2 * H:], self.qkv_bias[2 * H:])
        self.q_proj = ParamLinear(self.qkv_weight[:H], self.qkv_bias[:H])
        self.out_proj = ParamLinear(torch.randn(H, H, device=device, dtype=dtype) * std, torch.zeros(H, device=device, dtype=dtype))


class _MLP(nn.Module):
    def __init__(self, c, device, dtype, std=0.02):
        super().__init__()
        H, I = c.hidden_size, c.intermediate_size
        self.fc1 = ParamLinear(torch.randn(I, H, device=device, dtype=dtype) * std, torch.zeros(I, device=device, dtype=dtype))
        self.fc2 = ParamLinear(torch.randn(H, I, device=device, dtype=dtype) * std, torch.zeros(H, device=device, dtype=dtype))


class _Layer(nn.Module):
    def __init__(self, c, device, dtype):
        super().__init__()
        H = c.hidden_size
        ones = lambda: torch.ones(H, device=device, dtype=dtype)      # noqa: E731
        zeros = lambda: torch.zeros(H, device=device, dtype=dtype)    # noqa: E731
        self.self_attn = _Attn(c, device, dtype)
        self.layer_norm1 = ParamNorm(ones(), zeros(), c.layer_norm_eps)
        self.mlp = _MLP(c, device, dtype)
        self.layer_norm2 = ParamNorm(ones(), zeros(), c.layer_norm_eps)


class _Encoder(nn.Module):
    def __init__(self, c, device, dtype):
        super().__init__()
        self.layers = nn.ModuleList([_Layer(c, device, dtype) for _ in range(c.num_hidden_layers)])


class _VisionTransformer(nn.Module):
    def __init__(self, c, device, dtype):
        super().__init__()
        H = c.hidden_size
        self.embeddings = _Embeddings(c, device, dtype)
        self.pre_layrnorm = ParamNorm(torch.ones(H, device=device, dtype=dtype), torch.zeros(H, device=device, dtype=dtype), c.layer_norm_eps)
        self.encoder = _Encoder(c, device, dtype)
        self.post_layernorm = ParamNorm(torch.ones(H, device=device, dtype=dtype), torch.zeros(H, device=device, dtype=dtype), c.layer_norm_eps)


class CLIPVisionModel(nn.Module):
    """Parameter container + forward of the frozen tower (``hidden_states[select_layer]`` only)."""

    def __init__(self, config, device="cuda", dtype=torch.bfloat16):
        super().__init__()
        self.config = config
        self.vision_model = _VisionTransformer(config, device, dtype)
        self.requires_grad_(False)

    @property
    def dtype(self):
        return self.vision_model.pre_layrnorm.weight.dtype

    @property
    def device(self):
        return self.vision_model.pre_layrnorm.weight.device

    @torch.no_grad()
    def hidden_state(self, images, select_layer=-2):
        c = self.config
        n_run = c.num_hidden_layers + 1 + select_layer if select_layer < 0 else select_layer
        if not 0 <= n_run <= c.num_hidden_layers:      # hidden_states has num_hidden_layers + 1 entries; a slice would clamp silently
            raise IndexError("select_layer %d out of range for a tower with hidden states 0..%d" % (select_layer, c.num_hidden_layers))
        vm = self.vision_model
        n = images.shape[0]
        p, g = c.patch_size, c.image_size // c.patch_size
        H, nh = c.hidden_size, c.num_attention_heads
        x = images.to(device=self.device, dtype=self.dtype)
        w2, kp = vm.embeddings.patch_weight_2d()
        # im2col: [n,3,g,p,g,p] -> [n*g*g, 3*p*p] (channel-major within a patch == conv weight layout)
        cols = x.view(n, c.num_channels, g, p, g, p).permute(0, 2, 4, 1, 3, 5).reshape(n * g * g, c.num_channels * p * p)
        if kp != cols.shape[1]:
            cols = torch.nn.functional.pad(cols, (0, kp - cols.shape[1]))
        pe = K.mm_nt(cols.contiguous(), w2).view(n, g * g, H)
        T = g * g + 1
        seq = torch.empty(n, T, H, device=x.device, dtype=x.dtype)
        seq[:, 0] = vm.embeddings.class_embedding
        seq[:, 1:] = pe
        pos = vm.embeddings.position_embedding.weight[None].expand(n, T, H).contiguous()
        K.add_(seq, pos)
        h = K.layernorm(seq.view(n * T, H), vm.pre_layrnorm.weight, vm.pre_layrnorm.bias, c.layer_norm_eps)
        hd = H // nh
        for layer in vm.encoder.layers[:n_run]:
            a = layer.self_attn
            y = K.layernorm(h, layer.layer_norm1.weight, layer.layer_norm1.bias, c.layer_norm_eps)
            qkv = K.mm_nt(y, a.qkv_weight, a.qkv_bias)
            o = K.attention(qkv, n, T, nh, nh, hd, causal=False, scale=hd ** -0.5)
            o = K.mm_nt(o, a.out_proj.weight, a.out_proj.bias)
            K.add_(h, o)
            y = K.layernorm(h, layer.layer_norm2.weight, layer.layer_norm2.bias, c.layer_norm_eps)
            f = K.mm_nt(y, layer.mlp.fc1.weight)
            f = K.bias_act(f, layer.mlp.fc1.bias, K.ACT_QUICK_GELU)
            f = K.mm_nt(f, layer.mlp.fc2.weight, layer.mlp.fc2.bias)
            K.add_(h, f)
        return h.view(n, T, H)


class CLIPVisionTower(nn.Module):
    """Same surface as the reference's CLIPVisionTower (clip_encoder.py:7-84)."""

    def __init__(self, image_tower, args, delay_load=False, cache_dir="./cache_dir", device="cuda", dtype=torch.bfloat16):
        super().__init__()
        self.is_loaded = False
        self.image_tower_name = image_tower
        self.select_layer = args.mm_vision_select_layer
        self.select_feature = getattr(args, "mm_vision_select_feature", "patch")
        self._device, self._dtype = device, dtype
        self.cfg_only = self._load_config()
        if not delay_load:
            self.load_model()

    def _load_config(self):
        name = self.image_tower_name
        if isinstance(name, CLIPVisionConfig):
            return name
        if isinstance(name, dict):
            return CLIPVisionConfig(**name)
        if os.path.isdir(str(name)) and os.path.exists(os.path.join(name, "config.json")):
            return CLIPVisionConfig.from_pretrained(name)
        base = os.path.basename(str(name).rstrip("/"))
        if base in KNOWN_TOWERS and os.environ.get("LLAVAMOD_ALLOW_RANDOM_INIT", "0") == "1":
            return CLIPVisionConfig(**KNOWN_TOWERS[base])
        raise FileNotFoundError("image tower %r: no local checkpoint directory (no network here); set "
                                "LLAVAMOD_ALLOW_RANDOM_INIT=1 to build a known architecture with random weights" % (name,))

    def load_model(self):
        if self.is_loaded:
            return
        self.image_tower = CLIPVisionModel(self.cfg_only, self._device, self._dtype)
        name = self.image_tower_name
        if isinstance(name, str) and os.path.isdir(name):
            from ..builder_io import load_state_dict_files
            sd = load_state_dict_files(name)
            sd = {k: v for k, v in sd.items() if k.startswith("vision_model.")}
            if sd:
                from ..builder_io import load_into
                load_into(self.image_tower, sd, strict=False)
        self.image_tower.requires_grad_(False)
        self.is_loaded = True

    def feature_select(self, hidden):
        if self.select_feature == "patch":
            return hidden[:, 1:]
        if self.select_feature == "cls_patch":
            return hidden
        raise ValueError(f"Unexpected select feature: {self.select_feature}")

    @torch.no_grad()
    def forward(self, images):
        if type(images) is list:
            return [self.feature_select(self.image_tower.hidden_state(im.unsqueeze(0), self.select_layer)).to(im.dtype) for im in images]
        return self.feature_select(self.image_tower.hidden_state(images, self.select_layer)).to(images.dtype)

    @property
    def image_processor(self):
        """CLIPImageProcessor for the data pipeline (reference clip_encoder.py:29: CLIPImageProcessor.from_pretrained(tower)).  Built from
        the checkpoint's preprocessor_config.json when there is one, else from the tower's image size with CLIP's mean / std."""
        if getattr(self, "_image_processor", None) is None:
            from transformers import CLIPImageProcessor
            name = self.image_tower_name
            if isinstance(name, str) and os.path.exists(os.path.join(name, "preprocessor_config.json")):
                self._image_processor = CLIPImageProcessor.from_pretrained(name)
            else:
                s = self.config.image_size
                self._image_processor = CLIPImageProcessor(size={"shortest_edge": s}, crop_size={"height": s, "width": s})
        return self._image_processor

    @property
    def dummy_feature(self):
        return torch.zeros(1, self.hidden_size, device=self.device, dtype=self.dtype)

    @property
    def dtype(self):
        return self.image_tower.dtype if self.is_loaded else self._dtype

    @property
    def device(self):
        return self.image_tower.device if self.is_loaded else torch.device(self._device)

    @property
    def config(self):
        return self.image_tower.config if self.is_loaded else self.cfg_only

    @property
    def hidden_size(self):
        return self.config.hidden_size

    @property
    def num_patches(self):
        return (self.config.image_size // self.config.patch_size) ** 2
