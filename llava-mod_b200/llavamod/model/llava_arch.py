"""LLaVA glue: vision-module construction, ``encode_images`` and the multimodal splice.

Stands in for ``llavamod/model/llava_arch.py`` (LlavaMetaModel :27-128, encode_images :143-148,
prepare_inputs_labels_for_multimodal :155-334; image branch only -- 4-D video entries are out of scope).

The splice is split in two: the INTEGER plan (which embedding row / image-feature row feeds every output
position, the new labels, mask and position ids) is computed on the host from the host copy of ``input_ids`` --
the reference does the same work on the device with two host syncs (llava_arch.py:237,247) -- and the float part
is one gather kernel (``lmod_splice_embed``) whose backward scatters into the projector output.
"""
from abc import ABC, abstractmethod

import numpy as np
import torch

from .. import kernels as K
from ..constants import IGNORE_INDEX, IMAGE_TOKEN_INDEX
from .multimodal_encoder.builder import build_image_tower
from .multimodal_projector.builder import build_projector

PAD_SRC = -(1 << 40)


def splice_plan(input_ids, attention_mask, labels, n_patches, padding_side="right", max_len=None):
    """Host-side integer plan (numpy).  input_ids/labels [B,Tt] int64, attention_mask [B,Tt] bool or None.
    Returns src, new_labels, new_mask, position_ids, img_index (all [B,T'] numpy arrays).
    src >= 0: token id ; src = -1-k: row k of image ``img_index`` ; PAD_SRC: padding (zero embedding)."""
    ids = np.asarray(input_ids)
    B, Tt = ids.shape
    mask = np.ones_like(ids, dtype=bool) if attention_mask is None else np.asarray(attention_mask).astype(bool)
    labs = np.full_like(ids, IGNORE_INDEX) if labels is None else np.asarray(labels)
    rows, cur_img = [], 0
    ar = np.arange(n_patches, dtype=np.int64)
    for b in range(B):
        cid, clab = ids[b][mask[b]], labs[b][mask[b]]
        where = np.nonzero(cid == IMAGE_TOKEN_INDEX)[0]
        if where.size == 0:
            rows.append((cid.astype(np.int64), clab.astype(np.int64), np.full(cid.shape, -1, np.int64)))
            cur_img += 1                                   # llava_arch.py:238-245: still consumes one feature entry
            continue
        src_parts, lab_parts, img_parts = [], [], []
        prev = 0
        for w in where:
            src_parts.append(cid[prev:w]); lab_parts.append(clab[prev:w]); img_parts.append(np.full(w - prev, -1, np.int64))
            src_parts.append(-1 - ar); lab_parts.append(np.full(n_patches, IGNORE_INDEX, np.int64))
            img_parts.append(np.full(n_patches, cur_img, np.int64))
            cur_img += 1
            prev = w + 1
        src_parts.append(cid[prev:]); lab_parts.append(clab[prev:]); img_parts.append(np.full(cid.shape[0] - prev, -1, np.int64))
        rows.append((np.concatenate(src_parts).astype(np.int64), np.concatenate(lab_parts).astype(np.int64), np.concatenate(img_parts)))
    if max_len is not None:                                # tokenizer_model_max_length truncation (llava_arch.py:280-283)
        rows = [(s[:max_len], l[:max_len], i[:max_len]) for s, l, i in rows]
    Tm = max(r[0].shape[0] for r in rows)
    src = np.full((B, Tm), PAD_SRC, np.int64)
    nl = np.full((B, Tm), IGNORE_INDEX, np.int64)
    nm = np.zeros((B, Tm), bool)
    pos = np.zeros((B, Tm), np.int64)
    img = np.full((B, Tm), -1, np.int64)
    for b, (s, l, i) in enumerate(rows):
        n = s.shape[0]
        if n == 0:
            continue
        sl = slice(Tm - n, Tm) if padding_side == "left" else slice(0, n)
        src[b, sl], nl[b, sl], nm[b, sl], pos[b, sl], img[b, sl] = s, l, True, np.arange(n), i
    return src, nl, nm, pos, img


class MaskInfo:
    """Attention mask + the host-side knowledge whether it contains padding, so the decoder never has to ask the device
    (``bool(mask.all())`` would be a host sync and would break CUDA-graph capture)."""

    def __init__(self, mask, all_true):
        self.mask = mask
        self.all_true = bool(all_true)

    def all(self):
        return self.all_true


class LlavaMetaModel:
    """Mixin for the ``model`` attribute (reference: llava_arch.py:27-128)."""

    def _init_vision(self, config, device, dtype):
        if getattr(config, "mm_image_tower", None) is not None:
            self.image_tower = build_image_tower(config, delay_load=True, device=device, dtype=dtype)
            self.mm_projector = build_projector(config, device=device, dtype=dtype)

    def get_image_tower(self):
        image_tower = getattr(self, "image_tower", None)
        if type(image_tower) is list:
            image_tower = image_tower[0]
        return image_tower

    def get_video_tower(self):
        return None

    def initialize_vision_modules(self, model_args, fsdp=None):
        image_tower = model_args.image_tower
        if getattr(model_args, "video_tower", None) is not None:
            raise NotImplementedError("video towers are outside the distillation hot path")
        assert image_tower is not None
        dev, dt = self.embed_tokens.weight.device, self.embed_tokens.weight.dtype
        self.config.mm_image_tower = image_tower
        if self.get_image_tower() is None:
            tower = build_image_tower(model_args, device=dev, dtype=dt)
            self.image_tower = [tower] if (fsdp is not None and len(fsdp) > 0) else tower
        else:
            tower = self.get_image_tower()
            tower.load_model()
        self.config.mm_video_tower = None
        self.config.use_mm_proj = True
        self.config.image_projector_type = getattr(model_args, "image_projector_type", None)
        self.config.mm_hidden_size = tower.hidden_size
        self.config.mm_vision_select_layer = model_args.mm_vision_select_layer
        self.config.mm_vision_select_feature = getattr(model_args, "mm_vision_select_feature", "patch")
        if getattr(self, "mm_projector", None) is None:
            self.mm_projector = build_projector(self.config, device=dev, dtype=dt)
        else:
            for p in self.mm_projector.parameters():        # "In case it is frozen by LoRA" (llava_arch.py:117-120)
                p.requires_grad = True
        pre = getattr(model_args, "pretrain_mm_mlp_adapter", None)
        if pre is not None:
            w = torch.load(pre, map_location="cpu", weights_only=True)
            sd = {k.split("mm_projector.")[1]: v for k, v in w.items() if "mm_projector" in k}
            from .builder_io import load_into
            load_into(self.mm_projector, sd, strict=True)


class LlavaMetaForCausalLM(ABC):
    @abstractmethod
    def get_model(self):
        pass

    def get_image_tower(self):
        return self.get_model().get_image_tower()

    def get_video_tower(self):
        return None

    def encode_images(self, images, tower_features=None):
        """CLIP tower (frozen, no grad) -> projector (trainable).  ``tower_features`` lets a trainer share one tower pass
        between a teacher and a student that hold identical frozen towers (SURVEY.md Appendix B)."""
        if tower_features is None:
            tower_features = self.get_model().get_image_tower()(images)
        n, P, C = tower_features.shape
        out = self.get_model().mm_projector.forward_image(tower_features.reshape(n * P, C))
        return out.view(n, P, -1)

    def make_splice_plan(self, input_ids, attention_mask, labels, n_patches=None, device=None):
        """Host integer plan -> device tensors; reusable across the teacher and the student forward of one micro-batch."""
        tower = self.get_image_tower()
        n_patches = n_patches if n_patches is not None else tower.num_patches
        dev = device if device is not None else self.get_model().embed_tokens.weight.device
        ids_h = input_ids.cpu().numpy() if torch.is_tensor(input_ids) else input_ids
        am_h = None if attention_mask is None else (attention_mask.cpu().numpy() if torch.is_tensor(attention_mask) else attention_mask)
        lb_h = None if labels is None else (labels.cpu().numpy() if torch.is_tensor(labels) else labels)
        side = getattr(self.config, "tokenizer_padding_side", "right")
        src, nl, nm, pos, img = splice_plan(ids_h, am_h, lb_h, n_patches, side, getattr(self.config, "tokenizer_model_max_length", None))
        host = torch.from_numpy(np.stack([src, nl, pos, img, nm.astype(np.int64)]))
        if dev.type == "cuda":
            host = host.pin_memory()
        plan = host.to(dev, non_blocking=True)
        return dict(src=plan[0].contiguous(), labels=plan[1], pos=plan[2], img=plan[3].contiguous(), mask=plan[4].bool(),
                    all_true=bool(nm.all()), has_labels=labels is not None, has_mask=attention_mask is not None, n_patches=n_patches)

    def prepare_inputs_labels_for_multimodal(self, input_ids, position_ids, attention_mask, past_key_values, labels, images,
                                             tower_features=None, plan=None):
        tower = self.get_image_tower()
        if tower is None or images is None or input_ids.shape[1] == 1:
            return input_ids, position_ids, attention_mask, past_key_values, None, labels
        if any(getattr(im, "ndim", 3) != 3 for im in images):
            raise NotImplementedError("video inputs (4-D entries of `images`) are outside the distillation hot path")
        dev = self.get_model().embed_tokens.weight.device
        imgs = torch.stack([im.to(dev, non_blocking=True) for im in images]) if not torch.is_tensor(images) else images.to(dev)
        feats = self.encode_images(imgs, tower_features)                                   # [n_img, P, H]
        n_patches = feats.shape[1]
        if plan is None:   # host-side integer plan (a device tensor costs one sync, exactly like the reference's .sum()/.tolist())
            plan = self.make_splice_plan(input_ids, attention_mask, labels, n_patches, dev)
        core = self.get_model()
        embeds = K.splice_embed(feats, core.embed_tokens.weight, plan["src"], plan["img"], n_patches,
                                embed_grad=core.gview(core.embed_tokens.weight) if torch.is_grad_enabled() else None)
        if not plan["has_mask"]:
            new_mask = None
        else:       # "no padding" is known on the host, the decoder must not sync to find out
            new_mask = MaskInfo(plan["mask"], plan["all_true"])
        return None, plan["pos"], new_mask, past_key_values, embeds, (plan["labels"] if plan["has_labels"] else None)
