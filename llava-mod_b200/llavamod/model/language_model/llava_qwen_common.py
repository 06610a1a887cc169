"""Shared implementation of the LLaVA-Qwen causal-LM wrappers (dense teacher/student and sparse-MoE student).

Reference classes mirrored here:
  * dense : ``LlavaQwen1_5ForCausalLM`` llava_qwen1_5.py:56-167 over ``Qwen2ForCausalLM`` modeling_qwen2.py:1110-1217
  * sparse: ``LLaVAMoDQwen1_5ForCausalLM`` llava_qwen1_5_moe.py:342-560, ``...FineTune`` :564-626, ``Eval...`` :629-681
The Qwen-1.5 and Qwen-2 files of the reference differ only in names, so the concrete classes in
``llava_qwen1_5*.py`` / ``llava_qwen2*.py`` just bind names to this implementation.
"""
import os
import warnings
from typing import List, Optional

import torch
import torch.nn as nn
from torch.autograd import Function

from ... import kernels as K
from ...constants import IGNORE_INDEX, IMAGE_TOKEN_INDEX
from ..builder_io import load_into, load_state_dict_files
from ..llava_arch import LlavaMetaForCausalLM, LlavaMetaModel
from ..utils import CausalLMOutputWithPast, MoECausalLMOutputWithPast
from .qwen2_core import KVCache, MoE, ParamLinear, Qwen2Config, Qwen2Model

CACHE_ROOM = 512          # positions a cache allocated by forward(use_cache=True) keeps free after the prompt


class LlavaQwenModelBase(LlavaMetaModel, Qwen2Model):
    def __init__(self, config, device="cuda", dtype=torch.bfloat16):
        Qwen2Model.__init__(self, config, device, dtype)
        self._init_vision(config, device, dtype)


class ShiftedCEFn(Function):
    """CrossEntropyLoss over shifted logits/labels (modeling_qwen2.py:1196-1204) on our log-prob kernels:
    loss = -(sum of gathered log-probs over non-ignored shifted labels) / count."""

    @staticmethod
    def forward(ctx, logits, labels):
        labels = labels.contiguous()
        seq, tok, lse = K.logp_gather(logits, labels)
        cnt = (labels[:, 1:] != IGNORE_INDEX).sum().to(torch.float32)
        ctx.save_for_backward(logits, labels, lse, cnt)
        return -seq.sum() / cnt

    @staticmethod
    def backward(ctx, g):
        logits, labels, lse, cnt = ctx.saved_tensors
        gseq = (-g.to(torch.float32) / cnt).expand(logits.shape[0]).contiguous()
        return K.logp_gather_bwd(logits, labels, lse, gseq, torch.empty_like(logits)), None


class LlavaQwenForCausalLMBase(nn.Module, LlavaMetaForCausalLM):
    config_class = Qwen2Config
    model_class = LlavaQwenModelBase
    is_moe = False
    is_fp8 = False            # quantize_fp8_ has run: the decoder linears hold e4m3 weights, the model is forward-only

    def __init__(self, config, device="cuda", dtype=torch.bfloat16):
        nn.Module.__init__(self)
        self.config = config
        self.model = self.model_class(config, device, dtype)
        self.vocab_size = config.vocab_size
        if getattr(config, "tie_word_embeddings", False):
            self.lm_head = ParamLinear(self.model.embed_tokens.weight.detach())
            self.lm_head.weight = self.model.embed_tokens.weight            # one shared Parameter, like HF weight tying
        else:
            w = torch.empty(config.vocab_size, config.hidden_size, device=device, dtype=dtype).normal_(0.0, config.initializer_range)
            self.lm_head = ParamLinear(w)
        self.router_aux_loss_coef = getattr(config, "moe", {}).get("router_aux_loss_coef", 0.01) if hasattr(config, "moe") else 0.01
        self.lm_head_grad = None

    # ---- HF-like surface ---------------------------------------------------------------------------
    def get_model(self):
        return self.model

    @property
    def device(self):
        return self.model.embed_tokens.weight.device

    @property
    def dtype(self):
        return self.model.embed_tokens.weight.dtype

    def get_input_embeddings(self):
        return self.model.embed_tokens

    # ---- gradient checkpointing (HF PreTrainedModel surface) -----------------------------------------
    supports_gradient_checkpointing = True
    _input_require_grads = False

    def gradient_checkpointing_enable(self, gradient_checkpointing_kwargs=None):
        """From now on every decoder layer of the language model that has something to differentiate runs as one checkpointed segment
        while the model trains with autograd recording: its activations are recomputed in the backward instead of kept (Qwen2Model._layers,
        kernels.CheckpointFn).  Loss, routing and gradients are those of the run without it.  gradient_checkpointing_kwargs (e.g.
        use_reentrant) is accepted for HF compatibility and has no effect: there is one implementation."""
        self.model.gradient_checkpointing = True

    def gradient_checkpointing_disable(self):
        self.model.gradient_checkpointing = False

    @property
    def is_gradient_checkpointing(self):
        return self.model.gradient_checkpointing

    def enable_input_require_grads(self):
        """The embeddings the decoder receives require grad while autograd records (HF registers a forward hook on the input embeddings
        for this).  A checkpointed layer delivers its parameter gradients without it; the reference's trainers call it with checkpointing."""
        self._input_require_grads = True

    def disable_input_require_grads(self):
        self._input_require_grads = False

    def state_dict_reference_layout(self):
        """state_dict with tied lm_head de-duplicated the way HF saves it."""
        return {k: v for k, v in self.state_dict().items()}

    _FP8_NO_SAVE = ("this model's decoder weights were quantised to e4m3 in place (quantize_fp8_): their bf16 values are gone and there is "
                    "no e4m3 checkpoint format -- save the model before quantising it, or reload the bf16 checkpoint")

    def quantize_fp8_(self):
        """Run the decoder linears (q|k|v, o_proj, gate|up, down_proj of every layer) of this frozen dense model in FP8 from now on: e4m3
        weights with one scale per output channel, activations quantised per token on the fly, fp32 accumulation (csrc/gemm_fp8.cu,
        csrc/quant.cu).  Embeddings, norms, RoPE, attention, the residual stream, lm_head, the CLIP tower and the projector stay bf16.
        In place and one-way: the bf16 decoder weights are released.  Afterwards the model is forward-only -- labels, autograd through
        the decoder and saving raise.  The counterpart of the reference's 8-bit loading of a frozen model (align_train.py:536-553)."""
        if self.is_moe or any(isinstance(l.mlp, MoE) for l in self.model.layers):
            raise ValueError("quantize_fp8_ is for frozen dense models (the teacher); %s has trainable sparse-MoE experts" % type(self).__name__)
        if self.is_fp8:
            raise ValueError("this model is already quantised to e4m3")
        for n, p in self.model.layers.named_parameters():
            if p.requires_grad:
                raise ValueError("quantize_fp8_ needs a frozen decoder: model.layers.%s requires grad (an e4m3 weight cannot be trained)" % n)
        if self.training:
            raise ValueError("quantize_fp8_ needs the model in eval mode (call .eval() first): an FP8 model is forward-only")
        if self.device.type != "cuda":
            raise ValueError("quantize_fp8_ needs the model on the GPU (the weights are quantised by a CUDA kernel); it is on %s" % self.device)
        self.model.quantize_fp8_()
        self.is_fp8 = True
        return self

    def state_dict(self, *args, **kwargs):
        if self.is_fp8:
            raise RuntimeError(self._FP8_NO_SAVE)
        return super().state_dict(*args, **kwargs)

    def train(self, mode=True):
        if mode and self.is_fp8:
            raise RuntimeError("an e4m3-quantised model is forward-only and stays in eval mode")
        return super().train(mode)

    def save_pretrained(self, path, state_dict=None):
        if self.is_fp8:
            raise RuntimeError(self._FP8_NO_SAVE)
        os.makedirs(path, exist_ok=True)
        cfg = self.config
        cfg.architectures = [type(self).__name__]
        cfg.save_pretrained(path)
        sd = state_dict if state_dict is not None else self.state_dict()
        torch.save({k: v.detach().cpu() for k, v in sd.items()}, os.path.join(path, "pytorch_model.bin"))

    @classmethod
    def from_pretrained(cls, path, config=None, device="cuda", torch_dtype=torch.bfloat16, **kw):
        cfg = config if config is not None else cls.config_class.from_pretrained(path)
        model = cls(cfg, device=device, dtype=torch_dtype)
        sd = load_state_dict_files(path)
        if sd:
            tower = model.get_image_tower()
            if tower is not None and not tower.is_loaded and any(k.startswith("model.image_tower.") for k in sd):
                tower.load_model()          # the reference's final pytorch_model.bin carries the tower weights (align_train.py:623-631)
            load_into(model, sd, strict=False)
        return model

    # ---- eval path (SURVEY 8f N4) ---------------------------------------------------------------------
    def generate(self, inputs=None, images=None, **kw):
        """HF-style entry used by the reference's eval scripts (eval/model_vqa_loader.py:119-130); see model/generation.py."""
        from ..generation import generate
        if inputs is None:
            inputs = kw.pop("input_ids")
        return generate(self, inputs, images=images, **kw)

    def resize_token_embeddings(self, new_num_tokens=None):
        """builder.load_pretrained_model calls this with len(tokenizer) (builder.py:588).  HF would cut (or grow) the embedding / lm_head
        matrices; here the storage keeps its checkpoint size and decoding masks the logits beyond the active vocabulary -- the same
        distribution over the same tokens.  Growing past the checkpoint's vocabulary would need new rows and is refused."""
        if new_num_tokens is None:
            return self.model.embed_tokens
        if new_num_tokens > self.model.embed_tokens.weight.shape[0]:
            raise NotImplementedError("resize_token_embeddings beyond the checkpoint vocabulary (%d > %d)" %
                                      (new_num_tokens, self.model.embed_tokens.weight.shape[0]))
        self._active_vocab = int(new_num_tokens)
        return self.model.embed_tokens

    # ---- forward -------------------------------------------------------------------------------------
    def new_kv_cache(self, batch, max_len, share=1, suffix=None):
        """A KVCache for `batch` sequences of up to max_len spliced positions each (prompt incl. image patches + new tokens).  share = n > 1:
        the shared form generate uses for num_return_sequences, `batch` prompts of n sequences each (see KVCache)."""
        return KVCache(self.model, batch, max_len, share=share, suffix=suffix)

    def forward_hidden(self, input_ids=None, attention_mask=None, position_ids=None, inputs_embeds=None, labels=None,
                       images=None, moe_noise=None, tower_features=None, plan=None, cache=None):
        """Splice + decoder.  Returns dict(hidden [B,T',H], labels [B,T'], attention_mask, l_aux list).
        cache: a KVCache -- empty: prefill into it; holding a prefix: input_ids [B,T] is one cached step of T tokens per sequence (no
        splice, as llava_arch.py:162); T > 1 for dense models only."""
        if cache is not None and cache.length > 0 and inputs_embeds is None:
            ids = input_ids.to(self.device)
            inputs_embeds = torch.nn.functional.embedding(ids, self.model.embed_tokens.weight)
            attention_mask = None
        if inputs_embeds is None:
            (_, position_ids, attention_mask, _, inputs_embeds, labels) = self.prepare_inputs_labels_for_multimodal(
                input_ids, position_ids, attention_mask, None, labels, images, tower_features=tower_features, plan=plan)
            if inputs_embeds is None:                       # text-only batch
                ids = input_ids.to(self.device)
                inputs_embeds = torch.nn.functional.embedding(ids, self.model.embed_tokens.weight)
                if attention_mask is not None:
                    attention_mask = attention_mask.to(self.device)
                if labels is not None:
                    labels = labels.to(self.device)
        if self._input_require_grads and torch.is_grad_enabled() and not inputs_embeds.requires_grad:
            inputs_embeds = inputs_embeds.detach().requires_grad_(True)
        hidden, l_auxes, records = self.model(inputs_embeds, attention_mask, position_ids, moe_noise=moe_noise,
                                              training_moe=self.training, cache=cache)
        if hasattr(attention_mask, "mask"):
            attention_mask = attention_mask.mask
        return dict(hidden=hidden, labels=labels, attention_mask=attention_mask, l_aux=l_auxes, records=records)

    def moe_loss_from(self, l_auxes):
        if len(l_auxes) == 0:
            return None
        return self.router_aux_loss_coef * sum(l_auxes)                       # llava_qwen1_5_moe.py:431

    def forward_train_loss(self, input_ids=None, attention_mask=None, labels=None, images=None, moe_noise=None, plan=None):
        """Training-time `.loss` of `forward` without materialising the fp32 logits the reference returns (llava_qwen1_5_moe.py:408-434;
        dense: modeling_qwen2.py:1195-1207): shifted CE (+ moe_loss).  -> (loss, ce.detach(), moe_loss or None)"""
        if self.is_fp8:
            raise RuntimeError("an e4m3-quantised model is forward-only: it has no training loss")
        r = self.forward_hidden(input_ids, attention_mask, None, None, labels, images, moe_noise, plan=plan)
        hidden = r["hidden"]
        B, T, H = hidden.shape
        logits_lp = K.linear(hidden.reshape(B * T, H), self.lm_head.weight, None, self.lm_head_grad, None).view(B, T, -1)
        ce = ShiftedCEFn.apply(logits_lp, r["labels"])
        moe_loss = self.moe_loss_from(r["l_aux"]) if self.is_moe else None
        return (ce if moe_loss is None else ce + moe_loss), ce.detach(), moe_loss

    def forward(self, input_ids=None, attention_mask=None, position_ids=None, past_key_values=None, inputs_embeds=None,
                labels=None, use_cache=None, output_attentions=None, output_hidden_states=None, images=None,
                return_dict=None, moe_noise=None):
        cache = None
        if self.is_fp8 and labels is not None:
            raise RuntimeError("an e4m3-quantised model is forward-only: call it without labels")
        if use_cache and self.model.gradient_checkpointing and self.training and torch.is_grad_enabled():
            warnings.warn("`use_cache=True` is incompatible with gradient checkpointing. Setting `use_cache=False`...")     # modeling_qwen2.py:993-998
            use_cache = False
        if past_key_values is not None or use_cache:
            # KV-cache path (modeling_qwen2.py:1110-1217 with past_key_values; llava_arch.py:162-172 for the cached multimodal step).
            # Without a cache one is allocated for the prompt plus CACHE_ROOM positions; pass new_kv_cache(B, max_len) for longer runs.
            # A padded prompt batch prefills each sequence's real rows; the step's attention_mask is not read (the cache's lengths decide).
            if past_key_values is not None and not isinstance(past_key_values, KVCache):
                raise NotImplementedError("past_key_values must be the KVCache this model returned (or new_kv_cache made)")
            if past_key_values is not None and past_key_values.shared:
                raise NotImplementedError("past_key_values must be a plain KVCache; the shared form is internal to generate")
            if labels is not None:
                raise NotImplementedError("labels with a KV cache: the cached path is for decoding")
            cache = past_key_values
            if cache is None:
                n = inputs_embeds.shape[1] if inputs_embeds is not None else max(self.spliced_length(input_ids, images, attention_mask))
                cache = self.new_kv_cache(input_ids.shape[0] if input_ids is not None else inputs_embeds.shape[0], n + CACHE_ROOM)
        r = self.forward_hidden(input_ids, attention_mask, position_ids, inputs_embeds, labels, images, moe_noise, cache=cache)
        hidden, labels = r["hidden"], r["labels"]
        B, T, H = hidden.shape
        logits_lp = K.linear(hidden.reshape(B * T, H), self.lm_head.weight, None, self.lm_head_grad, None).view(B, T, -1)
        loss = None
        if labels is not None:
            loss = ShiftedCEFn.apply(logits_lp, labels)
        moe_loss = self.moe_loss_from(r["l_aux"]) if self.is_moe else None
        if moe_loss is not None and loss is not None:
            loss = loss + moe_loss                                            # llava_qwen1_5_moe.py:434
        logits = logits_lp.float()                                            # reference returns fp32 logits (:408)
        if self.is_moe:
            return MoECausalLMOutputWithPast(loss=loss, moe_loss=moe_loss, logits=logits, labels=labels,
                                             moe_loss_list=tuple(r["l_aux"]), past_key_values=cache)
        return CausalLMOutputWithPast(loss=loss, logits=logits, labels=labels, past_key_values=cache)

    def spliced_length(self, input_ids, images=None, attention_mask=None):
        """Per sequence, the number of real decoder positions of its prompt: its real tokens (attention_mask, or all of them), every image
        placeholder among them counting as the tower's patch count, cut at tokenizer_model_max_length as the splice cuts.  -> [B] ints."""
        ids = input_ids.cpu()
        real = torch.ones_like(ids, dtype=torch.bool) if attention_mask is None else attention_mask.cpu().bool()
        n = real.sum(1)
        tower = self.get_image_tower()
        if images is not None and tower is not None:
            n = n + ((ids == IMAGE_TOKEN_INDEX) & real).sum(1) * (tower.num_patches - 1)
        cap = getattr(self.config, "tokenizer_model_max_length", None)
        return [min(int(x), cap) if cap is not None else int(x) for x in n]



class LLaVAMoDForCausalLMBase(LlavaQwenForCausalLMBase):
    """Sparse student.  ``initialize_moe_modules`` follows llava_qwen1_5_moe.py:475-560."""
    is_moe = True

    def initialize_moe_modules(self, model_args):
        cfg = self.config
        cfg.moe["moe_enable"] = model_args.moe_enable
        cfg.moe["train_modules"] = model_args.train_modules
        cfg.moe["moe_mode"] = model_args.moe_mode
        cfg.moe["moe_layers_idx"] = model_args.moe_layers_idx
        cfg.moe["ep_size"] = model_args.ep_size
        cfg.moe["top_k_experts"] = model_args.top_k_experts
        cfg.moe["capacity_factor"] = model_args.capacity_factor
        cfg.moe["eval_capacity_factor"] = model_args.eval_capacity_factor
        cfg.moe["min_capacity"] = model_args.min_capacity
        cfg.moe["use_residual"] = model_args.use_residual
        cfg.moe["router_aux_loss_coef"] = self.router_aux_loss_coef = model_args.router_aux_loss_coef
        tm = cfg.moe["train_modules"]
        if tm is not None and len(tm) > 0:                                    # freeze by substring BEFORE wrapping (:501-506)
            for n, p in self.named_parameters():
                if not any(name in n for name in tm):
                    p.requires_grad = False
        L = cfg.num_hidden_layers
        idx = model_args.moe_layers_idx
        if idx is not None:
            model_args.moe_mode = "custom"
            assert len(idx) <= L and max(idx) < L and min(idx) >= 0
        else:
            mode = model_args.moe_mode
            if mode == "first_half":
                idx = list(range(0, L // 2))
            elif mode == "second_half":
                idx = list(range(L // 2, L))
            elif mode == "sparse":
                idx = list(range(L))[::2]
            elif mode == "dense":
                idx = list(range(L))
            else:
                raise NotImplementedError(f'Only support ["first_half", "second_half", "sparse", "dense"], but found {mode}')
        cfg.moe["moe_layers_idx"] = idx
        ne = list(model_args.num_experts)
        if len(ne) == 1:
            cfg.moe["num_experts"] = ne * len(idx)
        assert len(cfg.moe["num_experts"]) == len(idx)
        self._wrap_moe(cfg.moe["num_experts"], idx, model_args.ep_size, model_args.top_k_experts, model_args.capacity_factor,
                       model_args.eval_capacity_factor, model_args.min_capacity, model_args.use_residual)

    def _wrap_moe(self, num_experts, idx, ep_size, k, cf, ecf, min_cap, use_residual):
        for E, li in zip(num_experts, idx):
            dense = self.model.layers[li].mlp
            moe = MoE(self.config, expert=dense, num_experts=E, ep_size=ep_size, k=k, capacity_factor=cf,
                      eval_capacity_factor=ecf, min_capacity=min_cap, use_residual=use_residual)
            for e in moe.deepspeed_moe.experts.deepspeed_experts:             # same sanity check as the reference (:547-550)
                assert torch.equal(e.gate_proj.weight, dense.gate_proj.weight) and torch.equal(e.down_proj.weight, dense.down_proj.weight)
            if use_residual:                                                  # MoE(use_residual=True) keeps the dense module itself
                assert moe.mlp is dense
            self.model.layers[li].mlp = moe


class LLaVAMoDFineTuneBase(LLaVAMoDForCausalLMBase):
    """Builds the MoE layers from a saved ``config.moe`` so a sparse checkpoint loads directly (:564-626)."""

    def __init__(self, config, device="cuda", dtype=torch.bfloat16):
        super().__init__(config, device, dtype)
        m = config.moe
        self.router_aux_loss_coef = m["router_aux_loss_coef"]
        self._wrap_moe(m["num_experts"], m["moe_layers_idx"], m["ep_size"], m["top_k_experts"], m["capacity_factor"],
                       m["eval_capacity_factor"], m["min_capacity"], m["use_residual"])

    def initialize_moe_modules(self, model_args):
        self.config.moe["train_modules"] = model_args.train_modules
        tm = self.config.moe["train_modules"]
        if tm is not None and len(tm) > 0:
            for n, p in self.named_parameters():
                p.requires_grad = any(name in n for name in tm)


def make_moe_config(base_name, model_type_name):
    class _Cfg(Qwen2Config):
        model_type = model_type_name

        def __init__(self, moe_enable=True, moe_mode="sparse", moe_layers_idx=None, ep_size=1, top_k_experts=2,
                     capacity_factor=1.0, eval_capacity_factor=1.0, min_capacity=4, use_residual=False,
                     router_aux_loss_coef=0.01, **kwargs):
            moe = kwargs.pop("moe", None)
            lora = kwargs.pop("lora", {})
            self.moe = moe if moe is not None else dict(
                moe_enable=moe_enable, moe_mode=moe_mode, moe_layers_idx=moe_layers_idx, ep_size=ep_size,
                top_k_experts=top_k_experts, capacity_factor=capacity_factor, eval_capacity_factor=eval_capacity_factor,
                min_capacity=min_capacity, use_residual=use_residual, router_aux_loss_coef=router_aux_loss_coef,
                train_modules=[])
            self.lora = lora
            super().__init__(**kwargs)

    _Cfg.__name__ = base_name
    _Cfg.__qualname__ = base_name
    return _Cfg
