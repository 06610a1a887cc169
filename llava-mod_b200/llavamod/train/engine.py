"""Training state for the data-parallel distillation step: flat parameter / gradient / optimizer arenas in HBM,
fused AdamW, gradient all-reduce over NCCL.

Replaces what the reference gets from HF Trainer + accelerate + DeepSpeed ZeRO-2 with CPU-offloaded Adam
(llavamod/train/align_trainer.py:326-453, llavamod/config/dpconfig/zero2_offload.json): on an 80 GB H100 nothing is
sharded or offloaded -- the trainable student parameters (0.5B-4E: 521 M) keep bf16 model copy + fp32 master + two fp32
moments + a bf16 gradient buffer resident (16 B/param = 8.3 GB), the frozen teacher is replicated, and the only
collective of a step is ONE all-reduce over the flat gradient buffer (student grads only; SURVEY.md section 8e).

Layout: every trainable *storage unit* (a fused q|k|v / gate|up buffer, an [E,2I,H] expert stack, or a plain parameter)
is packed into one contiguous bf16 arena (fp32 units -- the router ``wg`` -- into a second, tiny fp32 arena), each unit
aligned to 256 bytes.  The ``nn.Parameter``s the reference exposes are re-pointed to views of the arena, their ``.grad``
to views of the gradient arena, so the wgrad GEMMs accumulate straight into the buffer NCCL reduces.
"""
import math

import torch
import torch.distributed as dist

from .. import kernels as K
from ..model.language_model.qwen2_core import Experts, Qwen2Attention, Qwen2MLP

ALIGN = 128  # elements


def _units(model):
    """Yields (storage_tensor, [member Parameters]) -- fused buffers first, then every remaining parameter."""
    seen = set()
    out = []

    def add(storage, members):
        members = [m for m in members if m is not None]
        for m in members:
            seen.add(id(m))
        out.append((storage, members))

    for mod in model.modules():
        if isinstance(mod, Qwen2Attention):
            add(mod.qkv_weight, [mod.q_proj.weight, mod.k_proj.weight, mod.v_proj.weight])
            add(mod.qkv_bias, [mod.q_proj.bias, mod.k_proj.bias, mod.v_proj.bias])
        elif isinstance(mod, Experts):
            add(mod.gu_weight, [p for e in mod.deepspeed_experts for p in (e.gate_proj.weight, e.up_proj.weight)])
            add(mod.dn_weight, [e.down_proj.weight for e in mod.deepspeed_experts])
    for mod in model.modules():
        if isinstance(mod, Qwen2MLP) and id(mod.gate_proj.weight) not in seen:
            add(mod.gu_weight, [mod.gate_proj.weight, mod.up_proj.weight])
    for p in model.parameters():
        if id(p) not in seen:
            add(p, [p])
    return out


def param_group_of(name, in_layernorm, projector_lr_set):
    """The reference's optimizer groups (align_trainer.py:341-398, same in dpo_trainer.py:348 / llava_trainer.py:167):
    decay = every parameter that is not inside an nn.LayerNorm (Qwen2RMSNorm is NOT in ALL_LAYERNORM_LAYERS, so RMSNorm weights decay)
    and whose name does not contain "bias"; with --mm_projector_lr the names containing "mm_projector" form their own two groups.
    -> (is_projector_group, no_decay)"""
    no_decay = in_layernorm or ("bias" in name)
    return (bool(projector_lr_set and "mm_projector" in name), bool(no_decay))


class TrainState:
    def __init__(self, model, lr=2e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, max_grad_norm=1.0,
                 process_group=None, mm_projector_lr=None):
        self.model = model
        self.lr, self.betas, self.eps, self.wd, self.max_grad_norm = lr, betas, eps, weight_decay, max_grad_norm
        self.mm_projector_lr = mm_projector_lr
        self.pg = process_group
        self.world = dist.get_world_size(process_group) if dist.is_available() and dist.is_initialized() else 1
        self.step_count = 0
        dev = next(model.parameters()).device
        # every trainable parameter must have a kernel that writes its gradient view: language-model linears / biases / norms / embeddings,
        # lm_head, router wg, experts and the projector do; the CLIP tower is forward-only (frozen in every recipe of the reference)
        orphans = [n for n, p in model.named_parameters() if p.requires_grad and "image_tower" in n]
        if orphans:
            raise NotImplementedError("trainable vision-tower parameters (%s ...): the tower's backward is not built -- the reference's "
                                      "recipes keep it frozen" % orphans[0])
        names = {id(p_): n for n, p_ in model.named_parameters()}
        ln_params = {id(p_) for mod in model.modules() if isinstance(mod, torch.nn.LayerNorm) or getattr(mod, "is_layernorm", False)
                     for p_ in mod.parameters(recurse=False)}
        u16, u32 = [], []
        for storage, members in _units(model):
            rg = [m.requires_grad for m in members]
            if not any(rg):
                continue
            if not all(rg):
                raise NotImplementedError("a fused buffer with mixed frozen/trainable members (e.g. only gate_proj of gate|up) "
                                          "is not supported; train or freeze q/k/v and gate/up together")
            keys = {param_group_of(names.get(id(m), ""), id(m) in ln_params, mm_projector_lr is not None) for m in members}
            if len(keys) != 1:
                raise NotImplementedError("a fused buffer whose members fall into different optimizer groups")
            (u32 if storage.dtype == torch.float32 else u16).append((storage, members, keys.pop()))
        # units of one optimizer group (decay / no-decay x projector-lr) are laid out contiguously, so a group is ONE slice of the arenas
        u16.sort(key=lambda u: u[2])
        u32.sort(key=lambda u: u[2])
        self.segments = {}
        self.n16 = self._pack(u16, torch.bfloat16, dev, "16")
        self.n32 = self._pack(u32, torch.float32, dev, "32")
        self.master = self.w16.float() if self.n16 else None
        self.m16 = torch.zeros_like(self.master) if self.n16 else None
        self.v16 = torch.zeros_like(self.master) if self.n16 else None
        self.m32 = torch.zeros_like(self.w32) if self.n32 else None
        self.v32 = torch.zeros_like(self.w32) if self.n32 else None
        self.gnorm_sq = torch.zeros(1, dtype=torch.float32, device=dev)
        self.grads_reduced = False           # set by the trainer when the all-reduce already ran inside the last micro-batch's CUDA graph
        gv = {}
        for storage, g in self._views:
            gv[id(storage)] = g
        # hand the gradient views to the modules whose forward issues the wgrad GEMMs
        core = model.get_model() if hasattr(model, "get_model") else model
        core.grad_views = gv
        if getattr(core, "mm_projector", None) is not None:
            core.mm_projector.grad_views = gv
        if hasattr(model, "lm_head") and id(model.lm_head.weight) in gv:
            model.lm_head_grad = gv[id(model.lm_head.weight)]
        self.num_trainable = self.n16 + self.n32

    def _pack(self, units, dtype, dev, tag):
        off, plan, segs = 0, [], []
        for storage, members, key in units:
            plan.append((storage, members, off))
            nxt = off + (storage.numel() + ALIGN - 1) // ALIGN * ALIGN
            if segs and segs[-1][0] == key:
                segs[-1][2] = nxt
            else:
                segs.append([key, off, nxt])
            off = nxt
        self.segments[tag] = [(k, a, b) for k, a, b in segs]
        w = torch.zeros(max(off, 1), dtype=dtype, device=dev)
        g = torch.zeros(max(off, 1), dtype=dtype, device=dev)
        views = getattr(self, "_views", [])
        for storage, members, o in plan:
            n = storage.numel()
            base_ptr = storage.data_ptr()
            rel = [((m.data_ptr() - base_ptr) // storage.element_size(), m.shape) for m in members]
            new = w[o:o + n].view(storage.shape)
            new.copy_(storage.detach())
            gview = g[o:o + n].view(storage.shape)
            is_param = any(m is storage for m in members)
            if is_param:
                storage.data = new
                storage.grad = gview
            else:
                storage.data = new                                   # plain fused tensor re-pointed in place (id preserved)
                for m, (r, shp) in zip(members, rel):
                    k = m.numel()
                    m.data = w[o + r:o + r + k].view(shp)
                    m.grad = g[o + r:o + r + k].view(shp)
            views.append((storage, gview))
        self._views = views
        setattr(self, "w" + tag, w)
        setattr(self, "g" + tag, g)
        return off

    # ---------------------------------------------------------------------------------------------
    def zero_grad(self):
        self.grads_reduced = False
        if self.n16:
            self.g16.zero_()
        if self.n32:
            self.g32.zero_()

    def refresh_master(self):
        """fp32 master copy <- current bf16 weights (after a checkpoint / adaptor was loaded into the model)."""
        if self.n16:
            self.master.copy_(self.w16.float())

    def allreduce_grads(self):
        """The one exchange step of data parallelism: sum the flat student gradient buffers over NVLink (NCCL)."""
        if self.world > 1:
            if self.n16:
                dist.all_reduce(self.g16, group=self.pg)
            if self.n32:
                dist.all_reduce(self.g32, group=self.pg)

    def step(self, lr=None, grad_scale=1.0):
        """AdamW step on the accumulated gradients.  ``grad_scale`` folds 1/(accumulation * world) into the update
        (HF Trainer divides the loss instead; same arithmetic up to bf16 rounding of the scaled loss)."""
        lr = self.lr if lr is None else lr
        self.step_count += 1
        if not self.grads_reduced:
            self.allreduce_grads()
        self.grads_reduced = False
        use_clip = self.max_grad_norm is not None and self.max_grad_norm > 0
        if use_clip:
            self.gnorm_sq.zero_()
            if self.n16:
                K.sumsq_(self.g16, self.gnorm_sq)
            if self.n32:
                K.sumsq_(self.g32, self.gnorm_sq)
        gn = self.gnorm_sq if use_clip else None
        mx = float(self.max_grad_norm) if use_clip else 0.0
        # one fused AdamW launch per optimizer group (a contiguous slice of the arenas); the clip coefficient is global (one norm over
        # every group, as torch.nn.utils.clip_grad_norm_ over all parameters), the projector group follows the same schedule scaled to its
        # own base LR (HF schedulers multiply each group's initial lr by the same lambda)
        for (is_proj, no_decay), a, b in (self.segments["16"] if self.n16 else []):
            g_lr = lr * (self.mm_projector_lr / self.lr) if (is_proj and self.lr) else lr
            K.adamw_(self.master[a:b], self.m16[a:b], self.v16[a:b], self.g16[a:b], self.w16[a:b], g_lr, self.betas[0], self.betas[1], self.eps,
                     0.0 if no_decay else self.wd, self.step_count, gn, mx, grad_scale)
        for (is_proj, no_decay), a, b in (self.segments["32"] if self.n32 else []):
            g_lr = lr * (self.mm_projector_lr / self.lr) if (is_proj and self.lr) else lr
            K.adamw_(self.w32[a:b], self.m32[a:b], self.v32[a:b], self.g32[a:b], None, g_lr, self.betas[0], self.betas[1], self.eps,
                     0.0 if no_decay else self.wd, self.step_count, gn, mx, grad_scale)

    def grad_norm(self, grad_scale=1.0):
        return float(torch.sqrt(self.gnorm_sq)[0]) * grad_scale


def warmup_steps_of(total, warmup_ratio=0.0, warmup_steps=0):
    """HF TrainingArguments.get_warmup_steps: --warmup_steps wins when > 0, else ceil(ratio * total)."""
    return int(warmup_steps) if warmup_steps and warmup_steps > 0 else math.ceil(warmup_ratio * total)


def cosine_lr(step, total, base_lr, warmup_ratio=0.03, warmup_steps=0):
    """transformers.get_cosine_schedule_with_warmup with HF's warm-up step count; ``step`` = number of completed optimizer steps."""
    warm = warmup_steps_of(total, warmup_ratio, warmup_steps)
    if step < warm:
        return base_lr * step / max(1, warm)
    prog = (step - warm) / max(1, total - warm)
    return base_lr * max(0.0, 0.5 * (1.0 + math.cos(math.pi * prog)))
