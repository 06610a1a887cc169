"""Minimal trainer loop with the HF ``Trainer`` surface the reference's trainers rely on
(``compute_loss`` / ``training_step`` / ``create_optimizer`` / ``log`` / ``save_model`` / ``_save_checkpoint``).

The reference subclasses ``transformers.Trainer`` and runs under accelerate + DeepSpeed ZeRO-2
(llavamod/train/align_trainer.py:180-309).  Here one process drives one GPU; gradient accumulation is local, the
optimizer is the fused AdamW of ``engine.TrainState`` and the only collective is the student-gradient all-reduce.
"""
import contextlib
import glob
import json
import os
import re
import time
from collections import defaultdict
from typing import Dict, Literal, Optional

import torch
import torch.distributed as dist

from ..model.utils import create_reference_model, disable_dropout_in_model
from .engine import TrainState, cosine_lr, optim_bits_of, warmup_steps_of


def _with_lookahead(iterable):
    """(item, next_item) pairs; next_item is None for the last element."""
    it = iter(iterable)
    try:
        cur = next(it)
    except StopIteration:
        return
    for nxt in it:
        yield cur, nxt
        cur = nxt
    yield cur, None


class _Wrapped:
    """Gives a bare module the ``.module`` attribute the reference dereferences on the DeepSpeed-wrapped teacher
    (align_trainer.py:305,309); the build accepts wrapped and bare teachers (SURVEY.md Appendix B)."""

    def __init__(self, module):
        self.module = module

    def __call__(self, *a, **kw):
        return self.module(*a, **kw)

    def __getattr__(self, k):
        return getattr(self.module, k)


def same_frozen_tower(a, b):
    ta, tb = a.get_image_tower(), b.get_image_tower()
    if ta is None or tb is None or not (ta.is_loaded and tb.is_loaded):
        return False
    sa, sb = ta.state_dict(), tb.state_dict()
    if sa.keys() != sb.keys() or any(p.requires_grad for p in ta.parameters()) or any(p.requires_grad for p in tb.parameters()):
        return False
    return ta.select_layer == tb.select_layer and all(torch.equal(sa[k], sb[k]) for k in sa)


def quantize_ref_fp8(ref, ref_fp8):
    """--ref_fp8 / LLAVAMOD_REF_FP8=1: the frozen teacher's decoder linears run in FP8 (e4m3) from here on (quantize_fp8_ of the dense
    causal-LM classes).  Opt-in: it changes the teacher's logits.  The quantisers and the e4m3 GEMM are plain stream-ordered launches, so
    the teacher keeps its side stream, its one-micro-batch lead and its place in the captured step."""
    if (ref_fp8 or bool(int(os.environ.get("LLAVAMOD_REF_FP8", "0")))) and not ref.is_fp8:
        ref.quantize_fp8_()


def image_count_shape(images):
    """(number of images, shape of one image) of a batch's images: one tensor [n, ...] or a list of n tensors."""
    if torch.is_tensor(images):
        return images.shape[0], tuple(images.shape[1:])
    return len(images), tuple(images[0].shape)


class TrainerState:
    def __init__(self):
        self.global_step = 0
        self.epoch = 0.0
        self.log_history = []


class BaseTrainer:
    def __init__(self, model=None, args=None, data_collator=None, train_dataset=None, eval_dataset=None, tokenizer=None,
                 model_init=None, compute_metrics=None, callbacks=None, optimizers=(None, None),
                 preprocess_logits_for_metrics=None):
        self.model = model
        self.args = args
        self.data_collator = data_collator
        self.train_dataset = train_dataset
        self.eval_dataset = eval_dataset
        self.tokenizer = tokenizer
        self.state = TrainerState()
        self.optimizer = None
        self.is_deepspeed_enabled = False
        self.world_size = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank() if self.world_size > 1 else 0
        self._accum = 0
        self._total_steps = None
        # CUDA graphs: the forward+backward of a micro-batch is captured once per input signature and replayed, which
        # removes the per-launch host cost (~1000 launches per micro-batch) -- "CUDA streams and graphs instead of a tracing compiler"
        self.use_cuda_graphs = bool(int(os.environ.get("LLAVAMOD_CUDA_GRAPHS", "1")))
        self._graphs = {}                    # signature -> captured graph (LRU, bounded) ; or {"warm": n} while still eager
        # real data (per_device_train_batch_size 1, variable lengths) produces a new signature per distinct length: every captured graph
        # pins its activations, so the cache is bounded (least-recently-used graph dropped) and all graphs share ONE memory pool
        self.max_graphs = int(os.environ.get("LLAVAMOD_MAX_GRAPHS", "6"))
        self._graph_pool = None
        self._suppress_store = False
        self.graph_replayed_launches = 0     # liblmod kernels executed through graph replays (not seen by the host-side counter)
        self._stored_metrics = defaultdict(lambda: defaultdict(list))
        if getattr(args, "gradient_checkpointing", False) and hasattr(model, "enable_input_require_grads"):
            model.enable_input_require_grads()         # align_trainer.py:243-246, dpo_trainer.py:243-246

    # ---- frozen teacher (AlignTrainer, DPOTrainer) ---------------------------------------------------------------
    def _init_teacher(self, ref_model, disable_dropout, ref_fp8):
        """Builds (a deep copy of the student) or takes the reference model, wraps a bare module in ``_Wrapped``, puts it in eval mode
        and freezes it; then --ref_fp8, whether the two models share one frozen CLIP tower, and the teacher's side stream."""
        ref = ref_model if ref_model else create_reference_model(self.model)
        self.ref_model = ref if hasattr(ref, "module") else _Wrapped(ref)
        if disable_dropout:
            disable_dropout_in_model(self.model)
            disable_dropout_in_model(self.ref_model.module)
        self.ref_model.module.eval()
        for p in self.ref_model.module.parameters():
            p.requires_grad = False
        self.share_tower = same_frozen_tower(self.model, self.ref_model.module)
        quantize_ref_fp8(self.ref_model.module, ref_fp8)
        self.overlap_teacher = bool(int(os.environ.get("LLAVAMOD_OVERLAP_TEACHER", "1"))) and next(self.model.parameters()).is_cuda
        self._teacher_stream = torch.cuda.Stream() if self.overlap_teacher else None

    @contextlib.contextmanager
    def _teacher_side(self):
        """Runs the block without grad on the teacher's side stream, after the work already queued on the main stream (on the main
        stream when the overlap is off).  The main stream waits for it in ``_join_teacher``."""
        main = torch.cuda.current_stream()
        side = self._teacher_stream if self.overlap_teacher else None
        if side is not None:
            side.wait_stream(main)
        with torch.no_grad(), torch.cuda.stream(side if side is not None else main):
            yield

    def _join_teacher(self, *tensors):
        """With the overlap on, the main stream waits for the side stream and ``tensors``, allocated there, are marked as used by the
        main stream."""
        if self.overlap_teacher:
            main = torch.cuda.current_stream()
            main.wait_stream(self._teacher_stream)
            for t in tensors:
                t.record_stream(main)

    # ---- optimizer ---------------------------------------------------------------------------------------
    def create_optimizer(self):
        """Fused AdamW over the flat arenas with the reference's parameter groups (align_trainer.py:326-434): decay / no-decay (names
        containing "bias", nn.LayerNorm parameters) and, with --mm_projector_lr, the projector's own LR groups -- each a contiguous slice
        of the arenas (engine.TrainState).  DeepSpeed's split into MoE expert groups changes no hyper-parameter and is not mirrored.
        ``--optim adamw_bnb_8bit`` / ``adamw_8bit`` (HF's bitsandbytes 8-bit AdamW, align_trainer.py:409-429) keep the moments of the bf16
        arena as 8-bit block-wise codes; every other value keeps fp32 moments."""
        if self.optimizer is None:
            a = self.args
            self.optimizer = TrainState(self.model, lr=a.learning_rate, betas=(a.adam_beta1, a.adam_beta2), eps=a.adam_epsilon,
                                        weight_decay=a.weight_decay, max_grad_norm=a.max_grad_norm,
                                        mm_projector_lr=getattr(a, "mm_projector_lr", None),
                                        optim_bits=optim_bits_of(getattr(a, "optim", "adamw_torch")))
        return self.optimizer

    def current_lr(self):
        a = self.args
        if self._total_steps is None or a.lr_scheduler_type == "constant":
            return a.learning_rate
        wsteps = getattr(a, "warmup_steps", 0) or 0
        if a.lr_scheduler_type == "cosine":
            return cosine_lr(self.state.global_step, self._total_steps, a.learning_rate, a.warmup_ratio, wsteps)
        if a.lr_scheduler_type == "linear":
            warm = warmup_steps_of(self._total_steps, a.warmup_ratio, wsteps)
            s = self.state.global_step
            if s < warm:
                return a.learning_rate * s / max(1, warm)
            return a.learning_rate * max(0.0, (self._total_steps - s) / max(1, self._total_steps - warm))
        raise NotImplementedError("lr_scheduler_type %r" % a.lr_scheduler_type)

    # ---- one micro-batch -----------------------------------------------------------------------------------
    def compute_loss(self, model, inputs, return_outputs=False):
        raise NotImplementedError

    def training_step(self, model, inputs, next_inputs=None):
        """forward + backward of one micro-batch; the optimizer step happens every ``gradient_accumulation_steps`` calls.
        Gradients are accumulated UNSCALED; 1/(accum*world) is folded into the AdamW kernel.
        ``next_inputs`` (optional look-ahead, the batch the NEXT call will receive) lets the trainer run the frozen teacher one
        micro-batch ahead, overlapped with this micro-batch's student forward/backward."""
        opt = self.create_optimizer()
        model.train()
        if self._accum == 0:
            opt.zero_grad()
        from ..kernels import nvtx
        loss = None
        with nvtx("micro_batch"):
            if self.use_cuda_graphs and hasattr(self, "_graph_signature"):
                loss = self._graphed_micro_batch(model, inputs, next_inputs)
            if loss is None:
                with nvtx("forward+loss"):
                    loss = self.compute_loss(model, inputs)
                with nvtx("backward"):
                    loss.backward()
        self._accum += 1
        if self._accum == self.args.gradient_accumulation_steps:
            with nvtx("allreduce+clip+adamw"):
                opt.step(lr=self.current_lr(), grad_scale=1.0 / (self._accum * self.world_size))
            self._accum = 0
            self.state.global_step += 1
        return loss.detach()

    # ---- CUDA-graph replay of one micro-batch ----------------------------------------------------------------------
    def _graphed_micro_batch(self, model, inputs, next_inputs=None):
        """Returns the loss tensor (detached, static buffer clone) or None when this batch must run eagerly.
        Subclasses provide ``_graph_signature(inputs, next_inputs)`` (hashable, or None = not capturable) and may override
        ``_graph_static_inputs``."""
        sig = self._graph_signature(inputs, next_inputs)
        if sig is None:
            return None
        pipelined = sig[-1] == "pipelined"
        ent = self._graphs.pop(sig, None)                # re-inserted below: dict order = recency
        if ent is None:
            ent = {"warm": 0}
            if len(self._graphs) > 4096:                 # rarely seen signatures never reach capture; forget the oldest counters
                for k in [k for k, v in self._graphs.items() if "graph" not in v][:2048]:
                    del self._graphs[k]
        self._graphs[sig] = ent
        if "graph" not in ent:
            ent["warm"] += 1
            if ent["warm"] <= 2:                         # eager warm-up (lazy init, autotune, workspace allocation)
                return None
            captured = [k for k, v in self._graphs.items() if "graph" in v]
            while len(captured) >= max(1, self.max_graphs):      # drop the least recently used graph with its static buffers
                self._graphs.pop(captured.pop(0)).clear()
            static = self._graph_static_inputs(inputs, None, next_inputs, pipelined)
            torch.cuda.synchronize()
            from .. import _C
            g = torch.cuda.CUDAGraph()
            if self._graph_pool is None:
                self._graph_pool = torch.cuda.graph_pool_handle()
            self._suppress_store = True
            n0 = _C.launch_count()
            try:
                with torch.cuda.graph(g, pool=self._graph_pool):
                    loss, outputs = self.compute_loss(model, static, return_outputs=True)
                    loss.backward()
                    if hasattr(self, "_graph_epilogue"):
                        self._graph_epilogue(static)
            finally:
                self._suppress_store = False
            ent.update(graph=g, static=static, loss=loss.detach(), outputs={k: v for k, v in outputs.items()},
                       launches=_C.launch_count() - n0)
            # the capture pass does not execute: fall through to a replay for this very batch
        self._graph_static_inputs(inputs, ent["static"], next_inputs, pipelined)
        ent["graph"].replay()
        self.graph_replayed_launches += ent["launches"]
        self.store_metrics({k: (v.clone() if hasattr(v, "clone") else v) for k, v in ent["outputs"].items()}, train_eval="train")
        return ent["loss"].clone()

    # static device inputs of a captured micro-batch: images + the precomputed splice plans (ids / labels / masks stay host-side: the
    # plans already encode them).  _static_keys are carried as they are, _static_plans are the splice plans' keys.
    _static_keys = ("input_ids", "labels", "attention_mask")
    _static_plans = ("splice_plan",)

    def _graph_static_inputs(self, inputs, static, next_inputs=None, pipelined=False):
        """Allocates (static None) and refills the static inputs of a captured micro-batch."""
        if static is None:
            static = self._new_static(inputs)
        self._fill_static(static, inputs)
        return static

    def _fill_static(self, static, inputs):
        images = inputs["images"]
        if torch.is_tensor(images):
            static["images"].copy_(images, non_blocking=True)
        else:
            for i, im in enumerate(images):
                static["images"][i].copy_(im, non_blocking=True)
        for name in self._static_plans:
            for k, v in inputs[name].items():
                if torch.is_tensor(v):
                    static[name][k].copy_(v, non_blocking=True)
        if static.get("moe_noise") is not None:           # explicit router noise (parity runs): static buffers like every other device input
            for dst, src in zip(static["moe_noise"], inputs["moe_noise"]):
                dst.copy_(src, non_blocking=True)

    def _new_static(self, inputs):
        dev = self.model.device
        n, ish = image_count_shape(inputs["images"])
        noise = inputs.get("moe_noise")
        static = {k: inputs.get(k) for k in self._static_keys}
        static["moe_noise"] = [torch.empty(tuple(t.shape), dtype=torch.float32, device=dev) for t in noise] if noise is not None else None
        static["images"] = torch.empty((n,) + ish, dtype=self.model.dtype, device=dev)
        for name in self._static_plans:
            static[name] = {k: (torch.empty_like(v) if torch.is_tensor(v) else v) for k, v in inputs[name].items()}
        return static

    # ---- loop ------------------------------------------------------------------------------------------------
    def get_train_dataloader(self):
        from torch.utils.data import DataLoader, DistributedSampler
        if getattr(self.args, "group_by_modality_length", False) and hasattr(self.train_dataset, "modality_lengths"):
            # reference: _get_train_sampler (align_trainer.py:311-322) -- global length-grouped order, then per-rank batches
            from .sampler import LengthGroupedSampler, RankShard
            a = self.args
            grouped = LengthGroupedSampler(a.per_device_train_batch_size, world_size=self.world_size * a.gradient_accumulation_steps,
                                           lengths=self.train_dataset.modality_lengths, group_by_modality=True)
            sampler = RankShard(grouped, a.per_device_train_batch_size, self.rank, self.world_size)
            return DataLoader(self.train_dataset, batch_size=a.per_device_train_batch_size, sampler=sampler, collate_fn=self.data_collator,
                              num_workers=a.dataloader_num_workers, pin_memory=True, drop_last=True)
        if self.world_size > 1:
            sampler = DistributedSampler(self.train_dataset, shuffle=True, seed=self.args.seed)
        else:
            from .sampler import EpochSeededRandomSampler       # order is a function of (seed, epoch): a resumed run sees the same batches
            sampler = EpochSeededRandomSampler(self.train_dataset, seed=self.args.seed)
        return DataLoader(self.train_dataset, batch_size=self.args.per_device_train_batch_size, sampler=sampler,
                          collate_fn=self.data_collator, num_workers=self.args.dataloader_num_workers, pin_memory=True, drop_last=True)

    def _grad_ckpt_key(self):
        """Part of every _graph_signature: a graph captured with checkpointing on holds the recompute, one captured with it off does not."""
        return ("grad_ckpt", bool(getattr(self.model, "is_gradient_checkpointing", False)))

    def train(self, resume_from_checkpoint=None):
        a = self.args
        if getattr(a, "gradient_checkpointing", False):  # transformers Trainer._inner_training_loop
            self.model.gradient_checkpointing_enable(gradient_checkpointing_kwargs=getattr(a, "gradient_checkpointing_kwargs", None))
        dl = self.get_train_dataloader()
        steps_per_epoch = max(1, len(dl) // a.gradient_accumulation_steps)
        self._total_steps = a.max_steps if a.max_steps > 0 else int(steps_per_epoch * a.num_train_epochs)
        rng = None
        if resume_from_checkpoint:
            rng = self._load_checkpoint(resume_from_checkpoint)
        # resume where the interrupted run stopped (HF Trainer: epochs_trained / skip_first_batches): same epoch, the micro-batches the
        # finished optimizer steps consumed are skipped, and the RNG streams (router Gumbel noise, samplers) continue from the saved state
        epoch = self.state.global_step // steps_per_epoch
        skip = (self.state.global_step % steps_per_epoch) * a.gradient_accumulation_steps
        t0 = time.time()
        tr_loss, n_loss = 0.0, 0
        done = self.state.global_step >= self._total_steps
        while not done:
            if hasattr(dl.sampler, "set_epoch"):
                dl.sampler.set_epoch(epoch)
            it = iter(dl)
            for _ in range(skip):
                next(it, None)
            skip = 0
            if rng is not None:                          # after the skipped batches were drawn: the loop below continues the saved streams
                self._restore_rng(rng)
                rng = None
            for batch, nxt in _with_lookahead(it):
                before = self.state.global_step
                loss = self.training_step(self.model, batch, nxt)     # look-ahead: the frozen teacher runs one micro-batch ahead
                tr_loss += float(loss); n_loss += 1
                if self.state.global_step != before:
                    s = self.state.global_step
                    if a.logging_steps and s % a.logging_steps == 0:
                        self.log({"loss": tr_loss / max(1, n_loss), "learning_rate": self.current_lr(), "epoch": s / steps_per_epoch})
                        tr_loss, n_loss = 0.0, 0
                    if a.save_strategy == "steps" and a.save_steps and s % a.save_steps == 0:
                        self._save_checkpoint(self.model, None)
                    if s >= self._total_steps:
                        done = True
                        break
            epoch += 1
        return {"train_runtime": time.time() - t0, "global_step": self.state.global_step}

    # ---- logging / saving --------------------------------------------------------------------------------------
    def store_metrics(self, metrics: Dict[str, float], train_eval: Literal["train", "eval"] = "train") -> None:
        if self._suppress_store:          # graph capture: the static output tensors are cloned after every replay instead
            return
        for key, value in metrics.items():
            self._stored_metrics[train_eval][key].append(value)

    def log(self, logs: Dict[str, float]) -> None:
        """store_metrics/log of the reference (align_trainer.py:596-614): the means of the stored metrics join the logged values."""
        train_eval = "train" if "loss" in logs else "eval"
        for key, metrics in self._stored_metrics[train_eval].items():
            logs[key] = torch.stack([torch.as_tensor(m, dtype=torch.float32).detach().cpu() for m in metrics]).mean().item()
        del self._stored_metrics[train_eval]
        logs = dict(logs)
        logs["step"] = self.state.global_step
        self.state.log_history.append(logs)
        if self.rank == 0:
            os.makedirs(self.args.output_dir, exist_ok=True)
            with open(os.path.join(self.args.output_dir, "trainer_log.jsonl"), "a") as f:
                f.write(json.dumps(logs) + "\n")
            print(logs, flush=True)

    def _get_output_dir(self, trial=None):
        return self.args.output_dir

    def save_model(self, output_dir=None):
        self._save(output_dir or self.args.output_dir)

    def _save(self, output_dir=None, state_dict=None):
        if self.rank == 0:
            self.model.save_pretrained(output_dir or self.args.output_dir, state_dict=state_dict)

    def _save_checkpoint(self, model, trial, metrics=None):
        """checkpoint-N/: HF-layout model + optimizer arenas + trainer state (reference: HF Trainer + DeepSpeed engine
        checkpoints under each checkpoint-N/, align_train.py:601-604 auto-resume)."""
        d = os.path.join(self._get_output_dir(trial), f"checkpoint-{self.state.global_step}")
        if self.rank == 0:
            self.model.save_pretrained(d)
            opt = self.optimizer
            if opt is not None and opt.optim_bits == 8:
                torch.save({"optim": "adamw_8bit", "master": opt.master, "m8": opt.m8, "v8": opt.v8, "absmax": opt.absmax,
                            "w32": getattr(opt, "w32", None), "m32": opt.m32, "v32": opt.v32, "step_count": opt.step_count},
                           os.path.join(d, "optimizer.pt"))
            elif opt is not None:
                torch.save({"master": opt.master, "m16": opt.m16, "v16": opt.v16, "w32": getattr(opt, "w32", None), "m32": opt.m32,
                            "v32": opt.v32, "step_count": opt.step_count}, os.path.join(d, "optimizer.pt"))
            with open(os.path.join(d, "trainer_state.json"), "w") as f:
                json.dump({"global_step": self.state.global_step, "log_history": self.state.log_history}, f)
            torch.save(self._rng_state(), os.path.join(d, "rng_state.pth"))
            lim = self.args.save_total_limit
            if lim:
                cks = sorted(glob.glob(os.path.join(self._get_output_dir(trial), "checkpoint-*")),
                             key=lambda p: int(re.findall(r"checkpoint-(\d+)", p)[-1]))
                import shutil
                for old in cks[:-lim]:
                    shutil.rmtree(old, ignore_errors=True)
        if self.world_size > 1:
            dist.barrier()

    def _rng_state(self):
        st = {"cpu": torch.get_rng_state()}
        if torch.cuda.is_available():
            st["cuda"] = torch.cuda.get_rng_state()
        return st

    def _restore_rng(self, st):
        torch.set_rng_state(st["cpu"].cpu())
        if "cuda" in st and torch.cuda.is_available():
            torch.cuda.set_rng_state(st["cuda"].cpu())

    def _load_checkpoint(self, d):
        """Restores weights, optimizer arenas, step count and returns the saved RNG state (or None).  Adaptor-only checkpoints
        (mm_projector.bin, written under --tune_mm_mlp_adapter) carry no optimizer state: the weights are loaded and the optimizer
        starts fresh, as the reference does when it re-reads --pretrain_mm_mlp_adapter."""
        from ..model.builder_io import load_into, load_state_dict_files
        if d is True:
            cks = sorted(glob.glob(os.path.join(self.args.output_dir, "checkpoint-*")),
                         key=lambda p: int(re.findall(r"checkpoint-(\d+)", p)[-1]))
            d = cks[-1]
        opt = self.create_optimizer()
        adaptor = os.path.join(d, "mm_projector.bin")
        if os.path.exists(adaptor) and not glob.glob(os.path.join(d, "pytorch_model*.bin")) and not glob.glob(os.path.join(d, "*.safetensors")):
            sd = torch.load(adaptor, map_location="cpu", weights_only=True)
            load_into(self.model, sd, strict=False)
        else:
            load_into(self.model, load_state_dict_files(d), strict=False)
        opt.refresh_master()                                 # fp32 master copy follows the weights just loaded
        op = os.path.join(d, "optimizer.pt")
        if os.path.exists(op):
            st = torch.load(op, map_location=self.model.device, weights_only=True)
            saved_bits = 8 if st.get("optim") == "adamw_8bit" else 32          # checkpoints without the key hold fp32 moments
            if saved_bits != opt.optim_bits:
                raise ValueError("%s holds %d-bit AdamW state (%s) but this run has --optim %s (%d-bit state); resume with the --optim the "
                                 "checkpoint was saved with -- the state is not converted" % (
                                     op, saved_bits, "--optim adamw_bnb_8bit / adamw_8bit" if saved_bits == 8 else "--optim adamw_torch",
                                     self.args.optim, opt.optim_bits))
            for k in ("master", "m16", "v16", "m8", "v8", "absmax", "m32", "v32"):
                if st.get(k) is not None and getattr(opt, k) is not None:
                    getattr(opt, k).copy_(st[k])
            opt.step_count = st["step_count"]
        else:
            print("[resume] %s has no optimizer.pt (adaptor-only checkpoint): weights restored, optimizer state starts fresh" % d, flush=True)
        m = re.findall(r"checkpoint-(\d+)", d)
        ts = os.path.join(d, "trainer_state.json")
        if os.path.exists(ts):
            with open(ts) as f:
                self.state.global_step = json.load(f)["global_step"]
        elif m:
            self.state.global_step = int(m[-1])
        rp = os.path.join(d, "rng_state.pth")
        return torch.load(rp, map_location="cpu", weights_only=True) if os.path.exists(rp) else None


class AdapterCheckpointMixin:
    """`--tune_mm_mlp_adapter`: checkpoints hold config.json + mm_projector.bin only (llava_trainer.py:249-281, align_trainer.py:616-643)."""

    def _save_checkpoint(self, model, trial, metrics=None):
        if not getattr(self.args, "tune_mm_mlp_adapter", False):
            return super()._save_checkpoint(model, trial, metrics)
        d = os.path.join(self._get_output_dir(trial), f"checkpoint-{self.state.global_step}")
        if self.rank == 0:
            os.makedirs(d, exist_ok=True)
            self.model.config.save_pretrained(d)
            torch.save({k: v.detach().cpu() for k, v in self.model.state_dict().items() if "mm_projector" in k}, os.path.join(d, "mm_projector.bin"))

    def _save(self, output_dir: Optional[str] = None, state_dict=None):
        if not getattr(self.args, "tune_mm_mlp_adapter", False):
            super()._save(output_dir, state_dict)
