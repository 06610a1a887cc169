"""Minimal trainer loop with the HF ``Trainer`` surface the reference's trainers rely on
(``compute_loss`` / ``training_step`` / ``create_optimizer`` / ``log`` / ``save_model`` / ``_save_checkpoint``).

The reference subclasses ``transformers.Trainer`` and runs under accelerate + DeepSpeed ZeRO-2
(llavamod/train/align_trainer.py:180-309).  Here one process drives one GPU; gradient accumulation is local, the
optimizer is the fused AdamW of ``engine.TrainState`` and the only collective is the student-gradient all-reduce.
"""
import glob
import json
import os
import re
import time
from collections import defaultdict

import torch
import torch.distributed as dist

from .engine import TrainState, cosine_lr, warmup_steps_of


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
        self._statics = {}                   # base signature -> static input buffers shared by the graphs of that signature
        # data parallel experiment (LLAVAMOD_GRAPH_ALLREDUCE=1, OFF by default): capture the gradient all-reduce INSIDE the graph of the step's
        # last micro-batch, behind the student's backward and ahead of the join with the teacher stream.  NCCL's CTAs then compete with the
        # teacher's persistent GEMMs instead of hiding behind them, and c10d aborts at shutdown with captured NCCL work outstanding.
        self.graph_allreduce = bool(int(os.environ.get("LLAVAMOD_GRAPH_ALLREDUCE", "0")))
        self._suppress_store = False
        self.graph_replayed_launches = 0     # liblmod kernels executed through graph replays (not seen by the host-side counter)

    # ---- optimizer ---------------------------------------------------------------------------------------
    def create_optimizer(self):
        """Fused AdamW over the flat arenas with the reference's parameter groups (align_trainer.py:326-434): decay / no-decay (names
        containing "bias", nn.LayerNorm parameters) and, with --mm_projector_lr, the projector's own LR groups -- each a contiguous slice
        of the arenas (engine.TrainState).  DeepSpeed's split into MoE expert groups changes no hyper-parameter and is not mirrored."""
        if self.optimizer is None:
            a = self.args
            self.optimizer = TrainState(self.model, lr=a.learning_rate, betas=(a.adam_beta1, a.adam_beta2), eps=a.adam_epsilon,
                                        weight_decay=a.weight_decay, max_grad_norm=a.max_grad_norm,
                                        mm_projector_lr=getattr(a, "mm_projector_lr", None))
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
        Subclasses provide ``_graph_signature(inputs)`` (hashable, or None = not capturable) and
        ``_graph_static_inputs(inputs, static=None)`` (allocate / refill the static device inputs)."""
        import torch
        try:
            sig = self._graph_signature(inputs, next_inputs)
        except TypeError:
            sig = self._graph_signature(inputs)
        if sig is None:
            return None
        pipelined = isinstance(sig, tuple) and sig[-1] == "pipelined"
        closing = (self.graph_allreduce and self.world_size > 1 and self._accum + 1 == self.args.gradient_accumulation_steps)
        base_sig = sig
        if closing:
            sig = ("closing",) + tuple(sig)                 # its own graph: the same micro-batch + the captured gradient all-reduce
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
                old = self._graphs.pop(captured.pop(0))
                old_base = old.get("base")
                old.clear()
                if not any(v.get("base") == old_base for v in self._graphs.values()):
                    self._statics.pop(old_base, None)
            # the plain and the step-closing graph of one signature are captured against the SAME static buffers: they take turns on one
            # stream of micro-batches, and the teacher's look-ahead state (logits / tower features of the next batch) must carry over
            static = self._statics.get(base_sig)
            if static is None:
                static = self._graph_static_inputs(inputs, None, next_inputs, pipelined) if pipelined else self._graph_static_inputs(inputs, None)
                self._statics[base_sig] = static
            elif pipelined:
                self._graph_static_inputs(inputs, static, next_inputs, True)
            else:
                self._graph_static_inputs(inputs, static)
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
                    if closing:
                        self.optimizer.allreduce_grads()          # NCCL nodes in the graph, ahead of the join with the teacher stream
                    if hasattr(self, "_graph_epilogue"):
                        self._graph_epilogue(static)
            finally:
                self._suppress_store = False
            ent.update(graph=g, static=static, base=base_sig, loss=loss.detach(), outputs={k: v for k, v in outputs.items()},
                       launches=_C.launch_count() - n0)
            # the capture pass does not execute: fall through to a replay for this very batch
        if pipelined:
            self._graph_static_inputs(inputs, ent["static"], next_inputs, True)
        else:
            self._graph_static_inputs(inputs, ent["static"])
        ent["graph"].replay()
        if closing:
            self.optimizer.grads_reduced = True              # TrainState.step() must not reduce again
        self.graph_replayed_launches += ent["launches"]
        self.store_metrics({k: (v.clone() if hasattr(v, "clone") else v) for k, v in ent["outputs"].items()}, train_eval="train")
        return ent["loss"].clone()

    # static device inputs of a captured micro-batch: images + the precomputed splice plan (ids / labels / masks stay host-side: the
    # plan already encodes them)
    def _fill_static(self, static, inputs):
        images, plan = inputs["images"], inputs["splice_plan"]
        if torch.is_tensor(images):
            static["images"].copy_(images, non_blocking=True)
        else:
            for i, im in enumerate(images):
                static["images"][i].copy_(im, non_blocking=True)
        for k, v in plan.items():
            if torch.is_tensor(v):
                static["splice_plan"][k].copy_(v, non_blocking=True)
        if static.get("moe_noise") is not None:           # explicit router noise (parity runs): static buffers like every other device input
            for dst, src in zip(static["moe_noise"], inputs["moe_noise"]):
                dst.copy_(src, non_blocking=True)

    def _new_static(self, inputs):
        dev = self.model.device
        images, plan = inputs["images"], inputs["splice_plan"]
        n = len(images) if not torch.is_tensor(images) else images.shape[0]
        ish = tuple(images[0].shape) if not torch.is_tensor(images) else tuple(images.shape[1:])
        noise = inputs.get("moe_noise")
        return dict(input_ids=inputs["input_ids"], labels=inputs["labels"], attention_mask=inputs.get("attention_mask"),
                    moe_noise=[torch.empty(tuple(t.shape), dtype=torch.float32, device=dev) for t in noise] if noise is not None else None,
                    images=torch.empty((n,) + ish, dtype=self.model.dtype, device=dev),
                    splice_plan={k: (torch.empty_like(v) if torch.is_tensor(v) else v) for k, v in plan.items()})

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

    def train(self, resume_from_checkpoint=None):
        a = self.args
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
    def log(self, logs):
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
            if opt is not None:
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
            for k in ("master", "m16", "v16", "m32", "v32"):
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
