#!/usr/bin/env python
"""Gradient checkpointing (``--gradient_checkpointing True``) against the plain step, on the H100.

    python scripts/bench_grad_checkpoint.py [--steps 2] [--warmup 2] [--only NAME ...] [--out FILE]

Every (configuration, arm) runs in a child process of its own with CUDA graphs on (except the SFT step that trains the embedding, which
runs eagerly), so each peak is that arm's alone.  Per run: the optimizer-step time (median over --steps after --warmup) and torch.cuda.max_memory_allocated over the whole run.
  * config2            0.5B-4E <- 7B mimic, T' = 2048, 8 micro-batches (bench.py's headline)
  * config5-mimic      1.8B-4E <- 7B mimic, T' = 4096, 8 micro-batches
  * finetune           dense Qwen1.5-1.8B SFT, 4 samples of 2048 per micro-batch (shells/train/qwen/finetune.sh)
  * pretrain           projector-only pre-training on the dense 1.8B, 8 samples of 2048 per micro-batch (pretrain.sh)
  * 1.8B-8E-pref-8bit  1.8B-8E <- 7B preference, T' = 2048, --optim adamw_bnb_8bit
  * 1.8B-8E-mimic-8bit 1.8B-8E <- 7B mimic, T' = 4096, --optim adamw_bnb_8bit
A run that does not fit reports the allocation failure.  Prints one JSON line with the card's name, power limit and maximum SM clock."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "llava-mod_b200"))

import torch  # noqa: E402

import bench  # noqa: E402

CONFIGS = {
    "config2": dict(wl="mimic-0.5B-4E-from-7B-seq2048", bits=32),
    "config5-mimic": dict(wl="mimic-1.8B-4E-from-7B-seq4096", bits=32),
    "finetune": dict(sft="qwen1.5-1.8b", batch=4, seq=2048, projector_only=False),
    "pretrain": dict(sft="qwen1.5-1.8b", batch=8, seq=2048, projector_only=True),
    "1.8B-8E-pref-8bit": dict(wl=dict(kind="dpo", student="qwen1.5-1.8b", teacher="qwen1.5-7b", clip="clip-l-336", seq=2048, accum=8,
                                      experts=8), bits=8),
    "1.8B-8E-mimic-8bit": dict(wl=dict(kind="mimic", student="qwen1.5-1.8b", teacher="qwen1.5-7b", clip="clip-l-336", seq=4096, accum=8,
                                       experts=8), bits=8),
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return dict(gpu=name, power_limit_w=float(power), max_sm_clock_mhz=float(clock))
    except Exception:                                  # noqa: BLE001 -- reported when it can be read
        return dict(gpu=torch.cuda.get_device_name(), power_limit_w=None, max_sm_clock_mhz=None)


def _distill_job(c, dev):
    from llavamod.model import synthetic as S
    from llavamod.train.engine import TrainState
    name = c["wl"] if isinstance(c["wl"], str) else "grad-ckpt-probe"
    if not isinstance(c["wl"], str):
        bench.WORKLOADS[name] = c["wl"]
    wl = bench.WORKLOADS[name]
    teacher = S.make_teacher(wl["teacher"], wl["clip"], device=dev, seed=0)
    student = S.make_student(wl["student"], wl["clip"], device=dev, seed=1, margs=S.moe_args(num_experts=wl["experts"]),
                             share_tower_with=teacher)
    ts = TrainState(student, lr=2e-5, weight_decay=0.0, max_grad_norm=1.0, optim_bits=c["bits"])
    return student, bench.Job(name, student, teacher, wl["accum"], 0, 1, dev, optimizer=ts)


class _SFTJob:
    """LLaVATrainer (plain CE) on the dense model, `batch` samples of `seq` spliced positions per micro-batch, 8 micro-batches per step."""

    def __init__(self, c, dev):
        from llavamod.config.args import TrainingArguments
        from llavamod.model import synthetic as S
        from llavamod.train.llava_trainer import LLaVATrainer
        self.student = S.make_teacher(c["sft"], "clip-l-336", device=dev, seed=1).train()
        for n, p in self.student.named_parameters():
            p.requires_grad = ("mm_projector" in n) if c["projector_only"] else ("image_tower" not in n)
        self.accum = 8
        args = TrainingArguments(output_dir="/tmp/lmod_gc", per_device_train_batch_size=c["batch"], gradient_accumulation_steps=self.accum,
                                 learning_rate=2e-5, lr_scheduler_type="constant", max_steps=1000, logging_steps=0, save_strategy="no", bf16=True)
        self.tr = LLaVATrainer(model=self.student, args=args)
        wl = dict(clip="clip-l-336", seq=c["seq"])
        V = self.student.config.vocab_size
        self.batches = []
        for i in range(2):
            parts = [bench.synth_batch(wl, 0, i * c["batch"] + j, V) for j in range(c["batch"])]
            b = dict(input_ids=torch.cat([p["input_ids"] for p in parts]), labels=torch.cat([p["labels"] for p in parts]),
                     attention_mask=torch.cat([p["attention_mask"] for p in parts]),
                     images=torch.stack([p["images"][0] for p in parts]).to(dev))
            self.batches.append(b)
        # a trainable embedding needs the splice plan's row order, which the captured step's precomputed plan does not carry: the SFT
        # step with the embedding trained runs eagerly, the projector-only step is captured
        self.tr.use_cuda_graphs = c["projector_only"]
        if c["projector_only"]:
            for b in self.batches:
                b["splice_plan"] = self.student.make_splice_plan(b["input_ids"], b["attention_mask"], b["labels"])
        self.i = 0

    def run(self, n_steps):
        last = None
        for _ in range(n_steps * self.accum):
            last = self.tr.training_step(self.student, self.batches[self.i % 2])
            self.i += 1
        return last


def child(name, arm, steps, warmup):
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.manual_seed(0)
    c = CONFIGS[name]
    try:
        if "sft" in c:
            job = _SFTJob(c, dev)
            student = job.student
        else:
            student, job = _distill_job(c, dev)
        if arm == "ckpt":
            student.gradient_checkpointing_enable()
            student.enable_input_require_grads()
        job.run(warmup)
        torch.cuda.synchronize()
        ms = []
        for _ in range(steps):
            t0 = time.perf_counter()
            last = job.run(1)
            torch.cuda.synchronize()
            ms.append((time.perf_counter() - t0) * 1e3)
        loss = float(last)
        graphs = bool(getattr(getattr(job, "tr", None), "use_cuda_graphs", True))
        return dict(fits=True, cuda_graphs=graphs, step_ms=statistics.median(ms), step_ms_all=ms, peak_gb=torch.cuda.max_memory_allocated() / 1e9,
                    loss=loss)
    except torch.OutOfMemoryError as e:
        return dict(fits=False, error="out of memory: %s" % str(e).splitlines()[0][:200], peak_gb=torch.cuda.max_memory_allocated() / 1e9)


def run_child(args, name, arm):
    cmd = [sys.executable, os.path.abspath(__file__), "--child", name, arm, "--steps", str(args.steps), "--warmup", str(args.warmup)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    if r.returncode != 0 or not lines:
        return {"error": ((r.stderr or r.stdout).strip().splitlines() or ["exit %d" % r.returncode])[-1]}
    return json.loads(lines[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", nargs="+", default=None, choices=sorted(CONFIGS))
    ap.add_argument("--child", nargs=2, default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_grad_checkpoint.py measures on the GPU; no CUDA device is visible")
    if args.child:
        print(json.dumps(child(args.child[0], args.child[1], args.steps, args.warmup)))
        return
    res = dict(card(), steps=args.steps, warmup=args.warmup, runs={})
    for name in args.only or CONFIGS:
        res["runs"][name] = {arm: run_child(args, name, arm) for arm in ("plain", "ckpt")}
        print(name, json.dumps(res["runs"][name]), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
