#!/usr/bin/env python
"""bench.py -- LLaVA-MoD distillation step on H100 (distill samples/s at 1/2/4/8 GPUs; KL-kernel HBM GB/s vs peak; next to the
reference CPU path).

    python bench.py --gpus N --steps K --warmup W            # our path (one process per GPU; torchrun for N > 1)
    python bench.py ... --dump-outputs DIR                   # + what the last timed step computed, as DIR/<name>.npy
    python bench.py --impl reference --gpus N --steps K ...  # the reference's own algorithm on the host cores (oracle)

Headline (`value`, BASELINE config 2): a "step" = one optimizer step of the reference recipe on every GPU: 8 micro-batches of one
sample each (per_device_train_batch_size 1 x gradient_accumulation_steps 8, dense2sparse_distillation.sh:70-72), each micro-batch =
CLIP tower forward + frozen 7B teacher forward + 0.5B-4E sparse student forward/backward + fused mimic-KL/LM loss, then gradient
all-reduce (N > 1), global-norm clip and fused AdamW.  Synthetic inputs of the named shape (SURVEY.md section 8d): 336x336 image, 1473
text ids with one <image> -> spliced length 2048, first 40% masked.

`secondary` (BASELINE configs 3, 4 and 5 in front of the driver at every N; 3 and 4 in the same process after the headline):
  config3  the same mimic step at GLOBAL batch 256 (256 / N micro-batches per GPU and optimizer step);
  config4  the preference (DPO) stage on the same 0.5B-4E <- 7B pair: chosen + rejected of T' = 2048, 2 reference + 2 policy forwards,
           2 policy backwards per pair (preference_distillation.sh:48-88), with the log-prob-gather kernel's roofline;
  config5  1.8B-4E student <- 7B teacher at T' = 2048 (the recipe's model_max_length), mimic micro-batches and preference pairs in one
           step (4 experts: with 8 the trainable state alone exceeds 80 GB).  It runs in a child process of its own, started before this
           process builds its models, and eagerly: the CUDA-graph pools of its two stages (~17 GB) do not fit next to the 1.8B student's
           optimizer state and the teacher in 80 GB.
           The mimic stage alone at T' = 4096 runs as --workload mimic-1.8B-4E-from-7B-seq4096.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "llava-mod_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

WORKLOADS = {
    # name: kind, student arch, teacher arch, clip, spliced seq len, accumulation (micro-batches per optimizer step and GPU), experts
    "mimic-0.5B-4E-from-7B-seq2048": dict(kind="mimic", student="qwen1.5-0.5b", teacher="qwen1.5-7b", clip="clip-l-336", seq=2048, accum=8, experts=4),
    "preference-0.5B-4E-from-7B-seq2048": dict(kind="dpo", student="qwen1.5-0.5b", teacher="qwen1.5-7b", clip="clip-l-336", seq=2048, accum=8, experts=4),
    "mimic-1.8B-4E-from-7B-seq4096": dict(kind="mimic", student="qwen1.5-1.8b", teacher="qwen1.5-7b", clip="clip-l-336", seq=4096, accum=8, experts=4),
    "mimic+pref-1.8B-4E-from-7B-seq2048": dict(kind="mimic+dpo", student="qwen1.5-1.8b", teacher="qwen1.5-7b", clip="clip-l-336", seq=2048, accum=8, experts=4),
    "tiny": dict(kind="mimic", student="tiny", teacher="tiny", clip="tiny", seq=64, accum=2, experts=4),
    "tiny-pref": dict(kind="dpo", student="tiny", teacher="tiny", clip="tiny", seq=64, accum=2, experts=4),
    "tiny-mimic+pref": dict(kind="mimic+dpo", student="tiny", teacher="tiny", clip="tiny", seq=64, accum=2, experts=4),
}
# nominal dense FLOP per unit (SURVEY.md 8d): mimic sample; preference pair = 2 teacher fwd + 2 student fwd/bwd + CLIP
FLOP_PER_SAMPLE = {"mimic-0.5B-4E-from-7B-seq2048": 38.5e12, "mimic-1.8B-4E-from-7B-seq4096": 115.7e12,
                   "preference-0.5B-4E-from-7B-seq2048": (2 * 30.17 + 2 * 7.6 + 0.38) * 1e12}
HEADLINE = "mimic-0.5B-4E-from-7B-seq2048"


def peaks():
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            d = json.load(f)
        return d["hbm_gbs"], d.get("bf16_tflops_sustained", d["bf16_tflops"]), "measured"
    except Exception:
        return 3350.0, 989.0, "H100 SXM data sheet (HBM3 3.35 TB/s, dense BF16 989 TFLOP/s)"


def synth_batch(wl, rank, idx, vocab, device=None, pinned=False):
    """One mimic sample (SURVEY.md 8d): ids with position 5 = -200, 40% instruction mask, all-true attention mask."""
    from llavamod.model import synthetic as S
    clip = S.CLIP[wl["clip"]]
    P = (clip["image_size"] // clip["patch_size"]) ** 2
    Tt = wl["seq"] - P + 1
    g = torch.Generator().manual_seed(1234 + 1000 * rank + idx)
    ids = torch.randint(0, vocab, (1, Tt), generator=g)
    ids[0, 5] = -200
    labels = ids.clone()
    labels[0, : int(0.4 * Tt)] = -100
    mask = torch.ones(1, Tt, dtype=torch.bool)
    img = torch.randn(3, clip["image_size"], clip["image_size"], generator=g).to(torch.bfloat16)
    if pinned:
        ids, labels, mask, img = ids.pin_memory(), labels.pin_memory(), mask.pin_memory(), img.pin_memory()
    return dict(input_ids=ids, labels=labels, attention_mask=mask, images=[img])


def synth_pair(wl, rank, idx, vocab, pinned=False):
    """One preference pair (SURVEY.md 8d): chosen / rejected share the first 40 % (instruction incl. the image) and differ in the response."""
    b = synth_batch(wl, rank, idx, vocab)
    g = torch.Generator().manual_seed(987654 + 1000 * rank + idx)
    Tt = b["input_ids"].shape[1]
    k = int(0.4 * Tt)
    rej = b["input_ids"].clone()
    rej[0, k:] = torch.randint(0, vocab, (Tt - k,), generator=g)
    rl = rej.clone()
    rl[0, :k] = -100
    out = dict(chosen_input_ids=b["input_ids"], chosen_labels=b["labels"], chosen_attention_mask=b["attention_mask"],
               rejected_input_ids=rej, rejected_labels=rl, rejected_attention_mask=b["attention_mask"].clone(), images=b["images"])
    if pinned:
        out = {k2: ([t.pin_memory() for t in v] if isinstance(v, list) else v.pin_memory()) for k2, v in out.items()}
    return out


class ClockSampler(threading.Thread):
    """nvidia-smi clocks / throttle reasons DURING the timed region."""

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.rows, self.stop_flag, self.proc = index, [], False, None

    def run(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q, "--format=csv,noheader,nounits", "-lms", "200"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            for line in self.proc.stdout:
                if self.stop_flag:
                    break
                self.rows.append([x.strip() for x in line.split(",")])
        except Exception:
            pass

    def finish(self):
        self.stop_flag = True
        if self.proc is not None:
            self.proc.terminate()
        sm, mx, reasons = [], 0.0, set()
        for r in self.rows:
            try:
                sm.append(float(r[0])); mx = max(mx, float(r[1]))
                for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[3:7]):
                    if v.lower().startswith("active"):
                        reasons.add(name)
            except Exception:
                continue
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx or None, "reasons": sorted(reasons), "samples": len(sm)}


# ---------------------------------------------------------------------------------------------------------------------
# the reference arm / cpu_baseline: the oracle (CPU restatement of the reference's algorithm) on the host cores.
# One "step" of this arm EXECUTES one micro-batch of the named workload through every layer -- 32 teacher layers, 12 dense + 12 MoE
# student layers forward and backward, 2 x 23 CLIP layers, both lm_heads over the full vocabulary, the mimic + LM losses -- on a BOUNDED
# number of sequence positions (REF_TOKENS of the T' positions; the image's 576 come first) so that a --steps K --warmup W run ends in
# minutes.  Layers of one kind share ONE set of random weights (memory; timing does not depend on values).  `ms_per_step` is the time
# really spent per step; `value` scales it to full samples linearly in tokens (labelled estimated; the quadratic attention term makes
# a full-length sample slower, so the scaling favours the reference).  The optimizer update is not included (also favours it).
# ---------------------------------------------------------------------------------------------------------------------
_CPU_CACHE = {}
REF_TOKENS = int(os.environ.get("LMOD_REF_TOKENS", "512"))


def _alias_layers(sd, n_layers, moe_layers):
    """state dict of `n_layers` layers whose tensors alias layer 0 (MoE pattern) / layer 1 (dense pattern) of a 2-layer init."""
    out = {k: v for k, v in sd.items() if ".layers." not in k}
    for i in range(n_layers):
        src = 0 if i in moe_layers else 1
        pre = "model.layers.%d." % src
        for k, v in sd.items():
            if k.startswith(pre):
                out["model.layers.%d.%s" % (i, k[len(pre):])] = v
    return out


def _cpu_setup(wl_name):
    from oracle import restated as R
    from llavamod.model import synthetic as S
    if wl_name in _CPU_CACHE:
        return _CPU_CACHE[wl_name]
    wl = WORKLOADS[wl_name]
    g = torch.Generator().manual_seed(0)
    sa, ta, ca = S.ARCH[wl["student"]], S.ARCH[wl["teacher"]], S.CLIP[wl["clip"]]
    T = wl["seq"]
    Tr = min(T, REF_TOKENS)
    V = sa["vocab_size"]
    E = wl["experts"]

    def lm(arch, layers, moe_layers=()):
        return R.LMCfg(hidden=arch["hidden_size"], inter=arch["intermediate_size"], layers=layers, heads=arch["num_attention_heads"],
                       kv_heads=arch["num_key_value_heads"], vocab=64, rope_theta=arch["rope_theta"], moe_layers=list(moe_layers),
                       num_experts=E, capacity_factor=1.5, kd_vocab=64)

    c = dict(T=T, Tr=Tr, V=V, wl=wl, sa=sa, ta=ta, ca=ca)
    Lt, Ls = ta["num_hidden_layers"], sa["num_hidden_layers"]
    s_moe = list(range(Ls))[::2]
    c["tc"] = lm(ta, Lt)
    c["t_sd"] = _alias_layers(R.init_lm(lm(ta, 2), 8, g), Lt, ())
    c["sc"] = lm(sa, Ls, s_moe)
    base = R.init_lm(lm(sa, 2, (0,)), 8, g)
    for k in R.trainable_keys(base):
        base[k].requires_grad_(True)
    c["s_sd"] = _alias_layers(base, Ls, s_moe)
    c["s_params"] = [v for v in base.values() if v.requires_grad]
    c["noise"] = [R.gumbel_noise((Tr, E), g) for _ in s_moe]
    c["t_x"] = torch.randn(1, Tr, ta["hidden_size"], generator=g)
    c["s_x"] = torch.randn(1, Tr, sa["hidden_size"], generator=g)
    cc2 = R.ClipCfg(hidden=ca["hidden_size"], inter=ca["intermediate_size"], layers=2, heads=ca["num_attention_heads"],
                    image=ca["image_size"], patch=ca["patch_size"], select_layer=-2)
    csd = R.init_clip(cc2, g)
    c["cc"] = R.ClipCfg(hidden=ca["hidden_size"], inter=ca["intermediate_size"], layers=ca["num_hidden_layers"], heads=ca["num_attention_heads"],
                        image=ca["image_size"], patch=ca["patch_size"], select_layer=-2)
    pre = R.P_CLIP + "encoder.layers."
    c["c_sd"] = {k: v for k, v in csd.items() if not k.startswith(pre)}
    for i in range(ca["num_hidden_layers"]):
        for k, v in csd.items():
            if k.startswith(pre + "0."):
                c["c_sd"][pre + "%d.%s" % (i, k[len(pre) + 2:])] = v
    c["img"] = torch.randn(1, 3, ca["image_size"], ca["image_size"], generator=g)
    c["wt"] = torch.empty(V, ta["hidden_size"]).normal_(0, 0.02, generator=g)
    c["ws"] = torch.empty(V, sa["hidden_size"]).normal_(0, 0.02, generator=g).requires_grad_(True)
    lab = torch.randint(0, V, (1, Tr), generator=g)
    lab[0, : int(0.4 * Tr)] = -100
    c["labels"] = lab
    _CPU_CACHE[wl_name] = c
    return c


def cpu_step_sample(wl_name, threads):
    """One executed micro-batch on REF_TOKENS positions.  Returns (seconds spent, fraction of a full sample it stands for, description, parts)."""
    from oracle import restated as R
    torch.set_num_threads(threads)
    c = _cpu_setup(wl_name)
    T, Tr, V = c["T"], c["Tr"], c["V"]
    t = {}
    t_all = time.perf_counter()
    with torch.no_grad():
        t0 = time.perf_counter()
        R.clip_tower(c["c_sd"], c["cc"], c["img"])                     # teacher's tower pass ...
        R.clip_tower(c["c_sd"], c["cc"], c["img"])                     # ... and the student's own (llava_arch.py:184)
        t["clip_2x%d_layers" % (c["cc"].layers - 1)] = time.perf_counter() - t0
        t0 = time.perf_counter()
        th, _ = R.lm_forward(c["t_sd"], c["tc"], c["t_x"], None, None)
        tl = torch.nn.functional.linear(th, c["wt"]).float()
        t["teacher_%d_layers_fwd+lm_head" % c["tc"].layers] = time.perf_counter() - t0
    for p in c["s_params"]:
        p.grad = None
    c["ws"].grad = None
    x = c["s_x"].clone().requires_grad_(True)
    t0 = time.perf_counter()
    h, la = R.lm_forward(c["s_sd"], c["sc"], x, None, None, c["noise"])
    sl = torch.nn.functional.linear(h, c["ws"]).float()
    moe_loss = c["sc"].aux_coef * sum(la)
    out = dict(logits=sl, labels=c["labels"], loss=R.shifted_ce(sl, c["labels"], V) + moe_loss, moe_loss=moe_loss)
    loss, _ = R.mimic_compute_loss(out, tl, "kd_lm", True, False, V)
    loss.backward()
    t["student_%d_layers_fwd_bwd+lm_head+losses" % c["sc"].layers] = time.perf_counter() - t0
    spent = time.perf_counter() - t_all
    desc = ("oracle (CPU restatement of the reference, fp32, %d threads): ONE micro-batch executed through all layers (2x%d CLIP, %d teacher, "
            "%d student fwd+bwd of which %d MoE, both lm_heads over V=%d, mimic+LM+aux losses, backward) on %d of the %d sequence positions; "
            "weights of same-kind layers shared; samples/s = (%d/%d) / measured seconds (estimated: linear in tokens); no optimizer update"
            % (threads, c["cc"].layers - 1, c["tc"].layers, c["sc"].layers, len(c["sc"].moe_layers), V, Tr, T, Tr, T))
    return spent, Tr / T, desc, t


def pick_threads(wl_name):
    """All the host threads the oracle can USE: torch's intra-op pool stops scaling (and on 100+ core boxes degrades) well
    before the core count for these shapes, so time one teacher-shaped GEMM chain at a few pool sizes and keep the fastest."""
    c = _cpu_setup(wl_name)
    n = os.cpu_count() or 1
    cands = sorted({n, max(1, n // 2), max(1, n // 4), min(n, 32), min(n, 16), min(n, 8)}, reverse=True)
    H = c["ta"]["hidden_size"]
    x = torch.randn(min(c["Tr"], 512), H)
    w = torch.randn(c["ta"]["intermediate_size"], H)
    best, best_t = n, None
    for th in cands:
        torch.set_num_threads(th)
        with torch.no_grad():
            torch.nn.functional.linear(x, w)
            t0 = time.perf_counter()
            for _ in range(3):
                torch.nn.functional.linear(x, w)
            dt = time.perf_counter() - t0
        if best_t is None or dt < best_t:
            best, best_t = th, dt
    return best


def our_config(wl_name, accum, world, cuda_graphs=True, compact=True):
    """`config` of the JSON line -- identical for our arm and the reference arm (same workload, same recipe)."""
    wl = WORKLOADS[wl_name]
    return {"workload": wl_name, "student": wl["student"] + "-%dE-top2" % wl["experts"], "teacher": wl["teacher"], "vision": wl["clip"],
            "seq_len": wl["seq"], "micro_batch": 1, "grad_accum": accum, "global_batch": accum * world,
            "loss": {"mimic": "kd_lm (mimic KL + LM + aux)", "dpo": "sigmoid DPO + aux", "mimic+dpo": "kd_lm micro-batches + sigmoid-DPO pairs"}[wl["kind"]],
            "parallelism": "dp%d" % world,
            # timing rule: no explicit L2 flush between timed steps -- one step streams the 15.4 GB of frozen teacher weights, the student's
            # weights / gradients / optimizer arenas and ~2 GB of activations and logits per micro-batch through a 50 MB L2
            "l2": "inputs larger than L2 (>= 17 GB touched per micro-batch); no flush"}


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    wl_name = args.workload
    if WORKLOADS[wl_name]["kind"] != "mimic":
        print(json.dumps({"impl": "reference", "unavailable": "the CPU arm is built for the mimic workloads"}), flush=True)
        return
    threads = pick_threads(wl_name)
    accum = args.accum if args.accum else WORKLOADS[wl_name]["accum"]
    for _ in range(args.warmup):
        cpu_step_sample(wl_name, threads)
    t0 = time.perf_counter()
    spent, frac, desc = 0.0, 1.0, ""
    for _ in range(args.steps):
        s, frac, desc, parts = cpu_step_sample(wl_name, threads)
        spent += s
    wall = time.perf_counter() - t0
    value = args.steps * frac / spent
    world = int(os.environ.get("WORLD_SIZE", str(args.gpus)))
    line = {"impl": "reference", "metric": "distill_samples_per_sec", "value": value, "unit": "samples/s", "n_gpus": args.gpus, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": 1e3 * spent / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic", "config": our_config(wl_name, accum, world),
            "step_definition": "one micro-batch executed on %d of %d sequence positions (bounded sample); value = estimated full samples/s" % (min(WORKLOADS[wl_name]["seq"], REF_TOKENS), WORKLOADS[wl_name]["seq"]),
            "cpu_baseline": {"value": value, "unit": "samples/s", "cores": threads, "kind": "port", "sample": desc, "estimated": True, "parts_s": parts},
            "e2e": {"value": value, "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "wall_s": wall}
    print(json.dumps(line), flush=True)


# ---------------------------------------------------------------------------------------------------------------------
# our arm  (nothing in it imports oracle/ or tests/: the oracle is used by the cpu_baseline / --impl reference legs only)
# ---------------------------------------------------------------------------------------------------------------------
def make_trainer(student, teacher, kind="mimic", accum=1, lr=2e-5, max_steps=1000, optimizer=None, world=1):
    from llavamod.config.args import TrainingArguments
    from llavamod.train.align_trainer import AlignTrainer
    from llavamod.train.dpo_trainer import DPOTrainer
    targs = TrainingArguments(output_dir="/tmp/lmod_out", per_device_train_batch_size=1, gradient_accumulation_steps=accum, learning_rate=lr,
                              weight_decay=0.0, warmup_ratio=0.03, lr_scheduler_type="cosine", max_steps=max_steps, logging_steps=0,
                              save_strategy="no", bf16=True)
    targs.moe_enable = True
    if kind == "mimic":
        tr = AlignTrainer(model=student, ref_model=teacher, args=targs, loss_type="kd_lm", moe_loss_enable=True)
    else:
        tr = DPOTrainer(model=student, ref_model=teacher, args=targs, loss_type="sigmoid", moe_loss_enable=True)
    tr._total_steps = max_steps
    tr.world_size = world
    if optimizer is not None:
        tr.optimizer = optimizer                 # stages of one run share the flat arenas / AdamW state
    return tr


class Job:
    """One workload on this rank: trainers, host (pinned) batches, device-resident batches, and the step function."""

    def __init__(self, wl_name, student, teacher, accum, rank, world, dev, optimizer=None, n_batches=None):
        self.wl_name, self.wl = wl_name, WORKLOADS[wl_name]
        self.accum, self.rank, self.world, self.dev, self.student = accum, rank, world, dev, student
        kinds = self.wl["kind"].split("+")
        self.trainers = {}
        for k in kinds:
            self.trainers[k] = make_trainer(student, teacher, k, accum, optimizer=optimizer, world=world)
            optimizer = self.trainers[k].create_optimizer()
        self.optimizer = optimizer
        V = student.config.vocab_size
        nb = n_batches if n_batches else min(accum * 2, 16)
        self.nb = nb
        self.host, self.res = {}, {}
        for k in kinds:
            if k == "mimic":
                hb = [synth_batch(self.wl, rank, i, V, pinned=True) for i in range(nb)]
                rb = []
                for b in hb:
                    plan = student.make_splice_plan(b["input_ids"], b["attention_mask"], b["labels"])
                    rb.append(dict(input_ids=b["input_ids"], labels=b["labels"], attention_mask=b["attention_mask"],
                                   images=torch.stack(b["images"]).to(dev), splice_plan=plan))
            else:
                hb = [synth_pair(self.wl, rank, i, V, pinned=True) for i in range(nb)]
                rb = []
                for b in hb:
                    r = dict(b)
                    r["images"] = torch.stack(b["images"]).to(dev)
                    r["splice_plan_chosen"] = student.make_splice_plan(b["chosen_input_ids"], b["chosen_attention_mask"], b["chosen_labels"])
                    r["splice_plan_rejected"] = student.make_splice_plan(b["rejected_input_ids"], b["rejected_attention_mask"], b["rejected_labels"])
                    rb.append(r)
            self.host[k], self.res[k] = hb, rb
        self.it = {k: 0 for k in kinds}
        self.units_per_step = accum * len(kinds)            # samples (mimic) + pairs (preference) per optimizer round and GPU

    def run(self, n_steps, resident=True, read_loss=False):
        """n_steps rounds: `accum` micro-batches of every stage kind, each stage closing with its optimizer step."""
        last = None
        for _ in range(n_steps):
            for k, tr in self.trainers.items():
                batches = (self.res if resident else self.host)[k]
                for _ in range(self.accum):
                    i = self.it[k]
                    nxt = batches[(i + 1) % self.nb] if k == "mimic" else None     # look-ahead: the mimic teacher runs one batch ahead
                    last = tr.training_step(self.student, batches[i % self.nb], nxt)
                    self.it[k] = i + 1
            if read_loss:
                _ = float(last)           # D2H read of the step's loss
        return last

    def replayed(self):
        return sum(t.graph_replayed_launches for t in self.trainers.values())

    def reset_counters(self):
        for t in self.trainers.values():
            t.graph_replayed_launches = 0

    def h2d_bytes_per_step(self):
        n = 0
        for k, hb in self.host.items():
            b = hb[0]
            img = b["images"][0].numel() * 2
            T = self.wl["seq"]
            plans = (1 if k == "mimic" else 2) * 5 * T * 8
            n += self.accum * (img + plans) * (2 if k == "mimic" else 1)      # mimic uploads the look-ahead batch too
        return n


def timed_steps(job, steps, barrier, resident=True, read_loss=False):
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    last = job.run(steps, resident, read_loss)
    e1.record()
    barrier()
    return e0.elapsed_time(e1), last


def kernel_rooflines(job, hbm_peak, src):
    """One extra round runs EAGERLY (graphs off; same inputs, kernels and stream) with CUDA events around the loss-head kernels.
    Not part of any throughput number."""
    from llavamod import kernels as K
    saved = {k: t.use_cuda_graphs for k, t in job.trainers.items()}
    for t in job.trainers.values():
        t.use_cuda_graphs = False
    K.TIMERS = {}
    job.run(1)
    torch.cuda.synchronize()
    timers, K.TIMERS = K.TIMERS, None
    for k, t in job.trainers.items():
        t.use_cuda_graphs = saved[k]
    T, V = job.wl["seq"], job.student.config.vocab_size
    out = {}
    if "mimic" in job.trainers:
        lab = job.res["mimic"][0]["splice_plan"]["labels"].cpu()
        m_kd = lab != -100
        m_ce = torch.cat([lab[:, 1:] != -100, torch.zeros(lab.shape[0], 1, dtype=torch.bool)], 1)
        active = int((m_kd | m_ce).sum())
        kd_vocab = min(151936, V)
        compact = bool(getattr(job.trainers["mimic"], "compact_head", False))
        bytes_launch = active * 6 * kd_vocab + (0 if compact else (T - active) * 2 * kd_vocab)
        ev = timers.get("kl_fwd_bwd", [])
        kl_ms = sum(a.elapsed_time(b) for a, b in ev) / max(1, len(ev))
        ach = bytes_launch / (kl_ms * 1e-3) / 1e9 if kl_ms > 0 else None
        traffic = None                       # measured DRAM traffic: no hardware-counter capture is stored with the project
        out["kl"] = {"kernel": "kl_stream_kernel (lmod_kl_fwd_bwd_rows)" if compact else "kl_stream_kernel (lmod_kl_fwd_bwd)", "bound": "hbm",
                     "achieved": ach, "peak": hbm_peak, "unit": "GB/s",
                     "frac": (ach / hbm_peak) if ach else None, "peak_source": src, "traffic": traffic,
                     "algorithmic_bytes_per_launch": bytes_launch, "avg_launch_ms": kl_ms, "launches_timed": len(ev),
                     "note": ("%d of %d rows active (6V B each); " % (active, T))
                             + ("the loss head runs on the active rows only (row compaction), masked rows cost nothing; "
                                if compact else "masked rows zero-filled (2V B); ")
                             + "survey-style 6V*N would read %.1f GB/s" % ((T * 6 * kd_vocab) / (kl_ms * 1e-3) / 1e9 if kl_ms > 0 else 0.0)}
    if "dpo" in job.trainers:
        f, b = timers.get("logp_fwd", []), timers.get("logp_bwd", [])
        f_ms = sum(x.elapsed_time(y) for x, y in f) / max(1, len(f))
        b_ms = sum(x.elapsed_time(y) for x, y in b) / max(1, len(b))
        # SURVEY 8d: log-prob gather = 2V B/token forward (reference + policy forwards), 4V B/token forward+backward (policy)
        fwd_gbs = T * 2 * V / (f_ms * 1e-3) / 1e9 if f_ms > 0 else None
        fb_gbs = T * 4 * V / ((f_ms + b_ms) * 1e-3) / 1e9 if (f_ms > 0 and b_ms > 0) else None
        out["logp"] = {"kernel": "logp_fwd_kernel + logp_bwd_kernel (lmod_logp_gather_fwd / _bwd)", "bound": "hbm", "achieved": fb_gbs, "peak": hbm_peak,
                       "unit": "GB/s", "frac": (fb_gbs / hbm_peak) if fb_gbs else None, "peak_source": src, "traffic": None,
                       "algorithmic_bytes_per_launch": T * 4 * V, "fwd_only_gbs": fwd_gbs, "fwd_only_frac": (fwd_gbs / hbm_peak) if fwd_gbs else None,
                       "avg_fwd_ms": f_ms, "avg_bwd_ms": b_ms, "launches_timed": [len(f), len(b)],
                       "note": "4V B/token for fwd+bwd of a policy forward (the backward re-reads the bf16 logits it overwrites: 6V B of real traffic), "
                               "2V B/token for the forward-only reference forwards"}
    return out


DUMP_SAMPLE = 4 << 20          # trainable-parameter elements written by --dump-outputs (fixed, seeded positions; 16 MB as float32)


def dump_outputs(out_dir, loss, student):
    """What the timed path hands its caller after the last timed step: the step's loss and the updated trainable weights (a fixed,
    seeded sample of them, in name order) -- float64 / float32 .npy files, so that two builds can be compared output for output."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    torch.cuda.synchronize()
    np.save(os.path.join(out_dir, "loss.npy"), np.array([float(loss)], dtype=np.float64))
    params = [p for _, p in sorted(student.named_parameters(), key=lambda kv: kv[0]) if p.requires_grad]
    total = sum(p.numel() for p in params)
    g = torch.Generator(device="cpu").manual_seed(0)
    idx = torch.randint(0, total, (DUMP_SAMPLE,), generator=g).sort().values        # positions in the name-ordered concatenation
    parts, off = [], 0
    for p in params:
        lo, hi = torch.searchsorted(idx, off), torch.searchsorted(idx, off + p.numel())
        if hi > lo:
            parts.append(p.detach().reshape(-1)[(idx[lo:hi] - off).to(p.device)].float().cpu())
        off += p.numel()
    np.save(os.path.join(out_dir, "trainable_params_sample.npy"), torch.cat(parts).numpy().astype(np.float32))


def run_ours(args):
    import torch.distributed as dist
    from llavamod import _C
    from llavamod.model import synthetic as S
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        # the one JSON line is all rank 0 may print on stdout, but NCCL printf()s its "NCCL version ..." banner there whenever NCCL_DEBUG is
        # VERSION / WARN / INFO: send the C-level stdout to stderr while the communicator comes up (init + first collective)
        sys.stdout.flush()
        saved = os.dup(1)
        os.dup2(2, 1)
        try:
            dist.init_process_group("nccl", device_id=torch.device("cuda", local))
            warm = torch.zeros(1, device=torch.device("cuda", local))
            dist.all_reduce(warm)
            torch.cuda.synchronize()
        finally:
            sys.stdout.flush()
            os.dup2(saved, 1)
            os.close(saved)
    dev = torch.device("cuda", local)
    sec5 = config5_child(world, rank) if (args.workload == HEADLINE and not args.no_secondary) else None
    torch.manual_seed(0)                               # host-side draws (router noise) repeat from run to run
    wl_name = args.workload
    wl = WORKLOADS[wl_name]
    accum = args.accum if args.accum else wl["accum"]
    train_modules = S.TRAIN_MODULES + (["deepspeed_experts"] if "dpo" in wl["kind"] else [])      # preference_distillation.sh:60
    teacher = S.make_teacher(wl["teacher"], wl["clip"], device=dev, seed=0)
    student = S.make_student(wl["student"], wl["clip"], device=dev, seed=1, margs=S.moe_args(num_experts=wl["experts"], train_modules=train_modules),
                             share_tower_with=teacher)
    job = Job(wl_name, student, teacher, accum, rank, world, dev)
    torch.cuda.synchronize()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def reduce_max(*vals):
        if world > 1:
            tt = torch.tensor(list(vals), device=dev, dtype=torch.float64)
            dist.all_reduce(tt, op=dist.ReduceOp.MAX)
            return tt.tolist()
        return list(vals)

    # ---- value: device-resident inputs ----
    job.run(args.warmup)
    if args.torch_profile:
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            job.run(1)
            torch.cuda.synchronize()
        with open(args.torch_profile, "w") as f:
            f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=70, max_name_column_width=90))
    sampler = ClockSampler(local)
    sampler.start()
    _C.launch_count_reset()
    job.reset_counters()
    if os.environ.get("LMOD_PROFILE") == "1":          # ncu --profile-from-start off: capture only the timed region
        torch.cuda.cudart().cudaProfilerStart()
    ms, last = timed_steps(job, args.steps, barrier)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last, student)
    if os.environ.get("LMOD_PROFILE") == "1":
        torch.cuda.synchronize()
        torch.cuda.cudart().cudaProfilerStop()
    launches = _C.launch_count() + job.replayed()
    clocks = sampler.finish()
    final_loss = float(last)
    # ---- e2e: host (pinned) buffers through the public trainer call, H2D copies + loss read inside the timed region ----
    if args.no_e2e:
        ms_e2e = float("nan")
    else:
        job.run(1, resident=False, read_loss=True)
        ms_e2e, _ = timed_steps(job, args.steps, barrier, resident=False, read_loss=True)
    hbm_peak, tf_peak, src = peaks()
    roofs = kernel_rooflines(job, hbm_peak, src)
    ms, ms_e2e = reduce_max(ms, ms_e2e)
    units = args.steps * job.units_per_step * world
    value = units / (ms / 1e3)
    e2e = units / (ms_e2e / 1e3)
    T = wl["seq"]
    cfg = our_config(wl_name, accum, world)
    mimic_tr = job.trainers.get("mimic")
    line = {
        "metric": "distill_samples_per_sec", "value": value, "unit": "samples/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
        "config": cfg,
        "implementation": {"l2": "working set per micro-batch (15.4 GB of teacher weights) >> 50 MB L2; no explicit flush",
                           "kernels": "hand-written wgmma+TMA GEMM / grouped expert GEMM, wgmma flash-attention forward AND backward, router, "
                                      "loss heads (liblmod_b200); no library GEMM or attention kernel on the path",
                           "cuda_graphs": all(bool(t.use_cuda_graphs) for t in job.trainers.values()),
                           "loss_head": ("supervised rows only (device-side row compaction, dynamic-extent GEMMs)"
                                         if (mimic_tr is not None and getattr(mimic_tr, "compact_head", False)) else "all rows"),
                           "unit": "a mimic sample or a preference pair counts as one sample"},
        "clocks": clocks, "gpu_launches": launches,
        "e2e": {"value": e2e, "unit": "samples/s", "h2d_bytes_per_step": job.h2d_bytes_per_step(), "d2h_bytes_per_step": 4,
                "note": "each mimic micro-batch uploads its own inputs and the look-ahead inputs of the next one (teacher runs one batch ahead)",
                "ms_per_step": ms_e2e / args.steps},
        "roofline": roofs.get("kl") or roofs.get("logp"),
        "step_tensor_util": ({"tflops_per_gpu": FLOP_PER_SAMPLE[wl_name] * value / world / 1e12, "peak_tflops": tf_peak,
                              "frac": FLOP_PER_SAMPLE[wl_name] * value / world / 1e12 / tf_peak} if wl_name in FLOP_PER_SAMPLE else None),
        "final_loss": final_loss,
        "peak_memory_gb": torch.cuda.max_memory_allocated() / 2 ** 30,
    }
    if "kl" in roofs and "logp" in roofs:
        line["roofline_logp"] = roofs["logp"]
    # ---- secondary: BASELINE configs 3 / 4 in this process after the headline, config 5 from its own process (measured first) ----
    if wl_name == HEADLINE and not args.no_secondary:
        sec = secondary(args, job, teacher, student, rank, world, dev, barrier, reduce_max, hbm_peak, tf_peak, src)
        sec.update(sec5)
        line["secondary"] = sec
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    if world == 1 and not args.no_cpu_baseline and wl["kind"] == "mimic":
        threads = pick_threads(wl_name)
        s, frac, desc, parts = cpu_step_sample(wl_name, threads)
        line["cpu_baseline"] = {"value": frac / s, "unit": "samples/s", "cores": threads, "kind": "port", "sample": desc, "estimated": True,
                                "seconds_spent": s, "parts_s": parts}
    print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


def secondary(args, job, teacher, student, rank, world, dev, barrier, reduce_max, hbm_peak, tf_peak, src):
    """BASELINE configs 3 and 4 measured with the same rules (CUDA events, barrier both sides, max over ranks).  Each entry is
    independent: a failure is recorded in place and the headline line is still printed."""
    from llavamod import _C
    out = {}
    # config 3: the headline workload at GLOBAL batch 256 (256 / N micro-batches per GPU per optimizer step); graphs are warm
    try:
        gb = 256
        acc3 = max(1, gb // world)
        tr = job.trainers["mimic"]
        old = (tr.args.gradient_accumulation_steps, job.accum, job.units_per_step)
        tr.args.gradient_accumulation_steps, job.accum, job.units_per_step = acc3, acc3, acc3
        tr._accum = 0
        ms3, _ = timed_steps(job, 1, barrier)
        (ms3,) = reduce_max(ms3)
        out["config3_global_batch_256"] = {"workload": HEADLINE, "global_batch": acc3 * world, "grad_accum": acc3, "steps": 1, "ms_per_step": ms3,
                                            "value": acc3 * world / (ms3 / 1e3), "unit": "samples/s", "n_gpus": world}
        tr.args.gradient_accumulation_steps, job.accum, job.units_per_step = old
        tr._accum = 0
    except Exception as e:          # noqa: BLE001
        out["config3_global_batch_256"] = {"error": "%s: %s" % (type(e).__name__, e)}
    # config 4: preference stage, same models, same optimizer arenas.  preference_distillation.sh trains the same modules (+ the
    # `deepspeed_experts` substring, which names the same expert weights)
    try:
        name4 = "preference-0.5B-4E-from-7B-seq2048"
        j4 = Job(name4, student, teacher, WORKLOADS[name4]["accum"], rank, world, dev, optimizer=job.optimizer, n_batches=8)
        j4.run(2)
        _C.launch_count_reset(); j4.reset_counters()
        steps4 = 3
        ms4, last4 = timed_steps(j4, steps4, barrier)
        l4 = _C.launch_count() + j4.replayed()
        roofs4 = kernel_rooflines(j4, hbm_peak, src)
        (ms4,) = reduce_max(ms4)
        pairs = steps4 * j4.accum * world
        v4 = pairs / (ms4 / 1e3)
        out["config4_preference"] = {"workload": name4, "config": our_config(name4, j4.accum, world), "steps": steps4, "warmup": 2,
                                     "ms_per_step": ms4 / steps4, "value": v4, "unit": "pairs/s", "n_gpus": world, "gpu_launches": l4,
                                     "final_loss": float(last4), "roofline": roofs4.get("logp"),
                                     "cuda_graphs": any(("graph" in e) for e in j4.trainers["dpo"]._graphs.values()),
                                     "step_tensor_util": {"tflops_per_gpu": FLOP_PER_SAMPLE[name4] * v4 / world / 1e12, "peak_tflops": tf_peak,
                                                          "frac": FLOP_PER_SAMPLE[name4] * v4 / world / 1e12 / tf_peak}}
        del j4
    except Exception as e:          # noqa: BLE001
        out["config4_preference"] = {"error": "%s: %s" % (type(e).__name__, e)}
    return out


CONFIG5 = "mimic+pref-1.8B-4E-from-7B-seq2048"


def config5_child(world, rank):
    """BASELINE config 5 measured by a child `bench.py --workload CONFIG5` (same rules: CUDA events, barrier both sides, max over ranks);
    with N ranks every rank starts its own child and the children form their own process group.  Returns the `secondary` entry."""
    key = "config5_mimic+pref_1.8B-4E_seq2048"
    acc5, steps5 = 2, 2
    cmd = [sys.executable, os.path.abspath(__file__), "--workload", CONFIG5, "--accum", str(acc5), "--steps", str(steps5), "--warmup", "2",
           "--min-warmup", "2", "--no-secondary", "--no-cpu-baseline", "--no-e2e"]
    env = dict(os.environ, LLAVAMOD_CUDA_GRAPHS="0")        # eager: see the module docstring
    if world > 1:
        env["MASTER_PORT"] = str(int(env.get("MASTER_PORT", "29500")) + 1)
    try:
        r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=3600)
    except subprocess.TimeoutExpired:
        return {key: {"error": "config 5 child timed out"}}
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or (rank == 0 and not lines):
        return {key: {"error": "config 5 child exited %d: %s" % (r.returncode, r.stderr[-3000:])}}
    if not lines:
        return {}
    d = json.loads(lines[-1])
    return {key: {"workload": CONFIG5, "config": d["config"], "steps": d["steps"], "warmup": d["warmup"], "ms_per_step": d["ms_per_step"],
                  "value": d["value"], "unit": "samples/s (mimic samples + preference pairs)", "n_gpus": d["n_gpus"],
                  "gpu_launches": d["gpu_launches"], "final_loss": d["final_loss"], "roofline_kl": d.get("roofline"),
                  "roofline_logp": d.get("roofline_logp"), "peak_memory_gb": d.get("peak_memory_gb"), "process": "own",
                  "cuda_graphs": d["implementation"]["cuda_graphs"],
                  "note": "grad_accum 2 (a step = 2 mimic micro-batches + optimizer step + 2 preference pairs + optimizer step) to keep the "
                          "bench short; per-sample cost does not depend on the accumulation count"}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default=HEADLINE, choices=sorted(WORKLOADS))
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-secondary", action="store_true", help="skip the config 3 / 4 / 5 block")
    ap.add_argument("--no-e2e", action="store_true", help="profiling aid: skip the host-buffer leg")
    ap.add_argument("--accum", type=int, default=None, help="profiling aid: override gradient accumulation (micro-batches per step)")
    ap.add_argument("--min-warmup", type=int, default=3)
    ap.add_argument("--torch-profile", default=None, help="profiling aid: write a per-kernel device-time table of one step to this file")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR", help="write what the last timed step computed to DIR/<name>.npy")
    args = ap.parse_args()
    args.warmup = max(args.warmup, args.min_warmup) if args.impl == "ours" else args.warmup
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
