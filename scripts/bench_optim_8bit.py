#!/usr/bin/env python
"""8-bit block-wise AdamW state (``--optim adamw_bnb_8bit``) against the fp32 moments, on the H100.

    python scripts/bench_optim_8bit.py [--steps 3] [--warmup 3] [--rounds 3] [--opt-reps 20] [--out FILE]

1. The optimizer step alone (gradient sum of squares + one AdamW launch per group slice) on the 0.5B-4E student's arenas, 32-bit and
   8-bit alternating, CUDA events; the bytes each pass must move (counted from the layout) over its time, against 3.35 TB/s.
2. The config-2 step (0.5B-4E <- 7B mimic, T' = 2048, 8 micro-batches, CUDA graphs on) with each optimizer: both students share the
   teacher in one process and alternate round by round, as scripts/bench_moe_top1.py does.
3. Peak device memory after warm-up, config 2 and config 5 (1.8B-4E <- 7B, T' = 4096), each optimizer in a child process of its own.
4. A 1.8B-8E <- 7B mimic step at T' = 2048 with 8-bit state in a child process: peak memory and samples/s, only when enough device
   memory is free (the fp32-state run is never attempted: its arena size is printed from the counted bytes).
Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "llava-mod_b200"))

import torch  # noqa: E402

import bench  # noqa: E402

HBM_BYTES_PER_S = 3.35e12            # H100 SXM data sheet


def card():
    name = torch.cuda.get_device_name()
    try:
        p = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(p.splitlines()[0])
    except Exception:                                  # noqa: BLE001 -- the power limit is reported when it can be read
        power = None
    return name, power


def make_state(student, bits):
    from llavamod.train.engine import TrainState
    return TrainState(student, lr=2e-5, weight_decay=0.0, max_grad_norm=1.0, optim_bits=bits)


def pass_bytes(ts):
    """Bytes one optimizer step must move over HBM: the sumsq read of the gradients, then per element of the bf16 arena the gradient,
    the master (read + write), the bf16 weight (write) and the moments (fp32 m, v read + write, or the two codes read + write, plus two
    scales per block read + write); the fp32 arena likewise with fp32 gradients and no bf16 copy."""
    n16, n32 = ts.n16, ts.n32
    b = 2 * n16 + 4 * n32                                        # sumsq
    b += n16 * (2 + 8 + 2) + n32 * (4 + 8 + 16)
    if ts.optim_bits == 8:
        b += n16 * 4 + 2 * ts.absmax.numel() * 4
    else:
        b += n16 * 16
    return b


def time_optimizer(states, reps, rounds):
    for ts in states.values():
        ts.g16.normal_(0, 1e-2)
        if ts.n32:
            ts.g32.normal_(0, 1e-2)
        for _ in range(3):
            ts.grads_reduced = True
            ts.step()
    torch.cuda.synchronize()
    ms = {k: [] for k in states}
    for _ in range(rounds):
        for k, ts in states.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                ts.grads_reduced = True                          # time sumsq + the AdamW launches, not the (single-GPU no-op) all-reduce
                ts.step()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / reps)
    return {k: statistics.median(v) for k, v in ms.items()}, ms


def student_of(wl, experts, teacher, dev):
    from llavamod.model import synthetic as S
    return S.make_student(wl["student"], wl["clip"], device=dev, seed=1, margs=S.moe_args(num_experts=experts, train_modules=S.TRAIN_MODULES),
                          share_tower_with=teacher)


def child_peak(workload, experts, bits, seq, steps, warmup):
    """One workload with one optimizer in this (fresh) process: peak memory after warm-up and the timed step rate."""
    from llavamod.model import synthetic as S
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.manual_seed(0)
    name = "optim8-probe"
    bench.WORKLOADS[name] = dict(bench.WORKLOADS[workload], seq=seq, experts=experts)
    wl = bench.WORKLOADS[name]
    teacher = S.make_teacher(wl["teacher"], wl["clip"], device=dev, seed=0)
    student = student_of(wl, experts, teacher, dev)
    ts = make_state(student, bits)
    job = bench.Job(name, student, teacher, wl["accum"], 0, 1, dev, optimizer=ts)
    job.run(warmup)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t, last = bench.timed_steps(job, steps, torch.cuda.synchronize)
    assert float(last) == float(last), "non-finite loss"
    return dict(peak_gb=torch.cuda.max_memory_allocated() / 1e9, step_ms=t / steps, samples_per_s=wl["accum"] * steps / (t / 1e3),
                trainable=ts.num_trainable, state_gb=ts.state_bytes() / 1e9)


def run_child(args, workload, experts, bits, seq):
    cmd = [sys.executable, os.path.abspath(__file__), "--child", workload, str(experts), str(bits), str(seq), "--steps", str(args.steps),
           "--warmup", str(args.warmup)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    if r.returncode != 0 or not lines:
        return {"error": (r.stderr or r.stdout).strip().splitlines()[-1:] or ["exit %d" % r.returncode]}
    return json.loads(lines[-1])


def counted_arena_gb(wl_student, experts, bits):
    """Optimizer state and whole arena (state + bf16 weight + gradient) of a student under --train_modules mlp.gate_proj mlp.up_proj
    mlp.down_proj wg, counted from its shapes (nothing is allocated): 3 H I per expert in every other layer (the MoE layers), 3 H I per
    dense MLP in the rest, the router wg (E H, fp32) per MoE layer.  One decay group."""
    from llavamod.model import synthetic as S
    from llavamod.train.engine import state_bytes
    c = S.ARCH[wl_student]
    H, I, L = c["hidden_size"], c["intermediate_size"], c["num_hidden_layers"]
    moe = L // 2
    n16 = moe * experts * 3 * H * I + (L - moe) * 3 * H * I
    n32 = moe * experts * H
    sb = state_bytes([n16], n16, n32, bits)
    return dict(trainable=n16 + n32, state_gb=sb / 1e9, arena_gb=(sb + 4 * n16 + 8 * n32) / 1e9)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--opt-reps", type=int, default=20)
    ap.add_argument("--child", nargs=4, default=None)
    ap.add_argument("--skip-peaks", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.child:
        wl, experts, bits, seq = args.child
        print(json.dumps(child_peak(wl, int(experts), int(bits), int(seq), args.steps, args.warmup)))
        return
    from llavamod.model import synthetic as S
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.manual_seed(0)
    name, power = card()
    res = dict(gpu=name, power_limit_w=power, steps=args.steps, rounds=args.rounds)
    # 3. + 4. peaks, in child processes started before this process allocates anything
    if not args.skip_peaks:
        peaks = {}
        for label, wln, experts, seq in (("config2", bench.HEADLINE, 4, 2048), ("1.8B-4E-seq4096", "mimic-1.8B-4E-from-7B-seq4096", 4, 4096)):
            for bits in (32, 8):
                peaks["%s/%dbit" % (label, bits)] = run_child(args, wln, experts, bits, seq)
        res["peak"] = peaks
        free, _ = torch.cuda.mem_get_info()
        res["free_gb_before_1.8B-8E"] = free / 1e9
        if free >= 72e9:
            res["1.8B-8E-seq2048/8bit"] = run_child(args, "mimic-1.8B-4E-from-7B-seq4096", 8, 8, 2048)
        else:
            res["1.8B-8E-seq2048/8bit"] = "not measured: %.1f GB free" % (free / 1e9)
        res["1.8B-8E/32bit"] = dict(counted_arena_only=counted_arena_gb(bench.WORKLOADS["mimic-1.8B-4E-from-7B-seq4096"]["student"], 8, 32))
        res["1.8B-8E/8bit_counted"] = counted_arena_gb(bench.WORKLOADS["mimic-1.8B-4E-from-7B-seq4096"]["student"], 8, 8)
    wl = bench.WORKLOADS[bench.HEADLINE]
    teacher = S.make_teacher(wl["teacher"], wl["clip"], device=dev, seed=0)
    jobs, states = {}, {}
    for bits in (32, 8):
        student = student_of(wl, wl["experts"], teacher, dev)
        states[bits] = make_state(student, bits)
        jobs[bits] = bench.Job(bench.HEADLINE, student, teacher, wl["accum"], 0, 1, dev, optimizer=states[bits])
    # 1. the optimizer step alone
    opt_ms, opt_rounds = time_optimizer(states, args.opt_reps, args.rounds)
    opt = {}
    for bits, ts in states.items():
        b = pass_bytes(ts)
        opt["%dbit" % bits] = dict(ms=opt_ms[bits], ms_rounds=opt_rounds[bits], counted_bytes=b, tb_per_s=b / (opt_ms[bits] / 1e3) / 1e12,
                                   of_hbm_peak=b / (opt_ms[bits] / 1e3) / HBM_BYTES_PER_S, state_gb=ts.state_bytes() / 1e9)
    # 2. the config-2 step, alternating
    for job in jobs.values():
        job.run(args.warmup)
    torch.cuda.synchronize()
    ms = {32: [], 8: []}
    for _ in range(args.rounds):
        for bits, job in jobs.items():
            t, last = bench.timed_steps(job, args.steps, torch.cuda.synchronize)
            ms[bits].append(t / args.steps)
            assert float(last) == float(last), "non-finite loss"
    step = {b: statistics.median(v) for b, v in ms.items()}
    res.update(optimizer_step=opt,
               config2_step_ms={"32bit": step[32], "8bit": step[8]}, config2_step_ms_rounds={"32bit": ms[32], "8bit": ms[8]},
               config2_samples_per_s={"32bit": wl["accum"] * 1e3 / step[32], "8bit": wl["accum"] * 1e3 / step[8]})
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
