#!/usr/bin/env python
"""Step rate of a top-1 sparse student (--top_k_experts 1) against the top-2 one on the headline mimic workload (BASELINE config 2:
0.5B-4E student distilled from the 7B teacher, 2048 positions, 8 micro-batches per step, CUDA graphs on), and the router's launches
at S = 2048, E = 4, H = 1024.

    python scripts/bench_moe_top1.py [--steps 3] [--warmup 3] [--rounds 3] [--accum N] [--out FILE]

The two students share one teacher and run in the same process, alternating round by round; each round times `--steps` optimizer steps
with CUDA events, and the reported figure is the median over the rounds.  Prints one JSON line with the card's name and power limit.
Top-1 gives the expert GEMMs at most S rows instead of 2S (C = ceil(S/E * cf) instead of ceil(S/E * cf * 2)) and adds one launch (the
random token selection) to every MoE layer's router."""
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


def card():
    name = torch.cuda.get_device_name()
    try:
        p = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(p.splitlines()[0])
    except Exception:                                  # noqa: BLE001 -- the power limit is reported when it can be read
        power = None
    return name, power


def time_router(k, reps=200, rounds=5):
    from llavamod import kernels as K
    S, H, E = 2048, 1024, 4
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(S, H, device="cuda", generator=g).to(torch.bfloat16)
    wg = torch.randn(E, H, device="cuda", generator=g) * 0.02
    noise = torch.rand(S, E, device="cuda", generator=g) if k == 1 else -torch.log(-torch.log(torch.rand(S, E, device="cuda", generator=g)))
    for _ in range(10):
        K.moe_route_scatter(x, wg, noise, 1.5, 0, K.LAYOUT_ALIGNED, k=k)
    out = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            K.moe_route_scatter(x, wg, noise, 1.5, 0, K.LAYOUT_ALIGNED, k=k)
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) * 1e3 / reps)
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--accum", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from llavamod.model import synthetic as S
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.manual_seed(0)
    wl = bench.WORKLOADS[bench.HEADLINE]
    accum = args.accum or wl["accum"]
    teacher = S.make_teacher(wl["teacher"], wl["clip"], device=dev, seed=0)
    jobs = {}
    for k in (2, 1):
        student = S.make_student(wl["student"], wl["clip"], device=dev, seed=1,
                                 margs=S.moe_args(num_experts=wl["experts"], train_modules=S.TRAIN_MODULES, top_k=k), share_tower_with=teacher)
        jobs[k] = bench.Job(bench.HEADLINE, student, teacher, accum, 0, 1, dev)
    for k, job in jobs.items():
        job.run(args.warmup)
    torch.cuda.synchronize()
    ms = {1: [], 2: []}
    for _ in range(args.rounds):
        for k, job in jobs.items():
            t, last = bench.timed_steps(job, args.steps, torch.cuda.synchronize)
            ms[k].append(t / args.steps)
            assert float(last) == float(last), "non-finite loss"
    step = {k: statistics.median(v) for k, v in ms.items()}
    router = {k: time_router(k) for k in (2, 1)}
    name, power = card()
    res = dict(workload=bench.HEADLINE, accum=accum, steps=args.steps, rounds=args.rounds, gpu=name, power_limit_w=power,
               step_ms={"top2": step[2], "top1": step[1]}, step_ms_rounds={"top2": ms[2], "top1": ms[1]},
               steps_per_s={"top2": 1e3 / step[2], "top1": 1e3 / step[1]}, top1_over_top2_step_rate=step[2] / step[1],
               router_us_S2048_E4_H1024={"top2": router[2], "top1": router[1]})
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
