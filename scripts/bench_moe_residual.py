#!/usr/bin/env python
"""Step time and peak memory of a Residual-MoE student (--use_residual True) against the plain top-2 student on the headline mimic
workload (BASELINE config 2: 0.5B-4E student distilled from the 7B teacher, 2048 positions, 8 micro-batches per step, CUDA graphs on), and
the two mix kernels alone at S = 2048, H = 1024.

    python scripts/bench_moe_residual.py [--steps 3] [--warmup 3] [--rounds 3] [--accum N] [--out FILE]

The two students share one teacher and run in the same process, alternating round by round; each round times `--steps` optimizer steps
with CUDA events, and the reported figure is the median over the rounds (every round is printed too).  Memory is, per student, what torch allocated
for it above the shared teacher: resident after its warm-up steps (weights, gradient and optimizer arenas, captured graphs) and the
peak while it was built and warmed up.  The kernel figures are CUDA-event medians after a warm-up, with the bytes each kernel must
move computed from the shapes and set against the H100 SXM data-sheet bandwidth (3.35 TB/s).  Prints one JSON line with the card's name
and power limit.  The residual student runs one more dense MLP forward and backward per MoE layer (12 at config 2)."""
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

DATASHEET_BW = 3.35e12          # bytes/s, H100 SXM5 80 GB data sheet (HBM3)


def card():
    name = torch.cuda.get_device_name()
    try:
        p = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(p.splitlines()[0])
    except Exception:                                  # noqa: BLE001 -- the power limit is reported when it can be read
        power = None
    return name, power


def _time(fn, reps=200, rounds=5):
    for _ in range(20):
        fn()
    out = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) * 1e3 / reps)
    return statistics.median(out)


def time_mix(S=2048, H=1024):
    from llavamod import kernels as K
    g = torch.Generator(device="cuda").manual_seed(0)
    x, moe, mlp, res, gr = (torch.randn(S, H, device="cuda", generator=g).to(torch.bfloat16) for _ in range(5))
    wc = (torch.randn(2, H, device="cuda", generator=g) * 0.03).to(torch.bfloat16)
    bc = torch.zeros(2, device="cuda", dtype=torch.bfloat16)
    dwc, dbc = torch.zeros_like(wc), torch.zeros_like(bc)
    _, coef = K.moe_residual_mix(x, moe, mlp, res, wc, bc)
    fwd = _time(lambda: K.moe_residual_mix(x, moe, mlp, res, wc, bc))
    bwd = _time(lambda: K.moe_residual_mix_bwd(gr, x, moe, mlp, coef, wc, dwc, dbc))
    t = S * H * 2
    fwd_bytes = 5 * t                              # reads x, moe, mlp, res; writes the stream
    bwd_bytes = 7 * t                              # reads g, moe, mlp and x (coefficient gradient); writes d_moe, d_mlp, the dx term
    return dict(S=S, H=H, fwd_us=fwd, bwd_us=bwd, fwd_bytes=fwd_bytes, bwd_bytes=bwd_bytes,
                fwd_TBps=fwd_bytes / fwd / 1e6, bwd_TBps=bwd_bytes / bwd / 1e6,
                fwd_of_datasheet=fwd_bytes / (fwd * 1e-6) / DATASHEET_BW, bwd_of_datasheet=bwd_bytes / (bwd * 1e-6) / DATASHEET_BW)


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
    jobs, resident, peak = {}, {}, {}
    for name, residual in (("top2", False), ("residual", True)):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        student = S.make_student(wl["student"], wl["clip"], device=dev, seed=1,
                                 margs=S.moe_args(num_experts=wl["experts"], train_modules=S.TRAIN_MODULES, use_residual=residual),
                                 share_tower_with=teacher)
        jobs[name] = bench.Job(bench.HEADLINE, student, teacher, accum, 0, 1, dev)
        jobs[name].run(args.warmup)
        torch.cuda.synchronize()
        resident[name] = torch.cuda.memory_allocated(dev) - base
        peak[name] = torch.cuda.max_memory_allocated(dev) - base
    ms = {n: [] for n in jobs}
    for _ in range(args.rounds):
        for n, job in jobs.items():
            t, last = bench.timed_steps(job, args.steps, torch.cuda.synchronize)
            ms[n].append(t / args.steps)
            assert float(last) == float(last), "non-finite loss"
    step = {n: statistics.median(v) for n, v in ms.items()}
    name, power = card()
    res = dict(workload=bench.HEADLINE, accum=accum, steps=args.steps, rounds=args.rounds, gpu=name, power_limit_w=power,
               step_ms=step, step_ms_rounds=ms, steps_per_s={n: 1e3 / v for n, v in step.items()},
               residual_over_top2_step_time=step["residual"] / step["top2"],
               student_resident_GiB={n: v / 2 ** 30 for n, v in resident.items()}, student_peak_GiB={n: v / 2 ** 30 for n, v in peak.items()}, mix_kernels=time_mix(), datasheet_bw_TBps=DATASHEET_BW / 1e12)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
