#!/usr/bin/env python
"""A/B two or more prebuilt kernel libraries in one process tree on one GPU.

    python scripts/ab_lib.py --arm parent=ab_libs/parent.so --arm branch=ab_libs/branch.so \
        [--arm fuse1=ab_libs/branch.so,LLAVAMOD_FUSE_SWIGLU=1 ...] [--runs 3] [--detail parent,branch [--reports] [--full]] --out DIR

An arm is NAME=LIB[,VAR=VALUE...]: the library is copied over llavamod/liblmod_b200.so while the arm runs (the original is put back at
the end), and the variables are set in the arm's child processes.  Build each library beforehand with llava-mod_b200/build_ext.py from
the sources it stands for, and keep it in an ignored directory (ab_libs/).  For every arm the script

  * runs the GEMM in every epilogue form at the teacher's shapes (and the teacher lm_head on 1229 compact rows), the grouped expert
    GEMM and the attention forward (hd 64 / 128, causal and padded) on seeded inputs, writes the outputs as .npy and times each call
    with CUDA events, next to the same dense product through torch.mm (`<case>_torch_mm`);
  * runs `bench.py --no-secondary --no-cpu-baseline` --runs times, the arms alternating, the first run also with --dump-outputs;
  * for the arms named in --detail: with --reports the GEMM and attention throughput reports of the test suite and one
    `bench.py --torch-profile` run, with --full one `bench.py --no-cpu-baseline` run (the headline and configs 3, 4 and 5).

It then compares the outputs of every arm byte for byte with the first arm's and writes DIR/ab.json (plus the logs and profiles).
The card's name, power limit and maximum SM clock are recorded in the same process.
"""
import argparse
import hashlib
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "llava-mod_b200")
LIB = os.path.join(PKG, "llavamod", "liblmod_b200.so")


# ---------------------------------------------------------------------------------------------------------------------------------
# child: seeded kernel outputs of one library
# ---------------------------------------------------------------------------------------------------------------------------------
def dump_kernels(out_dir):
    import numpy as np
    import torch
    sys.path.insert(0, PKG)
    from llavamod import kernels as K
    os.makedirs(out_dir, exist_ok=True)
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    times = {}

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, device=dev, generator=g) * scale).to(torch.bfloat16)

    def timed(fn):
        for _ in range(2):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 10

    def case(name, fn, dump=True, mm=None):
        """mm: the same product through torch.mm (cuBLAS), timed as name + "_torch_mm" for the fraction of cuBLAS"""
        out = fn()
        torch.cuda.synchronize()
        outs = out if isinstance(out, tuple) else (out,)
        for i, o in enumerate(x for x in outs if x is not None and dump):
            a = o.detach().contiguous().cpu()
            a = a.view(torch.int16).numpy() if a.dtype == torch.bfloat16 else a.numpy()
            np.save(os.path.join(out_dir, "%s%s.npy" % (name, "" if i == 0 else "_%d" % i)), a)
        times[name] = timed(fn)
        if mm is not None:
            times[name + "_torch_mm"] = timed(mm)

    M = 2048
    # teacher (qwen1.5-7b): H 4096, I 11008, 32 heads of 128
    H, I, nh, hd = 4096, 11008, 32, 128
    x, w_qkv, b_qkv = rnd(M, H), rnd(3 * H, H, scale=H ** -0.5), rnd(3 * H, scale=0.1)
    pos = torch.arange(M, device=dev, dtype=torch.int64)
    ang = torch.arange(M, device=dev).float()[:, None] * (1e6 ** (-torch.arange(0, hd, 2, device=dev).float() / hd))[None]
    ang = torch.cat([ang, ang], 1)
    cos, sin = ang.cos().to(torch.bfloat16), ang.sin().to(torch.bfloat16)
    w_o, w_gu, w_dn = rnd(H, H, scale=H ** -0.5), rnd(2 * I, H, scale=H ** -0.5), rnd(H, I, scale=I ** -0.5)
    res, act = rnd(M, H), rnd(M, I)
    dy, h1 = rnd(M, H), rnd(M, 2 * I)
    with torch.no_grad():
        case("teacher_plain_MxNxK_2048x4096x4096", lambda: K.gemm(x, w_o), mm=lambda: torch.mm(x, w_o.t()))
        case("teacher_bias_2048x12288x4096", lambda: K.gemm(x, w_qkv, bias=b_qkv), mm=lambda: torch.mm(x, w_qkv.t()))
        case("teacher_qkv_rope_2048x12288x4096", lambda: K.qkv_rope(x, w_qkv, b_qkv, cos, sin, pos, nh, nh, hd))
        case("teacher_swiglu_2048x22016x4096", lambda: K.gemm_swiglu(x, w_gu, True), mm=lambda: torch.mm(x, w_gu.t()))
        case("teacher_residual_2048x4096x11008", lambda: K.gemm_residual(act, w_dn, None, res))
        case("teacher_down_2048x4096x11008", lambda: K.gemm(act, w_dn), mm=lambda: torch.mm(act, w_dn.t()))
        case("teacher_silu_bwd_2048x11008x4096", lambda: K.gemm_silu_bwd(dy, w_dn, h1), mm=lambda: torch.mm(dy, w_dn))
        case("teacher_dgrad_2048x4096x4096", lambda: K.mm_nn(dy, w_o), mm=lambda: torch.mm(dy, w_o))
        case("teacher_wgrad_4096x4096x2048", lambda: K.gemm(dy, x, a_mn=True, b_mn=True), mm=lambda: torch.mm(dy.t(), x))
        # a ragged M: an odd number of 128-row tiles, the last one partial
        case("odd_m_tiles_1282x4096x4096", lambda: K.gemm(x[:1282], w_o), mm=lambda: torch.mm(x[:1282], w_o.t()))
        # teacher lm_head on the supervised rows of a compact batch: 1229 of 2048 rows, row count read from device memory
        w_lmt = rnd(151936, H, scale=0.02)
        cnt = torch.tensor([1229], device=dev, dtype=torch.int32)
        lm_out = torch.zeros(M, 151936, device=dev, dtype=torch.bfloat16)
        case("teacher_lm_head_1229x151936x4096", lambda: K.gemm(x, w_lmt, out=lm_out, m_dev=cnt), dump=False,
             mm=lambda: torch.mm(x[:1229], w_lmt.t()))
        # the full output is 622 MB: the first rows and the last supervised ones are compared
        np.save(os.path.join(out_dir, "teacher_lm_head_rows_0_64.npy"), lm_out[:64].cpu().view(torch.int16).numpy())
        np.save(os.path.join(out_dir, "teacher_lm_head_rows_1165_1229.npy"), lm_out[1165:1229].cpu().view(torch.int16).numpy())
        del w_lmt, lm_out
        # student (qwen1.5-0.5b): H 1024, I 2816, 16 heads of 64; the experts' grouped GEMM on 4 groups of compact rows
        Hs, Is = 1024, 2816
        xs, w_s, w_gus = rnd(M, Hs), rnd(3 * Hs, Hs, scale=Hs ** -0.5), rnd(2 * Is, Hs, scale=Hs ** -0.5)
        dys = rnd(M, 3 * Hs)
        case("student_plain_2048x3072x1024", lambda: K.gemm(xs, w_s), mm=lambda: torch.mm(xs, w_s.t()))
        case("student_plain_2048x1024x1024", lambda: K.gemm(xs, w_s[:Hs]), mm=lambda: torch.mm(xs, w_s[:Hs].t()))
        case("student_swiglu_2048x5632x1024", lambda: K.gemm_swiglu(xs, w_gus, True), mm=lambda: torch.mm(xs, w_gus.t()))
        case("student_wgrad_3072x1024x2048", lambda: K.gemm(dys, xs, a_mn=True, b_mn=True), mm=lambda: torch.mm(dys.t(), xs))
        w_lm = rnd(151936, Hs, scale=0.02)
        case("student_lm_head_2048x151936x1024", lambda: K.gemm(xs, w_lm), dump=False,    # timed only: a 622 MB output
             mm=lambda: torch.mm(xs, w_lm.t()))
        del w_lm
        E, R = 4, 4096
        offsets = torch.tensor([0, 1152, 2048, 3200, 4096], device=dev, dtype=torch.int32)
        xe, dye = rnd(R, Hs), rnd(R, Hs)
        w_gue, w_dne = rnd(E, 2 * Is, Hs, scale=Hs ** -0.5), rnd(E, Hs, Is, scale=Is ** -0.5)
        acte = rnd(R, Is)
        case("grouped_fwd_4x1024x2816", lambda: K.grouped_gemm(acte, w_dne, torch.empty(R, Hs, device=dev, dtype=torch.bfloat16), offsets, 0))
        case("grouped_dgrad_4x2816x1024", lambda: K.grouped_gemm(dye, w_dne, torch.empty(R, Is, device=dev, dtype=torch.bfloat16), offsets, 1))
        case("grouped_wgrad_4x1024x2816", lambda: K.grouped_gemm(dye, acte, torch.zeros(E, Hs, Is, device=dev, dtype=torch.bfloat16), offsets, 2))
        dwe = torch.zeros(E, Hs, Is, device=dev, dtype=torch.bfloat16)
        case("grouped_wgrad_accumulate_4x1024x2816", lambda: K.grouped_gemm(dye, acte, dwe, offsets, 2, accumulate=True), dump=False)
        case("grouped_swiglu_4x5632x1024", lambda: K.grouped_gemm_swiglu(xe, w_gue, offsets, R, True))
        # attention forward: teacher heads (hd 128) and student heads (hd 64), causal; a padded batch of two
        for hdx, nhx in ((128, 32), (64, 16)):
            qkv = rnd(M, 3 * nhx * hdx)
            case("attn_fwd_hd%d_causal" % hdx, lambda: K.attention_fwd(qkv, 1, M, nhx, nhx, hdx, True, need_lse=True))
            qkv2 = rnd(2 * M, 3 * nhx * hdx)
            lo = torch.tensor([0, 300], device=dev, dtype=torch.int32)
            hi = torch.tensor([M, M], device=dev, dtype=torch.int32)
            case("attn_fwd_hd%d_padded" % hdx, lambda: K.attention_fwd(qkv2, 2, M, nhx, nhx, hdx, True, need_lse=True, pad=(lo, hi)))
    with open(os.path.join(out_dir, "times_ms.json"), "w") as f:
        json.dump(times, f, indent=1)


# ---------------------------------------------------------------------------------------------------------------------------------
# parent: arms, alternating runs, comparison
# ---------------------------------------------------------------------------------------------------------------------------------
def parse_arm(s):
    name, rest = s.split("=", 1)
    parts = rest.split(",")
    env = dict(p.split("=", 1) for p in parts[1:])
    return {"name": name, "lib": os.path.abspath(parts[0]), "env": env}


def run(cmd, env, log, timeout=3600):
    t0 = time.time()
    r = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ, **env), capture_output=True, text=True, timeout=timeout)
    with open(log, "w") as f:
        f.write("$ %s\n# exit %d, %.0f s\n%s\n---- stderr ----\n%s" % (" ".join(cmd), r.returncode, time.time() - t0, r.stdout, r.stderr))
    return r


def json_line(stdout):
    lines = [ln for ln in stdout.splitlines() if ln.startswith("{")]
    return json.loads(lines[-1]) if lines else None


def gpu_info():
    q = "name,power.limit,clocks.max.sm,driver_version"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    except OSError as e:
        return {"error": str(e)}
    return dict(zip(q.split(","), [x.strip() for x in r.stdout.splitlines()[0].split(",")])) if r.returncode == 0 and r.stdout else {"error": r.stderr}


def compare(dir_a, dir_b):
    import numpy as np
    out = {}
    for f in sorted(os.listdir(dir_a)):
        if not f.endswith(".npy"):
            continue
        pb = os.path.join(dir_b, f)
        if not os.path.exists(pb):
            out[f] = "missing"
            continue
        ba, bb = open(os.path.join(dir_a, f), "rb").read(), open(pb, "rb").read()
        if ba == bb:
            out[f] = "identical"
            continue
        a, b = np.load(os.path.join(dir_a, f)), np.load(pb)
        if a.dtype == np.int16:               # bf16 stored as its bits
            a = (a.astype(np.int32) << 16).view(np.float32)
            b = (b.astype(np.int32) << 16).view(np.float32)
        d = np.abs(a.astype(np.float64) - b.astype(np.float64))
        out[f] = {"max_abs_diff": float(np.nanmax(d)), "differing": int((d > 0).sum()), "of": int(d.size),
                  "max_abs_ref": float(np.nanmax(np.abs(a.astype(np.float64))))}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arm", action="append", default=[], help="NAME=LIB[,VAR=VALUE...]; the first arm is the base of the comparisons")
    ap.add_argument("--runs", type=int, default=3, help="bench.py runs per arm, arms alternating")
    ap.add_argument("--detail", default="", help="comma-separated arms that get --reports and --full")
    ap.add_argument("--reports", action="store_true", help="the throughput reports of the test suite and a torch profile per --detail arm")
    ap.add_argument("--full", action="store_true", help="one bench.py run with configs 3, 4 and 5 per --detail arm")
    ap.add_argument("--out", required=True)
    ap.add_argument("--dumps", default=None, help="where the .npy outputs go (default: a temporary directory)")
    ap.add_argument("--dump-kernels", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.dump_kernels:
        dump_kernels(args.dump_kernels)
        return
    arms = [parse_arm(a) for a in args.arm]
    assert len(arms) >= 2 and len({a["name"] for a in arms}) == len(arms), "give at least two arms with distinct names"
    for a in arms:
        assert os.path.isfile(a["lib"]), a["lib"]
    detail = [d for d in args.detail.split(",") if d]
    os.makedirs(args.out, exist_ok=True)
    logs = os.path.join(args.out, "logs")
    os.makedirs(logs, exist_ok=True)
    dumps = args.dumps or tempfile.mkdtemp(prefix="ab_dumps_")
    report = {"gpu": gpu_info(), "arms": {a["name"]: {"lib": os.path.relpath(a["lib"], ROOT), "env": a["env"],
                                                       "lib_sha256": hashlib.sha256(open(a["lib"], "rb").read()).hexdigest()} for a in arms}}
    path = os.path.join(args.out, "ab.json")

    def save():
        with open(path, "w") as f:
            json.dump(report, f, indent=1)

    backup = LIB + ".ab_backup"
    had_lib = os.path.exists(LIB)
    if had_lib:
        shutil.copy2(LIB, backup)
    py = sys.executable
    try:
        def use(arm):
            shutil.copyfile(arm["lib"], LIB)

        # seeded kernel outputs and per-call times; an arm whose kernels fail is dropped from the runs
        live = []
        for a in arms:
            use(a)
            d = os.path.join(dumps, a["name"])
            r = run([py, os.path.abspath(__file__), "--dump-kernels", d, "--out", args.out], a["env"], os.path.join(logs, "kernels_%s.log" % a["name"]))
            rep = report["arms"][a["name"]]
            rep["kernels_exit"] = r.returncode
            if r.returncode == 0:
                rep["kernel_ms"] = json.load(open(os.path.join(d, "times_ms.json")))
                live.append(a)
            save()
        # step-level runs, arms alternating
        for i in range(args.runs):
            for a in live:
                use(a)
                cmd = [py, "bench.py", "--no-secondary", "--no-cpu-baseline"]
                if i == 0:
                    cmd += ["--dump-outputs", os.path.join(dumps, a["name"], "bench")]
                r = run(cmd, a["env"], os.path.join(logs, "bench_%s_%d.log" % (a["name"], i)))
                line = json_line(r.stdout)
                rep = report["arms"][a["name"]]
                rep.setdefault("runs", []).append({"value": line["value"], "ms_per_step": line["ms_per_step"], "clocks": line.get("clocks"),
                                                   "final_loss": line["final_loss"]} if (r.returncode == 0 and line) else {"exit": r.returncode})
                vals = [x["value"] for x in rep["runs"] if "value" in x]
                if vals:
                    rep["value_median"], rep["value_min"], rep["value_max"] = statistics.median(vals), min(vals), max(vals)
                save()
        for a in live:
            if a["name"] not in detail:
                continue
            use(a)
            rep = report["arms"][a["name"]]
            if args.reports:
                r = run([py, "-m", "pytest", "-q", "-s", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gemm_gpu.py::test_gemm_throughput_report",
                         "tests/test_attn_gpu.py::test_attn_throughput_report", "tests/test_attn_gpu.py::test_attn_bwd_throughput_report"],
                        a["env"], os.path.join(logs, "throughput_%s.log" % a["name"]))
                rep["throughput_reports"] = [ln for ln in r.stdout.splitlines() if "TFLOP/s" in ln]
                prof = os.path.join(os.path.abspath(args.out), "profile_%s.txt" % a["name"])
                r = run([py, "bench.py", "--no-secondary", "--no-cpu-baseline", "--torch-profile", prof], a["env"],
                        os.path.join(logs, "profile_%s.log" % a["name"]))
                rep["profile_exit"] = r.returncode
            if args.full:
                r = run([py, "bench.py", "--no-cpu-baseline"], a["env"], os.path.join(logs, "full_%s.log" % a["name"]))
                line = json_line(r.stdout)
                rep["full"] = {"exit": r.returncode, "value": line and line.get("value"), "secondary": line and line.get("secondary")}
            save()
        base = arms[0]["name"]
        for a in live[1:]:
            if base in [x["name"] for x in live]:
                rep = report["arms"][a["name"]]
                rep["vs_" + base] = compare(os.path.join(dumps, base), os.path.join(dumps, a["name"]))
                bd = os.path.join(dumps, base, "bench")
                if os.path.isdir(bd) and os.path.isdir(os.path.join(dumps, a["name"], "bench")):
                    rep["bench_outputs_vs_" + base] = compare(bd, os.path.join(dumps, a["name"], "bench"))
        save()
    finally:
        if had_lib:
            shutil.move(backup, LIB)
        if not args.dumps:
            shutil.rmtree(dumps, ignore_errors=True)
    for name, rep in report["arms"].items():
        print(name, {k: rep.get(k) for k in ("value_median", "value_min", "value_max")})
    print("wrote", path)


if __name__ == "__main__":
    main()
