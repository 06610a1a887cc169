"""Decoding benchmark: tokens/s of `generate` with and without the KV cache, decode-attention bandwidth, and the device time per
kernel family of one cached decode step.

    python scripts/bench_decode.py [--models student,teacher] [--new 128,512] [--batch 1,8] [--profile] [--out DIR]

* generate: the 0.5B-4E student and the 7B teacher (random weights, CLIP-L/336) on a prompt that splices to T' = 650 positions, greedy,
  use_cache False / True, CUDA graphs on / off (LLAVAMOD_CUDA_GRAPHS).  Tokens/s = B * new tokens / wall time of the call, which ends in
  a device synchronise; one full-length warm-up call per setting, then --repeat timed calls (median, min and max).  The no-cache loop at 512 new tokens is skipped unless asked (it re-runs the
  whole prompt every token).
* attention: lmod_attn_decode alone, B = 1 and 8, lengths 1k to 32k, CUDA events over 50 launches; bytes = 2 * len * nkv * hd * 2 per
  sequence (K and V) plus q and out, against the 3.35 TB/s of the H100 SXM data sheet.
* --profile: torch.profiler over 20 graph-less decode steps of the student at B = 1, device time summed per kernel family.
The card's name and power limit are read in the same process and printed with the results (one JSON line per measurement)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "llava-mod_b200")]

import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def emit(out, rec):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(os.path.join(out, "bench_decode.jsonl"), "a") as f:
            f.write(line + "\n")


def prompt(B, seed=0):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, 150000, (B, 75), generator=g)
    ids[:, 3] = -200                                   # 74 text tokens + 576 patches = T' 650
    imgs = [torch.randn(3, 336, 336, generator=g).to(torch.bfloat16) for _ in range(B)]
    return ids, imgs


def bench_generate(model, name, B, new, use_cache, graphs, out, info, repeat):
    os.environ["LLAVAMOD_CUDA_GRAPHS"] = "1" if graphs else "0"
    ids, imgs = prompt(B)
    model.generate(ids, images=imgs, max_new_tokens=new, use_cache=use_cache, eos_token_id=-1)      # warm-up (and graph capture)
    rates = []
    for _ in range(repeat):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = model.generate(ids, images=imgs, max_new_tokens=new, use_cache=use_cache, eos_token_id=-1)
        torch.cuda.synchronize()
        rates.append(B * (res.shape[1] - ids.shape[1]) / (time.perf_counter() - t0))
    rates.sort()
    emit(out, dict(kind="generate", model=name, B=B, new=res.shape[1] - ids.shape[1], use_cache=use_cache, graphs=graphs, runs=repeat,
                   tokens_per_s=round(rates[len(rates) // 2], 1), min=round(rates[0], 1), max=round(rates[-1], 1), card=info))


def bench_attention(out, info):
    from llavamod import kernels as K
    for hd, nh, nkv in [(64, 16, 16), (64, 14, 2), (128, 28, 4), (128, 32, 32)]:
        for B in (1, 8):
            for n in (1024, 4096, 16384, 32768):
                q = torch.randn(B, nh * hd, device="cuda").to(torch.bfloat16)
                k = torch.randn(B, nkv, n, hd, device="cuda").to(torch.bfloat16)
                v = torch.randn_like(k)
                lens = torch.full((B,), n, dtype=torch.int32, device="cuda")
                ws = torch.empty(K.attn_decode_ws_elems(B, nh, nkv, hd, n), dtype=torch.float32, device="cuda")
                for _ in range(5):
                    K.attn_decode(q, nh, nkv, hd, k, v, lens, ws)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(50):
                    K.attn_decode(q, nh, nkv, hd, k, v, lens, ws)
                b.record()
                torch.cuda.synchronize()
                t = a.elapsed_time(b) / 50 * 1e-3
                nbytes = B * (2 * n * nkv * hd * 2 + 2 * nh * hd * 2)
                emit(out, dict(kind="attn_decode", hd=hd, nh=nh, nkv=nkv, B=B, len=n, us=round(t * 1e6, 2),
                               TBps=round(nbytes / t / 1e12, 3), of_peak=round(nbytes / t / HBM_BYTES_PER_S, 3), card=info))
                del q, k, v, ws


def family(name):
    n = name.lower()
    for key, fam in (("attn_decode", "attn_decode"), ("kv_append", "kv_append"), ("moe", "moe"), ("grouped", "moe"),
                     ("swiglu", "gemm"), ("gemm", "gemm"), ("rmsnorm", "rmsnorm"), ("rope", "rope"), ("silu", "elementwise"),
                     ("embedding", "embedding")):
        if key in n:
            return fam
    return "other"


def profile_step(model, name, out, info):
    from torch.profiler import ProfilerActivity, profile
    from llavamod.model.generation import next_token_logits
    os.environ["LLAVAMOD_CUDA_GRAPHS"] = "0"
    ids, imgs = prompt(1)
    cache = model.new_kv_cache(1, 1024)
    tok = torch.zeros(1, 1, dtype=torch.int64, device="cuda")
    with torch.no_grad():
        next_token_logits(model, ids, images=imgs, cache=cache)
        for _ in range(3):
            next_token_logits(model, tok, cache=cache)
        torch.cuda.synchronize()
        steps = 20
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                next_token_logits(model, tok, cache=cache)
            torch.cuda.synchronize()
    fams = {}
    for e in prof.key_averages():
        t = getattr(e, "self_device_time_total", None)           # kernels only: host ops have no self device time
        if t is None:
            t = e.self_cuda_time_total
        if t > 0:
            fams[family(e.key)] = fams.get(family(e.key), 0.0) + t / steps
    emit(out, dict(kind="step_profile", model=name, B=1, us_per_step={k: round(v, 1) for k, v in sorted(fams.items(), key=lambda kv: -kv[1])},
                   card=info))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="student,teacher")
    ap.add_argument("--new", default="128,512")
    ap.add_argument("--batch", default="1,8")
    ap.add_argument("--nocache-max-new", type=int, default=128)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--skip-generate", action="store_true")
    ap.add_argument("--skip-attention", action="store_true")
    ap.add_argument("--repeat", type=int, default=3, help="timed generate calls per setting (median, min and max are reported)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_decode.py measures on the GPU"
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    info = card()
    from llavamod.model import synthetic as S
    if not a.skip_attention and not a.profile:
        bench_attention(a.out, info)
    for name in a.models.split(","):
        model = (S.make_student("qwen1.5-0.5b", "clip-l-336", seed=1) if name == "student" else
                 S.make_teacher("qwen1.5-7b", "clip-l-336", seed=0)).eval()
        if a.profile:
            profile_step(model, name, a.out, info)
        elif not a.skip_generate:
            for B in [int(x) for x in a.batch.split(",")]:
                for new in [int(x) for x in a.new.split(",")]:
                    for use_cache, graphs in ((True, True), (True, False), (False, False)):
                        if not use_cache and new > a.nocache_max_new:
                            continue
                        bench_generate(model, name, B, new, use_cache, graphs, a.out, info, a.repeat)
        del model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
