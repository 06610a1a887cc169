"""FP8 (e4m3) teacher against the bf16 one, kernel by kernel and as a whole forward / cached decode step.  One process, CUDA events,
every shape warmed up, bf16 and e4m3 alternating; the card, its power limit and the SM clock under load are printed with the numbers.

    python scripts/bench_fp8_teacher.py [--iters 30] [--layers 8] [--out FILE.json]

Share of peak is against NVIDIA's data-sheet figures for the H100 SXM at 700 W (989 TFLOP/s dense BF16, 1,979 dense FP8, 3.35 TB/s): figures
from the data sheet, not reached ones.  torch._scaled_mm, where the installed torch offers it, is a yardstick only (as torch.mm is for
the bf16 kernel); the library never calls it."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "llava-mod_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from llavamod import kernels as K  # noqa: E402

PEAK = dict(bf16=989e12, fp8=1979e12, hbm=3.35e12)


def smi(fields):
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:                                   # the numbers still stand, without the card's description
        return "nvidia-smi unavailable (%s)" % e


def timed(fns, iters):
    """ms per call of each fn, the fns alternating inside one timed loop per round (median of 5 rounds)."""
    for f in fns:
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    res = [[] for _ in fns]
    for _ in range(5):
        for i, f in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                f()
            b.record()
            torch.cuda.synchronize()
            res[i].append(a.elapsed_time(b) / iters)
    return [sorted(r)[len(r) // 2] for r in res]


def gemm_rows(iters):
    from llavamod.model.language_model.qwen2_core import rope_tables
    M = 2048
    rows = []
    shapes = [("q|k|v + RoPE", "rope", 12288, 4096, (32, 32, 128)), ("o_proj", "plain", 4096, 4096, None), ("gate|up + SwiGLU", "swiglu", 22016, 4096, None),
              ("down_proj", "plain", 4096, 11008, None), ("Qwen2-7B q|k|v + RoPE", "rope", 4608, 3584, (28, 4, 128)), ("Qwen2-7B o_proj", "plain", 3584, 3584, None),
              ("Qwen2-7B gate|up + SwiGLU", "swiglu", 37888, 3584, None), ("Qwen2-7B down_proj", "plain", 3584, 18944, None)]
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, form, N, Kd, heads in shapes:
        x = torch.randn(M, Kd, device="cuda", generator=g).to(torch.bfloat16)
        w = (torch.randn(N, Kd, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
        xq, wq = K.quant_rows(x), K.quant_rows(w)
        if form == "rope":
            nh, nkv, hd = heads
            cos, sin = rope_tables(hd, 4096, 1e6, torch.bfloat16, "cuda")
            pos = torch.arange(M, device="cuda")
            bias = torch.zeros(N, device="cuda", dtype=torch.bfloat16)
            f16 = lambda: K.qkv_rope(x, w, bias, cos, sin, pos, nh, nkv, hd)          # noqa: E731
            f8 = lambda: K.qkv_rope_fp8(xq, wq, bias, cos, sin, pos, nh, nkv, hd)      # noqa: E731
        elif form == "swiglu":
            f16 = lambda: K.gemm_swiglu(x, w)                                          # noqa: E731
            act = torch.empty(M, N // 2, dtype=torch.bfloat16, device="cuda")
            f8 = lambda: K.call("lmod_gemm_e4m3_swiglu", K.ptr(xq.q), Kd, K.ptr(xq.scale), K.ptr(wq.q), Kd, K.ptr(wq.scale), K.ptr(act), N // 2, M, N // 2, Kd)  # noqa: E731
        else:
            f16 = lambda: K.gemm(x, w)                                                 # noqa: E731
            f8 = lambda: K.gemm_fp8(xq, wq)                                            # noqa: E731
        fns = [f16, f8]
        if hasattr(torch, "_scaled_mm"):
            a8, b8 = xq.q.view(torch.float8_e4m3fn), wq.q.view(torch.float8_e4m3fn).t()
            sa, sb = xq.scale[:, None].contiguous(), wq.scale[None, :].contiguous()
            try:
                torch._scaled_mm(a8, b8, scale_a=sa, scale_b=sb, out_dtype=torch.bfloat16)
                fns.append(lambda: torch._scaled_mm(a8, b8, scale_a=sa, scale_b=sb, out_dtype=torch.bfloat16))
            except Exception:
                pass
        ms = timed(fns, iters)
        flop = 2.0 * M * N * Kd
        rows.append(dict(gemm=name, M=M, N=N, K=Kd, bf16_ms=ms[0], e4m3_ms=ms[1], scaled_mm_ms=ms[2] if len(ms) > 2 else None,
                         bf16_tflops=flop / ms[0] / 1e9, e4m3_tflops=flop / ms[1] / 1e9, e4m3_share_of_datasheet_fp8=flop / ms[1] / 1e9 / (PEAK["fp8"] / 1e12),
                         bf16_share_of_datasheet_bf16=flop / ms[0] / 1e9 / (PEAK["bf16"] / 1e12)))
    return rows


def quant_rows_rows(iters):
    rows = []
    g = torch.Generator(device="cuda").manual_seed(1)
    for M, Kd in ((2048, 4096), (2048, 11008)):
        x = torch.randn(M, Kd, device="cuda", generator=g).to(torch.bfloat16)
        (ms,) = timed([lambda: K.quant_rows(x)], iters)
        rows.append(dict(kernel="quant_rows", M=M, K=Kd, ms=ms, gbytes_per_s=(M * Kd * 3 + M * 4) / ms / 1e6))
    x = torch.randn(2048, 4096, device="cuda", generator=g).to(torch.bfloat16)
    r = torch.randn(2048, 4096, device="cuda", generator=g).to(torch.bfloat16)
    w = torch.ones(4096, device="cuda", dtype=torch.bfloat16)
    with torch.no_grad():
        ms = timed([lambda: K.rmsnorm(x, w, 1e-6, res=r), lambda: K.rmsnorm_quant(x, w, 1e-6, res=r)], iters)
    rows.append(dict(kernel="rmsnorm (+res) -> bf16", M=2048, K=4096, ms=ms[0], gbytes_per_s=2048 * 4096 * 8 / ms[0] / 1e6))
    rows.append(dict(kernel="rmsnorm_quant (+res) -> e4m3", M=2048, K=4096, ms=ms[1], gbytes_per_s=(2048 * 4096 * 7 + 2048 * 4) / ms[1] / 1e6))
    return rows


def model_rows(layers, iters):
    """A teacher-shaped decoder (H 4096, I 11008, 32 heads) of `layers` layers: one forward at T' = 2048 and a cached decode step at B = 1, 8;
    two copies of the same weights, one quantised."""
    from llavamod.model.language_model.qwen2_core import KVCache, Qwen2Config, Qwen2Model
    cfg = Qwen2Config(vocab_size=64, hidden_size=4096, intermediate_size=11008, num_hidden_layers=layers, num_attention_heads=32, rope_theta=1e6)
    models = []
    for _ in range(2):
        torch.manual_seed(3)
        m = Qwen2Model(cfg, "cuda", torch.bfloat16).eval()
        for p in m.parameters():
            p.requires_grad = False
        models.append(m)
    models[1].quantize_fp8_()
    x = torch.randn(1, 2048, 4096, device="cuda").to(torch.bfloat16)
    out = []
    with torch.no_grad():
        ms = timed([lambda: models[0](x), lambda: models[1](x)], max(3, iters // 5))
        out.append(dict(what="decoder forward, T' = 2048, %d layers" % layers, bf16_ms=ms[0], fp8_ms=ms[1]))
        for B in (1, 8):
            caches = [KVCache(m, B, 1024) for m in models]
            pre = torch.randn(B, 512, 4096, device="cuda").to(torch.bfloat16)
            tok = torch.randn(B, 1, 4096, device="cuda").to(torch.bfloat16)
            for m, c in zip(models, caches):
                m(pre, cache=c)

            def step(m, c):
                def f():
                    m(tok, cache=c)
                    c.rollback(1)
                    c.len.sub_(1)
                return f
            ms = timed([step(models[0], caches[0]), step(models[1], caches[1])], iters)
            out.append(dict(what="cached decode step (eager), B = %d, 512 cached, %d layers" % (B, layers), bf16_ms=ms[0], fp8_ms=ms[1]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--layers", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8_teacher.py measures on a GPU; none found")
    res = dict(card=smi("name,power.limit,clocks.max.sm"), datasheet_peaks=PEAK)
    res["gemm"] = gemm_rows(a.iters)
    res["sm_clock_under_load"] = smi("clocks.sm,power.draw")
    res["quant"] = quant_rows_rows(a.iters)
    res["model"] = model_rows(a.layers, a.iters)
    print("card:", res["card"], "| under load:", res["sm_clock_under_load"])
    for r in res["gemm"]:
        print("%-28s %5dx%5dx%5d  bf16 %.3f ms (%4.0f TFLOP/s, %.0f%% of data-sheet BF16)  e4m3 %.3f ms (%4.0f TFLOP/s, %.0f%% of data-sheet FP8)  _scaled_mm %s"
              % (r["gemm"], r["M"], r["N"], r["K"], r["bf16_ms"], r["bf16_tflops"], 100 * r["bf16_share_of_datasheet_bf16"], r["e4m3_ms"], r["e4m3_tflops"],
                 100 * r["e4m3_share_of_datasheet_fp8"], "%.3f ms" % r["scaled_mm_ms"] if r["scaled_mm_ms"] else "n/a"))
    for r in res["quant"]:
        print("%-30s [%d, %d]  %.4f ms  %.0f GB/s (%.0f%% of data-sheet HBM)" % (r["kernel"], r["M"], r["K"], r["ms"], r["gbytes_per_s"], 100 * r["gbytes_per_s"] * 1e9 / PEAK["hbm"]))
    for r in res["model"]:
        print("%-60s bf16 %.3f ms  fp8 %.3f ms  (x%.2f)" % (r["what"], r["bf16_ms"], r["fp8_ms"], r["bf16_ms"] / r["fp8_ms"]))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
