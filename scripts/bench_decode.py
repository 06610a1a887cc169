"""Decoding benchmark: tokens/s of `generate` with and without the KV cache, decode-attention bandwidth, and the device time per
kernel family of one cached decode step.

    python scripts/bench_decode.py [--models student,teacher] [--new 128,512] [--batch 1,8] [--profile] [--ragged] [--assisted]
                                   [--num-return 4,8] [--num-beams 2,3,4] [--out DIR]

* generate: the 0.5B-4E student and the 7B teacher (random weights, CLIP-L/336) on a prompt that splices to T' = 650 positions, greedy,
  use_cache False / True, CUDA graphs on / off (LLAVAMOD_CUDA_GRAPHS).  Tokens/s = B * new tokens / wall time of the call, which ends in
  a device synchronise; one full-length warm-up call per setting, then --repeat timed calls (median, min and max).  The no-cache loop at 512 new tokens is skipped unless asked (it re-runs the
  whole prompt every token).
* attention: lmod_attn_decode alone, B = 1 and 8, lengths 1k to 32k, CUDA events over 50 launches; bytes = 2 * len * nkv * hd * 2 per
  sequence (K and V) plus q and out, against the 3.35 TB/s of the H100 SXM data sheet.
* --profile: torch.profiler over 20 graph-less decode steps of the student at B = 1, device time summed per kernel family.
* --ragged: B = 8 seeded prompts of different lengths (one image each, left-padded, spliced to 600-1100 positions), greedy, graphs on,
  2 new tokens (a short-answer eval, dominated by the prefill) and 128: one padded B = 8 call, eight B = 1 calls on the same prompts,
  and the equal-length B = 8 row (T' = 650), each as prompts/s and tokens/s (median of --repeat timed passes after one warm-up pass).
* --assisted: the 7B teacher with the 0.5B-4E student as draft (random weights, T' = 650, greedy, graphs on, the first --new value of new
  tokens), B from --batch, k = 2 and 4: tokens/s of the teacher alone, of assisted decoding with the teacher as its own assistant (every
  draft kept: the pure overhead of the scheme) and with the random student (almost every draft rejected: the worst case); and the device
  time (CUDA events over 20 graph replays / launches) of one draft step, one verify step of k + 1 tokens, one teacher step and one accept
  launch, with the per-token acceptance alpha at which a round breaks even with the teacher alone.  alpha of a trained pair is not
  measured here (random weights).
* --num-return N[,N...]: sampled generate with num_return_sequences = n, the 7B teacher and the 0.5B-4E student (random weights, graphs on,
  the first --new value of new tokens), B from --batch at T' = 650 and B = 1 at T' = 8175 (a 7600-token prompt with one image), against
  the explicitly expanded call (inputs repeat_interleave'd to B*n, n = 1): tokens/s (B*n*new over the call), time to the first token
  (a call with max_new_tokens = 1: tower, prefill and one draw), the K / V bytes of the decode cache each allocates, and the decode
  attention of one layer at the middle step of the run: lmod_attn_decode_shared on the shared cache against lmod_attn_decode on the
  expanded one, CUDA events over 50 launches each, alternated, with the bytes each must read (K / V rows, q, out).  The sparse student
  runs the expanded call in both rows (its copies cannot share the cache), so its rows differ only by noise.
* --num-beams NB[,NB...]: beam search (num_beams = nb, eos_token_id -1 so every call runs all its steps), the 7B teacher and the
  0.5B-4E student (random weights, graphs on), B from --batch, each --new value, T' = 650: prompts/s and steps/s of the shared-cache path
  against the expanded form (generation._beam_search(expand=True)) for the dense teacher, the expanded form only for the sparse student,
  and the K / V bytes each allocates.  Then lmod_kv_beam_reorder alone at each model's shapes, B and nb: the suffix reorder of the shared
  cache at 128, 512 and 1024 rows past the prompt, and the whole-cache reorder of the expanded form (650 + those rows), each one launch
  over every layer's K and V with a map that moves half the beams (the call's host checks and operand copy included); CUDA events over
  20 calls, median of three alternated rounds, with the bytes it must move (sources read once, changed beams written) over 3.35 TB/s.
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


def ragged_prompts(B=8, seed=7):
    """B prompts of 24-524 text tokens plus one image (576 patches): 600-1100 spliced positions, left-padded with token 0."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(25, 526, (B,), generator=g).tolist()
    T = max(lens)
    ids = torch.zeros(B, T, dtype=torch.long)
    mask = torch.zeros(B, T, dtype=torch.bool)
    for b, n in enumerate(lens):
        p = torch.randint(0, 150000, (n,), generator=g)
        p[3] = -200
        ids[b, T - n:], mask[b, T - n:] = p, True
    imgs = [torch.randn(3, 336, 336, generator=g).to(torch.bfloat16) for _ in range(B)]
    return ids, mask, imgs


def bench_ragged(model, name, new, out, info, repeat):
    """prompts/s and tokens/s of one padded B = 8 call, of eight B = 1 calls on the same prompts, and of the equal-length B = 8 call."""
    os.environ["LLAVAMOD_CUDA_GRAPHS"] = "1"
    ids, mask, imgs = ragged_prompts()
    B = ids.shape[0]
    eq_ids, eq_imgs = prompt(B)
    runs = {
        "padded_B8": lambda: [model.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=new, use_cache=True, eos_token_id=-1)],
        "eight_B1": lambda: [model.generate(ids[b:b + 1, mask[b]], images=imgs[b:b + 1], max_new_tokens=new, use_cache=True, eos_token_id=-1)
                             for b in range(B)],
        "equal_length_B8": lambda: [model.generate(eq_ids, images=eq_imgs, max_new_tokens=new, use_cache=True, eos_token_id=-1)],
    }
    n_b = model.spliced_length(ids, imgs, mask)
    for row, fn in runs.items():
        fn()                                                                     # warm-up (and graph capture)
        secs = []
        for _ in range(repeat):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            secs.append(time.perf_counter() - t0)
        secs.sort()
        t = secs[len(secs) // 2]
        emit(out, dict(kind="ragged", model=name, row=row, B=B, new=new, spliced=(min(n_b), max(n_b)) if row != "equal_length_B8" else (650, 650),
                       runs=repeat, seconds=round(t, 4), prompts_per_s=round(B / t, 2), tokens_per_s=round(B * new / t, 1),
                       min_s=round(secs[0], 4), max_s=round(secs[-1], 4), card=info))


def _timed_generate(fn, repeat):
    fn()                                                                         # warm-up (and graph capture)
    secs = []
    for _ in range(repeat):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        secs.append(time.perf_counter() - t0)
    return sorted(secs)


def _replay_ms(fn, n=20):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def _step_graph(model, B, T, ids, imgs):
    """A captured cached step of T tokens per sequence after the prompt, on its own cache (replays move the device lengths only)."""
    from llavamod.model import generation as Gm
    ent = dict(cache=model.new_kv_cache(B, 2048), graph=None)
    with torch.no_grad():
        Gm.next_token_logits(model, ids, images=imgs, cache=ent["cache"])
        tok = torch.zeros((B,) if T == 1 else (B, T), dtype=torch.int64, device="cuda")
        Gm._decode_step(model, ent, tok, eager=True)
        Gm._decode_step(model, ent, tok, eager=False)
    return ent["graph"]


def _break_even(ratio, k):
    """alpha with (1 - alpha^(k+1)) / (1 - alpha) = ratio (tokens per round needed to match the teacher alone); None past k + 1."""
    if ratio >= k + 1:
        return None
    lo, hi = 0.0, 1.0
    for _ in range(60):
        mid = (lo + hi) / 2
        if sum(mid ** i for i in range(k + 1)) < ratio:
            lo = mid
        else:
            hi = mid
    return round(lo, 3)


def bench_assisted(teacher, student, batches, new, out, info, repeat):
    from llavamod import kernels as K
    from llavamod.model import generation as Gm
    os.environ["LLAVAMOD_CUDA_GRAPHS"] = "1"
    for B in batches:
        ids, imgs = prompt(B)
        kw = dict(images=imgs, max_new_tokens=new, use_cache=True, eos_token_id=-1)
        rows = [("teacher_alone", None, 0)] + [(n, d, k) for k in (2, 4) for n, d in (("self_assisted", teacher), ("student_assisted", student))]
        for row, draft, k in rows:
            extra = dict(assistant_model=draft, num_assistant_tokens=k) if draft is not None else {}
            secs = _timed_generate(lambda: teacher.generate(ids, **kw, **extra), repeat)
            st = Gm.last_assisted_stats if draft is not None else None
            rec = dict(kind="assisted", row=row, B=B, k=k, new=new, runs=repeat, tokens_per_s=round(B * new / secs[len(secs) // 2], 1),
                       min=round(B * new / secs[-1], 1), max=round(B * new / secs[0], 1), card=info)
            if st:
                rec.update(rounds=st["rounds"], acceptance=round(sum(st["accepted"]) / max(1, sum(st["drafted"])), 3))
            emit(out, rec)
        t_step = _replay_ms(_step_graph(teacher, B, 1, ids, imgs).replay)
        t_draft = _replay_ms(_step_graph(student, B, 1, ids, imgs).replay)
        V = teacher.config.vocab_size
        for k in (2, 4):
            t_verify = _replay_ms(_step_graph(teacher, B, k + 1, ids, imgs).replay)
            P = torch.randn(B, k + 1, V, device="cuda")
            d = torch.randint(0, V, (B, k), device="cuda")
            t_accept = _replay_ms(lambda: K.spec_accept(P, d))
            round_ms = (k + 1) * t_draft + t_verify + t_accept
            emit(out, dict(kind="assisted_step_ms", B=B, k=k, teacher_step=round(t_step, 3), draft_step=round(t_draft, 3),
                           verify_step=round(t_verify, 3), accept=round(t_accept, 4), round=round(round_ms, 3),
                           break_even_alpha=_break_even(round_ms / t_step, k), card=info))
        torch.cuda.empty_cache()


def long_prompt(B, n_text=7600, seed=3):
    """B prompts of n_text tokens with one image: T' = n_text - 1 + 576."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, 150000, (B, n_text), generator=g)
    ids[:, 3] = -200
    imgs = [torch.randn(3, 336, 336, generator=g).to(torch.bfloat16) for _ in range(B)]
    return ids, imgs


def _kv_bytes(model, rows, length):
    cfg = model.config
    from llavamod import kernels as K
    hp = K.attn_head_dim(cfg.hidden_size // cfg.num_attention_heads)
    return cfg.num_hidden_layers * 2 * rows * cfg.num_key_value_heads * length * hp * 2


def _attn_shared_vs_expanded(model, B, n, P, S, max_len, suffix_cap):
    """us per launch and bytes of lmod_attn_decode_shared and lmod_attn_decode at one layer's shapes, every copy at P + S keys."""
    from llavamod import kernels as K
    cfg = model.config
    nh, nkv = cfg.num_attention_heads, cfg.num_key_value_heads
    hd = cfg.hidden_size // nh
    hp = K.attn_head_dim(hd)
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g).to(torch.bfloat16)  # noqa: E731
    q = rnd(B * n, nh * hd)
    kp, vp = rnd(B, nkv, max_len, hp), rnd(B, nkv, max_len, hp)
    ks, vs = rnd(B * n, nkv, suffix_cap, hp), rnd(B * n, nkv, suffix_cap, hp)
    km, vm = kp.repeat_interleave(n, 0), vp.repeat_interleave(n, 0)
    km[:, :, P:P + S], vm[:, :, P:P + S] = ks[:, :, :S], vs[:, :, :S]
    plen = torch.full((B,), P, dtype=torch.int32, device="cuda")
    lens = torch.full((B * n,), P + S, dtype=torch.int32, device="cuda")
    ws1 = torch.empty(K.attn_decode_ws_elems(B * n, nh, nkv, hd, max_len), dtype=torch.float32, device="cuda")
    ws2 = torch.empty(K.attn_decode_shared_ws_elems(B, n, nh, nkv, hd, max_len), dtype=torch.float32, device="cuda")
    runs = {"expanded": lambda: K.attn_decode(q, nh, nkv, hd, km, vm, lens, ws1),
            "shared": lambda: K.attn_decode_shared(q, n, nh, nkv, hd, kp, vp, plen, ks, vs, lens, max_len, ws2)}
    a, b = runs["expanded"]()[0], runs["shared"]()[0]
    same = bool(torch.equal(a.view(torch.int16), b.view(torch.int16)))
    ms = {k: [] for k in runs}
    for _ in range(3):                                                     # alternated rounds of 50 launches
        for k, fn in runs.items():
            ms[k].append(_replay_ms(fn, 50))
    row = nkv * hp * 2 * 2                                                 # K and V bytes of one key of one sequence
    rows_per_cta = min(n, 8 // (nh // nkv))
    qo = B * n * nh * hd * 2 * 2
    nbytes = {"expanded": B * n * (P + S) * row + qo,
              "shared": B * -(-n // rows_per_cta) * P * row + B * n * S * row + qo}
    res = {}
    for k in runs:
        t = sorted(ms[k])[1] * 1e-3
        res[k] = dict(us=round(t * 1e6, 2), us_spread=[round(x * 1e3, 2) for x in sorted(ms[k])], MB=round(nbytes[k] / 1e6, 2),
                      TBps=round(nbytes[k] / t / 1e12, 3))
    return res, same


def bench_num_return(models, ns, batches, new, out, info, repeat):
    from llavamod.model import generation as Gm
    from llavamod.model import synthetic as S
    os.environ["LLAVAMOD_CUDA_GRAPHS"] = "1"
    for name in models:
        model = (S.make_student("qwen1.5-0.5b", "clip-l-336", seed=1) if name == "student" else
                 S.make_teacher("qwen1.5-7b", "clip-l-336", seed=0)).eval()
        shapes = [(B, prompt(B), 650) for B in batches] + [(1, long_prompt(1), 7600 - 1 + 576)]
        for B, (ids, imgs), P in shapes:
            for n in ns:
                e_ids, e_imgs = ids.repeat_interleave(n, 0), [im for im in imgs for _ in range(n)]
                kw = dict(use_cache=True, do_sample=True, eos_token_id=-1)
                calls = {"expanded": lambda m: model.generate(e_ids, images=e_imgs, max_new_tokens=m, **kw),
                         "shared": lambda m: model.generate(ids, images=imgs, max_new_tokens=m, num_return_sequences=n, **kw)}
                rec = dict(kind="num_return", model=name, B=B, n=n, prompt_len=P, new=new, runs=repeat, card=info)
                for row, fn in calls.items():
                    Gm._STEP_GRAPHS.clear()
                    torch.cuda.empty_cache()
                    try:
                        secs = _timed_generate(lambda: fn(new), repeat)
                    except torch.OutOfMemoryError:
                        rec[row] = dict(out_of_memory=True)
                        Gm._STEP_GRAPHS.clear()
                        torch.cuda.empty_cache()
                        continue
                    ents = list(Gm._STEP_GRAPHS.values())
                    cache = ents[-1]["cache"]
                    ttft = _timed_generate(lambda: fn(1), repeat)
                    rec[row] = dict(tokens_per_s=round(B * n * new / secs[len(secs) // 2], 1), min=round(B * n * new / secs[-1], 1),
                                    max=round(B * n * new / secs[0], 1), ttft_ms=round(ttft[len(ttft) // 2] * 1e3, 2),
                                    ttft_spread_ms=[round(ttft[0] * 1e3, 2), round(ttft[-1] * 1e3, 2)],
                                    cache_MB=round(cache.nbytes / 1e6, 1), shared_cache=cache.shared)
                    del ents, cache
                Gm._STEP_GRAPHS.clear()
                torch.cuda.empty_cache()
                max_len = Gm._bucket(P + new)
                suffix = -(-new // Gm.SUFFIX_BUCKET) * Gm.SUFFIX_BUCKET
                attn, same = _attn_shared_vs_expanded(model, B, n, P, new // 2, max_len, suffix)
                if all("tokens_per_s" in rec[row] for row in calls):
                    rec.update(speedup=round(rec["shared"]["tokens_per_s"] / rec["expanded"]["tokens_per_s"], 3))
                rec.update(attn_layer_step=dict(attn, same_bytes=same, keys=P + new // 2))
                emit(out, rec)
                torch.cuda.empty_cache()
        del model
        torch.cuda.empty_cache()


def _reorder_case(model, B, nb, rows, cap):
    """(bufs, parent) for one reorder launch over every layer's K and V of B prompts of nb beams, and the bytes it moves: beams
    1 .. nb//2 take beam 0's rows (the rest keep theirs), so one source is read and nb // 2 beams are written per prompt."""
    from llavamod import kernels as K
    cfg = model.config
    hd = cfg.hidden_size // cfg.num_attention_heads
    hp = K.attn_head_dim(hd)
    bufs = [torch.empty(B * nb, cfg.num_key_value_heads, cap, hp, device="cuda", dtype=torch.bfloat16)
            for _ in range(2 * cfg.num_hidden_layers)]
    parent = [0 if 1 <= j <= nb // 2 else j for _ in range(B) for j in range(nb)]
    nbytes = len(bufs) * B * (1 + nb // 2) * cfg.num_key_value_heads * rows * hd * 2
    return bufs, parent, hd, nbytes


def bench_num_beams(models, nbs, batches, news, out, info, repeat):
    from llavamod import kernels as K
    from llavamod.model import generation as Gm
    from llavamod.model import synthetic as S
    os.environ["LLAVAMOD_CUDA_GRAPHS"] = "1"
    for name in models:
        model = (S.make_student("qwen1.5-0.5b", "clip-l-336", seed=1) if name == "student" else
                 S.make_teacher("qwen1.5-7b", "clip-l-336", seed=0)).eval()
        for B in batches:
            ids, imgs = prompt(B)
            for new in news:
                for nb in nbs:
                    kw = dict(use_cache=True, eos_token_id=-1, num_beams=nb, max_new_tokens=new)
                    calls = {"expanded": lambda: Gm._beam_search(model, ids, images=imgs, expand=True, **kw)}
                    if not model.is_moe:
                        calls["shared"] = lambda: model.generate(ids, images=imgs, **kw)
                    rec = dict(kind="num_beams", model=name, B=B, nb=nb, prompt_len=650, new=new, runs=repeat, card=info)
                    for row, fn in calls.items():
                        Gm._STEP_GRAPHS.clear()
                        torch.cuda.empty_cache()
                        try:
                            secs = _timed_generate(fn, repeat)
                        except torch.OutOfMemoryError:
                            rec[row] = dict(out_of_memory=True)
                            continue
                        cache = list(Gm._STEP_GRAPHS.values())[-1]["cache"]
                        med = secs[len(secs) // 2]
                        rec[row] = dict(prompts_per_s=round(B / med, 3), steps_per_s=round(new / med, 1),
                                        spread_s=[round(secs[0], 3), round(secs[-1], 3)], cache_MB=round(cache.nbytes / 1e6, 1),
                                        shared_cache=cache.shared)
                        del cache
                    Gm._STEP_GRAPHS.clear()
                    torch.cuda.empty_cache()
                    if all("steps_per_s" in rec.get(r, {}) for r in ("shared", "expanded")):
                        rec.update(speedup=round(rec["shared"]["steps_per_s"] / rec["expanded"]["steps_per_s"], 3))
                    emit(out, rec)
        for B in batches:
            for nb in nbs:
                for rows in (128, 512, 1024):
                    cases = {"suffix": (rows, -(-rows // Gm.SUFFIX_BUCKET) * Gm.SUFFIX_BUCKET),
                             "whole": (650 + rows, Gm._bucket(650 + rows))}
                    rec = dict(kind="beam_reorder", model=name, B=B, nb=nb, rows_past_prompt=rows, card=info)
                    runs, ms, nbytes = {}, {}, {}
                    try:
                        for k, (r, cap) in cases.items():
                            bufs, parent, hd, nbytes[k] = _reorder_case(model, B, nb, r, cap)
                            runs[k] = (lambda bufs=bufs, parent=parent, hd=hd, r=r: K.kv_beam_reorder(bufs, nb, hd, [r] * B, parent))
                            ms[k] = []
                    except torch.OutOfMemoryError:
                        rec["out_of_memory"] = True
                    for _ in range(3):
                        for k, fn in runs.items():
                            ms[k].append(_replay_ms(fn, 20))
                    for k in runs:
                        t = sorted(ms[k])[1] * 1e-3
                        rec[k] = dict(rows=cases[k][0], us=round(t * 1e6, 1), us_spread=[round(x * 1e3, 1) for x in sorted(ms[k])],
                                      MB=round(nbytes[k] / 1e6, 1), TBps=round(nbytes[k] / t / 1e12, 3),
                                      of_3_35TBps=round(nbytes[k] / t / 3.35e12, 3))
                    emit(out, rec)
                    runs.clear()
                    torch.cuda.empty_cache()
        del model
        torch.cuda.empty_cache()


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
    ap.add_argument("--ragged", action="store_true", help="padded batches of prompts of different lengths (see the module docstring)")
    ap.add_argument("--assisted", action="store_true", help="assisted decoding, teacher with the student as draft (module docstring)")
    ap.add_argument("--num-return", default=None, help="num_return_sequences values: shared against expanded (module docstring)")
    ap.add_argument("--num-beams", default=None, help="num_beams values: beam search shared against expanded (module docstring)")
    ap.add_argument("--repeat", type=int, default=3, help="timed generate calls per setting (median, min and max are reported)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_decode.py measures on the GPU"
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    info = card()
    from llavamod.model import synthetic as S
    if a.num_return:
        bench_num_return(a.models.split(","), [int(x) for x in a.num_return.split(",")], [int(x) for x in a.batch.split(",")],
                         int(a.new.split(",")[0]), a.out, info, a.repeat)
        return
    if a.num_beams:
        bench_num_beams(a.models.split(","), [int(x) for x in a.num_beams.split(",")], [int(x) for x in a.batch.split(",")],
                        [int(x) for x in a.new.split(",")], a.out, info, a.repeat)
        return
    if a.assisted:
        teacher = S.make_teacher("qwen1.5-7b", "clip-l-336", seed=0).eval()
        student = S.make_student("qwen1.5-0.5b", "clip-l-336", seed=1, share_tower_with=teacher).eval()
        bench_assisted(teacher, student, [int(x) for x in a.batch.split(",")], int(a.new.split(",")[0]), a.out, info, a.repeat)
        return
    if not a.skip_attention and not a.profile and not a.ragged:
        bench_attention(a.out, info)
    for name in a.models.split(","):
        model = (S.make_student("qwen1.5-0.5b", "clip-l-336", seed=1) if name == "student" else
                 S.make_teacher("qwen1.5-7b", "clip-l-336", seed=0)).eval()
        if a.profile:
            profile_step(model, name, a.out, info)
        elif a.ragged:
            for new in (2, 128):
                bench_ragged(model, name, new, a.out, info, a.repeat)
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
