"""Top-1 MoE routing with random token selection (--top_k_experts 1) on the GPU: the router against the restated top1gating bit for bit,
the MoE block stage by stage against float64, a tiny top-1 student against oracle autograd, the training entry point, and cached
decoding.  The uniform of the token selection is an input tensor throughout."""
import math
import os

import pytest
import torch

from oracle import restated as R
from tests import helpers as Hh
from tests import moe_top1_oracle as O

pytestmark = pytest.mark.gpu
u24 = 2.0 ** -24


def planted(S, H, E, counts, seed):
    """x [S,H] bf16 and wg [E,H] fp32 that route counts[e] tokens to expert e (in a shuffled order), with a clear margin."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.cat([torch.full((n,), e, dtype=torch.long) for e, n in enumerate(counts)])
    assert idx.numel() == S
    idx = idx[torch.randperm(S, generator=g)]
    x = torch.randn(S, H, generator=g) * 0.05
    x[torch.arange(S), idx] += 1.0
    wg = torch.randn(E, H, generator=g) * 0.01
    wg[torch.arange(E), torch.arange(E)] += 4.0
    return x.to(torch.bfloat16).cuda(), wg.cuda(), idx


def check_route(x, wg, u, cf, mc, idx_want=None):
    from llavamod import kernels as K
    S, H = x.shape
    E = wg.shape[0]
    r = K.moe_route_scatter(x, wg, u, cf, mc, K.LAYOUT_ALIGNED, k=1)
    o = O.top1gating(r["logits"].cpu(), u.cpu(), cf, mc)
    C = o["capacity"]
    assert r["capacity"] == C == K.moe_capacity(S, E, cf, mc, k=1) == R.moe_capacity(S, E, cf, mc, 1)
    idx, row, w = r["idx"].cpu().long(), r["row"].cpu().long(), r["w"].cpu()
    assert torch.equal(idx[:, 0], o["idx1"]) and bool((idx[:, 1] == -1).all())
    if idx_want is not None:
        assert torch.equal(idx[:, 0], idx_want)
    keep = row[:, 0] >= 0
    assert torch.equal(keep, o["keep1"]) and bool((row[:, 1] == -1).all())
    counts = torch.bincount(o["idx1"], minlength=E)
    used = torch.minimum(counts, torch.tensor(C))
    offs = torch.zeros(E + 1, dtype=torch.long)
    offs[1:] = ((used + 127) // 128 * 128).cumsum(0)
    assert torch.equal(r["offsets"].cpu().long(), offs)
    assert torch.equal(row[keep, 0], offs[o["idx1"][keep]] + o["slot1"][keep])
    meta = r["meta"].cpu()
    assert meta[1] == C and meta[2] == int(used.sum()) and meta[3] == int(offs[-1])
    assert torch.equal(meta[4:].long(), o["exp_counts"].long())
    gates = r["gates"].cpu()
    torch.testing.assert_close(gates, torch.softmax(r["logits"].cpu().double(), 1).float(), rtol=2e-6, atol=1e-9)
    g1 = gates.gather(1, idx[:, :1].clamp(min=0))[:, 0]
    assert torch.equal(w[:, 0], torch.where(keep, g1, torch.zeros_like(g1))) and bool((w[:, 1] == 0).all())
    tpb = Hh.moe_route_tpb(S)
    laux = E * (gates.double().mean(0) * counts.double() / S).sum()
    assert abs(float(meta[0]) - float(laux)) <= (tpb + -(-S // tpb) + E + 8) * u24 * abs(float(laux)) + 1e-30
    xp = r["xp"].cpu()
    n = int(offs[-1])
    want = torch.zeros(n, H, dtype=torch.bfloat16)
    want[row[keep, 0]] = x.cpu()[keep]
    assert torch.equal(xp[:n], want)                  # routed rows are the tokens, pad rows zero
    r2 = K.moe_route_scatter(x, wg, u, cf, mc, K.LAYOUT_ALIGNED, k=1)
    for key in ("idx", "row", "w", "offsets", "meta"):
        assert torch.equal(r[key], r2[key]), key
    return r, o


# id, S, H, E, cf, min_cap, counts
ROUTE_CASES = [
    ("config2", 2048, 1024, 4, 1.5, 0, [1600, 200, 120, 128]),             # C = 768, expert 0 overflows
    ("S2047", 2047, 1024, 4, 1.1, 0, [1300, 400, 247, 100]),
    ("E8-empty-mincap", 2048, 1024, 8, 1.0, 400, [900, 300, 200, 200, 150, 129, 169, 0]),   # ceil rule 256, min_capacity 400
    ("E2", 333, 256, 2, 0.6, 0, [220, 113]),
    ("decode-S1", 1, 1024, 4, 2.0, 0, [0, 0, 1, 0]),
    ("decode-S8", 8, 1024, 4, 2.0, 0, [5, 1, 2, 0]),                       # C = 4
]


@pytest.mark.parametrize("case", ROUTE_CASES, ids=[c[0] for c in ROUTE_CASES])
def test_router_bit_exact_against_top1gating(case):
    name, S, H, E, cf, mc, counts = case
    x, wg, idx = planted(S, H, E, counts, S + E)
    u = torch.rand(S, E, generator=torch.Generator().manual_seed(S)).cuda()
    r, o = check_route(x, wg, u, cf, mc, idx)
    C = o["capacity"]
    for e, n in enumerate(counts):
        assert int(o["keep1"][o["idx1"] == e].sum()) == min(n, C)
    if name == "config2":
        toks = (idx == 0).nonzero()[:, 0]
        kept = o["keep1"][toks]
        assert not bool(kept.all()) and bool(kept.any())
        first_kept = int(kept.nonzero()[0])
        assert bool((~kept[first_kept + 1:]).any()), "drops are not only a tail in token order"


def test_router_threshold_tie_and_zero_uniform():
    S, H, E, cf = 256, 512, 4, 1.0                # C = 64
    x, wg, idx = planted(S, H, E, [150, 60, 30, 16], 3)
    u = torch.rand(S, E, generator=torch.Generator().manual_seed(4)) * 0.5
    t0 = (idx == 0).nonzero()[:, 0].tolist()
    for s in t0[:60]:
        u[s, 0] = 0.75                            # 60 keys above the threshold
    tied = t0[60:70]                              # ten equal keys straddle the cut: the first 4 in token order are kept
    for s in tied:
        u[s, 0] = 0.5
    z = (idx == 1).nonzero()[0, 0]                # expert 1 is under-full: a routed uniform of exactly 0 keeps its seat
    u[z, 1] = 0.0
    r, o = check_route(x, wg, u.cuda(), cf, 0, idx)
    keep = (r["row"][:, 0] >= 0).cpu()
    assert keep[tied].tolist() == [True] * 4 + [False] * 6
    assert bool(keep[z])
    # a threshold of 0.0 itself: more zero keys than free seats
    u2 = torch.rand(S, E, generator=torch.Generator().manual_seed(5)) + 0.0
    for s in t0[:100]:
        u2[s, 0] = 0.0
    u2[t0[100:], 0] = 0.9                         # 50 keys above, then 14 of the 100 zeros by token order
    r, o = check_route(x, wg, u2.cuda(), cf, 0, idx)
    keep = (r["row"][:, 0] >= 0).cpu()
    assert keep[t0[:100]].tolist() == [True] * 14 + [False] * 86


def test_router_host_errors():
    from llavamod import kernels as K
    x, wg, _ = planted(8, 256, 4, [2, 2, 2, 2], 1)
    u = torch.rand(8, 4, device="cuda")
    with pytest.raises(ValueError, match="min_capacity"):
        K.moe_route_scatter(x, wg, u, 1.0, 9, k=1)
    with pytest.raises(ValueError, match="capacity"):
        K.moe_route_scatter(x, wg, u, 8.0, 0, k=1)          # C = 16 > 8
    from llavamod._C import LmodError, call, ptr
    e = torch.empty(64, dtype=torch.float32, device="cuda")
    i = torch.empty(64, dtype=torch.int32, device="cuda")
    with pytest.raises(LmodError, match="min_capacity"):
        call("lmod_moe_route_scatter_top1", ptr(x), ptr(wg), ptr(u), 8, 256, 4, 1.0, 9, 2, ptr(e), ptr(e), ptr(i), ptr(i), ptr(e), ptr(i),
             ptr(e), ptr(e), ptr(i))


# ---------------------------------------------------------------------------------------------------------------------------------
# the MoE block stage by stage against float64 (bounds of tests/helpers.py)
# ---------------------------------------------------------------------------------------------------------------------------------
BLOCK_CASES = [
    ("config2", 2048, 1024, 2816, 4, 1.5, 0, [1600, 200, 120, 128]),
    ("1.8B-4E-S2048", 2048, 2048, 5504, 4, 1.5, 0, [1600, 200, 120, 128]),
    ("I320-E2", 333, 256, 320, 2, 0.6, 0, [220, 113]),
]


def _per_expert(A, Wf, offs, used, n_out, K_):
    want = torch.zeros(A.shape[0], n_out, dtype=torch.float64, device=A.device)
    tol = torch.zeros_like(want)
    for e in range(len(used)):
        r0, r1 = int(offs[e]), int(offs[e]) + int(used[e])
        if r1 > r0:
            a = A[r0:r1].double()
            B = Wf(e)
            want[r0:r1] = a @ B
            tol[r0:r1] = Hh._gemm_tol(want[r0:r1], a.abs() @ B.abs(), K_)
    return want, tol


@pytest.mark.parametrize("case", BLOCK_CASES, ids=[c[0] for c in BLOCK_CASES])
def test_moe_block_top1_stage_by_stage(case):
    from llavamod import kernels as K
    name, S, H, I, E, cf, mc, counts = case
    x, wg, _ = planted(S, H, E, counts, S + H)
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(S + I)
    u = torch.rand(S, E, device=dev, generator=g)
    w_gu = (torch.randn(E, 2 * I, H, device=dev, generator=g) / math.sqrt(H)).to(torch.bfloat16)
    w_dn = (torch.randn(E, H, I, device=dev, generator=g) / math.sqrt(I)).to(torch.bfloat16)
    res = torch.randn(S, H, device=dev, generator=g).to(torch.bfloat16)
    dout = (torch.randn(S, H, device=dev, generator=g) * 0.1).to(torch.bfloat16)
    old = dict(wg=torch.randn(E, H, device=dev, generator=g) * 1e-2,
               w_gu=(torch.randn(E, 2 * I, H, device=dev, generator=g) * 1e-2).to(torch.bfloat16),
               w_dn=(torch.randn(E, H, I, device=dev, generator=g) * 1e-2).to(torch.bfloat16))
    g_laux = 0.37
    grads = {k: v.clone() for k, v in old.items()}
    st = K.moe_forward_stages(x, res, wg, w_gu, w_dn, u, cf, mc, k=1)
    bw = K.moe_backward_stages(st, x, wg, w_gu, w_dn, dout, torch.tensor(g_laux, device=dev), grads)
    _, o = check_route(x, wg, u, cf, mc)
    row, keep = st["row"][:, 0].long(), st["row"][:, 0] >= 0
    idx = st["idx"][:, :1].long()
    offs, used = st["offsets"].long().cpu(), torch.minimum(torch.bincount(idx[:, 0], minlength=E).cpu(), torch.tensor(st["capacity"]))
    n = int(offs[-1])
    # expert forward
    want, tol = _per_expert(st["xp"][:n], lambda e: w_gu[e].double().t(), offs, used, 2 * I, H)
    Hh.check_moe("h1", st["h1"][:n], want, tol)
    h1 = st["h1"][:n].double()
    gg, uu = h1[:, :I], h1[:, I:]
    sg = torch.sigmoid(gg)
    act = gg * sg * uu
    Hh.check_moe("act", st["act"][:n], act, (2.0 ** -7 + 2.0 ** -16) * act.abs())
    want, tol = _per_expert(st["act"][:n], lambda e: w_dn[e].double().t(), offs, used, H, I)
    Hh.check_moe("y", st["y"][:n], want, tol)
    # combine: bit exact from the kernel's y and w
    wb = st["w"][:, :1].to(torch.bfloat16).float()
    ysel = torch.where(keep[:, None], st["y"][row.clamp(min=0)].float(), torch.zeros(S, H, device=dev))
    Hh.check_moe("out", st["out"], (res.float() + (wb * ysel).to(torch.bfloat16).float()).to(torch.bfloat16))
    # combine backward
    dy = torch.zeros(st["xp"].shape[0], H, dtype=torch.bfloat16, device=dev)
    dy[row[keep]] = (wb[keep] * dout[keep].float()).to(torch.bfloat16)
    Hh.check_moe("dy", bw["dy"], dy)
    d64 = dout.double()
    yr = st["y"][row.clamp(min=0)].double()
    dw = torch.where(keep, (d64 * yr).sum(1), torch.zeros(S, dtype=torch.float64, device=dev))
    lane_fmas = 8 * -(-H // 256)
    dwt = (lane_fmas + 6) * u24 * (d64.abs() * yr.abs()).sum(1) * keep
    Hh.check_moe("dw", bw["dw"][:, 0], dw, dwt)
    assert bool((bw["dw"][:, 1] == 0).all())
    # expert backward
    dact, dact_tol = _per_expert(bw["dy"][:n], lambda e: w_dn[e].double(), offs, used, I, H)
    Hh.check_moe("dact", bw["dact"][:n], dact, dact_tol)
    cg, cu = uu * sg * (1 + gg * (1 - sg)), gg * sg
    dh1 = torch.cat([dact * cg, dact * cu], 1)
    derr = dact_tol + 2.0 ** -16 * dact.abs()
    Hh.check_moe("dh1", bw["dh1"][:n], dh1, 2.0 ** -8 * dh1.abs() + (1 + 2.0 ** -8) * torch.cat([derr * cg.abs(), derr * cu.abs()], 1))
    want, tol = _per_expert(bw["dh1"][:n], lambda e: w_gu[e].double(), offs, used, H, 2 * I)
    Hh.check_moe("dxp", bw["dxp"][:n], want, tol)
    for gname, a, b, M, N in (("w_dn", bw["dy"], st["act"], H, I), ("w_gu", bw["dh1"], st["xp"], 2 * I, H)):
        for e in range(E):
            r0, r1, r2 = int(offs[e]), int(offs[e]) + int(used[e]), int(offs[e + 1])
            o_e = old[gname][e].double()
            if r1 > r0:
                A, B = a[r0:r1].double(), b[r0:r1].double()
                ref = A.t() @ B + o_e
                Hh.check_moe("g_" + gname, grads[gname][e], ref, Hh._gemm_tol(ref, A.abs().t() @ B.abs(), r2 - r0) + 2.0 ** -23 * ref.abs())
            else:
                Hh.check_moe("g_" + gname, grads[gname][e], o_e.to(grads[gname].dtype))
    # gate backward: dgates[s, idx1] += dw (kept), the l_aux term, the softmax
    gk = st["gates"].double()
    dwk = bw["dw"][:, 0].double() * keep
    lterm = (g_laux * E * o["exp_counts"].to(dev).double() / S / S)[None].expand(S, E)
    rterm = torch.zeros(S, E, dtype=torch.float64, device=dev).scatter_add_(1, idx, dwk[:, None])
    dg = lterm + rterm
    D = lterm.abs() + rterm.abs()
    dl = gk * (dg - (gk * dg).sum(1, keepdim=True))
    dl_tol = gk * (16 * u24 * D + (gk * (16 * u24 * D + E * u24 * dg.abs())).sum(1, keepdim=True)) + 2 * u24 * dl.abs() + 2.0 ** -140
    Hh.check_moe("dlogits", bw["dlogits"], dl, dl_tol)
    dlk = bw["dlogits"].double()
    wg64 = wg.double()
    dx = dlk @ wg64
    maj = dlk.abs() @ wg64.abs()
    v = bw["dxp"][row.clamp(min=0)].double() * keep[:, None]
    dx, maj = dx + v, maj + v.abs()
    Hh.check_moe("dx", bw["dx"], dx, 2.0 ** -8 * dx.abs() + (1 + 2.0 ** -8) * (E + 2) * u24 * maj)
    dwg = old["wg"].double() + dlk.t() @ x.double()
    Hh.check_moe("g_wg", grads["wg"], dwg, (-(-S // 32) + 34) * u24 * (dlk.abs().t() @ x.double().abs() + old["wg"].double().abs()))
    # MoEFn and the no-grad path give the stage functions' bytes
    grads_want = grads
    grads = {k: v.clone() for k, v in old.items()}
    xd, rd = x.clone().requires_grad_(True), res.clone().requires_grad_(True)
    out, l_aux = K.MoEFn.apply(xd, rd, wg, w_gu, w_dn, u, cf, mc, grads, 1)
    ((out.float() * dout.float()).sum() + g_laux * l_aux).backward()
    assert torch.equal(out, st["out"]) and torch.equal(l_aux, st["meta"][0]) and torch.equal(xd.grad, bw["dx"])
    for k in grads:
        assert torch.equal(grads[k], grads_want[k]), k
    with torch.no_grad():
        out_ng, la_ng, _ = K.moe_forward_nograd(x, res, wg, w_gu, w_dn, u, cf, mc, 1)
    assert torch.equal(out_ng, st["out"]) and torch.equal(la_ng, st["meta"][0])


# ---------------------------------------------------------------------------------------------------------------------------------
# a tiny top-1 student end to end
# ---------------------------------------------------------------------------------------------------------------------------------
def top1_pair(seed=0, vocab=512):
    from llavamod.model import synthetic as S
    teacher = S.make_teacher(dict(S.ARCH["tiny"], vocab_size=vocab, intermediate_size=320), "tiny", seed=seed)
    student = S.make_student(dict(S.ARCH["tiny"], vocab_size=vocab), "tiny", seed=seed + 1, margs=S.moe_args(top_k=1),
                             share_tower_with=teacher)
    return student, teacher


def uniforms(student, B, Tn, seed):
    g = torch.Generator().manual_seed(seed)
    n_moe = sum(1 for l in student.model.layers if hasattr(l.mlp, "deepspeed_moe"))
    return [torch.rand(B * Tn, 4, generator=g) for _ in range(n_moe)]


def oracle_student(student, batch, noise, sd=None, record=None):
    lc, cc = Hh.cfgs_of(student)
    lc.top_k = 1
    sd = sd if sd is not None else Hh.oracle_state(student)
    return O.llava_forward(sd, lc, cc, batch["input_ids"], batch["attention_mask"], batch["labels"],
                           [im.float() for im in batch["images"]], noise, record), lc


def test_tiny_top1_student_forward_backward_match_oracle_autograd():
    student, teacher = top1_pair()
    assert all(l.mlp.k == 1 for l in student.model.layers if hasattr(l.mlp, "deepspeed_moe"))
    batch, _ = Hh.tiny_batch(student, seed=4)
    noise = uniforms(student, 2, 55, 5)
    # routing agrees first: the no-grad forward's records against the oracle's
    rec = []
    with torch.no_grad():
        r = student.forward_hidden(input_ids=batch["input_ids"], attention_mask=batch["attention_mask"], labels=batch["labels"],
                                   images=batch["images"], moe_noise=[n.cuda() for n in noise])
    oracle_student(student, batch, noise, record=rec)
    assert len(r["records"]) == len(rec) == 1
    for gr, o in zip(r["records"], rec):
        assert torch.equal(gr["idx"][:, 0].long().cpu(), o["idx1"])
        assert torch.equal((gr["row"][:, 0] >= 0).cpu(), o["keep1"])
        assert int((~o["keep1"]).sum()) >= 0
    sd_s = Hh.oracle_state(student)
    keys = [n for n, p in student.named_parameters() if p.requires_grad]
    for k in keys:
        sd_s[k].requires_grad_(True)
    with torch.no_grad():
        t_out, _ = Hh.oracle_forward(teacher, batch)
    s_out, lc = oracle_student(student, batch, noise, sd=sd_s)
    ref_loss, ref_m = R.mimic_compute_loss(s_out, t_out["logits"], "kd_lm", True, False, lc.kd_vocab)
    ref_loss.backward()
    tr = Hh.make_trainer(student, teacher, "kd_lm")
    opt = tr.create_optimizer()
    opt.zero_grad()
    loss, m = tr.compute_loss(student, dict(batch, moe_noise=[n.cuda() for n in noise]), return_outputs=True)
    for k in ("loss", "loss/align", "loss/lm", "loss/moe_balance"):
        assert abs(float(m[k]) - float(ref_m[k])) < 1e-2 * abs(float(ref_m[k])) + 1e-4, (k, float(m[k]), float(ref_m[k]))
    loss.backward()
    torch.cuda.synchronize()
    for n, p in student.named_parameters():
        if p.requires_grad:
            gr, rr = p.grad.float().cpu(), sd_s[n].grad
            rel = (gr - rr).norm().item() / (rr.norm().item() + 1e-12)
            assert rel < 0.08, (n, rel)            # the tolerance of test_model_gpu.py's top-2 gradient check


def test_graphed_micro_batch_equals_eager_for_injected_uniforms():
    losses = {}
    for graphs in (False, True):
        student, teacher = top1_pair(seed=2)
        tr = Hh.make_trainer(student, teacher, "kd_lm", accum=1, lr=0.0)
        tr.use_cuda_graphs = graphs
        got = []
        for i in range(5):
            batch, _ = Hh.tiny_batch(student, seed=60 + i)
            got.append(float(tr.training_step(student, dict(batch, moe_noise=[n.cuda() for n in uniforms(student, 2, 55, 70 + i)]))))
        if graphs:
            assert tr._graphs, "no graph was captured"
        losses[graphs] = got
    assert losses[True] == losses[False], losses


def test_align_train_entry_point_with_top1(tmp_path, golden_dir):
    import json
    from llavamod.train import align_train
    from tests.test_entrypoints_gpu import _check_final_save, _common_flags, _save_tiny_checkpoints
    policy, teacher, tower, _ = _save_tiny_checkpoints(str(tmp_path), golden_dir)
    out = str(tmp_path / "out_top1")
    argv = _common_flags(policy, teacher, tower, out, golden_dir, "data_sft.json") + ["--loss_type", "kd_lm", "--learning_rate", "1e-3"]
    argv[argv.index("--top_k_experts") + 1] = "1"
    tr = align_train.train(argv)
    assert tr.state.global_step == 2
    assert all(l.mlp.k == 1 for l in tr.model.model.layers if hasattr(l.mlp, "deepspeed_moe"))
    _check_final_save(out, tr, (2,))
    assert json.load(open(os.path.join(out, "config.json")))["moe"]["top_k_experts"] == 1
    from llavamod.model import EvalLLaVAMoDQwen1_5ForCausalLM
    m = EvalLLaVAMoDQwen1_5ForCausalLM.from_pretrained(out)
    assert all(l.mlp.k == 1 for l in m.model.layers if hasattr(l.mlp, "deepspeed_moe"))


def test_cached_step_equals_recompute_and_assists_the_teacher():
    student, teacher = top1_pair(seed=6)
    student.eval()
    moes = [l.mlp for l in student.model.layers if hasattr(l.mlp, "deepspeed_moe")]
    batch, _ = Hh.tiny_batch(student, B=2, Tt=20, seed=7)
    ids, images = batch["input_ids"].cuda(), batch["images"]
    Tn = 20 - 1 + 16
    g = torch.Generator().manual_seed(8)
    cache = student.new_kv_cache(2, 64)
    pre = [torch.rand(2 * Tn, 4, generator=g).cuda() for _ in moes]
    tok = torch.randint(0, 512, (2, 1), generator=g).cuda()
    step = [torch.rand(2, 4, generator=g).cuda() for _ in moes]
    with torch.no_grad():
        student.forward_hidden(input_ids=ids, images=images, moe_noise=pre, cache=cache)
        a = student.forward_hidden(input_ids=tok, moe_noise=step, cache=cache)
        # the same step through forward(past_key_values=...)
        cache2 = student.new_kv_cache(2, 64)
        student.forward_hidden(input_ids=ids, images=images, moe_noise=pre, cache=cache2)
        b = student(input_ids=tok, past_key_values=cache2, use_cache=True, moe_noise=step, return_dict=True)
    assert a["records"][0]["capacity"] == math.ceil(2 / 4 * moes[0].eval_capacity_factor)
    assert torch.equal(a["records"][0]["idx"][:, 1], torch.full((2,), -1, dtype=torch.int32, device="cuda"))
    from llavamod import kernels as K
    logits_a = K.linear(a["hidden"].reshape(2, -1), student.lm_head.weight).float()
    assert torch.equal(logits_a, b.logits.reshape(2, -1))
    assert cache.lengths == cache2.lengths
    for li in range(len(cache.k)):
        assert torch.equal(cache[li][0], cache2[li][0]) and torch.equal(cache[li][1], cache2[li][1])
    # as an assistant, a top-1 student leaves the teacher's greedy tokens unchanged
    one_ids, one_img = batch["input_ids"][:1], batch["images"][:1]
    want = teacher.generate(one_ids, images=one_img, max_new_tokens=12, use_cache=True)
    got = teacher.generate(one_ids, images=one_img, max_new_tokens=12, use_cache=True, assistant_model=student, num_assistant_tokens=3)
    assert torch.equal(got, want)
