"""Residual-MoE (--use_residual True) on the GPU: the two mix kernels element by element against float64, the whole residual block stage by
stage at config 2, a tiny residual student against oracle autograd, graphs, the training entry points with save / reload, and decoding."""
import json
import math
import os

import pytest
import torch

from oracle import restated as R
from tests import helpers as Hh
from tests import moe_residual_oracle as O

pytestmark = pytest.mark.gpu
bf = torch.bfloat16


def mix_inputs(S, H, seed, saturate=False, dropped=()):
    """x, moe, mlp, res [S,H] bf16 and a coefficient (wc [2,H], bc [2]).  saturate: rows 0 and 1 (when present) push z apart by
    hundreds, so c is exactly (1, 0) and (0, 1); dropped: token rows whose routed output is 0 (both choices dropped)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(S, H, device="cuda", generator=g).to(bf)
    moe = torch.randn(S, H, device="cuda", generator=g).to(bf)
    mlp = (torch.randn(S, H, device="cuda", generator=g) * 3).to(bf)
    res = torch.randn(S, H, device="cuda", generator=g).to(bf)
    wc = (torch.randn(2, H, device="cuda", generator=g) / math.sqrt(H)).to(bf)
    bc = (torch.randn(2, device="cuda", generator=g) * 0.1).to(bf)
    if saturate:
        wc[0, :8] = 1.0
        wc[1, :8] = -1.0
        x[0, :8] = 64.0
        if S > 1:
            x[1, :8] = -64.0
    for s in dropped:
        if s < S:
            moe[s] = 0
    return x, moe, mlp, res, wc, bc


MIX_S = [1, 8, 2047, 2048, 4096]
MIX_H = [1024, 2048]                          # config 2 (Qwen1.5-0.5B) and the 1.8B hidden size


@pytest.mark.parametrize("H", MIX_H)
@pytest.mark.parametrize("S", MIX_S)
def test_mix_forward_against_float64(S, H):
    from llavamod import kernels as K
    x, moe, mlp, res, wc, bc = mix_inputs(S, H, S + H, saturate=True, dropped=(2, S - 1))
    with Hh.poisoned_uninitialised_memory():
        out, coef = K.moe_residual_mix(x, moe, mlp, res, wc, bc)
        torch.cuda.synchronize()
    ref = O.mix_reference_fp64(x, moe, mlp, res, wc, bc, coef)
    Hh.check_moe("coef", coef, *ref["coef"])
    Hh.check_moe("out", out, ref["out"][0])
    assert coef[0].tolist() == [1.0, 0.0]
    if S > 1:
        assert coef[1].tolist() == [0.0, 1.0]
    # a token whose two choices were both dropped: only c1 * mlp passes
    s = S - 1
    want = (res[s].float() + (mlp[s].float() * coef[s, 1].float()).to(bf).float()).to(bf)
    assert torch.equal(out[s], want)
    out2, coef2 = K.moe_residual_mix(x, moe, mlp, res, wc, bc)
    assert torch.equal(out, out2) and torch.equal(coef, coef2)


@pytest.mark.parametrize("H", MIX_H)
@pytest.mark.parametrize("S", [1, 8, 2048, 4096])
def test_mix_backward_against_float64(S, H):
    from llavamod import kernels as K
    x, moe, mlp, res, wc, bc = mix_inputs(S, H, 7 * S + H, saturate=True, dropped=(2,))
    _, coef = K.moe_residual_mix(x, moe, mlp, res, wc, bc)
    gen = torch.Generator(device="cuda").manual_seed(S)
    g = (torch.randn(S, H, device="cuda", generator=gen) * 0.1).to(bf)
    old_w = (torch.randn(2, H, device="cuda", generator=gen) * 0.01).to(bf)
    old_b = (torch.randn(2, device="cuda", generator=gen) * 0.01).to(bf)
    runs = []
    for _ in range(2):
        dwc, dbc = old_w.clone(), old_b.clone()
        with Hh.poisoned_uninitialised_memory():
            d = K.moe_residual_mix_bwd(g, x, moe, mlp, coef, wc, dwc, dbc)
            torch.cuda.synchronize()
        runs.append((d, dwc, dbc))
    d, dwc, dbc = runs[0]
    ref = O.mix_bwd_reference_fp64(g, x, moe, mlp, coef, wc, d["dz"], old_w, old_b)
    for name in ("d_moe", "d_mlp"):
        Hh.check_moe(name, d[name], ref[name][0])
    for name, got in (("dz", d["dz"]), ("dx", d["dx"]), ("dwc", dwc), ("dbc", dbc)):
        Hh.check_moe(name, got, *ref[name])
    assert float(d["dz"][0].abs().max()) == 0.0                 # c = (1, 0) exactly: the softmax passes no gradient
    # the reduction is deterministic: a second run gives the same bytes
    d2, dwc2, dbc2 = runs[1]
    for k in d:
        assert torch.equal(d[k], d2[k]), k
    assert torch.equal(dwc, dwc2) and torch.equal(dbc, dbc2)
    # frozen coefficient: nothing written to its gradient, every other output the same
    fw, fb = old_w.clone(), old_b.clone()
    d3 = K.moe_residual_mix_bwd(g, x, moe, mlp, coef, wc, None, None)
    assert torch.equal(fw, old_w) and torch.equal(fb, old_b)
    for k in d:
        assert torch.equal(d[k], d3[k]), k


# ---------------------------------------------------------------------------------------------------------------------------------
# the whole residual block at config 2, stage by stage
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [2, 1])
def test_residual_block_stage_by_stage(k):
    from llavamod import kernels as K
    S, H, I, E, cf = 2048, 1024, 2816, 4, 0.8
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(11 + k)
    x = torch.randn(S, H, device=dev, generator=g)
    x[:, 0] += 3.0
    x = x.to(bf)
    wg = torch.randn(E, H, device=dev, generator=g) * 0.05
    wg[:2, 0] = 2.0                               # experts 0 and 1 draw most tokens and overflow: some tokens lose every choice
    noise = torch.rand(S, E, device=dev, generator=g) if k == 1 else R.gumbel_noise((S, E)).to(dev)
    w_gu = (torch.randn(E, 2 * I, H, device=dev, generator=g) / math.sqrt(H)).to(bf)
    w_dn = (torch.randn(E, H, I, device=dev, generator=g) / math.sqrt(I)).to(bf)
    r_gu = (torch.randn(2 * I, H, device=dev, generator=g) / math.sqrt(H)).to(bf)
    r_dn = (torch.randn(H, I, device=dev, generator=g) / math.sqrt(I)).to(bf)
    wc = (torch.randn(2, H, device=dev, generator=g) / math.sqrt(H)).to(bf)
    bc = (torch.randn(2, device=dev, generator=g) * 0.1).to(bf)
    res = torch.randn(S, H, device=dev, generator=g).to(bf)
    dout = (torch.randn(S, H, device=dev, generator=g) * 0.1).to(bf)
    old = dict(wg=torch.randn(E, H, device=dev, generator=g) * 1e-2,
               w_gu=(torch.randn(E, 2 * I, H, device=dev, generator=g) * 1e-2).to(bf),
               w_dn=(torch.randn(E, H, I, device=dev, generator=g) * 1e-2).to(bf),
               r_gu=(torch.randn(2 * I, H, device=dev, generator=g) * 1e-2).to(bf),
               r_dn=(torch.randn(H, I, device=dev, generator=g) * 1e-2).to(bf),
               wc=(torch.randn(2, H, device=dev, generator=g) * 1e-2).to(bf), bc=(torch.randn(2, device=dev, generator=g) * 1e-2).to(bf))
    gl = torch.tensor(0.37, device=dev)
    grads = {n: v.clone() for n, v in old.items()}
    st = K.moe_residual_forward_stages(x, res, wg, w_gu, w_dn, noise, cf, 0, r_gu, r_dn, wc, bc, k)
    bw = K.moe_residual_backward_stages(st, x, wg, w_gu, w_dn, r_gu, r_dn, wc, dout, gl, grads)
    # the routed part is the plain MoE path with no residual, bit for bit, forward and backward (dres as its extra addend)
    plain = K.moe_forward_stages(x, None, wg, w_gu, w_dn, noise, cf, 0, k)
    assert torch.equal(plain["out"], st["moe"]) and torch.equal(plain["row"], st["row"])
    pg = {n: old[n].clone() for n in ("wg", "w_gu", "w_dn")}
    pb = K.moe_backward_stages(plain, x, wg, w_gu, w_dn, bw["mix"]["d_moe"], gl, pg, dres=bw["dres"])
    assert torch.equal(pb["dx"], bw["dx"])
    for n in pg:
        assert torch.equal(pg[n], grads[n]), n
    # some tokens lost both choices (k = 2) or their only one (k = 1), and their moe rows are zero
    lost = (st["row"] < 0).all(1) if k == 2 else st["row"][:, 0] < 0
    assert bool(lost.any()) and float(st["moe"][lost].float().abs().max()) == 0.0
    # the dense MLP against float64
    xd = x.double()
    h1 = xd @ r_gu.double().t()
    Hh.check_moe("mlp_h1", st["mlp_h1"], h1, Hh._gemm_tol(h1, xd.abs() @ r_gu.double().abs().t(), H))
    hk = st["mlp_h1"].double()
    gg, uu = hk[:, :I], hk[:, I:]
    sg = torch.sigmoid(gg)
    act = gg * sg * uu
    Hh.check_moe("mlp_act", st["mlp_act"], act, (2.0 ** -7 + 2.0 ** -16) * act.abs())
    ad = st["mlp_act"].double()
    y = ad @ r_dn.double().t()
    Hh.check_moe("mlp", st["mlp"], y, Hh._gemm_tol(y, ad.abs() @ r_dn.double().abs().t(), I))
    # the mix
    ref = O.mix_reference_fp64(x, st["moe"], st["mlp"], res, wc, bc, st["coef"])
    Hh.check_moe("coef", st["coef"], *ref["coef"])
    Hh.check_moe("out", st["out"], ref["out"][0])
    rb = O.mix_bwd_reference_fp64(dout, x, st["moe"], st["mlp"], st["coef"], wc, bw["mix"]["dz"], old["wc"], old["bc"])
    for n in ("d_moe", "d_mlp"):
        Hh.check_moe(n, bw["mix"][n], rb[n][0])
    Hh.check_moe("dz", bw["mix"]["dz"], *rb["dz"])
    Hh.check_moe("g_wc", grads["wc"], *rb["dwc"])
    Hh.check_moe("g_bc", grads["bc"], *rb["dbc"])
    # the dense MLP backward: dh1, the accumulated dx addend, the two weight gradients
    dm = bw["mix"]["d_mlp"].double()
    dact = dm @ r_dn.double()
    dact_tol = Hh._gemm_tol(dact, dm.abs() @ r_dn.double().abs(), H)
    cg, cu = uu * sg * (1 + gg * (1 - sg)), gg * sg
    dh1 = torch.cat([dact * cg, dact * cu], 1)
    derr = dact_tol + 2.0 ** -16 * dact.abs()
    Hh.check_moe("mlp_dh1", bw["mlp_dh1"], dh1, 2.0 ** -8 * dh1.abs() + (1 + 2.0 ** -8) * torch.cat([derr * cg.abs(), derr * cu.abs()], 1))
    dhk = bw["mlp_dh1"].double()
    zk, wcd = bw["mix"]["dz"].double(), wc.double()
    dres = zk @ wcd + dhk @ r_gu.double()
    maj = zk.abs() @ wcd.abs() + dhk.abs() @ r_gu.double().abs()
    Hh.check_moe("dres", bw["dres"], dres, 2.0 ** -7 * dres.abs() + 2 * Hh._gemm_tol(dres, maj, 2 * I) + 2.0 ** -8 * maj)
    for n, a, b_ in (("r_dn", bw["mix"]["d_mlp"], st["mlp_act"]), ("r_gu", bw["mlp_dh1"], x)):
        A, B = a.double(), b_.double()
        want = A.t() @ B + old[n].double()
        Hh.check_moe("g_" + n, grads[n], want, Hh._gemm_tol(want, A.abs().t() @ B.abs() + old[n].double().abs(), S))
    # ResidualMoEFn and the no-grad path give the stage functions' bytes
    g2 = {n: v.clone() for n, v in old.items()}
    xg, rg = x.clone().requires_grad_(True), res.clone().requires_grad_(True)
    out, l_aux = K.ResidualMoEFn.apply(xg, rg, wg, w_gu, w_dn, noise, cf, 0, r_gu, r_dn, wc, bc, g2, k)
    ((out.float() * dout.float()).sum() + 0.37 * l_aux).backward()
    assert torch.equal(out, st["out"]) and torch.equal(xg.grad, bw["dx"]) and torch.equal(rg.grad, dout)
    for n in g2:
        assert torch.equal(g2[n], grads[n]), n
    with torch.no_grad():
        out_ng, _, rec = K.moe_residual_forward_nograd(x, res, wg, w_gu, w_dn, noise, cf, 0, r_gu, r_dn, wc, bc, k)
    assert torch.equal(out_ng, st["out"]) and torch.equal(rec["coef"], st["coef"])


# ---------------------------------------------------------------------------------------------------------------------------------
# a tiny residual student end to end
# ---------------------------------------------------------------------------------------------------------------------------------
def residual_pair(seed=0, vocab=512, k=2):
    from llavamod.model import synthetic as S
    teacher = S.make_teacher(dict(S.ARCH["tiny"], vocab_size=vocab, intermediate_size=320), "tiny", seed=seed)
    student = S.make_student(dict(S.ARCH["tiny"], vocab_size=vocab), "tiny", seed=seed + 1, margs=S.moe_args(top_k=k, use_residual=True),
                             share_tower_with=teacher)
    return student, teacher


def noises(student, B, Tn, seed, k=2):
    g = torch.Generator().manual_seed(seed)
    n_moe = sum(1 for l in student.model.layers if hasattr(l.mlp, "deepspeed_moe"))
    if k == 1:
        return [torch.rand(B * Tn, 4, generator=g) for _ in range(n_moe)]
    return [R.gumbel_noise((B * Tn, 4), generator=g) for _ in range(n_moe)]


def oracle_student(student, batch, noise, sd=None, record=None, k=2):
    lc, cc = Hh.cfgs_of(student)
    lc.top_k = k
    sd = sd if sd is not None else Hh.oracle_state(student)
    return O.llava_forward(sd, lc, cc, batch["input_ids"], batch["attention_mask"], batch["labels"],
                           [im.float() for im in batch["images"]], noise, record), lc


@pytest.mark.parametrize("k", [2, 1])
def test_tiny_residual_student_matches_oracle_autograd(k):
    student, teacher = residual_pair(k=k)
    moes = [l.mlp for l in student.model.layers if hasattr(l.mlp, "deepspeed_moe")]
    assert moes and all(m.use_residual and m.k == k for m in moes)
    # fresh up-cycling makes every expert a copy of the dense MLP, so for top-2 moe == mlp up to rounding and the coefficient's true
    # gradient cancels to ~0; move the dense MLP away from the experts so the comparison measures the gradient, not rounding noise
    g = torch.Generator(device="cuda").manual_seed(40 + k)
    with torch.no_grad():
        for m in moes:
            for t in (m.mlp.gu_weight, m.mlp.down_proj.weight):
                t.add_((torch.randn(t.shape, device="cuda", generator=g) * 0.02).to(t.dtype))
    batch, _ = Hh.tiny_batch(student, seed=4)
    noise = noises(student, 2, 55, 5, k)
    rec = []
    with torch.no_grad():
        r = student.forward_hidden(input_ids=batch["input_ids"], attention_mask=batch["attention_mask"], labels=batch["labels"],
                                   images=batch["images"], moe_noise=[n.cuda() for n in noise])
    oracle_student(student, batch, noise, record=rec, k=k)
    assert len(r["records"]) == len(rec) == len(moes)
    for gr, o in zip(r["records"], rec):                # routing agrees before anything is compared
        assert torch.equal(gr["idx"][:, 0].long().cpu(), o["idx1"])
        assert torch.equal((gr["row"][:, 0] >= 0).cpu(), o["keep1"])
        torch.testing.assert_close(gr["coef"].float().cpu(), o["coef"].float(), atol=2e-2, rtol=0)
    sd_s = Hh.oracle_state(student)
    keys = [n for n, p in student.named_parameters() if p.requires_grad]
    assert any(".mlp.mlp.gate_proj." in n for n in keys) and any(".mlp.coefficient.bias" in n for n in keys)
    for n in keys:
        sd_s[n].requires_grad_(True)
    with torch.no_grad():
        t_out, _ = Hh.oracle_forward(teacher, batch)
    s_out, lc = oracle_student(student, batch, noise, sd=sd_s, k=k)
    ref_loss, ref_m = R.mimic_compute_loss(s_out, t_out["logits"], "kd_lm", True, False, lc.kd_vocab)
    ref_loss.backward()
    tr = Hh.make_trainer(student, teacher, "kd_lm")
    opt = tr.create_optimizer()
    opt.zero_grad()
    loss, m = tr.compute_loss(student, dict(batch, moe_noise=[n.cuda() for n in noise]), return_outputs=True)
    for n in ("loss", "loss/align", "loss/lm", "loss/moe_balance"):
        assert abs(float(m[n]) - float(ref_m[n])) < 1e-2 * abs(float(ref_m[n])) + 1e-4, (n, float(m[n]), float(ref_m[n]))
    loss.backward()
    torch.cuda.synchronize()
    for n, p in student.named_parameters():
        if p.requires_grad:
            gr, rr = p.grad.float().cpu(), sd_s[n].grad
            rel = (gr - rr).norm().item() / (rr.norm().item() + 1e-12)
            assert rel < 0.08, (n, rel)


def test_graphed_micro_batch_equals_eager():
    losses = {}
    for graphs in (False, True):
        student, teacher = residual_pair(seed=2)
        tr = Hh.make_trainer(student, teacher, "kd_lm", accum=1, lr=0.0)
        tr.use_cuda_graphs = graphs
        got = []
        for i in range(5):
            batch, _ = Hh.tiny_batch(student, seed=60 + i)
            got.append(float(tr.training_step(student, dict(batch, moe_noise=[n.cuda() for n in noises(student, 2, 55, 70 + i)]))))
        if graphs:
            assert tr._graphs, "no graph was captured"
        losses[graphs] = got
    assert losses[True] == losses[False], losses


def test_align_then_dpo_entry_points_with_residual(tmp_path, golden_dir):
    from llavamod.train import align_train, dpo_train
    from tests.test_entrypoints_gpu import _check_final_save, _common_flags, _save_tiny_checkpoints
    policy, teacher, tower, tok = _save_tiny_checkpoints(str(tmp_path), golden_dir)
    out = str(tmp_path / "tiny-qwen1.5-residual")            # the FineTune class is picked by the path's family name
    argv = _common_flags(policy, teacher, tower, out, golden_dir, "data_sft.json") + ["--loss_type", "kd_lm", "--learning_rate", "1e-3"]
    argv[argv.index("--use_residual") + 1] = "True"
    policy_before = torch.load(os.path.join(policy, "pytorch_model.bin"), map_location="cpu", weights_only=True)
    tr = align_train.train(argv)
    assert tr.state.global_step == 2
    _check_final_save(out, tr, (2,))
    sd = torch.load(os.path.join(out, "pytorch_model.bin"), map_location="cpu", weights_only=True)
    p = "model.layers.0.mlp."
    keys = [n for n in sd if n.startswith(p)]
    want = ([p + "deepspeed_moe.gate.wg.weight"] + [p + "deepspeed_moe.experts.deepspeed_experts.%d.%s.weight" % (e, w)
                                                    for e in range(4) for w in ("gate_proj", "up_proj", "down_proj")]
            + [p + "mlp.%s.weight" % w for w in ("gate_proj", "up_proj", "down_proj")] + [p + "coefficient.weight", p + "coefficient.bias"])
    assert keys == want
    assert sd[p + "coefficient.weight"].shape == (2, 128) and sd[p + "coefficient.weight"].dtype == bf and sd[p + "coefficient.bias"].shape == (2,)
    # --train_modules matched mlp.gate_proj on the dense module before wrapping, and the new coefficient trains: both moved
    assert not torch.equal(sd[p + "mlp.gate_proj.weight"], policy_before[p + "gate_proj.weight"])
    assert json.load(open(os.path.join(out, "config.json")))["moe"]["use_residual"] is True
    from llavamod.model import EvalLLaVAMoDQwen1_5ForCausalLM
    m = EvalLLaVAMoDQwen1_5ForCausalLM.from_pretrained(out)
    sd_m = m.state_dict()
    assert [n for n in sd_m if n.startswith(p)] == want
    for n in want:
        assert torch.equal(sd_m[n].cpu(), sd[n]), n
    # the preference stage from that checkpoint (FineTune class): the coefficient matches no --train_modules name and stays frozen
    tok.save_pretrained(out)                                 # the final save holds the weights and config; the tokenizer goes beside them
    out2 = str(tmp_path / "out_residual_dpo")
    argv2 = _common_flags(out, teacher, tower, out2, golden_dir, "data_dpo.json") + ["--loss_type", "sigmoid", "--learning_rate", "2e-4",
                                                                                        "--moe_finetune", "True"]
    argv2[argv2.index("--use_residual") + 1] = "True"
    tr2 = dpo_train.train(argv2)
    assert tr2.state.global_step == 1
    named = dict(tr2.model.named_parameters())
    assert not named[p + "coefficient.weight"].requires_grad and not named[p + "coefficient.bias"].requires_grad
    assert named[p + "mlp.gate_proj.weight"].requires_grad
    sd2 = torch.load(os.path.join(out2, "pytorch_model.bin"), map_location="cpu", weights_only=True)
    assert [n for n in sd2 if n.startswith(p)] == want
    assert torch.equal(sd2[p + "coefficient.weight"], sd[p + "coefficient.weight"])


def test_cached_padded_and_assisted_decoding():
    student, teacher = residual_pair(seed=6)
    student.eval()
    moes = [l.mlp for l in student.model.layers if hasattr(l.mlp, "deepspeed_moe")]
    batch, _ = Hh.tiny_batch(student, B=2, Tt=20, seed=7)
    ids, images = batch["input_ids"].cuda(), batch["images"]
    Tn = 20 - 1 + 16
    g = torch.Generator().manual_seed(8)
    cache = student.new_kv_cache(2, 64)
    pre = [R.gumbel_noise((2 * Tn, 4), generator=g).cuda() for _ in moes]
    tok = torch.randint(0, 512, (2, 1), generator=g).cuda()
    step = [R.gumbel_noise((2, 4), generator=g).cuda() for _ in moes]
    with torch.no_grad():
        student.forward_hidden(input_ids=ids, images=images, moe_noise=pre, cache=cache)
        a = student.forward_hidden(input_ids=tok, moe_noise=step, cache=cache)
        cache2 = student.new_kv_cache(2, 64)
        student.forward_hidden(input_ids=ids, images=images, moe_noise=pre, cache=cache2)
        b = student(input_ids=tok, past_key_values=cache2, use_cache=True, moe_noise=step, return_dict=True)
    assert a["records"][0]["coef"].shape == (2, 2)
    from llavamod import kernels as K
    logits_a = K.linear(a["hidden"].reshape(2, -1), student.lm_head.weight).float()
    assert torch.equal(logits_a, b.logits.reshape(2, -1))
    assert cache.lengths == cache2.lengths
    for li in range(len(cache.k)):
        assert torch.equal(cache[li][0], cache2[li][0]) and torch.equal(cache[li][1], cache2[li][1])
    # a padded batch decodes (prompts of different lengths, with and without the cache)
    pb, _ = Hh.tiny_batch(student, B=2, Tt=20, seed=9, pad=(0, 6))
    mask = pb["attention_mask"].cuda()
    out_c = student.generate(pb["input_ids"].cuda(), images=pb["images"], attention_mask=mask, max_new_tokens=6, use_cache=True)
    assert out_c.shape[0] == 2 and out_c.shape[1] >= 1
    # as an assistant, a residual student leaves the teacher's greedy tokens unchanged
    one_ids, one_img = batch["input_ids"][:1], batch["images"][:1]
    want = teacher.generate(one_ids, images=one_img, max_new_tokens=12, use_cache=True)
    got = teacher.generate(one_ids, images=one_img, max_new_tokens=12, use_cache=True, assistant_model=student, num_assistant_tokens=3)
    assert torch.equal(got, want)


def test_plain_moe_state_dict_is_untouched():
    from llavamod.model import synthetic as S
    plain = S.make_student(dict(S.ARCH["tiny"], vocab_size=512), "tiny", seed=1, margs=S.moe_args())
    resid = S.make_student(dict(S.ARCH["tiny"], vocab_size=512), "tiny", seed=1, margs=S.moe_args(use_residual=True))
    kp, kr = list(plain.state_dict()), list(resid.state_dict())
    assert not any(".mlp.mlp." in n or "coefficient" in n for n in kp)
    extra = [n for n in kr if n not in kp]
    assert sorted(extra) == sorted("model.layers.0.mlp.%s" % s for s in
                                   ("mlp.gate_proj.weight", "mlp.up_proj.weight", "mlp.down_proj.weight", "coefficient.weight", "coefficient.bias"))
    assert [n for n in kr if n in kp] == kp
    assert all(not l.mlp.use_residual for l in plain.model.layers if hasattr(l.mlp, "deepspeed_moe"))
