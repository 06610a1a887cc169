"""Layer-level GPU-vs-oracle parity at BASELINE config-2 SHAPES (the tiny-config model tests never reach them):
one teacher layer (H 4096, I 11008, 32 heads x 128: CTA-pair GEMM at N 22016 / K 11008, fused SwiGLU epilogue, hd-128 attention at
T 2048), one student decoder layer forward+backward (H 1024, I 2816, hd 64: dgrad / wgrad GEMMs, attention backward), the student's
sparse-MoE block forward+backward (E 4, T 2048: router + grouped fwd / dgrad / wgrad at I 2816) and the loss head on the bench's
885 / 2048 supervised rows against the full vocabulary (151936: dynamic-extent GEMMs, split-K lm_head dgrad, fused KL+CE).

Oracle = oracle/restated.py in fp32 on the CPU with the SAME bf16-rounded weights and inputs (seconds per layer).  Tolerances are
relative Frobenius errors: bf16 activations / gradients against an fp32 computation give ~0.4 % per rounding stage.
"""
import pytest
import torch

from oracle import restated as R

pytestmark = pytest.mark.gpu
T2 = 2048


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def build_lm(hidden, inter, heads, layers=1, vocab=256, seed=0, moe=None, train=()):
    """A bare Qwen2Model of the build at the given layer shape + the oracle's state dict of the same (bf16-rounded) weights."""
    from llavamod.model.language_model.qwen2_core import MoE, Qwen2Config, Qwen2Model
    torch.manual_seed(seed)
    cfg = Qwen2Config(vocab_size=vocab, hidden_size=hidden, intermediate_size=inter, num_hidden_layers=layers, num_attention_heads=heads,
                      num_key_value_heads=heads, rope_theta=1e6, rms_norm_eps=1e-6, max_position_embeddings=4096)
    m = Qwen2Model(cfg, device="cuda", dtype=torch.bfloat16)
    with torch.no_grad():
        for n, p in m.named_parameters():                  # non-trivial norms / biases
            if n.endswith("layernorm.weight") or n == "norm.weight":
                p.copy_((1 + 0.1 * torch.randn_like(p.float())).to(p.dtype))
            if n.endswith("bias"):
                p.copy_((0.1 * torch.randn_like(p.float())).to(p.dtype))
    for p in m.parameters():
        p.requires_grad = False
    moe_layers = []
    if moe:
        for i, layer in enumerate(m.layers):
            layer.mlp = MoE(cfg, layer.mlp, num_experts=moe, capacity_factor=1.5, eval_capacity_factor=2.0, min_capacity=0)
            moe_layers.append(i)
    for n, p in m.named_parameters():
        p.requires_grad = any(t in n for t in train)
    lc = R.LMCfg(hidden=hidden, inter=inter, layers=layers, heads=heads, kv_heads=heads, vocab=vocab, rope_theta=1e6, eps=1e-6,
                 moe_layers=moe_layers, num_experts=moe or 4, capacity_factor=1.5, min_capacity=0)
    sd = {"model." + k: v.detach().float().cpu() for k, v in m.state_dict().items()}
    return m, lc, sd


def test_teacher_layer_forward_at_7b_shape():
    """Frozen Qwen-1.5-7B decoder layer: qkv GEMM (+bias) -> RoPE -> hd-128 attention -> o_proj -> fused-residual RMSNorm ->
    gate|up GEMM with the SwiGLU epilogue (CTA-pair kernel, N 22016) -> down GEMM (K 11008) -> final norm."""
    m, lc, sd = build_lm(4096, 11008, 32, seed=1)
    g = torch.Generator().manual_seed(11)
    x = torch.randn(1, T2, 4096, generator=g).to(torch.bfloat16)
    with torch.no_grad():
        from llavamod import _C
        n0 = _C.launch_count()
        out, _, _ = m(x.cuda())
        # rmsnorm, qkv GEMM with the RoPE epilogue, attention, o_proj, rmsnorm(+residual), gate|up GEMM with the SwiGLU epilogue, down GEMM,
        # final norm: the fused-epilogue paths are the ones that ran (separate rope / silu_mul launches would make it 10)
        assert _C.launch_count() - n0 == 8, _C.launch_count() - n0
        ref, _ = R.lm_forward(sd, lc, x.float(), None, None)
    assert rel(out, ref) < 1.2e-2, rel(out, ref)
    err = (out.float().cpu() - ref).abs()
    assert err.max().item() < 0.25 and err.mean().item() < 1.2e-2 * ref.abs().mean().item() + 1e-3


def test_student_layer_forward_backward_at_0p5b_shape():
    """Qwen-1.5-0.5B dense decoder layer with a trainable MLP (the recipe's --train_modules): forward, d(input) through the hd-64
    attention backward, and the gate|up / down weight gradients accumulated into the flat gradient arena."""
    from llavamod.train.engine import TrainState
    m, lc, sd = build_lm(1024, 2816, 16, seed=2, train=("mlp.gate_proj", "mlp.up_proj", "mlp.down_proj"))
    st = TrainState(m, max_grad_norm=0.0)
    st.zero_grad()
    g = torch.Generator().manual_seed(12)
    x = torch.randn(1, T2, 1024, generator=g).to(torch.bfloat16)
    go = (torch.randn(1, T2, 1024, generator=g) / 32).to(torch.bfloat16)
    xd = x.cuda().requires_grad_(True)
    out, _, _ = m(xd)
    (out.float() * go.cuda().float()).sum().backward()
    torch.cuda.synchronize()
    keys = [k for k in sd if any(t in k for t in ("mlp.gate_proj", "mlp.up_proj", "mlp.down_proj"))]
    for k in keys:
        sd[k].requires_grad_(True)
    xo = x.float().requires_grad_(True)
    ref, _ = R.lm_forward(sd, lc, xo, None, None)
    (ref * go.float()).sum().backward()
    assert rel(out, ref) < 1.2e-2
    assert rel(xd.grad, xo.grad) < 2.5e-2, rel(xd.grad, xo.grad)
    grads = {n: p.grad for n, p in m.named_parameters() if p.requires_grad}
    assert len(grads) == 3
    for n, gq in grads.items():
        assert rel(gq, sd["model." + n].grad) < 2e-2, (n, rel(gq, sd["model." + n].grad))


def test_moe_block_forward_backward_at_config2_shape():
    """The student's sparse block alone (x given, so routing is decided from identical logits): 2048 tokens, H 1024, I 2816, 4 experts,
    capacity 1536 -- router, token scatter, grouped fwd / dgrad / wgrad GEMMs on ragged 128-aligned groups, combine."""
    from llavamod import kernels as K
    S, H, I, E, cf = T2, 1024, 2816, 4, 1.5
    g = torch.Generator().manual_seed(13)
    cfg = R.LMCfg(hidden=H, inter=I, layers=1, heads=16, kv_heads=16, vocab=64, moe_layers=[0], num_experts=E, capacity_factor=cf)
    pre = "m."
    sd = {pre + "gate.wg.weight": torch.randn(E, H, generator=g) * 0.1}
    for e in range(E):
        sd[pre + f"experts.deepspeed_experts.{e}.gate_proj.weight"] = (torch.randn(I, H, generator=g) * 0.03).to(torch.bfloat16).float()
        sd[pre + f"experts.deepspeed_experts.{e}.up_proj.weight"] = (torch.randn(I, H, generator=g) * 0.03).to(torch.bfloat16).float()
        sd[pre + f"experts.deepspeed_experts.{e}.down_proj.weight"] = (torch.randn(H, I, generator=g) * 0.03).to(torch.bfloat16).float()
    x = torch.randn(S, H, generator=g).to(torch.bfloat16)
    x[:, 0] += 1.5                                         # skew the gate so that one expert overflows its capacity (drops happen)
    sd[pre + "gate.wg.weight"][0, 0] += 0.6
    res = torch.randn(S, H, generator=g).to(torch.bfloat16)
    noise = R.gumbel_noise((S, E), g)
    go = (torch.randn(S, H, generator=g) / 32).to(torch.bfloat16)
    xd, rd = x.cuda().requires_grad_(True), res.cuda().requires_grad_(True)
    wg = sd[pre + "gate.wg.weight"].cuda()
    w_gu = torch.stack([torch.cat([sd[pre + f"experts.deepspeed_experts.{e}.gate_proj.weight"],
                                   sd[pre + f"experts.deepspeed_experts.{e}.up_proj.weight"]]) for e in range(E)]).to(torch.bfloat16).cuda()
    w_dn = torch.stack([sd[pre + f"experts.deepspeed_experts.{e}.down_proj.weight"] for e in range(E)]).to(torch.bfloat16).cuda()
    grads = dict(wg=torch.zeros_like(wg), w_gu=torch.zeros_like(w_gu), w_dn=torch.zeros_like(w_dn))
    out, l_aux = K.MoEFn.apply(xd, rd, wg, w_gu, w_dn, noise.cuda(), cf, 0, grads)
    (out.float() * go.cuda().float()).sum().add(0.37 * l_aux).backward()
    torch.cuda.synchronize()
    xo, ro = x.float().requires_grad_(True), res.float().requires_grad_(True)
    sdo = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    y, la, _ = R.moe_layer(sdo, pre, cfg, xo, noise)
    ((ro + y) * go.float()).sum().add(0.37 * la).backward()
    # integer record: bit exact (and the overflow case is really exercised)
    r = K.moe_route_scatter(x.cuda(), wg, noise.cuda(), cf, 0)
    o = R.top2gating(r["logits"].cpu(), noise, cf, 0)
    assert torch.equal(r["idx"].cpu().long()[:, 0], o["idx1"]) and torch.equal(r["idx"].cpu().long()[:, 1], o["idx2"])
    assert torch.equal(r["row"].cpu()[:, 0] >= 0, o["keep1"]) and torch.equal(r["row"].cpu()[:, 1] >= 0, o["keep2"])
    assert int((~o["keep1"]).sum() + (~o["keep2"]).sum()) > 0
    assert abs(l_aux.item() - la.item()) < 1e-4 * abs(la.item())
    assert rel(rd.grad, ro.grad) < 1e-6 + 2.0 ** -8
    # element by element: every stage against the float64 reference from the kernels' previous stage (a missing or misrouted token row,
    # about 2 % of the Frobenius norm here, fails), and MoEFn gives the stage functions' bytes
    from tests.helpers import check_moe_stages, moe_reference_fp64, moe_run_stages
    zeros = {k: torch.zeros_like(v) for k, v in grads.items()}
    k = moe_run_stages(xd.detach(), rd.detach(), wg, w_gu, w_dn, noise.cuda(), cf, 0, go.cuda(), 0.37, zeros)
    assert torch.equal(out, k["out"]) and torch.equal(xd.grad, k["dx"])
    for name in ("wg", "w_gu", "w_dn"):
        assert torch.equal(grads[name], k["g_" + name]), name
    ref = moe_reference_fp64(xd.detach(), rd.detach(), wg, w_gu, w_dn, noise, cf, 0, dout=go.cuda(), g_laux=0.37, old=zeros, k=k,
                             store=torch.float32)
    check_moe_stages(k, ref, E, zeros)


def test_loss_head_full_vocab_on_supervised_rows():
    """lm_head (V 151936, tied-embedding shape [V, 1024]) + mimic KL + shifted CE on the bench's label layout (40 % of the text ids
    masked -> 885 of 2048 post-splice rows supervised): compact head (row gather, dynamic-extent GEMMs, split-K dgrad, fused loss
    kernel) against the oracle's fp32 log-softmax formulas on the same rows; and the compact head against the dense head."""
    from llavamod import kernels as K
    V, H, Ht = 151936, 1024, 512
    g = torch.Generator().manual_seed(14)
    hs = torch.randn(T2, H, generator=g).to(torch.bfloat16)
    ht = torch.randn(T2, Ht, generator=g).to(torch.bfloat16)
    ws = (torch.randn(V, H, generator=g) * 0.02).to(torch.bfloat16)
    wt = (torch.randn(V, Ht, generator=g) * 0.05).to(torch.bfloat16)
    labels = torch.randint(0, V, (1, T2), generator=g)
    labels[0, :1164] = -100                               # 576 image positions + 40 % of 1473 text ids: 884 supervised + 1 CE-only row
    hsd = hs.cuda().requires_grad_(True)
    wsd = ws.cuda()
    head_grad = torch.zeros_like(wsd)
    lab = labels.cuda()
    rows = K.active_rows(lab.reshape(-1), T2)
    assert int(rows[1]) == 885
    t_logits = K.gemm(K.gather_rows(ht.cuda(), *rows), wt.cuda(), m_dev=rows[1])
    total, align, ce = K.distill_head(hsd.view(1, T2, H), wsd, t_logits, lab, V, 1.0, 1.0, False, head_grad, rows=rows)
    total.backward()
    torch.cuda.synchronize()
    # oracle on the active rows only (the masked rows contribute exact zeros to every sum)
    act = rows[0][:885].cpu().long()
    ho = hs.float().requires_grad_(True)
    wo = ws.float().requires_grad_(True)
    s_log = ho[act] @ wo.t()
    with torch.no_grad():
        t_log = (ht.float()[act] @ wt.float().t()).to(torch.bfloat16).float()      # the teacher's logits are a bf16 tensor in the reference too
    logp = torch.log_softmax(s_log, -1)
    m_kd = (labels[0, act] != -100).float()
    x_t = (torch.softmax(t_log, -1) * logp).sum(-1)
    align_o = -(x_t * m_kd).sum() / m_kd.sum()
    nxt = torch.cat([labels[0, 1:], torch.full((1,), -100)])[act]
    m_ce = nxt != -100
    ce_o = -(logp[m_ce, nxt[m_ce]]).sum() / m_ce.sum()
    (align_o + ce_o).backward()
    assert abs(float(align) - float(align_o)) < 2e-3 * abs(float(align_o)), (float(align), float(align_o))
    assert abs(float(ce) - float(ce_o)) < 2e-3 * abs(float(ce_o)), (float(ce), float(ce_o))
    assert rel(hsd.grad, ho.grad) < 2e-2, rel(hsd.grad, ho.grad)
    assert rel(head_grad, wo.grad) < 2e-2, rel(head_grad, wo.grad)
    assert float(hsd.grad[:1163].abs().max()) == 0.0      # unsupervised rows receive exact zeros
    # dense head (all rows through the GEMMs and the kernel) gives the same numbers
    hs2 = hs.cuda().requires_grad_(True)
    hg2 = torch.zeros_like(wsd)
    t_dense = K.gemm(ht.cuda(), wt.cuda())
    tot2, al2, ce2 = K.distill_head(hs2.view(1, T2, H), wsd, t_dense, lab, V, 1.0, 1.0, False, hg2, rows=None)
    tot2.backward()
    assert abs(float(al2) - float(align)) < 1e-5 * abs(float(align)) and abs(float(ce2) - float(ce)) < 1e-5 * abs(float(ce))
    assert rel(hs2.grad, hsd.grad) < 2e-3 and rel(hg2, head_grad) < 2e-3
