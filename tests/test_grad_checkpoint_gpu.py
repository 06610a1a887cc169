"""Gradient checkpointing (--gradient_checkpointing True): every decoder layer of the trained model runs as one checkpointed segment
(kernels.CheckpointFn) whose activations are recomputed in the backward.  The forward must give the bytes of the plain run, the recompute
the bytes of the first forward, and the gradients those of the plain run (byte for byte where the plain backward repeats its own bytes)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests import helpers as Hh  # noqa: E402

# kind -> (hidden, heads, kv heads) at the tiny / config-2 shapes, MoE width k (None: dense MLP), Residual-MoE
KINDS = {
    "dense": dict(tiny=(128, 2, 2), cfg2=(1024, 16, 16), k=None, res=False),
    "top2": dict(tiny=(128, 2, 2), cfg2=(1024, 16, 16), k=2, res=False),
    "top1": dict(tiny=(128, 2, 2), cfg2=(1024, 16, 16), k=1, res=False),
    "residual2": dict(tiny=(128, 2, 2), cfg2=(1024, 16, 16), k=2, res=True),
    "residual1": dict(tiny=(128, 2, 2), cfg2=(1024, 16, 16), k=1, res=True),
    "gqa_hd128": dict(tiny=(512, 4, 2), cfg2=(1024, 8, 2), k=None, res=False),
    "hd32": dict(tiny=(128, 4, 4), cfg2=(1024, 32, 32), k=2, res=False),
}
SHAPES = {"tiny": dict(inter=256, B=2, T=64), "cfg2": dict(inter=2816, B=2, T=1024)}
PADS = ("none", "left", "right")


def _decoder(kind, shape, layers=2, seed=0):
    from llavamod.model.language_model.qwen2_core import MoE, Qwen2Config, Qwen2Model
    H, nh, nkv = KINDS[kind][shape]
    cfg = Qwen2Config(vocab_size=64, hidden_size=H, intermediate_size=SHAPES[shape]["inter"], num_hidden_layers=layers,
                      num_attention_heads=nh, num_key_value_heads=nkv, rope_theta=1e6)
    torch.manual_seed(seed)
    m = Qwen2Model(cfg, device="cuda").train()
    with torch.no_grad():
        for layer in m.layers:                               # non-trivial norms and biases
            for t in (layer.input_layernorm.weight, layer.post_attention_layernorm.weight):
                t.uniform_(0.5, 1.5)
            layer.self_attn.qkv_bias.normal_(0.0, 0.05)
    k = KINDS[kind]["k"]
    if k is not None:
        for layer in m.layers:
            layer.mlp = MoE(cfg, expert=layer.mlp, num_experts=4, k=k, capacity_factor=1.5, min_capacity=4, use_residual=KINDS[kind]["res"])
    return m


def _mask(B, T, pad):
    if pad == "none":
        return None
    m = torch.ones(B, T, dtype=torch.bool, device="cuda")
    p = T // 5
    if pad == "left":
        m[1, :p] = False
    else:
        m[1, T - p:] = False
    return m


def _noise(m, S, seed):
    from llavamod.model.language_model.qwen2_core import MoE
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for layer in m.layers:
        if isinstance(layer.mlp, MoE):
            u = torch.rand(S, layer.mlp.num_experts, generator=g, device="cuda")
            out.append(u if layer.mlp.k == 1 else -torch.log(-torch.log(u.clamp(1e-20, 1.0 - 1e-7))))
    return out or None


def _arena(m, seed):
    """Gradient views of every trainable storage of the decoder: bf16 ones in a helpers.Arena, the fp32 router weights apart."""
    from llavamod.train.engine import _units
    units = [(s, mem) for s, mem in _units(m) if all(p.requires_grad for p in mem)]
    bf = [s for s, _ in units if s.dtype == torch.bfloat16]
    f32 = {id(s): torch.randn(s.shape, device="cuda") * 0.5 for s, _ in units if s.dtype == torch.float32}
    arena = Hh.Arena([tuple(s.shape) for s in bf], seed) if bf else None
    gv = dict(f32)
    if arena is not None:
        gv.update({id(s): v for s, v in zip(bf, arena.views)})
    m.grad_views = gv
    return arena, f32


class _Recorder:
    """Per checkpointed segment, the bytes of every call of its run (the first forward, then the recompute): the segment outputs and the
    q|k|v, gate|up pre-activations (h1) and SwiGLU outputs (act) the backward kernels read."""

    def __init__(self, monkeypatch):
        from llavamod import kernels as K
        self.calls, self.cur = {}, None
        orig_ckpt, orig_attn, orig_silu, orig_moe = K.checkpoint, K.attention, K.silu_mul, K.moe_forward_stages
        self.in_moe = False

        def checkpoint(run, *inputs):
            def rec_run(*xs):
                self.cur = []
                outs = run(*xs)
                self.calls.setdefault(id(rec_run), []).append(self.cur + [o.detach().clone() for o in outs])
                self.cur = None
                return outs
            return orig_ckpt(rec_run, *inputs)

        def attention(qkv, *a, **kw):
            if self.cur is not None:
                self.cur.append(qkv.detach().clone())
            return orig_attn(qkv, *a, **kw)

        def silu_mul(gu):
            act = orig_silu(gu)
            if self.cur is not None and not self.in_moe:
                self.cur += [gu.detach().clone(), act.detach().clone()]
            return act

        def moe_forward_stages(*a, **kw):
            self.in_moe = True
            try:
                st = orig_moe(*a, **kw)
            finally:
                self.in_moe = False
            if self.cur is not None:                # rows past offsets[E] are never written nor read (kernels.moe_forward_stages)
                n = int(st["offsets"][-1])
                self.cur += [st[k][:n].clone() for k in ("xp", "h1", "act", "y")] + [st[k].clone() for k in ("row", "w", "meta")]
            return st

        monkeypatch.setattr(K, "checkpoint", checkpoint)
        monkeypatch.setattr(K, "attention", attention)
        monkeypatch.setattr(K, "silu_mul", silu_mul)
        monkeypatch.setattr(K, "moe_forward_stages", moe_forward_stages)

    def check(self, tag, n_segments):
        assert len(self.calls) == n_segments, (tag, len(self.calls))
        for i, runs in enumerate(self.calls.values()):
            assert len(runs) == 2, f"{tag}: segment {i} ran {len(runs)} times (first forward + recompute expected)"
            Hh.same_bytes(f"{tag} segment {i} recompute", runs[0], runs[1])
        self.calls = {}


def _run(m, x, mask, noise, dout, ckpt, x_grad=True, arena=None, f32=None):
    """Decoder forward + backward of (dout, 0.01 per l_aux) -> [out, l_aux..., dx, grad views...]."""
    m.gradient_checkpointing = ckpt
    if arena is not None:
        arena.buf.copy_(arena.fresh)
    f32_0 = {k: v.clone() for k, v in (f32 or {}).items()}
    xi = x.clone().requires_grad_(x_grad)
    out, l_aux, _ = m(xi, mask, moe_noise=noise)
    outs, grads = [out] + list(l_aux), [dout] + [torch.full_like(l, 0.01) for l in l_aux]
    torch.autograd.backward([o for o in outs if o.requires_grad], [g for o, g in zip(outs, grads) if o.requires_grad])
    res = [out.detach().clone()] + [l.detach().clone() for l in l_aux]
    if x_grad:
        res.append(xi.grad.clone())
    if arena is not None:
        res += [v.clone() for v in arena.views]
    for k, v in (f32 or {}).items():
        res.append(v.clone())
        v.copy_(f32_0[k])
    return res


@pytest.mark.parametrize("pad", PADS)
@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_segment_outputs_and_recompute_bytes(shape, kind, pad, monkeypatch):
    """Per layer kind: the checkpointed decoder's outputs and l_aux equal the plain decoder's byte for byte, and each segment's recompute
    reproduces its first forward (outputs, q|k|v, h1, act)."""
    m = _decoder(kind, shape)
    B, T = SHAPES[shape]["B"], SHAPES[shape]["T"]
    H = m.config.hidden_size
    x = Hh.randn(B, T, H, seed=1)
    dout = Hh.randn(B, T, H, seed=2, scale=0.1)
    mask, noise = _mask(B, T, pad), _noise(m, B * T, 3)
    plain = _run(m, x, mask, noise, dout, False)
    rec = _Recorder(monkeypatch)
    got = _run(m, x, mask, noise, dout, True)
    rec.check(f"{shape}/{kind}/{pad}", len(m.layers))
    n_fwd = 1 + (len(noise) if noise else 0)
    Hh.same_bytes(f"{shape}/{kind}/{pad} forward", plain[:n_fwd], got[:n_fwd])


@pytest.mark.parametrize("train", ["all", "params_only", "input_only"])
@pytest.mark.parametrize("pad", PADS)
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_gradients_byte_equal_at_a_deterministic_shape(kind, pad, train):
    """T = 64 (one key block in the attention backward's dQ): dx and every arena gradient of the checkpointed decoder equal the plain run's
    bytes, nothing outside the views is written, and nothing reads unwritten memory.  params_only: a trainable layer whose input does not
    require grad (frozen embedding); input_only: frozen layers that still pass the gradient back (projector-only pre-training)."""
    m = _decoder(kind, "tiny")
    if train == "input_only":
        m.requires_grad_(False)
    arena, f32 = _arena(m, seed=10)
    B, T = SHAPES["tiny"]["B"], SHAPES["tiny"]["T"]
    x = Hh.randn(B, T, m.config.hidden_size, seed=1)
    dout = Hh.randn(B, T, m.config.hidden_size, seed=2, scale=0.1)
    mask, noise = _mask(B, T, pad), _noise(m, B * T, 3)
    x_grad = train != "params_only"
    tag = f"{kind}/{pad}/{train}"
    plain = _run(m, x, mask, noise, dout, False, x_grad, arena, f32)
    Hh.same_bytes(tag + " plain twice", plain, _run(m, x, mask, noise, dout, False, x_grad, arena, f32))
    got = _run(m, x, mask, noise, dout, True, x_grad, arena, f32)
    Hh.same_bytes(tag + " checkpointed vs plain", plain, got)
    if arena is not None:
        arena.check_sentinels(tag)
    with Hh.poisoned_uninitialised_memory():
        poisoned = _run(m, x, mask, noise, dout, True, x_grad, arena, f32)
    Hh.no_nan(tag, **{"t%d" % i: t for i, t in enumerate(poisoned)})
    Hh.same_bytes(tag + " poisoned", plain, poisoned)


# ---- whole steps on helpers.tiny_pair ---------------------------------------------------------------------------------------------
def _count_segments(monkeypatch):
    from llavamod import kernels as K
    n = [0]
    orig = K.checkpoint

    def checkpoint(run, *inputs):
        n[0] += 1
        return orig(run, *inputs)
    monkeypatch.setattr(K, "checkpoint", checkpoint)
    return n


def _grads(tr):
    o = tr.optimizer
    return [g.clone() for g in (o.g16, o.g32) if g is not None]


def _step(make, ckpt, inputs):
    """One micro-batch (accumulation 2, so the gradients stay in the arena) -> (loss, arena gradients)."""
    model, tr = make()
    tr.use_cuda_graphs = False
    if ckpt:
        model.gradient_checkpointing_enable()
        model.enable_input_require_grads()
    loss = tr.training_step(model, inputs)
    torch.cuda.synchronize()
    return [loss.reshape(1).clone()], _grads(tr)


def _compare_steps(tag, make, inputs, monkeypatch):
    l0, g0 = _step(make, False, inputs)
    l1, g1 = _step(make, False, inputs)
    n = _count_segments(monkeypatch)
    lc, gc = _step(make, True, inputs)
    assert n[0] > 0, f"{tag}: no layer ran as a checkpointed segment"
    Hh.same_bytes(tag + " plain loss twice", l0, l1)
    Hh.same_bytes(tag + " loss", l0, lc)
    repeat = all(torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a, b.view(torch.int16) if b.dtype == torch.bfloat16 else b)
                 for a, b in zip(g0, g1))
    if repeat:
        Hh.same_bytes(tag + " gradients", g0, gc)
    else:
        for a, c in zip(g0, gc):
            assert float((a.float() - c.float()).norm()) <= 1e-2 * float(a.float().norm()), tag
    print(f"\n{tag}: loss bytes equal, gradients {'byte-equal' if repeat else 'within 1e-2 (plain step not repeatable)'}; {n[0]} segments")


def _align(loss_type, dense_student=False):
    def make():
        student, teacher = Hh.tiny_pair()
        if dense_student:
            from llavamod.model import synthetic as S
            student = S.make_teacher(dict(S.ARCH["tiny"], vocab_size=512), "tiny", seed=5).train()
            student.get_image_tower().load_state_dict(teacher.get_image_tower().state_dict())
            for n, p in student.named_parameters():
                p.requires_grad = "image_tower" not in n
        return student, Hh.make_trainer(student, teacher, loss_type, accum=2)
    return make


@pytest.mark.parametrize("case", ["kd_lm", "only_kd_dense_student", "dpo_sigmoid", "dpo_kto_pair", "sft_dense", "pretrain_projector"])
def test_whole_steps_equal_the_plain_step(case, monkeypatch):
    student, _ = Hh.tiny_pair()
    batch, noise = Hh.tiny_batch(student, seed=11)
    if case == "kd_lm":
        _compare_steps(case, _align("kd_lm"), dict(batch, moe_noise=[n.cuda() for n in noise]), monkeypatch)
    elif case == "only_kd_dense_student":
        _compare_steps(case, _align("only_kd", dense_student=True), dict(batch), monkeypatch)
    elif case.startswith("dpo"):
        from tests.test_model_gpu import _dpo_inputs
        inputs = _dpo_inputs(student)[-1]

        def make():
            s, t = Hh.tiny_pair()
            return s, Hh.make_trainer(s, t, case[4:], accum=2, kind="dpo")
        _compare_steps(case, make, inputs, monkeypatch)
    else:
        from tests.test_sft_gpu import _dense_student, _sft_trainer

        def make():
            m = _dense_student()
            if case == "pretrain_projector":
                m.requires_grad_(False)
                for p in m.get_model().mm_projector.parameters():
                    p.requires_grad = True
            return m, _sft_trainer(m, 1e-3, 10, accum=2)
        m = _dense_student()
        b, _ = Hh.tiny_batch(m, seed=11)
        _compare_steps(case, make, dict(b), monkeypatch)


def test_config1_loss_curve_over_100_steps_is_the_plain_curve():
    """Config 1 (tiny pair, mimic kd_lm), 100 steps with CUDA graphs and the router noise drawn from the device generator: the checkpointed
    run's losses are the plain run's, byte for byte."""
    def curve(ckpt):
        student, teacher = Hh.tiny_pair()
        tr = Hh.make_trainer(student, teacher, "kd_lm", accum=1, lr=1e-3, max_steps=100)
        if ckpt:
            student.gradient_checkpointing_enable()
            student.enable_input_require_grads()
        batches = [Hh.tiny_batch(student, seed=200 + i)[0] for i in range(4)]
        torch.manual_seed(123)
        out = [tr.training_step(student, dict(batches[s % 4])).reshape(1) for s in range(100)]
        assert any("graph" in v for v in tr._graphs.values())
        return torch.cat(out)
    plain, got = curve(False), curve(True)
    Hh.same_bytes("config 1 loss curve", [plain], [got])
    print("\nconfig 1, 100 steps: checkpointed curve == plain curve; first %.5f last %.5f" % (float(plain[0]), float(plain[-1])))


def test_captured_checkpointed_step_replays_the_eager_bytes():
    """The captured forward+backward holds the recompute: three replays give the losses and weights of the eager checkpointed steps."""
    def run(graphs):
        student, teacher = Hh.tiny_pair()
        student.gradient_checkpointing_enable()
        student.enable_input_require_grads()
        tr = Hh.make_trainer(student, teacher, "kd_lm", accum=1, lr=1e-3)
        tr.use_cuda_graphs = graphs
        batch, noise = Hh.tiny_batch(student, seed=21)
        inputs = dict(batch, moe_noise=[n.cuda() for n in noise])
        losses = [tr.training_step(student, dict(inputs)).reshape(1) for _ in range(5)]     # 2 eager warm-ups, capture, 3 replays
        if graphs:
            sigs = [k for k, v in tr._graphs.items() if "graph" in v]
            assert len(sigs) == 1 and ("grad_ckpt", True) in sigs[0]
        return losses, [p.detach().clone() for p in student.parameters()]
    le, we = run(False)
    lg, wg = run(True)
    Hh.same_bytes("graph replays: losses", le, lg)
    Hh.same_bytes("graph replays: weights", we, wg)


# ---- config-2 student: 24 layers, T' = 2048 --------------------------------------------------------------------------------------
def _saved_bytes(model, S):
    """Saved-activation bytes of layers 1 .. L-1 of the plain student (kernels.py's Functions: 16H + 6I bytes per token for a dense layer,
    24H + 12I for a top-2 MoE layer), minus the two [S, H] bf16 boundary tensors a checkpointed layer keeps."""
    from llavamod.model.language_model.qwen2_core import MoE
    H, I = model.config.hidden_size, model.config.intermediate_size
    n = 0
    for layer in model.model.layers[1:]:
        per_tok = (24 * H + 12 * I) if isinstance(layer.mlp, MoE) else (16 * H + 6 * I)
        n += S * (per_tok - 4 * H)
    return n


def test_config2_student_loss_gradients_and_memory():
    from llavamod.model import synthetic as S
    from llavamod.train.engine import TrainState
    student = S.make_student("qwen1.5-0.5b", "tiny", seed=1, margs=S.moe_args()).train()
    ts = TrainState(student)
    batch, noise = Hh.tiny_batch(student, B=1, Tt=2048 - 15, seed=5)
    noise = [n.cuda() for n in noise]
    Tn = 2048

    def step(ckpt):
        if ckpt:
            student.gradient_checkpointing_enable()
        else:
            student.gradient_checkpointing_disable()
        ts.zero_grad()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        loss, _, _ = student.forward_train_loss(batch["input_ids"], batch["attention_mask"], batch["labels"], batch["images"], noise)
        loss.backward()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        return loss.detach().reshape(1).clone(), [g.float().clone() for _, g in ts._views], peak

    l0, g0, p0 = step(False)
    l1, g1, _ = step(False)
    lc, gc, pc = step(True)
    Hh.same_bytes("config-2 loss", [l0], [lc])
    worst, spread = 0.0, 0.0
    for a, b, c in zip(g0, g1, gc):
        na = float(a.norm())
        if na == 0.0:
            continue
        worst = max(worst, float((c - a).norm()) / na)
        spread = max(spread, float((b - a).norm()) / na)
        assert float((c - a).norm()) <= 1e-2 * na
    counted = _saved_bytes(student, Tn)
    print("\nconfig-2 student (24 layers, T' = 2048): max ||g_ckpt - g_plain|| / ||g_plain|| = %.3g (plain vs plain %.3g); peak over "
          "forward+backward plain %.1f MiB, checkpointed %.1f MiB (saved %.1f MiB; counted activations %.1f MiB)"
          % (worst, spread, p0 / 2 ** 20, pc / 2 ** 20, (p0 - pc) / 2 ** 20, counted / 2 ** 20))
    assert p0 - pc >= 0.5 * counted, (p0, pc, counted)
