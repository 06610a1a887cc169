"""The FP8 (e4m3) frozen teacher end to end: quantize_fp8_ on tiny dense models against the fake-quantised CPU oracle
(tests/fp8_oracle.py), one config-2-shape layer, the trainers with ref_fp8, and the decoding guarantees (padded batches, assisted
decoding, the T-token verify step) re-asserted under per-row activation scales."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import restated as R  # noqa: E402
from tests import fp8_oracle as O  # noqa: E402
from tests import helpers as Hh  # noqa: E402
from tests.test_decode_gpu import _logit_tol, _teacher  # noqa: E402
from tests.test_ragged_decode_gpu import _decode, _prompts  # noqa: E402


def _freeze(m):
    for p in m.parameters():
        p.requires_grad = False
    return m.eval()


def _fp8_teacher(heads=2, kv_heads=2, seed=21, inter=None):
    """(quantised model, fake-quantised fp32 oracle state of the same weights)"""
    from llavamod.model import synthetic as S
    arch = dict(S.ARCH["tiny"], num_attention_heads=heads, num_key_value_heads=kv_heads)
    if inter:
        arch["intermediate_size"] = inter
    m = _freeze(S.make_teacher(arch, "tiny", seed=seed))
    sd = O.fake_quant_state(Hh.oracle_state(m))
    return m, sd


@pytest.mark.parametrize("heads,kv_heads,inter", [(4, 4, 320), (4, 2, 256), (2, 2, 256)])      # MHA hd 32 (unfused RoPE / SwiGLU), GQA 4:2, hd 64
def test_quantised_model_matches_the_fake_quantised_oracle(heads, kv_heads, inter):
    m, sd = _fp8_teacher(heads, kv_heads, seed=61, inter=inter)
    batch, _ = Hh.tiny_batch(m, B=2, Tt=40, seed=62, pad=(0, 7))
    kw = dict(input_ids=batch["input_ids"], attention_mask=batch["attention_mask"], images=batch["images"])
    with torch.no_grad():
        bf16 = m(**kw).logits.float().cpu()
    ptrs = [p.data_ptr() for p in m.parameters()]
    m.quantize_fp8_()
    from llavamod import kernels as Kk
    assert m.is_fp8 and isinstance(m.model.layers[0].self_attn.qkv_weight, Kk.Fp8Rows)
    assert len(list(m.parameters())) < len(ptrs) and m.model.layers[0].mlp.down_proj.weight is None
    with torch.no_grad():
        got = m(**kw).logits.float().cpu()
    with O.fp8_decoder(R):
        want, _ = Hh.oracle_forward(m, batch, sd=sd)
    valid = want["attention_mask"].bool()
    ref = want["logits"][valid]
    err = (got[valid] - ref).abs().max().item()
    assert err < _logit_tol(ref), (err, _logit_tol(ref))
    # against its own bf16 self -- on random weights, so informative only: a trained teacher's logits are far more peaked
    p = torch.log_softmax(bf16[valid], -1)
    q = torch.log_softmax(got[valid], -1)
    print("\nFP8 vs bf16 (random weights, heads %d/%d): max |dlogit| %.4f of range %.3f, mean KL(p_bf16 || p_fp8) %.3e"
          % (heads, kv_heads, (got[valid] - bf16[valid]).abs().max().item(), bf16[valid].abs().max().item(), (p.exp() * (p - q)).sum(-1).mean().item()))


def test_quantised_model_is_forward_only():
    m, _ = _fp8_teacher(seed=63)
    m.quantize_fp8_()
    batch, _ = Hh.tiny_batch(m, B=1, Tt=24, seed=64)
    with pytest.raises(RuntimeError, match="forward-only"):
        m(input_ids=batch["input_ids"], labels=batch["labels"], images=batch["images"])
    with pytest.raises(RuntimeError, match="forward-only"):
        m.forward_train_loss(input_ids=batch["input_ids"], labels=batch["labels"], images=batch["images"])
    with pytest.raises(RuntimeError, match="e4m3"):
        m.state_dict()
    with pytest.raises(RuntimeError, match="e4m3"):
        m.save_pretrained("/tmp/lmod_fp8_never_written")
    with pytest.raises(RuntimeError, match="eval"):
        m.train()
    with pytest.raises(ValueError, match="already"):
        m.quantize_fp8_()
    emb = torch.randn(1, 8, m.config.hidden_size, device="cuda").to(torch.bfloat16).requires_grad_()
    with pytest.raises(RuntimeError, match="forward-only"):
        m.model(emb)


def test_config2_shape_layer_matches_the_fake_quantised_oracle():
    """One teacher layer at H 4096, I 11008, 32 heads of 128, T 2048 (the fused RoPE and SwiGLU e4m3 forms, BN = 256 tiles)."""
    from llavamod import kernels as Kk
    from llavamod.model.language_model.qwen2_core import Qwen2Config, Qwen2Model
    cfg = Qwen2Config(vocab_size=64, hidden_size=4096, intermediate_size=11008, num_hidden_layers=1, num_attention_heads=32, rope_theta=1e6)
    torch.manual_seed(5)
    model = _freeze(Qwen2Model(cfg, "cuda", torch.bfloat16))
    model.layers[0].self_attn.qkv_bias.normal_(0, 0.02)
    sd = O.fake_quant_state({"model." + k: v.detach().float().cpu() for k, v in model.state_dict().items()})
    x = (torch.randn(1, 2048, 4096, generator=torch.Generator().manual_seed(6)) * 0.5).to(torch.bfloat16)
    model.quantize_fp8_()
    with torch.no_grad():
        got, _, _ = model(x.cuda())
    lc = R.LMCfg(hidden=4096, inter=11008, layers=1, heads=32, kv_heads=32, vocab=64, rope_theta=1e6, eps=cfg.rms_norm_eps)
    with O.fp8_decoder(R):
        want, _ = R.lm_forward(sd, lc, x.float(), None, None)
    err = (got.float().cpu() - want).abs()
    print("\nFP8 cfg-2 layer vs fake-quantised fp32 oracle: max err %.4f mean err %.5f, output range %.3f" % (err.max().item(), err.mean().item(), want.abs().max().item()))
    # bf16 activations against an fp32 oracle: an activation that rounds the other way in bf16 lands in the next e4m3 bucket (a 6 - 12 %
    # step on that element), a few per cent of the elements of each of the four GEMM inputs do, and downstream of the first flip the two
    # chains quantise different numbers.  So this bounds the layer loosely (measured on an H100: max 0.357, mean 0.046 on unit-RMS output
    # rows of range 5.3); the tight checks are the kernels' own (test_gemm_fp8_gpu.py, test_fp8_quant_gpu.py) and the tiny models above
    assert err.max().item() < 0.1 * want.abs().max().item() + 3e-2, (err.max().item(), want.abs().max().item())
    assert err.mean().item() < 8e-2, err.mean().item()
    assert isinstance(model.layers[0].mlp.gu_weight, Kk.Fp8Rows)


def _trainer(student, teacher, kind="align", ref_fp8=False, loss_type="kd_lm", lr=2e-5):
    from llavamod.config.args import TrainingArguments
    from llavamod.train.align_trainer import AlignTrainer
    from llavamod.train.dpo_trainer import DPOTrainer
    args = TrainingArguments(output_dir="/tmp/lmod_out", per_device_train_batch_size=1, gradient_accumulation_steps=1, learning_rate=lr,
                             weight_decay=0.0, warmup_ratio=0.03, lr_scheduler_type="cosine", max_steps=100, logging_steps=0,
                             save_strategy="no", bf16=True)
    args.moe_enable = True
    tr = (AlignTrainer if kind == "align" else DPOTrainer)(model=student, ref_model=teacher, args=args, loss_type=loss_type,
                                                           moe_loss_enable=True, ref_fp8=ref_fp8)
    tr._total_steps = 100
    return tr


def test_align_trainer_with_ref_fp8_matches_the_oracle_fed_the_fake_quantised_teacher():
    student, teacher = Hh.tiny_pair(seed=70)
    batch, noise = Hh.tiny_batch(student, seed=71)
    sd_t = O.fake_quant_state(Hh.oracle_state(teacher))
    with torch.no_grad(), O.fp8_decoder(R):
        t_out, _ = Hh.oracle_forward(teacher, batch, sd=sd_t)
    s_out, lc = Hh.oracle_forward(student, batch, noise)
    ref_loss, ref_m = R.mimic_compute_loss(s_out, t_out["logits"], "kd_lm", True, False, lc.kd_vocab)
    tr = _trainer(student, teacher, ref_fp8=True)
    assert teacher.is_fp8 and tr.share_tower
    loss, m = tr.compute_loss(student, dict(batch, moe_noise=[n.cuda() for n in noise]), return_outputs=True)
    for k in ("loss", "loss/align", "loss/lm", "loss/moe_balance"):
        assert abs(float(m[k]) - float(ref_m[k])) < 1e-2 * abs(float(ref_m[k])) + 1e-4, (k, float(m[k]), float(ref_m[k]))
    loss.backward()
    torch.cuda.synchronize()
    assert all(torch.isfinite(p.grad).all() for p in student.parameters() if p.grad is not None)


def test_ref_fp8_false_quantises_nothing():
    student, teacher = Hh.tiny_pair(seed=72)
    student2, teacher2 = Hh.tiny_pair(seed=72)
    ptrs = [p.data_ptr() for p in teacher.parameters()]
    tr = _trainer(student, teacher, ref_fp8=False)
    assert not teacher.is_fp8 and [p.data_ptr() for p in teacher.parameters()] == ptrs
    batch, _ = Hh.tiny_batch(student, seed=73)
    with torch.no_grad():
        a = teacher(input_ids=batch["input_ids"], attention_mask=batch["attention_mask"], images=batch["images"]).logits
        b = _freeze(teacher2)(input_ids=batch["input_ids"], attention_mask=batch["attention_mask"], images=batch["images"]).logits
    assert torch.equal(a, b) and tr.ref_model.module is teacher


def test_ten_pipelined_graph_steps_with_an_fp8_teacher_track_the_eager_losses():
    student, teacher = Hh.tiny_pair(seed=74)
    batches = [Hh.tiny_batch(student, seed=80 + i)[0] for i in range(4)]
    tr = _trainer(student, teacher, ref_fp8=True, lr=0.0)
    tr.use_cuda_graphs = False
    ref = []
    for i in range(10):
        torch.manual_seed(100 + i)
        ref.append(float(tr.training_step(student, dict(batches[i % 4]))))
    student2, teacher2 = Hh.tiny_pair(seed=74)
    tr2 = _trainer(student2, teacher2, ref_fp8=True, lr=0.0)
    assert tr2.use_cuda_graphs and tr2.overlap_teacher and teacher2.is_fp8
    got = [float(tr2.training_step(student2, batches[i % 4], batches[(i + 1) % 4])) for i in range(10)]
    assert any("pipelined" in str(k) for k in tr2._graphs), "the pipelined graph was not captured"
    for a, b in zip(ref, got):                              # router noise differs between the eager and the replayed RNG streams
        assert abs(a - b) < 2e-2 * abs(a), (ref, got)


def test_dpo_trainer_with_ref_fp8_runs_a_step():
    student, teacher = Hh.tiny_pair(seed=75)
    tr = _trainer(student, teacher, kind="dpo", ref_fp8=True, loss_type="sigmoid")
    assert teacher.is_fp8
    from llavamod.train.dpo_train import SyntheticDPODataset, collate_dpo
    tower = student.get_image_tower()
    ds = SyntheticDPODataset(2, 40, student.config.vocab_size, tower.config.image_size, 0)
    loss = tr.training_step(student, collate_dpo([ds[0], ds[1]]))
    assert torch.isfinite(torch.as_tensor(float(loss)))


# ---- decoding guarantees under per-row scales ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("heads,kv_heads", [(2, 2), (4, 2)])
def test_padded_batch_equals_each_prompt_alone_with_a_quantised_target(heads, kv_heads):
    m, _ = _fp8_teacher(heads, kv_heads, seed=81)
    m.quantize_fp8_()
    m.config.tokenizer_padding_side = "right"
    lens, N = [21, 6, 13], 5
    ids, mask, imgs = _prompts(m.config.vocab_size, lens, "right", seed=82)
    toks = torch.randint(0, m.config.vocab_size, (3, N), generator=torch.Generator().manual_seed(83))
    got, _ = _decode(m, ids, mask, imgs, toks, 512)
    for b in range(3):
        one, _ = _decode(m, ids[b:b + 1, mask[b]], torch.ones(1, lens[b], dtype=torch.bool), imgs[b:b + 1], toks[b:b + 1], 512)
        assert torch.equal(got[:, b], one[:, 0]), (b, (got[:, b] - one[:, 0]).abs().max().item())
    want = m.generate(ids, images=imgs, attention_mask=mask, max_new_tokens=8, use_cache=True)
    for b in range(3):
        alone = m.generate(ids[b:b + 1, mask[b]], images=imgs[b:b + 1], max_new_tokens=8, use_cache=True)
        assert torch.equal(alone[0, -8:], want[b, -8:]), b


@pytest.mark.parametrize("graphs", ["1", "0"])
def test_assisted_greedy_equals_the_quantised_target(monkeypatch, graphs):
    monkeypatch.setenv("LLAVAMOD_CUDA_GRAPHS", graphs)
    student, teacher = Hh.tiny_pair(seed=84)
    _freeze(teacher).quantize_fp8_()
    batch, _ = Hh.tiny_batch(teacher, B=1, Tt=24, seed=85)
    ids, imgs = batch["input_ids"], batch["images"]
    want = teacher.generate(ids, images=imgs, max_new_tokens=20, use_cache=True)
    for k in (1, 4):
        assert torch.equal(teacher.generate(ids, images=imgs, max_new_tokens=20, use_cache=True, assistant_model=teacher, num_assistant_tokens=k), want)
        assert torch.equal(teacher.generate(ids, images=imgs, max_new_tokens=20, use_cache=True, assistant_model=student.eval(), num_assistant_tokens=k), want)


def test_verify_step_equals_one_token_steps_bitwise_with_a_quantised_target():
    m, _ = _fp8_teacher(4, 2, seed=86)
    m.quantize_fp8_()
    ids, mask, imgs = _prompts(m.config.vocab_size, [17, 6, 11], "right", seed=87)
    toks = torch.randint(0, m.config.vocab_size, (3, 7), generator=torch.Generator().manual_seed(88)).cuda()

    def prefill():
        cache = m.new_kv_cache(3, 256)
        with torch.no_grad():
            m(input_ids=ids.cuda(), attention_mask=mask.cuda(), images=imgs, past_key_values=cache, use_cache=True)
        return cache
    a, b = prefill(), prefill()
    with torch.no_grad():
        one = [m(input_ids=toks[:, t:t + 1], past_key_values=a, use_cache=True).logits for t in range(7)]
        two = [m(input_ids=toks[:, :3], past_key_values=b, use_cache=True).logits, m(input_ids=toks[:, 3:], past_key_values=b, use_cache=True).logits]
    assert torch.equal(torch.cat(one, 1), torch.cat(two, 1))
