"""GPU parity of the assembled path against the CPU oracle: dense teacher vs the REFERENCE's golden outputs, sparse student
forward/backward, AlignTrainer / DPOTrainer losses and a short loss curve."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import restated as R  # noqa: E402
from tests import helpers as Hh  # noqa: E402
from tests.golden import shards  # noqa: E402


def _rel(a, b):
    return (a.float().cpu() - b.float().cpu()).abs().max().item() / (b.float().abs().max().item() + 1e-12)


@pytest.mark.parametrize("name", ["dense_mha", "dense_gqa", "dense_nopad", "dense_hd64"])
def test_dense_model_matches_reference_golden(name, golden_dir):
    """Reference outputs (fp32, from the reference's own code) vs our bf16 CUDA model loaded with the same weights."""
    from llavamod.model import LlavaQwen1_5Config, LlavaQwen1_5ForCausalLM
    from llavamod.model.builder_io import load_into
    fx = shards.load(golden_dir, name)
    kw = fx["kw"]
    clip = dict(hidden_size=64, intermediate_size=128, num_hidden_layers=3, num_attention_heads=kw.get("clip_heads", 4), image_size=32, patch_size=8)
    cfg = LlavaQwen1_5Config(vocab_size=kw["vocab"], hidden_size=kw["hidden"], intermediate_size=kw["inter"], num_hidden_layers=kw["layers"],
                             num_attention_heads=kw["heads"], num_key_value_heads=kw["kv_heads"], rope_theta=1e6, mm_image_tower=clip,
                             image_projector_type="mlp2x_gelu", mm_hidden_size=64, mm_vision_select_layer=-2)
    m = LlavaQwen1_5ForCausalLM(cfg, device="cuda", dtype=torch.bfloat16)
    m.get_model().get_image_tower().load_model()
    load_into(m, {k: v for k, v in fx["state_dict"].items() if "position_ids" not in k}, strict=True)
    with torch.no_grad():
        out = m(input_ids=fx["input_ids"], labels=fx["labels"], attention_mask=fx["attention_mask"],
                images=[im.to(torch.bfloat16) for im in fx["images"]], return_dict=True)
    assert torch.equal(out.labels.cpu(), fx["out_labels"])                      # integer splice: bit exact vs the reference
    valid = fx["out_labels"].new_ones(fx["out_labels"].shape, dtype=torch.bool)
    if name not in ("dense_nopad", "dense_hd64"):
        valid = R.splice_plan(fx["input_ids"], fx["attention_mask"], fx["labels"], 16)[2]
    # bf16 weights + activations vs fp32 reference: 3e-2 of the logit range (stated tolerance for logits), loss 1e-2 relative
    err = (out.logits.float().cpu() - fx["logits"])[valid].abs().max().item()
    assert err < 3e-2 * fx["logits"][valid].abs().max().item() + 3e-2, err
    assert abs(out.loss.item() - fx["loss"].item()) < 1e-2 * fx["loss"].item()


def test_student_forward_and_trainer_loss_match_oracle():
    student, teacher = Hh.tiny_pair()
    batch, noise = Hh.tiny_batch(student, seed=1)
    ref_loss, ref_m = Hh.oracle_mimic_loss(student, teacher, batch, noise, "kd_lm")
    tr = Hh.make_trainer(student, teacher, "kd_lm")
    assert tr.share_tower
    loss, m = tr.compute_loss(student, dict(batch, moe_noise=[n.cuda() for n in noise]), return_outputs=True)
    # bf16 GPU path vs fp32 oracle on bf16-rounded weights: loss within 1e-2 relative at random init (V=512 -> loss ~ 6)
    for k in ("loss", "loss/align", "loss/lm", "loss/moe_balance"):
        assert abs(float(m[k]) - float(ref_m[k])) < 1e-2 * abs(float(ref_m[k])) + 1e-4, (k, float(m[k]), float(ref_m[k]))
    # only_kd + disabled moe loss: sentinel metric -1.0 (align_trainer.py:579)
    tr2 = Hh.make_trainer(student, teacher, "only_kd", moe_loss_enable=False)
    ref2, ref_m2 = Hh.oracle_mimic_loss(student, teacher, batch, noise, "only_kd", moe_loss_enable=False)
    loss2, m2 = tr2.compute_loss(student, dict(batch, moe_noise=[n.cuda() for n in noise]), return_outputs=True)
    assert float(m2["loss/moe_balance"]) == -1.0 and float(ref_m2["loss/moe_balance"]) == -1.0
    assert abs(float(loss2) - float(ref2)) < 1e-2 * abs(float(ref2))


@pytest.mark.parametrize("distill_all", [False, True])
def test_qwen2_like_pair_gqa_teacher_with_wider_vocab(distill_all):
    """Shell-default Qwen-2 shapes (SURVEY 8, shape table): GQA in both models and a teacher vocabulary LARGER than the student's, so the
    reference's hard-coded logits[:, :, :151936] slice (align_trainer.py:473,497; here min(kd_vocab, student vocab)) really cuts columns;
    plus --distill_all_tokens (align_trainer.py:512-515)."""
    from llavamod.model import synthetic as S
    arch_s = dict(S.ARCH["tiny"], num_key_value_heads=1, vocab_size=512, tie_word_embeddings=True)
    arch_t = dict(S.ARCH["tiny"], num_key_value_heads=1, vocab_size=640, intermediate_size=320)
    teacher = S.make_teacher(arch_t, "tiny", seed=3)
    student = S.make_student(arch_s, "tiny", seed=4, margs=S.moe_args(), share_tower_with=teacher)
    batch, noise = Hh.tiny_batch(student, seed=5)
    with torch.no_grad():
        t_out, _ = Hh.oracle_forward(teacher, batch)
    s_out, lc = Hh.oracle_forward(student, batch, noise)
    assert t_out["logits"].shape[-1] == 640 and s_out["logits"].shape[-1] == 512
    ref_loss, ref_m = R.mimic_compute_loss(s_out, t_out["logits"], "kd_lm", True, distill_all, 512)
    tr = Hh.make_trainer(student, teacher, "kd_lm")
    tr.args.distill_all_tokens = distill_all
    loss, m = tr.compute_loss(student, dict(batch, moe_noise=[n.cuda() for n in noise]), return_outputs=True)
    for k in ("loss", "loss/align", "loss/lm", "loss/moe_balance"):
        assert abs(float(m[k]) - float(ref_m[k])) < 1e-2 * abs(float(ref_m[k])) + 1e-4, (k, float(m[k]), float(ref_m[k]))
    loss.backward()
    torch.cuda.synchronize()


def test_real_data_batch_through_trainer_matches_oracle(golden_dir):
    """SURVEY 8f N1 end to end: records -> LazySupervisedDataset -> collator (tokeniser + CLIP processor; golden-checked against the
    reference in tests/test_data_pipeline.py) -> AlignTrainer on the GPU, against the CPU oracle on the same batch.  The batch is ragged
    on purpose: one image, two images, a text-only record (a blank image is fed and its features are consumed by an empty slice,
    llava_arch.py:247-274) and an unreadable file (black fallback), right-padded to the longest sample."""
    import types
    from transformers import CLIPImageProcessor
    from llavamod import conversation as conversation_lib
    from llavamod.data import dataset as D
    from tests.golden.make_data_golden import load_tokenizer
    D.local_rank = 1
    conversation_lib.set_default_conversation("qwen")
    tok = load_tokenizer(os.path.join(golden_dir, "tiny_tokenizer.json"))
    args = types.SimpleNamespace(image_folder=os.path.join(golden_dir, "data_imgs"), image_aspect_ratio="pad", is_multimodal=True,
                                 image_processor=CLIPImageProcessor(size={"shortest_edge": 32}, crop_size={"height": 32, "width": 32}),
                                 mm_use_im_start_end=False, num_frames=8, data_path=[os.path.join(golden_dir, "data_sft.json")])
    mod = D.make_supervised_data_module(tok, args)
    batch = mod["data_collator"]([mod["train_dataset"][i] for i in range(4)])
    batch["images"] = [im.to(torch.bfloat16) for im in batch["images"]]
    assert batch["input_ids"].shape == (4, 112) and len(batch["images"]) == 5 and not bool(batch["attention_mask"].all())
    student, teacher = Hh.tiny_pair(vocab=424)            # >= len(tok) = 420, multiple of 8 (16-byte rows for the loss kernels)
    student.config.pad_token_id = teacher.config.pad_token_id = tok.pad_token_id
    Tn = 112 - 1 + 16                                      # longest spliced sample: record 0 (one image, 16 patches)
    g = torch.Generator().manual_seed(11)
    n_moe = sum(1 for l in student.model.layers if hasattr(l.mlp, "deepspeed_moe"))
    noise = [R.gumbel_noise((4 * Tn, 4), g) for _ in range(n_moe)]
    ref_loss, ref_m = Hh.oracle_mimic_loss(student, teacher, batch, noise, "kd_lm")
    tr = Hh.make_trainer(student, teacher, "kd_lm")
    loss, m = tr.compute_loss(student, dict(batch, moe_noise=[n.cuda() for n in noise]), return_outputs=True)
    for k in ("loss", "loss/align", "loss/lm", "loss/moe_balance"):
        assert abs(float(m[k]) - float(ref_m[k])) < 1e-2 * abs(float(ref_m[k])) + 1e-4, (k, float(m[k]), float(ref_m[k]))


def test_padded_batch_goes_through_masked_attention():
    student, teacher = Hh.tiny_pair()
    batch, noise = Hh.tiny_batch(student, seed=2, pad=(0, 7))
    ref_loss, ref_m = Hh.oracle_mimic_loss(student, teacher, batch, noise, "kd_lm")
    tr = Hh.make_trainer(student, teacher, "kd_lm")
    loss = tr.compute_loss(student, dict(batch, moe_noise=[n.cuda() for n in noise]))
    assert abs(float(loss) - float(ref_loss)) < 1e-2 * abs(float(ref_loss))


def test_gradients_match_oracle_autograd():
    student, teacher = Hh.tiny_pair()
    batch, noise = Hh.tiny_batch(student, seed=4)
    sd_s = Hh.oracle_state(student)
    train_keys = [n for n, p in student.named_parameters() if p.requires_grad]
    assert sorted(train_keys) == sorted(R.trainable_keys(sd_s))
    for k in train_keys:
        sd_s[k].requires_grad_(True)
    ref_loss, _ = Hh.oracle_mimic_loss(student, teacher, batch, noise, "kd_lm", sd_s=sd_s)
    ref_loss.backward()
    tr = Hh.make_trainer(student, teacher, "kd_lm")
    opt = tr.create_optimizer()
    opt.zero_grad()
    loss = tr.compute_loss(student, dict(batch, moe_noise=[n.cuda() for n in noise]))
    loss.backward()
    torch.cuda.synchronize()
    worst = 0.0
    for n, p in student.named_parameters():
        if not p.requires_grad:
            continue
        g, r = p.grad.float().cpu(), sd_s[n].grad
        rel = (g - r).norm().item() / (r.norm().item() + 1e-12)
        worst = max(worst, rel)
        assert rel < 0.08, (n, rel)            # bf16 activations + bf16 grad buffer vs fp32 autograd: 8% of the tensor norm
    print("worst relative grad error", worst)


def test_dense_student_full_parameter_gradients_match_oracle():
    """Dense-to-dense distillation (shells/train/qwen/dense2dense_distillation.sh: --policy_model_type dense, only_kd): no MoE wrap, so
    nothing is frozen by --train_modules and EVERY language-model parameter trains -- embeddings (through the splice), q/k/v biases,
    attention weights, the three kinds of RMSNorm weights and lm_head, next to the FFN and the projector.  Gradients of all of them against
    fp32 autograd of the oracle."""
    from llavamod.model import synthetic as S
    teacher = S.make_teacher(dict(S.ARCH["tiny"], intermediate_size=320), "tiny", seed=6)
    student = S.make_teacher(dict(S.ARCH["tiny"]), "tiny", seed=7).train()
    student.get_image_tower().load_state_dict(teacher.get_image_tower().state_dict())
    for n, p in student.named_parameters():
        p.requires_grad = "image_tower" not in n
    batch, noise = Hh.tiny_batch(student, seed=8)
    assert noise == []
    sd_s = Hh.oracle_state(student)
    names = [n for n, p in student.named_parameters() if p.requires_grad]
    assert any("embed_tokens" in n for n in names) and any("input_layernorm" in n for n in names) and any("q_proj.bias" in n for n in names)
    for k in names:
        sd_s[k].requires_grad_(True)
    ref_loss, _ = Hh.oracle_mimic_loss(student, teacher, batch, None, "only_kd", moe_loss_enable=False, sd_s=sd_s)
    ref_loss.backward()
    tr = Hh.make_trainer(student, teacher, "only_kd", moe_loss_enable=False)
    opt = tr.create_optimizer()
    opt.zero_grad()
    loss = tr.compute_loss(student, dict(batch))
    assert abs(float(loss) - float(ref_loss)) < 1e-2 * abs(float(ref_loss))
    loss.backward()
    torch.cuda.synchronize()
    worst = ("", 0.0)
    for n, p in student.named_parameters():
        if not p.requires_grad:
            continue
        g, r = p.grad.float().cpu(), sd_s[n].grad
        assert r is not None and r.norm().item() > 0, n
        rel = (g - r).norm().item() / (r.norm().item() + 1e-12)
        if rel > worst[1]:
            worst = (n, rel)
        assert rel < 0.08, (n, rel)
    print("worst relative grad error", worst)


def test_loss_curve_tracks_oracle_20_steps():
    """config 1 (2-layer/128-d student + teacher, 32x32 image): the GPU loss follows the fp32 CPU oracle step by step."""
    student, teacher = Hh.tiny_pair()
    lc, cc = Hh.cfgs_of(student)
    sd_s, sd_t = Hh.oracle_state(student), Hh.oracle_state(teacher)
    keys = [n for n, p in student.named_parameters() if p.requires_grad]
    params = [sd_s[k].requires_grad_(True) for k in keys]
    m = [torch.zeros_like(p) for p in params]
    v = [torch.zeros_like(p) for p in params]
    steps, lr = 20, 1e-3
    tr = Hh.make_trainer(student, teacher, "kd_lm", accum=1, lr=lr, max_steps=steps)
    dev = []
    for s in range(steps):
        batch, noise = Hh.tiny_batch(student, seed=100 + s)
        ref_loss, _ = Hh.oracle_mimic_loss(student, teacher, batch, noise, "kd_lm", sd_s=sd_s, sd_t=sd_t)
        grads = torch.autograd.grad(ref_loss, params)
        grads = [g.clone() for g in grads]
        R.clip_grad_norm(grads, 1.0)
        with torch.no_grad():
            R.adamw_step(params, grads, m, v, s + 1, R.cosine_lr(s, steps, lr))
        loss = tr.training_step(student, dict(batch, moe_noise=[n.cuda() for n in noise]))
        dev.append(abs(float(loss) - float(ref_loss)))
        assert dev[-1] < 2e-2 * abs(float(ref_loss)), (s, float(loss), float(ref_loss))
    print("max |loss_gpu - loss_oracle| over %d steps: %.4e" % (steps, max(dev)))


def test_loss_curve_100_steps_config1():
    """BASELINE.json config 1, 100 optimizer steps (AdamW + cosine schedule + clipping): bf16 CUDA path vs the fp32 CPU oracle started
    from the same weights and fed the same batches / router noise.  Stated tolerance (BASELINE.json north star): |loss - oracle| <= 1e-3
    at every step."""
    student, teacher = Hh.tiny_pair()
    sd_s, sd_t = Hh.oracle_state(student), Hh.oracle_state(teacher)
    keys = [n for n, p in student.named_parameters() if p.requires_grad]
    params = [sd_s[k].requires_grad_(True) for k in keys]
    m = [torch.zeros_like(p) for p in params]
    v = [torch.zeros_like(p) for p in params]
    steps, lr = 100, 2e-4
    tr = Hh.make_trainer(student, teacher, "kd_lm", accum=1, lr=lr, max_steps=steps)
    worst_abs, worst_rel = 0.0, 0.0
    for s in range(steps):
        batch, noise = Hh.tiny_batch(student, seed=1000 + s)
        ref_loss, _ = Hh.oracle_mimic_loss(student, teacher, batch, noise, "kd_lm", sd_s=sd_s, sd_t=sd_t)
        grads = [g.clone() for g in torch.autograd.grad(ref_loss, params)]
        R.clip_grad_norm(grads, 1.0)
        with torch.no_grad():
            R.adamw_step(params, grads, m, v, s + 1, R.cosine_lr(s, steps, lr))
        loss = tr.training_step(student, dict(batch, moe_noise=[n.cuda() for n in noise]))
        d = abs(float(loss) - float(ref_loss))
        worst_abs, worst_rel = max(worst_abs, d), max(worst_rel, d / abs(float(ref_loss)))
        assert d < 1e-3, (s, float(loss), float(ref_loss))
    print("100 steps: max |loss_gpu - loss_oracle| = %.3e (relative %.3e); final loss gpu %.4f oracle %.4f" % (worst_abs, worst_rel, float(loss), float(ref_loss)))


def test_pipelined_teacher_gives_the_same_losses():
    """training_step(inputs, next_inputs): the teacher runs one micro-batch ahead inside the CUDA graph; losses must equal the
    unpipelined eager path batch for batch (same weights: lr = 0)."""
    student, teacher = Hh.tiny_pair()
    batches = [Hh.tiny_batch(student, seed=50 + i)[0] for i in range(4)]
    tr = Hh.make_trainer(student, teacher, "kd_lm", accum=1, lr=0.0)
    tr.use_cuda_graphs = False
    torch.manual_seed(7)
    ref = []
    for i in range(8):
        torch.manual_seed(100 + i)                                 # router noise is drawn from the device generator
        ref.append(float(tr.training_step(student, dict(batches[i % 4]))))
    student2, teacher2 = Hh.tiny_pair()
    tr2 = Hh.make_trainer(student2, teacher2, "kd_lm", accum=1, lr=0.0)
    assert tr2.use_cuda_graphs and tr2.overlap_teacher
    got = []
    for i in range(8):
        got.append(float(tr2.training_step(student2, batches[i % 4], batches[(i + 1) % 4])))
    assert any("pipelined" in str(k) for k in tr2._graphs), "the pipelined graph was not captured"
    # noise differs between eager and graph-replayed RNG streams -> compare within the routing-noise spread, and exactly-shaped curves
    for a, b in zip(ref, got):
        assert abs(a - b) < 2e-2 * abs(a), (ref, got)


def test_checkpoint_resume_continues_the_same_run(tmp_path):
    """N2: checkpoint-N/ (HF-layout model + optimizer arenas + trainer state) -> a fresh trainer resumes and reproduces the next losses."""
    from llavamod.config.args import TrainingArguments
    from llavamod.train.align_trainer import AlignTrainer

    class DS(torch.utils.data.Dataset):
        def __init__(self, student):
            self.items = [Hh.tiny_batch(student, B=1, seed=300 + i)[0] for i in range(6)]

        def __len__(self):
            return len(self.items)

        def __getitem__(self, i):
            b = self.items[i]
            return dict(input_ids=b["input_ids"][0], labels=b["labels"][0], image=b["images"][0])

    from llavamod.train.align_train import collate

    def run(out_dir, max_steps, resume):
        student, teacher = Hh.tiny_pair(seed=3)
        args = TrainingArguments(output_dir=str(out_dir), per_device_train_batch_size=1, gradient_accumulation_steps=1, learning_rate=1e-3,
                                 lr_scheduler_type="constant", max_steps=max_steps, logging_steps=1, save_strategy="steps", save_steps=2, bf16=True, seed=1)
        args.moe_enable = True
        tr = AlignTrainer(model=student, ref_model=teacher, args=args, loss_type="only_kd", moe_loss_enable=False,
                          train_dataset=DS(student), data_collator=collate)
        tr.use_cuda_graphs = False
        tr.get_train_dataloader = lambda: torch.utils.data.DataLoader(tr.train_dataset, batch_size=1, shuffle=False, collate_fn=collate)
        torch.manual_seed(0)
        tr.train(resume_from_checkpoint=resume)
        return [h["loss"] for h in tr.state.log_history], student

    full, _ = run(tmp_path / "a", 4, False)
    assert (tmp_path / "a" / "checkpoint-2" / "pytorch_model.bin").exists() and (tmp_path / "a" / "checkpoint-2" / "config.json").exists()
    import shutil
    shutil.copytree(tmp_path / "a" / "checkpoint-2", tmp_path / "b" / "checkpoint-2")
    resumed, student = run(tmp_path / "b", 4, True)
    assert student is not None and len(resumed) == 2                      # steps 3 and 4 only
    # same data order is not replayed by this minimal loop (it restarts the epoch), so compare the optimizer/weight state instead:
    sd_a = torch.load(tmp_path / "a" / "checkpoint-4" / "pytorch_model.bin")
    sd_b = torch.load(tmp_path / "b" / "checkpoint-4" / "pytorch_model.bin")
    assert sd_a.keys() == sd_b.keys()
    k = "model.layers.1.mlp.down_proj.weight"
    assert not torch.equal(sd_a[k], torch.load(tmp_path / "a" / "checkpoint-2" / "pytorch_model.bin")[k])     # training moved the weights
    assert torch.isfinite(sd_b[k].float()).all()


def _dpo_inputs(student, seeds=(7, 8)):
    bc, nc = Hh.tiny_batch(student, seed=seeds[0])
    br, nr = Hh.tiny_batch(student, seed=seeds[1])
    br["images"] = bc["images"]
    br["input_ids"][:, :16] = bc["input_ids"][:, :16]
    br["labels"][:, :16] = bc["labels"][:, :16]
    inputs = dict(chosen_input_ids=bc["input_ids"], chosen_labels=bc["labels"], chosen_attention_mask=bc["attention_mask"],
                  rejected_input_ids=br["input_ids"], rejected_labels=br["labels"], rejected_attention_mask=br["attention_mask"],
                  images=bc["images"], moe_noise=([n.cuda() for n in nc], [n.cuda() for n in nr]))
    return bc, nc, br, nr, inputs


DPO_METRICS = ("loss", "loss/reward", "loss/moe_balance", "loss/policy_chosen", "rewards/chosen", "rewards/rejected", "rewards/accuracies",
               "rewards/margins", "logps/chosen", "logps/rejected")


def test_dpo_trainer_matches_oracle():
    """DPOTrainer.compute_loss (dpo_trainer.py:564-641): the loss and ALL TEN logged metrics of the four loss types against the oracle
    (whose formulas are pinned on the reference's own method bodies, tests/test_trainer_loss_pin.py), at the mimic tolerance.
    Sequence log-probs are sums of ~33 token terms of ~6 nats each, so 1 % of a reward / margin is an absolute 2e-2 on those."""
    student, teacher = Hh.tiny_pair()
    bc, nc, br, nr, inputs = _dpo_inputs(student)
    with torch.no_grad():
        tc, _ = Hh.oracle_forward(teacher, bc)
        trj, _ = Hh.oracle_forward(teacher, br)
    pc, _ = Hh.oracle_forward(student, bc, nc)
    pr, _ = Hh.oracle_forward(student, br, nr)
    for lt in ("sigmoid", "kto_pair", "hinge", "ipo"):
        ref_loss, ref_m = R.dpo_compute_loss(pc, pr, tc["logits"], tc["labels"], trj["logits"], trj["labels"], 0.1, lt, True)
        tr = Hh.make_trainer(student, teacher, lt, kind="dpo")
        loss, m = tr.compute_loss(student, inputs, return_outputs=True)
        assert sorted(m) == sorted(DPO_METRICS) == sorted(ref_m)
        assert abs(float(loss) - float(ref_loss)) < 1e-2 * abs(float(ref_loss)) + 5e-3, (lt, float(loss), float(ref_loss))
        for k in DPO_METRICS:
            got, want = float(m[k]), float(ref_m[k])
            if k == "rewards/accuracies":
                assert got == want, (lt, k, got, want)
            else:
                assert abs(got - want) < 1e-2 * abs(want) + (2e-2 if (k.startswith("rewards") or lt == "ipo") else 5e-3), (lt, k, got, want)


def test_dpo_graph_replay_matches_eager():
    """Un-padded pairs without explicit router noise are captured into a CUDA graph after two eager warm-ups; the replayed losses and
    all ten logged metrics equal the eager ones (dense policy, whose forward draws no router noise; lr = 0)."""
    from llavamod.model import synthetic as S
    teacher = S.make_teacher(dict(S.ARCH["tiny"]), "tiny", seed=0)
    student = S.make_teacher(dict(S.ARCH["tiny"]), "tiny", seed=9).train()
    student.get_image_tower().load_state_dict(teacher.get_image_tower().state_dict())
    for n, p in student.named_parameters():
        p.requires_grad = "image_tower" not in n
    pairs = []
    for i in range(3):
        inputs = _dpo_inputs(student, seeds=(60 + 2 * i, 61 + 2 * i))[-1]
        del inputs["moe_noise"]                                    # the dense policy draws none
        pairs.append(inputs)
    tr = Hh.make_trainer(student, teacher, "sigmoid", lr=0.0, kind="dpo")
    tr.use_cuda_graphs = False
    eager = [float(tr.training_step(student, dict(pairs[i % 3]))) for i in range(6)]
    tr2 = Hh.make_trainer(student, teacher, "sigmoid", lr=0.0, kind="dpo")
    tr2.optimizer = tr.optimizer
    got = [float(tr2.training_step(student, dict(pairs[i % 3]))) for i in range(6)]
    assert tr2._graphs and any("graph" in e for e in tr2._graphs.values())
    for a, b in zip(eager, got):
        assert abs(a - b) < 1e-5 * abs(a) + 1e-6, (eager, got)
    for k in DPO_METRICS:
        want = [float(v) for v in tr._stored_metrics["train"][k]]
        have = [float(v) for v in tr2._stored_metrics["train"][k]]
        assert len(want) == len(have) == 6, k
        for a, b in zip(want, have):
            assert abs(a - b) < 1e-5 * abs(a) + 1e-6, (k, want, have)


@pytest.mark.parametrize("loss_type", ["sigmoid", "ipo"])
def test_dpo_gradients_match_oracle_autograd(loss_type):
    """Backward of the preference step through the fused log-prob head (lmod_logp_gather_bwd), two student forwards sharing one set of
    weights: every trainable gradient against fp32 autograd of the oracle, same bar as the mimic step (8 % of the tensor norm)."""
    student, teacher = Hh.tiny_pair()
    # seeds whose top-2 gate logits are never closer than the bf16-vs-fp32 activation noise: one token routed to a
    # different expert on the two sides moves ~2 % of an expert's rows and would drown the arithmetic being compared -- the test first
    # proves that both sides route identically, then compares gradients
    bc, nc, br, nr, inputs = _dpo_inputs(student, seeds=(24, 26))
    sd_s = Hh.oracle_state(student)
    train_keys = [n for n, p in student.named_parameters() if p.requires_grad]
    for k in train_keys:
        sd_s[k].requires_grad_(True)
    with torch.no_grad():
        tc, _ = Hh.oracle_forward(teacher, bc)
        trj, _ = Hh.oracle_forward(teacher, br)
    lc, cc = Hh.cfgs_of(student)
    recs = []
    for b, nz in ((bc, nc), (br, nr)):
        rec = []
        R.llava_forward(Hh.oracle_state(student), lc, cc, b["input_ids"], b["attention_mask"], b["labels"], [im.float() for im in b["images"]], nz, record=rec)
        with torch.no_grad():
            g = student.forward_hidden(input_ids=b["input_ids"], labels=b["labels"], attention_mask=b["attention_mask"], images=b["images"],
                                       moe_noise=[n.cuda() for n in nz])["records"][0]
        assert torch.equal(g["idx"].cpu().long()[:, 0], rec[0]["idx1"]) and torch.equal(g["idx"].cpu().long()[:, 1], rec[0]["idx2"])
        assert torch.equal(g["row"].cpu()[:, 0] >= 0, rec[0]["keep1"]) and torch.equal(g["row"].cpu()[:, 1] >= 0, rec[0]["keep2"])
    pc, _ = Hh.oracle_forward(student, bc, nc, sd=sd_s)
    pr, _ = Hh.oracle_forward(student, br, nr, sd=sd_s)
    ref_loss, _ = R.dpo_compute_loss(pc, pr, tc["logits"], tc["labels"], trj["logits"], trj["labels"], 0.1, loss_type, True)
    ref_loss.backward()
    tr = Hh.make_trainer(student, teacher, loss_type, kind="dpo")
    opt = tr.create_optimizer()
    opt.zero_grad()
    loss = tr.compute_loss(student, inputs)
    loss.backward()
    torch.cuda.synchronize()
    worst = 0.0
    for n, p in student.named_parameters():
        if not p.requires_grad:
            continue
        g, r = p.grad.float().cpu(), sd_s[n].grad
        rel = (g - r).norm().item() / (r.norm().item() + 1e-12)
        worst = max(worst, rel)
        assert rel < 0.08, (loss_type, n, rel)
    print("dpo worst relative grad error", loss_type, worst)


def test_dpo_loss_known_answers():
    student, teacher = Hh.tiny_pair()
    # analytic known answers: policy == reference -> sigmoid loss log 2, kto_pair 0.5 (SURVEY.md 8c)
    z = torch.zeros(3, device="cuda")
    tr = Hh.make_trainer(student, teacher, "sigmoid", kind="dpo")
    assert abs(tr.dpo_loss(z, z, z, z)[0].mean().item() - 0.6931472) < 1e-6
    tr.loss_type = "kto_pair"
    assert abs(tr.dpo_loss(z, z, z, z)[0].mean().item() - 0.5) < 1e-6
