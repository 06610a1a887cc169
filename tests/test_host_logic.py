"""CPU tests of the host-side mirror of the reference interface: splice plan (integer, bit exact vs the oracle), flag
parsing, schedules, config/ checkpoint key layout (against the reference's own state_dict in tests/golden)."""
import os

import numpy as np
import pytest
import torch

from oracle import restated as R
from tests.golden import shards


def test_splice_plan_bit_exact_vs_oracle():
    from llavamod.model.llava_arch import splice_plan
    g = torch.Generator().manual_seed(0)
    for trial in range(20):
        B, Tt, P = 4, 17, 5
        ids = torch.randint(0, 99, (B, Tt), generator=g)
        for b in range(B):
            for _ in range(int(torch.randint(0, 3, (1,), generator=g))):
                ids[b, int(torch.randint(0, Tt, (1,), generator=g))] = -200
        mask = torch.ones(B, Tt, dtype=torch.bool)
        mask[1, int(torch.randint(1, Tt, (1,), generator=g)):] = False
        labels = ids.clone(); labels[:, :3] = -100
        for side in ("right", "left"):
            for m in (mask, None):
                o = R.splice_plan(ids, m, labels, P, side)
                p = splice_plan(ids.numpy(), None if m is None else m.numpy(), labels.numpy(), P, side)
                for a, b in zip(o, p):
                    assert torch.equal(a, torch.from_numpy(b))


def test_empty_and_ragged_inputs():
    from llavamod.model.llava_arch import splice_plan
    ids = np.array([[5, -200, 7, 0], [1, 2, 3, 4]])
    mask = np.array([[1, 1, 1, 0], [0, 0, 0, 0]], bool)          # second sample fully masked -> empty row
    src, nl, nm, pos, img = splice_plan(ids, mask, ids.copy(), 3)
    assert src.shape == (2, 5) and nm[1].sum() == 0 and (nl[1] == -100).all()
    assert list(src[0]) == [5, -1, -2, -3, 7] and list(img[0]) == [-1, 0, 0, 0, -1]


def test_args_parser_accepts_the_reference_shell_flags():
    from llavamod.config.args import (AlignArguments, DataArguments, ModelArguments, TrainingArguments, parse_args_into_dataclasses)
    argv = ("--deepspeed x.json --moe_enable True --moe_finetune False --num_experts 4 --top_k_experts 2 --capacity_factor 1.5 "
            "--moe_mode sparse --use_residual False --router_aux_loss_coef 0.01 --train_modules mlp.gate_proj mlp.up_proj mlp.down_proj wg "
            "--policy_model_name_or_path /x/qwen1.5-0.5b --ref_model_name_or_path /x/qwen1.5-7b --policy_model_type sparse --ref_model_type dense "
            "--loss_type kd_lm --moe_loss_enable True --distill_all_tokens False --version qwen --image_tower openai/clip-vit-large-patch14-336 "
            "--image_projector_type mlp2x_gelu --mm_vision_select_layer -2 --image_aspect_ratio pad --bf16 True --output_dir /tmp/o "
            "--per_device_train_batch_size 1 --gradient_accumulation_steps 8 --learning_rate 2e-5 --weight_decay 0. --warmup_ratio 0.03 "
            "--lr_scheduler_type cosine --logging_steps 1 --tf32 True --model_max_length 2048 --gradient_checkpointing False "
            "--dataloader_num_workers 4 --lazy_preprocess True --report_to wandb --save_steps 1000 --save_total_limit 2").split()
    m, d, t, a = parse_args_into_dataclasses((ModelArguments, DataArguments, TrainingArguments, AlignArguments), argv)
    assert m.moe_enable and m.num_experts == [4] and m.train_modules == ["mlp.gate_proj", "mlp.up_proj", "mlp.down_proj", "wg"]
    assert t.gradient_accumulation_steps == 8 and t.learning_rate == 2e-5 and t.deepspeed == "x.json" and t.bf16
    assert a.loss_type == "kd_lm" and a.moe_loss_enable and d.image_aspect_ratio == "pad"


def test_cosine_schedule_matches_oracle():
    from llavamod.train.engine import cosine_lr
    for total in (10, 100, 1234):
        for s in range(0, total + 1, max(1, total // 17)):
            assert cosine_lr(s, total, 2e-5) == R.cosine_lr(s, total, 2e-5)


@pytest.mark.parametrize("name", ["dense_mha", "dense_gqa"])
def test_checkpoint_key_layout_equals_reference(name, golden_dir):
    """The reference's own state_dict (golden fixture) must load into our dense class key-for-key, shape-for-shape."""
    from llavamod.model import LlavaQwen1_5Config, LlavaQwen1_5ForCausalLM
    fx = shards.load(golden_dir, name)
    kw = fx["kw"]
    clip = dict(hidden_size=64, intermediate_size=128, num_hidden_layers=3, num_attention_heads=kw.get("clip_heads", 4), image_size=32, patch_size=8)
    cfg = LlavaQwen1_5Config(vocab_size=kw["vocab"], hidden_size=kw["hidden"], intermediate_size=kw["inter"],
                             num_hidden_layers=kw["layers"], num_attention_heads=kw["heads"], num_key_value_heads=kw["kv_heads"],
                             rope_theta=1e6, mm_image_tower=clip, image_projector_type="mlp2x_gelu", mm_hidden_size=64,
                             mm_vision_select_layer=-2)
    m = LlavaQwen1_5ForCausalLM(cfg, device="cpu", dtype=torch.float32)
    m.get_model().get_image_tower().load_model()
    ours = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    ref = {k: tuple(v.shape) for k, v in fx["state_dict"].items() if "position_ids" not in k}
    assert ours == ref
    from llavamod.model.builder_io import load_into
    load_into(m, {k: v for k, v in fx["state_dict"].items() if k in ours}, strict=True)
    a = m.model.layers[0].self_attn
    H = kw["hidden"]
    assert torch.equal(a.qkv_weight[:H], fx["state_dict"]["model.layers.0.self_attn.q_proj.weight"])       # fused buffer stays fused
    assert torch.equal(m.model.layers[1].mlp.gu_weight[kw["inter"]:], fx["state_dict"]["model.layers.1.mlp.up_proj.weight"])


def test_moe_checkpoint_keys_and_upcycling():
    from llavamod.model import LLaVAMoDQwen1_5Config, LLaVAMoDQwen1_5ForCausalLM, LLaVAMoDQwen1_5ForCausalLMFineTune
    from llavamod.model import synthetic as S
    clip = S.CLIP["tiny"]
    cfg = LLaVAMoDQwen1_5Config(**dict(S.ARCH["tiny"], num_hidden_layers=4), mm_image_tower=dict(clip), image_projector_type="mlp2x_gelu",
                                mm_hidden_size=64, mm_vision_select_layer=-2)
    m = LLaVAMoDQwen1_5ForCausalLM(cfg, device="cpu", dtype=torch.float32)
    m.initialize_moe_modules(S.moe_args())
    m.get_model().initialize_vision_modules(S.vision_args(clip))
    keys = set(m.state_dict().keys())
    assert "model.layers.0.mlp.deepspeed_moe.gate.wg.weight" in keys and "model.layers.2.mlp.deepspeed_moe.experts.deepspeed_experts.3.down_proj.weight" in keys
    assert "model.layers.1.mlp.gate_proj.weight" in keys and "model.layers.0.mlp.gate_proj.weight" not in keys
    assert m.config.moe["moe_layers_idx"] == [0, 2] and m.config.moe["num_experts"] == [4, 4]
    train = sorted(n for n, p in m.named_parameters() if p.requires_grad)
    assert train == sorted(R.trainable_keys(m.state_dict()))                                          # freeze-by-name rule
    assert m.state_dict()["model.layers.0.mlp.deepspeed_moe.gate.wg.weight"].dtype == torch.float32
    # save -> FineTune class rebuilds the MoE from config.moe and loads the sparse checkpoint directly
    import tempfile
    d = tempfile.mkdtemp()
    m.save_pretrained(d)
    m2 = LLaVAMoDQwen1_5ForCausalLMFineTune.from_pretrained(d, device="cpu", torch_dtype=torch.float32)
    for k, v in m.state_dict().items():
        assert torch.equal(v, m2.state_dict()[k]), k


def test_auto_factories_resolve_the_registered_families(tmp_path):
    """llava_qwen1_5.py:170-171 / llava_qwen2.py:133-134 / llava_qwen*_moe.py:684-687: `AutoConfig.from_pretrained(dir)` picks the config class
    from config.json's model_type; the model class registered LAST for a config is the one the factory builds (the Eval class for MoE)."""
    import llavamod.model as M
    from llavamod.model.auto import _MODELS
    for mt, cfg_cls, model_cls in (("llava_qwen1_5", M.LlavaQwen1_5Config, M.LlavaQwen1_5ForCausalLM),
                                   ("llava_qwen2", M.LlavaQwen2Config, M.LlavaQwen2ForCausalLM),
                                   ("moe_llava_qwen1_5", M.LLaVAMoDQwen1_5Config, M.EvalLLaVAMoDQwen1_5ForCausalLM),
                                   ("moe_llava_qwen2", M.LLaVAMoDQwen2Config, M.EvalLLaVAMoDQwen2ForCausalLM)):
        d = tmp_path / mt
        cfg_cls(vocab_size=64, hidden_size=32, intermediate_size=48, num_hidden_layers=1, num_attention_heads=2).save_pretrained(str(d))
        cfg = M.AutoConfig.from_pretrained(str(d))
        assert type(cfg) is cfg_cls and cfg.model_type == mt and cfg.hidden_size == 32
        assert _MODELS[cfg_cls] is model_cls
        assert type(M.AutoConfig.for_model(mt, hidden_size=16)) is cfg_cls
    (tmp_path / "other").mkdir()
    (tmp_path / "other" / "config.json").write_text('{"model_type": "llama"}')
    with pytest.raises(ValueError):
        M.AutoConfig.from_pretrained(str(tmp_path / "other"))
    with pytest.raises(ValueError):
        M.AutoConfig.register("not_its_type", M.LlavaQwen2Config)
