"""Every flag of the reference's six Qwen training shells (shells/train/qwen/*.sh) must be accepted by the matching entry point's
argument dataclasses (SURVEY section 8b "Entry points").  The shells' launch lines are stored, parsed, in tests/golden/shell_argv.json
(tests/golden/make_ref_golden.py)."""
import json
import os

import pytest

ENTRY = {"pretrain.sh": "train", "finetune.sh": "train", "finetune_moe.sh": "train", "dense2dense_distillation.sh": "align",
         "dense2sparse_distillation.sh": "align", "preference_distillation.sh": "dpo"}


def shell_argv(golden_dir, shell):
    with open(os.path.join(golden_dir, "shell_argv.json")) as f:
        d = json.load(f)[shell]
    return d["argv"], d["script"]


@pytest.mark.parametrize("shell", sorted(ENTRY))
def test_shell_flags_parse(shell, golden_dir):
    from llavamod.config.args import (AlignArguments, DataArguments, DPOArguments, ModelArguments, TrainingArguments,
                                      parse_args_into_dataclasses)
    argv, script = shell_argv(golden_dir, shell)
    kind = ENTRY[shell]
    assert script.endswith({"train": "train.py", "align": "align_train.py", "dpo": "dpo_train.py"}[kind])
    classes = {"train": (ModelArguments, DataArguments, TrainingArguments),
               "align": (ModelArguments, DataArguments, TrainingArguments, AlignArguments),
               "dpo": (ModelArguments, DataArguments, TrainingArguments, DPOArguments)}[kind]
    out = parse_args_into_dataclasses(classes, argv)
    m, d, t = out[:3]
    assert t.output_dir and t.model_max_length >= 1024 and t.bf16 and d.data_path and d.image_folder
    if shell == "pretrain.sh":
        assert m.tune_mm_mlp_adapter and t.learning_rate == 1e-3
    if shell == "finetune_moe.sh":
        assert m.moe_enable and m.train_modules and m.num_experts
    if kind == "align":
        assert out[3].loss_type in ("kd_lm", "only_kd") and out[3].policy_model_type in ("dense", "sparse")
    if kind == "dpo":
        assert out[3].loss_type in ("sigmoid", "hinge", "ipo", "kto_pair")
    assert os.path.exists(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "llava-mod_b200", "llavamod", "train",
                                       os.path.basename(script)))
