"""--gradient_checkpointing on the host: the HF model surface, the flag's way from the reference's shell flags through the four entry points
to the policy's decoder (never the teacher's), the use_cache rule and the trainers' graph signatures.  Models are tiny and on the CPU."""
import json
import os

import pytest
import torch

EXPORTED = ("LlavaQwen1_5ForCausalLM", "LlavaQwen2ForCausalLM", "LLaVAMoDQwen1_5ForCausalLM", "LLaVAMoDQwen1_5ForCausalLMFineTune",
            "EvalLLaVAMoDQwen1_5ForCausalLM", "LLaVAMoDQwen2ForCausalLM", "LLaVAMoDQwen2ForCausalLMFineTune", "EvalLLaVAMoDQwen2ForCausalLM")


def _tiny(sparse, seed=0):
    from llavamod.model import synthetic as S
    if sparse:
        return S.make_student("tiny", "tiny", device="cpu", dtype=torch.float32, seed=seed)
    return S.make_teacher("tiny", "tiny", device="cpu", dtype=torch.float32, seed=seed)


@pytest.mark.parametrize("name", EXPORTED)
def test_every_exported_class_has_the_hf_checkpointing_surface(name):
    import llavamod.model.language_model.llava_qwen1_5_moe as m15
    import llavamod.model.language_model.llava_qwen2_moe as m2
    import llavamod.model as M
    cls = getattr(M, name, None) or getattr(m15, name, None) or getattr(m2, name)
    assert cls.supports_gradient_checkpointing is True
    for meth in ("gradient_checkpointing_enable", "gradient_checkpointing_disable", "enable_input_require_grads", "disable_input_require_grads"):
        assert callable(getattr(cls, meth)), meth
    m = _tiny(sparse=cls.is_moe)
    assert not m.is_gradient_checkpointing and m.get_model().gradient_checkpointing is False
    m.gradient_checkpointing_enable(gradient_checkpointing_kwargs={"use_reentrant": False})
    assert m.is_gradient_checkpointing and m.get_model().gradient_checkpointing is True
    m.gradient_checkpointing_disable()
    assert not m.is_gradient_checkpointing
    m.enable_input_require_grads()
    assert m._input_require_grads
    m.disable_input_require_grads()
    assert not m._input_require_grads


def test_training_forward_with_use_cache_warns_and_runs_without_a_cache(monkeypatch):
    m = _tiny(sparse=False).train()
    m.gradient_checkpointing_enable()
    seen = {}

    class Stop(Exception):
        pass

    def forward_hidden(*a, cache=None, **kw):
        seen["cache"] = cache
        raise Stop

    monkeypatch.setattr(m, "forward_hidden", forward_hidden)
    ids = torch.zeros(1, 4, dtype=torch.long)
    with pytest.warns(UserWarning, match="use_cache=True.*incompatible with gradient checkpointing"):
        with pytest.raises(Stop):
            m(input_ids=ids, use_cache=True)
    assert seen["cache"] is None
    m.eval()                                                      # generation keeps its cache
    with pytest.raises(Stop):
        m(input_ids=ids, use_cache=True)
    assert seen["cache"] is not None


def _entry_argv(golden_dir, shell, out, ckpt):
    with open(os.path.join(golden_dir, "shell_argv.json")) as f:
        argv = list(json.load(f)[shell]["argv"])
    argv[argv.index("--data_path") + 1] = "synthetic:4"
    argv[argv.index("--output_dir") + 1] = out
    return argv + ["--num_train_epochs", "0", "--max_steps", "-1", "--model_max_length", "64", "--gradient_checkpointing", ckpt,
                   "--dataloader_num_workers", "0"]


ENTRIES = [("pretrain.sh", "train"), ("finetune.sh", "train"), ("dense2sparse_distillation.sh", "align"),
           ("preference_distillation.sh", "dpo"), ("dense2sparse_distillation.sh", "train_mem")]


@pytest.mark.parametrize("ckpt", ["True", "False"])
@pytest.mark.parametrize("shell,entry", ENTRIES)
def test_the_flag_reaches_the_policy_through_every_entry_point(shell, entry, ckpt, golden_dir, tmp_path, monkeypatch):
    """The reference's shell flags (with --gradient_checkpointing set as given) through align_train / dpo_train / train / train_mem, up to
    the start of training: the policy's Qwen2Model has checkpointing on and its embeddings require grad iff the flag is True; the teacher's
    never does."""
    from llavamod.train import align_train, dpo_train, train as train_mod, train_mem
    from llavamod.train.trainer_base import BaseTrainer
    made = []

    def create_model_tokenizer(model_args, data_args, training_args, name_or_path, model_type, pretrain_adapter=None, device="cuda"):
        sparse = model_type == "sparse"
        if sparse:
            model_args.moe_enable = True
        m = _tiny(sparse, seed=len(made))
        m.config.use_cache = False
        made.append(m)
        return m, None

    for mod in (align_train, dpo_train, train_mod):
        monkeypatch.setattr(mod, "create_model_tokenizer", create_model_tokenizer)
        monkeypatch.setattr(mod, "init_process", lambda seed: torch.device("cpu"))
    seen = {}
    orig_train = BaseTrainer.train

    def train(self, resume_from_checkpoint=None):
        out = orig_train(self, resume_from_checkpoint)
        seen["trainer"] = self
        return out
    monkeypatch.setattr(BaseTrainer, "train", train)
    argv = _entry_argv(golden_dir, shell, str(tmp_path / "out"), ckpt)
    if entry == "train_mem":
        train_mem.main(argv + ["--stage", "mimic"])
    else:
        {"train": train_mod, "align": align_train, "dpo": dpo_train}[entry].train(argv)
    tr = seen["trainer"]
    on = ckpt == "True"
    assert tr.model is made[0]
    assert tr.model.get_model().gradient_checkpointing is on and tr.model._input_require_grads is on
    if hasattr(tr, "ref_model"):
        ref = tr.ref_model.module
        assert ref is made[1] and ref.get_model().gradient_checkpointing is False and not ref._input_require_grads


def test_toggling_checkpointing_changes_the_graph_signature():
    from llavamod.config.args import TrainingArguments
    from llavamod.train.llava_trainer import LLaVATrainer
    m = _tiny(sparse=False)
    tr = LLaVATrainer(model=m, args=TrainingArguments(output_dir="/tmp/lmod_sig"))
    ids = torch.randint(0, 100, (2, 12))
    ids[:, 3] = -200
    inputs = dict(input_ids=ids, labels=ids.clone(), attention_mask=None, images=[torch.zeros(3, 32, 32)] * 2)
    off = tr._graph_signature(dict(inputs))
    m.gradient_checkpointing_enable()
    on = tr._graph_signature(dict(inputs))
    assert off is not None and on is not None and off != on
    m.gradient_checkpointing_disable()
    assert tr._graph_signature(dict(inputs)) == off
