"""``--optim adamw_bnb_8bit`` / ``adamw_8bit`` through the entry points: align_train and dpo_train train to the final save with the
model layout unchanged, a resumed 8-bit run reproduces the uninterrupted loss sequence, a resume with the other --optim is refused, and
100 config-1 steps with 8-bit moments follow the 32-bit loss curve."""
import json
import os
import shutil

import pytest
import torch

pytestmark = pytest.mark.gpu

from tests import helpers as Hh  # noqa: E402
from tests.test_entrypoints_gpu import _check_final_save, _common_flags, _save_tiny_checkpoints  # noqa: E402


def test_align_train_8bit_runs_to_the_final_save(tmp_path, golden_dir):
    from llavamod.train import align_train
    policy, teacher, tower, tok = _save_tiny_checkpoints(str(tmp_path), golden_dir)
    out = str(tmp_path / "out_mimic")
    argv = _common_flags(policy, teacher, tower, out, golden_dir, "data_sft.json") + [
        "--loss_type", "kd_lm", "--learning_rate", "1e-3", "--num_train_epochs", "2", "--optim", "adamw_bnb_8bit"]
    tr = align_train.train(argv)
    assert tr.state.global_step == 4
    assert tr.optimizer.optim_bits == 8 and tr.optimizer.m16 is None and tr.optimizer.m8 is not None
    logs = [json.loads(l) for l in open(os.path.join(out, "trainer_log.jsonl"))]
    assert [l["step"] for l in logs] == [1, 2, 3, 4] and all(l["loss"] == l["loss"] for l in logs)
    _check_final_save(out, tr, (2, 4))
    st = torch.load(os.path.join(out, "checkpoint-4", "optimizer.pt"), map_location="cpu", weights_only=True)
    assert st["optim"] == "adamw_8bit" and st["m8"].dtype == torch.uint8 and "m16" not in st
    assert torch.equal(st["m8"], tr.optimizer.m8.cpu()) and torch.equal(st["absmax"], tr.optimizer.absmax.cpu())


def test_dpo_train_8bit_with_fp8_teacher_runs_to_the_final_save(tmp_path, golden_dir):
    from llavamod.train import dpo_train
    policy, teacher, tower, tok = _save_tiny_checkpoints(str(tmp_path), golden_dir)
    out = str(tmp_path / "out_pref")
    argv = _common_flags(policy, teacher, tower, out, golden_dir, "data_dpo.json") + [
        "--loss_type", "sigmoid", "--learning_rate", "2e-4", "--num_train_epochs", "2", "--save_steps", "1", "--optim", "adamw_8bit",
        "--ref_fp8", "True"]
    tr = dpo_train.train(argv)
    assert tr.state.global_step == 2 and tr.optimizer.optim_bits == 8
    _check_final_save(out, tr, (1, 2), use_cache=False)


def _run(policy, teacher, tower, golden_dir, out, max_steps, optim):
    from llavamod.train import align_train
    argv = _common_flags(policy, teacher, tower, out, golden_dir, "data_sft.json") + [
        "--loss_type", "kd_lm", "--learning_rate", "1e-3", "--per_device_train_batch_size", "1", "--save_steps", "2",
        "--max_steps", str(max_steps), "--seed", "7", "--optim", optim]
    os.environ["LLAVAMOD_CUDA_GRAPHS"] = "0"
    try:
        return align_train.train(argv)
    finally:
        os.environ.pop("LLAVAMOD_CUDA_GRAPHS", None)


def test_resumed_8bit_run_reproduces_the_uninterrupted_loss_sequence(tmp_path, golden_dir):
    """As test_resumed_run_reproduces_the_uninterrupted_loss_sequence, with 8-bit state: codes and scales are restored with the master."""
    policy, teacher, tower, tok = _save_tiny_checkpoints(str(tmp_path), golden_dir)
    full = _run(policy, teacher, tower, golden_dir, str(tmp_path / "a"), 5, "adamw_bnb_8bit")
    want = {h["step"]: (h["loss"], h["loss/align"], h["learning_rate"]) for h in full.state.log_history}
    assert sorted(want) == [1, 2, 3, 4, 5]
    os.makedirs(tmp_path / "b")
    shutil.copytree(tmp_path / "a" / "checkpoint-2", tmp_path / "b" / "checkpoint-2")
    resumed = _run(policy, teacher, tower, golden_dir, str(tmp_path / "b"), 5, "adamw_bnb_8bit")
    got = {h["step"]: (h["loss"], h["loss/align"], h["learning_rate"]) for h in resumed.state.log_history}
    assert sorted(got) == [3, 4, 5]
    for s in (3, 4, 5):
        assert got[s][2] == want[s][2], (s, got[s], want[s])
        for x, y in zip(got[s][:2], want[s][:2]):
            assert abs(x - y) <= 1e-5 * abs(y), (s, got[s], want[s])
    a = torch.load(tmp_path / "a" / "pytorch_model.bin", map_location="cpu", weights_only=True)
    b = torch.load(tmp_path / "b" / "pytorch_model.bin", map_location="cpu", weights_only=True)
    for k in a:
        assert (a[k].float() - b[k].float()).norm() <= 1e-4 * a[k].float().norm() + 1e-9, k
    assert any(abs(want[s][0] - want[2][0]) > 1e-4 for s in (3, 4, 5))


@pytest.mark.parametrize("saved,resumed", [("adamw_bnb_8bit", "adamw_torch"), ("adamw_torch", "adamw_8bit")])
def test_resume_with_the_other_optim_is_refused(tmp_path, golden_dir, saved, resumed):
    policy, teacher, tower, tok = _save_tiny_checkpoints(str(tmp_path), golden_dir)
    _run(policy, teacher, tower, golden_dir, str(tmp_path / "a"), 2, saved)
    with pytest.raises(ValueError) as e:
        _run(policy, teacher, tower, golden_dir, str(tmp_path / "a"), 4, resumed)
    msg = str(e.value)
    assert resumed in msg and ("adamw_bnb_8bit" in msg if saved != "adamw_torch" else "adamw_torch" in msg), msg


def test_100_steps_config1_8bit_follows_the_32bit_loss_curve():
    """BASELINE config 1, 100 optimizer steps (cosine schedule, clipping), the same batches and router noise for both optimizers.
    Bound: |loss_8bit - loss_32bit| <= 1e-3 * loss_32bit at every step.  Measured on an H100 80GB HBM3: the largest relative gap over
    the 100 steps was 4.6e-5 (step 54), so the bound leaves a factor of about 20 for other seeds and builds while staying the size of
    the 1e-3 the 32-bit path is held to against the fp32 oracle (test_loss_curve_100_steps_config1)."""
    steps, lr = 100, 2e-4
    curves = {}
    for optim in ("adamw_torch", "adamw_bnb_8bit"):
        student, teacher = Hh.tiny_pair()
        tr = Hh.make_trainer(student, teacher, "kd_lm", accum=1, lr=lr, max_steps=steps)
        tr.args.optim = optim
        assert tr.create_optimizer().optim_bits == (8 if optim == "adamw_bnb_8bit" else 32)
        losses = []
        for s in range(steps):
            batch, noise = Hh.tiny_batch(student, seed=1000 + s)
            losses.append(float(tr.training_step(student, dict(batch, moe_noise=[n.cuda() for n in noise]))))
        curves[optim] = losses
    l32, l8 = curves["adamw_torch"], curves["adamw_bnb_8bit"]
    rel = [abs(a - b) / abs(a) for a, b in zip(l32, l8)]
    print("config-1 loss, step: 32-bit / 8-bit")
    for s in range(0, steps, 5):
        print("  %3d  %.5f  %.5f" % (s + 1, l32[s], l8[s]))
    print("max relative gap %.3e at step %d" % (max(rel), rel.index(max(rel)) + 1))
    assert l8[-1] < l8[0]
    assert max(rel) <= 1e-3, (max(rel), rel.index(max(rel)) + 1)
