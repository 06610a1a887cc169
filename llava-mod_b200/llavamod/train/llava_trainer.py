"""Plain cross-entropy trainer of the stages either side of distillation (SURVEY section 8f row N3): adaptor pre-training
(`--tune_mm_mlp_adapter`, `--version plain`), dense SFT and MoE fine-tuning.

Reference: llavamod/train/llava_trainer.py:135-281 -- an HF `Trainer` whose loss is the model's own `.loss` (shifted CE, + moe_loss for
the sparse classes), with the length-grouped sampler (:137-150; ours lives in BaseTrainer.get_train_dataloader), the decay / no-decay /
projector-LR optimizer groups (:152-247; see BaseTrainer.create_optimizer for what the shells actually use) and adaptor-only
checkpoints (:249-281).  Every kernel is the distillation path's; the teacher, the KL head and the side stream drop out."""
import torch

from .trainer_base import AdapterCheckpointMixin, BaseTrainer, image_count_shape


class LLaVATrainer(AdapterCheckpointMixin, BaseTrainer):
    # ---- loss ------------------------------------------------------------------------------------------------------------------
    def compute_loss(self, model, inputs, return_outputs=False):
        images = inputs.get("images")
        if images is not None and not torch.is_tensor(images):
            images = [im.to(model.device, non_blocking=True) for im in images]
        loss, ce, moe = model.forward_train_loss(input_ids=inputs["input_ids"], attention_mask=inputs.get("attention_mask"), labels=inputs["labels"],
                                                 images=images, moe_noise=inputs.get("moe_noise"), plan=inputs.get("splice_plan"))
        outputs = {"loss/lm": ce}                        # no stored "loss": the logged loss is the train loop's average of the float losses
        if moe is not None:
            outputs["loss/moe_balance"] = moe.detach()
        self.store_metrics(outputs)
        return (loss, outputs) if return_outputs else loss

    # ---- CUDA-graph plumbing (BaseTrainer._graphed_micro_batch): un-padded batches with explicit router noise absent -----------
    def _graph_signature(self, inputs, next_inputs=None):
        images = inputs.get("images")
        if images is None or inputs.get("moe_noise") is not None:
            return None
        plan = inputs.get("splice_plan")
        if plan is None:
            plan = inputs["splice_plan"] = self.model.make_splice_plan(inputs["input_ids"], inputs.get("attention_mask"), inputs["labels"])
        if not plan["all_true"]:
            return None                                  # padded batches take the masked-attention path eagerly
        n, ish = image_count_shape(images)
        return ("sft", tuple(inputs["input_ids"].shape), tuple(plan["src"].shape), n, ish, plan["has_mask"], plan["has_labels"],
                self._grad_ckpt_key())
