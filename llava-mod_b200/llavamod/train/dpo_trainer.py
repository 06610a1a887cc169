"""DPOTrainer -- preference distillation (DPO / IPO / hinge / KTO-pair on sequence log-prob ratios).

Reference: llavamod/train/dpo_trainer.py (DPOTrainer :180; get_logp :462-495; dpo_loss :497-562; compute_loss :564-641).
Kept: shift by one, NO vocabulary slice, masked sequence SUM of gathered log-probs, the four loss types with beta=0.1,
``chosen_moe + rejected_moe`` added when enabled, the ten logged metrics.

Hot loop: two frozen-teacher forwards (no grad) and two student forwards; each lm_head GEMM feeds the fused
log-softmax+gather kernel (online LSE + pick, 2*V bytes/token) instead of materialising log_softmax over [B,T,V]; the DPO
scalar math runs on [B] device tensors; backward re-reads the bf16 logits once and writes d(logits) in place.
"""
from collections import defaultdict
from typing import Any, Dict, Literal, Tuple, Union

import torch
import torch.nn.functional as F

from .. import kernels as K
from ..model.utils import create_reference_model, disable_dropout_in_model
from .align_trainer import _Wrapped, same_frozen_tower
from .trainer_base import BaseTrainer


class DPOTrainer(BaseTrainer):
    def __init__(self, model=None, ref_model=None, args=None, data_collator=None, train_dataset=None, eval_dataset=None,
                 tokenizer=None, label_pad_token_id: int = -100, padding_value: int = 0, beta: float = 0.1,
                 label_smoothing: float = 0, loss_type: str = "sigmoid", moe_loss_enable: bool = False,
                 disable_dropout: bool = True, model_init=None, compute_metrics=None, callbacks=None,
                 optimizers=(None, None), preprocess_logits_for_metrics=None):
        self.ref_model = ref_model if ref_model else create_reference_model(model)
        if disable_dropout:
            disable_dropout_in_model(model)
        self.label_pad_token_id = label_pad_token_id
        self.padding_value = padding_value
        self.beta = beta
        self.label_smoothing = label_smoothing
        self.loss_type = loss_type
        self.moe_loss_enable = moe_loss_enable
        self._stored_metrics = defaultdict(lambda: defaultdict(list))
        super().__init__(model=model, args=args, data_collator=data_collator, train_dataset=train_dataset,
                         eval_dataset=eval_dataset, tokenizer=tokenizer, model_init=model_init,
                         compute_metrics=compute_metrics, callbacks=callbacks, optimizers=optimizers,
                         preprocess_logits_for_metrics=preprocess_logits_for_metrics)
        if not hasattr(self.ref_model, "module"):
            self.ref_model = _Wrapped(self.ref_model)
        self.ref_model.module.eval()
        for p in self.ref_model.module.parameters():
            p.requires_grad = False
        self.share_tower = same_frozen_tower(self.model, self.ref_model.module)
        import os
        self.overlap_teacher = bool(int(os.environ.get("LLAVAMOD_OVERLAP_TEACHER", "1"))) and next(model.parameters()).is_cuda
        self._teacher_stream = torch.cuda.Stream() if self.overlap_teacher else None

    def _seq_logp(self, model, fwd, tower_feats, noise=None, grad=True, plan=None):
        r = model.forward_hidden(**fwd, tower_features=tower_feats, moe_noise=noise, plan=plan)
        if r["hidden"].shape[:2] != r["labels"].shape:
            raise ValueError("Logits (batch and sequence length dim) and labels must have the same shape.")
        if grad:
            logps = K.logp_head(r["hidden"], model.lm_head.weight, r["labels"], model.lm_head_grad)
        else:
            h = r["hidden"]
            logits = K.mm_nt(h.reshape(-1, h.shape[-1]), model.lm_head.weight).view(h.shape[0], h.shape[1], -1)
            logps = K.logp_gather(logits, r["labels"].contiguous())[0]
        return logps, r

    def get_logp(self, model, inputs, average_log_prob: bool = False):
        """dpo_trainer.py:462-495 -> (sequence log-probs [B], sft_loss, moe_loss).  API-compat form (runs the public forward)."""
        outputs = model(**inputs, return_dict=True)
        logits, labels = outputs.logits, outputs.labels
        if logits.shape[:-1] != labels.shape:
            raise ValueError("Logits (batch and sequence length dim) and labels must have the same shape.")
        seq = K.logp_gather(logits.to(torch.bfloat16).contiguous(), labels.contiguous(), average=average_log_prob)[0]
        moe = outputs.moe_loss if (getattr(self.args, "moe_enable", False) and self.moe_loss_enable and getattr(outputs, "moe_loss", None) is not None) else None
        return seq, outputs.loss, moe

    def dpo_loss(self, policy_chosen_logps, policy_rejected_logps, reference_chosen_logps, reference_rejected_logps,
                 reference_free: bool = False) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """dpo_trainer.py:497-562 ([B]-sized device math; K18 is a trivial epilogue of K17)."""
        pi_logratios = policy_chosen_logps - policy_rejected_logps
        ref_logratios = 0 if reference_free else reference_chosen_logps - reference_rejected_logps
        logits = pi_logratios - ref_logratios
        if self.loss_type == "sigmoid":
            losses = (-F.logsigmoid(self.beta * logits) * (1 - self.label_smoothing)
                      - F.logsigmoid(-self.beta * logits) * self.label_smoothing)
        elif self.loss_type == "hinge":
            losses = torch.relu(1 - self.beta * logits)
        elif self.loss_type == "ipo":
            losses = (logits - 1 / (2 * self.beta)) ** 2
        elif self.loss_type == "kto_pair":
            chosen_KL = (policy_chosen_logps - reference_chosen_logps).mean().clamp(min=0)
            rejected_KL = (policy_rejected_logps - reference_rejected_logps).mean().clamp(min=0)
            chosen_logratios = policy_chosen_logps - reference_chosen_logps
            rejected_logratios = policy_rejected_logps - reference_rejected_logps
            losses = torch.cat((1 - torch.sigmoid(self.beta * (chosen_logratios - rejected_KL)),
                                1 - torch.sigmoid(self.beta * (chosen_KL - rejected_logratios))), 0)
        else:
            raise ValueError(f"Unknown loss type: {self.loss_type}. Should be one of ['sigmoid', 'hinge']")
        chosen_rewards = self.beta * (policy_chosen_logps - reference_chosen_logps).detach()
        rejected_rewards = self.beta * (policy_rejected_logps - reference_rejected_logps).detach()
        return losses, chosen_rewards, rejected_rewards

    def compute_loss(self, model, inputs: Dict[str, Union[torch.Tensor, Any]], return_outputs=False):
        assert self.ref_model is not None, "ref model can not be none!"
        ref = self.ref_model.module
        images = inputs.get("images", None)
        tower_feats = None
        if self.share_tower and images is not None:
            with torch.no_grad():
                dev = model.device
                images = torch.stack([im.to(dev, non_blocking=True) for im in images]) if not torch.is_tensor(images) else images.to(dev)
                tower_feats = model.get_image_tower()(images.to(model.dtype))                 # once instead of 4x (dpo_trainer.py:595-607)
        ch = dict(input_ids=inputs["chosen_input_ids"], labels=inputs["chosen_labels"], attention_mask=inputs["chosen_attention_mask"], images=images)
        rj = dict(input_ids=inputs["rejected_input_ids"], labels=inputs["rejected_labels"], attention_mask=inputs["rejected_attention_mask"], images=images)
        # one host splice plan per side, shared by the reference and the policy forward when their towers emit the same patch count
        plan_c, plan_r = inputs.get("splice_plan_chosen"), inputs.get("splice_plan_rejected")
        if plan_c is None and images is not None and model.get_image_tower() is not None and \
                model.get_image_tower().num_patches == ref.get_image_tower().num_patches:
            plan_c = model.make_splice_plan(ch["input_ids"], ch["attention_mask"], ch["labels"])
            plan_r = model.make_splice_plan(rj["input_ids"], rj["attention_mask"], rj["labels"])
        # the two frozen reference forwards are independent of the policy until dpo_loss: they run on a side stream so the 0.5B policy's
        # small kernels fill the gaps of the 7B reference's machine-filling GEMMs (a fork/join inside the CUDA graph), as in AlignTrainer
        main = torch.cuda.current_stream()
        side = self._teacher_stream if self.overlap_teacher else None
        if side is not None:
            side.wait_stream(main)
        with torch.no_grad(), torch.cuda.stream(side if side is not None else main):
            reference_chosen_logps, _ = self._seq_logp(ref, ch, tower_feats, grad=False, plan=plan_c)
            reference_rejected_logps, _ = self._seq_logp(ref, rj, tower_feats, grad=False, plan=plan_r)
        noise = inputs.get("moe_noise") or (None, None)
        policy_chosen_logps, rc = self._seq_logp(model, ch, tower_feats, noise[0], plan=plan_c)
        policy_rejected_logps, rr = self._seq_logp(model, rj, tower_feats, noise[1], plan=plan_r)
        if side is not None:
            main.wait_stream(side)
            reference_chosen_logps.record_stream(main)
            reference_rejected_logps.record_stream(main)
        reward_losses, chosen_rewards, rejected_rewards = self.dpo_loss(policy_chosen_logps, policy_rejected_logps,
                                                                        reference_chosen_logps, reference_rejected_logps)
        enabled = getattr(self.args, "moe_enable", False) and self.moe_loss_enable and getattr(model, "is_moe", False)
        if enabled and len(rc["l_aux"]) and len(rr["l_aux"]):
            moe_loss = model.moe_loss_from(rc["l_aux"]) + model.moe_loss_from(rr["l_aux"])
            losses = reward_losses + moe_loss
        else:
            moe_loss = torch.full_like(reward_losses, -1.0)
            losses = reward_losses
        reward_accuracies = (chosen_rewards > rejected_rewards).float()
        # the reference logs the chosen forward's model loss (dpo_trainer.py:626): shifted CE averaged over the batch's supervised tokens
        # (+ the model's own moe_loss, llava_qwen1_5_moe.py:431-434).  The gathered token log-probs of the fused head ARE that CE's terms.
        n_tok = (rc["labels"][:, 1:] != self.label_pad_token_id).sum().clamp(min=1)
        policy_chosen_sft = -policy_chosen_logps.detach().sum() / n_tok
        if getattr(model, "is_moe", False) and len(rc["l_aux"]):
            policy_chosen_sft = policy_chosen_sft + model.moe_loss_from(rc["l_aux"]).detach()
        outputs = {"loss": losses.detach().mean(), "loss/reward": reward_losses.detach().mean(),
                   "loss/moe_balance": moe_loss.detach().mean(),
                   "loss/policy_chosen": policy_chosen_sft,
                   "rewards/chosen": chosen_rewards.mean(), "rewards/rejected": rejected_rewards.mean(),
                   "rewards/accuracies": reward_accuracies.mean(), "rewards/margins": (chosen_rewards - rejected_rewards).mean(),
                   "logps/chosen": policy_chosen_logps.detach().mean(), "logps/rejected": policy_rejected_logps.detach().mean()}
        self.store_metrics(outputs, train_eval="train")
        if return_outputs:
            return losses.mean(), outputs
        return losses.mean()

    def store_metrics(self, metrics: Dict[str, float], train_eval: Literal["train", "eval"] = "train") -> None:
        if self._suppress_store:          # graph capture: the static output tensors are cloned after every replay instead
            return
        for key, value in metrics.items():
            self._stored_metrics[train_eval][key].append(value)

    # ---- CUDA-graph plumbing (see BaseTrainer._graphed_micro_batch): the four forwards + two backwards of a pair are captured once per
    # input signature; static inputs = the image tensor and the two splice plans ------------------------------------------------------
    def _graph_signature(self, inputs, next_inputs=None):
        images = inputs.get("images")
        if images is None or inputs.get("moe_noise") is not None or not self.share_tower:
            return None
        for side in ("chosen", "rejected"):
            if inputs.get("splice_plan_" + side) is None:
                inputs["splice_plan_" + side] = self.model.make_splice_plan(inputs[side + "_input_ids"], inputs.get(side + "_attention_mask"),
                                                                            inputs[side + "_labels"])
        pc, pr = inputs["splice_plan_chosen"], inputs["splice_plan_rejected"]
        if not (pc["all_true"] and pr["all_true"]):
            return None                   # padded pairs run eagerly
        n_img = len(images) if not torch.is_tensor(images) else images.shape[0]
        ish = tuple(images[0].shape) if not torch.is_tensor(images) else tuple(images.shape[1:])
        return ("dpo", tuple(pc["src"].shape), tuple(pr["src"].shape), n_img, ish, pc["has_mask"], pr["has_mask"], self.loss_type)

    def _graph_static_inputs(self, inputs, static):
        images = inputs["images"]
        if static is None:
            dev = self.model.device
            n = len(images) if not torch.is_tensor(images) else images.shape[0]
            ish = tuple(images[0].shape) if not torch.is_tensor(images) else tuple(images.shape[1:])
            static = {k: inputs[k] for k in ("chosen_input_ids", "chosen_labels", "chosen_attention_mask", "rejected_input_ids",
                                             "rejected_labels", "rejected_attention_mask")}
            static["images"] = torch.empty((n,) + ish, dtype=self.model.dtype, device=dev)
            for side in ("chosen", "rejected"):
                static["splice_plan_" + side] = {k: (torch.empty_like(v) if torch.is_tensor(v) else v) for k, v in inputs["splice_plan_" + side].items()}
        if torch.is_tensor(images):
            static["images"].copy_(images, non_blocking=True)
        else:
            for i, im in enumerate(images):
                static["images"][i].copy_(im, non_blocking=True)
        for side in ("chosen", "rejected"):
            for k, v in inputs["splice_plan_" + side].items():
                if torch.is_tensor(v):
                    static["splice_plan_" + side][k].copy_(v, non_blocking=True)
        return static

    def log(self, logs: Dict[str, float]) -> None:
        train_eval = "train" if "loss" in logs else "eval"
        for key, metrics in self._stored_metrics[train_eval].items():
            logs[key] = torch.stack([torch.as_tensor(m, dtype=torch.float32).detach().cpu() for m in metrics]).mean().item()
        del self._stored_metrics[train_eval]
        return super().log(logs)
