"""AlignTrainer -- mimic distillation (teacher-weighted CE over the vocabulary, "KL") of a sparse-MoE student.

Reference: llavamod/train/align_trainer.py (AlignTrainer :180; get_p :455-477; get_logp :479-501; compute_align_loss
:503-528; compute_loss :530-594; store_metrics/log :596-614).  Semantics kept: un-shifted mask, hard-coded vocabulary
slice 151936, ``moe_loss`` counted inside the model loss AND again by the trainer under ``kd_lm``, ``-1.0`` sentinel metric,
0/0 -> NaN for a fully masked batch.

Hot loop (``compute_loss``): frozen teacher forward (no grad) -> bf16 teacher logits; student forward; the student's
lm_head GEMM output goes straight into ONE fused kernel that produces the mimic loss, the LM loss and d(logits) in a single
sweep (no fp32 [N,V] probability tensors -- the reference materialises five of them); when teacher and student hold the
same frozen CLIP tower it runs once per micro-batch instead of twice.
"""
import os
from typing import Any, Dict, Union

import torch

from .. import kernels as K
from ..constants import KD_VOCAB_SIZE
from .trainer_base import AdapterCheckpointMixin, BaseTrainer, image_count_shape
from .trainer_base import quantize_ref_fp8  # noqa: F401  (--ref_fp8's switch, still importable from the trainer that takes it)


class AlignTrainer(AdapterCheckpointMixin, BaseTrainer):
    def __init__(self, model=None, ref_model=None, args=None, data_collator=None, train_dataset=None, eval_dataset=None,
                 tokenizer=None, label_pad_token_id: int = -100, padding_value: int = 0, beta: float = 0.1,
                 label_smoothing: float = 0, loss_type: str = "sigmoid", moe_loss_enable: bool = False,
                 disable_dropout: bool = True, model_init=None, compute_metrics=None, callbacks=None,
                 optimizers=(None, None), preprocess_logits_for_metrics=None, ref_fp8: bool = False):
        self.label_pad_token_id = label_pad_token_id
        self.padding_value = padding_value
        self.beta = beta
        self.label_smoothing = label_smoothing
        self.loss_type = loss_type
        self.moe_loss_enable = moe_loss_enable
        super().__init__(model=model, args=args, data_collator=data_collator, train_dataset=train_dataset,
                         eval_dataset=eval_dataset, tokenizer=tokenizer, model_init=model_init,
                         compute_metrics=compute_metrics, callbacks=callbacks, optimizers=optimizers,
                         preprocess_logits_for_metrics=preprocess_logits_for_metrics)
        self._init_teacher(ref_model, disable_dropout, ref_fp8)
        self.kd_vocab = KD_VOCAB_SIZE
        self.pipeline_teacher = bool(int(os.environ.get("LLAVAMOD_PIPELINE_TEACHER", "1")))
        # loss head on the batch's supervised rows only (csrc/rows.cu): both lm_head GEMMs, the fused KL+CE kernel and the lm_head
        # backward skip the positions the reference multiplies by zero
        self.compact_head = bool(int(os.environ.get("LLAVAMOD_COMPACT_HEAD", "1")))

    # ---- API-compat pieces (materialising forms, our kernels) ------------------------------------------------
    def _moe_loss_of(self, outputs):
        if getattr(self.args, "moe_enable", False) and self.moe_loss_enable and getattr(outputs, "moe_loss", None) is not None:
            return outputs.moe_loss
        return None

    def get_p(self, model, inputs):
        """align_trainer.py:455-477 -> (softmax(logits[:, :, :151936]) fp32, sft_loss, moe_loss)"""
        outputs = model(**inputs, return_dict=True)
        logits, labels = outputs.logits, outputs.labels
        if logits.shape[:-1] != labels.shape:
            raise ValueError("Logits (batch and sequence length dim) and labels must have the same shape.")
        v = min(self.kd_vocab, logits.shape[-1])
        probs = K.softmax_rows(logits.to(torch.bfloat16), v, log_mode=False)
        return probs, outputs.loss, self._moe_loss_of(outputs)

    def get_logp(self, model, inputs):
        """align_trainer.py:479-501 -> (log_softmax fp32, sft_loss, moe_loss, labels).  Forward-only values; the training
        path is ``compute_loss`` (fused)."""
        outputs = model(**inputs, return_dict=True)
        logits, labels = outputs.logits, outputs.labels
        if logits.shape[:-1] != labels.shape:
            raise ValueError("Logits (batch and sequence length dim) and labels must have the same shape.")
        v = min(self.kd_vocab, logits.shape[-1])
        logprobs = K.softmax_rows(logits.to(torch.bfloat16), v, log_mode=True)
        return logprobs, outputs.loss, self._moe_loss_of(outputs), labels

    def compute_align_loss(self, policy_logprobs, reference_probs, labels):
        """align_trainer.py:503-528 on materialised fp32 tensors."""
        return K.align_loss_dense(policy_logprobs, reference_probs, labels, bool(getattr(self.args, "distill_all_tokens", False)))

    # ---- the hot loop body ---------------------------------------------------------------------------------------
    def _device_images(self, model, images):
        dev = model.device
        return torch.stack([im.to(dev, non_blocking=True) for im in images]) if not torch.is_tensor(images) else images.to(dev)

    @staticmethod
    def _forward_args(inputs, images):
        """Keyword arguments of ``forward_hidden`` for the batch ``inputs`` with ``images`` (host list, device tensor or static buffer)."""
        return dict(input_ids=inputs["input_ids"], labels=inputs["labels"], attention_mask=inputs.get("attention_mask"), images=images)

    def _teacher_forward(self, fwd, tower_feats, plan):
        """Frozen teacher -> bf16 logits (get_p's forward, align_trainer.py:458-461; its softmax lives in the fused kernel).
        -> (logits, (B, T'), rows): with the compact head `rows` = (perm, count) of the supervised rows of the post-splice labels and
        logits[j] belongs to row perm[j]; otherwise rows is None and logits is [B*T', Vt]."""
        ref = self.ref_model.module
        t = ref.forward_hidden(**fwd, tower_features=tower_feats, plan=plan)
        th = t["hidden"]
        h2 = th.reshape(-1, th.shape[-1])
        rows = None
        if self.compact_head and t["labels"] is not None:
            lab = t["labels"]
            rows = K.active_rows(lab.reshape(-1), lab.shape[-1], bool(getattr(self.args, "distill_all_tokens", False)))
            h2 = K.gather_rows(h2, *rows)
        return K.gemm(h2, ref.lm_head.weight, m_dev=rows[1] if rows is not None else None), th.shape[:2], rows

    def compute_loss(self, model, inputs: Dict[str, Union[torch.Tensor, Any]], return_outputs=False):
        assert self.ref_model is not None, "ref model can not be none!"
        ref = self.ref_model.module
        images = inputs.get("images", None)
        fwd = self._forward_args(inputs, images)
        pipe = inputs.get("_pipeline")          # software pipeline across micro-batches (see _graph_static_inputs): teacher logits and tower
        tower_feats = None                      # features of THIS batch were produced during the previous micro-batch
        with torch.no_grad():
            if pipe is not None:
                fwd["images"] = inputs["images"]
                tower_feats = pipe["tower_cur"]
            elif self.share_tower and images is not None:
                fwd["images"] = self._device_images(model, images)
                tower_feats = model.get_image_tower()(fwd["images"].to(model.dtype))
            plan = inputs.get("splice_plan")
            if plan is None and images is not None and model.get_image_tower() is not None and \
                    model.get_image_tower().num_patches == ref.get_image_tower().num_patches:
                plan = model.make_splice_plan(fwd["input_ids"], fwd["attention_mask"], fwd["labels"])     # one host plan for both models
        # The frozen teacher forward is independent of the student until the loss: it runs on a side stream so the student's small
        # kernels (H=1024: launch/tail bound) fill the gaps of the teacher's machine-filling GEMMs (a fork/join inside the CUDA graph).
        # Pipelined form: the side stream computes the teacher for the NEXT micro-batch while the main stream runs the student's
        # forward, the loss and the backward of THIS one against teacher logits produced one micro-batch earlier.
        with self._teacher_side():
            if pipe is not None:
                nxt = pipe["next"]
                tower_next = model.get_image_tower()(nxt["images"].to(model.dtype))
                t_next, _, rows_next = self._teacher_forward(self._forward_args(nxt, nxt["images"]), tower_next, nxt["splice_plan"])
                t_logits, t_shape, rows = pipe["t_cur"], pipe["t_shape"], pipe["rows_cur"]
            else:
                with K.nvtx("teacher_forward"):
                    t_logits, t_shape, rows = self._teacher_forward(fwd, tower_feats, plan)
        with K.nvtx("student_forward"):
            s = model.forward_hidden(**fwd, tower_features=tower_feats, moe_noise=inputs.get("moe_noise"), plan=plan)
        if pipe is None:
            self._join_teacher(t_logits, *(rows or ()))
        labels = s["labels"]
        if s["hidden"].shape[:2] != labels.shape or tuple(t_shape) != tuple(labels.shape):
            raise ValueError("Logits (batch and sequence length dim) and labels must have the same shape.")
        vocab = min(self.kd_vocab, model.config.vocab_size, t_logits.shape[-1])
        w_ce = 0.0 if self.loss_type == "only_kd" else 1.0
        with K.nvtx("loss_head"):
            total, align_loss, ce = K.distill_head(s["hidden"], model.lm_head.weight, t_logits, labels, vocab, 1.0, w_ce,
                                                   bool(getattr(self.args, "distill_all_tokens", False)), model.lm_head_grad, rows=rows)
        model_moe_loss = model.moe_loss_from(s["l_aux"]) if getattr(model, "is_moe", False) else None
        # model.loss = CE (+ moe_loss)   llava_qwen1_5_moe.py:421,434
        policy_sft_loss = ce if model_moe_loss is None else ce + model_moe_loss.detach()
        losses = total
        if w_ce != 0.0 and model_moe_loss is not None:
            losses = losses + model_moe_loss                       # the moe_loss already inside the model's loss
        policy_moe_loss = model_moe_loss if (getattr(self.args, "moe_enable", False) and self.moe_loss_enable) else None
        if policy_moe_loss is not None:                             # `if policy_moe_loss:` -- l_aux > 0 always; no host sync here
            moe_loss = policy_moe_loss
            losses = losses + moe_loss                              # ... and counted again by the trainer (align_trainer.py:575-577)
        else:
            moe_loss = torch.full_like(align_loss, -1.0)
        outputs = {"loss": losses.detach().mean(), "loss/align": align_loss.detach().mean(),
                   "loss/moe_balance": moe_loss.detach().mean(), "loss/lm": policy_sft_loss.detach().mean()}
        self.store_metrics(outputs, train_eval="train")
        if pipe is not None:
            pipe["t_next"], pipe["tower_next"], pipe["rows_next"] = t_next, tower_next, rows_next   # -> "current" buffers after the backward
        if return_outputs:
            return losses.mean(), outputs
        return losses.mean()

    # ---- CUDA-graph plumbing (see BaseTrainer._graphed_micro_batch) -------------------------------------------------
    def _graph_signature(self, inputs, next_inputs=None):
        images = inputs.get("images")
        if images is None:
            return None
        noise = inputs.get("moe_noise")
        ids = inputs["input_ids"]
        plan = inputs.get("splice_plan")
        if plan is None:
            plan = self.model.make_splice_plan(ids, inputs.get("attention_mask"), inputs["labels"])
            inputs["splice_plan"] = plan
        if not self.share_tower or not plan["all_true"]:
            return None                   # padded batches take the masked-attention path eagerly
        n_img, ish = image_count_shape(images)
        sig = ("align", tuple(ids.shape), tuple(plan["src"].shape), n_img, ish, plan["has_mask"], plan["has_labels"], self.loss_type,
               tuple(tuple(t.shape) for t in noise) if noise is not None else None, self._grad_ckpt_key())
        if next_inputs is not None and self.overlap_teacher and self.pipeline_teacher:
            nsig = self._graph_signature(next_inputs)
            if nsig == sig:
                return sig + ("pipelined",)
        return sig

    def _graph_static_inputs(self, inputs, static, next_inputs=None, pipelined=False):
        if static is None:
            static = self._new_static(inputs)
            if pipelined:
                nxt = self._new_static(next_inputs)
                # teacher logits / tower features of the CURRENT batch: filled by the prologue (eager) or by the previous replay
                with torch.no_grad():
                    self._fill_static(nxt, inputs)
                    tower = self.model.get_image_tower()(nxt["images"].to(self.model.dtype))
                    t_cur, t_shape, rows_cur = self._teacher_forward(self._forward_args(inputs, nxt["images"]), tower, nxt["splice_plan"])
                static["_pipeline"] = dict(next=nxt, t_cur=t_cur.clone(), tower_cur=tower.clone(), t_shape=tuple(t_shape), holds=inputs,
                                           rows_cur=tuple(r.clone() for r in rows_cur) if rows_cur is not None else None)
        self._fill_static(static, inputs)
        if pipelined:
            pipe = static["_pipeline"]
            if pipe["holds"] is not inputs:       # the "current" buffers do not belong to this batch (first call / caller skipped ahead)
                with torch.no_grad():
                    tower = self.model.get_image_tower()(static["images"].to(self.model.dtype))
                    t_cur, _, rows_cur = self._teacher_forward(self._forward_args(inputs, static["images"]), tower, static["splice_plan"])
                    pipe["t_cur"].copy_(t_cur)
                    if rows_cur is not None:
                        for dst, src in zip(pipe["rows_cur"], rows_cur):
                            dst.copy_(src)
                    pipe["tower_cur"].copy_(tower)
            self._fill_static(pipe["next"], next_inputs)
            pipe["holds"] = next_inputs           # after this replay the "current" buffers describe next_inputs
        return static

    def _graph_epilogue(self, static):
        """Captured at the end of the graph: hand the side stream's results (teacher logits / tower features of the next batch) over."""
        pipe = static.get("_pipeline")
        if pipe is not None:
            main = torch.cuda.current_stream()
            main.wait_stream(self._teacher_stream)
            if pipe.get("rows_cur") is not None:
                # hand over only the supervised rows of the next batch's teacher logits (+ their index list), not the whole [N, Vt] buffer
                K.gather_rows(pipe["t_next"], None, pipe["rows_next"][1], out=pipe["t_cur"])
                for dst, src in zip(pipe["rows_cur"], pipe["rows_next"]):
                    dst.copy_(src)
            else:
                pipe["t_cur"].copy_(pipe["t_next"])
            pipe["tower_cur"].copy_(pipe["tower_next"])
