"""DPO loss / step on the H100 kernels -- mirror of align_anything/trainers/text_to_text/dpo.py
(DPOTrainer.compute_log_probs :122-142, .loss :144-203, .train_step :205-237).

The methods read exactly what the reference's methods read from `self`:
    self.model.module, self.reference_model.module   (engine-wrapped HF models: `.logits`)
    self.infer_batch, self.tokenizer.pad_token_id, self.cfgs.train_cfgs.scale_coeff
    self.model.backward(loss), self.model.step(), self.model.optimizer.param_groups
so they can be bound onto the reference class unchanged (align_anything_b200.patch).
"""
from __future__ import annotations

from typing import Any

import torch

from ... import ops
from ...utils.multi_process import all_reduce_packed, fused_allreduce

__all__ = ['DPOTrainer', 'strip_pad']

METRIC_KEYS = ('train/loss', 'train/reward', 'train/better_sample_reward', 'train/worse_sample_reward',
               'train/reward_accuracy', 'train/reward_margin')


def strip_pad(seq: torch.Tensor, pad_token_id: int):
    """trainers/text_to_text/dpo.py:52-54 (kept for API parity; see ops.strip_pad_tail)."""
    return seq[seq != pad_token_id]


class DPOTrainer:
    """Hot-path half of the reference DPOTrainer.  `strip_pad_tokens` / `skip_identical_pairs` select
    the text+image (strip, keep all pairs) or audio (no strip, drop identical pairs) behaviour."""

    strip_pad_tokens = True  # trainers/text_to_text/dpo.py:135 ; False: text_audio_to_text/dpo.py:100
    skip_identical_pairs = False  # True: text_audio_to_text/dpo.py:138-139
    mode = None  # None -> 'faithful' (reference rounding); 'f32' for fp32 outputs
    # Opt-in (SURVEY.md 8f rank 1, first step): never build the (2B, L, V) logits tile.  The model is asked for its
    # last hidden states (`output_hidden_states=True, logits_to_keep=1`: the lm_head runs on one position only) and
    # the scored rows go through ops.sequence_log_probs_from_hidden (chunked lm_head GEMM + K1 / K1b).
    fused_lm_head = False
    lm_head_chunk_rows = None

    def __init__(self, cfgs, model, reference_model, tokenizer, infer_batch=None) -> None:
        self.cfgs = cfgs
        self.model = model
        self.reference_model = reference_model
        self.tokenizer = tokenizer
        self.infer_batch = infer_batch or (lambda batch: {k: v for k, v in batch.items() if k != 'meta_info'})
        self.global_step = 0

    # -- trainers/text_to_text/dpo.py:122-142 --------------------------------------------------
    def _hidden_and_head(self, model, batch):
        out = model(**self.infer_batch(batch), output_hidden_states=True, logits_to_keep=1)
        return out.hidden_states[-1], ops.lm_head_weight(model)

    def compute_log_probs(self, model, batch) -> torch.Tensor:
        """(2B, max(R)-1) response log-probs, right-padded with 0: one K1 launch for all samples."""
        if self.fused_lm_head:
            hidden, weight = self._hidden_and_head(model, batch)
            return ops.sequence_log_probs_from_hidden(
                hidden, weight, batch['input_ids'], batch['meta_info']['response_lens'], self.tokenizer.pad_token_id,
                strip=self.strip_pad_tokens, chunk_rows=self.lm_head_chunk_rows, mode=self.mode)
        logits = model(**self.infer_batch(batch)).logits
        return ops.sequence_log_probs(
            logits, batch['input_ids'], batch['meta_info']['response_lens'], self.tokenizer.pad_token_id,
            strip=self.strip_pad_tokens, mode=self.mode,
        )

    # -- trainers/text_to_text/dpo.py:144-203 --------------------------------------------------
    def loss(self, batch) -> dict[str, torch.Tensor]:
        if self.fused_lm_head:
            policy_lp = self.compute_log_probs(self.model.module, batch)
            with torch.no_grad():
                ref_lp = self.compute_log_probs(self.reference_model.module, batch)
            return ops.dpo_loss_from_log_probs(policy_lp, ref_lp, float(self.cfgs.train_cfgs.scale_coeff), batch['input_ids'],
                                               skip_identical_pairs=self.skip_identical_pairs, mode=self.mode)
        policy_logits = self.model.module(**self.infer_batch(batch)).logits
        with torch.no_grad():
            ref_logits = self.reference_model.module(**self.infer_batch(batch)).logits
        out = ops.dpo_fused_loss(
            policy_logits, ref_logits, batch['input_ids'], batch['meta_info']['response_lens'],
            self.tokenizer.pad_token_id, float(self.cfgs.train_cfgs.scale_coeff),
            strip=self.strip_pad_tokens, skip_identical_pairs=self.skip_identical_pairs, mode=self.mode)
        # inside train_step on several GPUs the packed metrics are all-reduced over NVLink peer memory by a one-warp
        # kernel on a side stream, launched HERE so that its wait for the slowest rank overlaps the backward (K1b);
        # every rank runs the same number of steps; a bare loss() call never enters a collective
        fused = fused_allreduce(policy_logits.device) if getattr(self, '_in_train_step', False) else None
        if fused is not None:
            out['_stats_pending'] = fused.all_reduce_async(out['_stats'], max_lanes=(7,))  # lane 7 = status word: MAX
        return out

    # -- trainers/text_to_text/dpo.py:205-237 --------------------------------------------------
    def train_step(self, batch) -> dict[str, Any]:
        self._in_train_step = True
        try:
            loss_dict = self.loss(batch=batch)
        finally:
            self._in_train_step = False
        self.model.backward(loss_dict['loss'])
        self.model.step()
        with torch.no_grad():
            if '_stats_pending' in loss_dict:  # reduced over NVLink on the side stream while K1b ran
                stats = loss_dict['_stats_pending'].wait()
            else:
                stats = all_reduce_packed(loss_dict['_stats'].clone(), max_lanes=(7,))  # ONE collective (reference: 6)
            values = stats.tolist()  # ONE host sync (reference: 7 .item())
        # lane 7 carries the device status word (label out of range, short sequence ...): the reference raises eagerly
        # at those points, we raise here -- same exception class, no extra sync, every rank together
        ops.raise_for_status(values[7], stats.device)
        out = dict(zip(METRIC_KEYS, values[:6]))
        out['train/lr'] = self.model.optimizer.param_groups[0]['lr']
        return out
