"""SFT loss / step on the H100 kernels -- mirror of align_anything/trainers/text_to_text/sft.py
(SupervisedTrainer.loss :95-98, .train_step :100-109).  The reference takes `outputs.loss` from the HF
model, which upcasts the whole logits tile to fp32 and materialises a (rows, V) log-softmax; here the
model is called WITHOUT labels and the cross-entropy comes from K1 + the mean-NLL epilogue
(ops.causal_lm_loss; SURVEY.md section 8f row 4)."""
from __future__ import annotations

from typing import Any

import torch

from ... import ops

__all__ = ['SupervisedTrainer']


class SupervisedTrainer:
    ignore_index = -100

    def __init__(self, cfgs, model, tokenizer=None, infer_batch=None) -> None:
        self.cfgs = cfgs
        self.model = model
        self.tokenizer = tokenizer
        self.infer_batch = infer_batch or (lambda batch: {k: v for k, v in batch.items() if k != 'meta_info'})

    def loss(self, sft_batch) -> dict[str, torch.Tensor]:
        """trainers/text_to_text/sft.py:95-98."""
        batch = dict(self.infer_batch(sft_batch))
        labels = batch.pop('labels')
        logits = self.model(**batch).logits
        return {'loss': ops.causal_lm_loss(logits, labels, self.ignore_index)}

    def train_step(self, sft_batch) -> dict[str, Any]:
        """trainers/text_to_text/sft.py:100-109."""
        loss = self.loss(sft_batch)['loss']
        self.model.backward(loss)
        self.model.step()
        with torch.no_grad():  # the loss and the device status word (out-of-range label ...) in ONE host read
            loss_val, status = torch.cat([loss.detach().float().reshape(1), ops.status_lane(loss.device)]).tolist()
        ops.raise_for_status(status, loss.device)
        return {'train/loss': loss_val, 'train/lr': self.model.optimizer.param_groups[0]['lr']}
