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
    # Opt-in: no (B, L, V) logits tile and no gradient tile.  The model is asked for its last hidden states
    # (`output_hidden_states=True, logits_to_keep=1`: the lm_head runs on one position only) and the loss comes from
    # ops.causal_lm_loss_from_hidden over the rows whose next label is not ignored; the gradient is formed in the forward.
    fused_lm_head = False
    lm_head_chunk_rows = None
    # the class attributes above that the grafted methods read: patch.install() copies them onto the reference's classes
    SWITCHES = ('ignore_index', 'fused_lm_head', 'lm_head_chunk_rows')

    def __init__(self, cfgs, model, tokenizer=None, infer_batch=None) -> None:
        self.cfgs = cfgs
        self.model = model
        self.tokenizer = tokenizer
        self.infer_batch = infer_batch or (lambda batch: {k: v for k, v in batch.items() if k != 'meta_info'})

    def loss(self, sft_batch) -> dict[str, torch.Tensor]:
        """trainers/text_to_text/sft.py:95-98."""
        batch = dict(self.infer_batch(sft_batch))
        labels = batch.pop('labels')
        if self.fused_lm_head:
            # refuse a head the fused path would get wrong, then the valid-row index (the step's first host read: the
            # previous step's read has drained the queue), both before the forward
            weight = ops.lm_head_weight(getattr(self.model, 'module', self.model))
            rows = ops.causal_lm_valid_rows(labels, self.ignore_index)
            out = self.model(**batch, output_hidden_states=True, logits_to_keep=1)
            loss = ops.causal_lm_loss_from_hidden(out.hidden_states[-1], weight, labels, self.ignore_index,
                                                  chunk_rows=self.lm_head_chunk_rows, valid_rows=rows)[0]
            return {'loss': loss}
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
