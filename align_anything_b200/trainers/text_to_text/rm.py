"""Reward-model training loss / step on the H100 kernels -- mirror of
align_anything/trainers/text_to_text/rm.py (RMTrainer.loss :97-132, .train_step :133-152).  The model
forward goes through the K3 score head (models.reward_model); the pairwise log-sigmoid loss, its
regularisation term, the accuracy and the gradient w.r.t. the end scores come from one launch."""
from __future__ import annotations

from typing import Any

import torch

from ... import ops
from ...utils.multi_process import all_reduce_packed

__all__ = ['RMTrainer']


class RMTrainer:
    def __init__(self, cfgs, model, tokenizer=None, infer_batch=None) -> None:
        self.cfgs = cfgs
        self.model = model
        self.tokenizer = tokenizer
        self.infer_batch = infer_batch or (lambda batch: {k: v for k, v in batch.items() if k != 'meta_info'})

    def loss(self, batch) -> dict[str, torch.Tensor]:
        """trainers/text_to_text/rm.py:97-132."""
        n = batch['input_ids'].size(0)
        assert n % 2 == 0, 'batch size mismatch!'
        output = self.model(**self.infer_batch(batch))
        higher_rewards, lower_rewards = output.scores.squeeze(dim=-1).chunk(chunks=2, dim=0)
        reg = float(getattr(self.cfgs.train_cfgs, 'regularization', 0.0) or 0.0)
        res = ops.rm_pair_loss(output.end_scores, reg)
        return {
            'loss': res['loss'], 'higher_end_reward': res['higher_end_reward'], 'lower_end_reward': res['lower_end_reward'],
            'higher_rewards': higher_rewards, 'lower_rewards': lower_rewards, 'accuracy': res['accuracy'],
            '_stats': res['_stats'],
        }

    def train_step(self, batch) -> dict[str, Any]:
        """trainers/text_to_text/rm.py:133-152: ONE packed collective + ONE sync (reference: 2 + 2)."""
        loss_dict = self.loss(batch)
        self.model.backward(loss_dict['loss'])
        self.model.step()
        with torch.no_grad():
            stats = torch.cat([loss_dict['_stats'], ops.status_lane(loss_dict['_stats'].device)])
            loss, acc, status = all_reduce_packed(stats, max_lanes=(2,)).tolist()  # lane 2 = device status word
        ops.raise_for_status(status, stats.device)
        return {'train/loss': loss, 'train/accuracy': acc, 'train/lr': self.model.optimizer.param_groups[0]['lr']}
