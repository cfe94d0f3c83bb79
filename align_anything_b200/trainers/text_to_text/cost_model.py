"""Cost-model training loss on the H100 kernels -- mirror of align_anything/trainers/text_to_text/cost_model.py
(CMTrainer.loss :95-145; .train_step :147-167 is the RM step), inherited unchanged by
trainers/text_image_to_text/cost_model.py.  The model forward goes through the K3 score head
(models.reward_model); the signed cost terms, the pairwise term, the regularisation, the accuracy and the gradient
w.r.t. the end scores come from one launch."""
from __future__ import annotations

import torch

from ... import ops
from .rm import RMTrainer

__all__ = ['CMTrainer']


class CMTrainer(RMTrainer):
    def __init__(self, cfgs, model, tokenizer=None, infer_batch=None) -> None:
        super().__init__(cfgs, model, tokenizer, infer_batch)
        self.scale_coeff = cfgs.train_cfgs.scale_coeff

    def loss(self, batch) -> dict[str, torch.Tensor]:
        """trainers/text_to_text/cost_model.py:97-144.  The safety signs are read before the forward, so a batch
        without them (the text PreferenceDataset has none) raises the reference's KeyError before any launch."""
        n = batch['input_ids'].size(0)
        assert n % 2 == 0, 'batch size mismatch!'
        better_signs = batch['meta_info']['is_better_safe']
        worse_signs = batch['meta_info']['is_worse_safe']
        output = self.model(**self.infer_batch(batch))
        higher_rewards, lower_rewards = output.scores.squeeze(dim=-1).chunk(chunks=2, dim=0)
        res = ops.cost_pair_loss(output.end_scores, better_signs, worse_signs, self.scale_coeff,
                                 float(self.cfgs.train_cfgs.regularization))
        return {
            'loss': res['loss'], 'higher_end_reward': res['higher_end_reward'], 'lower_end_reward': res['lower_end_reward'],
            'higher_rewards': higher_rewards, 'lower_rewards': lower_rewards, 'accuracy': res['accuracy'],
            '_stats': res['_stats'],
        }
