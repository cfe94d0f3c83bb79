"""ORPO loss on the H100 kernels -- mirror of align_anything/trainers/text_to_text/orpo.py
(ORPOTrainer.loss :41-113, .train_step :115-146).  Reads self.cfgs.train_cfgs.scale_coeff."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from ._sliced_pairs import SlicedPairTrainer, div_by_length

__all__ = ['ORPOTrainer']


class ORPOTrainer(SlicedPairTrainer):
    def loss(self, batch) -> dict[str, torch.Tensor]:
        sequence_log_probs = self.compute_log_probs(self.model.module, batch)
        _, [(better_sum, worse_sum)], better_len, worse_len = self._pair_terms(batch, sequence_log_probs)
        beta = self.cfgs.train_cfgs.scale_coeff
        better_log_ratio = div_by_length(better_sum, better_len)  # orpo.py:80
        worse_log_ratio = div_by_length(worse_sum, worse_len)
        log_odds = (better_log_ratio - worse_log_ratio) - (  # orpo.py:82-85
            torch.log1p(-torch.exp(better_log_ratio)) - torch.log1p(-torch.exp(worse_log_ratio))
        )
        odds_ratio_loss = -F.logsigmoid(log_odds)
        sft_loss = -better_log_ratio
        losses = sft_loss + beta * odds_ratio_loss  # orpo.py:88-92
        return self._pack(losses, beta * better_log_ratio.detach(), beta * worse_log_ratio.detach())
