"""SimPO loss on the H100 kernels -- mirror of align_anything/trainers/text_to_text/simpo.py
(SimPOTrainer.loss :41-108, .train_step :110-141).  Reads self.cfgs.train_cfgs.{scale_coeff, gamma}."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from ._sliced_pairs import SlicedPairTrainer, div_by_length

__all__ = ['SimPOTrainer']


class SimPOTrainer(SlicedPairTrainer):
    def loss(self, batch) -> dict[str, torch.Tensor]:
        sequence_log_probs = self.compute_log_probs(self.model.module, batch)
        _, [(better_sum, worse_sum)], better_len, worse_len = self._pair_terms(batch, sequence_log_probs)
        beta, gamma = self.cfgs.train_cfgs.scale_coeff, self.cfgs.train_cfgs.gamma
        better_log_ratio = div_by_length(better_sum, better_len)  # simpo.py:80
        worse_log_ratio = div_by_length(worse_sum, worse_len)
        losses = -F.logsigmoid(beta * (better_log_ratio - worse_log_ratio) - gamma)  # simpo.py:82-87
        return self._pack(losses, beta * better_log_ratio.detach(), beta * worse_log_ratio.detach())
