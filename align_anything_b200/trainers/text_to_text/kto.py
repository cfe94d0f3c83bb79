"""KTO loss on the H100 kernels -- mirror of align_anything/trainers/text_to_text/kto.py
(KTOTrainer.loss :83-159, .train_step :161-192; compute_kl :49-81 calls compute_log_probs, i.e. K1).
Reads self.cfgs.train_cfgs.{scale_coeff, scale_better, scale_worse} and self.kl."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from ._sliced_pairs import SlicedPairTrainer

__all__ = ['KTOTrainer']


class KTOTrainer(SlicedPairTrainer):
    kl = 0.0

    def compute_kl_from_batches(self, batches) -> None:
        """kto.py:70-81 for an iterable of batches (dataset construction stays in the reference)."""
        for batch in batches:
            log_probs = self.compute_log_probs(self.model.module, batch=batch)
            ref_log_probs = self.compute_log_probs(self.reference_model.module, batch=batch)
            kl = (log_probs - ref_log_probs).mean()
            self.kl = max(kl, 0)

    def loss(self, batch) -> dict[str, torch.Tensor]:
        sequence_log_probs = self.compute_log_probs(self.model.module, batch)
        with torch.no_grad():
            ref_sequence_log_probs = self.compute_log_probs(self.reference_model.module, batch)
        _, [(better, worse), (ref_better, ref_worse)], _, _ = self._pair_terms(
            batch, sequence_log_probs, ref_sequence_log_probs)
        cfg = self.cfgs.train_cfgs
        better_log_ratio = better - ref_better  # kto.py:123-124
        worse_log_ratio = worse - ref_worse
        losses = (cfg.scale_better * (1 - F.sigmoid(cfg.scale_coeff * (better_log_ratio - self.kl)))  # kto.py:126-131
                  - cfg.scale_worse * (1 - F.sigmoid(cfg.scale_coeff * (self.kl - worse_log_ratio))))
        return self._pack(losses, cfg.scale_coeff * better_log_ratio.detach(), cfg.scale_coeff * worse_log_ratio.detach())
