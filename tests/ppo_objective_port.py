"""The PPO actor objective with clip-higher, dual-clip and token-mean aggregation, restated in the reference's own style:
eager ATen ops in the tensors' dtypes (trainers/text_to_text/ppo.py:291-307 + utils/tools.py:460-467).  With every
option at its default this is the reference's actor_loss_fn, op for op.  The kernels (K5 and K1f) are held to it."""
from __future__ import annotations

import torch


def masked_mean(x: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """utils/tools.py:460-467."""
    return ((x * mask).sum(dim=-1) / mask.sum(dim=-1)).mean()


def objective_terms(log_probs, old_log_probs, advantages, clip_low: float, clip_high: float, dual_clip=None):
    """-> (s, s1, s2, dual_wins): the per-token objective and the pieces the clip fractions count."""
    ratios = torch.exp(log_probs - old_log_probs)
    s1 = advantages * ratios
    s2 = advantages * torch.clamp(ratios, 1.0 - clip_low, 1.0 + clip_high)
    s = torch.minimum(s1, s2)
    dual_wins = torch.zeros_like(s, dtype=torch.bool)
    if dual_clip is not None:
        ca = dual_clip * advantages
        dual_wins = (advantages < 0) & (s < ca)
        s = torch.where(advantages < 0, torch.maximum(s, ca), s)
    return s, s1, s2, dual_wins


def actor_loss(log_probs, old_log_probs, advantages, mask, clip_low: float, clip_high: float, dual_clip=None,
               agg: str = 'seq-mean-token-mean'):
    s, _, _, _ = objective_terms(log_probs, old_log_probs, advantages, clip_low, clip_high, dual_clip)
    if agg == 'seq-mean-token-mean':
        return -masked_mean(s, mask)
    return -(s * mask).sum() / mask.sum()


def clip_fractions(log_probs, old_log_probs, advantages, mask, clip_low: float, clip_high: float, dual_clip=None,
                   agg: str = 'seq-mean-token-mean') -> tuple[float, float]:
    """(clipped fraction, dual-clip fraction) in float64, aggregated like the loss: the masked mean of the indicator
    `s2 < s1`, and the ratio of the masked means of `c * A wins` and `A < 0` (0 without a negative advantage)."""
    _, s1, s2, dual_wins = objective_terms(log_probs, old_log_probs, advantages, clip_low, clip_high, dual_clip)
    m = mask.bool()
    clipped = ((s2 < s1) & m).double()
    dual = (dual_wins & m).double()
    neg = ((advantages < 0) & m).double()
    if agg == 'seq-mean-token-mean':
        cnt = m.double().sum(-1)
        fc = (clipped.sum(-1) / cnt).mean()
        fd, fn = (dual.sum(-1) / cnt).sum(), (neg.sum(-1) / cnt).sum()
    else:
        fc = clipped.sum() / m.double().sum()
        fd, fn = dual.sum(), neg.sum()
    return float(fc), float(fd / fn) if float(fn) > 0 else 0.0
