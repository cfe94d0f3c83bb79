"""High-entropy token masking for GRPO (Wang et al. 2025, "Beyond the 80/20 Rule"; TRL's top_entropy_quantile = rho),
restated in eager ATen ops on top of the token-level port (tests/ppo_objective_port.py, tests/kl_objective_port.py)
and GSPO's (tests/gspo_port.py).  ops.entropy_quantile_threshold and aa_grpo_loss_topent are held to it.

    thr  = torch.quantile(H[counted], 1 - rho)             over every rank's counted tokens; N == 0: keep nothing
    keep = counted & (H >= thr)
    per-token loss = -(s * keep - beta * KL)                s: the clipped (or GSPO) objective, KL: unmasked

The denominators of the aggregation stay the completion-mask counts, and GSPO's ratio averages every counted token."""
from __future__ import annotations

import torch

from gspo_port import sequence_log_weights
from kl_objective_port import kl_estimate
from ppo_objective_port import objective_terms


def quantile_threshold(values: torch.Tensor, q: float) -> torch.Tensor:
    """torch.quantile(values, q) (linear) restated over a sort, also past the 2^24 values torch.quantile accepts:
    rank = fp32 q * (N - 1) (capped at N - 1), lo = floor(rank), hi = ceil(rank), lerp(v_lo, v_hi, rank - lo).
    fp32 0-dim; NaN for no value or any NaN."""
    v = values.reshape(-1).float()
    n = v.numel()
    if n == 0 or bool(torch.isnan(v).any()):
        return torch.tensor(float('nan'), device=v.device)
    srt = torch.sort(v).values
    rank = torch.tensor(q, dtype=torch.float32, device=v.device) * (n - 1)
    lo = rank.long().clamp(max=n - 1)
    hi = rank.ceil().long().clamp(max=n - 1)
    return torch.lerp(srt[lo], srt[hi], rank - lo)


def entropy_keep(entropy: torch.Tensor, mask: torch.Tensor, rho: float, thr=None) -> torch.Tensor:
    """keep (bool (B, K)): the counted tokens (mask) whose entropy is >= the threshold at q = 1 - rho (thr: given, e.g.
    the one over every rank)."""
    counted = mask.bool()
    if thr is None:
        thr = quantile_threshold(entropy[counted], 1.0 - rho)
    return counted & (entropy >= thr)


def grpo_loss(per_token_logps, ref_per_token_logps, advantages, mask, beta: float, keep, old_per_token_logps=None,
              clip_low: float = 0.2, clip_high: float = 0.2, dual_clip=None, agg: str = 'token-mean',
              estimator: str = 'k3', sequence: bool = False):
    """GRPO's clipped objective (sequence: GSPO's one ratio per row, which needs old_per_token_logps) under the
    top-entropy mask `keep` (bool (B, K)).  old_per_token_logps None: the log-probs themselves, detached (ratio 1).
    The KL is created before the ratio, as TRL and the reference create it."""
    K = per_token_logps.size(1)
    per_token_kl = kl_estimate(per_token_logps, ref_per_token_logps, estimator)
    old = per_token_logps.detach() if old_per_token_logps is None else old_per_token_logps
    if sequence:
        w = torch.exp(sequence_log_weights(per_token_logps, old, mask)).unsqueeze(-1)
        s = torch.minimum(advantages * w, advantages * torch.clamp(w, 1.0 - clip_low, 1.0 + clip_high))
        if dual_clip is not None:
            s = torch.where(advantages < 0, torch.maximum(s, dual_clip * advantages), s)
    else:
        s, _, _, _ = objective_terms(per_token_logps, old, advantages.expand(-1, K), clip_low, clip_high, dual_clip)
    per_token_loss = -(s * keep - beta * per_token_kl)
    m = mask.to(per_token_loss.dtype)
    if agg == 'token-mean':
        return (per_token_loss * m).sum() / m.sum()
    if agg == 'seq-mean-token-mean':
        return ((per_token_loss * m).sum(-1) / m.sum(-1)).mean()
    if agg == 'seq-mean-token-sum-norm':
        return (per_token_loss * m).sum() / (per_token_loss.size(0) * K)
    raise ValueError(agg)
