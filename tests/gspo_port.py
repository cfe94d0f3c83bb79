"""GSPO's sequence-level importance ratio for GRPO (Zheng et al. 2025), restated as TRL writes it for
importance_sampling_level="sequence": eager ATen ops in the tensors' dtypes, on top of the token-level port
(tests/grpo_objective_port.py, tests/kl_objective_port.py).  aa_grpo_loss_seq is held to it.

    log_w = (log_ratio * m).sum(-1) / m.sum(-1).clamp(min=1.0)      (B,)  fp32: the count is fp32
    w     = exp(log_w)                                              (B, 1)
    s     = min(A * w, A * clamp(w, 1 - eps_low, 1 + eps_high))     fp32, dual-clip as at token level

The mask is an integer tensor, so the row sum of the log-ratios rounds once to the log-prob dtype; everything after
it is fp32, even for 16-bit log-probs."""
from __future__ import annotations

import torch

from kl_objective_port import kl_estimate
from ppo_objective_port import clip_fractions as _ppo_clip_fractions


def sequence_log_weights(per_token_logps, old_per_token_logps, mask):
    """log_w (B,): the mean log-ratio of each sequence's counted tokens (mask: an integer (B, K) tensor)."""
    log_ratio = per_token_logps - old_per_token_logps
    return (log_ratio * mask).sum(-1) / mask.sum(-1).clamp(min=1.0)


def grpo_loss(per_token_logps, ref_per_token_logps, advantages, mask, beta: float, old_per_token_logps=None,
              clip_low: float = 0.2, clip_high: float = 0.2, dual_clip=None, agg: str = 'token-mean',
              estimator: str = 'k3'):
    """GRPO's loss with the sequence-level ratio.  advantages (B, 1) fp32; mask (B, K) integer 0 / 1 (the completion
    mask); old_per_token_logps None: the log-probs themselves, detached (w = 1).  The KL is created before the ratio,
    as TRL and the reference create it."""
    K = per_token_logps.size(1)
    per_token_kl = kl_estimate(per_token_logps, ref_per_token_logps, estimator)
    old = per_token_logps.detach() if old_per_token_logps is None else old_per_token_logps
    w = torch.exp(sequence_log_weights(per_token_logps, old, mask)).unsqueeze(-1)
    s = torch.minimum(advantages * w, advantages * torch.clamp(w, 1.0 - clip_low, 1.0 + clip_high))
    if dual_clip is not None:
        s = torch.where(advantages < 0, torch.maximum(s, dual_clip * advantages), s)
    per_token_loss = -(s - beta * per_token_kl)
    m = mask.to(per_token_loss.dtype)
    if agg == 'token-mean':
        return (per_token_loss * m).sum() / m.sum()
    if agg == 'seq-mean-token-mean':
        return ((per_token_loss * m).sum(-1) / m.sum(-1)).mean()
    if agg == 'seq-mean-token-sum-norm':
        return (per_token_loss * m).sum() / (per_token_loss.size(0) * K)
    raise ValueError(agg)


def clip_fractions(per_token_logps, old_per_token_logps, advantages, mask, clip_low: float, clip_high: float,
                   dual_clip=None, agg: str = 'token-mean') -> tuple[float, float]:
    """(clipped fraction, dual-clip fraction) in float64 with the token-level definitions: every counted token of a
    sequence carries the sequence's w, so the counts are of clipped sequences (seq-mean-token-mean) or of the tokens in
    them.  The token-level counter sees w as the ratio exp(log_w - 0)."""
    log_w = sequence_log_weights(per_token_logps, old_per_token_logps, mask)
    x = log_w.unsqueeze(-1).expand(-1, per_token_logps.size(1))
    a = advantages.expand(-1, per_token_logps.size(1))
    return _ppo_clip_fractions(x, torch.zeros_like(x), a, mask.bool(), clip_low, clip_high, dual_clip,
                               'seq-mean-token-mean' if agg == 'seq-mean-token-mean' else 'token-mean')
