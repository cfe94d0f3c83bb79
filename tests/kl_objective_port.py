"""The KL regularisation options, restated in the reference's own style: eager ATen ops in the tensors' dtypes.  With
every option at its default this is the reference's arithmetic op for op: the k1 reward penalty of
add_kl_divergence_regularization (trainers/text_to_text/ppo.py:528-547) and the k3 KL of GRPO's per-token loss
(trainers/text_to_text/grpo.py:290-312).  The kernels (K4, aa_grpo_loss_kl and K1f's GRPO node) are held to it."""
from __future__ import annotations

import torch

from grpo_objective_port import is_reference
from ppo_objective_port import objective_terms


def kl_estimate(log_probs, ref_log_probs, estimator: str):
    """k1 lp - ref ; k2 0.5 * (lp - ref) ** 2 ; k3 exp(ref - lp) - (ref - lp) - 1 (the reference GRPO's expression)."""
    if estimator == 'k1':
        return log_probs - ref_log_probs
    if estimator == 'k2':
        return 0.5 * (log_probs - ref_log_probs) ** 2
    if estimator == 'k3':
        return torch.exp(ref_log_probs - log_probs) - (ref_log_probs - log_probs) - 1
    raise ValueError(estimator)


def kl_rewards(reward, log_probs, ref_log_probs, sequence_mask, kl_coeff: float, clip_range_score: float,
               estimator: str = 'k1'):
    """add_kl_divergence_regularization with the penalty formed from `estimator`."""
    end_index = torch.cat([m.nonzero()[-1] for m in sequence_mask])
    kl_penalty_rewards = -kl_coeff * kl_estimate(log_probs, ref_log_probs, estimator)
    rewards = torch.scatter_add(kl_penalty_rewards, dim=-1, index=end_index.unsqueeze(dim=-1),
                                src=reward.to(kl_penalty_rewards.dtype).unsqueeze(dim=-1))
    return torch.clamp(rewards, min=-clip_range_score, max=clip_range_score)


def kl_divergence_metric(log_probs, ref_log_probs, sequence_mask, start: int = 0) -> float:
    """train/kl_divergence under every estimator: the k1 sum over each row's response, averaged over rows (float64)."""
    d = (log_probs.double() - ref_log_probs.double())[:, start:] * sequence_mask[:, start:]
    return float(d.sum(-1).mean())


def grpo_loss(per_token_logps, ref_per_token_logps, advantages, mask, beta: float, estimator: str = 'k3',
              old_per_token_logps=None, clip_low=None, clip_high=None, dual_clip=None, agg: str = 'token-mean',
              clip: float = 0.2):
    """grpo_objective_port.grpo_loss with the per-token KL taken by `estimator` (created before the ratio term, as the
    reference creates its KL).  Every option at its default: the reference's loss; otherwise the clipped objective."""
    K = per_token_logps.size(1)
    per_token_kl = kl_estimate(per_token_logps, ref_per_token_logps, estimator)
    advantages_expanded = advantages.expand(-1, K)
    if is_reference(old_per_token_logps, clip_low, clip_high, dual_clip, agg) and estimator == 'k3':
        s = torch.exp(per_token_logps - per_token_logps.detach()) * advantages_expanded
    else:
        old = per_token_logps.detach() if old_per_token_logps is None else old_per_token_logps
        lo = clip if clip_low is None else clip_low
        hi = clip if clip_high is None else clip_high
        s, _, _, _ = objective_terms(per_token_logps, old, advantages_expanded, lo, hi, dual_clip)
    per_token_loss = -(s - beta * per_token_kl)
    m = mask.to(per_token_loss.dtype)
    if agg == 'token-mean':
        return (per_token_loss * m).sum() / m.sum()
    if agg == 'seq-mean-token-mean':
        return ((per_token_loss * m).sum(-1) / m.sum(-1)).mean()
    if agg == 'seq-mean-token-sum-norm':
        return (per_token_loss * m).sum() / (per_token_loss.size(0) * K)
    raise ValueError(agg)


def adaptive_kl_coeffs(kl_coeff: float, kls, n: int, target: float, horizon: float) -> list[float]:
    """The coefficient each step uses under the adaptive controller (Ziegler et al. 2019): after a step with KL `kl`,
    e = clip(kl / target - 1, -0.2, 0.2) and kl_coeff <- kl_coeff * (1 + e * n / horizon)."""
    out = []
    for kl in kls:
        out.append(kl_coeff)
        e = min(max(kl / target - 1.0, -0.2), 0.2)
        kl_coeff = kl_coeff * (1.0 + e * n / horizon)
    return out
