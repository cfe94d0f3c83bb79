"""The KL term in the PPO actor loss, restated in the reference's own style: eager ATen ops in the tensors' dtypes.

    total = actor_loss + kl_loss_coeff * agg(KL(lp, ref), mask)

actor_loss is ppo_objective_port.actor_loss, KL kl_objective_port.kl_estimate and agg the objective's aggregation over
the same mask.  The KL is created before the ratio term, so autograd adds its gradient to lp after the ratio's, the
order kl_grad (csrc/ppo_math.cuh) adds them in.  K5 and K1f's actor node with the KL term are held to it."""
from __future__ import annotations

import torch

from kl_objective_port import kl_estimate
from ppo_objective_port import actor_loss as clipped_loss
from ppo_objective_port import masked_mean


def aggregate(x, mask, agg: str = 'seq-mean-token-mean'):
    """The actor objective's aggregation of a per-token term (without the objective's sign)."""
    if agg == 'seq-mean-token-mean':
        return masked_mean(x, mask)
    return (x * mask).sum() / mask.sum()


def kl_loss(log_probs, ref_log_probs, mask, estimator: str, agg: str = 'seq-mean-token-mean'):
    """agg(KL): train/actor_kl_loss, the term without its coefficient."""
    return aggregate(kl_estimate(log_probs, ref_log_probs, estimator), mask, agg)


def actor_loss(log_probs, old_log_probs, advantages, mask, clip_low: float, clip_high: float, dual_clip=None,
               agg: str = 'seq-mean-token-mean', ref_log_probs=None, kl_loss_coeff: float = 0.0,
               estimator: str = 'k3'):
    """-> the total loss.  With kl_loss_coeff 0 this is ppo_objective_port.actor_loss, bit for bit."""
    if kl_loss_coeff == 0.0:
        return clipped_loss(log_probs, old_log_probs, advantages, mask, clip_low, clip_high, dual_clip, agg)
    kl = kl_estimate(log_probs, ref_log_probs, estimator)  # before the ratio
    loss = clipped_loss(log_probs, old_log_probs, advantages, mask, clip_low, clip_high, dual_clip, agg)
    return loss + kl_loss_coeff * aggregate(kl, mask, agg)
