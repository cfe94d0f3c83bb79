"""CISPO (MiniMax-M1, 2025) and SAPO (Qwen's Soft Adaptive Policy Optimization, 2025; TRL's GRPO loss_type 'cispo' /
'sapo') restated in eager ATen ops in the tensors' dtypes: the specification of the AA_PM_* entry points (K5's
aa_ppo_actor_loss_pm, aa_grpo_loss_pm and K1f's aa_logprob_*_fused_pm).

s is the negated per-token loss term that the aggregation takes exactly as it takes the clipped objective's:
    cispo   w = clamp(ratio, max = hi).detach() ;  s = w * adv * lp           (hi = 1 + eps_high in the log-prob dtype)
    sapo    tau = where(adv > 0, tau_pos, tau_neg) (fp32) ;  s = sigmoid(tau * (ratio - 1)) * 4 / tau * adv
with ratio = exp(lp - old).  The kernels round where these ops round (FAITHFUL) and nowhere in F32 mode."""
from __future__ import annotations

import torch

from ppo_objective_port import masked_mean

DEFAULT_TAU = (1.0, 1.05)


def policy_terms(mode: str, lp, old, adv, eps_high: float = 0.2, tau_pos: float = 1.0, tau_neg: float = 1.05):
    """-> (s, over): the per-token objective and CISPO's truncation indicator (all False under SAPO)."""
    ratio = torch.exp(lp - old)
    if mode == 'cispo':
        hi = torch.tensor(1.0 + eps_high, dtype=torch.float64).to(lp.dtype).item()  # rounded as clamp rounds it
        w = torch.clamp(ratio, max=hi).detach()
        return w * adv * lp, (ratio > hi).detach()
    if mode != 'sapo':
        raise ValueError(mode)
    tau = torch.where(adv > 0, tau_pos, tau_neg)  # fp32, whatever adv's dtype
    s = torch.sigmoid(tau * (ratio - 1)) * 4 / tau * adv
    return s, torch.zeros_like(ratio, dtype=torch.bool)


def aggregate(s, mask, agg: str):
    """The actor's and GRPO's aggregations of s (the loss is the negation, applied by the callers)."""
    m = mask.to(s.dtype)
    if agg == 'seq-mean-token-mean':
        return masked_mean(s, mask)
    if agg == 'token-mean':
        return (s * m).sum() / m.sum()
    if agg == 'seq-mean-token-sum-norm':
        return (s * m).sum() / (s.size(0) * s.size(1))
    raise ValueError(agg)


def actor_loss(mode, lp, old, adv, mask, agg='seq-mean-token-mean', eps_high=0.2, tau_pos=1.0, tau_neg=1.05):
    """The PPO actor loss under CISPO / SAPO: -agg(s)."""
    s, _ = policy_terms(mode, lp, old, adv, eps_high, tau_pos, tau_neg)
    return -aggregate(s, mask, agg)


def actor_loss_kl(mode, lp, old, adv, mask, agg, eps_high, tau_pos, tau_neg, ref, kl_coeff: float, estimator: str):
    """-> (loss, agg(KL), loss + kl_coeff * agg(KL)).  The KL is created before the ratio (kl_loss_port's order)."""
    from kl_loss_port import kl_loss

    kl = kl_loss(lp, ref, mask, estimator, agg)
    loss = actor_loss(mode, lp, old, adv, mask, agg, eps_high, tau_pos, tau_neg)
    return loss, kl, loss + kl_coeff * kl


def clip_fraction(mode, lp, old, adv, mask, agg='seq-mean-token-mean', eps_high=0.2) -> float:
    """train/actor_clip_fraction in float64: the share of counted tokens with ratio > 1 + eps_high under CISPO,
    aggregated like the loss (per-row shares averaged under seq-mean-token-mean); 0 under SAPO."""
    _, over = policy_terms(mode, lp, old, adv, eps_high)
    m = mask.bool()
    o = (over & m).double()
    if agg == 'seq-mean-token-mean':
        return float((o.sum(-1) / m.double().sum(-1)).mean())
    return float(o.sum() / m.double().sum())


def grpo_loss(mode, lp, ref, old, adv, mask, beta: float, agg='token-mean', eps_high=0.2, tau_pos=1.0, tau_neg=1.05,
              estimator='k3'):
    """GRPO under CISPO / SAPO: per-token loss -(s - beta * KL), the KL created before s; adv (B,) or (B, 1) fp32, old
    None: the log-probs themselves, detached (ratio 1)."""
    from kl_objective_port import kl_estimate

    old = lp.detach() if old is None else old
    kl = kl_estimate(lp, ref, estimator)
    s, _ = policy_terms(mode, lp, old, adv.reshape(-1, 1).expand(-1, lp.size(1)), eps_high, tau_pos, tau_neg)
    ptl = -(s - beta * kl)
    m = mask.to(ptl.dtype)
    if agg == 'token-mean':
        return (ptl * m).sum() / m.sum()
    if agg == 'seq-mean-token-mean':
        return ((ptl * m).sum(-1) / m.sum(-1)).mean()
    return (ptl * m).sum() / (ptl.size(0) * ptl.size(1))
