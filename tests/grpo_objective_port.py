"""GRPO's objective with several updates per rollout, clip-higher, dual-clip and the three aggregations, restated in the
reference's own style: eager ATen ops in the tensors' dtypes (trainers/text_to_text/grpo.py:268-312).  With every
option at its default this is the reference's train_step arithmetic, op for op.  The kernels (aa_grpo_loss_obj and
K1f's GRPO node) are held to it."""
from __future__ import annotations

import torch

from ppo_objective_port import clip_fractions as _ppo_clip_fractions
from ppo_objective_port import objective_terms


def completion_mask(completion_tokens: torch.Tensor, eos_token_id: int) -> torch.Tensor:
    """trainers/text_to_text/grpo.py:300-307: ones up to and including the first eos of each row."""
    mask = torch.ones_like(completion_tokens)
    for i in range(completion_tokens.size(0)):
        eos = (completion_tokens[i] == eos_token_id).nonzero(as_tuple=False)
        if eos.numel() > 0:
            mask[i, eos[0].item() + 1:] = 0
    return mask


def group_advantages(rewards: torch.Tensor, num_generations: int, scale: bool = True) -> torch.Tensor:
    """grpo.py:268-274; scale=False (Dr. GRPO): r - group mean."""
    r = rewards.view(-1, num_generations)
    adv = r - r.mean(dim=1, keepdim=True)
    if scale:
        adv = adv / (r.std(dim=1, keepdim=True) + 1e-4)
    return adv.view(-1, 1)


def is_reference(old_per_token_logps, clip_low, clip_high, dual_clip, agg) -> bool:
    return old_per_token_logps is None and clip_low is None and clip_high is None and dual_clip is None and \
        agg == 'token-mean'


def grpo_loss(per_token_logps, ref_per_token_logps, advantages, mask, beta: float, old_per_token_logps=None,
              clip_low=None, clip_high=None, dual_clip=None, agg: str = 'token-mean', clip: float = 0.2,
              clipped: bool | None = None):
    """advantages (B, 1); mask (B, K) of 0 / 1.  old_per_token_logps None: the log-probs themselves, detached (the
    first update: the ratio is 1).  clip_low / clip_high None: `clip`.  clipped None: the reference's expression when
    every option is at its default, the clipped objective otherwise (True / False force one of the two)."""
    K = per_token_logps.size(1)
    if clipped is None:
        clipped = not is_reference(old_per_token_logps, clip_low, clip_high, dual_clip, agg)
    per_token_kl = (
        torch.exp(ref_per_token_logps - per_token_logps) - (ref_per_token_logps - per_token_logps) - 1
    )
    advantages_expanded = advantages.expand(-1, K)
    if clipped:
        old = per_token_logps.detach() if old_per_token_logps is None else old_per_token_logps
        lo = clip if clip_low is None else clip_low
        hi = clip if clip_high is None else clip_high
        s, _, _, _ = objective_terms(per_token_logps, old, advantages_expanded, lo, hi, dual_clip)
    else:
        s = torch.exp(per_token_logps - per_token_logps.detach()) * advantages_expanded
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
    """(clipped fraction, dual-clip fraction) in float64: the PPO definition, aggregated like the loss under
    seq-mean-token-mean and as token fractions over the completion mask otherwise."""
    old = per_token_logps if old_per_token_logps is None else old_per_token_logps
    a = advantages.expand(-1, per_token_logps.size(1))
    return _ppo_clip_fractions(per_token_logps, old, a, mask.bool(), clip_low, clip_high, dual_clip,
                               'seq-mean-token-mean' if agg == 'seq-mean-token-mean' else 'token-mean')
