"""TEST INFRASTRUCTURE ONLY -- Multi-PPO's advantage estimators restated twice:

  * with the same ATen ops as the reference (trainers/text_to_text/multi_ppo.py:510-591), so that running it on CUDA
    tensors is "the reference's own arithmetic on the GPU" (the STRICT comparator of tests/test_gpu_multi_ppo.py), and
  * in float64 numpy with explicit flat-index loops: an independent statement of the grouping (SURVEY.md H9) and of
    the return recursion, used as a plausibility check on the port.

Nothing in the package imports this module.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import ref_port as O

ESTIMATORS = ('gae', 'reinforce', 'rloo', 'reinforce_baseline', 'group_norm')


def cumulative_returns(rewards, mask, start: int, gamma: float):
    """multi_ppo.py:572-591."""
    response_length = rewards.size(1) - start
    returns = torch.zeros_like(rewards)
    cumulative_return = torch.zeros(rewards.size(0), device=rewards.device)
    returns = returns[:, start:]
    if mask is not None:
        rewards = mask * rewards
    rewards = rewards[:, start:]
    for t in reversed(range(response_length)):
        cumulative_return = rewards[:, t] + gamma * cumulative_return
        returns[:, t] = cumulative_return
    return returns


def advantages_and_returns(values, rewards, sequence_mask, start: int, estimator: str, n: int, gamma: float,
                           gae_lambda: float = 0.95, mask_outputs: bool = True):
    """multi_ppo.py:510-570.  mask_outputs=False leaves out the final `*= sequence_mask` (`cumulative_returns` on its
    own, as `ops.estimator_returns(..., mask_outputs=False)` computes it)."""
    values = values * sequence_mask
    rewards = rewards * sequence_mask
    if estimator == 'gae':
        adv, ret = O.gae_advantages_and_returns(values, rewards, sequence_mask, start, gamma, gae_lambda)
        advantages, returns = adv, ret
    elif estimator in ('rloo', 'reinforce_baseline', 'group_norm'):
        shape = rewards.shape
        rewards = rewards.reshape(-1, n)
        if estimator == 'rloo':
            baseline = (rewards.sum(-1, keepdim=True) - rewards) / (n - 1)
            rewards = rewards - baseline
        elif estimator == 'reinforce_baseline':
            rewards = rewards - rewards.mean(-1, keepdim=True)
        else:
            mean = rewards.mean(-1, keepdim=True)
            std = rewards.std(-1, keepdim=True) + 1e-9
            rewards = (rewards - mean) / std
        rewards = rewards.view(shape)
        returns = cumulative_returns(rewards, sequence_mask, start, gamma)
        advantages = returns.clone()
    elif estimator == 'reinforce':
        returns = cumulative_returns(rewards, sequence_mask, start, gamma)
        advantages = returns.clone()
    else:
        raise ValueError(f'Unknown estimator: {estimator}')
    if mask_outputs:
        advantages *= sequence_mask[:, start:]
        returns *= sequence_mask[:, start:]
    return advantages, returns


def returns_f64(rewards, mask, start: int, estimator: str, n: int, gamma: float, mask_outputs: bool = True) -> np.ndarray:
    """The four non-GAE estimators in float64, group by group over the flat (B, W) index."""
    r = rewards.detach().double().cpu().numpy() * mask.cpu().numpy()
    B, W = r.shape
    flat = r.reshape(-1)
    x = flat.copy()
    if estimator != 'reinforce':
        for g0 in range(0, flat.size, n):
            grp = flat[g0:g0 + n]
            for k in range(n):
                if estimator == 'rloo':
                    x[g0 + k] = grp[k] - (grp.sum() - grp[k]) / (n - 1)
                elif estimator == 'reinforce_baseline':
                    x[g0 + k] = grp[k] - grp.mean()
                else:
                    x[g0 + k] = (grp[k] - grp.mean()) / (grp.std(ddof=1) + 1e-9)
    x = x.reshape(B, W) * mask.cpu().numpy()
    out = np.zeros((B, W - start))
    for b in range(B):
        c = 0.0
        for t in range(W - 1, start - 1, -1):
            c = x[b, t] + gamma * c
            out[b, t - start] = c
    return out * mask.cpu().numpy()[:, start:] if mask_outputs else out


def rl_step(rollout, new_actor_logits, new_critic_scores, input_ids, attention_mask, start: int, estimator: str,
            n: int, hp: dict | None = None) -> dict[str, torch.Tensor]:
    """multi_ppo.py:330-419 without the engines: oracle/ref_port.ppo_text_rl_step with the estimator switch."""
    hp = {**O.PPO_DEFAULTS, **(hp or {})}
    old_lp, ref_lp = rollout['log_probs'], rollout['ref_log_probs']
    reward, old_values = rollout['reward'], rollout['reward_values']
    seq_mask = attention_mask[:, 1:]
    with torch.no_grad():
        old_rewards = O.kl_shaped_rewards(reward, old_lp, ref_lp, seq_mask, hp['kl_coeff'], hp['clip_range_score'])
        adv, ret = advantages_and_returns(old_values, old_rewards, seq_mask, start, estimator, n, hp['gamma'],
                                          hp['gae_lambda'])
    lp = O.token_log_probs(new_actor_logits[:, :-1], input_ids[:, 1:])
    a_loss = O.actor_loss(lp[:, start:], old_lp[:, start:], adv, seq_mask[:, start:], hp['clip_range_ratio'])
    new_values = new_critic_scores.squeeze(dim=-1)[:, :-1]
    c_loss = O.critic_loss(new_values[:, start:], old_values[:, start:], ret, seq_mask[:, start:],
                           hp['clip_range_value'])
    with torch.no_grad():
        m = seq_mask[:, start:]
        out = {
            'actor_loss': a_loss,
            'reward_critic_loss': c_loss,
            'reward': reward.mean(),
            'reward_with_kl_penalty': (old_rewards[:, start:] * m).sum(dim=-1).mean(),
            'reward_advantage': O.masked_mean(adv, m),
            'reward_return': O.masked_mean(ret, m),
            'reward_value': O.masked_mean(new_values[:, start:], m),
            'kl_divergence': ((old_lp - ref_lp)[:, start:] * m).sum(dim=-1).mean(),
            'mean_generated_length': m.sum(dim=-1).float().mean(),
            'max_generated_length': m.sum(dim=-1).float().max(),
        }
    out['_old_rewards'] = old_rewards
    out['_advantages'] = adv
    out['_returns'] = ret
    return out
