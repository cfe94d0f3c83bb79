"""ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU restatement (plain PyTorch ops on whatever device the inputs live on; used
on CPU) of the reference's RLHF loss hot path.  The reference defines its
results as "whatever these ATen ops return in the input dtype" -- including the
bf16 rounding points -- so the restatement uses the same ops in the same order
and dtype, one function per reference function, each citing the reference
file:line it follows (paths relative to the reference's align_anything/ directory).

Pinned: `tests/golden/*.pt`, generated from the *unmodified* reference by
tests/golden/make_golden.py (through oracle/ref_shim.py), hold the reference's
outputs; `tests/test_oracle_golden.py` and `tests/test_oracle_vs_reference.py`
compare every function here against them.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
reference legs may import this module.  Nothing under align_anything_b200/
imports it; the product path has no CPU fallback.
"""
from __future__ import annotations

from typing import Sequence

import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------------------
# a1 / a13 / a3 -- utils/tools.py:402-413, :460-467 ; trainers/text_to_text/dpo.py:52-54
# --------------------------------------------------------------------------------------


def token_log_probs(logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """utils/tools.py:402-413 `gather_log_probabilities`: row log-softmax over V in the
    logits dtype, then pick the label column.  (b, l, V), (b, l) -> (b, l)."""
    full = F.log_softmax(logits, dim=-1)
    picked = full.gather(-1, labels.to(torch.int64).unsqueeze(-1))
    return picked.squeeze(-1)


def masked_mean(x: torch.Tensor, mask: torch.Tensor | None = None) -> torch.Tensor:
    """utils/tools.py:460-467: mean over rows of (masked row sum / row count)."""
    if mask is None:
        return x.mean()
    row = (x * mask).sum(dim=-1) / mask.sum(dim=-1)
    return row.mean()


def drop_pad(seq: torch.Tensor, pad_id: int) -> torch.Tensor:
    """trainers/text_to_text/dpo.py:52-54 `strip_pad`: every pad-valued token is removed,
    wherever it sits."""
    return seq[seq != pad_id]


# --------------------------------------------------------------------------------------
# a2 / a4 / a5 -- trainers/text_to_text/dpo.py:122-237 (+ TI2T :85-166, TA2T :86-171)
# --------------------------------------------------------------------------------------


def dpo_sequence_log_probs(
    logits: torch.Tensor,  # (2B, L, V)
    input_ids: torch.Tensor,  # (2B, L)
    response_lens: Sequence[int],
    pad_id: int,
    strip: bool = True,
) -> torch.Tensor:
    """trainers/text_to_text/dpo.py:122-142 (strip=True; same body in
    text_image_to_text/dpo.py:85-105) and text_audio_to_text/dpo.py:86-105 (strip=False):
    per sample, the last R logits rows against the last R (pad-stripped) ids, shifted by one;
    rows right-padded with 0.0 to the longest."""
    rows = []
    for i, r in enumerate(response_lens):
        ids = drop_pad(input_ids[i], pad_id) if strip else input_ids[i]
        tail_logits = logits[i][-r:].unsqueeze(0)
        tail_ids = ids[-r:].unsqueeze(0)
        rows.append(token_log_probs(tail_logits[:, :-1], tail_ids[:, 1:]).squeeze(0))
    return torch.nn.utils.rnn.pad_sequence(rows, batch_first=True, padding_value=0.0)


def dpo_loss(
    policy_lp: torch.Tensor,  # (2B, W)
    ref_lp: torch.Tensor,  # (2B, W)
    scale_coeff: float,
    input_ids: torch.Tensor | None = None,
    skip_identical_pairs: bool = False,
) -> dict[str, torch.Tensor]:
    """trainers/text_to_text/dpo.py:150-203.  `skip_identical_pairs` reproduces
    text_audio_to_text/dpo.py:134-139 (pairs with equal chosen/rejected id rows are dropped)."""
    better, worse = policy_lp.chunk(2, dim=0)
    ref_better, ref_worse = ref_lp.chunk(2, dim=0)
    if skip_identical_pairs:
        ids_better, ids_worse = input_ids.chunk(2, dim=0)
    per_pair, r_better, r_worse = [], [], []
    for i in range(better.size(0)):
        if skip_identical_pairs and bool(torch.all(torch.eq(ids_better[i], ids_worse[i]))):
            continue
        pc = better[i, :].sum(dim=-1)
        pr = worse[i, :].sum(dim=-1)
        rc = ref_better[i, :].sum(dim=-1)
        rr = ref_worse[i, :].sum(dim=-1)
        ratio_c = pc - rc
        ratio_r = pr - rr
        per_pair.append(-F.logsigmoid(scale_coeff * (ratio_c - ratio_r)))
        r_better.append(scale_coeff * ratio_c.detach())
        r_worse.append(scale_coeff * ratio_r.detach())
    loss = torch.stack(per_pair).mean()
    r_better = torch.stack(r_better)
    r_worse = torch.stack(r_worse)
    return {
        'loss': loss,
        'reward': r_better + r_worse,
        'better_sample_reward': r_better,
        'worse_sample_reward': r_worse,
        'reward_accuracy': (r_better > r_worse).float().mean(),
        'reward_margin': r_better - r_worse,
    }


def dpo_step_metrics(loss_dict: dict[str, torch.Tensor]) -> dict[str, torch.Tensor]:
    """trainers/text_to_text/dpo.py:215-227: the six local scalars that are then
    all-reduced with AVG (world size 1: unchanged)."""
    with torch.no_grad():
        return {
            'train/loss': loss_dict['loss'].detach(),
            'train/reward': loss_dict['reward'].mean(),
            'train/better_sample_reward': loss_dict['better_sample_reward'].mean(),
            'train/worse_sample_reward': loss_dict['worse_sample_reward'].mean(),
            'train/reward_accuracy': loss_dict['reward_accuracy'],
            'train/reward_margin': loss_dict['reward_margin'].mean(),
        }


def dpo_forward_backward(
    policy_logits: torch.Tensor,
    ref_logits: torch.Tensor,
    input_ids: torch.Tensor,
    response_lens: Sequence[int],
    pad_id: int,
    scale_coeff: float,
    strip: bool = True,
    skip_identical_pairs: bool = False,
) -> tuple[dict[str, torch.Tensor], torch.Tensor]:
    """One DPO unit of work as bench.py times it: policy log-probs (with grad), reference
    log-probs (no grad), loss, backward down to the policy logits (dpo.py:144-213 minus the
    model forward/optimizer).  Returns (loss dict, d loss / d policy_logits)."""
    leaf = policy_logits.detach().requires_grad_(True)
    lp = dpo_sequence_log_probs(leaf, input_ids, response_lens, pad_id, strip)
    with torch.no_grad():
        rlp = dpo_sequence_log_probs(ref_logits, input_ids, response_lens, pad_id, strip)
    out = dpo_loss(lp, rlp, scale_coeff, input_ids, skip_identical_pairs)
    out['loss'].backward()
    return out, leaf.grad


# --------------------------------------------------------------------------------------
# a8 -- models/llama.py:62-93 (opt.py, qwen2_audio.py:75-104 same), llava.py:62-66,
#       qwen2_vl.py:58-64 ; models/reward_model.py:22-32
# --------------------------------------------------------------------------------------


def score_head(
    last_hidden: torch.Tensor,  # (B, L, H)
    weight: torch.Tensor,  # (1, H)
    attention_mask: torch.Tensor | None,
    end_mode: str = 'mask',  # 'mask': last attended position ; 'last': position L-1
    upcast_scores: bool = True,
) -> dict[str, torch.Tensor]:
    """Scalar head of the reward / critic models.
    end_mode='mask', upcast: models/llama.py:62-93 (OPT identical; Qwen2-Audio passes the
    expanded mask, qwen2_audio.py:75-80).  end_mode='last': models/llava.py:62-66
    (scores upcast) and models/qwen2_vl.py:58-64 (scores NOT upcast, upcast_scores=False;
    end_scores always float)."""
    scores = F.linear(last_hidden, weight)
    if upcast_scores:
        scores = scores.float()
    bsz = last_hidden.size(0)
    if end_mode == 'mask':
        if attention_mask is None:
            if bsz > 1:
                raise ValueError("'attention_mask' is required when batch size > 1.")
            attention_mask = last_hidden.new_ones(bsz, last_hidden.size(1), dtype=torch.bool)
        end_index = torch.cat([m.nonzero()[-1] for m in attention_mask])
        pick = end_index.view(bsz, 1, 1)
        end_hidden = last_hidden.gather(1, pick.expand(-1, -1, last_hidden.size(-1))).squeeze(1)
        end_scores = scores.gather(1, pick.expand(-1, -1, scores.size(-1))).squeeze(1)
    elif end_mode == 'last':
        end_index = -torch.ones((bsz,))
        end_hidden = last_hidden[:, -1, :]
        end_scores = F.linear(end_hidden.unsqueeze(1), weight).float().squeeze(1)
    else:
        raise ValueError(end_mode)
    return {
        'scores': scores,
        'end_scores': end_scores,
        'end_last_hidden_state': end_hidden,
        'end_index': end_index,
    }


# --------------------------------------------------------------------------------------
# a9 - a12 -- trainers/text_to_text/ppo.py:291-307, :487-547
# --------------------------------------------------------------------------------------


def kl_shaped_rewards(
    reward: torch.Tensor,  # (B,)
    log_probs: torch.Tensor,  # (B, L')
    ref_log_probs: torch.Tensor,  # (B, L')
    sequence_mask: torch.Tensor,  # (B, L') bool
    kl_coeff: float,
    clip_range_score: float,
) -> torch.Tensor:
    """trainers/text_to_text/ppo.py:528-547: -kl_coeff * (logp - ref) per token, the scalar
    reward added at the last attended position, clamped to +-clip_range_score."""
    end_index = torch.cat([m.nonzero()[-1] for m in sequence_mask])
    penalty = -kl_coeff * (log_probs - ref_log_probs)
    shaped = torch.scatter_add(
        penalty, -1, end_index.unsqueeze(-1), reward.to(penalty.dtype).unsqueeze(-1)
    )
    return torch.clamp(shaped, min=-clip_range_score, max=clip_range_score)


def gae_advantages_and_returns(
    values: torch.Tensor,  # (B, L')
    rewards: torch.Tensor,  # (B, L')
    sequence_mask: torch.Tensor,  # (B, L') bool
    start: int,
    gamma: float,
    gae_lambda: float,
) -> tuple[torch.Tensor, torch.Tensor]:
    """trainers/text_to_text/ppo.py:487-508: reverse recurrence over t in [start, L')."""
    carry = 0.0
    rev = []
    values = values * sequence_mask
    rewards = rewards * sequence_mask
    width = rewards.size(-1)
    for t in range(width - 1, start - 1, -1):
        nxt = values[:, t + 1] if t < width - 1 else 0.0
        delta = rewards[:, t] + gamma * nxt - values[:, t]
        carry = delta + gamma * gae_lambda * carry
        rev.append(carry)
    adv = torch.stack(rev[::-1], dim=1)
    ret = adv + values[:, start:]
    return adv.detach(), ret


def actor_loss(log_probs, old_log_probs, advantages, mask, clip_range_ratio: float):
    """trainers/text_to_text/ppo.py:291-307."""
    ratio = torch.exp(log_probs - old_log_probs)
    unclipped = advantages * ratio
    clipped = advantages * torch.clamp(ratio, 1.0 - clip_range_ratio, 1.0 + clip_range_ratio)
    return -masked_mean(torch.minimum(unclipped, clipped), mask)


def critic_loss(values, old_values, returns, mask, clip_range_value: float):
    """trainers/text_to_text/ppo.py:510-526."""
    clipped = torch.clamp(values, old_values - clip_range_value, old_values + clip_range_value)
    worst = torch.maximum(torch.square(values - returns), torch.square(clipped - returns))
    return 0.5 * masked_mean(worst, mask)


# --------------------------------------------------------------------------------------
# a6 / a14 (text) -- trainers/text_to_text/ppo.py:244-289, :309-398, given the model outputs
# --------------------------------------------------------------------------------------

PPO_DEFAULTS = dict(
    kl_coeff=0.02,
    clip_range_ratio=0.2,
    clip_range_score=50.0,
    clip_range_value=5.0,
    gamma=1.0,
    gae_lambda=0.95,
)


def ppo_text_rollout_scoring(actor_logits, ref_logits, input_ids, reward_end_scores, critic_scores):
    """trainers/text_to_text/ppo.py:237-240, :266-271: the scoring half of rollout() once
    generation and the four forwards are done.  critic_scores: (B, L, 1)."""
    with torch.no_grad():
        return {
            'log_probs': token_log_probs(actor_logits[:, :-1], input_ids[:, 1:]),
            'ref_log_probs': token_log_probs(ref_logits[:, :-1], input_ids[:, 1:]),
            'reward': reward_end_scores.squeeze(dim=-1),
            'reward_values': critic_scores.squeeze(dim=-1)[:, :-1],
        }


def ppo_text_rl_step(
    rollout: dict[str, torch.Tensor],
    new_actor_logits: torch.Tensor,  # (B, L, V), leaf or not
    new_critic_scores: torch.Tensor,  # (B, L, 1)
    input_ids: torch.Tensor,
    attention_mask: torch.Tensor,
    start: int,
    hp: dict | None = None,
) -> dict[str, torch.Tensor]:
    """trainers/text_to_text/ppo.py:309-381 without the engines: returns the two losses
    (autograd-attached) and the ten local metric scalars (before all-reduce)."""
    hp = {**PPO_DEFAULTS, **(hp or {})}
    old_lp, ref_lp = rollout['log_probs'], rollout['ref_log_probs']
    reward, old_values = rollout['reward'], rollout['reward_values']
    seq_mask = attention_mask[:, 1:]
    with torch.no_grad():
        old_rewards = kl_shaped_rewards(
            reward, old_lp, ref_lp, seq_mask, hp['kl_coeff'], hp['clip_range_score']
        )
        adv, ret = gae_advantages_and_returns(
            old_values, old_rewards, seq_mask, start, hp['gamma'], hp['gae_lambda']
        )
    lp = token_log_probs(new_actor_logits[:, :-1], input_ids[:, 1:])
    a_loss = actor_loss(
        lp[:, start:], old_lp[:, start:], adv, seq_mask[:, start:], hp['clip_range_ratio']
    )
    new_values = new_critic_scores.squeeze(dim=-1)[:, :-1]
    c_loss = critic_loss(
        new_values[:, start:], old_values[:, start:], ret, seq_mask[:, start:], hp['clip_range_value']
    )
    with torch.no_grad():
        m = seq_mask[:, start:]
        out = {
            'actor_loss': a_loss,
            'reward_critic_loss': c_loss,
            'reward': reward.mean(),
            'reward_with_kl_penalty': (old_rewards[:, start:] * m).sum(dim=-1).mean(),
            'reward_advantage': masked_mean(adv, m),
            'reward_return': masked_mean(ret, m),
            'reward_value': masked_mean(new_values[:, start:], m),
            'kl_divergence': ((old_lp - ref_lp)[:, start:] * m).sum(dim=-1).mean(),
            'mean_generated_length': m.sum(dim=-1).float().mean(),
            'max_generated_length': m.sum(dim=-1).float().max(),
        }
    out['_old_rewards'] = old_rewards
    out['_advantages'] = adv
    out['_returns'] = ret
    out['_log_probs'] = lp
    return out


# --------------------------------------------------------------------------------------
# a6 / a14 / a15 / a16 (multimodal) -- trainers/text_image_to_text/ppo.py:56-87, :190-379
# --------------------------------------------------------------------------------------


def move_padding_left(ids: torch.Tensor, pad_id: int) -> torch.Tensor:
    """trainers/text_image_to_text/ppo.py:56-87 (dup utils/tools.py:615-639): circular shift
    of each row by (number of pads that are NOT leading), via gather with modular indices."""
    width = ids.size(1)
    is_pad = ids == pad_id
    leading = is_pad.cumsum(dim=1).eq(torch.arange(1, width + 1, device=ids.device)).sum(dim=1)
    kept = (~is_pad).sum(dim=1)
    cols = torch.arange(width, device=ids.device).expand(ids.size(0), width)
    shift = width - kept.unsqueeze(1) - leading.unsqueeze(1)
    return torch.gather(ids, 1, (cols - shift) % width)


def response_lengths(prompt_ids: torch.Tensor, sequences: torch.Tensor, pad_id: int) -> list[int]:
    """trainers/text_image_to_text/ppo.py:190-203: len(non-pad(sequence)[n_prompt:]) with
    n_prompt = number of non-pad prompt tokens."""
    out = []
    for b in range(sequences.size(0)):
        n_prompt = int((prompt_ids[b] != pad_id).sum())
        n_seq = int((sequences[b] != pad_id).sum())
        out.append(max(n_seq - n_prompt, 0))
    return out


def _tail_rows(x2d_list, fill=0.0):
    return torch.nn.utils.rnn.pad_sequence(x2d_list, batch_first=True, padding_value=fill)


def ppo_mm_rollout_scoring(actor_logits, ref_logits, input_ids, response_lens, reward, reward_values):
    """trainers/text_image_to_text/ppo.py:224-250: per-sample response tails, right padded
    with 0; response_mask = (log_probs != 0).  reward_values: (B, L-1)."""
    with torch.no_grad():
        lp, rlp, vals = [], [], []
        for b, r in enumerate(response_lens):
            ids = input_ids[b, 1:][-r:].unsqueeze(0)
            lp.append(token_log_probs(actor_logits[b, :-1][-r:].unsqueeze(0), ids).squeeze())
            rlp.append(token_log_probs(ref_logits[b, :-1][-r:].unsqueeze(0), ids).squeeze())
            vals.append(reward_values[b][-r:].unsqueeze(0).squeeze())
        log_probs = _tail_rows(lp)
        return {
            'response_lens': list(response_lens),
            'log_probs': log_probs,
            'ref_log_probs': _tail_rows(rlp),
            'reward': reward,
            'reward_values': _tail_rows(vals),
            'response_mask': (log_probs != 0).bool(),
        }


def ppo_mm_rl_step(
    rollout: dict,
    new_actor_logits: torch.Tensor,
    new_critic_scores: torch.Tensor,  # (B, L, 1)
    input_ids: torch.Tensor,
    hp: dict | None = None,
) -> dict[str, torch.Tensor]:
    """trainers/text_image_to_text/ppo.py:271-347 without the engines (GAE start = 0,
    losses over the whole padded width under response_mask)."""
    hp = {**PPO_DEFAULTS, **(hp or {})}
    lens = rollout['response_lens']
    old_lp, ref_lp = rollout['log_probs'], rollout['ref_log_probs']
    reward, old_values, mask = rollout['reward'], rollout['reward_values'], rollout['response_mask']
    with torch.no_grad():
        old_rewards = kl_shaped_rewards(
            reward, old_lp, ref_lp, mask, hp['kl_coeff'], hp['clip_range_score']
        )
        adv, ret = gae_advantages_and_returns(
            old_values, old_rewards, mask, 0, hp['gamma'], hp['gae_lambda']
        )
    rows = []
    for b, r in enumerate(lens):
        ids = input_ids[b, 1:][-r:].unsqueeze(0)
        rows.append(token_log_probs(new_actor_logits[b, :-1][-r:].unsqueeze(0), ids).squeeze())
    lp = _tail_rows(rows)
    a_loss = actor_loss(lp, old_lp, adv, mask, hp['clip_range_ratio'])
    raw = new_critic_scores.squeeze(dim=-1)[:, :-1]
    new_values = _tail_rows([raw[b][-r:].unsqueeze(0).squeeze() for b, r in enumerate(lens)])
    c_loss = critic_loss(new_values, old_values, ret, mask, hp['clip_range_value'])
    with torch.no_grad():
        out = {
            'actor_loss': a_loss,
            'reward_critic_loss': c_loss,
            'reward': reward.mean(),
            'reward_with_kl_penalty': (old_rewards * mask).sum(dim=-1).mean(),
            'reward_advantage': masked_mean(adv, mask),
            'reward_return': masked_mean(ret, mask),
            'reward_value': masked_mean(new_values, mask),
            'kl_divergence': ((old_lp - ref_lp) * mask).sum(dim=-1).mean(),
            'mean_generated_length': mask.sum(dim=-1).float().mean(),
            'max_generated_length': mask.sum(dim=-1).float().max(),
        }
    out['_old_rewards'] = old_rewards
    out['_advantages'] = adv
    out['_returns'] = ret
    out['_log_probs'] = lp
    return out


# --------------------------------------------------------------------------------------
# f4 -- the `outputs.loss` consumed by SupervisedTrainer.loss (trainers/text_to_text/sft.py:95-98) and
#       PPOTrainer.ptx_step (trainers/text_to_text/ppo.py:400-408).  The arithmetic lives in a third-party
#       dependency that is NOT part of the reference: transformers (pyproject.toml:37 pins ">=4.50.0";
#       installed here 5.5.0), `transformers.loss.loss_utils.ForCausalLMLoss`: logits upcast to fp32,
#       labels padded with ignore_index and shifted by one, mean cross-entropy over labels != ignore_index.
#       Pinned by tests/golden/sft.pt (a tiny LlamaForCausalLM run through the real HF forward).
# --------------------------------------------------------------------------------------


def causal_lm_loss(logits: torch.Tensor, labels: torch.Tensor, ignore_index: int = -100) -> torch.Tensor:
    upcast = logits.float()
    shifted = F.pad(labels, (0, 1), value=ignore_index)[..., 1:].contiguous()
    return F.cross_entropy(upcast.view(-1, upcast.size(-1)), shifted.view(-1), ignore_index=ignore_index,
                           reduction='mean')


# --------------------------------------------------------------------------------------
# f2 -- reward-model pairwise loss, trainers/text_to_text/rm.py:97-132
# --------------------------------------------------------------------------------------


def rm_pair_loss(scores: torch.Tensor, end_scores: torch.Tensor, regularization: float = 0.0) -> dict[str, torch.Tensor]:
    """scores (2B, L, 1), end_scores (2B, 1): higher rows first."""
    higher_rewards, lower_rewards = scores.squeeze(dim=-1).chunk(chunks=2, dim=0)
    higher_end, lower_end = end_scores.squeeze(dim=-1).chunk(chunks=2, dim=0)
    loss = -F.logsigmoid(higher_end - lower_end).mean()
    if regularization > 0.0:
        loss = loss + regularization * torch.stack([lower_end, higher_end]).square().mean()
    return {
        'loss': loss,
        'higher_end_reward': higher_end,
        'lower_end_reward': lower_end,
        'higher_rewards': higher_rewards,
        'lower_rewards': lower_rewards,
        'accuracy': (higher_end > lower_end).float().mean(),
    }


# --------------------------------------------------------------------------------------
# f2 -- GRPO, trainers/text_to_text/grpo.py:199-210 (_get_per_token_logps), :268-318 (train_step arithmetic)
# --------------------------------------------------------------------------------------


def grpo_per_token_logps(logits: torch.Tensor, input_ids: torch.Tensor, logits_to_keep: int) -> torch.Tensor:
    """trainers/text_to_text/grpo.py:203-210 given the model's logits."""
    tail = logits[:, :-1, :][:, -logits_to_keep:, :]
    log_probs = F.log_softmax(tail, dim=-1)
    target = input_ids[:, -logits_to_keep:]
    return log_probs.gather(dim=-1, index=target.unsqueeze(-1)).squeeze(-1)


def grpo_group_advantages(rewards: torch.Tensor, n_prompts: int, num_generations: int) -> torch.Tensor:
    """trainers/text_to_text/grpo.py:268-274."""
    r = rewards.view(n_prompts, num_generations)
    adv = (r - r.mean(dim=1, keepdim=True)) / (r.std(dim=1, keepdim=True) + 1e-4)
    return adv.view(-1, 1)


def grpo_loss(per_token_logps, ref_per_token_logps, advantages, sequences, prompt_length: int, eos_token_id: int,
              beta: float) -> torch.Tensor:
    """trainers/text_to_text/grpo.py:290-312."""
    keep = sequences.size(1) - prompt_length
    # NB: the reference evaluates (ref - logp) twice as separate ops; autograd then accumulates three gradient
    # contributions into logp in node order, each rounded in the logp dtype -- keep the same expression shape
    per_token_kl = (
        torch.exp(ref_per_token_logps - per_token_logps) - (ref_per_token_logps - per_token_logps) - 1
    )
    per_token_loss = torch.exp(per_token_logps - per_token_logps.detach()) * advantages.expand(-1, keep)
    per_token_loss = -(per_token_loss - beta * per_token_kl)
    completion = sequences[:, prompt_length:]
    mask = torch.ones_like(completion)
    for i in range(completion.size(0)):
        eos = (completion[i] == eos_token_id).nonzero(as_tuple=False)
        if eos.numel() > 0:
            mask[i, eos[0].item() + 1:] = 0
    mask = mask.to(per_token_loss.dtype)
    return (per_token_loss * mask).sum() / mask.sum()


# --------------------------------------------------------------------------------------
# f2 -- SimPO / ORPO / KTO, trainers/text_to_text/simpo.py:41-108, orpo.py:41-113, kto.py:83-159
#       (all three inherit DPOTrainer.compute_log_probs, i.e. dpo_sequence_log_probs above)
# --------------------------------------------------------------------------------------


def _pair_slices(ids_better, ids_worse, mask_better, mask_worse, i):
    """simpo.py:63-77: end indices from the attention masks, first index where the id rows differ."""
    end_b = mask_better[i].nonzero()[-1].squeeze().item()
    end_w = mask_worse[i].nonzero()[-1].squeeze().item()
    diverge = (ids_better[i] != ids_worse[i]).nonzero()[0].squeeze().item()
    assert 0 <= diverge <= end_b, 'diverge index is out of range!'
    assert 0 <= diverge <= end_w, 'diverge index is out of range!'
    return slice(diverge, end_b + 1), slice(diverge, end_w + 1), end_b + 1, end_w + 1


def _pair_metrics(losses, r_better, r_worse):
    loss = torch.stack(losses).mean()
    r_better, r_worse = torch.stack(r_better), torch.stack(r_worse)
    return {
        'loss': loss, 'reward': r_better + r_worse, 'better_sample_reward': r_better, 'worse_sample_reward': r_worse,
        'reward_accuracy': (r_better > r_worse).float().mean(), 'reward_margin': r_better - r_worse,
    }


def simpo_loss(policy_lp, input_ids, attention_mask, scale_coeff: float, gamma: float):
    """trainers/text_to_text/simpo.py:46-108."""
    better, worse = policy_lp.chunk(2, dim=0)
    ids_b, ids_w = input_ids.chunk(2, dim=0)
    m_b, m_w = attention_mask.chunk(2, dim=0)
    losses, rb, rw = [], [], []
    for i in range(ids_b.size(0)):
        if torch.all(torch.eq(ids_b[i], ids_w[i])).item():
            continue
        sl_b, sl_w, len_b, len_w = _pair_slices(ids_b, ids_w, m_b, m_w, i)
        ratio_b = better[i, sl_b].sum(dim=-1) / len_b
        ratio_w = worse[i, sl_w].sum(dim=-1) / len_w
        losses.append(-F.logsigmoid(scale_coeff * (ratio_b - ratio_w) - gamma))
        rb.append(scale_coeff * ratio_b.detach())
        rw.append(scale_coeff * ratio_w.detach())
    return _pair_metrics(losses, rb, rw)


def orpo_loss(policy_lp, input_ids, attention_mask, scale_coeff: float):
    """trainers/text_to_text/orpo.py:46-113."""
    better, worse = policy_lp.chunk(2, dim=0)
    ids_b, ids_w = input_ids.chunk(2, dim=0)
    m_b, m_w = attention_mask.chunk(2, dim=0)
    losses, rb, rw = [], [], []
    for i in range(ids_b.size(0)):
        if torch.all(torch.eq(ids_b[i], ids_w[i])).item():
            continue
        sl_b, sl_w, len_b, len_w = _pair_slices(ids_b, ids_w, m_b, m_w, i)
        ratio_b = better[i, sl_b].sum(dim=-1) / len_b
        ratio_w = worse[i, sl_w].sum(dim=-1) / len_w
        log_odds = (ratio_b - ratio_w) - (torch.log1p(-torch.exp(ratio_b)) - torch.log1p(-torch.exp(ratio_w)))
        odds_ratio_loss = -F.logsigmoid(log_odds)
        sft_loss = -ratio_b
        losses.append(sft_loss + scale_coeff * odds_ratio_loss)
        rb.append(scale_coeff * ratio_b.detach())
        rw.append(scale_coeff * ratio_w.detach())
    return _pair_metrics(losses, rb, rw)


def kto_loss(policy_lp, ref_lp, input_ids, attention_mask, scale_coeff: float, scale_better: float, scale_worse: float, kl):
    """trainers/text_to_text/kto.py:88-159."""
    better, worse = policy_lp.chunk(2, dim=0)
    ref_better, ref_worse = ref_lp.chunk(2, dim=0)
    ids_b, ids_w = input_ids.chunk(2, dim=0)
    m_b, m_w = attention_mask.chunk(2, dim=0)
    losses, rb, rw = [], [], []
    for i in range(ids_b.size(0)):
        if torch.all(torch.eq(ids_b[i], ids_w[i])).item():
            continue
        sl_b, sl_w, _, _ = _pair_slices(ids_b, ids_w, m_b, m_w, i)
        ratio_b = better[i, sl_b].sum(dim=-1) - ref_better[i, sl_b].sum(dim=-1)
        ratio_w = worse[i, sl_w].sum(dim=-1) - ref_worse[i, sl_w].sum(dim=-1)
        losses.append(scale_better * (1 - F.sigmoid(scale_coeff * (ratio_b - kl)))
                      - scale_worse * (1 - F.sigmoid(scale_coeff * (kl - ratio_w))))
        rb.append(scale_coeff * ratio_b.detach())
        rw.append(scale_coeff * ratio_w.detach())
    return _pair_metrics(losses, rb, rw)


# --------------------------------------------------------------------------------------
# f2 -- Safe RLHF-V, trainers/text_image_to_text/saferlhf.py:432-481 (+ :513-536, :772-793)
# --------------------------------------------------------------------------------------


def saferlhf_actor_loss(log_probs, old_log_probs, reward_advantages, cost_advantages, mask, multiplier: float,
                        clip_range_ratio: float) -> torch.Tensor:
    """saferlhf.py:432-451; multiplier = log_lambda.exp().item()."""
    advantages = (reward_advantages - multiplier * cost_advantages) / (1.0 + multiplier)
    return actor_loss(log_probs, old_log_probs, advantages, mask, clip_range_ratio)


def saferlhf_kl_rewards_and_costs(reward, cost, log_probs, ref_log_probs, sequence_mask, kl_coeff: float,
                                  clip_range_score: float):
    """saferlhf.py:453-481."""
    end_index = torch.cat([m.nonzero()[-1] for m in sequence_mask])
    penalty = -kl_coeff * (log_probs - ref_log_probs)
    rewards = torch.scatter_add(penalty, -1, end_index.unsqueeze(-1), reward.to(penalty.dtype).unsqueeze(-1))
    costs = torch.scatter_add(-penalty, -1, end_index.unsqueeze(-1), cost.to(penalty.dtype).unsqueeze(-1))
    return (torch.clamp(rewards, min=-clip_range_score, max=clip_range_score),
            torch.clamp(costs, min=-clip_range_score, max=clip_range_score))


def saferlhf_losses(c: dict, hp: dict | None = None) -> dict[str, torch.Tensor]:
    """The arithmetic of SafeRLHFVTrainer.rl_step (saferlhf.py:513-600) on given tensors: all-ones mask,
    KL-shaped rewards / costs, two GAE passes from 0, Lagrangian actor loss, two critic losses."""
    hp = {**PPO_DEFAULTS, **(hp or {})}
    lp, rlp = c['log_probs'], c['ref_log_probs']
    mask = torch.ones_like(lp, dtype=torch.bool)
    with torch.no_grad():
        rew, cst = saferlhf_kl_rewards_and_costs(c['reward'], c['cost'], lp, rlp, mask, hp['kl_coeff'],
                                                 hp['clip_range_score'])
        radv, rret = gae_advantages_and_returns(c['reward_values'], rew, mask, 0, hp['gamma'], hp['gae_lambda'])
        cadv, cret = gae_advantages_and_returns(c['cost_values'], cst, mask, 0, hp['gamma'], hp['gae_lambda'])
    a = saferlhf_actor_loss(c['new_log_probs'], lp, radv, cadv, mask, c['multiplier'], hp['clip_range_ratio'])
    rc = critic_loss(c['new_reward_values'], c['reward_values'], rret, mask, hp['clip_range_value'])
    cc = critic_loss(c['new_cost_values'], c['cost_values'], cret, mask, hp['clip_range_value'])
    return dict(rewards=rew, costs=cst, reward_advantages=radv, reward_returns=rret, cost_advantages=cadv,
                cost_returns=cret, actor_loss=a, reward_critic_loss=rc, cost_critic_loss=cc)
