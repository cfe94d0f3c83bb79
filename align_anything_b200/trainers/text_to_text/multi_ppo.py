"""Multi-PPO rollout and rl_step on the H100 kernels -- mirror of
align_anything/trainers/text_to_text/multi_ppo.py (__init__ :95-101, rollout :253-310, rl_step :330-419,
get_advantages_and_returns :510-570, cumulative_returns :572-591).

Multi-PPO is the text PPO trainer with two differences: rollout repeats every prompt `n_samples_per_prompt` times,
and get_advantages_and_returns picks one of five estimators.  'gae' is K4's scan, exactly as in the text trainer.
'reinforce', 'rloo', 'reinforce_baseline' and 'group_norm' run K4 for the KL-shaped rewards and the metric row sums,
then K4r (ops.estimator_returns) for the group statistic and the discounted returns: two launches and no host sync
where the reference loops over every response position.  The group estimators keep the reference's grouping of the
flattened (B, W) token rewards (SURVEY.md H9).

`fused_lm_head` (inherited from the text trainer) covers all five estimators: rollout scoring is the text trainer's
score_rollout, and both rl_step branches take the actor node of the text trainer (actor_loss_node).

Reads, besides what the text trainer reads, `self.advantage_estimator` and `self.n_samples_per_prompt`.
"""
from __future__ import annotations

from typing import Any

import torch

from ... import ops
from ...utils.multi_process import all_reduce_packed, fused_allreduce
from .ppo import (METRIC_KEYS, actor_loss_node, clip_metrics, lm_head_of, with_bonus_lane, with_clip_lanes,
                  with_entropy_lane)
from .ppo import PPOTrainer as _TextPPOTrainer

__all__ = ['PPOTrainer']

GROUP_ESTIMATORS = ('rloo', 'reinforce_baseline', 'group_norm')


class PPOTrainer(_TextPPOTrainer):
    def __init__(self, cfgs=None, actor_model=None, actor_reference_model=None, reward_model=None,
                 reward_critic_model=None, tokenizer=None, reward_tokenizer=None, *, advantage_estimator='reinforce',
                 n_samples_per_prompt=4, **kwargs) -> None:
        super().__init__(cfgs, actor_model, actor_reference_model, reward_model, reward_critic_model, tokenizer,
                         reward_tokenizer, **kwargs)
        tc = getattr(cfgs, 'train_cfgs', None) if cfgs is not None else None
        est = getattr(tc, 'advantage_estimator', None) if tc is not None else None
        n = getattr(tc, 'n_samples_per_prompt', None) if tc is not None else None
        self.advantage_estimator = advantage_estimator if est is None else est
        self.n_samples_per_prompt = n_samples_per_prompt if n is None else n
        if self.advantage_estimator in GROUP_ESTIMATORS:  # multi_ppo.py:98-101
            assert self.n_samples_per_prompt > 1, f'{self.advantage_estimator} requires n_samples_per_prompt > 1'

    # ---- multi_ppo.py:253-310 ---------------------------------------------------------------
    @torch.no_grad()
    def rollout(self, prompt_only_batch):
        """The text rollout with every prompt repeated n_samples_per_prompt times (tensors: repeat_interleave on dim 0,
        anything else: each item repeated) and `action_mask` added to each training batch."""
        self.set_train(mode=False)
        total = prompt_only_batch['input_ids'].size(0)
        micro = int(self.cfgs.train_cfgs.per_device_train_batch_size)
        n = self.n_samples_per_prompt
        inference_batches, training_batches = [], []
        for i in range(0, total, micro):
            pre_mini_batch = {key: prompt_only_batch[key][i:i + micro] for key in prompt_only_batch}
            mini_batch = {
                k: (v.repeat_interleave(n, dim=0) if isinstance(v, torch.Tensor) else [item for item in v for _ in range(n)])
                for k, v in pre_mini_batch.items()
            }
            actor_batch = self.actor_step(mini_batch)
            inference, training = self.score_rollout(actor_batch, mini_batch['input_ids'].size(-1))
            training['action_mask'] = actor_batch['attention_mask'][:, 1:].bool()
            mini_batch['input_ids'] = inference['input_ids']
            mini_batch['attention_mask'] = inference['attention_mask']
            inference_batches.append(mini_batch)
            training_batches.append(training)
        self.set_train()
        return inference_batches, training_batches

    # ---- multi_ppo.py:510-591 ---------------------------------------------------------------
    def get_advantages_and_returns(self, values, rewards, sequence_mask, start):
        if self.advantage_estimator == 'gae':
            adv, ret = _TextPPOTrainer.get_advantages_and_returns(self, values, rewards, sequence_mask, start)
            # :566-567 mask both in place after every estimator (exact: the value or a signed zero); unlike the text
            # trainer's GAE this zeroes masked positions inside the response.  rl_step never reads those positions.
            m = sequence_mask[:, start:]
            return adv.mul_(m), ret.mul_(m)
        return ops.estimator_returns(rewards, sequence_mask, start, self.advantage_estimator, self.n_samples_per_prompt,
                                     self.gamma, mode=self.mode)

    def cumulative_returns(self, rewards, mask, start):
        """Discounted returns of `rewards[:, start:]` (masked first when `mask` is given), not masked afterwards."""
        if mask is None:
            mask = torch.ones(rewards.shape, dtype=torch.bool, device=rewards.device)
        _, returns = ops.estimator_returns(rewards, mask, start, 'reinforce', 1, self.gamma, mode=self.mode,
                                           mask_outputs=False)
        return returns

    # ---- multi_ppo.py:330-419 ---------------------------------------------------------------
    def rl_step(self, inference_batch, training_batch) -> dict[str, Any]:
        if self.advantage_estimator == 'gae':  # textually the text trainer's rl_step
            return _TextPPOTrainer.rl_step(self, inference_batch, training_batch)
        old_log_probs = training_batch['log_probs']
        ref_log_probs = training_batch['ref_log_probs']
        reward = training_batch['reward']
        old_reward_values = training_batch['reward_values']
        start = training_batch['prompt_idx']
        input_ids = inference_batch['input_ids']
        sequence_mask = inference_batch['attention_mask'][:, 1:]
        head = lm_head_of(self.actor_model) if self.fused_lm_head else None  # refusals before any launch

        # K4 gives the KL-shaped rewards, the metric row sums and the status word (its GAE output is not used); K4r
        # then writes the estimator's advantages / returns and their row means into lanes 3 / 4 of row_stats
        old_rewards, _, _, row_stats = ops.kl_rewards_and_gae(
            reward, old_log_probs, ref_log_probs, old_reward_values, sequence_mask, start, self.kl_coeff,
            self.clip_range_score, self.gamma, self.gae_lambda, mode=self.mode)
        reward_advantages, reward_returns = ops.estimator_returns(
            old_rewards, sequence_mask, start, self.advantage_estimator, self.n_samples_per_prompt, self.gamma,
            mode=self.mode, row_stats=row_stats)

        actor_loss, actor_loss32, entropy_mean, clip_frac = actor_loss_node(
            self, inference_batch, input_ids, start, head, old_log_probs, reward_advantages, sequence_mask)
        self.actor_model.backward(actor_loss)
        self.actor_model.step()

        reward_values = self.reward_critic_model(**inference_batch).scores
        reward_values = reward_values.squeeze(dim=-1)[:, :-1]
        reward_critic_loss, value_row_mean = ops.critic_loss(
            reward_values[:, start:], old_reward_values[:, start:], reward_returns, sequence_mask[:, start:],
            self.clip_range_value, mode=self.mode, return_row_mean=True)
        self.reward_critic_model.backward(reward_critic_loss)
        self.reward_critic_model.step()

        with torch.no_grad():
            # see the text rl_step
            extra = self.log_entropy or entropy_mean is not None or clip_frac is not None
            fused = fused_allreduce(row_stats.device) if not extra else None
            stats = ops.ppo_pack_metrics(row_stats, reward, value_row_mean, actor_loss32, reward_critic_loss,
                                         coll=fused.next((9, 10)) if fused is not None else None)
            if self.log_entropy:
                stats = with_entropy_lane(stats, training_batch['entropy'][:, start:], sequence_mask[:, start:])
            if entropy_mean is not None:
                stats = with_bonus_lane(stats, entropy_mean)
            clip_lane = stats.numel()
            if clip_frac is not None:
                stats = with_clip_lanes(stats, clip_frac, self)
            if fused is None:
                stats = all_reduce_packed(stats, max_lanes=(9, 10))  # ONE collective (reference: 10 + barrier)
            v = stats.tolist()  # ONE host sync (reference: 12 .item())
        ops.raise_for_status(v[10], stats.device)
        out = dict(zip(METRIC_KEYS, v[:10]))
        if self.log_entropy:
            out['train/entropy'] = v[11]
        if entropy_mean is not None:
            out['train/actor_entropy'] = v[12]
        if clip_frac is not None:
            clip_metrics(out, v, clip_lane, self)
        out['train/actor_lr'] = self.actor_model.optimizer.param_groups[0]['lr']
        out['train/reward_critic_lr'] = self.reward_critic_model.optimizer.param_groups[0]['lr']
        self.last_rl_tensors = {'old_rewards': old_rewards, 'advantages': reward_advantages, 'returns': reward_returns}
        return out
