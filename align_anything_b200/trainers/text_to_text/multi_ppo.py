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
score_rollout, and rl_step is the text trainer's, with K4r's advantages and returns for the four non-GAE estimators.

Reads, besides what the text trainer reads, `self.advantage_estimator` and `self.n_samples_per_prompt`.
"""
from __future__ import annotations

from typing import Any

import torch

from ... import ops
from .ppo import PPOTrainer as _TextPPOTrainer
from .ppo import whiten_advantages_of, whiten_rollout

__all__ = ['PPOTrainer']

GROUP_ESTIMATORS = ('rloo', 'reinforce_baseline', 'group_norm')


def estimator_returns_of(tr):
    """The `returns` hook of the text trainer's rl_step for the advantage estimator in effect: None for 'gae' (K4's
    GAE), otherwise K4r's advantages and returns, with their row means written into lanes 3 / 4 of row_stats."""
    if tr.advantage_estimator == 'gae':
        return None

    def returns(old_rewards, sequence_mask, start, row_stats):
        return ops.estimator_returns(old_rewards, sequence_mask, start, tr.advantage_estimator, tr.n_samples_per_prompt,
                                     tr.gamma, mode=tr.mode, row_stats=row_stats)

    return returns


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
        anything else: each item repeated) and `action_mask` added to each training batch.  With whiten_advantages, the
        estimator's advantages whitened over the rollout (REINFORCE++ for 'reinforce'; the group estimators after their
        own group statistic)."""
        whiten = whiten_advantages_of(self)
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
        if whiten:
            whiten_rollout(self, training_batches, [b['attention_mask'][:, 1:] for b in inference_batches],
                           [t['prompt_idx'] for t in training_batches], estimator_returns_of(self))
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
        """The text trainer's rl_step.  Past 'gae', K4r's outputs replace K4's GAE ones: the estimator's advantages and
        returns, with their row means written into lanes 3 / 4 of row_stats (estimator_returns_of)."""
        return _TextPPOTrainer.rl_step(self, inference_batch, training_batch, returns=estimator_returns_of(self))
