"""Safe RLHF-V (PPO-Lagrangian with a cost model) on the H100 kernels -- mirror of the loss half of
align_anything/trainers/text_image_to_text/saferlhf.py: actor_step :289-319, rollout :343-430,
actor_loss_fn_with_cost :432-451, add_kl_divergence_regularization_with_cost :453-481, rl_step :483-675
(get_advantages_and_returns :772-793 is the text trainer's).  `model.generate`, cost_model_step / reward_model_step
(backbone forwards), the cost / reward / critic backbones and the dataset plumbing stay in the reference.

The cost side reuses K4 unchanged: costs = clamp(scatter_add(+kl_coeff * kl, end, cost)) is the reward
expression with `kl_coeff -> -kl_coeff` (negation is exact in every dtype), so ONE extra aa_ppo_prep launch
yields old_costs, cost advantages / returns and their metric row sums."""
from __future__ import annotations

from typing import Any

import torch
import torch.distributed as dist

from ... import ops
from ...utils.multi_process import all_reduce_packed
from .ppo import PPOTrainer as _MMPPOTrainer
from .ppo import _tail_values

__all__ = ['SafeRLHFVTrainer']

METRIC_KEYS = (
    'train/actor_loss', 'train/reward_critic_loss', 'train/reward', 'train/reward_with_kl_penalty',
    'train/reward_advantage', 'train/reward_return', 'train/reward_value', 'train/kl_divergence',
    'train/mean_generated_length', 'train/max_generated_length',
    'train/cost_critic_loss', 'train/cost', 'train/cost_with_kl_penalty', 'train/cost_advantage', 'train/cost_return',
    'train/cost_value',
)


class SafeRLHFVTrainer(_MMPPOTrainer):
    log_lambda: torch.Tensor  # nn.Parameter in the reference (saferlhf.py:107-110)

    # ---- saferlhf.py:343-430: the multimodal scoring plus the cost model's end score and the cost critic's values ----
    @torch.no_grad()
    def score_rollout(self, actor_batch, response_lens):
        inference, training = super().score_rollout(actor_batch, response_lens)
        cost_batch = self.cost_model_step(actor_batch)  # the reference's own method (backbone forwards + episode_costs)
        lens = training['response_lens']
        training['cost'] = cost_batch['cost']
        training['cost_values'] = _tail_values(cost_batch['cost_values'], lens)
        if lens.bound < 3 and min(lens.tolist()) == 1:  # (host read only in this corner: at most 2 generated positions)
            # a length-1 response is widened to [x, 0, 0] by the reference (:370-388), so pad_sequence yields width 3
            for k in ('log_probs', 'ref_log_probs', 'reward_values', 'cost_values'):
                training[k] = torch.nn.functional.pad(training[k], (0, 3 - training[k].size(-1)))
            training['response_mask'] = training['log_probs'] != 0
        return inference, training

    # ---- saferlhf.py:432-451 ---------------------------------------------------------------------------
    def actor_loss_fn_with_cost(self, log_probs, old_log_probs, reward_advantages, cost_advantages, mask) -> torch.Tensor:
        multiplier = self.log_lambda.exp().item()
        advantages = (reward_advantages - multiplier * cost_advantages) / (1.0 + multiplier)
        return ops.actor_loss(log_probs, old_log_probs, advantages, mask, self.clip_range_ratio, mode=self.mode)

    # ---- saferlhf.py:453-481 ---------------------------------------------------------------------------
    def add_kl_divergence_regularization_with_cost(self, reward, cost, log_probs, ref_log_probs, sequence_mask):
        zeros = torch.zeros_like(log_probs)
        rewards = ops.kl_rewards_and_gae(reward, log_probs, ref_log_probs, zeros, sequence_mask, 0, self.kl_coeff,
                                         self.clip_range_score, self.gamma, self.gae_lambda, mode=self.mode)[0]
        costs = ops.kl_rewards_and_gae(cost, log_probs, ref_log_probs, zeros, sequence_mask, 0, -self.kl_coeff,
                                       self.clip_range_score, self.gamma, self.gae_lambda, mode=self.mode)[0]
        return rewards, costs

    # ---- saferlhf.py:487-500 (scalar, host side: kept as the reference writes it) -------------------------
    def update_lambda(self, episode_cost: torch.Tensor) -> None:
        lambda_loss = -(episode_cost - self.threshold) * self.log_lambda.exp()
        lambda_loss = torch.clamp(lambda_loss, min=-1e6, max=1e6)
        self.log_lambda_optimizer.zero_grad()
        lambda_loss.backward()
        self.log_lambda_optimizer.step()
        if self.log_lambda_max is not None:
            with torch.no_grad():
                self.log_lambda.clamp_(max=self.log_lambda_max)

    def _lambda_step(self) -> None:
        """saferlhf.py:487-500: mean episode cost over the window, averaged onto rank 0, one SGD step on
        log_lambda there (after `lambda_update_delay_steps`), broadcast back."""
        costs = getattr(self, 'episode_costs', None)
        if not costs:
            return
        episode_cost = torch.tensor(list(costs), dtype=torch.float32).mean().to(self.log_lambda.device)
        multi = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
        if multi:
            dist.reduce(episode_cost, dst=0, op=dist.ReduceOp.SUM)
            episode_cost = episode_cost / dist.get_world_size()
        if (not multi or dist.get_rank() == 0) and \
                getattr(self, 'global_step', 0) >= getattr(self, 'lambda_update_delay_steps', 0):
            self.update_lambda(episode_cost)
        if multi:
            dist.broadcast(self.log_lambda.data, src=0)

    # ---- saferlhf.py:483-675 ---------------------------------------------------------------------------
    def rl_step(self, inference_batch, training_batch) -> dict[str, Any]:
        self._lambda_step()
        lens = ops.as_device_lens(training_batch['response_lens'], training_batch['log_probs'].device)
        old_log_probs = training_batch['log_probs']
        ref_log_probs = training_batch['ref_log_probs']
        reward, cost = training_batch['reward'], training_batch['cost']
        input_ids = inference_batch['input_ids']
        # the reference scores under an all-ones mask truncated to the narrowest of the three tensors (:513-520)
        new_size = min(training_batch['response_mask'].size(-1), training_batch['reward_values'].size(-1),
                       training_batch['cost_values'].size(-1))
        sequence_mask = torch.ones((old_log_probs.size(0), new_size), dtype=torch.bool, device=old_log_probs.device)
        old_reward_values = training_batch['reward_values'][:, :new_size]
        old_cost_values = training_batch['cost_values'][:, :new_size]

        old_rewards, reward_advantages, reward_returns, reward_stats = ops.kl_rewards_and_gae(
            reward, old_log_probs, ref_log_probs, old_reward_values, sequence_mask, 0, self.kl_coeff,
            self.clip_range_score, self.gamma, self.gae_lambda, mode=self.mode)
        old_costs, cost_advantages, cost_returns, cost_stats = ops.kl_rewards_and_gae(
            cost, old_log_probs, ref_log_probs, old_cost_values, sequence_mask, 0, -self.kl_coeff,
            self.clip_range_score, self.gamma, self.gae_lambda, mode=self.mode)

        batch = self.infer_batch(inference_batch)
        if self.fused_lm_head:
            log_probs = self._tail_log_probs(self.actor_model, batch, lens, input_ids, use_cache=False)
            actor_loss = self.actor_loss_fn_with_cost(log_probs, old_log_probs, reward_advantages, cost_advantages,
                                                      sequence_mask)
        else:
            logits = self._actor_logits(self.actor_model, batch, lens, use_cache=False)
            if ops._FUSED_ACTOR and ops._single_pass_ok(logits) and new_size == lens.bound == old_log_probs.size(-1):
                # actor_loss_fn_with_cost (:432-451) is the clipped-ratio loss on the Lagrangian mix of the two advantages:
                # the same single-pass actor node as the PPO trainers (K1f: log-probs, d loss / d log-prob, gradient tile)
                multiplier = self.log_lambda.exp().item()
                advantages = (reward_advantages - multiplier * cost_advantages) / (1.0 + multiplier)
                actor_loss, _, _ = ops.tail_actor_loss(logits, input_ids, lens, old_log_probs, advantages, sequence_mask,
                                                       self.clip_range_ratio, mode=self.mode)
            else:  # short rows / fp16: K1 over the response tails -> K5; backward K1b
                log_probs = ops.response_tail_log_probs(logits, input_ids, lens, mode=self.mode)
                actor_loss = self.actor_loss_fn_with_cost(log_probs, old_log_probs, reward_advantages, cost_advantages,
                                                          sequence_mask)
        self.actor_model.backward(actor_loss)
        self.actor_model.step()

        losses, row_means = [], []
        for engine, old_values, returns in ((self.reward_critic_model, old_reward_values, reward_returns),
                                            (self.cost_critic_model, old_cost_values, cost_returns)):
            raw = engine(**self.infer_batch(inference_batch)).scores.squeeze(dim=-1)[:, :-1]
            values = _tail_values(raw, lens)
            loss, row_mean = ops.critic_loss(values, old_values, returns, sequence_mask, self.clip_range_value,
                                             mode=self.mode, return_row_mean=True)
            engine.backward(loss)
            engine.step()
            losses.append(loss)
            row_means.append(row_mean)

        with torch.no_grad():  # 19 AVG + 1 MAX all-reduces and a barrier in the reference (:618-651): ONE collective
            r = ops.ppo_pack_metrics(reward_stats, reward, row_means[0], actor_loss, losses[0])
            c = ops.ppo_pack_metrics(cost_stats, cost, row_means[1], actor_loss, losses[1])
            stats = all_reduce_packed(torch.cat([r[:10], c[1:7], c[10:11]]), max_lanes=(9, 16))
            v = stats.tolist()
        ops.raise_for_status(v[16], stats.device)  # lane 16 = device status word
        out = dict(zip(METRIC_KEYS, v[:16]))
        out['train/log_lambda'] = self.log_lambda.item()
        out['train/lambda'] = self.log_lambda.exp().item()
        out['train/actor_lr'] = self.actor_model.optimizer.param_groups[0]['lr']
        out['train/reward_critic_lr'] = self.reward_critic_model.optimizer.param_groups[0]['lr']
        out['train/cost_critic_lr'] = self.cost_critic_model.optimizer.param_groups[0]['lr']
        # scalars only in the returned dict (it goes straight to Logger.log); per-token tensors for tests / debugging:
        self.last_rl_tensors = {'old_rewards': old_rewards, 'old_costs': old_costs, 'advantages': reward_advantages,
                                'cost_advantages': cost_advantages, 'returns': reward_returns, 'cost_returns': cost_returns}
        return out
