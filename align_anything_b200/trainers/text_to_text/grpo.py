"""GRPO loss / step on the H100 kernels -- mirror of align_anything/trainers/text_to_text/grpo.py
(GRPOTrainer._get_per_token_logps :199-210, the arithmetic of .train_step :268-318).  Generation
(`generate_completions`) and reward computation (`compute_rewards`: a reward-model forward) are out of
scope and stay in the reference; the methods below read self.actor_model, self.actor_reference_model,
self.tokenizer.{pad_token_id, eos_token_id}, self.beta, self.num_generations like the reference."""
from __future__ import annotations

from typing import Any

import torch

from ... import ops
from ...utils.multi_process import all_reduce_packed

__all__ = ['GRPOTrainer']


class GRPOTrainer:
    mode = None

    def __init__(self, cfgs=None, actor_model=None, actor_reference_model=None, tokenizer=None, *, beta=None,
                 num_generations=None) -> None:
        self.cfgs = cfgs
        self.actor_model = actor_model
        self.actor_reference_model = actor_reference_model
        self.tokenizer = tokenizer
        tc = getattr(cfgs, 'train_cfgs', None) if cfgs is not None else None
        self.beta = beta if beta is not None else getattr(tc, 'beta', 0.04)
        self.num_generations = num_generations if num_generations is not None else getattr(tc, 'num_generations', 4)

    # -- trainers/text_to_text/grpo.py:199-210 ---------------------------------------------------
    def _get_per_token_logps(self, model, input_ids, attention_mask, logits_to_keep):
        """Log-probs of the last `logits_to_keep` tokens: one K1 launch on the model's logits (the reference
        slices, log-softmaxes the whole (B, K, V) tile and gathers)."""
        logits = model(input_ids=input_ids, attention_mask=attention_mask).logits
        return ops.tail_token_log_probs(logits, input_ids, logits_to_keep, mode=self.mode)

    # -- the arithmetic of train_step, trainers/text_to_text/grpo.py:268-318 ---------------------------
    def step_from_rollout(self, sequences: torch.Tensor, prompt_length: int, rewards: torch.Tensor) -> dict[str, Any]:
        advantages = ops.group_advantages(rewards, self.num_generations)  # (B * G, 1)
        attention_mask = (sequences != self.tokenizer.pad_token_id).long()
        logits_to_keep = sequences.size(1) - prompt_length
        # the frozen reference model is scored FIRST (the reference scores it second, :284-288): with its per-token
        # log-probs at hand the policy's log-probs, the loss and d loss / d logits come out of ONE pass over the policy tile
        with torch.no_grad():
            ref_per_token_logps = self._get_per_token_logps(self.actor_reference_model, sequences, attention_mask,
                                                            logits_to_keep)
        logits = self.actor_model(input_ids=sequences, attention_mask=attention_mask).logits
        loss, _, _ = ops.grpo_loss_from_logits(logits, sequences, logits_to_keep, ref_per_token_logps, advantages,
                                               self.tokenizer.eos_token_id, self.beta, mode=self.mode)
        self.actor_model.zero_grad()
        self.actor_model.backward(loss)
        self.actor_model.step()
        with torch.no_grad():
            stats = torch.cat([torch.stack([loss.detach().float(), rewards.float().mean()]), ops.status_lane(loss.device)])
            # ONE collective, ONE sync (reference: 2 + 2); lane 2 = device status word, MAX over ranks
            loss_val, avg_reward, status = all_reduce_packed(stats, max_lanes=(2,)).tolist()
        ops.raise_for_status(status, loss.device)
        return {'train/loss': loss_val, 'train/reward': avg_reward}

    def train_step(self, prompt_batch: dict) -> dict[str, float]:
        """trainers/text_to_text/grpo.py:258-318; generate_completions / compute_rewards come from the reference."""
        device = next(self.actor_model.module.parameters()).device
        prompt_batch = {k: v.to(device) for k, v in prompt_batch.items()}
        prompt_length = prompt_batch['input_ids'].size(1)
        sequences = self.generate_completions(prompt_batch)
        self.actor_model.train()
        rewards = self.compute_rewards(sequences, prompt_length)
        return self.step_from_rollout(sequences, prompt_length, rewards)
