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
from .ppo import entropy_coeff_of, hidden_log_probs, lm_head_of

__all__ = ['GRPOTrainer']


class GRPOTrainer:
    mode = None
    # Opt-in: no (B * G, L, V) logits tile.  Both models are asked for their last hidden states (`output_hidden_states=
    # True, logits_to_keep=1`); the reference model's completion rows run through K6, the policy's through K6 + K6b + the
    # two backward GEMMs (ops.dense_log_probs_from_hidden), then the GRPO loss kernel (ops.grpo_loss).
    fused_lm_head = False
    lm_head_chunk_rows = None
    # Opt-in: `train/entropy`, the policy entropy of the completions (token mean over the completion mask, as the loss),
    # from the policy pass of the step (K1f's phase A, or K6 with fused_lm_head), in the step's one packed collective
    log_entropy = False
    # Entropy bonus: the policy minimises  loss - entropy_coeff * (H * mask).sum() / mask.sum()  over the completion
    # mask (H: the step's own policy pass).  `cfgs.train_cfgs.entropy_coeff` overrides it when set; 0 leaves the step
    # unchanged.  train/loss stays GRPO's loss, train/actor_entropy carries the entropy term.
    entropy_coeff = 0.0

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
    def _get_per_token_logps(self, model, input_ids, attention_mask, logits_to_keep, return_entropy=False,
                             entropy_grad=False):
        """Log-probs of the last `logits_to_keep` tokens: one K1 launch on the model's logits (the reference
        slices, log-softmaxes the whole (B, K, V) tile and gathers).  With fused_lm_head: from the hidden states
        (return_entropy: and the fp32 entropy of the same rows, from the same kernel; differentiable with entropy_grad)."""
        if self.fused_lm_head:
            return hidden_log_probs(model, {'input_ids': input_ids, 'attention_mask': attention_mask}, input_ids,
                                    input_ids.size(1) - 1 - logits_to_keep, lm_head_of(model), self.lm_head_chunk_rows,
                                    self.mode, return_entropy=return_entropy, entropy_grad=entropy_grad)
        logits = model(input_ids=input_ids, attention_mask=attention_mask).logits
        return ops.tail_token_log_probs(logits, input_ids, logits_to_keep, mode=self.mode)

    # -- the arithmetic of train_step, trainers/text_to_text/grpo.py:268-318 ---------------------------
    def step_from_rollout(self, sequences: torch.Tensor, prompt_length: int, rewards: torch.Tensor) -> dict[str, Any]:
        if self.fused_lm_head:  # refuse a head the fused path would get wrong before anything runs
            for model in (self.actor_reference_model, self.actor_model):
                lm_head_of(model)
        advantages = ops.group_advantages(rewards, self.num_generations)  # (B * G, 1)
        attention_mask = (sequences != self.tokenizer.pad_token_id).long()
        logits_to_keep = sequences.size(1) - prompt_length
        # the frozen reference model is scored FIRST (the reference scores it second, :284-288): with its per-token
        # log-probs at hand the policy's log-probs, the loss and d loss / d logits come out of ONE pass over the policy tile
        with torch.no_grad():
            ref_per_token_logps = self._get_per_token_logps(self.actor_reference_model, sequences, attention_mask,
                                                            logits_to_keep)
        entropy = None
        coeff = entropy_coeff_of(self)
        entropy_mean = plain = None  # with the bonus: its entropy term and GRPO's loss without it
        if self.fused_lm_head:  # the composed path: K1f needs a logits tile
            want_entropy = self.log_entropy or coeff != 0.0
            per_token_logps = self._get_per_token_logps(self.actor_model, sequences, attention_mask, logits_to_keep,
                                                        return_entropy=want_entropy, entropy_grad=coeff != 0.0)
            if want_entropy:
                per_token_logps, entropy = per_token_logps
            loss, row_end = ops.grpo_loss(per_token_logps, ref_per_token_logps, advantages,
                                          sequences[:, -logits_to_keep:], self.tokenizer.eos_token_id, self.beta,
                                          mode=self.mode)
            if coeff != 0.0:  # K6b adds the entropy's gradient in its epilogue
                entropy_mean = ops._completion_mean(entropy, row_end)
                plain, loss = loss, loss - coeff * entropy_mean
                entropy, entropy_mean = entropy.detach(), entropy_mean.detach()
        else:
            logits = self.actor_model(input_ids=sequences, attention_mask=attention_mask).logits
            scored = ops.grpo_loss_from_logits(logits, sequences, logits_to_keep, ref_per_token_logps, advantages,
                                               self.tokenizer.eos_token_id, self.beta, mode=self.mode,
                                               return_entropy=self.log_entropy,
                                               **({'entropy_coeff': coeff} if coeff != 0.0 else {}))
            loss, row_end = scored[0], scored[2]
            if coeff != 0.0:
                entropy_mean, plain = scored[3], scored[4]
            if self.log_entropy:
                entropy = scored[-1]
        self.actor_model.zero_grad()
        self.actor_model.backward(loss)
        self.actor_model.step()
        with torch.no_grad():
            # train/loss is GRPO's loss, without the bonus
            plain = (loss if plain is None else plain).detach().float()
            lanes = [torch.stack([plain, rewards.float().mean()]), ops.status_lane(loss.device)]
            if self.log_entropy:  # token mean over the completion mask (tokens up to and including the first eos)
                mask = torch.arange(logits_to_keep, device=row_end.device) < row_end.unsqueeze(1)
                lanes.append(((entropy * mask).sum() / mask.sum()).reshape(1))
            if entropy_mean is not None:
                lanes.append(entropy_mean.reshape(1))
            # ONE collective, ONE sync (reference: 2 + 2); lane 2 = device status word, MAX over ranks
            v = all_reduce_packed(torch.cat(lanes), max_lanes=(2,)).tolist()
        ops.raise_for_status(v[2], loss.device)
        out = {'train/loss': v[0], 'train/reward': v[1]}
        if self.log_entropy:
            out['train/entropy'] = v[3]
        if entropy_mean is not None:
            out['train/actor_entropy'] = v[-1]
        return out

    def train_step(self, prompt_batch: dict) -> dict[str, float]:
        """trainers/text_to_text/grpo.py:258-318; generate_completions / compute_rewards come from the reference."""
        device = next(self.actor_model.module.parameters()).device
        prompt_batch = {k: v.to(device) for k, v in prompt_batch.items()}
        prompt_length = prompt_batch['input_ids'].size(1)
        sequences = self.generate_completions(prompt_batch)
        self.actor_model.train()
        rewards = self.compute_rewards(sequences, prompt_length)
        return self.step_from_rollout(sequences, prompt_length, rewards)
