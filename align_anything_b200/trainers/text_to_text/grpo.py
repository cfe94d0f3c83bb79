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
from .ppo import cov_seed_of, entropy_coeff_of, hidden_log_probs, lm_head_of, switch_of

__all__ = ['GRPOTrainer']

GRPO_OBJECTIVE_KEYS = ('clip_range_ratio', 'clip_range_ratio_low', 'clip_range_ratio_high', 'dual_clip_ratio',
                       'loss_agg_mode', 'kl_estimator', 'importance_sampling_level', 'top_entropy_quantile',
                       'policy_loss_mode', 'clip_cov_ratio', 'clip_cov_lb', 'clip_cov_ub', 'kl_cov_ratio', 'ppo_kl_coef',
                       'sapo_temperature_pos', 'sapo_temperature_neg')


def num_iterations_of(tr) -> int:
    """The updates per rollout in effect (switch_of `num_iterations`).  The reference sizes its LR schedule by
    `train_cfgs.update_iters`, so a different `num_iterations` > 1 is refused here, before anything runs."""
    mu = switch_of(tr, 'num_iterations')
    if isinstance(mu, bool) or int(mu) != mu or int(mu) < 1:
        raise ValueError(f'num_iterations must be an integer >= 1, got {mu!r}')
    mu = int(mu)
    tc = getattr(getattr(tr, 'cfgs', None), 'train_cfgs', None)
    ui = getattr(tc, 'update_iters', None) if tc is not None else None
    if mu > 1 and ui is not None and int(ui) != mu:
        raise ValueError(f'num_iterations={mu} differs from train_cfgs.update_iters={ui}, which sizes the LR schedule')
    return mu


def grpo_objective_of(tr) -> ops.GrpoObjective | None:
    """The GRPO objective in effect (switch_of each of GRPO_OBJECTIVE_KEYS), or None for the reference's loss and
    today's launches: one update per rollout and every objective field at its default.  A bad value raises
    ValueError here, before anything runs."""
    fields = {k: switch_of(tr, k) for k in GRPO_OBJECTIVE_KEYS}
    fields = {k: v for k, v in fields.items() if v is not None}
    obj = ops.GrpoObjective(**fields)
    return None if obj.is_default and num_iterations_of(tr) == 1 else obj


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
    # GRPO's objective (ops.GrpoObjective).  num_iterations = mu updates per rollout (DeepSeekMath's GRPO; TRL's
    # `num_iterations`): the advantages and the reference log-probs are computed once, the first update's detached
    # log-probs are the old log-probs of the ratio exp(lp - old) for updates 2..mu.  The ratio is clipped to
    # [1 - clip_range_ratio_low, 1 + clip_range_ratio_high] (None: clip_range_ratio); dual_clip_ratio c > 1 (None =
    # off); loss_agg_mode 'token-mean' (the reference's), 'seq-mean-token-mean' or 'seq-mean-token-sum-norm' (Dr. GRPO,
    # with scale_rewards False: advantages r - group mean).  `cfgs.train_cfgs.<key>` overrides each when set; the
    # defaults are the reference's single-update step and today's launches.
    num_iterations = 1
    clip_range_ratio = 0.2
    clip_range_ratio_low = None
    clip_range_ratio_high = None
    dual_clip_ratio = None
    loss_agg_mode = 'token-mean'
    scale_rewards = True
    # The per-token KL of the loss -(s - beta * KL): 'k3' (the reference's exp(ref - lp) - (ref - lp) - 1), 'k1'
    # (lp - ref) or 'k2' (0.5 * (lp - ref) ** 2); ops.KL_ESTIMATORS.  `cfgs.train_cfgs.kl_estimator` overrides it.
    kl_estimator = 'k3'
    # GRPO's importance ratio: 'token' (exp(lp - old) per token, the default) or 'sequence' (GSPO, Zheng et al. 2025;
    # TRL's importance_sampling_level): one ratio per completion, exp of the mean of its tokens' log-ratios, clipped in
    # place of the token ratios.  It acts from update 2 on, so it wants num_iterations > 1; the first update (ratio 1)
    # runs the token-level launches.  `cfgs.train_cfgs.importance_sampling_level` overrides it.
    importance_sampling_level = 'token'
    # High-entropy token masking (Wang et al. 2025, "Beyond the 80/20 Rule"; TRL's top_entropy_quantile): rho in [0, 1].
    # Each update, only the top-rho fraction of the completion tokens by policy entropy (over every data-parallel rank)
    # keep the policy-gradient term; the others carry the KL term alone.  1 (the default) masks nothing and runs
    # today's launches; rho < 1 takes the composed path with the exact entropy quantile (ops.entropy_quantile_threshold)
    # on both the tile and the fused_lm_head paths.  `cfgs.train_cfgs.top_entropy_quantile` overrides it.
    top_entropy_quantile = 1.0
    # Clip-Cov / KL-Cov (Cui et al. 2025; verl's policy_loss.loss_mode, see ops.ActorObjective / ops.GrpoObjective):
    # policy_loss_mode 'clip_cov' or 'kl_cov' (None = 'vanilla') and their keys (None = verl's defaults), token level
    # only.  Each update selects over its own completion tokens on the device, on the composed path (tile and
    # fused_lm_head); train/actor_cov_fraction reports the selected share, the mean over the updates.  On the first
    # update (ratio 1) KL-Cov changes nothing.  `cfgs.train_cfgs.<key>` overrides each when set.
    policy_loss_mode = None
    clip_cov_ratio = None
    clip_cov_lb = None
    clip_cov_ub = None
    kl_cov_ratio = None
    ppo_kl_coef = None
    # CISPO / SAPO (TRL's GRPO loss_type 'cispo' / 'sapo', see ops.GrpoObjective): policy_loss_mode 'cispo' or 'sapo',
    # token level only, on K1f's single pass whenever it runs; SAPO's temperatures sapo_temperature_pos / _neg (None =
    # 1.0 / 1.05).  `cfgs.train_cfgs.<key>` overrides each when set.
    sapo_temperature_pos = None
    sapo_temperature_neg = None
    # Opt-in: train/actor_clip_fraction (and train/actor_dual_clip_fraction with dual-clip), the mean over the updates,
    # in the step's one packed all-reduce
    log_clip_fraction = False
    # the class attributes above that the grafted methods read: patch.install() copies them onto the reference's class
    SWITCHES = ('mode', 'fused_lm_head', 'lm_head_chunk_rows', 'log_entropy', 'entropy_coeff', 'num_iterations',
                'clip_range_ratio', 'clip_range_ratio_low', 'clip_range_ratio_high', 'dual_clip_ratio', 'loss_agg_mode',
                'scale_rewards', 'log_clip_fraction', 'kl_estimator', 'importance_sampling_level',
                'top_entropy_quantile', 'policy_loss_mode', 'clip_cov_ratio', 'clip_cov_lb', 'clip_cov_ub',
                'kl_cov_ratio', 'ppo_kl_coef', 'sapo_temperature_pos', 'sapo_temperature_neg')

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
        mu = num_iterations_of(self)
        objective = grpo_objective_of(self)
        log_cf = bool(switch_of(self, 'log_clip_fraction'))
        if self.fused_lm_head:  # refuse a head the fused path would get wrong before anything runs
            for model in (self.actor_reference_model, self.actor_model):
                lm_head_of(model)
        advantages = ops.group_advantages(rewards, self.num_generations,
                                          **({} if switch_of(self, 'scale_rewards') else {'scale': False}))  # (B * G, 1)
        attention_mask = (sequences != self.tokenizer.pad_token_id).long()
        logits_to_keep = sequences.size(1) - prompt_length
        # the frozen reference model is scored FIRST (the reference scores it second, :284-288): with its per-token
        # log-probs at hand the policy's log-probs, the loss and d loss / d logits come out of ONE pass over the policy
        # tile.  It is scored once per rollout, however many updates follow.
        with torch.no_grad():
            ref_per_token_logps = self._get_per_token_logps(self.actor_reference_model, sequences, attention_mask,
                                                            logits_to_keep)
        kw = {}
        if objective is not None:
            kw['objective'] = objective
        if log_cf:
            kw['return_clip_fraction'] = True
        old = None  # updates 2..mu: the first update's log-probs
        plains, entropies, entropy_means, fracs, shares = [], [], [], [], []
        cov = objective is not None and objective.policy_loss_mode in ops.COV_MODES
        for _ in range(mu):
            if old is not None:
                kw['old_per_token_logps'] = old
            if cov:
                kw['cov_seed'] = cov_seed_of(self, objective)
            loss, plain, entropy, entropy_mean, cf, lp, row_end, share = policy_update(
                self, sequences, attention_mask, logits_to_keep, ref_per_token_logps, advantages, kw)
            if old is None and mu > 1:
                old = lp
            plains.append(plain)
            entropies.append(entropy)
            entropy_means.append(entropy_mean)
            fracs.append(cf)
            shares.append(share)
        with torch.no_grad():
            # train/loss is GRPO's loss without the bonus, the mean over the updates; lane 2 = device status word, MAX
            packed = [torch.stack([_mean(plains), rewards.float().mean()]), ops.status_lane(loss.device)]
            lanes = {}  # the optional AVG lanes after those three, read back under their keys
            if self.log_entropy:  # token mean over the completion mask (tokens up to and including the first eos)
                mask = torch.arange(logits_to_keep, device=row_end.device) < row_end.unsqueeze(1)
                lanes['train/entropy'] = _mean([((e * mask).sum() / mask.sum()).reshape(1) for e in entropies])
            if entropy_means[0] is not None:
                lanes['train/actor_entropy'] = _mean([m.reshape(1) for m in entropy_means])
            if log_cf:  # the clip fraction (and the dual-clip fraction)
                cf = _mean(fracs)
                lanes['train/actor_clip_fraction'] = cf[:1]
                if objective is not None and objective.dual_clip_ratio is not None:
                    lanes['train/actor_dual_clip_fraction'] = cf[1:2]
            if cov:  # the share of completion tokens Clip-Cov / KL-Cov selected
                lanes['train/actor_cov_fraction'] = _mean(shares)
            # ONE collective, ONE sync per rollout (reference: 2 + 2 per update)
            v = all_reduce_packed(torch.cat([*packed, *lanes.values()]), max_lanes=(2,)).tolist()
        ops.raise_for_status(v[2], loss.device)
        return {'train/loss': v[0], 'train/reward': v[1], **dict(zip(lanes, v[3:]))}

    def train_step(self, prompt_batch: dict) -> dict[str, float]:
        """trainers/text_to_text/grpo.py:258-318; generate_completions / compute_rewards come from the reference."""
        device = next(self.actor_model.module.parameters()).device
        prompt_batch = {k: v.to(device) for k, v in prompt_batch.items()}
        prompt_length = prompt_batch['input_ids'].size(1)
        sequences = self.generate_completions(prompt_batch)
        self.actor_model.train()
        rewards = self.compute_rewards(sequences, prompt_length)
        return self.step_from_rollout(sequences, prompt_length, rewards)


def _mean(xs):
    """The mean over the updates (one update: the value itself, bit for bit)."""
    return xs[0] if len(xs) == 1 else torch.stack(xs).mean(0)


def policy_update(tr, sequences, attention_mask, logits_to_keep, ref_per_token_logps, advantages, kw):
    """One policy pass, backward and optimizer step of the trainer `tr` on the rollout -> (loss, GRPO's loss without
    the bonus (fp32, detached), entropy or None, entropy term or None, clip fractions or None, detached log-probs,
    row_end, the Clip-Cov / KL-Cov selected share or None).  A function rather than a method, so that the grafted step_from_rollout of the reference's class finds
    it without being grafted itself."""
    entropy = cf = share = None
    coeff = entropy_coeff_of(tr)
    entropy_mean = plain = None  # with the bonus: its entropy term and GRPO's loss without it
    if tr.fused_lm_head:  # the composed path: K1f needs a logits tile
        topent = ops._top_entropy(kw.get('objective'))  # the mask's threshold is taken from this pass's entropy
        want_entropy = tr.log_entropy or coeff != 0.0 or topent
        per_token_logps = tr._get_per_token_logps(tr.actor_model, sequences, attention_mask, logits_to_keep,
                                                    return_entropy=want_entropy, entropy_grad=coeff != 0.0)
        if want_entropy:
            per_token_logps, entropy = per_token_logps
        scored = ops.grpo_loss(per_token_logps, ref_per_token_logps, advantages,
                               sequences[:, -logits_to_keep:], tr.tokenizer.eos_token_id, tr.beta,
                               mode=tr.mode, **kw, **({'entropy': entropy} if topent else {}))
        loss, row_end = scored[0], scored[1]
        if kw.get('return_clip_fraction'):
            cf = scored[-1]
        if 'cov_seed' in kw:
            share = scored[2]
        lp = per_token_logps.detach()
        if coeff != 0.0:  # K6b adds the entropy's gradient in its epilogue
            entropy_mean = ops._completion_mean(entropy, row_end)
            plain, loss = loss, loss - coeff * entropy_mean
            entropy, entropy_mean = entropy.detach(), entropy_mean.detach()
        if not tr.log_entropy and coeff == 0.0:
            entropy = None  # taken for the mask alone
    else:
        logits = tr.actor_model(input_ids=sequences, attention_mask=attention_mask).logits
        scored = ops.grpo_loss_from_logits(logits, sequences, logits_to_keep, ref_per_token_logps, advantages,
                                           tr.tokenizer.eos_token_id, tr.beta, mode=tr.mode,
                                           return_entropy=tr.log_entropy,
                                           **({'entropy_coeff': coeff} if coeff != 0.0 else {}), **kw)
        if kw.get('return_clip_fraction'):
            scored, cf = scored[:-1], scored[-1]
        if 'cov_seed' in kw:
            scored, share = scored[:-1], scored[-1]
        loss, lp, row_end = scored[0], scored[1], scored[2]
        if coeff != 0.0:
            entropy_mean, plain = scored[3], scored[4]
        if tr.log_entropy:
            entropy = scored[-1]
    tr.actor_model.zero_grad()
    tr.actor_model.backward(loss)
    tr.actor_model.step()
    plain = (loss if plain is None else plain).detach().float()
    return loss, plain, entropy, entropy_mean, cf, lp, row_end, share
