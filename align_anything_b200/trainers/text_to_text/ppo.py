"""PPO rollout scoring and rl_step on the H100 kernels -- mirror of
align_anything/trainers/text_to_text/ppo.py (reward_model_step :224-242, rollout :244-289,
actor_loss_fn :291-307, rl_step :309-398, get_advantages_and_returns :487-508, critic_loss_fn
:510-526, add_kl_divergence_regularization :528-547).

Generation itself (`model.generate`), engine construction and the data loaders are out of scope and stay
in the reference; the methods below read the same attributes from `self`:
    self.actor_model, self.actor_reference_model, self.reward_model, self.reward_critic_model,
    self.kl_coeff, self.clip_range_ratio, self.clip_range_score, self.clip_range_value,
    self.gamma, self.gae_lambda, self.tokenizer, self.reward_tokenizer
"""
from __future__ import annotations

import copy
import math
from typing import Any

import torch

from ... import ops
from ...utils.multi_process import all_reduce_packed, fused_allreduce

__all__ = ['PPOTrainer']

METRIC_KEYS = ('train/actor_loss', 'train/reward_critic_loss', 'train/reward', 'train/reward_with_kl_penalty',
               'train/reward_advantage', 'train/reward_return', 'train/reward_value', 'train/kl_divergence',
               'train/mean_generated_length', 'train/max_generated_length')


def lm_head_of(model) -> torch.Tensor:
    """The lm_head weight of an engine (or bare module) for the fused lm_head path; ops.lm_head_weight refuses the heads
    that path would get wrong (ZeRO-3 placeholder, bias, soft-capping / logit scaling)."""
    return ops.lm_head_weight(getattr(model, 'module', model))


def hidden_log_probs(model, batch, input_ids, start, weight, chunk_rows, mode, return_entropy=False, entropy_grad=False,
                     **kw):
    """`gather_log_probabilities(model(**batch).logits[:, :-1], input_ids[:, 1:])[:, start:]` from the model's last
    hidden states: the lm_head runs on one position inside the model and on the scored rows in ops, no logits tile.
    return_entropy: -> (log_probs, fp32 policy entropy of the same rows) from the same kernel (differentiable with
    entropy_grad: its gradient enters K6b's epilogue)."""
    out = model(**batch, output_hidden_states=True, logits_to_keep=1, **kw)
    return ops.dense_log_probs_from_hidden(out.hidden_states[-1], weight, input_ids, start, chunk_rows=chunk_rows,
                                           mode=mode, return_entropy=return_entropy, entropy_grad=entropy_grad)


def switch_of(tr, name: str):
    """A trainer switch in effect: `cfgs.train_cfgs.<name>` when the config sets it (a yaml recipe), otherwise the
    class attribute `<name>`."""
    tc = getattr(getattr(tr, 'cfgs', None), 'train_cfgs', None)
    v = getattr(tc, name, None) if tc is not None else None
    return getattr(tr, name, None) if v is None else v


def entropy_coeff_of(tr) -> float:
    """The entropy-bonus coefficient in effect (switch_of `entropy_coeff`)."""
    return float(switch_of(tr, 'entropy_coeff'))


def kl_estimator_of(tr) -> str:
    """The KL estimator of the reward penalty in effect (switch_of `kl_estimator`; None: 'k1', the reference's)."""
    name = switch_of(tr, 'kl_estimator') or 'k1'
    ops.kl_estimator_code(name)
    return name


def kl_controller_of(tr) -> tuple[float, float] | None:
    """(kl_target, kl_horizon) of the adaptive KL coefficient in effect, or None when `kl_target` is unset (a fixed
    kl_coeff, the reference's).  Both, and kl_coeff, must be finite and > 0; anything else raises ValueError here."""
    target = switch_of(tr, 'kl_target')
    if target is None:
        return None
    horizon = switch_of(tr, 'kl_horizon')
    for name, v in (('kl_target', target), ('kl_horizon', horizon), ('kl_coeff', tr.kl_coeff)):
        if isinstance(v, bool) or not isinstance(v, (int, float)) or not (math.isfinite(v) and v > 0):
            raise ValueError(f'the adaptive KL coefficient needs a finite {name} > 0, got {v!r}')
    return float(target), float(horizon)


def adaptive_kl_coeff(kl_coeff: float, kl: float, n: int, target: float, horizon: float) -> float:
    """One update of the adaptive KL controller (Ziegler et al. 2019, TRL's AdaptiveKLController):
    e = clip(kl / target - 1, -0.2, 0.2), kl_coeff * (1 + e * n / horizon); n = samples in the step."""
    e = min(max(kl / target - 1.0, -0.2), 0.2)
    return kl_coeff * (1.0 + e * n / horizon)


def kl_loss_of(tr) -> tuple[float, str] | None:
    """(kl_loss_coeff, kl_loss_estimator) of the KL term in the actor loss, or None when `kl_loss_estimator` is unset
    (no term).  The term is on iff the estimator is set (switch_of each): then it must be one of ops.KL_ESTIMATORS and
    kl_loss_coeff finite and > 0.  A non-zero kl_loss_coeff without an estimator is refused rather than ignored.  Every
    error raises ValueError here, before anything runs."""
    est = switch_of(tr, 'kl_loss_estimator')
    c = switch_of(tr, 'kl_loss_coeff')
    if est is None:
        if c is not None and c != 0:
            raise ValueError(f'kl_loss_coeff={c!r} without kl_loss_estimator: the KL term in the PPO actor loss is '
                             f'turned on by kl_loss_estimator (k1, k2 or k3)')
        return None
    ops.kl_estimator_code(est)
    if isinstance(c, bool) or not isinstance(c, (int, float)) or not (math.isfinite(c) and c > 0):
        raise ValueError(f'kl_loss_estimator={est!r} needs a finite kl_loss_coeff > 0, got {c!r}')
    return float(c), est


def kl_rewards(tr, reward, log_probs, ref_log_probs, values, sequence_mask, start):
    """K4 of an rl_step under the trainer's KL switches: the KL-shaped rewards, GAE and the metric row sums
    (ops.kl_rewards_and_gae with kl_estimator_of(tr); checks the KL switches before the launch)."""
    kl_loss_of(tr)
    kl_controller_of(tr)
    est = kl_estimator_of(tr)
    return ops.kl_rewards_and_gae(reward, log_probs, ref_log_probs, values, sequence_mask, start, tr.kl_coeff,
                                  tr.clip_range_score, tr.gamma, tr.gae_lambda, mode=tr.mode,
                                  **({} if est == 'k1' else {'kl_estimator': est}))


def whiten_advantages_of(tr) -> bool:
    """Whether rollout() whitens the advantages (switch_of `whiten_advantages`; unset: False).  Anything but a bool
    raises ValueError."""
    v = switch_of(tr, 'whiten_advantages')
    if v is None:
        return False
    if not isinstance(v, bool):
        raise ValueError(f'whiten_advantages must be True or False, got {v!r}')
    return v


# the tensors a whitening rollout() stores in each training batch, in rl_step's order
ROLLOUT_ADVANTAGE_KEYS = ('old_rewards', 'advantages', 'returns', 'row_stats')


def micro_batch_advantages(tr, training_batch, sequence_mask, start, returns=None):
    """The KL-shaped rewards, advantages, returns and metric row sums of one micro-batch: K4 (kl_rewards) and, with
    `returns(old_rewards, sequence_mask, start, row_stats) -> (advantages, returns)`, K4r (Multi-PPO's estimators)."""
    old_rewards, advantages, ret, row_stats = kl_rewards(
        tr, training_batch['reward'], training_batch['log_probs'], training_batch['ref_log_probs'],
        training_batch['reward_values'], sequence_mask, start)
    if returns is not None:
        advantages, ret = returns(old_rewards, sequence_mask, start, row_stats)
    return old_rewards, advantages, ret, row_stats


def step_advantages(tr, training_batch, sequence_mask, start, returns=None):
    """rl_step's (old_rewards, advantages, returns, row_stats): micro_batch_advantages, or with whiten_advantages on
    the tensors rollout() stored (whiten_rollout), with no launch; the KL switches are checked first either way."""
    if not whiten_advantages_of(tr):
        return micro_batch_advantages(tr, training_batch, sequence_mask, start, returns)
    kl_loss_of(tr)
    kl_controller_of(tr)
    kl_estimator_of(tr)
    return tuple(training_batch[k] for k in ROLLOUT_ADVANTAGE_KEYS)


def whiten_rollout(tr, training_batches, sequence_masks, starts, returns=None) -> None:
    """rollout()'s advantages under whiten_advantages: K4 (+ K4r through `returns`) for each micro-batch at the
    kl_coeff in effect now, then ONE ops.whiten_advantages over the whole rollout with the actor-loss masks
    `sequence_mask[:, start:]`.  Stores ROLLOUT_ADVANTAGE_KEYS in each training batch for rl_step; row_stats keeps the
    pre-whitening advantage row means (train/reward_advantage), and the returns stay unwhitened."""
    for training, mask, start in zip(training_batches, sequence_masks, starts):
        training.update(zip(ROLLOUT_ADVANTAGE_KEYS, micro_batch_advantages(tr, training, mask, start, returns)))
    whitened = ops.whiten_advantages([t['advantages'] for t in training_batches],
                                     [m[:, s:] for m, s in zip(sequence_masks, starts)])
    for training, adv in zip(training_batches, whitened):
        training['advantages'] = adv


OBJECTIVE_KEYS = ('clip_range_ratio_low', 'clip_range_ratio_high', 'dual_clip_ratio', 'loss_agg_mode',
                  'policy_loss_mode', 'clip_cov_ratio', 'clip_cov_lb', 'clip_cov_ub', 'kl_cov_ratio', 'ppo_kl_coef',
                  'sapo_temperature_pos', 'sapo_temperature_neg')


def actor_objective_of(tr) -> ops.ActorObjective | None:
    """The actor objective in effect (switch_of each of OBJECTIVE_KEYS), or None when every key is unset: the
    reference's objective and today's launches.  A bad value raises ValueError here, before anything runs."""
    fields = {k: switch_of(tr, k) for k in OBJECTIVE_KEYS}
    fields = {k: v for k, v in fields.items() if v is not None}
    return ops.ActorObjective(**fields) if fields else None


def cov_seed_of(tr, objective) -> int:
    """The hash seed of this loss call under Clip-Cov (ops.cov_hash_seed of `train_cfgs.seed` (0 when absent), the
    data-parallel rank and tr's count of earlier Clip-Cov calls, which this advances); 0 for any other objective."""
    if objective is None or objective.policy_loss_mode != 'clip_cov':
        return 0
    tc = getattr(getattr(tr, 'cfgs', None), 'train_cfgs', None)
    seed = getattr(tc, 'seed', None)
    dist = torch.distributed
    rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
    n = getattr(tr, 'cov_calls', 0)
    tr.cov_calls = n + 1
    return ops.cov_hash_seed(int(seed or 0), rank, n)


def objective_kwargs(tr) -> dict:
    """The ops keywords of the actor objective switches: empty when they are all at their defaults (today's call)."""
    kw = {}
    objective = actor_objective_of(tr)
    if objective is not None:
        kw['objective'] = objective
        if objective.policy_loss_mode in ops.COV_MODES:
            kw['cov_seed'] = cov_seed_of(tr, objective)
    if tr.log_clip_fraction:
        kw['return_clip_fraction'] = True
    return kw


def actor_loss_node(tr, batch, input_ids, old_log_probs, advantages, mask, *, start=0, head=None, lens=None,
                    ref_log_probs=None):
    """The actor loss of an rl_step -> (loss, the loss for ppo_pack_metrics, the masked-mean entropy or None, the
    fp32[2] clip fractions or None, agg(KL) of the KL loss term or None, the Clip-Cov / KL-Cov selected share or
    None).  The rows scored are those of the text
    layout, `[start:]` of every row, or with `lens` the response tails of the multimodal layout (`old_log_probs`,
    `ref_log_probs`, `advantages` and `mask` already (B, W)).
    `head`: the lm_head weight of the text layout's fused path.  With an entropy bonus (entropy_coeff_of(tr) != 0) the loss is
    actor_loss - c * masked_mean(H, mask)  over the same rows and mask (a token mean under loss_agg_mode 'token-mean'),
    the second output stays the actor loss without it.  The actor objective switches (actor_objective_of) reach K5 and
    K1f; `tr.log_clip_fraction` asks K5 for the clip fractions.  With a KL loss term (kl_loss_of) the loss gains
    + kl_loss_coeff * agg(KL(lp, ref_log_probs), mask)  aggregated like the objective; the second output stays without
    it.  A function rather than a method, so that the grafted rl_step of the reference's classes finds it without
    being grafted itself."""
    coeff = entropy_coeff_of(tr)
    kw = objective_kwargs(tr)
    cf = kl = share = None
    if lens is None:
        old_log_probs, mask = old_log_probs[:, start:], mask[:, start:]
    term = kl_loss_of(tr)
    if term is not None:
        kw.update(ref_log_probs=ref_log_probs if lens is not None else ref_log_probs[:, start:], kl_loss_coeff=term[0],
                  kl_loss_estimator=term[1])
    if tr.fused_lm_head:  # K6 + K6b + backward GEMMs for the log-probs, then K5
        # with a bonus K6's entropy variant; K6b adds the entropy's gradient in its epilogue
        ent_kw = {'return_entropy': coeff != 0.0, 'entropy_grad': coeff != 0.0, 'use_cache': False}
        if lens is None:
            log_probs = hidden_log_probs(tr.actor_model, batch, input_ids, start, head, tr.lm_head_chunk_rows, tr.mode,
                                         **ent_kw)
        else:
            log_probs = tr._tail_log_probs(tr.actor_model, batch, lens, input_ids, **ent_kw)
        if coeff != 0.0:
            log_probs, ent = log_probs
        # ops.actor_loss, with the actor loss without the KL term beside the loss
        loss, loss32, kl, cf, share = ops._actor_loss(
            log_probs, old_log_probs, advantages, mask, tr.clip_range_ratio, tr.mode, kw.get('objective'),
            kw.get('return_clip_fraction', False), kw.get('ref_log_probs'), kw.get('kl_loss_coeff', 0.0),
            kw.get('kl_loss_estimator', 'k3'), kw.get('cov_seed', 0))
        if coeff == 0.0:
            return loss, loss32, None, cf, kl, share
        token = 'objective' in kw and kw['objective'].token_mean
        h_mean = (ops.token_mean if token else ops.masked_mean)(ent, mask)
        return loss - coeff * h_mean, loss32, h_mean.detach(), cf, kl, share
    # One autograd node (K1f): log-probs, d loss / d log-prob and the gradient tile in a single pass over the scored
    # rows.  The text layout reads only the rows `[start:]` the reference keeps after scoring every position
    # (:338-346); the prompt rows of the tile are written as zeros by the same kernel.
    if coeff != 0.0:
        kw['entropy_coeff'] = coeff
    if lens is None:
        logits = tr.actor_model(**batch, use_cache=False).logits
        out = ops.dense_actor_loss(logits, input_ids, start, old_log_probs, advantages, mask, tr.clip_range_ratio,
                                   mode=tr.mode, **kw)
    else:
        logits = tr._actor_logits(tr.actor_model, batch, lens, use_cache=False)
        out = ops.tail_actor_loss(logits, input_ids, lens, old_log_probs, advantages, mask, tr.clip_range_ratio,
                                  mode=tr.mode, **kw)
    if kw.get('return_clip_fraction'):
        out, cf = out[:-1], out[-1]
    if 'cov_seed' in kw:
        out, share = out[:-1], out[-1]
    if term is not None:
        out, kl = out[:-1], out[-1]
    return out[0], out[2], (out[3] if coeff != 0.0 else None), cf, kl, share


def ppo_metrics(tr, row_stats, reward, value_row_mean, actor_loss, critic_loss, tensors, *, entropy=None, mask=None,
                entropy_mean=None, clip_frac=None, kl_loss=None, cov_share=None) -> dict[str, Any]:
    """The metric dict of a PPO rl_step from ONE packed collective and ONE host sync (reference: 10 all-reduces, a
    barrier and 12 .item()).  ppo_pack_metrics packs the ten metrics of METRIC_KEYS, the device status word (lane 10,
    MAX-reduced with lane 9) and a spare lane 11 (0).  Optional AVG lanes follow, each read back under its key:
      * `entropy` (the rollout policy's, with `mask`; both over the scored rows) takes lane 11 as train/entropy, reduced
        like train/kl_divergence: summed over each row's masked tokens, averaged over rows and ranks;
      * `entropy_mean`, the entropy term of the bonus (train/actor_entropy);
      * `clip_frac`, K5's clip fraction (train/actor_clip_fraction) and with dual-clip its dual-clip fraction
        (train/actor_dual_clip_fraction);
      * `kl_loss`, agg(KL) of the KL loss term without its coefficient (train/actor_kl_loss);
      * `cov_share`, the share of counted tokens Clip-Cov / KL-Cov selected (train/actor_cov_fraction).
    Sets `tr.last_rl_tensors = tensors` (per-token tensors stay out of the dict: the reference hands it to Logger.log,
    which takes scalars only).  With `kl_target` set (kl_controller_of) the step's train/kl_coeff goes into the dict and
    tr.kl_coeff takes the adaptive controller's update from the step's (all-reduced) train/kl_divergence and its
    sample count over all ranks: every rank computes the same coefficient, from the values already read here."""
    with torch.no_grad():
        # an optional lane is filled in before the one packed all-reduce, so the NVLink reduction fused into
        # ppo_pack_metrics (which reduces the vector as it writes it) gives way to all_reduce_packed
        extra = entropy is not None or entropy_mean is not None or clip_frac is not None or kl_loss is not None or \
            cov_share is not None
        fused = fused_allreduce(row_stats.device) if not extra else None
        stats = ops.ppo_pack_metrics(row_stats, reward, value_row_mean, actor_loss, critic_loss,
                                     coll=fused.next((9, 10)) if fused is not None else None)
        lanes = {}
        if entropy is not None:
            lanes['train/entropy'] = (entropy * mask).sum(dim=-1).mean().reshape(1)
        if entropy_mean is not None:
            lanes['train/actor_entropy'] = entropy_mean.detach().float().reshape(1)
        if clip_frac is not None:
            lanes['train/actor_clip_fraction'] = clip_frac[:1]
            objective = actor_objective_of(tr)
            if objective is not None and objective.dual_clip_ratio is not None:
                lanes['train/actor_dual_clip_fraction'] = clip_frac[1:2]
        if kl_loss is not None:
            lanes['train/actor_kl_loss'] = kl_loss.detach().float().reshape(1)
        if cov_share is not None:
            lanes['train/actor_cov_fraction'] = cov_share.reshape(1)
        first = 11 if entropy is not None else 12  # the entropy takes the spare lane 11
        if lanes:
            stats = torch.cat([stats[:first], *lanes.values()])
        if fused is None:
            stats = all_reduce_packed(stats, max_lanes=(9, 10))
        v = stats.tolist()
    ops.raise_for_status(v[10], stats.device)  # the device status word (MAX over ranks): raise like the reference
    out = dict(zip(METRIC_KEYS, v[:10]))
    out.update(zip(lanes, v[first:]))
    controller = kl_controller_of(tr)
    if controller is not None:
        ranks = torch.distributed.get_world_size() if torch.distributed.is_available() and \
            torch.distributed.is_initialized() else 1
        out['train/kl_coeff'] = float(tr.kl_coeff)
        tr.kl_coeff = adaptive_kl_coeff(float(tr.kl_coeff), out['train/kl_divergence'], row_stats.size(0) * ranks,
                                        *controller)
    out['train/actor_lr'] = tr.actor_model.optimizer.param_groups[0]['lr']
    out['train/reward_critic_lr'] = tr.reward_critic_model.optimizer.param_groups[0]['lr']
    tr.last_rl_tensors = tensors
    return out


class PPOTrainer:
    mode = None  # None -> 'faithful'
    # Opt-in: no (B, L, V) logits tile.  The models are asked for their last hidden states (`output_hidden_states=True,
    # logits_to_keep=1`); rollout scoring (no gradient) runs K6 once per model, the actor's rl_step K6 + K6b + the two
    # backward GEMMs and then K5 (ops.dense_log_probs_from_hidden -> ops.actor_loss).  ptx_step keeps its logits.
    fused_lm_head = False
    lm_head_chunk_rows = None
    # Opt-in: `train/entropy`, the policy entropy of the rollout, taken from the pass that scores its log-probs (K1's
    # or K6's entropy variant: one more FMA per logit, no extra read) and reduced in the step's one packed collective
    log_entropy = False
    # Entropy bonus: the actor minimises  actor_loss - entropy_coeff * masked_mean(H, mask)  (H: the policy entropy of
    # rl_step's own pass, its gradient written by the log-prob kernels).  `cfgs.train_cfgs.entropy_coeff` overrides it
    # when set; 0 leaves the step unchanged.  train/actor_loss stays the loss without the bonus, train/actor_entropy
    # carries the entropy term.
    entropy_coeff = 0.0
    # The actor objective (ops.ActorObjective): clip-higher (clip_range_ratio_low / _high; None = clip_range_ratio),
    # dual-clip (dual_clip_ratio c > 1, None = off) and loss_agg_mode ('seq-mean-token-mean', the reference's
    # masked_mean, or 'token-mean').  `cfgs.train_cfgs.<key>` overrides each when set; all None is the reference's
    # objective and today's launches.
    clip_range_ratio_low = None
    clip_range_ratio_high = None
    dual_clip_ratio = None
    loss_agg_mode = None
    # Opt-in: train/actor_clip_fraction (and train/actor_dual_clip_fraction with dual-clip) from K5, reduced in the
    # step's one packed all-reduce
    log_clip_fraction = False
    # The KL penalty of the rewards, -kl_coeff * KL per token.  kl_estimator: 'k1' (lp - ref, the reference's; None),
    # 'k2' (0.5 * (lp - ref) ** 2) or 'k3' (exp(ref - lp) - (ref - lp) - 1); train/kl_divergence stays the k1 sum.
    # kl_target (None = a fixed kl_coeff): the adaptive KL coefficient of Ziegler et al. (2019), updated after every
    # rl_step from train/kl_divergence with horizon kl_horizon (adaptive_kl_coeff); train/kl_coeff reports the
    # coefficient each step used.  `cfgs.train_cfgs.<key>` overrides each when set.
    kl_estimator = None
    kl_target = None
    kl_horizon = 10000
    # The KL term in the actor loss (verl's use_kl_loss): kl_loss_estimator 'k1' / 'k2' / 'k3' (None = no term) turns
    # it on, and the actor minimises  actor_loss + kl_loss_coeff * agg(KL(lp, ref), mask)  with the objective's
    # aggregation.  kl_loss_coeff must then be finite and > 0; without an estimator anything but 0 raises
    # (kl_loss_of).  Independent of the reward penalty: kl_coeff 0 moves the KL from the reward into the loss.
    # train/actor_loss stays the clipped objective, train/actor_kl_loss reports agg(KL).
    kl_loss_coeff = 0.0
    kl_loss_estimator = None
    # Clip-Cov / KL-Cov (Cui et al. 2025; verl's policy_loss.loss_mode, see ops.ActorObjective): policy_loss_mode
    # 'clip_cov' or 'kl_cov' (None = 'vanilla'), and their keys clip_cov_ratio, clip_cov_lb, clip_cov_ub, kl_cov_ratio
    # and ppo_kl_coef (None = verl's defaults).  The selection runs on the device, local to each micro-batch's loss;
    # train/actor_cov_fraction reports the selected share.  `cfgs.train_cfgs.<key>` overrides each when set.
    policy_loss_mode = None
    clip_cov_ratio = None
    clip_cov_lb = None
    clip_cov_ub = None
    kl_cov_ratio = None
    ppo_kl_coef = None
    # CISPO / SAPO (TRL's loss_type 'cispo' / 'sapo', see ops.ActorObjective): policy_loss_mode 'cispo' truncates the
    # importance weight at 1 + clip_range_ratio_high (None = clip_range_ratio) and stops its gradient; 'sapo' gates the
    # ratio with a sigmoid of temperature sapo_temperature_pos (A > 0) or sapo_temperature_neg (None = 1.0 / 1.05).  Both
    # keep K1f's single pass.  `cfgs.train_cfgs.<key>` overrides each when set.
    sapo_temperature_pos = None
    sapo_temperature_neg = None
    # Advantage whitening (TRL's / verl's masked_whiten): rollout() forms every micro-batch's advantages with the
    # kl_coeff in effect then (K4, and K4r for Multi-PPO's other estimators) and whitens them with ONE mean and std over
    # the whole rollout's actor-loss mask, on every data-parallel rank (ops.whiten_advantages); rl_step reuses them (all
    # update_iters).  The returns stay unwhitened, train/reward_advantage stays the pre-whitening row mean.  A bool;
    # `cfgs.train_cfgs.whiten_advantages` overrides it when set; False leaves rollout and rl_step unchanged.
    whiten_advantages = False
    # the class attributes above that the grafted methods read: patch.install() copies them onto the reference's classes
    SWITCHES = ('mode', 'fused_lm_head', 'lm_head_chunk_rows', 'log_entropy', 'entropy_coeff', 'clip_range_ratio_low',
                'clip_range_ratio_high', 'dual_clip_ratio', 'loss_agg_mode', 'log_clip_fraction', 'kl_estimator',
                'kl_target', 'kl_horizon', 'kl_loss_coeff', 'kl_loss_estimator', 'whiten_advantages', 'policy_loss_mode',
                'clip_cov_ratio', 'clip_cov_lb', 'clip_cov_ub', 'kl_cov_ratio', 'ppo_kl_coef', 'sapo_temperature_pos',
                'sapo_temperature_neg')

    def __init__(self, cfgs=None, actor_model=None, actor_reference_model=None, reward_model=None,
                 reward_critic_model=None, tokenizer=None, reward_tokenizer=None, *, kl_coeff=0.02,
                 clip_range_ratio=0.2, clip_range_score=50.0, clip_range_value=5.0, gamma=1.0,
                 gae_lambda=0.95) -> None:
        self.cfgs = cfgs
        self.actor_model = actor_model
        self.actor_reference_model = actor_reference_model
        self.reward_model = reward_model
        self.reward_critic_model = reward_critic_model
        self.tokenizer = tokenizer
        self.reward_tokenizer = reward_tokenizer if reward_tokenizer is not None else tokenizer
        tc = getattr(cfgs, 'train_cfgs', None) if cfgs is not None else None

        def pick(name, default):  # trainers/text_to_text/ppo.py:87-93 reads these from cfgs.train_cfgs
            v = getattr(tc, name, None) if tc is not None else None
            return default if v is None else v

        self.kl_coeff = pick('kl_coeff', kl_coeff)
        self.clip_range_ratio = pick('clip_range_ratio', clip_range_ratio)
        self.clip_range_score = pick('clip_range_score', clip_range_score)
        self.clip_range_value = pick('clip_range_value', clip_range_value)
        self.gamma = pick('gamma', gamma)
        self.gae_lambda = pick('gae_lambda', gae_lambda)
        self.ptx_coeff = pick('ptx_coeff', 16.0)
        self.infer_batch = lambda batch: {k: v for k, v in batch.items() if k != 'meta_info'}
        self.reward_infer_batch = self.infer_batch

    # ---- the four loss-path functions, drop-in signatures -----------------------------------
    def actor_loss_fn(self, log_probs, old_log_probs, advantages, mask) -> torch.Tensor:
        """trainers/text_to_text/ppo.py:291-307."""
        return ops.actor_loss(log_probs, old_log_probs, advantages, mask, self.clip_range_ratio, mode=self.mode)

    def critic_loss_fn(self, values, old_values, returns, mask) -> torch.Tensor:
        """trainers/text_to_text/ppo.py:510-526."""
        return ops.critic_loss(values, old_values, returns, mask, self.clip_range_value, mode=self.mode)

    def add_kl_divergence_regularization(self, reward, log_probs, ref_log_probs, sequence_mask) -> torch.Tensor:
        """trainers/text_to_text/ppo.py:528-547 (K4; rl_step below fuses it with the GAE scan)."""
        W = log_probs.size(-1)
        dummy = torch.zeros((log_probs.size(0), W), dtype=torch.float32, device=log_probs.device)
        old_rewards, _, _, _ = kl_rewards(self, reward, log_probs, ref_log_probs, dummy, sequence_mask, W - 1)
        return old_rewards

    def get_advantages_and_returns(self, values, rewards, sequence_mask, start):
        """trainers/text_to_text/ppo.py:487-508."""
        adv, ret, _ = ops.gae_from_rewards(values, rewards, sequence_mask, start, self.gamma, self.gae_lambda,
                                           mode=self.mode)
        return adv.detach(), ret

    # ---- trainers/text_to_text/ppo.py:224-242 -----------------------------------------------
    def reward_model_step(self, actor_batch) -> dict[str, Any]:
        reward_batch = copy.copy(actor_batch)
        if self.reward_tokenizer is not self.tokenizer:
            raise NotImplementedError('re-tokenisation for a different reward tokenizer is host-side text '
                                      'processing (utils/tools.py batch_retokenize) and out of scope')
        reward_batch['reward'] = self.reward_model(**self.reward_infer_batch(reward_batch)).end_scores.squeeze(dim=-1)
        scores = self.reward_critic_model(**self.reward_infer_batch(actor_batch)).scores
        reward_batch['reward_values'] = scores.squeeze(dim=-1)[:, :-1]
        return reward_batch

    # ---- trainers/text_to_text/ppo.py:209-222 and base/rl_trainer.py:274-286 -------------------
    def actor_step(self, mini_prompt_only_batch) -> dict[str, Any]:
        """Generation + attention mask.  patch.install() keeps the reference's own method for the text trainer (it is
        already free of host syncs); this one serves the stand-alone mirror."""
        infer_batch = self.infer_batch(mini_prompt_only_batch)
        actor_batch = copy.deepcopy(infer_batch)
        sequences = self.actor_model.module.generate(**infer_batch, generation_config=self.generation_config,
                                                     synced_gpus=True, do_sample=True)
        actor_batch['input_ids'] = sequences
        actor_batch['attention_mask'] = sequences.not_equal(self.tokenizer.pad_token_id)
        return actor_batch

    def set_train(self, mode: bool = True) -> None:
        for engine in (self.actor_model, self.reward_critic_model):
            fn = getattr(engine, 'train' if mode else 'eval', None)
            if callable(fn):
                fn()

    # ---- trainers/text_to_text/ppo.py:244-289 -------------------------------------------------
    @torch.no_grad()
    def rollout(self, prompt_only_batch):
        """Micro-batched generation + scoring -> (inference_batches, training_batches), the lists the reference's
        train() loop zips into rl_step (:430-447); with whiten_advantages, the whitened advantages (whiten_rollout)."""
        whiten = whiten_advantages_of(self)
        self.set_train(mode=False)
        total = prompt_only_batch['input_ids'].size(0)
        micro = int(self.cfgs.train_cfgs.per_device_train_batch_size)
        inference_batches, training_batches = [], []
        for i in range(0, total, micro):
            mini_batch = {key: prompt_only_batch[key][i:i + micro] for key in prompt_only_batch}
            actor_batch = self.actor_step(mini_batch)
            inference, training = self.score_rollout(actor_batch, mini_batch['input_ids'].size(-1))
            mini_batch['input_ids'] = inference['input_ids']
            mini_batch['attention_mask'] = inference['attention_mask']
            inference_batches.append(mini_batch)
            training_batches.append(training)
        if whiten:
            whiten_rollout(self, training_batches, [b['attention_mask'][:, 1:] for b in inference_batches],
                           [t['prompt_idx'] for t in training_batches])
        self.set_train()
        return inference_batches, training_batches

    # ---- scoring half of rollout(), trainers/text_to_text/ppo.py:262-283 ---------------------
    @torch.no_grad()
    def score_rollout(self, actor_batch, prompt_len: int) -> tuple[dict, dict]:
        """Everything rollout() does after generation for one mini-batch: reward / critic scoring and
        the actor / reference log-probs of every next token."""
        if self.fused_lm_head:  # refuse a head the fused path would get wrong before anything runs
            heads = (lm_head_of(self.actor_model), lm_head_of(self.actor_reference_model))
        reward_batch = self.reward_model_step(actor_batch)
        ids = actor_batch['input_ids']
        entropy = None
        if self.fused_lm_head:  # every position, prompt and pad included: the width the tile path stores
            log_probs = hidden_log_probs(self.actor_model, actor_batch, ids, 0, heads[0], self.lm_head_chunk_rows,
                                         self.mode, return_entropy=self.log_entropy)
            if self.log_entropy:
                log_probs, entropy = log_probs
            ref_log_probs = hidden_log_probs(self.actor_reference_model, actor_batch, ids, 0, heads[1],
                                             self.lm_head_chunk_rows, self.mode)
        else:
            logits = self.actor_model(**actor_batch).logits
            ref_logits = self.actor_reference_model(**actor_batch).logits
            if self.log_entropy:
                log_probs, entropy = ops.gather_log_probabilities_with_entropy(logits[:, :-1], ids[:, 1:], mode=self.mode)
            else:
                log_probs = ops.gather_log_probabilities(logits[:, :-1], ids[:, 1:], mode=self.mode)
            ref_log_probs = ops.gather_log_probabilities(ref_logits[:, :-1], ids[:, 1:], mode=self.mode)
        training = {
            'prompt_idx': prompt_len - 1,
            'log_probs': log_probs,
            'ref_log_probs': ref_log_probs,
            'reward': reward_batch['reward'],
            'reward_values': reward_batch['reward_values'],
        }
        if entropy is not None:
            training['entropy'] = entropy  # (B, L - 1) fp32, the actor's, aligned with log_probs
        inference = {'input_ids': reward_batch['input_ids'], 'attention_mask': actor_batch['attention_mask']}
        return inference, training

    # ---- trainers/text_to_text/ppo.py:400-408 -----------------------------------------------
    def ptx_step(self, ptx_batch) -> dict[str, Any]:
        """PTX (pre-training mix) term: the HF causal-LM loss, taken from K1 instead of `outputs.loss`."""
        from ...utils.multi_process import get_all_reduce_mean

        batch = dict(self.infer_batch(ptx_batch))
        labels = batch.pop('labels')
        logits = self.actor_model(**batch).logits
        # `ptx_coeff * ptx_loss` (:405): the gradient tile comes out of the single pass already multiplied
        scaled_loss, ptx_loss = ops.causal_lm_loss_scaled(logits, labels, self.ptx_coeff)
        self.actor_model.backward(scaled_loss)
        self.actor_model.step()
        ptx_loss = get_all_reduce_mean(ptx_loss.detach())
        return {'train/ptx_loss': ptx_loss.item()}

    # ---- trainers/text_to_text/ppo.py:309-398 -----------------------------------------------
    def rl_step(self, inference_batch, training_batch, returns=None) -> dict[str, Any]:
        """returns: None for K4's GAE advantages and returns, or `returns(old_rewards, sequence_mask, start, row_stats)
        -> (advantages, returns)`, which also rewrites their metric lanes of row_stats (Multi-PPO's K4r).  With
        whiten_advantages, the rollout's stored tensors instead (step_advantages)."""
        old_log_probs = training_batch['log_probs']
        ref_log_probs = training_batch['ref_log_probs']
        reward = training_batch['reward']
        old_reward_values = training_batch['reward_values']
        start = training_batch['prompt_idx']
        input_ids = inference_batch['input_ids']
        sequence_mask = inference_batch['attention_mask'][:, 1:]
        head = lm_head_of(self.actor_model) if self.fused_lm_head else None  # refusals before any launch

        old_rewards, reward_advantages, reward_returns, row_stats = step_advantages(
            self, training_batch, sequence_mask, start, returns)

        actor_loss, actor_loss32, entropy_mean, clip_frac, kl_loss, cov_share = actor_loss_node(
            self, inference_batch, input_ids, old_log_probs, reward_advantages, sequence_mask, start=start, head=head,
            ref_log_probs=ref_log_probs)
        self.actor_model.backward(actor_loss)
        self.actor_model.step()

        reward_values = self.reward_critic_model(**inference_batch).scores
        reward_values = reward_values.squeeze(dim=-1)[:, :-1]
        reward_critic_loss, value_row_mean = ops.critic_loss(
            reward_values[:, start:], old_reward_values[:, start:], reward_returns, sequence_mask[:, start:],
            self.clip_range_value, mode=self.mode, return_row_mean=True)
        self.reward_critic_model.backward(reward_critic_loss)
        self.reward_critic_model.step()

        return ppo_metrics(
            self, row_stats, reward, value_row_mean, actor_loss32, reward_critic_loss,
            {'old_rewards': old_rewards, 'advantages': reward_advantages, 'returns': reward_returns},
            entropy=training_batch['entropy'][:, start:] if self.log_entropy else None, mask=sequence_mask[:, start:],
            entropy_mean=entropy_mean, clip_frac=clip_frac, kl_loss=kl_loss, cov_share=cov_share)
