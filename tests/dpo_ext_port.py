"""The further DPO objectives of ops.DpoObjective (f-divergences, exo_pair, discopop, aot, aot_pair) restated in the
reference's own style: eager ATen ops on 0-dim tensors of the log-prob dtype, pair by pair, as TRL's DPOTrainer.dpo_loss
writes them.  With those fields at their defaults this is tests/dpo_objective_port.py's dpo_loss, which it calls.  K2's
extended variant (aa_dpo_loss_ext) restates these rounding points, including the order in which autograd adds the
gradients of a value that reaches the loss along several paths."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from dpo_objective_port import dpo_loss as objective_loss
from dpo_objective_port import pair_loss

EXT_TYPES = ('exo_pair', 'discopop', 'aot', 'aot_pair')


def exp_cap(dtype: torch.dtype) -> float:
    """cap_exp's clamp, floor(log(finfo(dtype).max) * 1e4) / 1e4 in double: 88.7189 for bf16, 88.7228 for fp32,
    11.0898 for fp16."""
    return math.floor(math.log(torch.finfo(dtype).max) * 1e4) / 1e4


def f_divergence(a, b, kind: str, coef: float, cap: float):
    """h of a = pc - rc and b = pr - rr under the f-divergence."""
    if kind == 'alpha_divergence':
        eb = torch.exp(torch.clamp(b * -coef, max=cap))
        ea = torch.exp(torch.clamp(a * -coef, max=cap))
        return (eb - ea) / coef
    h = a - b
    if kind == 'js_divergence':
        return h - (F.softplus(a) - F.softplus(b))
    return h


def h_loss(h, beta: float, loss_type: str, eps: float, tau: float):
    """The per-pair loss of a type that reads z = beta * h."""
    if loss_type == 'exo_pair':
        e = eps if eps > 0 else 1e-3
        z = beta * h
        s1 = torch.sigmoid(z)
        t1 = F.logsigmoid(z) - math.log(1 - e)
        nz = -z
        s2 = torch.sigmoid(nz)
        t2 = F.logsigmoid(nz) - math.log(e)
        return s1 * t1 + s2 * t2
    if loss_type == 'discopop':
        z = beta * h
        m = torch.sigmoid(z / tau)
        lc = -F.logsigmoid(z)
        ec = torch.exp(-z)
        return lc * (1 - m) + ec * m
    return pair_loss(h, torch.zeros((), dtype=h.dtype, device=h.device), beta, loss_type, eps)  # h - 0 == h


def aot_losses(keys1, keys2, beta: float, eps: float):
    """AOT: both key lists sorted ascending (stable: ties to the smaller pair index, NaN last), then the sigmoid loss
    of delta_k = key1_(k) - key2_(k) at each position k."""
    s1, _ = torch.sort(torch.stack(keys1), stable=True)
    s2, _ = torch.sort(torch.stack(keys2), stable=True)
    delta = s1 - s2
    zero = torch.zeros((), dtype=delta.dtype, device=delta.device)
    return [pair_loss(delta[k], zero, beta, 'sigmoid', eps) for k in range(delta.numel())]


def dpo_loss(policy_lp, ref_lp, scale_coeff: float, input_ids=None, skip_identical_pairs: bool = False,
             loss_type: str = 'sigmoid', label_smoothing: float = 0.0, rpo_alpha: float = 0.0,
             reference_free: bool = False, response_lens=None, f_divergence_type: str = 'reverse_kl',
             f_alpha_divergence_coef: float = 1.0, discopop_tau: float = 0.05, cap: float | None = None):
    """-> the dict of tests/dpo_objective_port.py's dpo_loss.  cap: cap_exp's clamp (default: that of the log-prob
    dtype; a float64 restatement of a narrower dtype's run passes that dtype's)."""
    if loss_type not in EXT_TYPES and f_divergence_type == 'reverse_kl':
        return objective_loss(policy_lp, ref_lp, scale_coeff, input_ids, skip_identical_pairs, loss_type,
                              label_smoothing, rpo_alpha, reference_free, response_lens)
    cap = exp_cap(policy_lp.dtype) if cap is None else cap
    better, worse = policy_lp.chunk(2, dim=0)
    B = better.size(0)
    if not reference_free:
        ref_better, ref_worse = ref_lp.chunk(2, dim=0)
    if skip_identical_pairs:
        ids_better, ids_worse = input_ids.chunk(2, dim=0)
    per_pair, keys1, keys2, r_better, r_worse, chosen, n_chosen = [], [], [], [], [], [], 0
    for i in range(B):
        if skip_identical_pairs and bool(torch.all(torch.eq(ids_better[i], ids_worse[i]))):
            continue
        pc = better[i, :].sum(dim=-1)
        pr = worse[i, :].sum(dim=-1)
        zero = torch.zeros((), dtype=policy_lp.dtype, device=policy_lp.device)
        rc = zero if reference_free else ref_better[i, :].sum(dim=-1)
        rr = zero if reference_free else ref_worse[i, :].sum(dim=-1)
        a = pc - rc
        b = pr - rr
        if loss_type == 'aot':
            keys1.append(pc - pr)
            keys2.append(rc - rr)
        elif loss_type == 'aot_pair':
            keys1.append(a)
            keys2.append(b)
        else:
            h = f_divergence(a, b, f_divergence_type, f_alpha_divergence_coef, cap)
            per_pair.append(h_loss(h, scale_coeff, loss_type, label_smoothing, discopop_tau))
        r_better.append(scale_coeff * a.detach())
        r_worse.append(scale_coeff * b.detach())
        if rpo_alpha > 0:
            chosen.append(pc)
            n_chosen += int(response_lens[i]) - 1
    if keys1:
        per_pair = aot_losses(keys1, keys2, scale_coeff, label_smoothing)
    loss = torch.stack(per_pair).mean()
    out = {}
    if rpo_alpha > 0:
        nll = -(torch.stack(chosen).sum() / n_chosen)
        loss = loss + rpo_alpha * nll
        out['nll_loss'] = nll.detach()
    r_better = torch.stack(r_better)
    r_worse = torch.stack(r_worse)
    out.update({
        'loss': loss,
        'reward': r_better + r_worse,
        'better_sample_reward': r_better,
        'worse_sample_reward': r_worse,
        'reward_accuracy': (r_better > r_worse).float().mean(),
        'reward_margin': r_better - r_worse,
    })
    return out
