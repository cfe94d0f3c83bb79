"""The DPO objective options (ops.DpoObjective) restated in the reference's own style: eager ATen ops on 0-dim tensors
of the log-prob dtype, pair by pair (trainers/text_to_text/dpo.py:150-203).  With every option at its default this is
oracle/ref_port.py's dpo_loss, op for op.  K2's objective variant (aa_dpo_loss_obj) restates these rounding points."""
from __future__ import annotations

import torch
import torch.nn.functional as F


def pair_loss(a, b, beta: float, loss_type: str, eps: float):
    """The per-pair loss of a = pc - rc, b = pr - rr (IPO: of the count-normalised sums)."""
    c = 1 / (2 * beta)
    if loss_type in ('sigmoid', 'robust'):
        z = beta * (a - b)
        if eps == 0:
            return -F.logsigmoid(z)
        m1 = -F.logsigmoid(z) * (1 - eps)
        m2 = F.logsigmoid(-z) * eps
        return m1 - m2 if loss_type == 'sigmoid' else (m1 + m2) / (1 - 2 * eps)
    if loss_type == 'hinge':
        return torch.relu(1 - beta * (a - b))
    if loss_type == 'ipo':
        return ((a - b) - c) ** 2
    if loss_type == 'sppo_hard':
        return (a - c) ** 2 + (b + c) ** 2
    if loss_type == 'nca_pair':
        za, zb = beta * a, beta * b
        return -F.logsigmoid(za) - 0.5 * F.logsigmoid(-za) - 0.5 * F.logsigmoid(-zb)
    if loss_type == 'apo_zero':
        return (1 - torch.sigmoid(beta * a)) + torch.sigmoid(beta * b)
    if loss_type == 'apo_down':
        return torch.sigmoid(beta * a) + (1 - torch.sigmoid(beta * (a - b)))
    raise ValueError(loss_type)


def dpo_loss(policy_lp, ref_lp, scale_coeff: float, input_ids=None, skip_identical_pairs: bool = False,
             loss_type: str = 'sigmoid', label_smoothing: float = 0.0, rpo_alpha: float = 0.0,
             reference_free: bool = False, response_lens=None):
    """-> the dict of oracle/ref_port.py's dpo_loss, plus 'nll_loss' when rpo_alpha > 0.  ref_lp is not read when
    reference_free (the reference sums are 0).  response_lens: R_i per row (the counts are R_i - 1)."""
    better, worse = policy_lp.chunk(2, dim=0)
    B = better.size(0)
    if not reference_free:
        ref_better, ref_worse = ref_lp.chunk(2, dim=0)
    if skip_identical_pairs:
        ids_better, ids_worse = input_ids.chunk(2, dim=0)
    per_pair, r_better, r_worse, chosen, n_chosen = [], [], [], [], 0
    for i in range(B):
        if skip_identical_pairs and bool(torch.all(torch.eq(ids_better[i], ids_worse[i]))):
            continue
        pc = better[i, :].sum(dim=-1)
        pr = worse[i, :].sum(dim=-1)
        zero = torch.zeros((), dtype=policy_lp.dtype, device=policy_lp.device)
        rc = zero if reference_free else ref_better[i, :].sum(dim=-1)
        rr = zero if reference_free else ref_worse[i, :].sum(dim=-1)
        ratio_c = pc - rc
        ratio_r = pr - rr
        if loss_type == 'ipo':
            nc, nr = int(response_lens[i]) - 1, int(response_lens[B + i]) - 1
            per_pair.append(pair_loss(pc / nc - rc / nc, pr / nr - rr / nr, scale_coeff, loss_type, label_smoothing))
        else:
            per_pair.append(pair_loss(ratio_c, ratio_r, scale_coeff, loss_type, label_smoothing))
        r_better.append(scale_coeff * ratio_c.detach())
        r_worse.append(scale_coeff * ratio_r.detach())
        if rpo_alpha > 0:
            chosen.append(pc)
            n_chosen += int(response_lens[i]) - 1
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
