"""TEST INFRASTRUCTURE ONLY -- the cost-model loss of the reference restated on ATen, for the CPU goldens and as the
GPU tests' reference on ATen CUDA:

  * `cm_loss`: CMTrainer.loss (trainers/text_to_text/cost_model.py:97-144) after the model forward, op for op, so
    that dtypes, rounding points and autograd's chain are the reference's;
  * `cm_loss_f64`: the same formula in float64 from the values, as an independent cross-check;
  * `rm_loss`: the RM pairwise loss (trainers/text_to_text/rm.py:111-124, restated by the audio / video trainers)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F


def cm_loss(end_scores: torch.Tensor, better, worse, scale_coeff, regularization) -> dict:
    """end_scores (2B,) or (2B, 1), higher-cost rows first; better / worse: the meta_info lists."""
    h, lo = end_scores.squeeze(-1).chunk(2)
    sb = torch.tensor(better).to(h.device)
    sw = torch.tensor(worse).to(lo.device)
    cost = -F.logsigmoid(h * sb).mean() - F.logsigmoid(lo * sw).mean()
    origin = -F.logsigmoid(h - lo).mean()  # built before scale * cost: autograd's order of accumulation follows it
    loss = scale_coeff * cost + origin
    if regularization > 0.0:
        loss = loss + regularization * torch.stack([lo, h]).square().mean()
    return {'loss': loss, 'accuracy': (h > lo).float().mean(), 'higher_end_reward': h, 'lower_end_reward': lo}


def rm_loss(end_scores: torch.Tensor, regularization) -> dict:
    h, lo = end_scores.squeeze(-1).chunk(2)
    loss = -F.logsigmoid(h - lo).mean()
    if regularization > 0.0:
        loss = loss + regularization * torch.stack([lo, h]).square().mean()
    return {'loss': loss, 'accuracy': (h > lo).float().mean()}


def _log_sigmoid(x):
    return np.minimum(x, 0.0) - np.log1p(np.exp(-np.abs(x)))


def cm_loss_f64(end_scores, better, worse, scale_coeff, regularization):
    """(loss, d loss / d end_scores) in float64."""
    x = end_scores.detach().double().reshape(-1).cpu().numpy()
    B = x.size // 2
    h, lo = x[:B], x[B:]
    sb, sw = np.asarray(better, dtype=np.float64), np.asarray(worse, dtype=np.float64)
    sig = lambda z: 1.0 / (1.0 + np.exp(-z))
    loss = scale_coeff * (-_log_sigmoid(h * sb).mean() - _log_sigmoid(lo * sw).mean()) - _log_sigmoid(h - lo).mean()
    gh = -scale_coeff * sig(-h * sb) * sb / B - sig(lo - h) / B
    gl = -scale_coeff * sig(-lo * sw) * sw / B + sig(lo - h) / B
    if regularization > 0.0:
        loss += regularization * np.square(x).mean()
        gh = gh + regularization * h / B
        gl = gl + regularization * lo / B
    return loss, np.concatenate([gh, gl])
