"""TRL's / verl's masked_whiten(values, mask, shift_mean=True) restated in eager ATen ops over a whole rollout (a list of
micro-batches), with the masked-out positions written as 0 and the rounding points of ops.whiten_advantages:
    n = sum m,  mean = sum m A / n,  var = sum m (A - mean) ** 2 / (n - 1)    (float64, two passes)
    A' = (A - mean) * rsqrt(var + 1e-8) where m, 0 where not m
with mean and rstd rounded once to fp32, the difference and the product in fp32, and A' rounded once to A's dtype."""
from __future__ import annotations

import torch


def statistics(advantages, masks) -> tuple[float, float, float]:
    """(n, mean, var) in float64 over every micro-batch's masked elements (masked_mean / masked_var, unbiased)."""
    m = torch.cat([y.bool().flatten() for y in masks])
    a = torch.cat([x.double().flatten() for x in advantages])[m]  # a masked-out value is never read
    n = float(m.sum())
    mean = a.sum() / n
    var = ((a - mean) ** 2).sum() / (n - 1)
    return float(n), float(mean), float(var)


def whiten(advantages, masks) -> list[torch.Tensor]:
    """The whitened micro-batches, each in its own dtype; n < 2 returns them unchanged (the kernel's status bit)."""
    n, mean, var = statistics(advantages, masks)
    if not n >= 2:
        return [a.clone() for a in advantages]
    mean32 = torch.tensor(mean, dtype=torch.float64).float()
    rstd32 = torch.rsqrt(torch.tensor(var, dtype=torch.float64) + 1e-8).float()
    out = []
    for a, m in zip(advantages, masks):
        w = (a.float() - mean32.to(a.device)) * rstd32.to(a.device)
        out.append(torch.where(m.bool(), w, torch.zeros_like(w)).to(a.dtype))
    return out

