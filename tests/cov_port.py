"""Clip-Cov and KL-Cov (Cui et al. 2025; verl's compute_policy_loss_clip_cov / _kl_cov) restated in eager torch:
the specification of ops.cov_token_selection and of the Cov entry points of K5 and the GRPO loss kernel.

verl draws Clip-Cov's tokens with torch.randperm and KL-Cov's with torch.topk on the host; here both are exact,
deterministic top-k selections: Clip-Cov by the key fmix32(t ^ s) of the flat index t = b * W + j, KL-Cov by cov_t
with ties to the smaller flat index, -0.0 == +0.0 and NaN above +inf.  Runs are therefore not bit-identical to
verl's Clip-Cov draws; the selected counts and the loss expressions are verl's."""
from __future__ import annotations

import torch

U32 = 0xffffffff
DEFAULTS = {'clip_cov_ratio': 2e-4, 'clip_cov_lb': 1.0, 'clip_cov_ub': 5.0, 'kl_cov_ratio': 2e-4, 'ppo_kl_coef': 1.0}


def fmix32(h):
    """MurmurHash3's 32-bit finaliser, on a Python int or an int64 tensor of uint32 values."""
    h = h & U32
    h = h ^ (h >> 16)
    h = (h * 0x85ebca6b) & U32
    h = h ^ (h >> 13)
    h = (h * 0xc2b2ae35) & U32
    return h ^ (h >> 16)


def hash_seed(seed: int, rank: int, call: int) -> int:
    return fmix32(fmix32(fmix32(seed) ^ rank) ^ call)


def means(lp, adv, counted):
    """The fp64 token means of the advantages and the log-probs over the counted tokens, each rounded once to fp32."""
    c = counted.bool()
    n = int(c.sum())
    return (adv.double()[c].sum() / n).float(), (lp.double()[c].sum() / n).float()


def covariance(lp, adv, mean_a, mean_lp):
    """cov_t = (A_t - mean A) * (lp_t - mean lp) in fp32."""
    return (adv.float() - mean_a) * (lp.float() - mean_lp)


def n_select(ratio: float, n: int) -> int:
    """max(int(ratio * N), 1), the product in double as Python forms it; 0 without a counted token."""
    return 0 if n == 0 else max(int(ratio * n), 1)


def order_key(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> int64 keys in torch.topk's order: -0.0 == +0.0, NaN above +inf."""
    x = torch.where(x == 0, torch.zeros_like(x), x.float())
    u = x.view(torch.int32).to(torch.int64) & U32
    k = torch.where(u >= 0x80000000, U32 - u, u | 0x80000000)
    return torch.where(torch.isnan(x), torch.full_like(k, U32), k)


def top_k(keys: torch.Tensor, eligible: torch.Tensor, k: int) -> torch.Tensor:
    """The k eligible entries with the largest keys (ties to the smaller flat index) as a bool mask."""
    flat_keys, flat_e = keys.reshape(-1), eligible.reshape(-1).bool()
    idx = torch.nonzero(flat_e).squeeze(1)
    order = torch.sort(flat_keys[idx], descending=True, stable=True).indices
    out = torch.zeros_like(flat_e)
    out[idx[order[:k]]] = True
    return out.view(keys.shape)


def clipped(lp, old, adv, lo: float, hi: float):
    """The clip-fraction predicate: the clipped branch A * clamp(r) is strictly smaller than A * r."""
    r = torch.exp(lp - old)
    return adv * torch.clamp(r, 1 - lo, 1 + hi) < adv * r


def kl_cov_select(cov, counted, ratio):
    c = counted.bool()
    return top_k(order_key(cov), c, n_select(ratio, int(c.sum())))


def clip_cov_select(cov, counted, is_clipped, ratio, lb, ub, seed):
    c = counted.bool()
    eligible = c & ~is_clipped & (cov > lb) & (cov < ub)
    t = torch.arange(cov.numel(), dtype=torch.int64).view(cov.shape).to(cov.device)
    return top_k(fmix32(t ^ seed), eligible, min(n_select(ratio, int(c.sum())), int(eligible.sum())))


def aggregate(pg, mask, agg: str):
    m = mask.to(pg.dtype)
    if agg == 'token-mean':
        return (pg * m).sum() / m.sum()
    if agg == 'seq-mean-token-mean':
        return ((pg * m).sum(-1) / m.sum(-1)).mean()
    return (pg * m).sum() / (pg.size(0) * pg.size(1))  # 'seq-mean-token-sum-norm'


def pg_losses(mode, lp, old, adv, sel, lo=0.2, hi=0.2, coef=1.0):
    """verl's per-token policy-gradient losses (the negated objective) with the selection `sel` given."""
    ratio = torch.exp(lp - old)
    if mode == 'clip_cov':
        pg = torch.maximum(-adv * ratio, -adv * torch.clamp(ratio, 1 - lo, 1 + hi))
        return torch.where(sel, torch.zeros_like(pg), pg)
    return -adv * ratio + torch.where(sel, coef * (lp - old).abs(), torch.zeros_like(ratio))


def ppo_loss(mode, lp, old, adv, mask, sel, agg='seq-mean-token-mean', lo=0.2, hi=0.2, coef=1.0):
    return aggregate(pg_losses(mode, lp, old, adv, sel, lo, hi, coef), mask, agg)


def grpo_loss(mode, lp, ref, old, adv, mask, sel, beta, agg='token-mean', lo=0.2, hi=0.2, coef=1.0, estimator=None):
    """GRPO under Clip-Cov / KL-Cov: per-token loss pg + beta * k3 KL, `old` None: the ratio is 1.  estimator 'k1' /
    'k2' / 'k3': the KL of kl_objective_port.kl_estimate instead (op for op the kernel's, created before the ratio)."""
    old = lp.detach() if old is None else old
    if estimator is None:
        d = ref - lp
        kl = torch.exp(d) - d - 1
    else:
        from kl_objective_port import kl_estimate
        kl = kl_estimate(lp, ref, estimator)
    return aggregate(pg_losses(mode, lp, old, adv.view(-1, 1), sel, lo, hi, coef) + beta * kl, mask, agg)


def ppo_loss_kl(mode, lp, old, adv, mask, sel, agg, lo, hi, coef, ref, kl_coeff: float, estimator: str):
    """-> (the Cov objective's loss, agg(KL), the total loss + kl_coeff * agg(KL)).  The KL is created before the
    ratio, so autograd adds its gradient to lp after the objective's (kl_loss_port's order, K5's kl_grad)."""
    from kl_loss_port import kl_loss

    kl = kl_loss(lp, ref, mask, estimator, agg)
    loss = ppo_loss(mode, lp, old, adv, mask, sel, agg, lo, hi, coef)
    return loss, kl, loss + kl_coeff * kl


def stable_clip(lp, old, adv, lo: float, hi: float, ulps: int = 4):
    """True where `clipped` cannot change when exp moves by up to `ulps` fp32 ulps.  The kernel's expf and ATen's exp
    may differ by one fp32 ulp; where that ulp lands the dtype-rounded ratio on the other side of a clip bound the
    kernel and the port disagree by design.  The band is narrow (fp32 ulps of exp, not dtype ulps of the ratio): the
    ratios one dtype ulp from a bound stay, and with them the tokens on which the ratio's rounding dtype decides."""
    d = (lp - old).double()
    r = torch.exp(d)
    a = adv.to(torch.promote_types(lp.dtype, adv.dtype))
    out = []
    for f in (1.0 - ulps * 2.0 ** -24, 1.0 + ulps * 2.0 ** -24):
        rr = (r * f).float().to(lp.dtype)
        out.append(a * torch.clamp(rr, 1 - lo, 1 + hi) < a * rr)
    return out[0] == out[1]


def clear_clip_band(lp, old, adv, lo: float, hi: float, ulps: int = 4):
    """`old` with old = lp (ratio exactly 1, never clipped) on every token stable_clip rejects."""
    return torch.where(stable_clip(lp, old, adv, lo, hi, ulps), old, lp)


def state_words(keys, eligible, ratio: float, n: int):
    """The selection's state words of the reference: (E, k, T, need), as aa_cov_select_hi / _lo leave them.  keys: the
    int64 uint32 keys, eligible: bool, both over every token; k = min(max(int(ratio * N), 1), E), 0 when E = 0 (then
    T = 0xffffffff and need = 0); T is the k-th largest eligible key and need how many keys equal to T are taken."""
    ek = keys.reshape(-1)[eligible.reshape(-1).bool()]
    E = int(ek.numel())
    k = min(n_select(ratio, n), E)
    if k == 0:
        return E, 0, U32, 0
    top = torch.sort(ek, descending=True).values[:k]
    T = int(top[-1])
    return E, k, T, int((top == T).sum())
