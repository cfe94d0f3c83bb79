"""FAITHFUL K5 at mask counts a 16-bit dtype cannot hold, without a GPU.

The reference's `masked_mean` (utils/tools.py:460-467) divides `(x * mask).sum(-1)` by `mask.sum(-1)`, an int64 count.
With bf16 / fp16 `x`, ATen casts that count to the dividend's dtype before it divides, in the forward and in
DivBackward: a bf16 row of 257 masked-in tokens is divided by 256, an fp16 row of 2049 by 2048.  Powers of two and
every count up to 256 (bf16) / 2048 (fp16) are exact, so only longer responses see it.

`k5_actor` / `k5_critic` restate K5's seq-mean-token-mean loss, row means and per-token gradient in float64 with the
rounding points of csrc/ppo_math.cuh and csrc/ppo.cu (one 16-bit rounding after every op the reference rounds).  The
operands are exact: lp == old (the ratio is exactly 1, every token a minimum tie), dyadic advantages, values and
returns, so every sum is exact in fp32 in any order and the restatement equals ATen bit for bit.  These tests hold it
to `oracle/ref_port.py` on ATen CPU; tests/test_gpu_faithful_counts.py holds K5 and K1f to it and to the port on ATen
CUDA.  The token-mean aggregation stays out of this file: its divisor is a 0-dim tensor, which ATen CPU reads at its
exact value and ATen CUDA casts to the 16-bit dtype.
"""
from __future__ import annotations

import pytest
import torch

from oracle import ref_port as O

BF, F16 = torch.bfloat16, torch.float16
# counts around the first ones each dtype rounds (bf16: 257, fp16: 2049), ties that round up (259, 263), and counts
# the dtype holds exactly (255, 256, 300, 2047, 2048)
COUNTS = {BF: [255, 256, 257, 259, 263, 300, 511, 513, 1001, 1501, 4095], F16: [2047, 2048, 2049, 2051, 4097]}
CASES = [(dt, n) for dt, ns in COUNTS.items() for n in ns]
CASE_IDS = [f'{str(dt)[6:]}-{n}' for dt, n in CASES]
ACTOR_CLIP, CRITIC_CLIP = 0.2, 0.5


def r(x, dt):
    """One rounding of a float64 value to dt (float64 -> dt directly: for the single + - * / of two dt values this is
    the fp32 operation rounded to dt, since 53 >= 2 * 24 + 2)."""
    return torch.as_tensor(x, dtype=torch.float64).to(dt).double()


def count_divisor(cnt, dt, rounded: bool):
    """What K5 divides by: the count as ATen casts it to the dividend's dtype (rounded), or the exact count."""
    return r(cnt, dt) if rounded else torch.as_tensor(cnt, dtype=torch.float64)


def exact_mask(B, W, n, seed):
    """(B, W) bool with exactly n masked-in tokens per row, at random places."""
    g = torch.Generator().manual_seed(seed)
    order = torch.rand(B, W, generator=g).argsort(1)[:, :n]
    return torch.zeros(B, W, dtype=torch.bool).scatter_(1, order, True)


def actor_operands(B, n, seed, W=None):
    """float64 (lp, adv, mask): lp on the 2^-4 grid in [-4, -1/16], advantages k / 8 with |k| <= 32 (exact in bf16 and
    fp16), n masked-in tokens per row of W = n + 5."""
    W = n + 5 if W is None else W
    g = torch.Generator().manual_seed(seed)
    lp = -torch.randint(1, 65, (B, W), generator=g).double() / 16
    adv = torch.randint(-32, 33, (B, W), generator=g).double() / 8
    return lp, adv, exact_mask(B, W, n, seed + 1)


def critic_operands(B, n, seed, W=None):
    """float64 (values, old values, returns, mask) on the 2^-3 grid, |.| <= 2: value - return and its square are exact
    in both dtypes; some values sit outside old +- clip, some on it."""
    W = n + 5 if W is None else W
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-16, 17, (B, W), generator=g).double() / 8
    old = torch.randint(-16, 17, (B, W), generator=g).double() / 8
    ret = torch.randint(-16, 17, (B, W), generator=g).double() / 8
    t = torch.arange(W)[None, :].expand(B, W)
    x = torch.where(t % 5 == 1, old + CRITIC_CLIP, x)
    return x, old, ret, exact_mask(B, W, n, seed + 1)


def k5_actor(adv, mask, dt, rounded=True):
    """K5's actor loss at lp == old (ratio 1): -> (loss, row means, d loss / d lp), float64 holding dt values.
    g_rs = round(round(-1 / B) / count) is the coefficient of a row's masked sum (actor_row_coeff); on the minimum's
    tie each branch gets round(g_rs / 2), times the advantage, and the two halves add in dt (actor_token)."""
    B = adv.size(0)
    on = mask.double()
    den = count_divisor(on.sum(1), dt, rounded)
    g_rs = r(r(-1.0 / B, dt) / den, dt)[:, None]
    half = r(r(r(0.5 * g_rs, dt) * adv, dt), dt)
    grad = torch.where(mask, r(half + half, dt), 0.0)
    rows = r(r((adv * on).sum(1), dt) / den, dt)
    return -r(rows.sum() / B, dt), rows, grad


def k5_critic(x, old, ret, mask, dt, rounded=True):
    """K5's critic loss: -> (loss, row means, d loss / d values), float64 holding dt values (ppo_loss_kernel,
    ACTOR = false): g_rs = round(round(0.5 / B) / count); maximum's backward sends g_rs, or round(g_rs / 2) to each
    branch on a tie, through d (x - ret)^2 = 2 (x - ret); the clamp passes it only in range."""
    B = x.size(0)
    on = mask.double()
    den = count_divisor(on.sum(1), dt, rounded)
    g_rs = r(r(0.5 / B, dt) / den, dt)[:, None]
    lo, hi = r(old - CRITIC_CLIP, dt), r(old + CRITIC_CLIP, dt)
    vc = torch.minimum(torch.maximum(x, lo), hi)
    d1, d2 = r(x - ret, dt), r(vc - ret, dt)
    l1, l2 = r(d1 * d1, dt), r(d2 * d2, dt)
    in_range = (x >= lo) & (x <= hi)
    half = r(0.5 * g_rs, dt)
    g = torch.where(l1 == l2, half, g_rs)
    g1 = torch.where(l1 >= l2, r(g * 2 * d1, dt), 0.0)
    g2 = torch.where((l2 >= l1) & in_range, r(g * 2 * d2, dt), 0.0)
    grad = torch.where(mask, r(g1 + g2, dt), 0.0)
    rows = r(r((torch.maximum(l1, l2) * on).sum(1), dt) / den, dt)
    return r(0.5 * r(rows.sum() / B, dt), dt), rows, grad


def aten_actor(lp, adv, mask, dt):
    x = lp.to(dt).clone().requires_grad_(True)
    loss = O.actor_loss(x, lp.to(dt), adv.to(dt), mask, ACTOR_CLIP)
    loss.backward()
    return loss.detach(), x.grad


def aten_critic(x, old, ret, mask, dt):
    v = x.to(dt).clone().requires_grad_(True)
    loss = O.critic_loss(v, old.to(dt), ret.to(dt), mask, CRITIC_CLIP)
    loss.backward()
    return loss.detach(), v.grad


def mean_rounds_alike(rows, dt):
    """The 16-bit mean of the row means is the same whatever order fp32 sums them in: the float64 mean, moved by the
    fp32 summation bound either way, rounds to one dt value."""
    m = rows.sum() / rows.numel()
    tol = rows.numel() * 2.0 ** -24 * rows.abs().sum() / rows.numel()
    return bool(r(m - tol, dt) == r(m + tol, dt))


def test_aten_cpu_rounds_a_row_count_to_the_dividend_dtype():
    """The premise on ATen CPU: a 16-bit (B,) tensor divided by an int64 (B,) count divides by the rounded count.
    A one-element divisor is the exception: ATen CPU's division reads it at its exact value, as it reads the token
    mean's 0-dim count, so B = 1 stays out of the comparisons below (ATen CUDA casts it like any other count; the GPU
    file checks that)."""
    for dt, n in ((BF, 257), (F16, 2049)):
        x = torch.full((2,), -0.5, dtype=dt)
        q = x / torch.tensor([n, n])
        assert q.dtype == dt
        assert torch.equal(q.double(), r(-0.5 / r(n, dt), dt).expand(2))
        assert not torch.equal(q.double(), r(-0.5 / n, dt).expand(2)), (dt, n)
        one = x[:1] / torch.tensor([n])
        assert torch.equal(one.double(), r(-0.5 / n, dt).expand(1)), (dt, n)


def exact_actor_case(B, n, dt, seed):
    """actor_operands from the first seed (seed, seed + 1000, ...) whose loss does not depend on the fp32 summation
    order (mean_rounds_alike): so K5, ATen CPU and ATen CUDA all owe the restatement's loss bit for bit."""
    for s in range(seed, seed + 10000, 1000):
        lp, adv, mask = actor_operands(B, n, s)
        if mean_rounds_alike(k5_actor(adv, mask, dt)[1], dt):
            return lp, adv, mask
    raise AssertionError(f'no operand set for {dt} n={n} B={B}')


def exact_critic_case(B, n, dt, seed):
    """critic_operands, chosen like exact_actor_case."""
    for s in range(seed, seed + 10000, 1000):
        ops = critic_operands(B, n, s)
        if mean_rounds_alike(k5_critic(*ops, dt)[1], dt):
            return ops
    raise AssertionError(f'no operand set for {dt} n={n} B={B}')


@pytest.mark.parametrize('B', [3, 129])
@pytest.mark.parametrize('dt,n', CASES, ids=CASE_IDS)
def test_k5_actor_restatement_vs_ref_port(dt, n, B):
    lp, adv, mask = exact_actor_case(B, n, dt, seed=n + B)
    loss, rows, grad = k5_actor(adv, mask, dt)
    want, gwant = aten_actor(lp, adv, mask, dt)
    assert torch.equal(grad, gwant.double()), f'{dt} n={n} B={B}: gradient'
    assert float(loss) == float(want), f'{dt} n={n} B={B}: loss'
    # the masked row means themselves, as ref_port's masked_mean forms them before its .mean()
    x = (adv.to(dt) * mask).sum(-1) / mask.sum(-1)
    assert torch.equal(rows, x.double())


@pytest.mark.parametrize('B', [3, 129])
@pytest.mark.parametrize('dt,n', CASES, ids=CASE_IDS)
def test_k5_critic_restatement_vs_ref_port(dt, n, B):
    x, old, ret, mask = exact_critic_case(B, n, dt, seed=2 * n + B)
    loss, rows, grad = k5_critic(x, old, ret, mask, dt)
    want, gwant = aten_critic(x, old, ret, mask, dt)
    assert torch.equal(grad, gwant.double()), f'{dt} n={n} B={B}: gradient'
    assert float(loss) == float(want), f'{dt} n={n} B={B}: loss'


@pytest.mark.parametrize('dt,n', [(BF, 257), (F16, 2049)], ids=['bfloat16-257', 'float16-2049'])
def test_the_exact_count_rule_misses_the_reference(dt, n):
    """Dividing by the exact count (K5's rule before it rounded the count) differs from ATen in the gradient of almost
    every token and in the loss; at a count the dtype holds, both rules agree."""
    lp, adv, mask = actor_operands(3, n, seed=n)
    _, gwant = aten_actor(lp, adv, mask, dt)
    _, _, exact = k5_actor(adv, mask, dt, rounded=False)
    _, _, rounded = k5_actor(adv, mask, dt)
    assert torch.equal(rounded, gwant.double())
    on = mask & (adv != 0)
    assert float((exact[on] != gwant.double()[on]).double().mean()) > 0.5
    x, old, ret, cmask = critic_operands(3, n, seed=n)
    want, _ = aten_critic(x, old, ret, cmask, dt)
    assert float(k5_critic(x, old, ret, cmask, dt, rounded=False)[0]) != float(want)
    held = {BF: 256, F16: 2048}[dt]
    lp, adv, mask = actor_operands(3, held, seed=held)
    assert torch.equal(k5_actor(adv, mask, dt, rounded=False)[2], k5_actor(adv, mask, dt)[2])
