"""The references tests/test_gpu_cov_pin.py holds the Clip-Cov / KL-Cov kernels to, checked without a GPU: the
stable-sort top-k, the fp32 key order, the clip-band filter and the exactness of the faithful-count operands."""
from __future__ import annotations

import math

import pytest
import torch

import cov_port as port
from test_cpu_faithful_counts import BF, CASE_IDS, CASES, F16, exact_actor_case, k5_actor, r

F32 = torch.float32
# token-mean totals a 16-bit dtype cannot hold (1501 -> 1504 in bf16, 2049 -> 2048 in fp16), in one row or spread
TOKEN_MEAN_CASES = [(BF, [1501]), (BF, [500, 500, 501]), (F16, [2049]), (F16, [683, 683, 683])]
TOKEN_MEAN_IDS = ['bfloat16-1x1501', 'bfloat16-3x500', 'float16-1x2049', 'float16-3x683']


def token_mean_case(counts):
    """The operands of tests/test_gpu_cov_pin.py's token-mean totals, float64 on the CPU: log-probs on the 2^-4 grid in
    [-4, -1/16], advantages k / 8 with |k| <= 32, a mask with counts[b] tokens at random places of row b (W =
    max(counts) + 7) and a ~5 % selection on counted and uncounted tokens alike."""
    B, W = len(counts), max(counts) + 7
    g = torch.Generator().manual_seed(sum(counts))
    lp = -torch.randint(1, 65, (B, W), generator=g).double() / 16
    adv = torch.randint(-32, 33, (B, W), generator=g).double() / 8
    mask = torch.zeros(B, W, dtype=torch.bool)
    for b, n in enumerate(counts):
        mask[b, torch.randperm(W, generator=g)[:n]] = True
    sel = torch.rand(B, W, generator=g) < 0.05
    sel[torch.arange(B), (~mask).int().argmax(-1)] = True  # the first uncounted token of each row: must change nothing
    return lp, adv, mask, sel


def test_top_k_agrees_with_torch_topk_on_distinct_keys():
    g = torch.Generator().manual_seed(0)
    keys = torch.randperm(1 << 20, generator=g)[:5000].view(50, 100).to(torch.int64)
    eligible = torch.ones_like(keys, dtype=torch.bool)
    for k in (1, 17, 2500, 5000):
        want = torch.zeros(5000, dtype=torch.bool)
        want[torch.topk(keys.reshape(-1), k).indices] = True
        assert torch.equal(port.top_k(keys, eligible, k).reshape(-1), want), k


def test_top_k_breaks_ties_to_the_smaller_flat_index_and_skips_ineligible():
    keys = torch.tensor([[5, 7, 7, 3], [7, 9, 7, 7]])
    eligible = torch.tensor([[True, True, False, True], [True, True, True, True]])
    # 9 first, then the eligible 7s in flat order: (0, 1), (1, 0), (1, 2), (1, 3)
    assert port.top_k(keys, eligible, 3).tolist() == [[False, True, False, False], [True, True, False, False]]
    assert port.top_k(keys, eligible, 5).tolist() == [[False, True, False, False], [True, True, True, True]]
    assert port.state_words(keys, eligible, 3 / 8, 8) == (7, 3, 7, 2)  # E, k, T, need (two of the four 7s)
    assert port.state_words(keys, eligible, 1.0, 8) == (7, 7, 3, 1)
    assert port.state_words(keys, torch.zeros_like(eligible), 0.5, 8) == (0, 0, port.U32, 0)


def test_order_key_is_monotone_over_fp32():
    """Strictly increasing over an increasing fp32 sweep (-inf, normals, subnormals, +-0 as one key, +inf), NaN above
    +inf (either sign, any payload)."""
    tiny = torch.finfo(F32).tiny
    pos = [2.0 ** -149, 2.0 ** -140, tiny / 2, tiny, 1e-30, 0.5, 1.0, 1.0 + 2 ** -23, 3.0, 1e30,
           torch.finfo(F32).max]
    sweep = [-math.inf] + [-v for v in reversed(pos)] + [0.0] + pos + [math.inf]
    x = torch.tensor(sweep, dtype=F32)
    k = port.order_key(x)
    assert bool((k[1:] > k[:-1]).all()), k.tolist()
    assert int(port.order_key(torch.tensor([-0.0]))[0]) == int(port.order_key(torch.tensor([0.0]))[0])
    nans = torch.tensor([0x7fc00000, 0xffc00000, 0x7f800001, 0x7fffffff], dtype=torch.int64).to(torch.int32)
    nk = port.order_key(nans.view(F32))
    assert bool((nk == port.U32).all()) and bool((nk > k[-1]).all())
    assert bool((k >= 0).all()) and bool((k <= port.U32).all())


@pytest.mark.parametrize('dt', [F32, BF, F16])
def test_clip_band_filter_leaves_no_ambiguous_ratio(dt):
    """After clear_clip_band, perturbing exp by +-4 fp32 ulps changes no token's clip predicate; in fp32 that means no
    ratio within 4 ulps of a bound.  The filter keeps ratios one dtype ulp from a bound, whose side the dtype decides."""
    g = torch.Generator().manual_seed(1)
    B, W, lo, hi = 64, 512, 0.2, 0.28
    lp = (-torch.rand(B, W, generator=g) * 4).to(dt)
    old = (lp.float() + torch.randn(B, W, generator=g) * 0.3).to(dt)
    adv = torch.randn(B, W, generator=g).to(dt)
    if dt == F32:  # plant ratios right at the bounds
        old[:, :8] = lp[:, :8] - torch.log(torch.tensor([1 - lo, 1 + hi] * 4, dtype=torch.float64)).float()
    stable = port.stable_clip(lp, old, adv, lo, hi)
    if dt == F32:
        assert not bool(stable.all())  # the planted ratios sit in the band
    new = port.clear_clip_band(lp, old, adv, lo, hi)
    assert torch.equal(new[stable], old[stable]) and torch.equal(new[~stable], lp[~stable])
    assert bool(port.stable_clip(lp, new, adv, lo, hi).all())
    rr = torch.exp((lp - new).double())
    if dt == F32:  # the bound that decides: 1 - low for a negative advantage, 1 + high for a positive one
        for bound, side in ((1 - lo, adv < 0), (1 + hi, adv > 0)):
            b = torch.tensor(bound, dtype=F32).double()
            assert not bool((((rr - b).abs() <= 4 * 2.0 ** -24 * b) & side).any())
    else:  # ratios one dtype ulp from a bound survive
        ulp = 2.0 ** -8 if dt == BF else 2.0 ** -11
        near = (rr - (1 + hi)).abs() <= 2 * ulp
        assert bool((near & stable).any())


@pytest.mark.parametrize('dt,n', CASES, ids=CASE_IDS)
def test_exact_operands_are_exact(dt, n):
    """The operands of the faithful-count loss pins: lp == old (ratio exactly 1), advantages and log-probs the dtype
    holds exactly, and every masked row sum exact in fp32 (dyadic, below 2^24 units of 1/8)."""
    lp, adv, mask = exact_actor_case(3, n, dt, seed=n + 3)
    assert torch.equal(lp.to(dt).double(), lp) and torch.equal(adv.to(dt).double(), adv)
    assert float(torch.exp(lp.to(dt) - lp.to(dt)).max()) == 1.0 == float(torch.exp(lp.to(dt) - lp.to(dt)).min())
    sums = (adv * mask).sum(-1) * 8
    assert torch.equal(sums, sums.round()) and float(sums.abs().max()) < 2 ** 24
    assert torch.equal((adv * mask).sum(-1).float().double(), (adv * mask).sum(-1))
    loss, rows, grad = k5_actor(adv, mask, dt)
    assert torch.equal(r(loss, dt), loss) and torch.equal(r(grad, dt), grad)


@pytest.mark.parametrize('dt,counts', TOKEN_MEAN_CASES, ids=TOKEN_MEAN_IDS)
def test_token_mean_operands_are_exact(dt, counts):
    """token_mean_case: the counts asked for, a total the dtype rounds, operands the dtype holds, lp == old (ratio 1),
    and the masked sum with or without the selected terms exact in fp32 and in any order, so the only rounding left
    to tell ATen CUDA's divisor from the exact count is the count's own."""
    lp, adv, mask, sel = token_mean_case(counts)
    assert mask.sum(-1).tolist() == counts
    total = sum(counts)
    assert float(r(total, dt)) != total
    assert torch.equal(lp.to(dt).double(), lp) and torch.equal(adv.to(dt).double(), adv)
    assert float(torch.exp(lp.to(dt) - lp.to(dt)).max()) == 1.0 == float(torch.exp(lp.to(dt) - lp.to(dt)).min())
    assert bool((sel & mask).any()) and bool((sel & ~mask).any())
    for kept in (mask, mask & ~sel):
        s8 = (adv * kept).sum() * 8
        assert float(s8) == round(float(s8)) and abs(float(s8)) < 2 ** 24
        assert float((adv * kept).sum().float()) == float((adv * kept).sum())
