"""K4r (`aa_ppo_returns`, Multi-PPO's rloo / reinforce_baseline / group_norm / reinforce returns) pinned through the C
ABI on one H100 (`pytest -m gpu`), at the cases of tests/test_cpu_returns_pin.py: every n from 2 to 64 the group
estimators meet (n = 5, 6, 7, 12, 15, 17 leave some of ATen's reduction threads with one element fewer; n >= 16 takes
the 16- and 32-thread trees), groups that straddle rows and groups longer than a row, start 0, W // 4 and W - 1, more
CTAs than one resident wave, both modes, both output masks, two gammas and an output dtype wider than the rewards.

Every launch writes into guarded outputs (POISON between SENTINEL bands; `row_stats` must change in lanes 3-4 only) and
reads rewards and mask through strided rows between NaN-fenced rows, so a read past a row reaches the result as NaN.
Four checks per case:
  1. exact operands (gamma = 1): small dyadic rewards whose groups sum to exactly 0, so that every value K4r rounds is
     representable and every sum is exact in any order; the outputs equal `returns_f64` rounded once to their dtype;
  2. faithful mode on real-valued rollout rewards: the ATen port on CUDA at DESIGN section 4's bar (16-bit: every
     element within 1 ulp and >= 97 % bit-identical; fp32: 2e-5 relative), masked positions exactly zero, the NaN
     pattern of fp16 group_norm on a constant group the port's; lanes 3-4 of row_stats the masked row means of the
     port's returns (a 1-ulp fp16 flip in a short row moves its mean by ~1e-3, far past the 2e-5 allowed);
  3. F32 mode: `returns_f64` within 2e-5 relative, or the fp32 summation bound where that is larger;
  4. on the same real-valued rewards, every mode and dtype: bit for bit `k4r_restated`, the float32 restatement of
     K4r's own order (tests/test_cpu_returns_pin.py).  ATen's fp32 group order is not this one for n >= 4 (DESIGN
     section 4), so checks 2 and 3 cannot see an order change in fp32 and 16-bit rounding hides most of them; this
     check does at every n >= 3, which is what keeps `group_stats` from drifting to another order unnoticed."""
from __future__ import annotations

import pytest
import torch

import multi_ppo_port as P
from align_anything_b200 import _lib as Lb
from test_cpu_returns_pin import CASE_IDS, CASES, exact_case, exact_estimators, k4r_restated
from test_gpu_loss_kernels import CODE, FAITHFUL, F32MODE, Guarded, _stream, assert_same, assert_within, fenced, rc_ok
from test_gpu_multi_ppo import _rollout_like
from test_gpu_parity import assert_close_f32, assert_ulp_close, ops  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

DEV = 'cuda'
F32 = torch.float32
U = 2.0 ** -24


def launch(c, est, r, mask):
    """One aa_ppo_returns on guarded outputs, rewards at row stride W + 3 and the mask at W + 5 between fences.
    -> (advantages, returns, row_stats) after the guard checks."""
    B, W, nr = c.B, c.W, c.W - c.start
    from align_anything_b200 import ops

    rews = fenced(r.to(c.dt), W + 3)
    mt = fenced(mask.to(torch.bool), W + 5, pad=True)
    adv, ret, rs = Guarded(B, nr, c.out), Guarded(B, nr, c.out), Guarded(B, 8, F32)
    what = f'{c.id} {est}'
    rc_ok(Lb.lib().aa_ppo_returns(rews.data_ptr(), CODE[c.dt], rews.stride(0), mt.data_ptr(), mt.stride(0), B, W,
                                  c.start, ops.ESTIMATORS[est], c.n, c.gamma, FAITHFUL if c.mode == 'faithful' else
                                  F32MODE, c.mask_out, adv.ptr(), ret.ptr(), CODE[c.out], rs.ptr(), _stream()), what)
    torch.cuda.synchronize()
    adv.check(what + ' adv')
    ret.check(what + ' ret')
    lanes = torch.zeros(B, 8, dtype=torch.bool)
    lanes[:, 3:5] = True
    rs.check(what + ' row_stats lanes 3-4 only', lanes)
    assert_same(adv.t, ret.t, what + ' adv == ret')
    assert_same(rs.t[:, 4], rs.t[:, 3], what + ' row_stats lane 4 == lane 3')
    return adv.t.clone(), ret.t.clone(), rs.t.clone()


def real_case(c):
    """_rollout_like rewards (holes, left and right pads) at the case's shape, and one group of the constant 0.25, all
    masked in, inside the outputs: fp16 group_norm turns it into 0 / 0 (1e-9 rounds to 0 in fp16)."""
    gen = torch.Generator().manual_seed(c.n * 1009 + c.B * 31 + c.W)
    r, mask, _ = _rollout_like(c.B, c.W, c.dt, gen)
    if c.ests != ('reinforce',):
        g0 = (c.start + c.W - 1) // 2 // c.n * c.n  # the group holding flat index ~ (start + W) / 2 of row 0
        r.view(-1)[g0:g0 + c.n] = 0.25
        mask.view(-1)[g0:g0 + c.n] = True
    return r.to(DEV), mask.to(DEV)


@pytest.mark.parametrize('c', CASES, ids=CASE_IDS)
def test_returns_pin(ops, c):
    nr = c.W - c.start
    # 1. exact operands: returns_f64 rounded once to the output dtype, bit for bit
    if c.gamma == 1.0:
        r64, mask = exact_case(c, seed=c.n * 7 + c.W)
        for est in exact_estimators(c):
            adv, ret, rs = launch(c, est, r64.to(DEV), mask.to(DEV))
            want = torch.from_numpy(P.returns_f64(r64, mask, c.start, est, c.n, 1.0, bool(c.mask_out)))
            assert_same(ret, want.to(c.out), f'{c.id} {est} exact')
            m = mask[:, c.start:].to(DEV)
            assert_close_f32(rs[:, 3], (ret.float() * m).sum(-1) / m.sum(-1), what=f'{c.id} {est} row mean')
    # 2. / 3. real-valued rewards
    r, mask = real_case(c)
    off = ~mask[:, c.start:]
    for est in c.ests:
        what = f'{c.id} {est}'
        adv, ret, rs = launch(c, est, r, mask)
        assert_same(ret, k4r_restated(r, mask, c, est), what + ' vs the float32 restatement')
        if c.mode == 'faithful':
            _, w_ret = P.advantages_and_returns(torch.zeros_like(r), r, mask, c.start, est, c.n, c.gamma,
                                                mask_outputs=bool(c.mask_out))
            if c.out != c.dt:  # the faithful value, stored wider: exactly a value of the rewards' dtype
                assert_same(ret, ret.to(c.dt), what + ' representable in the rewards dtype')
                ret = ret.to(c.dt)
            assert_ulp_close(ret, w_ret, max_ulp=1, min_exact=0.97, what=what)
            if c.mask_out:
                assert not bool((ret[off].nan_to_num() != 0).any()), what + ' masked positions'
            if not (c.dt == torch.float16 and est == 'group_norm'):
                assert not bool(torch.isnan(ret).any()), what
            m = mask[:, c.start:]
            want_mean = torch.where(m, w_ret.float(), 0.0).sum(-1) / m.sum(-1)  # K4r sums the masked-in positions only
            assert_close_f32(rs[:, 3], want_mean, what=what + ' row mean')
        else:
            r64 = r.double().cpu()
            want = torch.from_numpy(P.returns_f64(r64, mask.cpu(), c.start, est, c.n, c.gamma, bool(c.mask_out)))
            # the summation bound: every estimator value is off by a few of its magnitude's ulps (|r| + |group
            # statistic|, over std for group_norm) and the chain adds one rounding per step
            x = r64 * mask.cpu()
            if est != 'reinforce':
                x = x.reshape(-1, c.n)
                mag = x.abs() + x.mean(-1, keepdim=True).abs() + x.abs().sum(-1, keepdim=True) / (c.n - 1)
                if est == 'group_norm':  # a constant group is exactly 0 in both
                    sd = x.std(-1, keepdim=True)
                    mag = torch.where(sd > 0, mag / sd, 0.0)
                x = mag.reshape(c.B, c.W)
            mag = (x.abs() * mask.cpu())[:, c.start:]
            suffix = torch.flip(torch.cumsum(torch.flip(mag, [1]), 1), [1])
            tol = torch.maximum(2e-5 * want.abs(), (nr + 16) * U * suffix)
            assert_within(ret.float(), want, tol, what + ' f32 mode')
