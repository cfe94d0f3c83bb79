"""The case table of tests/test_gpu_returns_pin.py (K4r, `aa_ppo_returns`, through the C ABI) and its premises, checked
without a GPU: every case has the edge its id claims, the exact operands make every value K4r rounds representable
and every sum exact in any order, the float64 restatement agrees with the ATen port run in float64, and the float32
restatement of K4r's own arithmetic (`k4r_restated`, which the GPU pin holds the kernel to bit for bit) agrees with
float64 on every case."""
from __future__ import annotations

import dataclasses

import numpy as np
import pytest
import torch

import multi_ppo_port as P
from test_gpu_loss_kernels import sum_exact  # importable without a GPU: it only touches the device inside tests

BF, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
GROUP = ('rloo', 'reinforce_baseline', 'group_norm')
NS = (2, 5, 6, 7, 12, 15, 16, 17, 32, 64)
RESIDENT_CTAS = 132 * 32  # H100 SXM: 132 SMs, at most 32 resident CTAs each (K4r's CTAs are one warp)
EXACT = 2 ** 24


@dataclasses.dataclass(frozen=True)
class Case:
    ests: tuple
    n: int
    B: int
    W: int
    start: int
    dt: torch.dtype           # rewards
    mode: str                 # 'faithful' | 'f32'
    out: torch.dtype          # advantages / returns
    mask_out: int
    gamma: float
    edges: tuple = ()         # 'straddle' (W % n != 0), 'n>W', 'idle' (some of the bw threads hold fewer
                              # elements), 'aligned' (W % n == 0), 'waves' (B above one resident wave)

    @property
    def id(self):
        e = ','.join(self.edges) or 'plain'
        est = 'reinforce' if self.ests == ('reinforce',) else 'group'
        return (f'{est}-n{self.n}-B{self.B}-W{self.W}-s{self.start}-{str(self.dt)[6:]}-{self.mode}-out'
                f'{str(self.out)[6:]}-m{self.mask_out}-g{self.gamma}-{e}')


def bw(n):
    """ATen's threads per group for a contiguous inner reduction of n (Reduce.cuh): min(largest power of two <= n, 32)."""
    return min(1 << (n.bit_length() - 1), 32)


def _edges(n, B, W):
    e = []
    e.append('aligned' if W % n == 0 else 'straddle')
    if n > W:
        e.append('n>W')
    if n % bw(n):
        e.append('idle')
    if B > RESIDENT_CTAS:
        e.append('waves')
    return tuple(e)


def _cases():
    out = []

    def add(ests, n, B, W, start, dt, mode, o, m, g):
        out.append(Case(ests, n, B, W, start, dt, mode, o, m, g, _edges(n, B, W)))

    W = 257  # prime: every n straddles rows
    for n in NS:
        B = n * -(-32 // n)
        add(GROUP, n, B, W, W // 4, BF, 'faithful', BF, 1, 1.0)
        add(GROUP, n, B, W, 0, F16, 'faithful', F16, 1, 0.99)
        add(GROUP, n, B, W, W // 4, F32, 'faithful', F32, 0, 0.99)
        add(GROUP, n, B, W, W - 1, F32, 'faithful', F32, 1, 1.0)
        add(GROUP, n, B, W, W // 4, BF, 'f32', F32, 1, 1.0)
    # one group spans several rows
    add(GROUP, 64, 64, 37, 9, BF, 'faithful', BF, 1, 1.0)
    add(GROUP, 64, 64, 37, 9, F32, 'faithful', F32, 0, 1.0)
    add(GROUP, 32, 8, 20, 0, F16, 'f32', F32, 1, 0.99)
    add(GROUP, 17, 17, 5, 1, F32, 'faithful', F32, 1, 1.0)
    # rows that hold whole groups
    add(GROUP, 12, 8, 96, 24, F32, 'faithful', F32, 1, 1.0)
    add(GROUP, 16, 8, 256, 64, BF, 'faithful', BF, 0, 0.99)
    # more CTAs than one resident wave
    add(GROUP, 16, 4500, 12, 3, F32, 'faithful', F32, 1, 1.0)
    add(GROUP, 16, 4500, 12, 3, F16, 'faithful', F16, 1, 1.0)
    # faithful rounding stored in a wider dtype; F32 mode on fp16
    add(GROUP, 6, 36, 257, 64, BF, 'faithful', F32, 1, 1.0)
    add(GROUP, 15, 45, 257, 64, F16, 'f32', F32, 0, 1.0)
    add(('reinforce',), 1, 32, 257, 64, BF, 'faithful', BF, 1, 0.99)
    add(('reinforce',), 1, 32, 257, 0, F32, 'faithful', F32, 0, 1.0)
    add(('reinforce',), 16, 32, 257, 64, F16, 'f32', F32, 1, 1.0)
    return out


CASES = _cases()
CASE_IDS = [c.id for c in CASES]


def rc_dtype(c):
    """The dtype K4r rounds to: the rewards' in faithful mode, fp32 in F32 mode."""
    return c.dt if c.mode == 'faithful' else F32


def exact_estimators(c):
    """The estimators whose every intermediate is exact on exact_case's operands: reinforce; reinforce_baseline (the
    group mean is 0 * 1/n); rloo where n - 1 is a power of two (its base is loo * 1/(n - 1), 1/(n - 1) exact).
    group_norm's std is a square root and has no exact case here: the real-valued checks hold it."""
    pow2 = lambda k: k & (k - 1) == 0  # noqa: E731
    return tuple(e for e in c.ests if e in ('reinforce', 'reinforce_baseline') or (e == 'rloo' and pow2(c.n - 1)))


def exact_case(c, seed):
    """float64 rewards and a bool mask (CPU): masked-in rewards are k / 8 with |k| <= 15 (a quarter of them 0); the
    masked-out ones are other values (k / 2), which K4r must not see.  For the group estimators every group's
    masked-in values come in +- pairs (an odd one out is 0), so each group sums to exactly 0 and its mean, sum * 1/n,
    is exactly 0 whatever n is.  About 15 % of the mask is holes."""
    B, W, n = c.B, c.W, c.n
    g = torch.Generator().manual_seed(seed)
    mask = torch.rand(B, W, generator=g) > 0.15
    v = torch.randint(-15, 16, (B, W), generator=g).double() / 8
    v = v * (torch.randint(0, 4, (B, W), generator=g) != 0)
    if c.ests != ('reinforce',):
        fv, fm = v.reshape(-1, n), mask.reshape(-1, n)
        for k in range(fv.shape[0]):
            on = fm[k].nonzero().flatten()
            on = on[torch.randperm(on.numel(), generator=g)]
            a = fv[k, on[0::2]][: on.numel() // 2]
            fv[k] = 0
            fv[k, on[0:2 * a.numel():2]] = a
            fv[k, on[1:2 * a.numel():2]] = -a
        v = fv.reshape(B, W)
    junk = torch.randint(-15, 16, (B, W), generator=g).double() / 2
    return torch.where(mask, v, junk), mask


def estimator_f64(r64, mask, est, n):
    """The estimator values and the quantities K4r rounds on the way, float64: {'x': (B, W), 'inter': [tensors]}."""
    x = (r64 * mask).reshape(-1, n)
    s = x.sum(-1, keepdim=True)
    if est == 'reinforce':
        return {'x': r64 * mask, 'inter': []}
    if est == 'reinforce_baseline':
        mu = s / n
        return {'x': (x - mu).reshape(r64.shape), 'inter': [s, mu]}
    loo = s - x
    base = loo / (n - 1)
    return {'x': (x - base).reshape(r64.shape), 'inter': [s, loo, base]}


def representable(v, dt):
    return torch.equal(v.to(dt).double(), v) and torch.equal(v.float().double(), v)


# ---- K4r's arithmetic restated in float32 (csrc/ppo.cu: group_stats, estimator_value, ppo_returns_kernel) ----------
F4, LD = np.float32, np.longdouble


def _fma(a, b, c):
    """fp32 fma: a * b is exact in the 64-bit significand of x86 long double and the sum rounds there first; a second
    rounding can differ from one only when that first result sits exactly on an fp32 midpoint (~2^-40 of cases)."""
    return (LD(1) * a.astype(LD) * b.astype(LD) + c.astype(LD)).astype(F4)


def _w_one(x):
    return (x, np.zeros_like(x), np.ones_like(x))


def _w_add(w, x):
    m0, m2, nf = w
    nf = nf + F4(1)
    d = x - m0
    m = m0 + d / nf
    return (m, _fma(d, x - m, m2), nf)


def _w_combine(a, b):
    d, nn = b[0] - a[0], a[2] + b[2]
    r = b[2] / nn
    return (_fma(d, r, a[0]), _fma((d * d) * a[2], r, a[1] + b[1]), nn)


def _tree(parts, combine):
    """ATen's shuffle-down tree over len(parts) (a power of two) thread partials: offset 1, 2, 4 ..., lower on the left."""
    parts, off = list(parts), 1
    while off < len(parts):
        for j in range(0, len(parts) - off, 2 * off):
            parts[j] = combine(parts[j], parts[j + off])
        off *= 2
    return parts[0]


def group_stats32(x, n):
    """x: float32 (G, n) masked rewards -> (sum, unbiased std) per group, in group_stats' order: bw = min(largest power
    of two <= n, 32) threads; thread j folds elements j + k * bw into sum accumulator k % 4 (from 0; then
    ((a0 + a1) + a2) + a3) and Welford accumulator k % 2 (then combined when the second is not empty), except that
    for n < 16 a thread's (at most two) elements are added directly; then the tree."""
    bw = min(1 << (n.bit_length() - 1), 32)
    sums, wels = [], []
    for j in range(bw):
        idx = list(range(j, n, bw))
        if n < 16:
            s = x[:, idx[0]] + x[:, idx[1]] if len(idx) == 2 else x[:, idx[0]]
            w = _w_combine(_w_one(x[:, idx[0]]), _w_one(x[:, idx[1]])) if len(idx) == 2 else _w_one(x[:, idx[0]])
        else:
            acc = [np.zeros(x.shape[0], F4) for _ in range(4)]
            wa = [None, None]
            for k, e in enumerate(idx):
                acc[k % 4] = acc[k % 4] + x[:, e]
                wa[k % 2] = _w_add(wa[k % 2], x[:, e]) if wa[k % 2] is not None else _w_one(x[:, e])
            s = ((acc[0] + acc[1]) + acc[2]) + acc[3]
            w = wa[0] if wa[1] is None else _w_combine(wa[0], wa[1])
        sums.append(s)
        wels.append(w)
    total = _tree(sums, lambda a, b: a + b)
    m2 = _tree(wels, _w_combine)[1]
    return total, np.sqrt(m2 / F4(n - 1))


def k4r_restated(r, mask, c, est):
    """K4r's returns for case c on rewards r (any float tensor; read as c.dt) and bool mask, in float32 numpy with the
    kernel's rounding points: every op one fp32 rounding, then `rnd` to the rounding dtype (the rewards' in faithful
    mode, fp32 in F32 mode); the carry of the chain stays fp32.  -> torch (B, W - start) of dtype c.out."""
    rc = rc_dtype(c)

    def rnd(v):
        return v if rc == F32 else torch.from_numpy(np.ascontiguousarray(v)).to(rc).float().numpy()

    B, W, n, start = c.B, c.W, c.n, c.start
    rv = r.to(c.dt).float().cpu().numpy()
    m = mask.cpu().numpy()
    x = np.where(m, rv, rv * F4(0))
    if est == 'reinforce':
        v = x
    else:
        xg = x.reshape(-1, n)
        s, sd = group_stats32(xg, n)
        s, sd = s[:, None], sd[:, None]
        if est == 'group_norm':
            mu = rnd(s * (F4(1) / F4(n)))
            with np.errstate(invalid='ignore'):  # fp16 0 / 0 of a constant group is part of what is restated
                v = rnd(rnd(xg - mu) / rnd(rnd(sd) + F4(1e-9)))
        elif est == 'rloo':
            v = rnd(xg - rnd(rnd(rnd(s) - xg) * (F4(1) / F4(n - 1))))
        else:
            v = rnd(xg - rnd(s * (F4(1) / F4(n))))
        v = v.reshape(B, W)
    v = np.where(m, v, v * F4(0))[:, start:]
    g, carry = F4(c.gamma), np.zeros(B, F4)
    out = np.empty_like(v)
    for t in range(W - start - 1, -1, -1):
        carry = v[:, t] + g * carry
        out[:, t] = rnd(carry)
    if c.mask_out:
        mo = m[:, start:]
        out = np.where(mo, out, out * F4(0))
    return torch.from_numpy(out).to(c.out)


@pytest.mark.parametrize('c', CASES, ids=CASE_IDS)
def test_case_has_its_edges(c):
    """Each case is valid for K4r and has the edge its id names: straddling groups, n > W, threads of ATen's
    reduction that hold one element fewer, B above one resident wave; and start is in range."""
    B, W, n = c.B, c.W, c.n
    assert 0 <= c.start < W
    if c.ests != ('reinforce',):
        assert (B * W) % n == 0 and n >= 2
    assert ('straddle' in c.edges) == (W % n != 0) and ('aligned' in c.edges) == (W % n == 0)
    assert ('n>W' in c.edges) == (n > W)
    assert ('idle' in c.edges) == (n % bw(n) != 0)
    assert ('waves' in c.edges) == (B > RESIDENT_CTAS)
    if 'straddle' in c.edges and c.ests != ('reinforce',):  # some group really has elements in two rows
        g0 = torch.arange(0, B * W, n)
        assert bool(((g0 // W) != ((g0 + n - 1) // W)).any())


def test_the_matrix_covers_every_edge():
    """Every n at every start kind, every dtype and mode, both mask_outputs and both gammas, n > W, a wave-crossing B."""
    group = [c for c in CASES if c.ests == GROUP]
    for n in NS:
        mine = [c for c in group if c.n == n]
        assert {c.start for c in mine} >= {0, 257 // 4, 256}, n
        assert {(c.dt, c.mode) for c in mine} >= {(BF, 'faithful'), (F16, 'faithful'), (F32, 'faithful'), (BF, 'f32')}
    assert {c.n for c in CASES if c.ests == ('reinforce',)} == {1, 16}
    assert {c.mask_out for c in CASES} == {0, 1} and {c.gamma for c in CASES} == {1.0, 0.99}
    assert any(c.out != c.dt and c.mode == 'faithful' for c in CASES)
    assert any('n>W' in c.edges for c in group) and any('waves' in c.edges for c in group)
    assert {bw(n) for n in NS} == {2, 4, 8, 16, 32}


@pytest.mark.parametrize('c', [c for c in CASES if c.gamma == 1.0], ids=[c.id for c in CASES if c.gamma == 1.0])
def test_exact_operands_are_exact(c):
    """For each exact estimator: the group sums are exact in any order, every value K4r rounds (sum, mean, loo, base,
    the estimator value) is representable in its rounding dtype, and each row's chain of masked values is exact in
    fp32 in any order, so K4r must equal returns_f64 bit for bit (rounded once to the output dtype)."""
    r64, mask = exact_case(c, seed=c.n * 7 + c.W)
    assert representable(r64, c.dt)
    ests = exact_estimators(c)
    assert ests, c.id
    for est in ests:
        q = estimator_f64(r64, mask, est, c.n)
        if est != 'reinforce':
            assert sum_exact((r64 * mask).reshape(-1, c.n), -1), est
        for t in q['inter'] + [q['x']]:
            assert representable(t, rc_dtype(c)), est
        assert sum_exact((q['x'] * mask)[:, c.start:], -1), est
        want = P.returns_f64(r64, mask, c.start, est, c.n, 1.0, bool(c.mask_out))
        chain = torch.flip(torch.cumsum(torch.flip((q['x'] * mask)[:, c.start:], [1]), 1), [1])
        if c.mask_out:
            chain = chain * mask[:, c.start:]
        assert torch.equal(torch.from_numpy(want), chain), est


@pytest.mark.parametrize('c', CASES[::3], ids=CASE_IDS[::3])
def test_returns_f64_agrees_with_the_port_in_float64(c):
    """The two statements of the estimators (ATen ops and explicit flat-index groups) agree in float64 on real-valued
    rewards, with holes and both output masks."""
    g = torch.Generator().manual_seed(c.n + c.B)
    r = torch.randn(c.B, c.W, generator=g, dtype=F64)
    mask = torch.rand(c.B, c.W, generator=g) > 0.1
    for est in c.ests:
        _, ret = P.advantages_and_returns(torch.zeros_like(r), r, mask, c.start, est, c.n, c.gamma,
                                          mask_outputs=bool(c.mask_out))
        want = torch.from_numpy(P.returns_f64(r, mask, c.start, est, c.n, c.gamma, bool(c.mask_out)))
        assert torch.allclose(ret, want, rtol=1e-10, atol=1e-10), (c.id, est)


@pytest.mark.parametrize('c', CASES, ids=CASE_IDS)
def test_float32_restatement(c):
    """k4r_restated on every case: bit for bit returns_f64 (rounded once) on the exact operands, and within the
    rounding of its dtype of returns_f64 on real-valued rewards, so the restatement the GPU pin holds K4r to bit
    for bit computes the estimators and not something else."""
    if c.gamma == 1.0:
        r64, mask = exact_case(c, seed=c.n * 7 + c.W)
        for est in exact_estimators(c):
            want = torch.from_numpy(P.returns_f64(r64, mask, c.start, est, c.n, 1.0, bool(c.mask_out)))
            got = k4r_restated(r64, mask, c, est)
            assert torch.equal(got.double(), want.to(c.out).double()), (c.id, est)
    g = torch.Generator().manual_seed(c.n * 3 + c.W)
    r = (0.3 * torch.randn(c.B, c.W, generator=g, dtype=F64)).to(c.dt)
    mask = torch.rand(c.B, c.W, generator=g) > 0.1
    eps = {BF: 2.0 ** -7, F16: 2.0 ** -10, F32: 2.0 ** -20}[rc_dtype(c)]
    for est in c.ests:
        want = torch.from_numpy(P.returns_f64(r.double(), mask, c.start, est, c.n, c.gamma, bool(c.mask_out)))
        got = k4r_restated(r, mask, c, est).double()
        nan = torch.isnan(got)  # fp16 group_norm of a constant group: 1e-9 rounds to 0 in fp16, 0 / 0
        assert not bool(nan.any()) or (c.dt == F16 and c.mode == 'faithful' and est == 'group_norm'), (c.id, est)
        got, want = got[~nan], want[~nan]
        scale = want.abs().max().clamp(min=1.0)
        assert float((got - want).abs().max()) <= 64 * eps * scale * (c.W - c.start + c.n) ** 0.5, (c.id, est)
