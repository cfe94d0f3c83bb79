"""The loss and score-head kernels pinned against float64 on guarded buffers (run on an H100: `pytest -m gpu`).

K2 `aa_dpo_loss`, K3 (`aa_score_head_fwd`, `aa_score_end`, `aa_score_head_bwd`), K4 `aa_ppo_prep`, K4r
`aa_ppo_returns` (its shared-memory opt-in and refusal), K5 `aa_ppo_actor_loss` / `aa_ppo_critic_loss`, the GRPO mask,
loss and group-advantage kernels, `aa_nll_mean`, `aa_masked_mean`, `aa_rm_pair_loss` and `aa_ppo_pack_metrics` are
called through the C ABI, so every stride, pitch, counter and scratch buffer is the test's own.  The shapes go past
each switch that only real sizes reach: more CTAs than one resident wave before a `last_block_arrives` reduction, the
strided warp loop of K3's capped grid, both `MAXV` instantiations of the K3 backward, every shared-memory opt-in and
refusal, and `nll_mean`'s capped grid.

Guarded buffers.  Every output sits in the middle of one allocation between guard bands of at least one row and 256
bytes.  Outputs start as a NaN bit pattern (POISON), guards and pad columns as a finite SENTINEL: a skipped write leaves
POISON, a stray write changes a SENTINEL.  Inputs with a row stride above their width carry NaN in the pad columns and
sit between NaN rows, so a read past a row reaches the result as a NaN.  Each launch gets its own zeroed counter word
and status word; after it the counter must read 0 again and the status word must hold exactly the predicted bits.

Exact arithmetic.  Most operands are small signed integers times a power of two.  Sizes and ranges are chosen so that
every sum the kernel forms is a multiple of one grid step g with sum |terms| <= 2^24 g: such a sum is exact in fp32 in
any order.  The float64 references (`ref_*` below) restate each kernel's rounding points: one fp32 rounding after
every + - * / sqrt, then the 16-bit rounding where faithful mode rounds.  Rounding a float64 result to fp32 after one
such operation on fp32 operands equals the fp32 operation itself, because 53 >= 2 * 24 + 2; for the same reason an fp32
result rounded to bf16 / f16 equals the correctly rounded 16-bit result.  So on these cases the kernels equal the
references bit for bit.  `test_exact_premise` checks the precondition for every exact operand set of the matrix on the
CPU, and `test_references_match_ref_port` holds each reference to `oracle/ref_port.py` run in float64.

Real-valued parts (log-sigmoid, exp, sums of inexact terms): f32 mode within 2e-5 relative of float64 (DESIGN section
4), or within the summation bound (n - 1) * 2^-24 * sum |x_i| where a sum's error can exceed that; faithful mode against
`oracle/ref_port.py` on ATen CUDA within 1 ulp and >= 97 % bit-identical.  K4's 16-bit chain is bit-identical.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from align_anything_b200 import _lib as Lb
from oracle import ref_port as O
from test_gpu_parity import assert_ulp_close, ops  # noqa: F401

DEV = 'cuda'
gpu = pytest.mark.gpu
BF, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
CODE = {BF: Lb.AA_BF16, F16: Lb.AA_F16, F32: Lb.AA_F32}
FAITHFUL, F32MODE = Lb.MODE_FAITHFUL, Lb.MODE_F32
# bit patterns: POISON is a NaN in bf16 / f16 (0x7FA5), fp32 (0x7FA5A5A5) and fp64; SENTINEL is finite (bytes: neither
# pattern is 0 or 1, so a byte mask output shows both a skipped and a stray write)
POISON = {1: 0xA5, 2: 0x7FA5, 4: 0x7FA5A5A5, 8: 0x7FA5A5A5A5A5A5A5}
SENTINEL = {1: 0x5A, 2: 0x3C5A, 4: 0x3C5A5A5A, 8: 0x3C5A5A5A5A5A5A5A}
INT = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}
EXACT = 2 ** 24
U = 2.0 ** -24
SEED = 4321
ERR_ALIGN, ERR_UNSUPPORTED = -3, -4  # AA_ERR_ALIGN, AA_ERR_UNSUPPORTED


def _up(x, m):
    return (x + m - 1) // m * m


def _stream():
    return Lb.stream_ptr(torch.device(DEV))


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- rounding restated -----------------------------------------------------------------------------------------------
def f32(x):
    """One fp32 rounding of a float64 value."""
    return x.float().double()


def rnd(x, dt):
    """The kernels' `round_to` after an fp32 operation: fp32 first, then the 16-bit dtype (None / fp32: fp32 only)."""
    x = x.float()
    return (x if dt in (None, F32) else x.to(dt)).double()


def grid_exp(v):
    """The smallest k with every v * 2^k an integer (v float64, finite)."""
    v = v[torch.isfinite(v)]
    for k in range(-30, 80):
        s = v * 2.0 ** k
        if bool((s == torch.round(s)).all()):
            return k
    return None


def sum_exact(v, dim=None):
    """True when every partial sum of v (along `dim`, in any order) is exact in fp32: all terms on one grid 2^-k and
    sum |v| <= 2^24 * 2^-k."""
    v = v.double()
    k = grid_exp(v)
    if k is None:
        return False
    a = v.abs().sum() if dim is None else v.abs().sum(dim)
    return bool((a * 2.0 ** k <= EXACT).all())


def same(got, want):
    """Equal values (NaN where the other is NaN; +0 == -0)."""
    got, want = got.double().cpu(), want.double().cpu()
    if got.shape != want.shape or not torch.equal(torch.isnan(got), torch.isnan(want)):
        return False
    return torch.equal(torch.nan_to_num(got), torch.nan_to_num(want))


def assert_same(got, want, what):
    if not same(got, want):
        g, w = got.double().cpu().reshape(-1), want.double().cpu().reshape(-1)
        bad = ~((g == w) | (torch.isnan(g) & torch.isnan(w)))
        i = int(bad.nonzero()[0]) if bool(bad.any()) else 0
        raise AssertionError(f'{what}: {int(bad.sum())} of {g.numel()} differ, first at {i}: got {float(g[i])!r}, '
                             f'want {float(w[i])!r}')


def assert_within(got, want, tol, what):
    """|got - want| <= tol element by element, NaN where want is NaN."""
    got, want = got.double().cpu(), want.double().cpu()
    tol = torch.as_tensor(tol, dtype=F64).cpu().expand_as(want)
    assert torch.equal(torch.isnan(got), torch.isnan(want)), f'{what}: NaN pattern differs'
    err = (torch.nan_to_num(got) - torch.nan_to_num(want)).abs()
    bad = err > tol
    assert not bool(bad.any()), (f'{what}: {int(bad.sum())} beyond the bar, max err {float(err.max()):.3e} '
                                 f'(bar there {float(tol.reshape(-1)[int(bad.reshape(-1).nonzero()[0])]):.3e})')


def rel(want, r=2e-5):
    """DESIGN section 4's bar: 2e-5 relative (the tiny floor keeps a zero reference from demanding an exact zero)."""
    return r * want.double().abs().cpu() + 1e-30


def half_ulp(want, dt):
    """Half an ulp of a 16-bit dtype at |want|: the final rounding of an fp32 result into a 16-bit output."""
    if dt in (None, F32):
        return torch.zeros_like(want.double().cpu())
    fi = torch.finfo(dt)
    a = want.double().abs().cpu().clamp(min=fi.tiny)
    return torch.exp2(torch.floor(torch.log2(a))) * fi.eps / 2 + fi.tiny * fi.eps / 2


# ---- guarded buffers, fenced operands, own words ---------------------------------------------------------------------
class Guarded:
    """A (rows, cols) region with row pitch `pitch` inside one allocation, 16-byte aligned, between guard bands of at
    least one row and 256 bytes.  Region elements start as POISON, guards and pad columns [cols, pitch) as SENTINEL."""

    def __init__(self, rows, cols, dtype, pitch=None):
        pitch = cols if pitch is None else pitch
        esz = torch.empty(0, dtype=dtype).element_size()
        q = max(1, 16 // esz)
        self.pre = _up(max(pitch, 256 // esz), q)
        post = _up(pitch + 256 // esz, q)
        self.rows, self.cols, self.pitch, self.esz, self.dtype = rows, cols, pitch, esz, dtype
        self.buf = torch.empty(self.pre + rows * pitch + post, dtype=dtype, device=DEV)
        self.bits = self.buf.view(INT[esz]) if dtype != INT[esz] else self.buf
        self.bits.fill_(SENTINEL[esz])
        self.region_bits().fill_(POISON[esz])
        self.fresh = self.bits.clone()
        self.t = self.buf.as_strided((rows, cols), (pitch, 1), self.pre)

    def region_bits(self):
        return self.bits.as_strided((self.rows, self.cols), (self.pitch, 1), self.pre)

    def ptr(self):
        return self.t.data_ptr()

    @property
    def flat(self):
        return self.t.reshape(-1)

    def outside_intact(self):
        m = torch.ones(self.buf.numel(), dtype=torch.bool, device=DEV)
        m.as_strided((self.rows, self.cols), (self.pitch, 1), self.pre).fill_(False)
        return torch.equal(self.bits[m], self.fresh[m])

    def untouched(self):
        return torch.equal(self.bits, self.fresh)

    def unwritten(self):
        """bool (rows, cols): elements still holding POISON."""
        return self.region_bits() == POISON[self.esz]

    def check(self, what, written=None):
        """Guards and pad columns unchanged; `written` (bool (rows, cols), default all) elements no longer POISON, the
        rest still POISON."""
        assert self.outside_intact(), f'{what}: a guard or pad word changed'
        un = self.unwritten()
        if written is None:
            assert not bool(un.any()), f'{what}: {int(un.sum())} elements left unwritten'
        else:
            written = written.to(DEV)
            assert not bool((un & written).any()), f'{what}: {int((un & written).sum())} elements left unwritten'
            assert bool(un[~written].all()), f'{what}: {int((~un[~written]).sum())} elements written outside the contract'


def fenced(values, stride=None, pad=None, reach=0):
    """`values` (rows, cols) placed between fence rows (>= 256 bytes and >= `reach` elements on each side) in an
    allocation of row stride `stride` >= cols; fence rows and pad columns hold `pad` (NaN for floats).  Returns the
    (rows, cols) view."""
    rows, cols = values.shape
    stride = cols if stride is None else stride
    if pad is None:
        pad = float('nan') if values.is_floating_point() else -7
    esz = values.element_size()
    extra = max(2, -(-max(256, reach * esz) // max(stride * esz, 1)))
    buf = torch.full((rows + 2 * extra, max(stride, 1)), pad, dtype=values.dtype, device=DEV)
    buf[extra:extra + rows, :cols] = values.to(DEV)
    return buf[extra:extra + rows, :cols]


def fenced_vec(values, pad=None):
    return fenced(values.reshape(1, -1), pad=pad)[0]


class Words:
    """Counter / status words of the test's own: int32 [n] in the middle of a zeroed block, starting at `value`."""

    def __init__(self, n=1, value=0):
        self.n = n
        self.buf = torch.zeros(32 + n, dtype=torch.int32, device=DEV)
        self.buf[16:16 + n] = value

    def ptr(self):
        return self.buf.data_ptr() + 64

    def values(self):
        return self.buf[16:16 + self.n].tolist()

    def check(self, want, what):
        assert self.values() == list(want), f'{what}: words {self.values()} != {list(want)}'
        assert int(self.buf[:16].abs().sum()) == 0 and int(self.buf[16 + self.n:].abs().sum()) == 0, f'{what}: guard'


def _p(t):
    """Device address of a view, also of an empty one (whose data_ptr() is 0)."""
    return t.data_ptr() or t.untyped_storage().data_ptr()


def rc_ok(rc, what):
    if rc != 0:
        raise AssertionError(f'{what}: rc {rc}: {Lb.lib().aa_last_error().decode(errors="replace")}')


def exact_ints(shape, q, e, seed, device=DEV, zero_share=4, nonpos=False):
    """float64 integers in [-q, q] (or [-q, 0]) times 2^e, roughly 1 in `zero_share` more of them zero."""
    gen = torch.Generator(device=device).manual_seed(seed)
    v = torch.randint(-q, 1 if nonpos else q + 1, shape, generator=gen, device=device, dtype=torch.int32)
    v = v * (torch.randint(0, zero_share, shape, generator=gen, device=device, dtype=torch.int32) != 0)
    return v.double() * 2.0 ** e


def pow2_mask(B, W, seed, device=DEV):
    """(B, W) bool with 2^floor(log2(W)) / 2 (at least 1) set positions per row, at random places."""
    cnt = max(1, (1 << (W.bit_length() - 1)) // 2) if W > 1 else 1
    gen = torch.Generator(device=device).manual_seed(seed)
    order = torch.rand(B, W, generator=gen, device=device).argsort(1)[:, :cnt]
    m = torch.zeros(B, W, dtype=torch.bool, device=device)
    m.scatter_(1, order, True)
    return m


# ---- float64 references ----------------------------------------------------------------------------------------------
def dlogsig(z):
    return torch.sigmoid(-z)


def ref_dpo(pol, ref, B, beta, valid, rd):
    """K2 with its rounding points (rd: the dtype faithful mode rounds to, None in f32 mode).  pol / ref (2B, W)
    float64.  -> dict of float64 tensors."""
    R = lambda x: rnd(x, rd)  # noqa: E731
    pc, pr = R(pol[:B].sum(1)), R(pol[B:].sum(1))
    qc, qr = R(ref[:B].sum(1)), R(ref[B:].sum(1))
    ratio_c, ratio_r = R(pc - qc), R(pr - qr)
    z = R(beta * R(ratio_c - ratio_r))
    loss = -R(F.logsigmoid(z))
    better, worse = R(beta * ratio_c), R(beta * ratio_r)
    v = valid.to(pol.device)
    n = v.double().sum()
    inv_n = f32(1.0 / n)
    mean = lambda x: R(f32(torch.where(v, x, 0.0).sum()) * inv_n)  # noqa: E731
    stats = torch.stack([mean(loss), mean(R(better + worse)), mean(better), mean(worse),
                         f32((v & (better > worse)).double().sum() * inv_n), mean(R(better - worse)), n])
    gl = R(inv_n)
    g = torch.where(v, R(R(-gl * dlogsig(z)) * beta), torch.zeros_like(z))
    return dict(loss=loss, better=better, worse=worse, g=g, valid=v.double(), stats=stats, z=z)


def ref_score(hidden64, w64, dt, out_dt, mode):
    s = f32(hidden64 @ w64)
    if mode == FAITHFUL:
        s = rnd(s, dt)
    return s.to(out_dt)


def last_true(mask):
    """Per row: index of the last True, -1 for an empty row."""
    W = mask.size(1)
    idx = torch.arange(W, device=mask.device).expand_as(mask)
    return torch.where(mask.bool(), idx, -1).max(1).values


def ref_prep(lp, rf, reward, values, mask, start, kc, clip, gamma, lam, rd, rew_dt, adv_dt):
    """K4 in f32-scan form (rd None, or fp32 tensors), float64.  lp / rf / values (B, W) float64 or None (GAE only:
    `reward` is then the (B, W) token rewards).  -> old_rewards, adv, ret (float64, rounded to their dtypes),
    row_stats (B, 8)."""
    B, W = values.shape
    m = mask.bool()
    end = last_true(m)
    end0 = end.clamp(min=0)
    R = lambda x: rnd(x, rd)  # noqa: E731
    if lp is not None:
        kl = R(lp - rf)
        r = R(-kc * kl)
        at_end = torch.arange(W, device=lp.device)[None, :] == end0[:, None]
        r = torch.where(at_end, R(r + R(reward)[:, None]), r)
        c = R(torch.tensor(clip, dtype=F64))
        r = torch.minimum(torch.maximum(r, -c), c)
        old = r.to(rew_dt).double()
    else:
        kl = torch.zeros_like(values)
        old = reward.to(rew_dt).double()
    sr = torch.where(m, old, 0.0)
    sv = torch.cat([torch.where(m, values, 0.0), torch.zeros(B, 1, dtype=F64, device=values.device)], 1)
    delta = sr[:, start:] + gamma * sv[:, start + 1:] - sv[:, start:W]
    assert gamma == 1.0 and lam == 1.0, 'the exact restatement is the gamma = lambda = 1 suffix sum'
    adv = delta.flip(1).cumsum(1).flip(1)
    ret = adv + sv[:, start:W]
    on = m[:, start:]
    cnt = on.double().sum(1)
    stats = torch.zeros(B, 8, dtype=F64, device=values.device)
    stats[:, 0] = R(torch.where(on, kl[:, start:], 0.0).sum(1))
    stats[:, 1] = R(torch.where(on, sr[:, start:], 0.0).sum(1))
    stats[:, 2] = cnt
    stats[:, 3] = f32(torch.where(on, adv, 0.0).sum(1) / cnt)
    stats[:, 4] = f32(torch.where(on, ret, 0.0).sum(1) / cnt)
    stats[:, 5] = end0.double()
    return old, adv.to(adv_dt).double(), ret.to(adv_dt).double(), stats, dict(delta=delta, adv=adv, ret=ret, sr=sr)


def ref_critic(x, old, ret, mask, clip, rx, rp, B):
    """K5 critic, float64 with the kernel's rounding points.  -> loss, grad (B, Wm), row_mean, row values."""
    m = mask.bool()
    cnt = m.double().sum(1)
    g_rs = rnd(rnd(rnd(torch.tensor(0.5, dtype=F64, device=x.device), rp) / B, rp)[None] / cnt, rp)[:, None]
    lo, hi = rnd(old - clip, rx), rnd(old + clip, rx)
    vc = torch.minimum(torch.maximum(x, lo), hi)
    d1, d2 = rnd(x - ret, rp), rnd(vc - ret, rp)
    l1, l2 = rnd(d1 * d1, rp), rnd(d2 * d2, rp)
    obj = torch.maximum(l1, l2)
    inr = (x >= lo) & (x <= hi)
    half = rnd(0.5 * g_rs, rp)  # a tie: maximum's backward sends round(grad / 2) down each branch
    g1 = torch.where(l1 > l2, rnd(g_rs * (2 * d1), rp), torch.where(l1 == l2, rnd(half * (2 * d1), rp), 0.0))
    g2 = torch.where(l1 < l2, torch.where(inr, rnd(g_rs * (2 * d2), rp), 0.0),
                     torch.where(l1 == l2, torch.where(inr, rnd(half * (2 * d2), rp), 0.0), 0.0))
    grad = torch.where(m, rnd(rnd(g1, rx) + rnd(g2, rx), rx), 0.0)
    rows = rnd(rnd(torch.where(m, rnd(obj, rp), 0.0).sum(1), rp) / cnt, rp)
    mm = rnd(f32(rows.sum()) / B, rp)
    loss = rnd(0.5 * mm, rp)
    row_mean = f32(f32(torch.where(m, x, 0.0).sum(1)) / cnt)
    return loss, grad, row_mean, rows


def ref_actor(x, old, adv, mask, clip, B):
    """K5 actor in float64 (f32 mode): loss, d loss / d x."""
    m = mask.bool().double()
    cnt = m.sum(1, keepdim=True)
    ratio = torch.exp(x - old)
    s1, s2 = adv * ratio, adv * ratio.clamp(1 - clip, 1 + clip)
    obj = torch.minimum(s1, s2)
    loss = -((obj * m).sum(1) / cnt[:, 0]).mean()
    g_rs = -1.0 / B / cnt
    inr = (ratio >= 1 - clip) & (ratio <= 1 + clip)
    gs = torch.where(s1 < s2, g_rs * adv, torch.where(s1 == s2, torch.where(inr, g_rs * adv, 0.5 * g_rs * adv), 0.0))
    return loss, gs * ratio * m, obj


def ref_grpo(lp, rf, A, row_end, beta):
    """GRPO loss, float64: loss, d loss / d lp, per-token loss, |terms| of the gradient."""
    K = lp.size(1)
    on = torch.arange(K, device=lp.device)[None, :] < row_end[:, None]
    total = on.double().sum()
    d = rf - lp
    e = torch.exp(d)
    kl = e - d - 1
    ptl = -(A[:, None] - beta * kl)
    loss = torch.where(on, ptl, 0.0).sum() / total
    gt = 1.0 / total
    c1, gkl, c2 = -gt * A[:, None].expand_as(lp), gt * beta, -gt * beta * e
    grad = torch.where(on, c1 + gkl + c2, 0.0)
    return loss, grad, ptl, on, (c1.abs() + abs(gkl) + c2.abs())


def grpo_row_end(tokens, eos):
    K = tokens.size(1)
    hit = tokens == eos
    first = torch.where(hit, torch.arange(K, device=tokens.device)[None, :], K).min(1).values
    return torch.where(first < K, first + 1, K)


def ref_group_adv(r):
    G = r.size(1)
    mean = r.mean(1, keepdim=True)
    sd = r.std(1, keepdim=True) if G > 1 else torch.full_like(mean, float('nan'))
    return (r - mean) / (sd + 1e-4)


def ref_rm(h, l, reg):
    B = h.numel()
    z = h - l
    loss = (-F.logsigmoid(z)).mean()
    if reg > 0:
        loss = loss + reg * torch.cat([l, h]).square().mean()
    ds = -dlogsig(z) / B
    r = reg / B if reg > 0 else 0.0
    return loss, torch.cat([ds + r * h, -ds + r * l]), (h > l).double().mean()


# ---- CPU: the premise and the references -----------------------------------------------------------------------------
DPO_B = [1, 2, 127, 128, 129, 1000, 4500]
DPO_W = [0, 1, 31, 129, 2047]
BETA = 2.0 ** -3


def dpo_shape(B, width):
    """(columns holding nonzero log-probs, integer range): B * nz * q <= 2^22 keeps every pair-level sum exact."""
    nz = min(width, 2 ** 22 // (B * 8))
    q = max(1, min(8, 2 ** 22 // (B * max(nz, 1))))
    return nz, q


def dpo_operands(B, width, seed, device=DEV):
    nz, q = dpo_shape(B, width)
    out = []
    for k in range(2):
        v = torch.zeros(2 * B, width, dtype=F64, device=device)
        v[:, :nz] = exact_ints((2 * B, nz), q, -3, seed + k, device, nonpos=True)
        out.append(v)
    return out


def dpo_valid(B, ids_kind):
    if ids_kind == 'none':
        return torch.ones(B, dtype=torch.bool)
    if ids_kind == 'all':
        return torch.zeros(B, dtype=torch.bool)
    return torch.arange(B) % 3 != 1


# K4: (W, start kind); the operands are sparse so that the suffix sums and their row sums stay exact
PREP_W = [1, 33, 4095, 4096, 17065]
PREP_START = ['0', 'half', 'last']
PREP_KC, PREP_CLIP = 0.5, 8.0


def prep_start(W, kind):
    return {'0': 0, 'half': W // 2, 'last': W - 1}[kind]


def prep_masks(W, start, with_empty, device=DEV):
    rows = [torch.ones(W, dtype=torch.bool)]
    holes = torch.ones(W, dtype=torch.bool)
    holes[1::3] = False
    if W > 8:
        holes[W // 2:W // 2 + 5] = False
    rows.append(holes)
    before = torch.zeros(W, dtype=torch.bool)
    before[:max(start, 1)] = True
    before[max(start, 1) - 1] = True
    rows.append(before)
    if with_empty:
        rows.append(torch.zeros(W, dtype=torch.bool))
    return torch.stack(rows).to(device)


def prep_operands(B, W, seed, device=DEV):
    """lp, ref, values (B, W) and reward (B,): integers times 2^-2, nonzero on at most 8 positions per row beyond
    W = 1024 (kl is nonzero only where lp and ref differ)."""
    gen = torch.Generator(device=device).manual_seed(seed)
    lp = exact_ints((B, W), 4, -2, seed, device, nonpos=True)
    rf = lp.clone()
    vals = exact_ints((B, W), 4, -2, seed + 1, device)
    dk = exact_ints((B, W), 4, -2, seed + 2, device)
    if W > 1024:
        keep = torch.zeros(B, W, dtype=torch.bool, device=device)
        keep.scatter_(1, torch.randint(0, W, (B, 8), generator=gen, device=device), True)
        dk = torch.where(keep, dk, 0.0)
        keep2 = torch.zeros(B, W, dtype=torch.bool, device=device)
        keep2.scatter_(1, torch.randint(0, W, (B, 8), generator=gen, device=device), True)
        vals = torch.where(keep2, vals, 0.0)
    rf = rf + dk
    reward = exact_ints((B,), 8, -2, seed + 3, device)
    return lp, rf, vals, reward


def prep_exact(delta, on_adv, adv, ret, start):
    """The premise of the f32 scan: suffix sums, their masked row sums and the returns exact in any order."""
    ok = sum_exact(delta, 1)
    # every partial sum of the scan is bounded by the suffix sums of |delta|; their row sum bounds the adv row sum
    k = grid_exp(torch.cat([delta.reshape(-1), ret.reshape(-1)]))
    bound = delta.abs().flip(1).cumsum(1).flip(1).sum(1) + ret.abs().sum(1)
    return ok and k is not None and bool((bound * 2.0 ** k <= EXACT).all())


def test_exact_premise():
    """No GPU: for every exact operand set of the matrix the values are exact in each dtype used, lie on their grid,
    and every sum the kernels form is exact in any order."""
    torch.manual_seed(0)
    for B in DPO_B:
        for width in DPO_W:
            nz, q = dpo_shape(B, width)
            assert B * max(nz, 1) * q <= 2 ** 22 or nz == 0
            pol, ref = dpo_operands(B, width, SEED + B + width, 'cpu')
            for dt in (BF, F16):
                assert torch.equal(pol.to(dt).double(), pol) and torch.equal(ref.to(dt).double(), ref)
            assert sum_exact(pol, 1) and sum_exact(ref, 1)
            for rd in (None, BF, F16):
                for kind in ('none', 'some'):
                    r = ref_dpo(pol, ref, B, BETA, dpo_valid(B, kind), rd)
                    v = r['valid'].bool()
                    for name, x in (('better', r['better']), ('worse', r['worse']),
                                    ('reward', rnd(r['better'] + r['worse'], rd)),
                                    ('margin', rnd(r['better'] - r['worse'], rd))):
                        assert sum_exact(x[v]), (B, width, rd, name)
    # K3: |hidden| <= 7 * 2^-3, |w| <= 7 * 2^-4, |g| <= 7 * 2^-2: H * 49 and rows * 49 products of one grid
    for H in SCORE_H[F32] + BWD_H[BF] + BWD_H[F32]:
        assert H * 7 * 7 <= EXACT
    for rows in SCORE_ROWS + BWD_ROWS:
        assert rows * 7 * 7 <= EXACT
    hs = exact_ints((64, 96), 7, -3, 1, 'cpu')
    for dt in (BF, F16):
        assert torch.equal(hs.to(dt).double(), hs)
        prod = hs * exact_ints((1, 96), 7, -4, 2, 'cpu')
        assert torch.equal(prod.to(dt).double(), prod)  # grad_hidden = g * w is exact in every dtype
    # K4: the f32 scan on every (W, start)
    for W in PREP_W:
        for sk in PREP_START:
            start = prep_start(W, sk)
            lp, rf, vals, rew = prep_operands(4, W, SEED + W, 'cpu')
            mask = prep_masks(W, start, True, 'cpu')
            for dt in (BF, F16):
                for x in (lp, rf, vals, rew):
                    assert torch.equal(x.to(dt).double(), x)
                old, adv, ret, stats, aux = ref_prep(lp, rf, rew, vals, mask, start, PREP_KC, PREP_CLIP, 1.0, 1.0,
                                                     None, dt, dt)
                assert torch.equal(old.to(dt).double(), old)
            assert prep_exact(aux['delta'], mask[:, start:], aux['adv'], aux['ret'], start), (W, start)
            assert sum_exact(torch.where(mask[:, start:], aux['sr'][:, start:], 0.0), 1)
    # K5 critic: per-token terms and the row sums on a power-of-two mask count
    for B in ACTOR_B:
        for Wm in ACTOR_W:
            x, old, ret, mask = critic_operands(B, Wm, SEED + B + Wm, 'cpu')
            for dt in (BF, F16):
                for t in (x, old, ret):
                    assert torch.equal(t.to(dt).double(), t)
            for rd in (None, BF, F16):
                _, _, _, rows = ref_critic(x, old, ret, mask, CRITIC_CLIP, rd, rd, B)
                d = (x - ret).abs().max() + CRITIC_CLIP
                assert Wm * float(d * d) * 2.0 ** 8 <= EXACT  # sum of squares on the 2^-8 grid
    # nll_mean and masked_mean
    for n in NLL_N:
        assert n * NLL_Q <= EXACT  # integers times 2^-3, |x| <= q: in units of 2^-3
    for B in MM_B:
        assert B * MM_W * 7 <= EXACT


def test_references_match_ref_port():
    """No GPU: every float64 reference of this file against oracle/ref_port.py run in float64 on small inputs."""
    gen = torch.Generator().manual_seed(7)
    B, W = 5, 9
    pol = -torch.rand(2 * B, W, generator=gen, dtype=F64) * 3
    rf = -torch.rand(2 * B, W, generator=gen, dtype=F64) * 3
    valid = torch.tensor([True, False, True, True, False])
    ids = torch.randint(0, 9, (2 * B, 4), generator=gen)
    ids[B:][~valid] = ids[:B][~valid]
    mine = ref_dpo(pol, rf, B, 0.1, valid, None)
    leaf = pol.clone().requires_grad_(True)
    want = O.dpo_loss(leaf, rf, 0.1, ids, skip_identical_pairs=True)
    want['loss'].backward()
    assert torch.allclose(mine['stats'][0], want['loss'], rtol=1e-6, atol=1e-9)
    assert torch.allclose(mine['better'][valid], want['better_sample_reward'], rtol=1e-6, atol=1e-9)
    assert torch.allclose(mine['stats'][4], want['reward_accuracy'].double(), rtol=1e-6)
    assert torch.allclose(mine['stats'][5], want['reward_margin'].mean(), rtol=1e-6, atol=1e-9)
    assert torch.allclose(mine['g'], leaf.grad[:B, 0], rtol=1e-6, atol=1e-9) and torch.allclose(-mine['g'], leaf.grad[B:, 0])

    h = torch.randn(3, 4, 16, generator=gen, dtype=F64)
    w = torch.randn(1, 16, generator=gen, dtype=F64)
    m = torch.tensor([[1, 1, 0, 0], [1, 1, 1, 1], [0, 1, 0, 1]], dtype=torch.bool)
    sh = O.score_head(h, w, m)
    assert torch.allclose(ref_score(h.reshape(-1, 16), w[0], F32, F64, F32MODE).reshape(3, 4), sh['scores'][..., 0].double(),
                          rtol=1e-6)
    assert torch.equal(last_true(m), sh['end_index'])

    W, start = 11, 4
    lp = -torch.rand(3, W, generator=gen, dtype=F64)
    rfl = -torch.rand(3, W, generator=gen, dtype=F64)
    vals = torch.randn(3, W, generator=gen, dtype=F64)
    rew = torch.randn(3, generator=gen, dtype=F64)
    mk = torch.ones(3, W, dtype=torch.bool)
    mk[1, 7:] = False
    mk[2, ::2] = False
    old, adv, ret, stats, _ = ref_prep(lp, rfl, rew, vals, mk, start, 0.1, 0.3, 1.0, 1.0, None, F64, F64)
    w_old = O.kl_shaped_rewards(rew, lp, rfl, mk, 0.1, 0.3)
    w_adv, w_ret = O.gae_advantages_and_returns(vals, w_old, mk, start, 1.0, 1.0)
    assert torch.allclose(old, w_old, rtol=1e-6, atol=1e-7)
    assert torch.allclose(adv, w_adv, rtol=1e-6, atol=1e-6) and torch.allclose(ret, w_ret, rtol=1e-6, atol=1e-6)
    mm = mk[:, start:]
    assert torch.allclose(stats[:, 3], (w_adv * mm).sum(1) / mm.sum(1), rtol=1e-6)

    x = torch.randn(4, 6, generator=gen, dtype=F64)
    o = x + 0.3 * torch.randn(4, 6, generator=gen, dtype=F64)
    rt = torch.randn(4, 6, generator=gen, dtype=F64)
    mk = torch.rand(4, 6, generator=gen) > 0.3
    mk[:, 0] = True
    leaf = x.clone().requires_grad_(True)
    want = O.critic_loss(leaf, o, rt, mk, 0.2)
    want.backward()
    loss, grad, _, _ = ref_critic(x, o, rt, mk, 0.2, F64, F64, 4)
    assert torch.allclose(loss, want, rtol=1e-6) and torch.allclose(grad, leaf.grad, rtol=1e-6, atol=1e-12)
    # the 16-bit rounding points, ties included, against autograd on ATen (CPU): at B = 4500 the halved tie gradients
    # are fp16 subnormals
    xc, oc, rc, mc = critic_operands(4500, 128, 99, 'cpu')
    for dt in (BF, F16):
        leaf16 = xc.to(dt).requires_grad_(True)
        O.critic_loss(leaf16, oc.to(dt), rc.to(dt), mc, CRITIC_CLIP).backward()
        _, grad16, _, _ = ref_critic(xc, oc, rc, mc, CRITIC_CLIP, dt, dt, 4500)
        assert_same(grad16.to(dt), leaf16.grad, f'critic {dt} gradient vs autograd')  # values: -0 == +0
    leaf = x.clone().requires_grad_(True)
    want = O.actor_loss(leaf, o, rt, mk, 0.2)
    want.backward()
    loss, grad, _ = ref_actor(x, o, rt, mk, 0.2, 4)
    assert torch.allclose(loss, want, rtol=1e-6, atol=1e-9) and torch.allclose(grad, leaf.grad, rtol=1e-6, atol=1e-9)

    lp = -torch.rand(4, 7, generator=gen, dtype=F64)
    rfl = -torch.rand(4, 7, generator=gen, dtype=F64)
    A = torch.randn(4, generator=gen, dtype=F64)
    tok = torch.randint(0, 5, (4, 7), generator=gen)
    leaf = lp.clone().requires_grad_(True)
    want = O.grpo_loss(leaf, rfl, A[:, None], tok, 0, 3, 0.04)
    want.backward()
    loss, grad, _, _, _ = ref_grpo(lp, rfl, A, grpo_row_end(tok, 3), 0.04)
    assert torch.allclose(loss, want, rtol=1e-6, atol=1e-9) and torch.allclose(grad, leaf.grad, rtol=1e-6, atol=1e-9)

    r = torch.randn(3, 5, generator=gen, dtype=F64)
    assert torch.allclose(ref_group_adv(r).reshape(-1, 1), O.grpo_group_advantages(r.reshape(-1), 3, 5), rtol=1e-6, atol=1e-9)
    assert torch.isnan(ref_group_adv(r[:, :1])).all()

    x = torch.randn(3, 5, generator=gen, dtype=F64)
    mk = torch.rand(3, 5, generator=gen) > 0.4
    mk[:, 0] = True
    assert torch.allclose(ref_masked_mean(x, mk), O.masked_mean(x, mk), rtol=1e-6, atol=1e-9)
    assert torch.allclose(ref_masked_mean(x, None), O.masked_mean(x), rtol=1e-6, atol=1e-9)

    es = torch.randn(8, generator=gen, dtype=F64)
    leaf = es.clone().requires_grad_(True)
    want = O.rm_pair_loss(leaf.view(8, 1, 1), leaf.view(8, 1), 0.01)
    want['loss'].backward()
    loss, grad, acc = ref_rm(es[:4], es[4:], 0.01)
    assert torch.allclose(loss, want['loss'], rtol=1e-6, atol=1e-9) and torch.allclose(grad, leaf.grad, rtol=1e-6, atol=1e-9)
    assert torch.allclose(acc, want['accuracy'].double())

    logits = torch.randn(2, 6, 5, generator=gen, dtype=F64)
    labels = torch.randint(0, 5, (2, 6), generator=gen)
    labels[0, 2] = -100
    shifted = F.pad(labels, (0, 1), value=-100)[..., 1:]
    lpt = O.token_log_probs(logits, shifted.clamp(min=0))
    assert torch.allclose(ref_nll(lpt.reshape(-1), shifted.reshape(-1), -100), O.causal_lm_loss(logits, labels).double(),
                          rtol=1e-6, atol=1e-9)


def ref_masked_mean(x, mask):
    if mask is None:
        return x.mean()
    return ((x * mask).sum(1) / mask.sum(1)).mean()


def ref_nll(logp, labels, ignore):
    keep = labels != ignore
    return -(torch.where(keep, logp, 0.0).sum()) / keep.sum()


# ---- K2 --------------------------------------------------------------------------------------------------------------
def _dpo_ids(B, L, kind):
    gen = torch.Generator().manual_seed(B + L)
    ids = torch.randint(0, 1000, (2 * B, L), generator=gen)
    same_rows = ~dpo_valid(B, kind)
    ids[B:][same_rows] = ids[:B][same_rows]
    if kind != 'all':
        ids[B:, L - 1][~same_rows] = ids[:B, L - 1][~same_rows] + 1  # differ only in the last column
    return ids


@gpu
@pytest.mark.parametrize('B', DPO_B)
@pytest.mark.parametrize('width', DPO_W)
def test_dpo_loss(ops, B, width):
    pol64, ref64 = dpo_operands(B, width, SEED + B + width)
    L = 9
    for stride in sorted({width, width + 5}):
        for dt in (BF, F16, F32):
            pol, ref = fenced(pol64.to(dt), stride), fenced(ref64.to(dt), stride)
            for mode in (FAITHFUL, F32MODE):
                rd = dt if mode == FAITHFUL and dt != F32 else None
                for kind in ('none', 'some', 'all'):
                    what = f'K2 B={B} w={width} stride={stride} {dt} mode={mode} ids={kind}'
                    ids = None if kind == 'none' else fenced(_dpo_ids(B, L, kind), L + 3)
                    valid = dpo_valid(B, kind)
                    per_pair = Guarded(5, B, F32)
                    grad_seg = Guarded(1, 2 * B, F32)
                    stats = Guarded(1, 8, F32)
                    counter, status = Words(), Words(value=6)
                    rc_ok(Lb.lib().aa_dpo_loss(_p(pol), _p(ref), CODE[dt], B, width, stride, BETA, mode,
                                               Lb.ptr(ids), L, L + 3, per_pair.ptr(), grad_seg.ptr(), stats.ptr(),
                                               counter.ptr(), None, None, status.ptr(), _stream()), what)
                    torch.cuda.synchronize()
                    per_pair.check(what + ' per_pair')
                    grad_seg.check(what + ' grad_seg')
                    stats.check(what + ' stats')
                    counter.check([0], what + ' counter')
                    status.check([6], what + ' status')
                    r = ref_dpo(pol64, ref64, B, BETA, valid.to(DEV), rd)
                    pp, st = per_pair.t.double(), stats.t[0].double()
                    for lane, key in ((1, 'better'), (2, 'worse'), (4, 'valid')):
                        assert_same(pp[lane], r[key], f'{what} per_pair[{lane}] {key}')
                    assert_same(st[1:7], r['stats'][1:7], what + ' stats[1:7]')
                    assert float(st[7]) == 6.0, what + ' stats[7] carries the status word'
                    gs = grad_seg.t[0]
                    assert torch.equal(gs[:B].view(torch.int32), per_pair.t[3].view(torch.int32)), what + ' +g'
                    assert torch.equal(gs[B:].view(torch.int32), (-per_pair.t[3]).view(torch.int32)), what + ' -g'
                    if kind == 'all':
                        assert bool((per_pair.t[3] == 0).all()) and float(st[6]) == 0.0
                        assert bool(torch.isnan(st[:6]).all()), what + ' empty mean is NaN'
                        continue
                    if rd is None:
                        assert_within(pp[0], r['loss'], rel(r['loss']) + 4 * U * r['loss'].abs().cpu(), what + ' loss')
                        assert_within(pp[3], r['g'], rel(r['g']), what + ' g')
                        n = float(r['stats'][6])
                        sl = torch.where(r['valid'].bool(), r['loss'], 0.0).abs().sum() / n
                        assert_within(st[0], r['stats'][0], rel(r['stats'][0]) + (n + 4) * U * sl.cpu(), what + ' loss')
                    else:
                        # faithful: the float64 restatement rounded to dt, within 1 ulp (the fp32 log-sigmoid / exp
                        # may sit on the other side of a 16-bit rounding boundary)
                        assert_ulp_close(pp[0].to(dt), r['loss'].to(dt), max_ulp=1, min_exact=0.97, what=what + ' loss')
                        assert_ulp_close(pp[3].to(dt), r['g'].to(dt), max_ulp=1, min_exact=0.97, what=what + ' g')
                        assert_ulp_close(st[:1].to(dt), r['stats'][:1].to(dt), max_ulp=1, min_exact=0.0,
                                         what=what + ' stats[0]')
                        if B <= 129 and width > 0 and stride == width:
                            _dpo_vs_ref_port(pol, ref, ids, kind, per_pair, stats, dt, B, what)


def _dpo_vs_ref_port(pol, ref, ids, kind, per_pair, stats, dt, B, what):
    leaf = pol.detach().clone().requires_grad_(True)
    want = O.dpo_loss(leaf, ref, BETA, ids, skip_identical_pairs=kind != 'none')
    want['loss'].backward()
    v = dpo_valid(B, kind).to(DEV)
    assert_ulp_close(stats.t[0, :1].to(dt), want['loss'].reshape(1), max_ulp=1, min_exact=0.0, what=what + ' vs ATen loss')
    assert_ulp_close(per_pair.t[1][v].to(dt), want['better_sample_reward'], min_exact=0.97, what=what + ' vs ATen better')
    assert_ulp_close(per_pair.t[3].to(dt), leaf.grad[:B, 0], min_exact=0.97, what=what + ' vs ATen g')


# ---- K3 forward ------------------------------------------------------------------------------------------------------
SCORE_H = {BF: [8, 100, 3584, 4096, 8192], F16: [8, 100, 3584, 4096, 8192], F32: [8, 100, 3584, 4096, 8192, 12289]}
SCORE_ROWS = [1, 9, 4224, 4225, 40000]
SCORE_CASES = [(dt, H, rows) for dt in (BF, F16, F32) for H in SCORE_H[dt] for rows in SCORE_ROWS]


def _layouts(values, H):
    """The same (rows, H) operand with row stride H, H + 8, and one element off 16-byte alignment (odd stride)."""
    yield 'contig', fenced(values, H)
    yield 'pitch', fenced(values, H + 8)
    rows = values.size(0)
    wide = torch.cat([torch.full((rows, 1), float('nan'), dtype=values.dtype, device=DEV), values.to(DEV)], 1)
    yield 'odd', fenced(wide, H + 9)[:, 1:]


@gpu
@pytest.mark.parametrize('dt,H,rows', SCORE_CASES, ids=[f'{str(d)[6:]}-H{h}-r{r}' for d, h, r in SCORE_CASES])
def test_score_head_forward(ops, dt, H, rows):
    h64 = exact_ints((rows, H), 7, -3, SEED + H + rows)
    w64 = exact_ints((H,), 7, -4, SEED + 3 * H)
    w = fenced_vec(w64.to(dt))
    hd = h64.to(dt)
    for lay, hidden in _layouts(hd, H):
        stride = hidden.stride(0)
        if lay == 'odd':
            assert hidden.data_ptr() % 16 != 0
        for mode in (FAITHFUL, F32MODE):
            for out_dt in sorted({F32, dt}, key=str):
                what = f'K3 fwd {dt} H={H} rows={rows} {lay} mode={mode} out={out_dt}'
                out = Guarded(rows, 1, out_dt)
                rc_ok(Lb.lib().aa_score_head_fwd(hidden.data_ptr(), CODE[dt], rows, H, stride, w.data_ptr(),
                                                 out.ptr(), CODE[out_dt], mode, _stream()), what)
                torch.cuda.synchronize()
                out.check(what)
                assert_same(out.t[:, 0], ref_score(h64, w64, dt, out_dt, mode), what)
    del hd


@gpu
@pytest.mark.parametrize('dt', [BF, F16, F32])
def test_score_head_forward_real_values(ops, dt):
    rows, H = 4225, 4096
    gen = torch.Generator(device=DEV).manual_seed(5)
    hidden = fenced(torch.randn(rows, H, generator=gen, device=DEV).to(dt), H + 8)
    w = fenced_vec((torch.randn(H, generator=gen, device=DEV) / 64).to(dt))
    for mode in (FAITHFUL, F32MODE):
        out = Guarded(rows, 1, F32)
        rc_ok(Lb.lib().aa_score_head_fwd(hidden.data_ptr(), CODE[dt], rows, H, H + 8, w.data_ptr(), out.ptr(), CODE[F32],
                                         mode, _stream()), 'fwd')
        torch.cuda.synchronize()
        out.check('fwd real')
        if mode == FAITHFUL and dt != F32:
            # an fp32 dot of H terms rounded once to dt: within the summation bound (H - 1) * 2^-24 * sum |h * w| of
            # the float64 dot, plus half an ulp of dt for the rounding (twice: at the result and at the reference)
            prod = hidden.double() * w.double()[None, :]
            want = prod.sum(1)
            tol = (H - 1) * U * prod.abs().sum(1).cpu() + 2 * half_ulp(want, dt)
            assert_within(out.t[:, 0], want, tol, f'fwd {dt} faithful')
        else:
            # fp32 dot of H terms: |err| <= (H - 1) * 2^-24 * sum |h * w| in any summation order
            prod = hidden.double() * w.double()[None, :]
            want = prod.sum(1)
            assert_within(out.t[:, 0], want, rel(want) + (H - 1) * U * prod.abs().sum(1).cpu(), f'fwd {dt} f32')


# ---- K3 end gather ---------------------------------------------------------------------------------------------------
def _end_masks(L):
    m = torch.zeros(5, L, dtype=torch.bool)
    m[0] = True
    m[1, ::2] = True
    m[1, L // 2] = True
    m[2, 0] = True
    m[4, L - 1] = True
    return m  # row 3 is empty


@gpu
@pytest.mark.parametrize('L', [1, 31, 32, 33, 4097])
def test_score_end(ops, L):
    B = 5
    mask = _end_masks(L)
    scores = fenced(torch.randn(B, L, device=DEV), L + 3)
    for hdt, H, off in ((BF, 64, 0), (BF, 100, 0), (BF, 64, 1), (F32, 100, 0), (F32, 100, 1), (F16, 40, 0)):
        hid = torch.randn(B * L, H, device=DEV).to(hdt)
        hidden = fenced(hid, H + 8)
        for kind in ('u8', 'i64', 'none'):
            what = f'score_end L={L} {hdt} H={H} off={off} mask={kind}'
            if kind == 'none':
                mptr, mk, mstride, want_end = None, Lb.MASK_U8, 0, torch.full((B,), L - 1)
            else:
                mt = fenced(mask.to(torch.uint8 if kind == 'u8' else torch.int64), L + 5, pad=1)
                mptr, mk, mstride = mt.data_ptr(), (Lb.MASK_U8 if kind == 'u8' else Lb.MASK_I64), L + 5
                want_end = last_true(mask).clamp(min=0)
            end_index = Guarded(B, 1, torch.int64)
            end_scores = Guarded(B, 1, F32)
            end_hidden = Guarded(1, B * H + off, hdt)
            status = Words()
            rc_ok(Lb.lib().aa_score_end(scores.data_ptr(), CODE[F32], L + 3, mptr, mk, mstride, B, L, end_index.ptr(),
                                        end_scores.ptr(), hidden.data_ptr(), CODE[hdt], L * (H + 8), H + 8, H,
                                        end_hidden.ptr() + off * end_hidden.esz, status.ptr(), _stream()), what)
            torch.cuda.synchronize()
            end_index.check(what + ' end_index')
            end_scores.check(what + ' end_scores')
            wr = torch.ones(1, B * H + off, dtype=torch.bool)
            wr[0, :off] = False
            end_hidden.check(what + ' end_hidden', wr)
            status.check([Lb.STATUS_EMPTY_MASK if kind != 'none' else 0], what + ' status')
            assert torch.equal(end_index.t[:, 0].cpu(), want_end), what
            e = want_end.to(DEV)
            assert torch.equal(end_scores.t[:, 0], scores[torch.arange(B, device=DEV), e]), what
            got_h = end_hidden.flat[off:].view(B, H)
            want_h = hid.view(B, L, H)[torch.arange(B, device=DEV), e]
            assert torch.equal(got_h.view(INT[end_hidden.esz]), want_h.view(INT[end_hidden.esz])), what + ' gather'


# ---- K3 backward -----------------------------------------------------------------------------------------------------
BWD_H = {BF: [8, 4096, 4104, 8192], F32: [2048, 2052, 4096]}
BWD_ROWS = [1, 5, 263, 264, 265, 40001]
BWD_CASES = [(dt, H, rows) for dt in (BF, F32) for H in BWD_H[dt] for rows in BWD_ROWS]


def _bwd_call(hidden, dt, rows, H, w, g, gdt, gh_ptr, gh_stride, gw_ptr, part_ptr, n_out):
    return Lb.lib().aa_score_head_bwd(hidden.data_ptr(), CODE[dt], rows, H, hidden.stride(0), w.data_ptr(),
                                      g.data_ptr(), CODE[gdt], gh_ptr, gh_stride, gw_ptr, part_ptr,
                                      ctypes.byref(n_out), FAITHFUL, _stream())


@gpu
@pytest.mark.parametrize('dt,H,rows', BWD_CASES, ids=[f'{str(d)[6:]}-H{h}-r{r}' for d, h, r in BWD_CASES])
def test_score_head_backward(ops, dt, H, rows):
    h64 = exact_ints((rows, H), 7, -3, SEED + 5 * H + rows)
    w64 = exact_ints((H,), 7, -4, SEED + 7 * H)
    g64 = exact_ints((rows,), 7, -2, SEED + rows)
    E = 16 // torch.empty(0, dtype=dt).element_size()
    hidden = fenced(h64.to(dt), H + E)
    w = fenced_vec(w64.to(dt))
    want_gw = f32(g64 @ h64)
    want_gh = (g64[:, None] * w64[None, :]).to(dt)
    n_part = min(2 * _sm_count(), rows)
    for gdt in (F32, BF, F16):
        g = fenced_vec(g64.to(gdt))
        for with_gh in (True, False):
            what = f'K3 bwd {dt} H={H} rows={rows} g={gdt} grad_hidden={with_gh}'
            gh = Guarded(rows, H, dt, pitch=H + E) if with_gh else None
            gw = Guarded(1, H, F32)
            part = Guarded(n_part, H, F32)
            n_out = ctypes.c_int32(-1)
            # the size query: n_partials, and nothing written
            rc_ok(_bwd_call(hidden, dt, rows, H, w, g, gdt, gh.ptr() if gh else None, H + E, gw.ptr(), None, n_out),
                  what + ' query')
            torch.cuda.synchronize()
            assert n_out.value == n_part, (what, n_out.value, n_part)
            assert gw.untouched() and part.untouched() and (gh is None or gh.untouched()), what + ' query wrote'
            rc_ok(_bwd_call(hidden, dt, rows, H, w, g, gdt, gh.ptr() if gh else None, H + E, gw.ptr(), part.ptr(),
                            n_out), what)
            torch.cuda.synchronize()
            gw.check(what + ' grad_weight')
            part.check(what + ' partial')
            assert_same(gw.t[0], want_gw, what + ' grad_weight')
            if gh is not None:
                gh.check(what + ' grad_hidden')
                assert torch.equal(gh.t, want_gh), what + ' grad_hidden'


@gpu
def test_score_head_backward_refusals(ops):
    """H not a multiple of the vector width, H / E > 1024 and misaligned rows are refused; nothing is written."""
    cases = [(BF, 100, 0, 0, ERR_UNSUPPORTED), (BF, 8200, 0, 0, ERR_UNSUPPORTED),
             (F32, 4100, 0, 0, ERR_UNSUPPORTED), (F32, 2050, 0, 0, ERR_UNSUPPORTED),
             (BF, 64, 1, 0, ERR_ALIGN), (BF, 64, 0, 4, ERR_ALIGN), (F32, 64, 0, 1, ERR_ALIGN)]
    for dt, H, base_off, extra_stride, code in cases:
        rows = 7
        buf = torch.zeros(rows + 2, H + 16, dtype=dt, device=DEV)
        hidden = buf.view(-1)[base_off:base_off + rows * (H + extra_stride)].view(rows, H + extra_stride)[:, :H]
        w = torch.zeros(H, dtype=dt, device=DEV)
        g = torch.zeros(rows, dtype=F32, device=DEV)
        gw = Guarded(1, H, F32)
        part = Guarded(rows, H, F32)
        n_out = ctypes.c_int32(-1)
        rc = Lb.lib().aa_score_head_bwd(hidden.data_ptr(), CODE[dt], rows, H, H + extra_stride, w.data_ptr(),
                                        g.data_ptr(), CODE[F32], None, 0, gw.ptr(), part.ptr(), ctypes.byref(n_out),
                                        FAITHFUL, _stream())
        torch.cuda.synchronize()
        assert rc == code, (dt, H, base_off, extra_stride, rc)
        assert gw.untouched() and part.untouched(), (dt, H, 'refused call wrote')


# ---- K4 --------------------------------------------------------------------------------------------------------------
def _prep_call(lp, rf, rew, vals, mask, B, W, start, kc, clip, gamma, lam, mode, dts, old, adv, ret, rs, status,
               gae_only=False):
    lpdt, vdt, rdt, adt = dts
    return Lb.lib().aa_ppo_prep(
        None if gae_only else lp.data_ptr(), None if gae_only else rf.data_ptr(), CODE[lpdt],
        0 if gae_only else lp.stride(0), None if gae_only else rew.data_ptr(), vals.data_ptr(), CODE[vdt],
        vals.stride(0), mask.data_ptr(), mask.stride(0), B, W, start, kc, clip, gamma, lam, mode, old, CODE[rdt], adv,
        ret, CODE[adt], rs, status, _stream())


@gpu
@pytest.mark.parametrize('W', PREP_W)
@pytest.mark.parametrize('sk', PREP_START)
def test_ppo_prep_scan(ops, W, sk):
    """The f32 scan with gamma = lambda = 1 (a suffix sum) on exact operands: rewards, advantages, returns and the row
    statistics bit-exact, the empty row flagged, every output written and nothing else."""
    start = prep_start(W, sk)
    n = W - start
    B = 4
    lp64, rf64, v64, rew64 = prep_operands(B, W, SEED + W)
    mask = prep_masks(W, start, True)
    mt = fenced(mask, W + 3, pad=True)
    rew = fenced_vec(rew64.float())
    for dt, mode in ((F32, FAITHFUL), (F32, F32MODE), (BF, F32MODE), (F16, F32MODE)):
        lp, rf, vals = fenced(lp64.to(dt), W + 2), fenced(rf64.to(dt), W + 2), fenced(v64.to(dt), W + 1)
        for gae_only in (False, True):
            what = f'K4 W={W} start={start} {dt} mode={mode} gae_only={gae_only}'
            old_want, adv_want, ret_want, st_want, aux = ref_prep(lp64, rf64, rew64, v64, mask, start, PREP_KC,
                                                                  PREP_CLIP, 1.0, 1.0, None, dt, dt)
            if gae_only:
                tok = old_want
                old_want, adv_want, ret_want, st_want, aux = ref_prep(None, None, tok, v64, mask, start, 0.0, 0.0, 1.0,
                                                                      1.0, None, dt, dt)
                old_in = fenced(tok.to(dt), W)
                old = None
            else:
                old = Guarded(B, W, dt)
            adv, ret, rs = Guarded(B, n, dt), Guarded(B, n, dt), Guarded(B, 8, F32)
            status = Words()
            rc_ok(_prep_call(lp, rf, rew, vals, mt, B, W, start, PREP_KC, PREP_CLIP, 1.0, 1.0, mode, (dt, dt, dt, dt),
                             old_in.data_ptr() if gae_only else old.ptr(), adv.ptr(), ret.ptr(), rs.ptr(),
                             status.ptr(), gae_only), what)
            torch.cuda.synchronize()
            status.check([Lb.STATUS_EMPTY_MASK], what + ' status')
            for name, buf in (('adv', adv), ('ret', ret), ('row_stats', rs)) + ((('old_rewards', old),) if old else ()):
                buf.check(f'{what} {name}')
            if gae_only:
                assert torch.equal(old_in.double(), tok), what + ' GAE-only must not write old_rewards'
            else:
                assert_same(old.t, old_want, what + ' old_rewards')
            assert_same(adv.t, adv_want, what + ' advantages')
            assert_same(ret.t, ret_want, what + ' returns')
            assert_same(rs.t[:, :6], st_want[:, :6], what + ' row_stats[0:6]')
            assert bool((rs.t[:, 6:] == 0).all()) and not bool(torch.signbit(rs.t[:, 6:]).any()), what + ' lanes 6-7'


@gpu
@pytest.mark.parametrize('W', PREP_W)
@pytest.mark.parametrize('sk', PREP_START)
def test_ppo_prep_16bit_chain(ops, W, sk):
    """Faithful bf16 / f16: rewards, advantages and returns bit-identical to kl_shaped_rewards +
    gae_advantages_and_returns on ATen CUDA (the sequential chain reproduces each eager rounding)."""
    start = prep_start(W, sk)
    n = W - start
    B = 3
    gen = torch.Generator(device=DEV).manual_seed(W + start)
    mask = prep_masks(W, start, False)
    mt = fenced(mask, W + 3, pad=True)
    for dt in (BF, F16):
        lp = fenced((-3 * torch.rand(B, W, generator=gen, device=DEV)).to(dt), W + 2)
        rf = fenced((lp.float() + 0.2 * torch.randn(B, W, generator=gen, device=DEV)).to(dt), W + 2)
        vals = fenced(torch.randn(B, W, generator=gen, device=DEV).to(dt), W + 1)
        rew = fenced_vec(torch.randn(B, generator=gen, device=DEV))
        hp = O.PPO_DEFAULTS
        what = f'K4 chain W={W} start={start} {dt}'
        old, adv, ret, rs = Guarded(B, W, dt), Guarded(B, n, dt), Guarded(B, 8, F32), None
        ret = Guarded(B, n, dt)
        rs = Guarded(B, 8, F32)
        status = Words()
        rc_ok(_prep_call(lp, rf, rew, vals, mt, B, W, start, hp['kl_coeff'], hp['clip_range_score'], hp['gamma'],
                         hp['gae_lambda'], FAITHFUL, (dt, dt, dt, dt), old.ptr(), adv.ptr(), ret.ptr(), rs.ptr(),
                         status.ptr()), what)
        torch.cuda.synchronize()
        status.check([0], what + ' status')
        for name, buf in (('old_rewards', old), ('adv', adv), ('ret', ret), ('row_stats', rs)):
            buf.check(f'{what} {name}')
        w_old = O.kl_shaped_rewards(rew.to(dt), lp, rf, mask, hp['kl_coeff'], hp['clip_range_score'])
        w_adv, w_ret = O.gae_advantages_and_returns(vals, w_old, mask, start, hp['gamma'], hp['gae_lambda'])
        for name, got, want in (('old_rewards', old.t, w_old), ('adv', adv.t, w_adv), ('ret', ret.t, w_ret)):
            assert got.dtype == want.dtype and torch.equal(got.view(torch.int16), want.view(torch.int16)), what + name
        m = mask[:, start:]
        assert_same(rs.t[:, 2], m.sum(1), what + ' count')
        assert_same(rs.t[:, 5], last_true(mask), what + ' end')
        assert bool((rs.t[:, 6:] == 0).all()), what + ' lanes 6-7'


@gpu
def test_ppo_prep_refuses_past_shared_memory(ops):
    W, B = 17066, 2
    vals = torch.zeros(B, W, dtype=F32, device=DEV)
    mask = torch.ones(B, W, dtype=torch.bool, device=DEV)
    old, adv, ret, rs = Guarded(B, W, F32), Guarded(B, W, F32), Guarded(B, W, F32), Guarded(B, 8, F32)
    rc = _prep_call(vals, vals, vals[0], vals, mask, B, W, 0, 0.5, 8.0, 1.0, 1.0, F32MODE, (F32,) * 4, old.ptr(),
                    adv.ptr(), ret.ptr(), rs.ptr(), None)
    torch.cuda.synchronize()
    assert rc == ERR_UNSUPPORTED, rc
    assert old.untouched() and adv.untouched() and ret.untouched() and rs.untouched()


@gpu
def test_ppo_returns_shared_memory_opt_in_and_refusal(ops):
    """K4r at W - start = 12289 (past 48 KB of shared memory) equals the float64 restatement bit for bit on exact
    operands (reinforce, gamma = 1: a suffix sum); W - start = 51201 is refused and writes nothing."""
    from multi_ppo_port import returns_f64

    B, start = 2, 3
    W = start + 12289
    r64 = exact_ints((B, W), 8, -3, 11)
    mask = torch.rand(B, W, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3)) > 0.2
    rews = fenced(r64.float(), W + 4)
    mt = fenced(mask, W + 1, pad=True)
    adv, ret, rs = Guarded(B, W - start, F32), Guarded(B, W - start, F32), Guarded(B, 8, F32)
    rc_ok(Lb.lib().aa_ppo_returns(rews.data_ptr(), CODE[F32], W + 4, mt.data_ptr(), W + 1, B, W, start,
                                  0, 1, 1.0, F32MODE, 1, adv.ptr(), ret.ptr(), CODE[F32], rs.ptr(), _stream()), 'K4r')
    torch.cuda.synchronize()
    want = torch.from_numpy(returns_f64(r64, mask, start, 'reinforce', 1, 1.0))
    assert sum_exact(torch.where(mask, r64, 0.0), 1), 'premise: every carry of the chain is exact'
    adv.check('K4r adv')
    ret.check('K4r ret')
    written = torch.zeros(B, 8, dtype=torch.bool)
    written[:, 3:5] = True
    rs.check('K4r row_stats lanes 3-4 only', written)
    assert_same(adv.t, want.float(), 'K4r adv')
    assert_same(ret.t, want.float(), 'K4r ret')
    W = start + 51201
    rews = torch.zeros(B, W, device=DEV)
    mt = torch.ones(B, W, dtype=torch.bool, device=DEV)
    adv, ret = Guarded(B, W - start, F32), Guarded(B, W - start, F32)
    rc = Lb.lib().aa_ppo_returns(rews.data_ptr(), CODE[F32], W, mt.data_ptr(), W, B, W, start, 0, 1, 1.0, F32MODE, 1,
                                 adv.ptr(), ret.ptr(), CODE[F32], None, _stream())
    torch.cuda.synchronize()
    assert rc == ERR_UNSUPPORTED, rc
    assert adv.untouched() and ret.untouched()


# ---- K5 --------------------------------------------------------------------------------------------------------------
ACTOR_B = [1, 127, 128, 129, 4500]
ACTOR_W = [1, 31, 128, 1000]
CRITIC_CLIP = 0.5
ACTOR_CLIP = 0.2


def critic_operands(B, Wm, seed, device=DEV):
    """values, old values, returns on the 2^-4 grid (|.| <= 2) and a mask with a power-of-two count per row.  Some
    values sit exactly at old +- clip, some returns halfway between a value and its clipped value (l1 == l2 with the
    value out of range)."""
    x = exact_ints((B, Wm), 16, -3, seed, device)
    old = exact_ints((B, Wm), 16, -3, seed + 1, device)
    ret = exact_ints((B, Wm), 32, -4, seed + 2, device)
    t = torch.arange(Wm, device=device)[None, :].expand(B, Wm)
    x = torch.where(t % 7 == 1, old + CRITIC_CLIP, torch.where(t % 7 == 2, old - CRITIC_CLIP, x))
    hi = old + CRITIC_CLIP
    ret = torch.where((t % 7 == 3) & (x > hi), (x + hi) / 2, ret)
    return x, old, ret, pow2_mask(B, Wm, seed + 3, device)


def _k5_buffers(B, Wm, dt, pitched_grad):
    pitch = Wm + 8 if pitched_grad else Wm
    return Guarded(B, Wm, dt, pitch=pitch), Guarded(1, 2, F32), Guarded(B, 1, F32), Guarded(B, 1, F32)


@gpu
@pytest.mark.parametrize('B', ACTOR_B)
@pytest.mark.parametrize('Wm', ACTOR_W)
def test_critic_loss(ops, B, Wm):
    x64, o64, r64, mask = critic_operands(B, Wm, SEED + B + Wm)
    mt = fenced(mask, Wm + 3, pad=True)
    for dt in (BF, F16, F32):
        x, old, ret = fenced(x64.to(dt), Wm + 2), fenced(o64.to(dt), Wm + 1), fenced(r64.to(dt), Wm + 3)
        for mode in (FAITHFUL, F32MODE):
            rd = dt if mode == FAITHFUL and dt != F32 else None
            for gkind in ('pitched', 'none'):
                what = f'critic B={B} Wm={Wm} {dt} mode={mode} grad={gkind}'
                grad, loss, row_mean, rows = _k5_buffers(B, Wm, dt, True)
                counter = Words()
                rc_ok(Lb.lib().aa_ppo_critic_loss(x.data_ptr(), Wm + 2, old.data_ptr(), Wm + 1, CODE[dt], ret.data_ptr(),
                                                  Wm + 3, CODE[dt], mt.data_ptr(), Wm + 3, B, Wm, CRITIC_CLIP, mode,
                                                  loss.ptr(), grad.ptr() if gkind == 'pitched' else None, Wm + 8,
                                                  row_mean.ptr(), rows.ptr(), counter.ptr(), None, 0, _stream()), what)
                torch.cuda.synchronize()
                counter.check([0], what + ' counter')
                loss.check(what + ' loss', torch.tensor([[True, rd is not None]]))
                row_mean.check(what + ' row_mean')
                rows.check(what + ' row_scratch')
                if gkind == 'pitched':
                    grad.check(what + ' grad')
                else:
                    assert grad.untouched(), what + ' grad NULL'
                w_loss, w_grad, w_rm, w_rows = ref_critic(x64, o64, r64, mask, CRITIC_CLIP, rd, rd, B)
                assert_same(row_mean.t[:, 0], w_rm, what + ' row_mean')
                assert_same(rows.t[:, 0], w_rows, what + ' row_scratch')
                if gkind == 'pitched':
                    assert_same(grad.t, w_grad.to(dt), what + ' grad')  # stored in the value dtype
                if sum_exact(w_rows):
                    assert_same(loss.t[0, :1], w_loss.reshape(1), what + ' loss')
                else:  # the mean over B of inexact row means: fp32 summation bound, then the 16-bit rounding
                    tol = rel(w_loss) + (B + 2) * U * 0.5 * w_rows.abs().sum().cpu() / B + 2 * half_ulp(w_loss, rd)
                    assert_within(loss.t[0, :1], w_loss.reshape(1), tol.reshape(1), what + ' loss')
                if rd is not None:
                    s16 = loss.t[0, 1:2].view(torch.int16)[:1].view(rd)
                    assert torch.equal(s16.float(), loss.t[0, :1].to(rd).float()), what + ' 16-bit loss scalar'
                    if gkind == 'pitched':  # the tie rows included: values at old +- clip, returns halfway
                        leaf = x.detach().clone().requires_grad_(True)
                        want = O.critic_loss(leaf, old, ret, mask, CRITIC_CLIP)
                        want.backward()
                        assert_ulp_close(s16, want.reshape(1), max_ulp=1, min_exact=0.0, what=what + ' loss vs ATen')
                        assert_ulp_close(grad.t, leaf.grad, max_ulp=1, min_exact=0.97, what=what + ' grad vs ATen')


@gpu
def test_critic_value_tail_lens(ops):
    """`value_tail_lens`: lengths below 0, 0, inside the range and above `value_src_width`."""
    B, Wm = 6, 40
    src_w = Wm + 4
    lens = torch.tensor([-3, 0, 5, Wm, src_w, src_w + 7], dtype=torch.int32)
    raw64 = exact_ints((B, src_w), 16, -3, 21)
    o64 = exact_ints((B, Wm), 16, -3, 22)
    r64 = exact_ints((B, Wm), 32, -4, 23)
    mask = pow2_mask(B, Wm, 24)
    R = lens.clamp(0, src_w)
    x64 = torch.zeros(B, Wm, dtype=F64, device=DEV)
    for b in range(B):
        for t in range(Wm):
            if t < int(R[b]):
                x64[b, t] = raw64[b, src_w - int(R[b]) + t]
    for dt in (BF, F32):
        raw, old, ret = fenced(raw64.to(dt), src_w + 3), fenced(o64.to(dt), Wm), fenced(r64.to(dt), Wm)
        mt = fenced(mask, Wm, pad=True)
        ln = fenced_vec(lens.to(DEV))
        grad, loss, row_mean, rows = _k5_buffers(B, Wm, dt, True)
        counter = Words()
        rc_ok(Lb.lib().aa_ppo_critic_loss(raw.data_ptr(), src_w + 3, old.data_ptr(), Wm, CODE[dt], ret.data_ptr(), Wm,
                                          CODE[dt], mt.data_ptr(), Wm, B, Wm, CRITIC_CLIP, F32MODE, loss.ptr(),
                                          grad.ptr(), Wm + 8, row_mean.ptr(), rows.ptr(), counter.ptr(), ln.data_ptr(),
                                          src_w, _stream()), 'tail lens')
        torch.cuda.synchronize()
        counter.check([0], 'tail lens counter')
        grad.check('tail lens grad')
        w_loss, w_grad, w_rm, w_rows = ref_critic(x64, o64, r64, mask, CRITIC_CLIP, None, None, B)
        assert_same(grad.t, w_grad.to(dt), f'tail lens grad {dt}')
        assert_same(row_mean.t[:, 0], w_rm, f'tail lens row_mean {dt}')
        assert_same(loss.t[0, :1], w_loss.reshape(1), f'tail lens loss {dt}')


def ratio_edges(dt, clip=ACTOR_CLIP):
    """Host search for d = x - old (representable in dt) whose exp() rounds onto round(1 - clip) / round(1 + clip)
    in dt, taking the d whose exp lies furthest inside the rounding interval."""
    out = []
    for target in (1 - clip, 1 + clip):
        t = torch.tensor(target, dtype=F32).to(dt)
        cands = torch.linspace(math.log(target) - 0.05, math.log(target) + 0.05, 4001, dtype=F64).to(dt).unique()
        e = torch.exp(cands.double())
        hit = e.to(dt) == t
        assert bool(hit.any()), (dt, target)
        ulp = float(t.double()) * torch.finfo(dt).eps
        margin = (ulp / 2 - (e - t.double()).abs())
        margin[~hit] = -1
        out.append(float(cands[int(margin.argmax())]))
    return out


@gpu
@pytest.mark.parametrize('B', ACTOR_B)
@pytest.mark.parametrize('Wm', ACTOR_W)
def test_actor_loss(ops, B, Wm):
    gen = torch.Generator(device=DEV).manual_seed(B * 7 + Wm)
    mask = pow2_mask(B, Wm, B + Wm)
    mt = fenced(mask, Wm + 3, pad=True)
    old64 = -3 * torch.rand(B, Wm, generator=gen, device=DEV, dtype=F64)
    x64 = old64 + 0.3 * torch.randn(B, Wm, generator=gen, device=DEV, dtype=F64)
    a64 = torch.randn(B, Wm, generator=gen, device=DEV, dtype=F64)
    for dt in (BF, F16, F32):
        old_d, x_d = old64.to(dt), x64.to(dt)
        if dt != F32:  # ratios that round onto 1 -+ clip
            dlo, dhi = ratio_edges(dt)
            old_d[:, ::3] = 0
            x_d[:, ::3] = dlo
            old_d[:, 1::3] = 0
            x_d[:, 1::3] = dhi
        xx, old, adv = fenced(x_d, Wm + 2), fenced(old_d, Wm + 1), fenced(a64.to(dt), Wm + 5)
        for mode in (FAITHFUL, F32MODE):
            for gkind in ('pitched', 'none'):
                what = f'actor B={B} Wm={Wm} {dt} mode={mode} grad={gkind}'
                grad, loss, _, rows = _k5_buffers(B, Wm, dt, True)
                counter = Words()
                rc_ok(Lb.lib().aa_ppo_actor_loss(xx.data_ptr(), Wm + 2, old.data_ptr(), Wm + 1, CODE[dt], adv.data_ptr(),
                                                 Wm + 5, CODE[dt], mt.data_ptr(), Wm + 3, B, Wm, ACTOR_CLIP, mode,
                                                 loss.ptr(), grad.ptr() if gkind == 'pitched' else None, Wm + 8,
                                                 rows.ptr(), counter.ptr(), _stream()), what)
                torch.cuda.synchronize()
                counter.check([0], what + ' counter')
                sixteen = mode == FAITHFUL and dt != F32
                loss.check(what + ' loss', torch.tensor([[True, sixteen]]))
                rows.check(what + ' row_scratch')
                if gkind == 'none':
                    assert grad.untouched(), what + ' grad NULL'
                else:
                    grad.check(what + ' grad')
                if sixteen:
                    leaf = xx.detach().clone().requires_grad_(True)
                    want = O.actor_loss(leaf, old, adv, mask, ACTOR_CLIP)
                    want.backward()
                    s16 = loss.t[0, 1:2].view(torch.int16)[:1].view(dt)
                    assert_ulp_close(s16, want.reshape(1), max_ulp=1, min_exact=0.0, what=what + ' loss')
                    assert torch.equal(s16.float(), loss.t[0, :1].to(dt).float()), what + ' 16-bit scalar'
                    if gkind == 'pitched':
                        assert_ulp_close(grad.t, leaf.grad, max_ulp=1, min_exact=0.97, what=what + ' grad')
                else:
                    w_loss, w_grad, obj = ref_actor(xx.double(), old.double(), adv.double(), mask, ACTOR_CLIP, B)
                    # per-row sums of Wm inexact terms, then the mean over B: the fp32 summation bound
                    m = mask.double()
                    cnt = m.sum(1)
                    bound = ((Wm + 4) * U * ((obj.abs() * m).sum(1) / cnt)).sum() / B + (B + 2) * U * (
                        (obj * m).sum(1) / cnt).abs().sum() / B
                    assert_within(loss.t[0, :1], w_loss.reshape(1), (rel(w_loss) + bound.cpu()).reshape(1), what + ' loss')
                    if gkind == 'pitched':
                        assert_within(grad.t, w_grad, rel(w_grad) + half_ulp(w_grad, dt), what + ' grad')


# ---- counters re-armed -----------------------------------------------------------------------------------------------
@gpu
def test_counters_rearm_after_the_largest_grid(ops):
    """Each `last_block_arrives` kernel at its largest grid here and then at one block, on the same counter: a counter
    that is not re-armed leaves the second result POISON (and the counter non-zero)."""
    counters = [Words(), Words(), Words(n=2), Words(), Words()]  # critic, masked_mean, GRPO (two), nll, DPO
    for B in (4500, 1):
        Wm = 31
        mask = pow2_mask(B, Wm, 5)
        x64, o64, r64, _ = critic_operands(B, Wm, 6)
        x, o, r = fenced(x64.float()), fenced(o64.float()), fenced(r64.float())
        mt = fenced(mask)
        # critic
        loss, rows = Guarded(1, 2, F32), Guarded(B, 1, F32)
        rc_ok(Lb.lib().aa_ppo_critic_loss(x.data_ptr(), Wm, o.data_ptr(), Wm, CODE[F32], r.data_ptr(), Wm, CODE[F32],
                                          mt.data_ptr(), Wm, B, Wm, CRITIC_CLIP, F32MODE, loss.ptr(), None, 0, None,
                                          rows.ptr(), counters[0].ptr(), None, 0, _stream()), 'critic')
        # masked mean
        out, rows2 = Guarded(1, 1, F32), Guarded(B, 1, F32)
        rc_ok(Lb.lib().aa_masked_mean(x.data_ptr(), CODE[F32], Wm, mt.data_ptr(), Wm, B, Wm, out.ptr(), rows2.ptr(),
                                      counters[1].ptr(), _stream()), 'masked_mean')
        # GRPO
        tok = fenced(torch.zeros(B, Wm, dtype=torch.int64, device=DEV))
        adv = fenced_vec(torch.zeros(B, device=DEV))
        gl, re, scr = Guarded(1, 1, F32), Guarded(B, 1, torch.int32), Guarded(1, B + 1, F32)
        rc_ok(Lb.lib().aa_grpo_loss(x.data_ptr(), Wm, o.data_ptr(), Wm, CODE[F32], adv.data_ptr(), tok.data_ptr(), Wm, 5,
                                    B, Wm, 0.04, F32MODE, gl.ptr(), None, 0, re.ptr(), scr.ptr(), counters[2].ptr(),
                                    _stream()), 'grpo')
        # nll_mean (256 blocks at B * Wm >= 65536)
        n = B * Wm * (1 if B == 1 else 2)
        lpn = fenced_vec(-torch.ones(n, device=DEV))
        lab = fenced_vec(torch.zeros(n, dtype=torch.int64, device=DEV))
        nl, ni, part = Guarded(1, 1, F32), Guarded(1, 1, F32), Guarded(1, 512, F32)
        rc_ok(Lb.lib().aa_nll_mean(lpn.data_ptr(), CODE[F32], lab.data_ptr(), n, -100, nl.ptr(), ni.ptr(), part.ptr(),
                                   counters[3].ptr(), _stream()), 'nll')
        # DPO
        npairs = max(B // 2, 1)
        pol = fenced(x64[:1].expand(2 * npairs, Wm).float().contiguous())
        pp, st = Guarded(5, npairs, F32), Guarded(1, 8, F32)
        rc_ok(Lb.lib().aa_dpo_loss(pol.data_ptr(), pol.data_ptr(), CODE[F32], npairs, Wm, Wm, BETA, F32MODE, None, 0, 0,
                                   pp.ptr(), None, st.ptr(), counters[4].ptr(), None, None, None, _stream()), 'dpo')
        torch.cuda.synchronize()
        for what, buf in (('critic loss', loss), ('masked_mean', out), ('grpo loss', gl), ('nll loss', nl),
                          ('dpo stats', st)):
            assert not bool(buf.unwritten()[0, 0]), f'{what} B={B}: left POISON (counter not re-armed?)'
            assert not bool(torch.isnan(buf.t[0, 0])), f'{what} B={B}: NaN'
        for i, c in enumerate(counters):
            c.check([0] * c.n, f'counter {i} after B={B}')


# ---- GRPO ------------------------------------------------------------------------------------------------------------
GRPO_B = [1, 129, 4500]
GRPO_K = [1, 7, 128, 1025]
EOS = 3


def grpo_tokens(B, K, device=DEV):
    """Rows cycle through: eos at 0, in the middle, at K - 1 (twice: a later eos does not count), and no eos."""
    gen = torch.Generator(device=device).manual_seed(B + K)
    tok = torch.randint(4, 100, (B, K), generator=gen, device=device)
    kind = torch.arange(B, device=device) % 4
    pos = torch.stack([torch.zeros_like(kind), torch.full_like(kind, K // 2), torch.full_like(kind, K - 1),
                       torch.full_like(kind, -1)], 1).gather(1, kind[:, None])[:, 0]
    rows = torch.arange(B, device=device)
    has = pos >= 0
    tok[rows[has], pos[has]] = EOS
    tok[rows[kind == 1], K - 1] = EOS  # a second eos after the first
    return tok


@gpu
@pytest.mark.parametrize('B', GRPO_B)
@pytest.mark.parametrize('K', GRPO_K)
def test_grpo_loss(ops, B, K):
    gen = torch.Generator(device=DEV).manual_seed(B * 3 + K)
    tok64 = grpo_tokens(B, K)
    tok = fenced(tok64, K + 3, pad=EOS)
    A = fenced_vec(torch.randn(B, generator=gen, device=DEV))
    lp64 = -2 * torch.rand(B, K, generator=gen, device=DEV, dtype=F64)
    rf64 = lp64 + 0.3 * torch.randn(B, K, generator=gen, device=DEV, dtype=F64)
    row_end_want = grpo_row_end(tok64, EOS)
    beta = 0.04
    for dt in (BF, F16, F32):
        lp, rf = fenced(lp64.to(dt), K + 2), fenced(rf64.to(dt), K + 1)
        for mode in (FAITHFUL, F32MODE):
            what = f'GRPO B={B} K={K} {dt} mode={mode}'
            loss, grad = Guarded(1, 1, F32), Guarded(B, K, dt, pitch=K + 8)
            row_end, scratch = Guarded(B, 1, torch.int32), Guarded(1, B + 1, F32)
            counter = Words(n=2)
            rc_ok(Lb.lib().aa_grpo_loss(lp.data_ptr(), K + 2, rf.data_ptr(), K + 1, CODE[dt], A.data_ptr(),
                                        tok.data_ptr(), K + 3, EOS, B, K, beta, mode, loss.ptr(), grad.ptr(), K + 8,
                                        row_end.ptr(), scratch.ptr(), counter.ptr(), _stream()), what)
            torch.cuda.synchronize()
            counter.check([0, 0], what + ' counters')
            for name, buf in (('loss', loss), ('grad', grad), ('row_end', row_end), ('scratch', scratch)):
                buf.check(f'{what} {name}')
            assert torch.equal(row_end.t[:, 0].long(), row_end_want), what + ' row_end'
            assert float(scratch.t[0, 0]) == float(row_end_want.sum()), what + ' total'
            if mode == FAITHFUL and dt != F32:
                if B <= 129:
                    leaf = lp.detach().clone().requires_grad_(True)
                    want = O.grpo_loss(leaf, rf, A[:, None], tok64, 0, EOS, beta)
                    want.backward()
                    assert_within(loss.t[0], want.double().reshape(1), rel(want.reshape(1)) +
                                  (K + B + 4) * U * float(want.abs()), what + ' loss vs ATen')
                    assert_ulp_close(grad.t, leaf.grad, max_ulp=1, min_exact=0.97, what=what + ' grad vs ATen')
            else:
                w_loss, w_grad, ptl, on, mag = ref_grpo(lp.double(), rf.double(), A.double(), row_end_want, beta)
                total = on.double().sum()
                bound = (K + B + 4) * U * torch.where(on, ptl, 0.0).abs().sum() / total
                assert_within(loss.t[0], w_loss.reshape(1), (rel(w_loss) + bound.cpu()).reshape(1), what + ' loss')
                assert_within(grad.t, w_grad, rel(w_grad) + 8 * U * torch.where(on, mag, 0.0).cpu() +
                              half_ulp(w_grad, dt), what + ' grad')


@gpu
@pytest.mark.parametrize('G', [1, 2, 31, 32, 33, 100])
def test_group_advantages(ops, G):
    n_groups = 4000 if G <= 33 else 1000
    r64 = exact_ints((n_groups, G), 8, -2, G)
    r = fenced(r64.float(), G)
    out = Guarded(n_groups, G, F32)
    rc_ok(Lb.lib().aa_group_advantages(r.data_ptr(), n_groups, G, out.ptr(), _stream()), 'group adv')
    torch.cuda.synchronize()
    out.check(f'group advantages G={G}')
    want = ref_group_adv(r64)
    if G == 1:
        assert bool(torch.isnan(out.t).all()), 'G = 1: std of one sample is NaN, as torch.std gives'
        return
    if G & (G - 1) == 0:  # the mean, the deviations and their squares on one grid: one rounding each after the sum
        mean = r64.mean(1, keepdim=True)
        sd = f32(f32(torch.sqrt(f32(((r64 - mean) ** 2).sum(1, keepdim=True) / (G - 1)))) + f32(torch.tensor(1e-4)))
        assert_same(out.t, f32((r64 - mean) / sd), f'group advantages G={G}')
    else:
        # mean: G-term sum plus one division; deviation, sum of squares, sqrt, division: a few ulps of each term
        tol = rel(want) + (2 * G + 8) * U * (r64.abs().amax(1, keepdim=True) / (r64.std(1, keepdim=True) + 1e-4)).cpu()
        assert_within(out.t, want, tol, f'group advantages G={G}')


# ---- nll_mean, masked_mean, rm_pair_loss, pack_metrics ---------------------------------------------------------------
NLL_N = [1, 255, 256, 257, 65535, 65536, 65537, 3 * 65536 + 1]
NLL_Q = 64


@gpu
@pytest.mark.parametrize('n', NLL_N)
def test_nll_mean(ops, n):
    x64 = exact_ints((n,), NLL_Q, -3, n, nonpos=True)
    gen = torch.Generator(device=DEV).manual_seed(n)
    blocks = min(256, -(-n // 256))
    for ign in (0.0, 0.5, 1.0):
        labels64 = torch.randint(0, 50, (n,), generator=gen, device=DEV)
        drop = torch.rand(n, generator=gen, device=DEV) < ign if ign < 1.0 else torch.ones(n, dtype=torch.bool,
                                                                                            device=DEV)
        labels64[drop] = -100
        labels = fenced_vec(labels64)
        keep = labels64 != -100
        c = keep.double().sum()
        for dt in (BF, F16, F32):
            what = f'nll n={n} ignored={ign} {dt}'
            x = fenced_vec(x64.to(dt))
            loss, nic = Guarded(1, 1, F32), Guarded(1, 1, F32)
            part = Guarded(1, 2 * blocks, F32)
            counter = Words()
            rc_ok(Lb.lib().aa_nll_mean(x.data_ptr(), CODE[dt], labels.data_ptr(), n, -100, loss.ptr(), nic.ptr(),
                                       part.ptr(), counter.ptr(), _stream()), what)
            torch.cuda.synchronize()
            counter.check([0], what + ' counter')
            for name, buf in (('loss', loss), ('neg_inv_count', nic), ('partial', part)):
                buf.check(f'{what} {name}')
            s = torch.where(keep, x64, 0.0).sum()
            assert_same(loss.t[0], f32(-s / c).reshape(1), what + ' loss')
            assert_same(nic.t[0], f32(-1.0 / c).reshape(1), what + ' neg_inv_count')
            if ign == 1.0:
                assert bool(torch.isnan(loss.t[0, 0])) and float(nic.t[0, 0]) == -math.inf


MM_B = [1, 129, 4500]
MM_W = 96


@gpu
@pytest.mark.parametrize('B', MM_B)
def test_masked_mean(ops, B):
    W = MM_W
    x64 = exact_ints((B, W), 7, -3, B)
    mask = pow2_mask(B, W, B + 1)
    for dt in (BF, F16, F32):
        x = fenced(x64.to(dt), W + 3)
        for kind in ('mask', 'none', 'empty_row'):
            what = f'masked_mean B={B} {dt} {kind}'
            m = mask.clone()
            if kind == 'empty_row':
                m[B // 2] = False
            mt = fenced(m, W + 5, pad=True)
            out, rows = Guarded(1, 1, F32), Guarded(B, 1, F32)
            counter = Words()
            rc_ok(Lb.lib().aa_masked_mean(x.data_ptr(), CODE[dt], W + 3, None if kind == 'none' else mt.data_ptr(),
                                          W + 5, B, W, out.ptr(), rows.ptr(), counter.ptr(), _stream()), what)
            torch.cuda.synchronize()
            counter.check([0], what + ' counter')
            out.check(what + ' out')
            rows.check(what + ' rows')
            if kind == 'none':
                want = f32(x64.sum() / (B * W))  # B * W is an exact fp32 product here
                assert_same(rows.t[:, 0], x64.sum(1), what + ' rows')
            else:
                rw = f32(torch.where(m, x64, 0.0).sum(1) / m.double().sum(1))
                assert_same(rows.t[:, 0], rw, what + ' rows')
                want = f32(rw.sum() / B) if kind == 'mask' else torch.tensor(float('nan'), dtype=F64)
            assert_same(out.t[0], want.reshape(1), what)


@gpu
@pytest.mark.parametrize('B', [1, 255, 256, 257, 10000])
def test_rm_pair_loss(ops, B):
    gen = torch.Generator(device=DEV).manual_seed(B)
    h = torch.randn(B, generator=gen, device=DEV, dtype=F64).float().double()
    l = torch.randn(B, generator=gen, device=DEV, dtype=F64).float().double()
    l[::5] = h[::5]  # ties
    if B >= 3:
        h[1], l[1] = 50.0, -50.0  # saturated: h - l = +100
        h[2], l[2] = -50.0, 50.0  # h - l = -100
    es = fenced_vec(torch.cat([h, l]).float())
    for reg in (0.0, 0.01):
        what = f'rm B={B} reg={reg}'
        out, grad = Guarded(1, 2, F32), Guarded(1, 2 * B, F32)
        rc_ok(Lb.lib().aa_rm_pair_loss(es.data_ptr(), B, reg, out.ptr(), grad.ptr(), _stream()), what)
        torch.cuda.synchronize()
        out.check(what + ' out')
        grad.check(what + ' grad')
        w_loss, w_grad, w_acc = ref_rm(h, l, reg)
        terms = (-F.logsigmoid(h - l)).abs().sum() / B + reg * torch.cat([h, l]).square().sum() / (2 * B)
        assert_within(out.t[0, :1], w_loss.reshape(1), (rel(w_loss) + (B + 8) * U * terms).cpu().reshape(1), what)
        assert_same(out.t[0, 1:], f32(f32((h > l).double().sum()) * f32(torch.tensor(1.0 / B, dtype=F64))).reshape(1),
                    what + ' accuracy')
        mag = (dlogsig(h - l).abs() / B).repeat(2) + (reg / B) * torch.cat([h, l]).abs()
        assert_within(grad.t[0], w_grad, rel(w_grad) + 8 * U * mag.cpu() + 1e-37, what + ' grad')


@gpu
@pytest.mark.parametrize('B', [1, 31, 32, 33, 1000])
def test_ppo_pack_metrics(ops, B):
    rs64 = exact_ints((B, 8), 64, -3, B)
    rs64[:, 2] = torch.randint(0, 100, (B,), device=DEV).double()
    rew64 = exact_ints((B,), 64, -3, B + 1)
    vm64 = exact_ints((B,), 64, -3, B + 2)
    rs, rew, vm = fenced(rs64.float()), fenced_vec(rew64.float()), fenced_vec(vm64.float())
    al, cl = fenced_vec(torch.tensor([1.25], device=DEV)), fenced_vec(torch.tensor([-0.5], device=DEV))
    inv = f32(torch.tensor(1.0 / B, dtype=F64))
    for with_vm in (True, False):
        what = f'pack B={B} value_row_mean={with_vm}'
        stats = Guarded(1, 12, F32)
        status = Words(value=Lb.STATUS_EMPTY_MASK | Lb.STATUS_LABEL_OOB)
        rc_ok(Lb.lib().aa_ppo_pack_metrics(rs.data_ptr(), rew.data_ptr(), vm.data_ptr() if with_vm else None,
                                           al.data_ptr(), cl.data_ptr(), B, stats.ptr(), None, status.ptr(), _stream()),
              what)
        torch.cuda.synchronize()
        stats.check(what)
        status.check([5], what + ' status')
        mean = lambda v: f32(v.sum() * inv)  # noqa: E731
        want = torch.stack([torch.tensor(1.25, dtype=F64, device=DEV), torch.tensor(-0.5, dtype=F64, device=DEV),
                            mean(rew64), mean(rs64[:, 1]), mean(rs64[:, 3]), mean(rs64[:, 4]),
                            mean(vm64) if with_vm else torch.tensor(0.0, dtype=F64, device=DEV), mean(rs64[:, 0]),
                            mean(rs64[:, 2]), rs64[:, 2].max().clamp(min=0), torch.tensor(5.0, dtype=F64, device=DEV),
                            torch.tensor(0.0, dtype=F64, device=DEV)])
        assert_same(stats.t[0], want, what)
