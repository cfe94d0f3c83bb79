"""float64 references for K2's objective variants (aa_dpo_loss_obj, aa_dpo_loss_ext), held to the ports on the CPU.

`ref_k2` restates the two variants of `dpo_loss_kernel` (csrc/dpo.cu) on whole pair vectors at once: one fp32 rounding
after every + - * /, then the 16-bit rounding wherever faithful mode rounds (`rd`), the autograd order of the
gradients that reach one value along several paths (`exo_discopop`, `fdiv_backward`), AOT's stable rank sort with NaN
last, the metric means, the RPO term and the seeds of the last block.  The per-pair Python ports
(dpo_objective_port.py, dpo_ext_port.py) say the same one pair at a time; they are too slow for the 4500 pairs of
tests/test_gpu_dpo_objective_pin.py, which compares the kernels against `ref_k2`.

Only expf / log1pf are not restated bit for bit: CUDA's are within 2 ulp of the correctly rounded value, the reference
rounds the float64 value once.  `_Ar(tw)` moves each such result by 4 fp32 ulps, all one way or alternating; twice
the spread of those references is the part of the GPU bar that cancellation after a libm call needs (hinge: none; JS and DiscoPOP
gradients: most of it).

Here, without a GPU:
- each reference against the ports run in float64 (to 1e-6: the fp32 scalar arguments) and in fp32 (the metrics bit for
  bit, seeds and loss within 1 ulp and the libm spread), for every type and f-divergence, on random and saturated operand sets;
- the exact premise of every operand set of the GPU matrix: the four sums, a, b, h and AOT's keys exact in fp32;
- the two AOT identities: one kept pair, and co-monotone keys, give `sigmoid` pair by pair;
- the RPO count case: its fp32 tree sum of the counts (the kernel's old reduction) is not the count rounded once.
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dpo_ext_port import dpo_loss as port_loss
from dpo_ext_port import exp_cap
from test_gpu_loss_kernels import DPO_B, DPO_W, EXACT, U, dpo_operands, dpo_shape, dpo_valid, f32, grid_exp, rnd, \
    sum_exact

BF, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
OBJ_TYPES = ('sigmoid', 'robust', 'hinge', 'ipo', 'sppo_hard', 'nca_pair', 'apo_zero', 'apo_down')
TYPES = {t: k for k, t in enumerate(OBJ_TYPES + ('exo_pair', 'discopop', 'aot', 'aot_pair'))}
FDIV = {'reverse_kl': 0, 'js_divergence': 1, 'alpha_divergence': 2}
SMOOTHABLE = ('sigmoid', 'robust', 'exo_pair', 'aot', 'aot_pair')
READS_H = ('sigmoid', 'robust', 'hinge', 'exo_pair')
AOT_MAX = 1024
SEED = 4321
# the GPU matrix's pair counts: the loss pin's, and AOT's limit (AOT runs up to it, the other types past it)
MATRIX_B = DPO_B + [AOT_MAX]


def c32(x):
    """A Python float as the kernel's fp32 scalar argument receives it."""
    return float(np.float32(x))


@dataclasses.dataclass(frozen=True)
class Opt:
    """One objective: the entry point ('obj' or 'ext') and the fields the C ABI takes."""
    entry: str
    loss_type: str
    eps: float = 0.0
    alpha: float = 0.0
    fdiv: str = 'reverse_kl'
    coef: float = 1.0
    tau: float = 0.05
    ref_free: bool = False

    @property
    def obj_arith(self):
        return self.loss_type in OBJ_TYPES and self.fdiv == 'reverse_kl'

    def port_kw(self):
        return dict(loss_type=self.loss_type, label_smoothing=self.eps, rpo_alpha=self.alpha,
                    reference_free=self.ref_free, f_divergence_type=self.fdiv, f_alpha_divergence_coef=self.coef,
                    discopop_tau=self.tau)


# the 8 types of aa_dpo_loss_obj and the 12 aa_dpo_loss_ext adds: its own 4 types and the f-divergences on the types
# that read h
KINDS = [('obj', t, 'reverse_kl') for t in OBJ_TYPES] + \
    [('ext', t, 'reverse_kl') for t in ('exo_pair', 'discopop', 'aot', 'aot_pair')] + \
    [('ext', t, f) for f in ('js_divergence', 'alpha_divergence') for t in READS_H]


def kind_opt(kind, j):
    """The options of `kind` at the j-th width of the matrix: label smoothing, RPO, reference-free, the alpha
    coefficient and DiscoPOP's temperature cycle over the widths, so that every one meets every pair count."""
    entry, t, fdiv = kind
    return Opt(entry, t, eps=[0.0, 0.25, 0.1, 0.125, 0.0][j] if t in SMOOTHABLE else 0.0,
               alpha=[0.0, 0.5, 0.0, 1.0, 0.5][j], fdiv=fdiv,
               coef=[1.0, 1.5, 2.0, 1.0, 1.25][j] if fdiv == 'alpha_divergence' else 1.0,
               tau=[0.05, 0.5, 0.05, 1.0, 0.05][j] if t == 'discopop' else 0.05, ref_free=j == 2)


# ---- the kernel's arithmetic ------------------------------------------------------------------------------------------
class _Ar:
    """r: round_to(x, rd) after an fp32 op; f: the fp32 rounding alone; t: an fp32 libm result (expf / log1pf), moved
    by tw * 4 ulps.  rd = F64: no rounding at all (the formulas and the autograd chain alone)."""

    def __init__(self, rd, tw=0):
        self.rd, self.tw, self.calls = rd, tw, 0

    def f(self, x):
        x = torch.as_tensor(x, dtype=F64)
        return x if self.rd == F64 else f32(x)

    def r(self, x):
        x = torch.as_tensor(x, dtype=F64)
        return x if self.rd == F64 else rnd(x, self.rd)

    def t(self, x):
        if not self.tw:
            return self.f(x)
        self.calls += 1  # tw = (even, odd): the calls alternate, so that errors of two terms may add or cancel
        return self.f(x * (1 + self.tw[self.calls % 2] * 4 * U))

    def exp(self, x):
        return self.t(torch.exp(x))

    def ls(self, z):  # log_sigmoid: fminf(z, 0) - log1pf(expf(-|z|)); fminf(NaN, 0) = 0, log1pf(expf(NaN)) = NaN
        return self.f(torch.nan_to_num(z.clamp(max=0.0), nan=0.0) - self.t(torch.log1p(self.exp(-z.abs()))))

    def dls(self, z):  # dlog_sigmoid
        e = self.exp(-z.abs())
        q = self.f(e / self.f(1 + e))
        return torch.where(z < 0, self.f(1 - q), q)

    def sig(self, z):
        return self.f(1 / self.f(1 + self.exp(-z)))

    def dsig(self, g, s):
        R = self.r
        return R(R(g * R(1 - s)) * s)

    def softplus(self, x):
        return torch.where(x > 20, x, self.t(torch.log1p(self.exp(x))))

    def dsoftplus(self, g, x):
        z = self.exp(x)
        return self.r(torch.where(x > 20, g, self.f(self.f(g * z) / self.f(z + 1))))

    def cap_exp(self, x, cap):
        return self.r(self.exp(self.r(torch.where(torch.isnan(x), x, x.clamp(max=cap)))))


def obj_forward(A, t, a, b, beta, eps):
    """dpo_obj_forward -> (loss, s0, s1)."""
    R = A.r
    c = c32(0.5 / beta)
    z0 = torch.zeros_like(a)
    if t in ('sigmoid', 'robust'):
        z = R(beta * R(a - b))
        t1 = R(A.ls(z))
        loss = -t1
        if eps != 0:
            m1 = R(-t1 * c32(1 - eps))
            m2 = R(R(A.ls(-z)) * eps)
            loss = R(m1 - m2) if t == 'sigmoid' else R(R(m1 + m2) * c32(1 / c32(1 - 2 * eps)))
        return loss, z, z0
    if t == 'hinge':
        u = R(1 - R(beta * R(a - b)))
        loss = torch.where((u > 0) | torch.isnan(u), u, z0)
        return loss, loss, z0
    if t == 'ipo':
        d = R(R(a - b) - c)
        return R(d * d), d, z0
    if t == 'sppo_hard':
        d1, d2 = R(a - c), R(b + c)
        return R(R(d1 * d1) + R(d2 * d2)), d1, d2
    if t == 'nca_pair':
        za, zb = R(beta * a), R(beta * b)
        t1, t2, t3 = R(A.ls(za)), R(A.ls(-za)), R(A.ls(-zb))
        return R(R(-t1 - 0.5 * t2) - 0.5 * t3), za, zb
    if t == 'apo_zero':
        sa, sb = R(A.sig(R(beta * a))), R(A.sig(R(beta * b)))
        return R(R(1 - sa) + sb), sa, sb
    sa, sh = R(A.sig(R(beta * a))), R(A.sig(R(beta * R(a - b))))  # apo_down
    return R(sa + R(1 - sh)), sa, sh


def obj_backward(A, t, gl, s0, s1, beta, eps, inv_nc=None, inv_nr=None):
    """dpo_obj_backward -> (d / d chosen, d / d rejected)."""
    R = A.r
    if t in ('sigmoid', 'robust'):
        if eps == 0:
            gz = R(-gl * A.dls(s0))
        else:
            g0 = R(gl * c32(1 / c32(1 - 2 * eps))) if t == 'robust' else gl
            dt1 = -R(g0 * c32(1 - eps))
            dt2 = R((g0 if t == 'robust' else -g0) * eps)
            gz = R(R(dt1 * A.dls(s0)) - R(dt2 * A.dls(-s0)))
        gh = R(gz * beta)
        return gh, -gh
    if t == 'hinge':
        gh = R(torch.where((s0 > 0) | torch.isnan(s0), -gl, 0.0) * beta)
        return gh, -gh
    if t == 'ipo':
        gd = R(gl * 2 * s0)
        return R(gd * inv_nc), R(-gd * inv_nr)
    if t == 'sppo_hard':
        return R(gl * 2 * s0), R(gl * 2 * s1)
    if t == 'nca_pair':
        hg = -gl * 0.5
        gza = R(R(-gl * A.dls(s0)) - R(hg * A.dls(-s0)))
        gzb = -R(hg * A.dls(-s1))
        return R(gza * beta), R(gzb * beta)
    if t == 'apo_zero':
        return R(A.dsig(-gl, s0) * beta), R(A.dsig(gl, s1) * beta)
    gh = R(A.dsig(-gl, s1) * beta)  # apo_down
    ga = R(A.dsig(gl, s0) * beta)
    return R(ga + gh), -gh


def fdiv_forward(A, o, a, b, cap):
    R = A.r
    if o.fdiv == 'alpha_divergence':
        eb = A.cap_exp(R(b * -o.coef), cap)
        ea = A.cap_exp(R(a * -o.coef), cap)
        return R(R(eb - ea) * c32(1 / o.coef))
    h = R(a - b)
    if o.fdiv == 'js_divergence':
        return R(h - R(R(A.softplus(a)) - R(A.softplus(b))))
    return h


def fdiv_backward(A, o, gh, a, b, cap):
    R = A.r
    if o.fdiv == 'alpha_divergence':
        gd = R(gh * c32(1 / o.coef))
        ta, tb = R(a * -o.coef), R(b * -o.coef)
        gta = torch.where(ta <= cap, R(-gd * A.cap_exp(ta, cap)), 0.0)
        gtb = torch.where(tb <= cap, R(gd * A.cap_exp(tb, cap)), 0.0)
        return R(gta * -o.coef), R(gtb * -o.coef)
    if o.fdiv == 'js_divergence':  # h = a - b and softplus(a) both reach a: two terms, added once
        return R(gh + A.dsoftplus(-gh, a)), R(-gh + A.dsoftplus(gh, b))
    return gh, -gh


def exo_discopop(A, o, h, gl, beta):
    """-> (loss, d (gl * loss) / d h); the sums follow autograd's order (the latest-created node first)."""
    R = A.r
    z = R(beta * h)
    if o.loss_type == 'exo_pair':
        e = o.eps if o.eps > 0 else 1e-3
        c1, c2 = c32(math.log(1 - e)), c32(math.log(e))
        s1, t1 = R(A.sig(z)), R(R(A.ls(z)) - c1)
        s2, t2 = R(A.sig(-z)), R(R(A.ls(-z)) - c2)
        loss = R(R(s1 * t1) + R(s2 * t2))
        g_nz = R(R(R(gl * s2) * A.dls(-z)) + A.dsig(R(gl * t2), s2))
        g_l1 = R(R(gl * s1) * A.dls(z))
        gz = R(R(-g_nz + g_l1) + A.dsig(R(gl * t1), s1))
        return loss, R(gz * beta)
    inv_tau = c32(1 / c32(o.tau))  # discopop
    m = R(A.sig(R(z * inv_tau)))
    lc, ec, om = -R(A.ls(z)), R(A.exp(-z)), R(1 - m)
    loss = R(R(lc * om) + R(ec * m))
    gm = R(R(gl * ec) - R(gl * lc))
    g_e = -R(R(gl * m) * ec)
    g_l = R(-R(gl * om) * A.dls(z))
    g_t = R(A.dsig(gm, m) * inv_tau)
    gz = R(R(g_e + g_l) + g_t)
    return loss, R(gz * beta)


def ext_pair(A, o, a, b, gl, beta, cap):
    """dpo_ext_pair -> (loss, d / d a, d / d b)."""
    h = fdiv_forward(A, o, a, b, cap)
    if o.loss_type in ('exo_pair', 'discopop'):
        loss, gh = exo_discopop(A, o, h, gl, beta)
    else:
        loss, s0, s1 = obj_forward(A, o.loss_type, h, torch.zeros_like(h), beta, o.eps)
        gh = obj_backward(A, o.loss_type, gl, s0, s1, beta, o.eps)[0]
    ga, gb = fdiv_backward(A, o, gh, a, b, cap)
    return loss, ga, gb, gh


def stable_ranks(x):
    """Positions of x's elements in torch.sort(x, stable=True): NaN last, ties to the smaller index."""
    order = torch.sort(x, stable=True).indices
    rank = torch.empty_like(order)
    rank[order] = torch.arange(x.numel())
    return rank


def ref_k2(pc, pr, rc, rr, valid, counts, o, beta, rd, cap, tw=0):
    """K2's objective variants on the four row sums (float64 [B], already the kernel's rounded sums; rc = rr = 0 when
    reference-free).  valid: bool [B]; counts: float64 [2B] or None.  -> dict of float64 tensors: per_pair (5, B),
    grad_seg (2B,), stats (8 or 9,), and seed_terms (2B,): the sum of the magnitudes of what each seed adds last
    (JS: gh and softplus' term; RPO: the chosen seed and g_nll), the scale of its rounding errors."""
    A = _Ar(rd, tw)
    R = A.r
    beta = c32(beta)
    cap = cap if rd == F64 else c32(cap)  # the kernel's fp32 cap: a key at it is not clamped
    B = pc.numel()
    eps = c32(o.eps)
    v = valid.to(pc.device).bool()
    ratio_c, ratio_r = R(pc - rc), R(pr - rr)
    a, b = ratio_c, ratio_r
    inv_c = inv_r = None
    if o.loss_type == 'ipo':
        inv_c, inv_r = A.f(1 / counts[:B]), A.f(1 / counts[B:])
        a = R(R(pc * inv_c) - R(rc * inv_c))
        b = R(R(pr * inv_r) - R(rr * inv_r))
    n = float(v.sum())
    inv_n = c32(1 / n) if n else math.inf
    gl = float(R(torch.tensor(inv_n, dtype=F64)))
    aot = o.loss_type in ('aot', 'aot_pair')
    terms = None
    if aot:
        k1, k2 = (R(pc - pr), R(rc - rr)) if o.loss_type == 'aot' else (a, b)
        loss = torch.zeros(B, dtype=F64)
        gc, gr = torch.zeros(B, dtype=F64), torch.zeros(B, dtype=F64)
        if n:
            kk1, kk2 = k1[v], k2[v]
            r1, r2 = stable_ranks(kk1), stable_ranks(kk2)
            pos2 = torch.empty_like(kk2)
            pos2[r2] = kk2
            lk, zk, _ = obj_forward(A, 'sigmoid', R(kk1 - pos2[r1]), torch.zeros_like(kk1), beta, eps)
            zpos = torch.empty_like(zk)
            zpos[r1] = zk
            loss[v] = lk
            g1 = obj_backward(A, 'sigmoid', gl, zpos[r1], None, beta, eps)[0]
            g2 = -g1 if o.loss_type == 'aot' else -obj_backward(A, 'sigmoid', gl, zpos[r2], None, beta, eps)[0]
            gc[v], gr[v] = g1, g2
    elif o.entry == 'obj' or o.obj_arith:
        loss, s0, s1 = obj_forward(A, o.loss_type, a, b, beta, eps)
        gc, gr = obj_backward(A, o.loss_type, gl, s0, s1, beta, eps, inv_c, inv_r)
    else:
        loss = ext_pair(A, o, a, b, 0.0, beta, cap)[0]
        _, gc, gr, gh = ext_pair(A, o, a, b, gl, beta, cap)
        if o.fdiv == 'js_divergence':  # each seed adds gh and softplus' term
            terms = (gh.abs() + A.dsoftplus(-gh, a).abs(), gh.abs() + A.dsoftplus(gh, b).abs())
    better, worse = R(beta * ratio_c), R(beta * ratio_r)
    mean = lambda x: R(A.f(torch.where(v, x, 0.0).sum()) * inv_n) if n else torch.tensor(math.nan, dtype=F64)  # noqa
    s_loss = A.f(torch.where(v, loss, 0.0).sum())
    stats = [mean(loss), mean(R(better + worse)), mean(better), mean(worse),
             A.f((v & (better > worse)).double().sum() * inv_n) if n else torch.tensor(math.nan, dtype=F64),
             mean(R(better - worse)), torch.tensor(n, dtype=F64), torch.tensor(0.0, dtype=F64)]
    if o.alpha > 0:
        cnt = float(counts[:B][v].sum())
        inv_cnt = c32(1 / c32(cnt)) if cnt else math.inf
        s_pc = A.f(torch.where(v, pc, 0.0).sum())
        nll = -R(R(s_pc) * inv_cnt) if n else torch.tensor(math.nan, dtype=F64)
        g_nll = float(R(torch.tensor(-float(R(torch.tensor(c32(o.alpha), dtype=F64))) * inv_cnt, dtype=F64)))
        stats[0] = R(R(s_loss * inv_n) + R(nll * c32(o.alpha))) if n else nll
        stats.append(nll)
        gc_terms = (gc.abs() if terms is None else terms[0]) + abs(g_nll)
        gc = R(gc + g_nll)
    else:
        gc_terms = gc.abs() if terms is None else terms[0]
    gr_terms = gr.abs() if terms is None else terms[1]
    gc = torch.where(v, gc, 0.0)
    gr = torch.where(v, gr, -0.0)
    per_pair = torch.stack([loss, better, worse, gc, v.double()])
    return dict(per_pair=per_pair, grad_seg=torch.cat([gc, gr]), stats=torch.stack([torch.as_tensor(s) for s in stats]),
                loss=loss, seed_terms=torch.cat([torch.where(v, gc_terms, 0.0), torch.where(v, gr_terms, 0.0)]))


def ref_spread(sums, valid, counts, o, beta, rd, cap):
    """-> (the reference, its spread): per output twice the largest move of the reference when every expf / log1pf
    result moves by 4 fp32 ulps, all one way or alternating (0 where it stays NaN)."""
    r0 = ref_k2(*sums, valid, counts, o, beta, rd, cap)
    spread = {}
    for tw in ((1, 1), (-1, -1), (1, -1), (-1, 1)):
        r = ref_k2(*sums, valid, counts, o, beta, rd, cap, tw)
        for k in ('per_pair', 'grad_seg', 'stats'):
            d = torch.nan_to_num((r[k] - r0[k]).abs(), nan=0.0)
            spread[k] = torch.maximum(spread.get(k, d), 2 * d)
    return r0, spread


def sums_of(pol, ref, B, rd, ref_free):
    """The kernel's four row sums of float64 (2B, W) operands: exact in fp32 (the premise), then rounded to rd."""
    pc, pr = rnd(pol[:B].sum(1), rd), rnd(pol[B:].sum(1), rd)
    if ref_free:
        return pc, pr, torch.zeros_like(pc), torch.zeros_like(pr)
    return pc, pr, rnd(ref[:B].sum(1), rd), rnd(ref[B:].sum(1), rd)


def ref_case(pol, ref, valid, counts, o, beta, dt, rd, tw=0):
    B = pol.size(0) // 2
    return ref_k2(*sums_of(pol.cpu(), ref.cpu(), B, rd, o.ref_free), valid.cpu(), counts, o, beta, rd, exp_cap(dt), tw)


# ---- the references against the ports ---------------------------------------------------------------------------------
PORT_OPTS = [Opt('obj', t) for t in OBJ_TYPES] + \
    [Opt('obj', 'sigmoid', eps=0.25, alpha=0.5), Opt('obj', 'robust', eps=0.125, ref_free=True),
     Opt('obj', 'ipo', alpha=1.0), Opt('obj', 'nca_pair', ref_free=True)] + \
    [Opt('ext', t, eps=e, alpha=al) for t, e, al in (('exo_pair', 0.0, 0.0), ('exo_pair', 0.1, 0.5),
                                                     ('discopop', 0.0, 0.0), ('aot', 0.25, 0.5), ('aot_pair', 0.0, 1.0),
                                                     ('aot', 0.0, 0.0), ('aot_pair', 0.125, 0.0))] + \
    [Opt('ext', 'discopop', tau=0.5), Opt('ext', 'discopop', tau=2.0 ** -9)] + \
    [Opt('ext', t, fdiv=f, coef=c, eps=0.125 if t in SMOOTHABLE else 0.0)
     for t in READS_H for f, c in (('js_divergence', 1.0), ('alpha_divergence', 1.0), ('alpha_divergence', 2.0))]


def _port_operands(kind, B, W, seed):
    """(pol, ref) float64 (2B, W): 'random' multiples of 1/8 in [-8, 0]; 'saturated' puts |beta h| past every threshold
    (softplus' 20, the exp caps, expf's overflow) and repeats pair 0 for ties."""
    g = torch.Generator().manual_seed(seed)
    pol = -torch.randint(0, 65, (2 * B, W), generator=g).double() / 8
    ref = -torch.randint(0, 65, (2 * B, W), generator=g).double() / 8
    if kind == 'saturated':
        scale = torch.tensor([1, 40, 3, 160, 12, 900, 2, 25, 600, 7, 90, 1])[torch.arange(2 * B) % 12].double()
        pol = pol * scale[:, None]
        ref = ref * scale.flip(0)[:, None]
        pol[4:B:4], ref[4:B:4] = pol[0], ref[0]
        pol[B + 4::4], ref[B + 4::4] = pol[B], ref[B]
    return pol, ref


@pytest.mark.parametrize('opt', PORT_OPTS, ids=lambda o: f'{o.entry}-{o.loss_type}-{o.fdiv}-e{o.eps}-a{o.alpha}'
                         f'-c{o.coef}-t{o.tau}-rf{int(o.ref_free)}')
@pytest.mark.parametrize('operands', ['random', 'saturated'])
def test_reference_against_the_port(opt, operands):
    """The float64 reference against the port pair by pair: without rounding against the port in float64 (to 1e-6: the
    kernel's fp32 scalar arguments), and with fp32's rounding points against the port on ATen CPU in fp32: every seed,
    metric bit for bit, every seed, the NLL and the mean loss within 1 ulp and the reference's libm spread (ATen
    CPU's vectorised expf / log1pf are not CUDA's; ATen CPU divides by n where ATen CUDA, and K2, multiply by 1 / n; IPO's seeds are held in float64 only).  The
    16-bit rounding points are ATen CUDA's (CPU rounds some chains once); tests/test_gpu_dpo_objective_pin.py holds
    them to the port there."""
    B, W, beta = 12, 5, 0.125
    pol, ref = _port_operands(operands, B, W, 100 + PORT_OPTS.index(opt))
    g = torch.Generator().manual_seed(5)
    lens = torch.randint(2, 40, (2 * B,), generator=g)
    ids = torch.randint(0, 9, (2 * B, 3), generator=g)
    ids[B + 1::3] = ids[1:B:3]
    valid = ~(ids[:B] == ids[B:]).all(1)
    counts = (lens - 1).double()
    for dt in (F64, F32):
        cap = exp_cap(F32)
        leaf = pol.to(dt).detach().clone().requires_grad_(True)
        want = port_loss(leaf, ref.to(dt), beta, ids, True, response_lens=lens.tolist(), cap=cap, **opt.port_kw())
        want['loss'].backward()
        got_g = leaf.grad[:, 0].double()
        what = f'{opt} {operands} {dt}'
        mine = ref_k2(*sums_of(pol, ref, B, None, opt.ref_free), valid, counts, opt, beta, dt if dt == F64 else None,
                      cap)
        if dt == F64:  # the formulas and the autograd chain without rounding (but for the fp32 scalar arguments)
            assert torch.allclose(mine['stats'][0], want['loss'], rtol=1e-6, atol=1e-12, equal_nan=True), what
            assert torch.allclose(mine['grad_seg'], got_g, rtol=1e-6, atol=1e-12, equal_nan=True), what
            continue
        sp = ref_spread(sums_of(pol, ref, B, None, opt.ref_free), valid, counts, opt, beta, None, cap)[1]
        if opt.loss_type != 'ipo':  # ATen CPU's pc / n is not K2's pc * (1 / n), and h - 1 / (2 beta) cancels
            _ulps(mine['grad_seg'], got_g, F32, 1, what + ' seeds', sp['grad_seg'])
        _same(mine['per_pair'][1][valid], want['better_sample_reward'].double(), what + ' better')
        _same(mine['per_pair'][2][valid], want['worse_sample_reward'].double(), what + ' worse')
        _same(mine['stats'][4], want['reward_accuracy'].double(), what + ' accuracy')
        if opt.alpha > 0:
            _ulps(mine['stats'][8], want['nll_loss'].double(), F32, 1, what + ' nll')
        _ulps(mine['stats'][0], want['loss'].detach().double(), F32, 1, what + ' loss', sp['stats'][0])


def _same(got, want, what):
    got, want = got.double().reshape(-1), want.double().reshape(-1)
    ok = (got == want) | (torch.isnan(got) & torch.isnan(want))
    assert bool(ok.all()), f'{what}: {int((~ok).sum())} of {ok.numel()} differ: {got[~ok][:4]} vs {want[~ok][:4]}'


def _ulps(got, want, dt, n, what, spread=0.0):
    """|got - want| <= n ulps of dt at want + spread (NaN where want is NaN)."""
    got, want = got.double().reshape(-1), want.double().reshape(-1)
    assert torch.equal(torch.isnan(got), torch.isnan(want)), what
    fi = torch.finfo(dt)
    ulp = torch.exp2(torch.floor(torch.log2(want.abs().clamp(min=fi.tiny)))) * fi.eps
    ok = ((got - want).abs() <= n * ulp + torch.as_tensor(spread).reshape(-1)) | torch.isnan(want) | (got == want)
    assert bool(ok.all()), f'{what}: {got[~ok]} vs {want[~ok]}'


# ---- the exact premise of the GPU matrix ------------------------------------------------------------------------------
def fp32_exact(x):
    """Every value of x (float64) is an fp32 value: on one grid 2^-k with |x| * 2^k <= 2^24."""
    x = x[torch.isfinite(x)]
    if x.numel() == 0:
        return True
    k = grid_exp(x)
    return k is not None and bool((x.abs() * 2.0 ** k <= EXACT).all())


def test_exact_premise_of_the_matrix():
    """For every (B, W) of the matrix (AOT's 1024 too): the operands hold in bf16 and fp16, every row sum is exact in
    fp32 in any order, and so are a = pc - rc, b = pr - rr, h = a - b and AOT's keys pc - pr, rc - rr."""
    for B in MATRIX_B:
        for W in DPO_W:
            pol, ref = dpo_operands(B, W, SEED + B + W, 'cpu')
            for dt in (BF, F16):
                assert torch.equal(pol.to(dt).double(), pol) and torch.equal(ref.to(dt).double(), ref)
            assert sum_exact(pol, 1) and sum_exact(ref, 1), (B, W)
            pc, pr, rc, rr = sums_of(pol, ref, B, None, False)
            a, b = pc - rc, pr - rr
            for x in (pc, pr, rc, rr, a, b, a - b, pc - pr, rc - rr):
                assert fp32_exact(x), (B, W)
            nz, q = dpo_shape(B, W)
            assert B * max(nz, 1) * q <= 2 ** 22 or nz == 0


# ---- AOT identities ---------------------------------------------------------------------------------------------------
def comonotone(B, W, loss_type, seed):
    """(pol, ref) float64 (2B, W) whose AOT keys are co-monotone across pairs (ties included): pair i's first key is
    x_i and its second y_i = 2 x_i - 1/8, so sorting either key list moves the pairs alike."""
    g = torch.Generator().manual_seed(seed)
    x = -torch.randint(0, 65, (B,), generator=g).double() / 8
    y = 2 * x - 0.125
    pol = torch.zeros(2 * B, W, dtype=F64)
    ref = torch.zeros(2 * B, W, dtype=F64)
    pol[:B, 0] = x
    if loss_type == 'aot_pair':  # a = pc - rc = x, b = pr - rr = y
        pol[B:, 0] = y
    else:  # aot: pc - pr = x, rc - rr = y
        ref[:B, 0] = y
    return pol, ref


@pytest.mark.parametrize('loss_type', ['aot', 'aot_pair'])
@pytest.mark.parametrize('rd', [None, BF, F16])
def test_aot_identities(loss_type, rd):
    """One kept pair: AOT is sigmoid DPO with the same label smoothing.  Co-monotone keys: AOT is sigmoid pair by pair."""
    B, W = 40, 3
    g = torch.Generator().manual_seed(9)
    pol = -torch.randint(0, 65, (2 * B, W), generator=g).double() / 8
    ref = -torch.randint(0, 65, (2 * B, W), generator=g).double() / 8
    one = torch.zeros(B, dtype=torch.bool)
    one[17] = True
    for eps in (0.0, 0.25):
        for pol_, ref_, valid in ((pol, ref, one), (*comonotone(B, W, loss_type, 3), torch.ones(B, dtype=torch.bool)),
                                  (*comonotone(B, W, loss_type, 4), torch.arange(B) % 3 != 1)):
            s = sums_of(pol_, ref_, B, rd, False)
            x = ref_k2(*s, valid, None, Opt('ext', loss_type, eps=eps), 0.125, rd, exp_cap(F32))
            y = ref_k2(*s, valid, None, Opt('ext', 'sigmoid', eps=eps), 0.125, rd, exp_cap(F32))
            _same(x['per_pair'][:, valid], y['per_pair'][:, valid], f'{loss_type} eps={eps} per_pair')
            _same(x['grad_seg'], y['grad_seg'], f'{loss_type} eps={eps} seeds')
            _same(x['stats'], y['stats'], f'{loss_type} eps={eps} stats')


def fp32_tree_sum(vals, threads=128):
    """The fp32 block reduction K2's last block used for the RPO counts: a strided per-thread sum, then xor-butterflies
    within each warp and over the warp totals."""
    vals = np.asarray(vals, dtype=np.float32)
    part = np.array([np.float32(0)] * threads, dtype=np.float32)
    for t in range(threads):
        acc = np.float32(0)
        for x in vals[t::threads]:
            acc = np.float32(acc + x)
        part[t] = acc
    w = part.reshape(threads // 32, 32)
    for o in (16, 8, 4, 2, 1):
        w = (w + w[:, np.arange(32) ^ o]).astype(np.float32)
    t = np.zeros(32, dtype=np.float32)
    t[:threads // 32] = w[:, 0]
    for o in (16, 8, 4, 2, 1):
        t = (t + t[np.arange(32) ^ o]).astype(np.float32)
    return float(t[0])


def test_rpo_count_case_has_teeth():
    """The RPO count case of the GPU file: 4500 kept pairs whose chosen counts sum past 2^25.  ATen converts the exact
    Python count to fp32 once; a fp32 tree sum rounds twice and lands on another fp32 value, so an NLL divided by it
    is not the reference's."""
    counts = rpo_counts()
    B = counts.numel() // 2
    n = int(counts[:B].sum())
    assert n > 2 ** 25
    assert fp32_tree_sum(counts[:B].numpy()) != c32(n)


def rpo_counts(B=4500, seed=3):
    """int64 [2B] row counts of the RPO count case: chosen responses of 8000-16000 scored tokens."""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(8000, 16000, (2 * B,), generator=g)
