"""K2's objective variants pinned against float64 on guarded buffers (run on an H100: `pytest -m gpu`).

`aa_dpo_loss_obj` (8 types) and `aa_dpo_loss_ext` (its own 4 types, and the JS and alpha f-divergences on the 4 types
that read h) are called through the C ABI with the loss pin's harness (tests/test_gpu_loss_kernels.py): outputs
poisoned between finite guard bands, NaN-padded strides, a zeroed counter and a status word of the test's own per
launch.  They are compared with `ref_k2` (tests/test_cpu_dpo_objective_pin.py), the float64 restatement of both
variants.

- **Matrix.** Every kind at the loss pin's pair counts and widths (`DPO_B` x `DPO_W`), AOT at B <= 1024 and at 1024
  itself, in bf16, fp16 and fp32, in both modes, with no, some or all pairs skipped.  Thinned: faithful mode runs on
  the padded stride (W + 5), f32 mode on the tight one, so each dtype meets both strides.  Label smoothing, RPO,
  reference-free, the alpha coefficient and DiscoPOP's temperature cycle over the widths (`kind_opt`).  At every
  shape: `aa_dpo_loss_ext` equals `aa_dpo_loss_obj` bit for bit on the 8 shared types, and `aa_dpo_loss_obj` at default
  fields equals `aa_dpo_loss`.
- **Bars** (DESIGN section 4.3).  The metrics (per_pair lanes 1, 2, 4, stats 1-6) and the NLL are exact on these
  operands and must match bit for bit.  The loss and the seeds (lanes 0, 3, grad_seg): f32 mode within 2e-5 relative
  (a seed that adds two terms, under JS or RPO: relative to the sum of their magnitudes),
  faithful mode within 1 ulp of the 16-bit dtype and >= 97 % bit-identical; both plus the reference's libm spread
  (`ref_spread`), and stats[0] plus the summation bound (n + 4) 2^-24 sum |loss_i| / n.
- **AOT identities** on the kernel up to 1024 pairs; **edge operand sets**; the **RPO count** past 2^25; the **refusal**
  of 1025 AOT pairs; one **node-level** case of `ops.dpo_fused_loss` at 1000 pairs.
"""
import json
import math
import os

import pytest
import torch

from align_anything_b200 import _lib as Lb
from dpo_ext_port import dpo_loss as port_loss
from dpo_ext_port import exp_cap
from oracle import ref_port as O
from test_cpu_dpo_objective_pin import AOT_MAX, FDIV, KINDS, MATRIX_B, OBJ_TYPES, SEED, TYPES, Opt, comonotone, \
    kind_opt, ref_k2, ref_spread, rpo_counts, sums_of
from test_gpu_loss_kernels import DPO_W, U, Guarded, Words, _dpo_ids, _p, _stream, assert_same, dpo_operands, \
    dpo_valid, fenced, rc_ok, rel
from test_gpu_parity import ops  # noqa: F401

DEV = 'cuda'
gpu = pytest.mark.gpu
BF, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
CODE = {BF: Lb.AA_BF16, F16: Lb.AA_F16, F32: Lb.AA_F32}
FAITHFUL, F32MODE = Lb.MODE_FAITHFUL, Lb.MODE_F32
BETA = 2.0 ** -3
L_IDS = 9
ERR_ARG = -2
# worst error of each output as a fraction of its bar, and the faithful bit-identical share (printed at the end)
WORST = {}
EXACT_SHARE = {'n': 0, 'same': 0}


def _valid(B, kind):
    if kind == 'one':
        v = torch.zeros(B, dtype=torch.bool)
        v[B // 2] = True
        return v
    return dpo_valid(B, kind)


def _ids(B, kind):
    if kind == 'none':
        return None
    if kind == 'one':
        ids = _dpo_ids(B, L_IDS, 'all')
        ids[B + B // 2, L_IDS - 1] += 1
    else:
        ids = _dpo_ids(B, L_IDS, kind)
    return fenced(ids, L_IDS + 3)


def launch(entry, pol, ref, dt, mode, o, counts, ids, stride, B, W, beta=BETA):
    """One guarded launch of entry 'obj', 'ext' or 'plain' -> (per_pair (5, B), grad_seg (2B,), stats) as float64 on
    the CPU, after the guard, counter and status checks."""
    per_pair, grad_seg = Guarded(5, B, F32), Guarded(1, 2 * B, F32)
    stats = Guarded(1, 9 if o.alpha > 0 else 8, F32)
    counter, status = Words(), Words(value=6)
    ids_args = (Lb.ptr(ids), L_IDS, L_IDS + 3 if ids is not None else 0)
    out = (per_pair.ptr(), grad_seg.ptr(), stats.ptr(), counter.ptr())
    if entry == 'plain':
        rc = Lb.lib().aa_dpo_loss(_p(pol), _p(ref), CODE[dt], B, W, stride, beta, mode, *ids_args, *out, None, None,
                                  status.ptr(), _stream())
    else:
        head = (_p(pol), None if o.ref_free else _p(ref), CODE[dt], B, W, stride, beta, mode, TYPES[o.loss_type], o.eps,
                o.alpha)
        if entry == 'obj':
            rc = Lb.lib().aa_dpo_loss_obj(*head, Lb.ptr(counts), *ids_args, *out, status.ptr(), _stream())
        else:
            e = o.eps or 1e-3
            rc = Lb.lib().aa_dpo_loss_ext(*head, FDIV[o.fdiv], o.coef, o.tau, math.log(1 - e), math.log(e),
                                          Lb.ptr(counts), *ids_args, *out, status.ptr(), _stream())
    rc_ok(rc, entry)
    torch.cuda.synchronize()
    for buf, what in ((per_pair, 'per_pair'), (grad_seg, 'grad_seg'), (stats, 'stats')):
        buf.check(f'{entry} {what}')
    counter.check([0], f'{entry} counter')
    status.check([6], f'{entry} status')
    return per_pair.t.double().cpu(), grad_seg.t[0].double().cpu(), stats.t[0].double().cpu()


def _bits_equal(x, y, what):
    for a, b, name in zip(x, y, ('per_pair', 'grad_seg', 'stats')):
        a, b = a.float(), b.float()
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f'{what}: {name} differs in its bits'


def _ulp(want, dt):
    fi = torch.finfo(dt)
    return torch.exp2(torch.floor(torch.log2(want.abs().clamp(min=fi.tiny)))) * fi.eps


def _bar(got, want, tol, what, key):
    assert torch.equal(torch.isnan(got), torch.isnan(want)), f'{what}: NaN pattern differs'
    fin = ~torch.isnan(want)
    g, w, t = got[fin], want[fin], tol.expand_as(want)[fin]
    inf = torch.isinf(w)
    assert torch.equal(g[inf], w[inf]), f'{what}: an infinite reference value differs'
    same_inf = (g == w)
    err = torch.where(same_inf, torch.zeros_like(g), (g - w).abs())
    bad = err > t
    assert not bool(bad.any()), (f'{what}: {int(bad.sum())} beyond the bar, first got {float(g[bad][0])!r} want '
                                 f'{float(w[bad][0])!r} bar {float(t[bad][0]):.3e}')
    if err.numel():
        frac = float((err / t.clamp(min=1e-300)).max())
        WORST[key] = max(WORST.get(key, 0.0), frac)


def check(got, r, sp, dt, rd, n_sum_abs, what):
    """got: the launch's outputs; r, sp: the reference and its spread."""
    pp, gs, st = got
    rp, rg, rs = r['per_pair'], r['grad_seg'], r['stats']
    v = rp[4].bool()
    n = int(v.sum())
    for lane, name in ((1, 'better'), (2, 'worse'), (4, 'valid')):
        assert_same(pp[lane], rp[lane], f'{what} per_pair[{lane}] {name}')
    assert_same(st[1:7], rs[1:7], what + ' stats[1:7]')
    assert float(st[7]) == 6.0, what + ' stats[7] carries the status word'
    if rs.numel() > 8:
        assert_same(st[8:9], rs[8:9], what + ' nll')
    assert torch.equal(gs[:gs.numel() // 2].float().view(torch.int32), pp[3].float().view(torch.int32)), what + ' g lane'
    if n == 0:  # the empty mean: NaN means, seeds (+0, -0), nothing else written (the guards above)
        assert bool(torch.isnan(st[:6]).all()) and float(st[6]) == 0.0, what + ' empty mean is NaN'
        B = pp.size(1)
        assert bool((gs[:B].float().view(torch.int32) == 0).all()), what + ' chosen seeds +0'
        assert bool((gs[B:].float().view(torch.int32) == -2 ** 31).all()), what + ' rejected seeds -0'
        if rs.numel() > 8:
            assert bool(torch.isnan(st[8])), what + ' empty NLL'
        return
    fam = 'f32' if rd is None else 'faithful'
    terms = r['seed_terms']  # a seed that adds two terms (JS, RPO) may cancel: f32 mode's bar is relative to the terms
    for got_, want, s, name, scale in ((pp[0], rp[0], sp['per_pair'][0], 'loss_i', rp[0]),
                                       (pp[3], rp[3], sp['per_pair'][3], 'g', terms[:rp.size(1)]),
                                       (gs, rg, sp['grad_seg'], 'grad_seg', terms)):
        base = rel(scale) if rd is None else _ulp(want, rd)
        _bar(got_, want, base + s, f'{what} {name}', f'{fam} {name}')
        if rd is not None:
            eq = (got_ == want) | (torch.isnan(got_) & torch.isnan(want))
            EXACT_SHARE['n'] += eq.numel()
            EXACT_SHARE['same'] += int(eq.sum())
            assert float(eq.double().mean()) >= 0.97 or int((~eq).sum()) <= 1, f'{what} {name}: < 97 % bit-identical'
    base = rel(rs[0]) if rd is None else _ulp(rs[0], rd)
    _bar(st[0:1], rs[0:1], base + sp['stats'][0] + (n + 4) * U * n_sum_abs / n, what + ' stats[0]', f'{fam} stats[0]')


def run_case(entry, pol64, ref64, B, W, stride, dt, mode, o, counts64, kind, what, beta=BETA):
    """Launch one case and hold it to the reference; -> the launch's outputs."""
    rd = dt if mode == FAITHFUL and dt != F32 else None
    pol, ref = fenced(pol64.to(dt), stride), fenced(ref64.to(dt), stride)
    counts = fenced(counts64.to(torch.int32).reshape(1, -1), pad=-7)[0]
    valid = _valid(B, kind)
    got = launch(entry, pol, ref, dt, mode, o, counts, _ids(B, kind), stride, B, W, beta)
    sums = sums_of(pol64.cpu(), ref64.cpu(), B, rd, o.ref_free)
    r, sp = ref_spread(sums, valid, counts64.double().cpu(), o, beta, rd, exp_cap(dt))
    check(got, r, sp, dt, rd, float(torch.where(valid, r['loss'], 0.0).abs().nan_to_num().sum()), what)
    return got, (pol, ref, counts)


def _counts(B, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(1, 4097, (2 * B,), generator=g)


MATRIX = [(k, B) for k in KINDS for B in MATRIX_B
          if (B <= AOT_MAX if k[1] in ('aot', 'aot_pair') else B != AOT_MAX)]


@gpu
@pytest.mark.parametrize('kind,B', MATRIX, ids=[f'{k[0]}-{k[1]}-{k[2]}-B{B}' for k, B in MATRIX])
def test_objective_matrix(ops, kind, B):
    for j, W in enumerate(DPO_W):
        o = kind_opt(kind, j)
        pol64, ref64 = dpo_operands(B, W, SEED + B + W)
        counts64 = _counts(B, B + W)
        for dt in (BF, F16, F32):
            for mode in (FAITHFUL, F32MODE):
                stride = W + 5 if mode == FAITHFUL else W
                for ids_kind in ('none', 'some', 'all'):
                    what = f'{o} B={B} W={W} stride={stride} {dt} mode={mode} ids={ids_kind}'
                    got, (pol, ref, counts) = run_case(o.entry, pol64, ref64, B, W, stride, dt, mode, o, counts64,
                                                       ids_kind, what)
                    ids = _ids(B, ids_kind)
                    if o.entry == 'obj':  # the extended entry computes the shared types bit for bit alike
                        _bits_equal(launch('ext', pol, ref, dt, mode, o, counts, ids, stride, B, W), got,
                                    what + ' ext == obj')
                        if o.loss_type == 'sigmoid':  # default fields: aa_dpo_loss bit for bit
                            d = Opt('obj', 'sigmoid')
                            a = launch('obj', pol, ref, dt, mode, d, None, ids, stride, B, W)
                            _bits_equal(launch('plain', pol, ref, dt, mode, d, None, ids, stride, B, W), a,
                                        what + ' obj default == aa_dpo_loss')


AOT_B = [1, 2, 127, 128, 129, 1000, AOT_MAX]


@gpu
@pytest.mark.parametrize('B', AOT_B)
@pytest.mark.parametrize('loss_type', ['aot', 'aot_pair'])
def test_aot_identities_on_the_kernel(ops, loss_type, B):
    """Co-monotone keys (skipped pairs interleaved or not), and one kept pair of random operands: AOT is sigmoid DPO
    with the same label smoothing, pair by pair and bit for bit."""
    W = 3
    counts = fenced(_counts(B, 1).to(torch.int32).reshape(1, -1), pad=-7)[0]
    for eps, alpha in ((0.0, 0.0), (0.25, 0.5)):
        sets = [(*comonotone(B, W, loss_type, B), 'none'), (*comonotone(B, W, loss_type, B + 1), 'some')]
        sets.append((*dpo_operands(B, W, B + 2, 'cpu'), 'one'))
        for pol64, ref64, kind in sets:
            v = _valid(B, kind)
            for dt in (BF, F16, F32):
                pol, ref = fenced(pol64.to(dt), W), fenced(ref64.to(dt), W)
                for mode in (FAITHFUL, F32MODE):
                    what = f'{loss_type} B={B} eps={eps} alpha={alpha} {dt} mode={mode} ids={kind}'
                    ids = _ids(B, kind)
                    x = launch('ext', pol, ref, dt, mode, Opt('ext', loss_type, eps=eps, alpha=alpha), counts, ids, W,
                               B, W)
                    y = launch('ext', pol, ref, dt, mode, Opt('ext', 'sigmoid', eps=eps, alpha=alpha), counts, ids, W,
                               B, W)
                    _bits_equal((x[0][:, v], x[1], x[2]), (y[0][:, v], y[1], y[2]), what)


# ---- edge operand sets ------------------------------------------------------------------------------------------------
def _pairs(vals, W=1):
    """(pol, ref) float64 (2B, W) whose row sums are the given (pc, pr, rc, rr) per pair (spread over W columns)."""
    v = torch.tensor(vals, dtype=F64)
    B = v.size(0)
    pol, ref = torch.zeros(2 * B, W, dtype=F64), torch.zeros(2 * B, W, dtype=F64)
    pol[:B, 0], pol[B:, 0], ref[:B, 0], ref[B:, 0] = v[:, 0], v[:, 1], v[:, 2], v[:, 3]
    return pol, ref


def edge_sets(name, dt):
    """-> list of (pol, ref, counts, [Opt], ids kind, beta)."""
    cap = exp_cap(dt)
    if name == 'hinge_kink':  # beta h = 1 exactly (h = 8) and its neighbours
        pol, ref = _pairs([(0, 0, -8, 0), (0, 0, -8.125, 0), (0, 0, -7.875, 0), (1, 0, -7, 0)])
        return [(pol, ref, torch.full((8,), 4), [Opt('obj', 'hinge'), Opt('ext', 'hinge', fdiv='js_divergence')],
                 'none', BETA)]
    if name == 'ipo_sppo_zero':  # h = 1 / (2 beta) = 4 with power-of-two counts (IPO); a = 4, b = -4 (SPPO)
        pol, ref = _pairs([(0, -8, -16, -8), (0, 0, -16, 0), (4, -8, -12, -8), (0, -2, -4, -2)])
        sp_pol, sp_ref = _pairs([(0, -4, -4, 0), (4, 0, 0, 4), (0, -4, -4.125, 0), (1, -3, -3, 1)])
        return [(pol, ref, torch.tensor([4, 4, 4, 4, 2, 2, 2, 2]), [Opt('obj', 'ipo')], 'none', BETA),
                (sp_pol, sp_ref, torch.full((8,), 4), [Opt('obj', 'sppo_hard')], 'none', BETA)]
    if name == 'js_20':  # a and b on both sides of softplus' threshold 20
        pol, ref = _pairs([(19.875, 20.125, 0, 0), (20, 20, 0, 0), (20.125, 19.875, 0, 0), (-20.125, 21, 0, 0),
                           (30, -3, 0, 0), (0, 19.875, -20.125, 0)])
        return [(pol, ref, torch.full((12,), 4), [Opt('ext', t, fdiv='js_divergence') for t in
                                                  ('sigmoid', 'robust', 'hinge', 'exo_pair')], 'none', BETA)]
    if name == 'alpha_clamp':  # -coef a past the cap on one key, on both, and exactly at it (coef = the cap, a = -1)
        big = math.ceil(cap) + 4
        pol, ref = _pairs([(-big, -2, 0, 0), (-2, -big, 0, 0), (-big, -big - 8, 0, 0), (-1, -2, 0, 0),
                           (-1, -1, 0, 0), (-0.5, -1, 0, 0)])
        c = float(torch.tensor(cap, dtype=F32))
        return [(pol, ref, torch.full((12,), 4),
                 [Opt('ext', t, fdiv='alpha_divergence', coef=k) for t in ('sigmoid', 'hinge') for k in (1.0, c)],
                 'none', BETA)]
    if name == 'exp_overflow':  # |z| = |beta h| past expf's overflow (88.72), DiscoPOP's NaN where exp(-z) * 0
        hs = [-800, -720, -712, -704, -8, 0, 8, 704, 720, 800]
        pol, ref = _pairs([(h, 0, 0, 0) for h in hs])
        opts = [Opt('ext', 'discopop'), Opt('ext', 'discopop', tau=2.0 ** -9), Opt('ext', 'discopop', tau=1.0),
                Opt('ext', 'exo_pair'), Opt('ext', 'exo_pair', eps=0.25)]
        return [(pol, ref, torch.full((20,), 4), opts, 'none', BETA)]
    if name == 'fp16_overflow':  # rows whose fp16 sums overflow to -inf in faithful mode (-4096 * 31 = -126976)
        W = 31
        pol = torch.zeros(8, W, dtype=F64)
        ref = torch.zeros(8, W, dtype=F64)
        pol[0], pol[5], ref[2], ref[3], ref[7] = -4096, -4096, -4096, -4096, -4096
        pol[1, :3] = -1
        opts = [Opt('obj', t) for t in ('sigmoid', 'ipo', 'nca_pair', 'apo_down')] + \
            [Opt('ext', 'exo_pair'), Opt('ext', 'aot_pair'), Opt('ext', 'sigmoid', fdiv='js_divergence'),
             Opt('ext', 'sigmoid', fdiv='alpha_divergence', coef=1.5)]
        return [(pol, ref, torch.full((8,), 31), opts, 'none', BETA)]
    if name == 'aot_nan_ties':  # 300 pairs: three passes of the last block; ties 128 apart, NaN keys, skips interleaved
        B, W = 300, 2
        g = torch.Generator().manual_seed(12)
        pol = -torch.randint(0, 9, (2 * B, W), generator=g).double() / 8
        ref = -torch.randint(0, 9, (2 * B, W), generator=g).double() / 8
        for i in range(0, B - 256, 7):
            pol[i + 128], pol[i + 256], ref[i + 128] = pol[i], pol[i], ref[i]
        pol[[5, 133, 261], 1] = math.nan  # a NaN first key (and a = pc - rc) in each pass
        ref[[B + 17, B + 200], 0] = math.nan  # NaN second keys
        opts = [Opt('ext', 'aot'), Opt('ext', 'aot_pair', eps=0.125), Opt('ext', 'aot', alpha=0.5)]
        return [(pol, ref, _counts(B, 3), opts, kind, BETA) for kind in ('none', 'some', 'all', 'one')]
    raise ValueError(name)


EDGES = ['hinge_kink', 'ipo_sppo_zero', 'js_20', 'alpha_clamp', 'exp_overflow', 'fp16_overflow', 'aot_nan_ties']


@gpu
@pytest.mark.parametrize('name', EDGES)
def test_edge_operands(ops, name):
    for dt in (BF, F16, F32):
        for pol64, ref64, counts64, opts, kind, beta in edge_sets(name, dt):
            B, W = pol64.size(0) // 2, pol64.size(1)
            for o in opts:
                for mode in (FAITHFUL, F32MODE):
                    what = f'{name} {o} {dt} mode={mode} ids={kind}'
                    (pp, gs, st), _ = run_case(o.entry, pol64, ref64, B, W, W, dt, mode, o, counts64, kind, what, beta)
                    if name == 'hinge_kink' and o.fdiv == 'reverse_kl':
                        assert float(pp[0, 0]) == 0.0 and float(gs[0]) == 0.0 and float(gs[B]) == 0.0, what
                    if name == 'ipo_sppo_zero':
                        assert float(pp[0, 0]) == 0.0 and float(gs[0]) == 0.0 and float(gs[B]) == 0.0, what
                    if name == 'exp_overflow' and o.loss_type == 'discopop' and o.tau != 1.0:  # NaN where TRL has it
                        assert bool(torch.isnan(pp[0, :3]).all()) and not bool(torch.isnan(pp[0, 4:]).any()), what
                    if name == 'fp16_overflow' and dt == F16 and mode == FAITHFUL:
                        assert bool(torch.isinf(st[2]) | torch.isnan(st[2])), what + ' -inf row sum reaches the metric'


@gpu
@pytest.mark.parametrize('entry,loss_type', [('obj', 'sigmoid'), ('ext', 'exo_pair'), ('ext', 'aot')])
def test_rpo_count_past_2_pow_25(ops, entry, loss_type):
    """4500 pairs (1024 under AOT) whose chosen counts sum past 2^25: the NLL divides by the count rounded to fp32
    once, bit for bit."""
    B, W = (4500, 2047) if loss_type != 'aot' else (AOT_MAX, 2047)
    counts64 = rpo_counts() if B == 4500 else rpo_counts(B=B) * 4
    assert int(counts64[:B].sum()) > 2 ** 25
    pol64, ref64 = dpo_operands(B, W, SEED + 7)
    o = Opt(entry, loss_type, alpha=0.5)
    for dt in (BF, F16, F32):
        for mode in (FAITHFUL, F32MODE):
            run_case(entry, pol64, ref64, B, W, W, dt, mode, o, counts64, 'some', f'RPO count {o} {dt} mode={mode}')


@gpu
def test_aot_refuses_past_its_limit(ops):
    """1025 AOT pairs: AA_ERR_ARG at the C ABI, and every guarded buffer, the counter and the status word untouched."""
    assert ops.DPO_AOT_MAX_PAIRS == AOT_MAX
    B, W = AOT_MAX + 1, 4
    pol, ref = fenced(torch.zeros(2 * B, W, dtype=BF), W), fenced(torch.zeros(2 * B, W, dtype=BF), W)
    for loss_type in ('aot', 'aot_pair'):
        per_pair, grad_seg, stats = Guarded(5, B, F32), Guarded(1, 2 * B, F32), Guarded(1, 8, F32)
        counter, status = Words(), Words(value=6)
        rc = Lb.lib().aa_dpo_loss_ext(_p(pol), _p(ref), CODE[BF], B, W, W, BETA, FAITHFUL, TYPES[loss_type], 0.0, 0.0,
                                      0, 1.0, 0.05, math.log(1 - 1e-3), math.log(1e-3), None, None, 0, 0,
                                      per_pair.ptr(), grad_seg.ptr(), stats.ptr(), counter.ptr(), status.ptr(),
                                      _stream())
        torch.cuda.synchronize()
        assert rc == ERR_ARG, rc
        for buf in (per_pair, grad_seg, stats):
            assert buf.untouched(), loss_type
        counter.check([0], 'counter')
        status.check([6], 'status')


@gpu
def test_fused_node_at_1000_pairs_against_float64(ops):
    """ops.dpo_fused_loss at 1000 pairs, exo_pair under JS with RPO and skipped identical pairs, against float64
    autograd through the port: ops passes the counts, ids and strides through at that size."""
    obj = ops.DpoObjective(loss_type='exo_pair', f_divergence_type='js_divergence', rpo_alpha=0.5)
    B, L_, V, pad = 1000, 12, 64, 0
    g = torch.Generator().manual_seed(31)
    logits = torch.randn(2 * B, L_, V, generator=g) * 2
    ref_logits = logits + torch.randn(2 * B, L_, V, generator=g) / 2
    ids = torch.randint(1, V, (2 * B, L_), generator=g)
    ids[B::7] = ids[:B:7]
    lens = torch.randint(2, L_, (2 * B,), generator=g).tolist()
    for i in range(0, B, 7):
        lens[B + i] = lens[i]
    leaf64 = logits.double().requires_grad_(True)
    lp = O.dpo_sequence_log_probs(leaf64, ids, lens, pad, True)
    rlp = O.dpo_sequence_log_probs(ref_logits.double(), ids, lens, pad, True)
    want = port_loss(lp, rlp, BETA, ids, True, 'exo_pair', 0.0, 0.5, False, lens, 'js_divergence', cap=exp_cap(F32))
    want['loss'].backward()
    leaf = logits.to(DEV).requires_grad_(True)
    out = ops.dpo_fused_loss(leaf, ref_logits.to(DEV), ids.to(DEV), lens, pad, BETA, skip_identical_pairs=True,
                             mode='f32', objective=obj)
    out['loss'].backward()
    for got, w, what in ((out['loss'], want['loss'], 'loss'), (out['nll_loss'], want['nll_loss'], 'nll'),
                         (leaf.grad, leaf64.grad, 'd logits')):
        got, w = got.detach().double().cpu(), w.detach().double().cpu()
        tol = 1e-4 * w.abs() + 1e-6 * float(w.abs().max())
        assert bool(((got - w).abs() <= tol).all()), f'{what}: max err {float((got - w).abs().max()):.3e}'


@gpu
def test_zz_report():
    """Runs last: prints the worst error of each output as a fraction of its bar, and the faithful bit-identical
    share, over the cases of this session (and writes them as JSON to $AA_PIN_REPORT when it is set)."""
    if not EXACT_SHARE['n']:
        pytest.skip('no case of this file ran in this session')
    rep = {'worst_fraction_of_bar': WORST, 'faithful_bit_identical': EXACT_SHARE['same'] / EXACT_SHARE['n']}
    print('\nK2 objective pin:', json.dumps(rep, indent=1, sort_keys=True))
    assert max(WORST.values()) <= 1.0
    out = os.environ.get('AA_PIN_REPORT')
    if out:
        with open(out, 'w') as f:
            json.dump(rep, f, indent=1, sort_keys=True)
