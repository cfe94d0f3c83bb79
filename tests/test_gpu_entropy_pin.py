"""The per-token entropy of the log-prob kernels pinned against float64 (run on an H100: `pytest -m gpu`).

Three entry points write or read the entropy H = -sum_j p_j log p_j that the `log_entropy` metric, the entropy bonus and
GRPO's top-entropy mask use; each runs here through the C ABI over the matrix of the earlier tile pins:
  * K1 `aa_logprob_fwd_entropy` over test_gpu_logprob_tiles.CASES (row plans, layouts, V from 1 to 128257, the
    ring / LDG switch at 128 KB rows), on the bulk-copy ring kernel, the LDG kernel and (long rows) the default route,
    plus a two-copy plan cut by n_entropy and planted rows (near one-hot, uniform, -inf peels, one finite logit, all
    -inf, fp16 at +-65504);
  * K6 `aa_linear_logprob_fwd_entropy` over test_gpu_lm_head_tiles.FWD_CASES at three `partial` budgets
    (test_cpu_entropy_pin: 'wide4', 'none' and the case's own kind counted at three floats per split);
  * K6b `aa_linear_dlogits_entropy` over test_gpu_lm_head_tiles.DLOGITS_CASES, fed its own K6 entropy launch, with g_H
    in bf16, fp16 and fp32.

The entropy bar is |H - H64| <= min(1e-4, 1e-5 * max(1, H64)).  It comes from the arithmetic: H = log s + |t| / s is a
sum of two non-negative terms (t = sum_j e^{x_j - m} (x_j - m) <= 0), so nothing cancels, and the error is that of
ex2.approx (<= 2^-22 relative, common to s and t, so it mostly drops out of t / s) and of fp32 partial sums of at most
a few thousand terms per thread -- around 1e-6 * H.  Every case prints its worst error / bar as a HEADROOM line.
"""
from __future__ import annotations

import math

import pytest
import torch

from align_anything_b200 import _lib as Lb
from test_cpu_entropy_pin import K6_IDS, K6_PARAMS, SPLIT_COUNTS_DIFFER, k6_budgets
from test_gpu_entropy import entropy64
from test_gpu_lm_head_tiles import (BM, BN, DLOGITS_CASES, _device_status_ptr, _dlogits_case_id, _fwd_operands,
                                    _half_ulp_bf16, _headroom, _ordered, _plant_labels, _plant_saturated, _stream, _up,
                                    _upstream, poisoned_operand, schedule, vec_guard)
from test_gpu_lm_head_tiles import Guarded as GuardedLM
from test_gpu_logprob_tiles import CASES, INT, POISON, Case, Guarded, _case_id, _status_take
from test_gpu_parity import ops  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

DEV = 'cuda'
BF, F16, F32 = torch.bfloat16, torch.float16, torch.float32
RING, LDG, DEFAULT = 1, 2, 0  # aa_logprob_set_tuning variants
ROUTE_NAME = {RING: 'ring', LDG: 'ldg', DEFAULT: 'default'}


def entropy_bar(h64):
    """min(1e-4, 1e-5 * max(1, H64)) per row (float64)."""
    return torch.clamp(1e-5 * h64.clamp(min=1.0), max=1e-4)


def check_entropy(got, want64, what):
    """got (fp32) against float64: same NaN pattern, every other row within entropy_bar -> worst err / bar."""
    want64 = want64.to(got.device)
    nan = torch.isnan(want64)
    assert torch.equal(torch.isnan(got), nan), f'{what}: NaN pattern of the entropy'
    if bool(nan.all()):
        return 0.0
    err = (got.double() - want64).abs()[~nan]
    tol = entropy_bar(want64[~nan])
    bad = ~(err <= tol)
    assert not bool(bad.any()), (f'{what}: {int(bad.sum())} entropies beyond the bar, max err {float(err.max()):.3e} '
                                 f'(H64 {float(want64[~nan][bad.nonzero()[0, 0]]):.6f})')
    return float((err / tol).max())


def _bits(t):
    return t.contiguous().view(INT[t.element_size()])


# ---- K1 --------------------------------------------------------------------------------------------------------------
def _set_route(route):
    Lb.check(Lb.lib().aa_logprob_set_tuning(route, 0))


def _k1(logits_ptr, dtype, row_stride, V, labels, ignore, plan, out, stats, ent=None, n_ent=0):
    """One aa_logprob_fwd (ent None) or aa_logprob_fwd_entropy launch -> the status word it raised."""
    from align_anything_b200 import ops as _ops

    p = plan.ptrs()
    args = (logits_ptr, Lb.dtype_code(dtype), row_stride, V, labels.data_ptr(), 0 if ignore is None else ignore,
            0 if ignore is None else 1, plan.n_seg, plan.n_rows, p[0], p[1], p[2], p[3], out.data_ptr(),
            Lb.dtype_code(out.dtype), stats[0].data_ptr(), stats[1].data_ptr(),
            _ops._device_scratch(torch.device(DEV))['status'].data_ptr())
    _status_take()
    if ent is None:
        Lb.check(Lb.lib().aa_logprob_fwd(*args, Lb.stream_ptr(torch.device(DEV))))
    else:
        Lb.check(Lb.lib().aa_logprob_fwd_entropy(*args, ent, n_ent, Lb.stream_ptr(torch.device(DEV))))
    torch.cuda.synchronize()
    return _status_take()


def _poisoned(shape, dtype):
    t = torch.empty(shape, dtype=dtype, device=DEV)
    t.view(INT[t.element_size()]).fill_(POISON[t.element_size()])
    return t


def _k1_pair(logits_ptr, dtype, row_stride, V, labels, ignore, plan, out_shape, out_dtype, n_out, n_ent):
    """The plain and the entropy launch into fresh poisoned buffers; the entropy into a guarded fp32 vector of n_out
    values -> (plain (out, stats, status), entropy (out, stats, status), guarded entropy)."""
    runs = []
    for with_ent in (False, True):
        out = _poisoned(out_shape, out_dtype)
        stats = _poisoned((2, max(plan.n_rows, 1)), F32)
        ent = Guarded(1, n_out, n_out, F32) if with_ent else None
        status = _k1(logits_ptr, dtype, row_stride, V, labels, ignore, plan, out, stats,
                     ent.tile.data_ptr() if ent else None, n_ent)
        runs.append((out, stats, status, ent))
    return runs[0][:3], runs[1][:3], runs[1][3]


def _same_outputs(a, b, what):
    """out, stat_max, stat_logsum and the status word of two launches are bit-identical."""
    assert torch.equal(_bits(a[0]), _bits(b[0])), f'{what}: log-probs differ with the entropy on'
    assert torch.equal(_bits(a[1]), _bits(b[1])), f'{what}: statistics differ with the entropy on'
    assert a[2] == b[2], f'{what}: status {a[2]:#x} with the entropy off, {b[2]:#x} with it on'


def _k1_routes(dtype, V):
    long_row = (dtype == F32 and V >= 32768) or (dtype != F32 and V == 128257)
    return [RING, LDG] + ([DEFAULT] if long_row else [])


K1_PARAMS = [(c, r) for c in CASES for r in _k1_routes(c[0], c[1])]
K1_IDS = [f'K1-{_case_id(c)}-{ROUTE_NAME[r]}' for c, r in K1_PARAMS]


@pytest.mark.parametrize('case_args,route', K1_PARAMS, ids=K1_IDS)
def test_k1_entropy_tile_matrix(ops, case_args, route):
    """aa_logprob_fwd_entropy on one log-prob tile pin case and one K1 kernel, with the out dtype of both modes:
      * out, stat_max, stat_logsum and the status word bit-identical to aa_logprob_fwd on the same route;
      * every scored row's entropy within entropy_bar of entropy64 of the fp32-upcast row (an out-of-range label
        included: the entropy does not depend on it), ignored rows exactly 0;
      * out positions the plan does not score, positions >= n_entropy and the guards keep their poison / sentinel
        bits (the second launch cuts n_entropy three scored rows before the end and writes the same bits below it)."""
    case = Case(ops, *case_args)
    what = K1_IDS[K1_PARAMS.index((case_args, route))]
    n_out = math.prod(case.out_shape)
    ig = -100 if case.ignore else None
    args = (case.logits.data_ptr(), case.dtype, case.lpitch, case.V, case.labels, ig, case.plan)
    written = torch.zeros(n_out, dtype=torch.bool)
    written[case.out_idx] = True
    written = written.to(DEV)
    x = case.logits[case.tile_row.to(DEV)]
    want = entropy64(x)
    ign = case.ignored.to(DEV)
    _set_route(route)
    try:
        worst = 0.0
        for out_dtype in sorted({case.dtype, F32}, key=str):
            plain, with_ent, ent = _k1_pair(*args, case.out_shape, out_dtype, n_out, n_out)
            _same_outputs(plain, with_ent, f'{what} out {out_dtype}')
            assert bool((with_ent[2] & Lb.STATUS_LABEL_OOB) != 0) == bool(case.oob.any()), f'{what}: status'
            keep = ent.outside()
            assert torch.equal(ent.bits[keep], ent.fresh[keep]), f'{what}: a guard of the entropy changed'
            eb = ent.row_bits(0)
            assert bool((eb[written] != POISON[4]).all()), f'{what}: an entropy was not written'
            assert bool((eb[~written] == POISON[4]).all()), f'{what}: an entropy written outside the scored rows'
            got = ent.tile[0][case.out_idx.to(DEV)]
            if bool(ign.any()):
                assert bool((got[ign] == 0).all()), f'{what}: an ignored row must have entropy 0'
            worst = max(worst, check_entropy(got[~ign], want[~ign], what))
            if bool(case.oob.any()):
                oob = case.oob.to(DEV)
                assert bool(torch.isfinite(got[oob]).all()), f'{what}: out-of-range label rows keep their entropy'
            # n_entropy three scored rows before the end: the same bits below it, poison from it on
            n_ent = int(case.out_idx[-3])
            cut = Guarded(1, n_out, n_out, F32)
            out = _poisoned(case.out_shape, out_dtype)
            stats = _poisoned((2, max(case.plan.n_rows, 1)), F32)
            st = _k1(*args, out, stats, cut.tile.data_ptr(), n_ent)
            _same_outputs(plain, (out, stats, st), f'{what} n_entropy {n_ent}')
            cb = cut.row_bits(0)
            assert torch.equal(cb[:n_ent], eb[:n_ent]), f'{what}: the cut launch wrote other entropies'
            assert bool((cb[n_ent:] == POISON[4]).all()), f'{what}: an entropy written at or past n_entropy'
            keep = cut.outside()
            assert torch.equal(cut.bits[keep], cut.fresh[keep]), f'{what}: a guard changed (cut launch)'
    finally:
        _set_route(DEFAULT)
    _headroom(f'{what} entropy (err / bar)', worst, 1.0)


@pytest.mark.parametrize('route', [RING, LDG], ids=['ring', 'ldg'])
@pytest.mark.parametrize('dtype', [BF, F16, F32], ids=['bf16', 'f16', 'f32'])
def test_k1_entropy_two_copy_plan(ops, dtype, route):
    """aa_tail_plan_build with copies = 2 (actor and reference in one launch) and n_entropy = copy_out_delta: the
    entropy buffer holds exactly copy_out_delta values; the first copy's entropies are written and match float64,
    unscored positions keep their poison, and the guard after the buffer is unchanged although the second copy's rows
    map past it.  Log-probs and statistics are bit-identical to aa_logprob_fwd's."""
    V, B, S = 4097, 6, 12
    lens = [S - 1, 0, 7, -2, 3, S // 2]
    W = S - 1
    gen = torch.Generator().manual_seed(V + len(str(dtype)))
    logits = (torch.randn(2, B * S, V, generator=gen) * 2.5).to(dtype).to(DEV)
    labels = torch.randint(0, V, (B, S), generator=gen).to(DEV)
    dl = ops.DeviceLens(torch.tensor(lens, dtype=torch.int32, device=DEV), W)
    plan = ops.DevicePlan(dl, S, S * V, V, S, S, 0, -1, W, copies=2, copy_logit_delta=B * S * V)
    _status_take()
    n_out = B * W  # copy_out_delta
    rows, out_idx = [], []
    for b, r in enumerate(lens):
        r = max(0, min(r, S - 1))
        for j in range(min(r, W)):
            rows.append(b * S + S - r - 1 + j)
            out_idx.append(b * W + j)
    what = f'K1 two-copy {dtype} V={V} {ROUTE_NAME[route]}'
    _set_route(route)
    try:
        plain, with_ent, ent = _k1_pair(logits.data_ptr(), dtype, V, V, labels, None, plan, plan.out_shape, F32,
                                        n_out, n_out)
    finally:
        _set_route(DEFAULT)
    _same_outputs(plain, with_ent, what)
    keep = ent.outside()
    assert torch.equal(ent.bits[keep], ent.fresh[keep]), f'{what}: the second copy wrote past copy_out_delta'
    written = torch.zeros(n_out, dtype=torch.bool)
    written[out_idx] = True
    eb = ent.row_bits(0)
    assert bool((eb[written.to(DEV)] != POISON[4]).all()) and bool((eb[~written.to(DEV)] == POISON[4]).all())
    got = ent.tile[0][torch.tensor(out_idx, device=DEV)]
    r = check_entropy(got, entropy64(logits[0][torch.tensor(rows, device=DEV)]), what)
    _headroom(f'{what} entropy (err / bar)', r, 1.0)


def _planted_rows(dtype, V, gen):
    """(R, V) rows in the 'odd' layout (the logits base one element off, so row 0 has a head peel):
    row 0: -inf in the head-peel and tail-peel elements, random in the body;  1: near one-hot (H ~ 0);  2: uniform
    (H = log V);  3 and 4: exactly one finite logit, in the body and at column 0 (H = 0 exactly: 0 * (-inf) would be
    NaN without the -3e38 clamp);  5: all -inf (NaN);  6 (fp16): logits at +-65504;  then random rows."""
    esz = torch.empty(0, dtype=dtype).element_size()
    E = 16 // esz
    R = 10
    x = torch.randn(R, V, generator=gen) * 2.5
    mis = (1 * esz % 16) // esz
    head = min(E - mis, V) if mis else 0
    tail0 = head + (V - head) // E * E
    x[0, :head] = float('-inf')
    x[0, tail0:] = float('-inf')
    x[1] = 0.0
    x[1, V // 3] = 40.0
    x[2] = 1.5
    x[3] = float('-inf')
    x[3, (3 * V) // 5] = 0.7
    x[4] = float('-inf')
    x[4, 0] = -3.25
    x[5] = float('-inf')
    if dtype == F16:
        sgn = torch.randint(0, 2, (V,), generator=gen) * 2 - 1
        x[6] = torch.where(torch.rand(V, generator=gen) < 0.5, sgn * 65504.0, x[6])
    return x.to(dtype)


@pytest.mark.parametrize('route', [RING, LDG], ids=['ring', 'ldg'])
@pytest.mark.parametrize('V', [7, 9, 4097, 32767, 32769])
@pytest.mark.parametrize('dtype', [BF, F16, F32], ids=['bf16', 'f16', 'f32'])
def test_k1_entropy_planted_rows(ops, dtype, V, route):
    """The rows where an online entropy goes wrong, on both K1 kernels, against float64; log-probs and statistics
    bit-identical to aa_logprob_fwd's."""
    gen = torch.Generator().manual_seed(V * 3 + len(str(dtype)))
    x = _planted_rows(dtype, V, gen)
    R = x.size(0)
    buf = torch.zeros(R * V + 16, dtype=dtype)
    buf[1:1 + R * V] = x.reshape(-1)
    buf = buf.to(DEV)
    logits = buf[1:1 + R * V].view(R, V)
    labels = torch.randint(0, V, (R,), generator=gen).to(DEV)
    plan = ops.RowPlan([0], [0], [0], [R], [0], (1, R), 0, DEV)
    what = f'K1 planted {dtype} V={V} {ROUTE_NAME[route]}'
    _set_route(route)
    try:
        plain, with_ent, ent = _k1_pair(logits.data_ptr(), dtype, V, V, labels, None, plan, (1, R), F32, R, R)
    finally:
        _set_route(DEFAULT)
    _same_outputs(plain, with_ent, what)
    keep = ent.outside()
    assert torch.equal(ent.bits[keep], ent.fresh[keep]), f'{what}: a guard of the entropy changed'
    got = ent.tile[0]
    want = entropy64(logits)
    assert bool((got[3:5] == 0).all()), f'{what}: one finite logit must give H = 0 exactly, got {got[3:5].tolist()}'
    assert bool(torch.isnan(got[5])), f'{what}: an all -inf row must give NaN'
    assert float(got[1]) <= 1e-6, f'{what}: near one-hot H = {float(got[1])}'
    assert abs(float(got[2]) - math.log(V)) <= entropy_bar(torch.tensor(math.log(V), dtype=torch.float64)), \
        f'{what}: uniform H = {float(got[2])}, log V = {math.log(V)}'
    r = check_entropy(got, want, what)
    _headroom(f'{what} entropy (err / bar)', r, 1.0)


# ---- K6 --------------------------------------------------------------------------------------------------------------
def _k6(hidden, weight, labels, mode, pf, n, V, H, entropy):
    """One K6 launch (entropy: the entropy variant) into guarded buffers -> (out, max, logsum, partial or None,
    entropy or None, status)."""
    out = vec_guard(n, BF if mode == Lb.MODE_FAITHFUL else F32)
    smax, slog = vec_guard(n, F32), vec_guard(n, F32)
    part = vec_guard(pf, F32) if pf else None
    ent = vec_guard(n, F32) if entropy else None
    args = (hidden.data_ptr(), n, H, hidden.stride(0), weight.data_ptr(), V, weight.stride(0), labels.data_ptr(),
            out.ptr(), Lb.dtype_code(out.t.dtype), smax.ptr(), slog.ptr(), part.ptr() if part else None, pf, mode,
            _device_status_ptr())
    _status_take()
    if entropy:
        Lb.check(Lb.lib().aa_linear_logprob_fwd_entropy(*args, ent.ptr(), _stream()))
    else:
        Lb.check(Lb.lib().aa_linear_logprob_fwd(*args, _stream()))
    torch.cuda.synchronize()
    return out, smax, slog, part, ent, _status_take()


def _k6_inputs(case):
    """test_k6_forward_exact's operands: exact hidden / weight, planted labels (-1 and V included unless n = 129),
    saturated rows, strided operands for even n."""
    n, H, V, kind, _ = case
    pf = {'none': 0, 'wide': n * torch.cuda.get_device_properties(0).multi_processor_count * 3, 'two': n * 2 * 3}[kind]
    splits, tps, _ = schedule(n, V, kind != 'none', pf)
    labels = _plant_labels(n, V, splits, tps, n + V, oob=n != 129)
    hidden, weight = _fwd_operands(n, H, V)
    sat_rows = [r for r in (n // 2, n - 1) if n > 8]
    _plant_saturated(hidden, weight, labels, sat_rows, H)
    hs, ws = (H, H) if n % 2 else (H + 8, H + 64)
    return poisoned_operand(hidden, hs), poisoned_operand(weight, ws), labels.to(DEV), sat_rows


@pytest.mark.parametrize('case,budget', K6_PARAMS, ids=[f'K6-{i}' for i in K6_IDS])
def test_k6_entropy_schedules(ops, case, budget):
    """aa_linear_logprob_fwd_entropy against float64 on exact operands, both modes, at one `partial` budget:
      * the entropy of every row within entropy_bar of entropy64 of the float64 logits (FAITHFUL: rounded to bf16
        first, exact on these operands), out-of-range labels included; saturated rows H <= 1e-6;
      * `partial` written over exactly n * splits * 4 floats (splits of the 4-float schedule; none when unsplit) and
        nowhere past, every output written, nothing outside the outputs;
      * out, stat_max and stat_logsum bit-identical to aa_linear_logprob_fwd with the same `partial` whenever the two
        launches run the same split count, as include/aa_b200.h promises (`partial` NULL, or room for 4 floats per
        row and split).  Where they do not (test_cpu_entropy_pin.SPLIT_COUNTS_DIFFER: a budget of 3 floats per split
        that holds the plain launch's two splits but not the entropy launch's), the statistics are merged in another
        order and the header promises no bit-identity -- on an H100 80GB HBM3 the two launches' outputs were not
        bit-identical at either such budget, in either mode.  Both launches then meet test_k6_forward_exact's bars against float64 (stat_max
        bit-exact, stat_logsum and f32 log-probs within 2e-5 * max(1, |ref|), faithful log-probs the bf16 rounding of
        the launch's own statistics), and whether the bits matched is printed."""
    n, H, V, kind, _ = case
    S = torch.cuda.get_device_properties(0).multi_processor_count
    pf = k6_budgets(case, S)[budget]
    cid = K6_IDS[K6_PARAMS.index((case, budget))]
    splits4 = schedule(n, V, pf > 0, pf, 4)[0]
    splits3 = schedule(n, V, pf > 0, pf, 3)[0]
    assert (splits3 != splits4) == (cid in SPLIT_COUNTS_DIFFER), 'test_cpu_entropy_pin lists the differing budgets'
    hidden, weight, labels, sat_rows = _k6_inputs(case)
    x64 = hidden.double() @ weight.double().T
    lab_ok = (labels >= 0) & (labels < V)
    y = torch.where(lab_ok, labels, torch.zeros_like(labels))
    worst = 0.0
    for mode in (Lb.MODE_FAITHFUL, Lb.MODE_F32):
        what = f'K6 {cid} mode {mode}'
        plain = _k6(hidden, weight, labels, mode, pf, n, V, H, False)
        out, smax, slog, part, ent, status = _k6(hidden, weight, labels, mode, pf, n, V, H, True)
        for gd in (out, smax, slog, ent):
            assert gd.outside_intact(), f'{what}: write outside an output'
            assert not bool((gd.region_bits() == POISON[gd.esz]).any()), f'{what}: an output was not written'
        if part is not None:
            assert part.outside_intact(), f'{what}: write outside partial'
            used = n * splits4 * 4 if splits4 > 1 else 0
            pb = part.region_bits()[:, 0]
            assert not bool((pb[:used] == POISON[4]).any()), f'{what}: partial not written'
            assert bool((pb[used:] == POISON[4]).all()), f'{what}: partial written past n * splits * 4'
        assert status == plain[5], f'{what}: status {status:#x}, plain launch {plain[5]:#x}'
        assert bool(status & Lb.STATUS_LABEL_OOB) == (not bool(lab_ok.all())), f'{what}: status {status:#x}'
        xr = x64.float().bfloat16().double() if mode == Lb.MODE_FAITHFUL else x64
        h64 = entropy64(xr)
        h = ent.vec
        worst = max(worst, check_entropy(h, h64, what))
        if not bool(lab_ok.all()):
            assert bool(torch.isfinite(h[~lab_ok]).all()), f'{what}: out-of-range label rows keep their entropy'
        others = x64.clone()
        others[torch.arange(n, device=DEV), y] = -math.inf
        sat = ((x64.gather(1, y[:, None])[:, 0] - others.max(dim=1).values) > 40) & lab_ok
        planted = [r for r in sat_rows if bool(lab_ok[r])]
        if planted and H >= 128:
            assert bool(sat[planted].all()), f'{what}: the planted rows must saturate'
        assert bool((h[sat] <= 1e-6).all()), f'{what}: a saturated row has H > 1e-6'
        same = all(torch.equal(a.region_bits(), b.region_bits()) for a, b in zip(plain[:3], (out, smax, slog)))
        if splits3 == splits4:
            assert same, f'{what}: out / stat_max / stat_logsum differ from aa_linear_logprob_fwd'
            continue
        print(f'SPLITS {what}: plain {splits3} splits, entropy {splits4}; bit-identical: {same}')
        for o, m, ls in (plain[:3], (out, smax, slog)):
            m_ref = xr.max(dim=1).values
            assert torch.equal(m.vec.double(), m_ref), f'{what}: stat_max'
            ls_ref = torch.logsumexp(xr - m_ref[:, None], dim=1)
            assert bool(((ls.vec.double() - ls_ref).abs() <= 2e-5 * ls_ref.abs().clamp(min=1.0)).all()), \
                f'{what}: stat_logsum'
            lp = o.vec
            assert torch.equal(torch.isnan(lp), ~lab_ok), f'{what}: NaN pattern of the log-probs'
            if mode == Lb.MODE_F32:
                ref = x64.gather(1, y[:, None])[:, 0] - m_ref - ls_ref
                e = (lp.double() - ref).abs()[lab_ok]
                assert bool((e <= 2e-5 * ref.abs().clamp(min=1.0)[lab_ok]).all()), f'{what}: f32 log-probs'
            else:
                xl = x64.gather(1, y[:, None])[:, 0].float().bfloat16().float()
                want = ((xl - m.vec) - ls.vec).bfloat16()
                assert torch.equal(lp[lab_ok].view(torch.int16), want[lab_ok].view(torch.int16)), \
                    f'{what}: faithful log-probs'
    _headroom(f'K6 {cid} entropy (err / bar)', worst, 1.0)


# ---- K6b -------------------------------------------------------------------------------------------------------------
def _grad_entropy(n, dtype, seed):
    """g_H per row, exact in bf16 and fp16: zeros on every seventh row (3, 10, ...), nonzero on row 1 (where the
    upstream g is 0: the row carries the entropy's gradient alone) and one NaN."""
    gen = torch.Generator().manual_seed(seed)
    gh = (torch.randn(n, generator=gen) * 2).bfloat16().float()
    gh = torch.where(gh.abs() < 2 ** -8, torch.full_like(gh, -1.5), gh)
    gh[3::7] = 0.0
    if n > 1:
        gh[1] = 0.625
    if n > 4:
        r = n // 2 + 1
        r = r + 1 if r % 7 == 3 else r
        gh[r] = float('nan')
    return gh.to(dtype).to(DEV)


def _k6b(hidden, weight, labels, smax, slog, g, ld, mode, n, V, H, ent=None, gh=None, row0=0, rows=None):
    """aa_linear_dlogits (ent None) or aa_linear_dlogits_entropy on rows [row0, row0 + rows) into a fresh guarded
    (n, roundup256(V)) region of pitch ld; the per-row vectors are offset by row0."""
    rows = n - row0 if rows is None else rows
    buf = GuardedLM(n, _up(V, BN), ld, BF, tail_rows=_up(n, BM) - n + BM)
    head = (hidden[row0].data_ptr(), rows, H, hidden.stride(0), weight.data_ptr(), V, weight.stride(0),
            labels[row0:].data_ptr(), smax[row0:].data_ptr(), slog[row0:].data_ptr(), g[row0:].data_ptr(),
            Lb.dtype_code(g.dtype))
    if ent is None:
        Lb.check(Lb.lib().aa_linear_dlogits(*head, buf.ptr(row0), ld, mode, _stream()))
    else:
        Lb.check(Lb.lib().aa_linear_dlogits_entropy(*head, ent[row0:].data_ptr(), gh[row0:].data_ptr(),
                                                    Lb.dtype_code(gh.dtype), buf.ptr(row0), ld, mode, _stream()))
    torch.cuda.synchronize()
    return buf


# the faithful share of bit-identical elements, measured on an H100 80GB HBM3: 99.986 % at the least (129 x 320 x 777),
# 100 % at V = 1 and V = 257
FAITHFUL_EXACT_FLOOR = 0.999

K6B_PARAMS = [(c, d) for c in DLOGITS_CASES for d in (BF, F16, F32)]
K6B_IDS = [f'K6b-{_dlogits_case_id(c)}-gH{str(d)[6:]}' for c, d in K6B_PARAMS]


@pytest.mark.parametrize('case,gh_dtype', K6B_PARAMS, ids=K6B_IDS)
def test_k6b_entropy_epilogue(ops, case, gh_dtype):
    """aa_linear_dlogits_entropy on one lm_head pin case, both modes, fed the case's own K6 entropy launch (stat_max,
    stat_logsum and H), with g_H in one dtype (zeros on every seventh row, g = 0 with g_H != 0, one NaN):
      * rows with g_H == 0 bit-identical to aa_linear_dlogits on the same layout; pad columns [V, roundup256(V))
        +0.0; columns up to ld, rows past n and the guards unchanged;
      * F32 mode: within 2e-5 * max(|g|, |g_H| p (|l| + H), |ref|) + half a bf16 ulp of float64
        g (onehot - p) - g_H p (l + H).  The entropy term is scaled by |l| + H rather than |l + H|: l + H cancels
        where l ~ -H, and the fp32 l = (x - m) - logsum and K6's fp32 H each carry an error relative to their own
        size, not to their sum;
      * FAITHFUL mode: the epilogue restated in torch fp32 from the saved statistics (test_k6b_dlogits_elementwise's
        restatement plus fma(p (max(ls, -3e38) + H), -g_H, d) on rows with g_H != 0, the fused multiply-add taken in
        float64 with one rounding to fp32, as the kernel rounds it: a restatement that rounds the product first is up
        to 3 bf16 ulp off where d and the entropy term cancel); every element within 1 bf16 ulp (ex2.approx may move a
        value across a rounding boundary), the share of bit-identical elements >= FAITHFUL_EXACT_FLOOR and printed;
      * row-locality: the (128, n - 128) and (0, 128) row-chunk launches, with entropy and grad_entropy offset by
        row0, give byte-identical rows."""
    n, H, V, ld_extra, gdt = case
    ld = _up(V, BN) + ld_extra
    cid = K6B_IDS[K6B_PARAMS.index((case, gh_dtype))]
    labels = _plant_labels(n, V, 1, 1, n + V + 1, oob=False).to(DEV)
    hidden, weight = _fwd_operands(n, H, V)
    hidden, weight = poisoned_operand(hidden, H + 16), poisoned_operand(weight, H + 8)
    g = _upstream(n, gdt, n + H)
    gh = _grad_entropy(n, gh_dtype, n + V)
    x64 = hidden.double() @ weight.double().T
    onehot = torch.zeros_like(x64)
    onehot[torch.arange(n, device=DEV), labels] = 1.0
    g64, gh64 = g.double(), gh.double()
    cold = (gh == 0).nonzero().flatten()
    S = torch.cuda.get_device_properties(0).multi_processor_count
    worst = 0.0
    for mode in (Lb.MODE_FAITHFUL, Lb.MODE_F32):
        what = f'{cid} mode {mode}'
        _, smax, slog, _, ent, _ = _k6(hidden, weight, labels, mode, n * S * 4, n, V, H, True)
        m, ls, h = smax.vec, slog.vec, ent.vec
        plain = _k6b(hidden, weight, labels, m, ls, g, ld, mode, n, V, H)
        buf = _k6b(hidden, weight, labels, m, ls, g, ld, mode, n, V, H, h, gh)
        assert buf.outside_intact(), f'{what}: write outside the (n, roundup256(V)) region (rows >= n, pad or guards)'
        assert bool((buf.region_bits()[:, V:] == 0).all()), f'{what}: pad columns [V, roundup256(V)) must be +0.0'
        assert torch.equal(buf.region_bits()[cold], plain.region_bits()[cold]), \
            f'{what}: a row with g_H == 0 differs from aa_linear_dlogits'
        got = buf.t[:, :V]
        if mode == Lb.MODE_F32:
            lse = torch.logsumexp(x64, dim=1, keepdim=True)
            l64 = x64 - lse
            p = torch.exp(l64)
            h64 = entropy64(x64)[:, None]
            ref = g64[:, None] * (onehot - p) - gh64[:, None] * p * (l64 + h64)
            assert torch.equal(torch.isnan(got), torch.isnan(ref)), f'{what}: NaN pattern'
            r = torch.nan_to_num(ref)
            scale = torch.maximum(torch.nan_to_num(g64).abs()[:, None],
                                  torch.nan_to_num(gh64).abs()[:, None] * p * (l64.abs() + h64))
            tol = 2e-5 * torch.maximum(scale, r.abs()) + _half_ulp_bf16(r)
            err = (torch.nan_to_num(got.double()) - r).abs()
            assert bool((err <= tol).all()), f'{what}: max err {float(err.max()):.3e}, {int((err > tol).sum())} beyond'
            worst = max(worst, float((err / tol).max()))
        else:
            xs = x64.float().bfloat16().float()
            lsr = ((xs - m[:, None]) - ls[:, None]).bfloat16().float()
            pe = torch.exp(lsr)
            d = -(pe * g.float()[:, None])
            lab_d = d.gather(1, labels[:, None])[:, 0] + g.float()
            d[torch.arange(n, device=DEV), labels] = lab_d
            ngh = -gh.float()[:, None]
            # fma(p (max(ls, -3e38) + H), -g_H, d): the float64 product of two fp32 values is exact, one rounding
            t2 = (pe * (lsr.clamp(min=-3.0e38) + h[:, None])).double() * ngh.double()
            c = (t2 + d.double()).float()
            want = torch.where(ngh != 0, c, d).bfloat16()
            assert torch.equal(torch.isnan(got), torch.isnan(want)), f'{what}: NaN pattern'
            diff = (_ordered(torch.nan_to_num(got)) - _ordered(torch.nan_to_num(want))).abs()
            exact = float((diff == 0).double().mean())
            assert int(diff.max()) <= 1, f'{what}: max {int(diff.max())} bf16 ulp'
            print(f'HEADROOM {cid} faithful: bit-identical share {exact:.6f}')
            assert exact >= FAITHFUL_EXACT_FLOOR, f'{what}: only {exact:.5f} bit-identical'
        if n > BM:
            for row0, rows in ((BM, n - BM), (0, BM)):
                part = _k6b(hidden, weight, labels, m, ls, g, ld, mode, n, V, H, h, gh, row0, rows)
                rb = part.region_bits()[row0:row0 + rows]
                assert torch.equal(rb, buf.region_bits()[row0:row0 + rows]), f'{what}: rows {row0}+{rows} differ'
                assert bool((part.region_bits()[:row0] == POISON[2]).all()), f'{what}: rows before {row0} written'
                assert bool((part.region_bits()[row0 + rows:] == POISON[2]).all()), f'{what}: rows past the launch'
                assert part.outside_intact()
    _headroom(f'{cid} f32 (err / bar)', worst, 1.0)
