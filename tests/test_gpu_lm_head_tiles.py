"""The lm_head tensor-core kernels pinned element by element (run on an H100: `pytest -m gpu`).

The four wgmma kernels of the fused lm_head path -- K6 `aa_linear_logprob_fwd`, K6b `aa_linear_dlogits`,
`aa_linear_dhidden` and `aa_linear_dweight` -- are called through the C ABI, so every stride, `ld`, `partial` buffer
and row-chunk cut is the test's choice.

Exact arithmetic.  Most operands come from `exact_operand`: small signed integers times a power of two, a share of
them zero.  For a GEMM over K terms with |a| <= qa * 2^ea and |b| <= qb * 2^eb every product is a multiple of
g = 2^(ea + eb), and the closed-form precondition K * qa * qb <= 2^20 keeps every partial sum an integer multiple of g
below 2^20 * g: exact in fp32 (24-bit significand, 3 bits to spare) in ANY summation order and under the tensor core's
truncating adds.  So the GEMM equals the float64 product exactly, its bf16 rounding equals `ref64.float().bfloat16()`
bit for bit, and logits and statistics can be held to float64 with no summation-order slack.  The one CPU test here
checks that premise for every operand of the matrix.

Guarded buffers.  Every output lives in the middle of one larger allocation, between guard bands of at least one row
and 256 bytes (plus the rest of the last 128-row tile after it, so a stray store of a whole tile row stays inside the
test's memory).  Outputs start as a NaN bit pattern, guards and pad columns as a finite sentinel: a skipped write
leaves a NaN, a stray write changes a sentinel.  Input operands sit between NaN rows (and NaN pad columns when their
row stride exceeds H), so a tensor map that reaches one row past its operand turns results into NaN instead of
reading TMA's silent zeros.
"""
import math

import pytest
import torch

from align_anything_b200 import _lib as Lb
from test_gpu_parity import ops  # noqa: F401

DEV = 'cuda'
gpu = pytest.mark.gpu
BF, F16, F32 = torch.bfloat16, torch.float16, torch.float32
# bit patterns: POISON is a NaN in bf16 (0x7FA5) and fp32 (0x7FA5A5A5); SENTINEL is a finite value
POISON = {2: 0x7FA5, 4: 0x7FA5A5A5}
SENTINEL = {2: 0x3C5A, 4: 0x3C5A5A5A}
INT = {2: torch.int16, 4: torch.int32}
BM, BN = 128, 256  # wgmma tile of every kernel: 128 rows x 256 columns
EXACT_LIMIT = 2 ** 20


def _up(x, m):
    return (x + m - 1) // m * m


# ---- exact-arithmetic operands ---------------------------------------------------------------------------------------
def exact_bound_ok(K, qa, qb):
    """The closed-form precondition: K * max|a| * max|b| <= 2^20 * g (in units of the grid step g)."""
    return K * qa * qb <= EXACT_LIMIT


def exact_q(K, q_other, cap=7):
    """The largest integer range |a| <= q (at most `cap`) that keeps a K-term GEMM against |b| <= q_other exact."""
    q = min(cap, EXACT_LIMIT // (K * q_other))
    assert q >= 1, f'K = {K} with |b| <= {q_other} cannot be made exact'
    return q


def logit_exponent(H, q=7):
    """Exponent e of the weight so that hidden (q * 2^-3) . weight (q * 2^e) logits spread over a few units: an entry is
    uniform in [-q, q] and zero a quarter of the time more, variance 0.75 * q (q + 1) / 3 per factor."""
    var = 0.75 * q * (q + 1) / 3
    return round(math.log2(2.0 / (var * math.sqrt(H)))) + 3


def exact_operand(rows, K, q, e, seed, device=DEV):
    """(rows, K) bf16: integers in [-q, q] times 2^e, about a quarter of them (plus the draws of 0) zero."""
    gen = torch.Generator(device=device).manual_seed(seed)
    v = torch.randint(-q, q + 1, (rows, K), generator=gen, device=device, dtype=torch.int8)
    v *= (torch.randint(0, 4, (rows, K), generator=gen, device=device, dtype=torch.int8) != 0).to(torch.int8)
    return v.to(BF) * (2.0 ** e)


# ---- guarded buffers and poisoned operands ---------------------------------------------------------------------------
class Guarded:
    """A (rows, cols) region with row pitch `pitch` inside one allocation.  The guard before it holds at least one row
    and 256 bytes; the guard after it that plus `tail_rows` more rows.  Both keep the region 16-byte aligned.  Region
    elements start as POISON, everything else (guards, pad columns [cols, pitch)) as SENTINEL."""

    def __init__(self, rows, cols, pitch, dtype, tail_rows=0):
        esz = torch.empty(0, dtype=dtype).element_size()
        q = 16 // esz
        self.pre = _up(max(pitch, 256 // esz), q)
        post = _up(pitch * (tail_rows + 1) + 256 // esz, q)
        self.rows, self.cols, self.pitch, self.esz = rows, cols, pitch, esz
        self.buf = torch.empty(self.pre + rows * pitch + post, dtype=dtype, device=DEV)
        self.bits = self.buf.view(INT[esz])
        self.bits.fill_(SENTINEL[esz])
        self._bits_region().fill_(POISON[esz])
        self.fresh = self.bits.clone()
        self.t = self.buf.as_strided((rows, cols), (pitch, 1), self.pre)

    def _bits_region(self):
        return self.bits.as_strided((self.rows, self.cols), (self.pitch, 1), self.pre)

    @property
    def vec(self):
        assert self.cols == 1
        return self.t[:, 0]

    def ptr(self, row=0):
        return self.t.data_ptr() + row * self.pitch * self.esz

    def region_bits(self):
        return self._bits_region()

    def outside_intact(self):
        m = torch.ones(self.buf.numel(), dtype=torch.bool, device=DEV)
        m.as_strided((self.rows, self.cols), (self.pitch, 1), self.pre).fill_(False)
        return torch.equal(self.bits[m], self.fresh[m])

    def untouched(self):
        return torch.equal(self.bits, self.fresh)


def vec_guard(n, dtype):
    return Guarded(n, 1, 1, dtype)


def poisoned_operand(values, stride, pad=float('nan')):
    """`values` (rows, K) placed between NaN rows (at least 256 bytes on each side) in an allocation of row stride
    `stride` >= K; the pad columns [K, stride) hold `pad`.  Returns the (rows, K) view, 16-byte aligned."""
    rows, K = values.shape
    extra = max(2, -(-256 // (stride * values.element_size())))
    buf = torch.full((rows + 2 * extra, stride), float('nan'), dtype=values.dtype, device=DEV)
    buf[extra:extra + rows, :K] = values
    if stride > K:
        buf[extra:extra + rows, K:] = pad
    v = buf[extra:extra + rows, :K]
    assert v.data_ptr() % 16 == 0
    return v


def _status_take():
    from align_anything_b200 import ops as _ops

    st = _ops._device_scratch(torch.device(DEV))['status']
    v = int(st.item())
    st.zero_()
    return v


def _stream():
    return Lb.stream_ptr(torch.device(DEV))


def _half_ulp_bf16(a64):
    """Half a bf16 ulp at |a| (float64)."""
    fi = torch.finfo(BF)
    a = a64.abs().clamp(min=fi.tiny)
    return torch.exp2(torch.floor(torch.log2(a))) * fi.eps / 2 + fi.tiny * fi.eps / 2


def _canon(t):
    """bf16 bits with -0 mapped to +0 (a tensor-core sum of signed zero products may carry either sign)."""
    return (t.float() + 0.0).bfloat16().view(torch.int16)


def _headroom(what, err, tol):
    print(f'HEADROOM {what}: max err {err:.3e}, bar {tol:.3e}')


def schedule(n, V, may_split, partial_floats, per_split=3, sms=None):
    """The host schedule of linear_logprob.cu restated: -> (splits, tiles per split, row units per group).
    per_split: floats of `partial` per (row, split) -- 3 for K6, 4 for its entropy variant; sms: the SM count (default:
    the device's)."""
    S = sms or torch.cuda.get_device_properties(0).multi_processor_count
    units = -(-n // BM)
    all_tiles = -(-V // BN)
    splits, group = 1, units
    if may_split:
        if units < S // 8:
            splits = S // units
        else:
            best, best_cost = 12, None
            for s in range(6, 17):
                tps = -(-all_tiles // s)
                live = units * (-(-all_tiles // tps))
                cost = (-(-live // S)) * tps * 64 + abs(s - 12)
                if best_cost is None or cost < best_cost:
                    best, best_cost = s, cost
            splits, group = best, S // best
        splits = max(1, min(splits, all_tiles))
        while partial_floats >= 0 and splits > 1 and n * splits * per_split > partial_floats:
            splits -= 1
        group = max(1, min(group, units))
    tps = -(-all_tiles // splits)
    return -(-all_tiles // tps), tps, group


# ---- the matrix ------------------------------------------------------------------------------------------------------
# K6 / K6b: (n, H, V, partial, note).  partial: 'none' (NULL: no split), 'wide' (room for every split the schedule
# wants), 'two' (exactly n * 2 * 3 floats: the schedule must cut its split count to 2)
FWD_CASES = [
    (1, 64, 1, 'wide', 'V = 1, one k-block'),
    (63, 192, 257, 'wide', 'split 1 is the partial last tile only, 3 k-blocks < 4 stages'),
    (129, 320, 777, 'none', 'no split, V tail of 9 columns'),
    (200, 64, 513, 'wide', 'split 2 is the partial last tile only, one k-block'),
    (129, 320, 777, 'two', 'partial_floats just large enough for 2 splits'),
    (300, 4096, 32064, 'wide', 'units < S / 8: the vocabulary spread over the idle SMs'),
    (300, 4096, 32064, 'none', 'no split at H = 4096'),
    (2100, 256, 32064, 'wide', 'grouped schedule: >= 16 row tiles, 6..16 splits'),
    (260, 4096, 128257, 'wide', 'full vocabulary, splits end inside the last tile'),
    (1000, 128, 5000, 'two', '16 splits cut to 2 by partial_floats'),
]
# K6b: (n, H, V, ld - roundup256(V), upstream gradient dtype)
DLOGITS_CASES = [
    (1, 64, 1, 64, BF),
    (63, 192, 257, 0, F16),
    (129, 320, 777, 64, F32),
    (200, 64, 513, 0, BF),
    (300, 4096, 32064, 64, BF),
    (2100, 256, 32064, 0, F16),
    (260, 4096, 128257, 0, F32),
]
# backward GEMMs: (n, H, V, ld kind, strided, chunk cuts of d(weight))
GEMM_CASES = [
    (1, 64, 1, 'r256', True, [0, 1]),
    (63, 192, 257, 'r64', True, [0, 1, 38, 63]),
    (129, 320, 777, 'r256+64', True, [0, 1, 70, 129]),
    (129, 320, 777, 'r256', False, [0, 65, 129]),
    (300, 4096, 32064, 'r256+64', True, [0, 1, 101, 300]),
    (260, 4096, 128257, 'r64', True, [0, 131, 260]),
]
SEED = 1234


def _ld(V, kind):
    return {'r64': _up(V, 64), 'r256': _up(V, 256), 'r256+64': _up(V, 256) + 64}[kind]


def _fwd_operands(n, H, V, device=DEV):
    """hidden (n, H) and weight (V, H): exact operands with logits that spread over a few units."""
    ew = logit_exponent(H)
    hidden = exact_operand(n, H, 7, -3, SEED + n + H, device)
    weight = exact_operand(V, H, 7, ew, SEED + V + 7 * H, device)
    return hidden, weight


def _gemm_operands(n, H, V, ld, device=DEV):
    """hidden, weight as for K6, and a d(logits) (n, V) whose range keeps both backward GEMMs exact."""
    hidden, weight = _fwd_operands(n, H, V, device)
    qd = min(exact_q(ld, 7), exact_q(n, 7))
    d = exact_operand(n, V, qd, -4, SEED + 3 * n + V, device)
    return hidden, weight, d, qd


def exact_specs():
    """Every exact operand pair of the matrix: (what, rows of a, K, (qa, ea), (qb, eb), seed, rows of b)."""
    specs = []
    for n, H, V, *_ in FWD_CASES + DLOGITS_CASES:
        specs.append((f'K6 {n}x{H}x{V}', n, H, (7, -3), (7, logit_exponent(H)), V))
    for n, H, V, kind, *_ in GEMM_CASES:
        ld = _ld(V, kind)
        qd = min(exact_q(ld, 7), exact_q(n, 7))
        specs.append((f'dhidden {n}x{H}x{V} ld {ld}', n, ld, (qd, -4), (7, logit_exponent(H)), H))
        specs.append((f'dweight {n}x{H}x{V}', V, n, (qd, -4), (7, -3), H))
    return specs


def test_exact_operand_premise():
    """No GPU: for every operand pair of the matrix the generator's values are exact in bf16, lie on their grid, hold
    the precondition K * max|a| * max|b| <= 2^20 * g, and small fp32 GEMMs summed in forward and in reversed k order
    (sequential fp32 adds) agree bit for bit with float64.  Rows are capped at 256 (the properties are per entry; K,
    which the bound depends on, is kept)."""
    for what, ra, K, (qa, ea), (qb, eb), rb in exact_specs():
        assert exact_bound_ok(K, qa, qb), what
        a = exact_operand(min(ra, 256), K, qa, ea, SEED + ra, 'cpu')
        b = exact_operand(min(rb, 256), K, qb, eb, SEED + rb + 1, 'cpu')
        for t, q, e in ((a, qa, ea), (b, qb, eb)):
            ints = t.double() * 2.0 ** -e
            assert torch.equal(ints, ints.round()) and float(ints.abs().max()) <= q, what
            assert torch.equal(t.float().bfloat16(), t), what
            if t.numel() >= 1000:
                assert 0.15 < float((t == 0).double().mean()) < 0.6, what
        m = 8 if K > 8192 else 16
        a64, b64 = a[:m].double(), b[:m].double()
        ref = a64 @ b64.T
        prod = (a[:m].float()[:, None, :] * b[:m].float()[None, :, :])  # exact: 8-bit x 8-bit significands
        fwd = prod.cumsum(-1)[..., -1]
        rev = prod.flip(-1).cumsum(-1)[..., -1]
        assert torch.equal(fwd.double(), ref) and torch.equal(rev.double(), ref), what
        assert torch.equal((a[:m].float() @ b[:m].float().T).double(), ref), what
        g = 2.0 ** (ea + eb)
        assert float(ref.abs().max()) <= EXACT_LIMIT * g, what


# ---- K6 ----------------------------------------------------------------------------------------------------------------
def _plant_labels(n, V, splits, tps, seed, oob=True):
    """Labels: columns 0 and V - 1, the partial last tile, the first and last column of every split, -1 and V (once
    each) and random columns elsewhere."""
    gen = torch.Generator().manual_seed(seed)
    lab = torch.randint(0, V, (n,), generator=gen)
    special = [0, V - 1, (V - 1) // BN * BN]
    for s in range(splits):
        special += [min(s * tps * BN, V - 1), min((s + 1) * tps * BN - 1, V - 1)]
    if oob:
        special += [-1, V]
    for i, c in enumerate(special[:n]):
        lab[(i * 7) % n if n > len(special) else i] = c
    return lab


def _plant_saturated(hidden, weight, labels, rows, H):
    """Rows whose label logit leads every other logit by a wide margin: the label's weight row is +-7 everywhere and
    the hidden row its sign pattern times 7 (still exact: the same integer ranges)."""
    ew = logit_exponent(H)
    for r in rows:
        y = int(labels[r])
        if not 0 <= y < weight.size(0):
            continue
        gen = torch.Generator().manual_seed(1000 + r)
        sgn = (torch.randint(0, 2, (H,), generator=gen) * 2 - 1).to(DEV)
        weight[y] = (7 * sgn).to(BF) * 2.0 ** ew
        hidden[r] = (7 * sgn).to(BF) * 2.0 ** -3


def _run_k6(hidden, weight, labels, mode, partial_kind, n, V, H):
    """One K6 launch into guarded buffers -> (out guard, max guard, logsum guard, partial guard or None, status)."""
    out = vec_guard(n, BF if mode == Lb.MODE_FAITHFUL else F32)
    smax, slog = vec_guard(n, F32), vec_guard(n, F32)
    pf = _partial_floats(partial_kind, n)
    part = vec_guard(pf, F32) if pf else None
    _status_take()
    Lb.check(Lb.lib().aa_linear_logprob_fwd(
        hidden.data_ptr(), n, H, hidden.stride(0), weight.data_ptr(), V, weight.stride(0), labels.data_ptr(),
        out.ptr(), Lb.dtype_code(out.t.dtype), smax.ptr(), slog.ptr(), part.ptr() if part else None, pf, mode,
        _device_status_ptr(), _stream()))
    torch.cuda.synchronize()
    return out, smax, slog, part, pf, _status_take()


def _partial_floats(kind, n):
    """'none': no partial buffer; 'wide': room for every split the schedule can pick; 'two': exactly 2 splits' worth."""
    S = torch.cuda.get_device_properties(0).multi_processor_count
    return {'none': 0, 'wide': n * S * 3, 'two': n * 2 * 3}[kind]


def _device_status_ptr():
    from align_anything_b200 import ops as _ops

    return _ops._device_scratch(torch.device(DEV))['status'].data_ptr()


def _fwd_case_id(c):
    return f'{c[0]}x{c[1]}x{c[2]}-{c[3]}'


@gpu
@pytest.mark.parametrize('case', FWD_CASES, ids=[_fwd_case_id(c) for c in FWD_CASES])
def test_k6_forward_exact(ops, case):
    """K6 on exact operands, both modes: stat_max bit-exact (the largest logit, faithful: the largest bf16-rounded
    logit), stat_logsum and f32 log-probs within 2e-5 * max(1, |ref|) of float64, faithful log-probs bit-identical to
    bf16((x_label_bf16 - m) - logsum) from the kernel's own stats, saturated rows exactly 0, out-of-range labels NaN in
    their row only with the status bit set, and nothing written outside the outputs (and the used part of
    `partial`)."""
    n, H, V, partial_kind, _ = case
    splits, tps, group = schedule(n, V, partial_kind != 'none', _partial_floats(partial_kind, n))
    S = torch.cuda.get_device_properties(0).multi_processor_count
    if partial_kind == 'two':
        assert splits == 2 and schedule(n, V, True, -1)[0] > 2, 'partial_floats must cut the split count to 2'
    if n >= 16 * BM and partial_kind == 'wide':
        assert 6 <= splits <= 16 and -(-n // BM) >= S // 8, 'grouped schedule'
    oob = n != 129  # the 129-row cases have in-range labels only: the status bit must stay clear
    labels = _plant_labels(n, V, splits, tps, n + V, oob=oob)
    hidden, weight = _fwd_operands(n, H, V)
    sat_rows = [r for r in (n // 2, n - 1) if n > 8]
    _plant_saturated(hidden, weight, labels, sat_rows, H)
    hs, ws = (H, H) if n % 2 else (H + 8, H + 64)  # odd n: contiguous; even n: row strides above H
    hidden, weight = poisoned_operand(hidden, hs), poisoned_operand(weight, ws)
    labels = labels.to(DEV)
    x64 = hidden.double() @ weight.double().T
    lab_ok = (labels >= 0) & (labels < V)
    y = torch.where(lab_ok, labels, torch.zeros_like(labels))
    worst = {}
    for mode in (Lb.MODE_FAITHFUL, Lb.MODE_F32):
        what = f'{_fwd_case_id(case)} mode {mode}'
        out, smax, slog, part, pf, status = _run_k6(hidden, weight, labels, mode, partial_kind, n, V, H)
        for gd in (out, smax, slog):
            assert gd.outside_intact(), f'{what}: write outside an output'
            assert not bool((gd.region_bits() == POISON[gd.esz]).any()), f'{what}: an output was not written'
        if part is not None:
            assert part.outside_intact(), f'{what}: write outside partial'
            used = n * splits * 3 if splits > 1 else 0
            pb = part.region_bits()[:, 0]
            assert not bool((pb[:used] == POISON[4]).any()), f'{what}: partial not written'
            assert bool((pb[used:] == POISON[4]).all()), f'{what}: partial written past n * splits * 3'
        assert bool(status & Lb.STATUS_LABEL_OOB) == (not bool(lab_ok.all())), f'{what}: status {status:#x}'
        xr = x64.float().bfloat16().double() if mode == Lb.MODE_FAITHFUL else x64
        m_ref = xr.max(dim=1).values
        assert torch.equal(smax.vec.double(), m_ref), f'{what}: stat_max'
        ls_ref = torch.logsumexp(xr - m_ref[:, None], dim=1)
        err = (slog.vec.double() - ls_ref).abs()
        tol = 2e-5 * ls_ref.abs().clamp(min=1.0)
        assert bool((err <= tol).all()), f'{what}: stat_logsum max err {float(err.max()):.3e}'
        worst[f'stat_logsum mode {mode}'] = float((err / tol).max())
        lp = out.vec
        assert torch.equal(torch.isnan(lp), ~lab_ok), f'{what}: NaN pattern of the log-probs'
        if mode == Lb.MODE_F32:
            ref = x64.gather(1, y[:, None])[:, 0] - m_ref - ls_ref
            e = (lp.double() - ref).abs()[lab_ok]
            t = 2e-5 * ref.abs().clamp(min=1.0)[lab_ok]
            assert bool((e <= t).all()), f'{what}: f32 log-probs max err {float(e.max()):.3e}'
            worst['f32 log-probs'] = float((e / t).max())
        else:
            xl = x64.gather(1, y[:, None])[:, 0].float().bfloat16().float()
            want = ((xl - smax.vec) - slog.vec).bfloat16()
            assert torch.equal(lp[lab_ok].view(torch.int16), want[lab_ok].view(torch.int16)), f'{what}: faithful log-probs'
        if V == 1:
            assert bool((lp[lab_ok] == 0).all()), f'{what}: V = 1 must give log p = 0'
        others = x64.clone()
        others[torch.arange(n, device=DEV), y] = -math.inf
        lead = x64.gather(1, y[:, None])[:, 0] - others.max(dim=1).values
        sat = (lead > 40) & lab_ok
        planted = [r for r in sat_rows if bool(lab_ok[r])]
        if planted and H >= 128:
            assert bool(sat[planted].all()), f'{what}: the planted rows must saturate'
        assert bool((lp[sat] == 0).all()), f'{what}: a saturated row must give exactly 0.0'
    for k, v in worst.items():
        _headroom(f'K6 {_fwd_case_id(case)} {k} (err / bar)', v, 1.0)


@gpu
@pytest.mark.parametrize('shape', [(300, 256, 777), (130, 4096, 128257)])
def test_k6_forward_random_vs_float64(ops, shape):
    """Real-valued operands (not exact): f32 log-probs and max + logsum within 2e-5 * max(1, |ref|) of float64."""
    n, H, V = shape
    gen = torch.Generator(device=DEV).manual_seed(n + V)
    hidden = poisoned_operand(torch.randn((n, H), generator=gen, device=DEV).bfloat16(), H + 8)
    weight = poisoned_operand((torch.randn((V, H), generator=gen, device=DEV) * (2.5 / H ** 0.5)).bfloat16(), H)
    labels = torch.randint(0, V, (n,), generator=gen, device=DEV)
    out, smax, slog, part, _, status = _run_k6(hidden, weight, labels, Lb.MODE_F32, 'wide', n, V, H)
    assert status == 0 and out.outside_intact() and smax.outside_intact() and part.outside_intact()
    x64 = hidden.double() @ weight.double().T
    lse = torch.logsumexp(x64, dim=1)
    ref = x64.gather(1, labels[:, None])[:, 0] - lse
    for what, got, want in (('log-probs', out.vec, ref), ('max + logsum', smax.vec + slog.vec, lse)):
        err = (got.double() - want).abs()
        tol = 2e-5 * want.abs().clamp(min=1.0)
        assert bool((err <= tol).all()), f'{shape} {what}: max err {float(err.max()):.3e}'
        _headroom(f'K6 random {shape} {what} (err / bar)', float((err / tol).max()), 1.0)


# ---- K6b ---------------------------------------------------------------------------------------------------------------
def _upstream(n, dtype, seed):
    """Upstream gradient per row: exact in bf16 and f16, negative values, zeros and NaNs."""
    gen = torch.Generator().manual_seed(seed)
    g = (torch.randn(n, generator=gen) * 2).bfloat16().float()
    g = torch.where(g.abs() < 2 ** -8, torch.full_like(g, 0.75), g)
    g[:: 5] = -g[:: 5].abs()
    if n > 2:
        g[1] = 0.0
        g[n - 2] = float('nan')
    return g.to(dtype).to(DEV)


def _run_k6b(hidden, weight, labels, smax, slog, g, ld, mode, n, V, H, row0=0, rows=None):
    """K6b on rows [row0, row0 + rows) into a fresh guarded (n, roundup256(V)) region of pitch ld."""
    rows = n - row0 if rows is None else rows
    Vp = _up(V, BN)
    buf = Guarded(n, Vp, ld, BF, tail_rows=_up(n, BM) - n + BM)
    Lb.check(Lb.lib().aa_linear_dlogits(
        hidden[row0].data_ptr(), rows, H, hidden.stride(0), weight.data_ptr(), V, weight.stride(0),
        labels[row0:].data_ptr(), smax[row0:].data_ptr(), slog[row0:].data_ptr(), g[row0:].data_ptr(),
        Lb.dtype_code(g.dtype), buf.ptr(row0), ld, mode, _stream()))
    torch.cuda.synchronize()
    return buf


def _dlogits_case_id(c):
    return f'{c[0]}x{c[1]}x{c[2]}-ld+{c[3]}-g{str(c[4])[6:]}'


@gpu
@pytest.mark.parametrize('case', DLOGITS_CASES, ids=[_dlogits_case_id(c) for c in DLOGITS_CASES])
def test_k6b_dlogits_elementwise(ops, case):
    """K6b element by element, both modes, on exact operands and the stats K6 saved:
      * f32 mode: |err| <= 2e-5 * max(|g|, |ref|) + half a bf16 ulp of float64 g * (onehot - exp(x - lse));
      * faithful mode: the epilogue restated in torch fp32 from the saved stats (xs = bf16(x), ls = bf16((xs - m) -
        logsum), p = exp(ls), bf16(-p * g), on the label column bf16(fp32(-p * g) + g)); every element within 1 bf16
        ulp (ex2.approx may move a value across a rounding boundary), >= 99.9 % bit-identical (measured on an H100
        80GB HBM3: 99.975 % at the least, in the 63 x 257 case; 100 % at V = 1 and V = 128257);
      * pad columns [V, roundup256(V)) exactly +0.0, also for NaN and zero g; columns [roundup256(V), ld), rows past
        n and the guards unchanged;
      * row-locality: a row's d(logits) is byte-identical whether the launch covers all n rows, the 128-aligned rows
        from 128 on, or the first 128 rows alone (a row count small enough to split the vocabulary)."""
    n, H, V, ld_extra, gdt = case
    ld = _up(V, BN) + ld_extra
    Vp = _up(V, BN)
    labels = _plant_labels(n, V, 1, 1, n + V + 1, oob=False).to(DEV)
    hidden, weight = _fwd_operands(n, H, V)
    hidden, weight = poisoned_operand(hidden, H + 16), poisoned_operand(weight, H + 8)
    g = _upstream(n, gdt, n + H)
    x64 = hidden.double() @ weight.double().T
    onehot = torch.zeros_like(x64)
    onehot[torch.arange(n, device=DEV), labels] = 1.0
    g64 = g.double()
    for mode in (Lb.MODE_FAITHFUL, Lb.MODE_F32):
        what = f'{_dlogits_case_id(case)} mode {mode}'
        out, smax, slog, _, _, _ = _run_k6(hidden, weight, labels, mode, 'wide', n, V, H)
        buf = _run_k6b(hidden, weight, labels, smax.vec, slog.vec, g, ld, mode, n, V, H)
        assert buf.outside_intact(), f'{what}: write outside the (n, roundup256(V)) region (rows >= n, pad or guards)'
        pad = buf.region_bits()[:, V:]
        assert bool((pad == 0).all()), f'{what}: pad columns [V, roundup256(V)) must be +0.0'
        got = buf.t[:, :V]
        if mode == Lb.MODE_F32:
            ref = g64[:, None] * (onehot - torch.exp(x64 - torch.logsumexp(x64, dim=1, keepdim=True)))
            assert torch.equal(torch.isnan(got), torch.isnan(ref)), f'{what}: NaN pattern'
            err = (torch.nan_to_num(got.double()) - torch.nan_to_num(ref)).abs()
            r = torch.nan_to_num(ref)
            tol = 2e-5 * torch.maximum(torch.nan_to_num(g64).abs()[:, None], r.abs()) + _half_ulp_bf16(r)
            assert bool((err <= tol).all()), f'{what}: max err {float(err.max()):.3e}, {int((err > tol).sum())} beyond'
            _headroom(f'K6b f32 {_dlogits_case_id(case)} (err / bar)', float((err / tol).max()), 1.0)
        else:
            xs = x64.float().bfloat16().float()
            ls = ((xs - smax.vec[:, None]) - slog.vec[:, None]).bfloat16().float()
            d = -(torch.exp(ls) * g.float()[:, None])
            want = d.bfloat16()
            lab_d = (d.gather(1, labels[:, None])[:, 0] + g.float()).bfloat16()
            want[torch.arange(n, device=DEV), labels] = lab_d
            assert torch.equal(torch.isnan(got), torch.isnan(want)), f'{what}: NaN pattern'
            gb = _ordered(torch.nan_to_num(got))
            wb = _ordered(torch.nan_to_num(want))
            diff = (gb - wb).abs()
            exact = float((diff == 0).double().mean())
            assert int(diff.max()) <= 1, f'{what}: max {int(diff.max())} bf16 ulp'
            assert exact >= 0.999, f'{what}: only {exact:.5f} bit-identical'
            print(f'HEADROOM K6b faithful {_dlogits_case_id(case)}: bit-identical share {exact:.6f}')
        # row-locality
        if n > BM:
            for row0, rows in ((BM, n - BM), (0, BM)):
                part = _run_k6b(hidden, weight, labels, smax.vec, slog.vec, g, ld, mode, n, V, H, row0, rows)
                rb = part.region_bits()[row0:row0 + rows]
                assert torch.equal(rb, buf.region_bits()[row0:row0 + rows]), f'{what}: rows {row0}+{rows} differ'
                assert bool((part.region_bits()[:row0] == POISON[2]).all()), f'{what}: rows before {row0} written'
                assert bool((part.region_bits()[row0 + rows:] == POISON[2]).all()), f'{what}: rows past the launch written'
                assert part.outside_intact()


def _ordered(t):
    bits = t.contiguous().view(torch.int16).to(torch.int32) & 0xFFFF
    return torch.where(bits >= 0x8000, 0x8000 - bits, bits)


# ---- aa_linear_dhidden / aa_linear_dweight -----------------------------------------------------------------------------
def _strides(H, strided):
    """(hidden, weight, d_hidden, acc, d_weight) row strides: all above H, or all H."""
    return (H + 8, H + 64, H + 24, H + 4, H + 16) if strided else (H,) * 5


def _dhidden(d, n, ld, weight, V, H, dhs):
    out = Guarded(n, H, dhs, BF, tail_rows=_up(n, BM) - n + BM)
    Lb.check(Lb.lib().aa_linear_dhidden(d.data_ptr(), n, ld, weight.data_ptr(), V, H, weight.stride(0), out.ptr(),
                                        dhs, _stream()))
    torch.cuda.synchronize()
    return out


def _dweight(d, hidden, cuts, ld, V, H, accs, dws, on_middle=None):
    """d(weight) over the row chunks `cuts`: first chunk writes acc (or, alone, d_weight directly with acc = NULL),
    later chunks add to it, the last one rounds into d_weight.  on_middle(i, r1, acc, dw) runs after each chunk that
    does not finish."""
    n_chunks = len(cuts) - 1
    tail = _up(V, BM) - V + BM
    dw = Guarded(V, H, dws, BF, tail_rows=tail)
    acc = Guarded(V, H, accs, F32, tail_rows=tail) if n_chunks > 1 else None
    for i in range(n_chunks):
        r0, r1 = cuts[i], cuts[i + 1]
        last = i == n_chunks - 1
        Lb.check(Lb.lib().aa_linear_dweight(
            d[r0].data_ptr(), r1 - r0, ld, hidden[r0].data_ptr(), H, hidden.stride(0), V, acc.ptr() if acc else None,
            accs, 1 if i else 0, dw.ptr() if last else None, dws, _stream()))
        torch.cuda.synchronize()
        if not last and on_middle:
            on_middle(i, r1, acc, dw)
    return dw, acc


def _gemm_case_id(c):
    return f'{c[0]}x{c[1]}x{c[2]}-{c[3]}' + ('-strided' if c[4] else '-contig')


def _bf16_exact(got, ref64, what):
    assert torch.equal(_canon(got), _canon(ref64.float().bfloat16())), \
        f'{what}: {int((_canon(got) != _canon(ref64.float().bfloat16())).sum())} elements differ from float64'


@gpu
@pytest.mark.parametrize('case', GEMM_CASES, ids=[_gemm_case_id(c) for c in GEMM_CASES])
def test_backward_gemms_exact(ops, case):
    """Exact operands: d(hidden) = d @ W and d(weight) = d^T @ hidden bit-identical (up to the sign of zero) to the
    float64 product rounded to bf16 -- d(weight) in one piece with acc = NULL and in row chunks through the fp32
    accumulator, which is itself exact after every middle chunk while d_weight stays unwritten.  Strides above H keep
    the pad columns' sentinel; operand rows past the tensors are NaN."""
    n, H, V, kind, strided, cuts = case
    ld = _ld(V, kind)
    hs, ws, dhs, accs, dws = _strides(H, strided)
    hidden, weight, d, _ = _gemm_operands(n, H, V, ld)
    hidden, weight = poisoned_operand(hidden, hs), poisoned_operand(weight, ws)
    d_zero = poisoned_operand(torch.nn.functional.pad(d, (0, ld - V)), ld, pad=0.0)  # K of d(hidden): columns >= V are 0
    d_nan = poisoned_operand(d, ld)  # d(weight) never reads columns >= V into a stored row: NaN there
    what = _gemm_case_id(case)
    dh = _dhidden(d_zero, n, ld, weight, V, H, dhs)
    assert dh.outside_intact(), f'{what}: d_hidden write outside (n, H)'
    _bf16_exact(dh.t, d.double() @ weight.double(), f'{what} d_hidden')
    want_w = d.double().T @ hidden.double()
    dw1, _ = _dweight(d_nan, hidden, [0, n], ld, V, H, accs, dws)
    assert dw1.outside_intact(), f'{what}: d_weight write outside (V, H)'
    _bf16_exact(dw1.t, want_w, f'{what} d_weight')
    del dw1
    if len(cuts) > 2:
        def middle(i, r1, acc, dw):
            assert dw.untouched(), f'{what}: chunk {i} wrote d_weight'
            assert acc.outside_intact(), f'{what}: chunk {i} wrote outside acc'
            part = d[:r1].double().T @ hidden[:r1].double()
            assert torch.equal(acc.t.double(), part), f'{what}: fp32 accumulator after chunk {i}'

        dwc, acc = _dweight(d_nan, hidden, cuts, ld, V, H, accs, dws, middle)
        assert dwc.outside_intact() and acc.outside_intact(), f'{what}: chunked d_weight write outside'
        _bf16_exact(dwc.t, want_w, f'{what} d_weight in chunks {cuts}')


def _bound(ref, absprod, K, extra_adds=0):
    """The provable bar of a bf16-rounded tensor-core GEMM: each of the <= K/16 + 1 truncating fp32 adds errs by less
    than 2^-23 of its running |sum| <= (|A| @ |B|); the fp32 result y then rounds to bf16 within half an ulp of |y|."""
    e = (K / 16 + 2 + extra_adds) * 2.0 ** -23 * absprod
    return _half_ulp_bf16(ref.abs() + e) + e


@gpu
@pytest.mark.parametrize('case', GEMM_CASES[1:], ids=[_gemm_case_id(c) for c in GEMM_CASES[1:]])
def test_backward_gemms_random_bound(ops, case):
    """Real-valued operands: every element within the provable bound of float64, in one piece and in row chunks (each
    chunk adds up to 1 truncating add and one rounded fp32 add of the accumulator)."""
    n, H, V, kind, strided, cuts = case
    ld = _ld(V, kind)
    hs, ws, dhs, accs, dws = _strides(H, strided)
    gen = torch.Generator(device=DEV).manual_seed(n + V + 5)
    d = (torch.randn((n, V), generator=gen, device=DEV) * 0.05).bfloat16()
    weight = poisoned_operand((torch.randn((V, H), generator=gen, device=DEV) * 0.3).bfloat16(), ws)
    hidden = poisoned_operand(torch.randn((n, H), generator=gen, device=DEV).bfloat16(), hs)
    d_zero = poisoned_operand(torch.nn.functional.pad(d, (0, ld - V)), ld, pad=0.0)
    what = _gemm_case_id(case)
    dh = _dhidden(d_zero, n, ld, weight, V, H, dhs)
    assert dh.outside_intact()
    ref = d.double() @ weight.double()
    tol = _bound(ref, d.double().abs() @ weight.double().abs(), ld)
    err = (dh.t.double() - ref).abs()
    assert bool((err <= tol).all()), f'{what} d_hidden: {int((err > tol).sum())} beyond the bound'
    _headroom(f'dhidden random {what} (err / bar)', float((err / tol).max()), 1.0)
    del ref, tol, err
    ref = d.double().T @ hidden.double()
    absprod = d.double().abs().T @ hidden.double().abs()
    for cc in ([0, n], cuts):
        dw, _ = _dweight(poisoned_operand(d, ld), hidden, cc, ld, V, H, accs, dws)
        assert dw.outside_intact()
        tol = _bound(ref, absprod, n, 2 * (len(cc) - 2))
        err = (dw.t.double() - ref).abs()
        assert bool((err <= tol).all()), f'{what} d_weight chunks {cc}: {int((err > tol).sum())} beyond the bound'
        _headroom(f'dweight random {what} chunks {cc} (err / bar)', float((err / tol).max()), 1.0)


# ---- the autograd wrapper ---------------------------------------------------------------------------------------------
# (N, H, V, chunk_rows, mode, grads): grads 'hw' both, 'h' hidden only, 'w' weight only
WRAP_CASES = [
    (300, 128, 2053, None, 'faithful', 'hw'),
    (300, 128, 2053, 128, 'faithful', 'hw'),
    (1100, 256, 5000, 1000, 'faithful', 'hw'),  # 2 chunks: 1000 becomes 768
    (301, 192, 777, 128, 'faithful', 'h'),
    (301, 192, 777, 128, 'faithful', 'w'),
    (517, 64, 1031, 256, 'f32', 'hw'),
]


@gpu
@pytest.mark.parametrize('case', WRAP_CASES, ids=[f'{c[0]}x{c[1]}x{c[2]}-c{c[3]}-{c[4]}-{c[5]}' for c in WRAP_CASES])
def test_linear_token_log_probs_composition(ops, case, monkeypatch):
    """ops.linear_token_log_probs (the K6 forward and the K6b + d(hidden) + d(weight) backward) against its parts:
    log-probs bit-identical to fused_linear_token_log_probs; d(hidden) byte-identical to one aa_linear_dhidden over
    one K6b call that covers all N rows (both kernels are row-local); d(weight) byte-identical to one aa_linear_dweight
    over that d(logits) when the backward takes one chunk, within the provable bound of float64 when it takes
    several, and finite everywhere.  The upstream gradient has zeros."""
    monkeypatch.setattr(ops, '_K6B', True)
    N, H, V, chunk, mode, grads = case
    labels = _plant_labels(N, V, 1, 1, N, oob=False).to(DEV)
    hidden, weight = _fwd_operands(N, H, V)
    code = Lb.MODE_FAITHFUL if mode == 'faithful' else Lb.MODE_F32
    g = _upstream(N, BF if code == Lb.MODE_FAITHFUL else F32, N + 3)
    g[g.isnan()] = 0.0
    h = hidden.clone().requires_grad_('h' in grads)
    w = weight.clone().requires_grad_('w' in grads)
    lp = ops.linear_token_log_probs(h, w, labels, chunk_rows=chunk, mode=mode)
    lp.backward(g)
    want_lp, stats = ops.fused_linear_token_log_probs(hidden, weight, labels, mode=mode, return_stats=True)
    assert torch.equal(lp.detach().view(INT[lp.element_size()]), want_lp.view(INT[lp.element_size()]))
    ld = _up(V, BN)
    dbuf = torch.empty((N, ld), dtype=BF, device=DEV)
    st = _stream()
    Lb.check(Lb.lib().aa_linear_dlogits(hidden.data_ptr(), N, H, H, weight.data_ptr(), V, H, labels.data_ptr(),
                                        stats[0].data_ptr(), stats[1].data_ptr(), g.data_ptr(), Lb.dtype_code(g.dtype),
                                        dbuf.data_ptr(), ld, code, st))
    if 'h' in grads:
        dh = torch.empty_like(hidden)
        Lb.check(Lb.lib().aa_linear_dhidden(dbuf.data_ptr(), N, ld, weight.data_ptr(), V, H, H, dh.data_ptr(), H, st))
        torch.cuda.synchronize()
        assert torch.equal(h.grad.view(torch.int16), dh.view(torch.int16)), 'd(hidden)'
    else:
        assert h.grad is None
    if 'w' in grads:
        n_chunks = -(-N // (chunk or N))
        if chunk is None:
            n_chunks = 1 if N <= max(128, (2 << 30) // (ld * 2) // 128 * 128) else 2
        assert bool(torch.isfinite(w.grad.float()).all()), 'd(weight) not finite'
        if n_chunks == 1:
            dw = torch.empty_like(weight)
            Lb.check(Lb.lib().aa_linear_dweight(dbuf.data_ptr(), N, ld, hidden.data_ptr(), H, H, V, None, 0, 0,
                                                dw.data_ptr(), H, st))
            torch.cuda.synchronize()
            assert torch.equal(w.grad.view(torch.int16), dw.view(torch.int16)), 'd(weight), one chunk'
        else:
            ref = dbuf[:, :V].double().T @ hidden.double()
            tol = _bound(ref, dbuf[:, :V].double().abs().T @ hidden.double().abs(), N, 2 * n_chunks)
            err = (w.grad.double() - ref).abs()
            assert bool((err <= tol).all()), f'd(weight) in {n_chunks} chunks: {int((err > tol).sum())} beyond the bound'
    else:
        assert w.grad is None
    ops.check_status()


@gpu
def test_first_launch_on_a_fresh_thread(ops):
    """The kernels encode their TMA tensor maps through the driver, which needs a current context.  A thread whose
    first CUDA work is one of these launches has none: the autograd engine's device thread when the lm_head backward
    is the first node it runs.  K6 and K6b launched from a new thread must work and write what the main thread's
    launches write."""
    import threading

    n, H, V = 130, 128, 777
    hidden, weight = _fwd_operands(n, H, V)
    labels = _plant_labels(n, V, 1, 1, 11, oob=False).to(DEV)
    g = _upstream(n, BF, 5)
    ld = _up(V, BN)
    st = _stream()

    def launch(out, stats, dl, errors):
        try:
            Lb.check(Lb.lib().aa_linear_logprob_fwd(
                hidden.data_ptr(), n, H, H, weight.data_ptr(), V, H, labels.data_ptr(), out.data_ptr(), Lb.AA_BF16,
                stats[0].data_ptr(), stats[1].data_ptr(), None, 0, Lb.MODE_FAITHFUL, None, st))
            Lb.check(Lb.lib().aa_linear_dlogits(
                hidden.data_ptr(), n, H, H, weight.data_ptr(), V, H, labels.data_ptr(), stats[0].data_ptr(),
                stats[1].data_ptr(), g.data_ptr(), Lb.AA_BF16, dl.data_ptr(), ld, Lb.MODE_FAITHFUL, st))
        except Exception as e:  # noqa: BLE001 -- reported on the main thread
            errors.append(e)

    bufs = [(torch.empty(n, dtype=BF, device=DEV), torch.empty((2, n), dtype=F32, device=DEV),
             torch.empty((n, ld), dtype=BF, device=DEV)) for _ in range(2)]
    errors = []
    th = threading.Thread(target=launch, args=(*bufs[0], errors))
    th.start()
    th.join()
    assert not errors, errors[0]
    launch(*bufs[1], errors)
    assert not errors, errors[0]
    torch.cuda.synchronize()
    for a, b in zip(*bufs):
        assert torch.equal(a.view(INT[a.element_size()]), b.view(INT[b.element_size()]))
