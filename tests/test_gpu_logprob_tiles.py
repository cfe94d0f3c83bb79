"""The gradient tile K1b and K1f write, pinned element by element (run on an H100: `pytest -m gpu`).

The tile-writing contract of the log-prob backward:
  1. scored rows hold g * (onehot - softmax(x));
  2. every unscored row inside the tile is zero;
  3. nothing else is touched: not the rows a scored-only plan leaves out, not the pad columns of a pitched tile, and
     not the bytes before or after the tile.

Every tile here lives in the middle of one larger allocation, between guard bands of at least one row and 256 bytes.
The tile starts as a NaN bit pattern, the guards and pad columns as a different sentinel, so a skipped write leaves
a NaN behind and a stray write changes a sentinel -- both inside memory the test owns.  The forward outputs (log-probs,
saved max / log-sum) are poisoned the same way.

Each case runs the TMA-staged K1b and the LDG row kernel, in both modes, through every route its plan allows, and
checks:
  * scored rows against float64 (f32 mode: |err| <= 2e-5 * max(|g|, |ref|), plus half an ulp of a 16-bit tile) or
    against the eager ATen chain in the tile dtype (faithful mode: DESIGN section 4's bar);
  * zero rows are exactly 0, rows outside a scored-only plan, pad columns and guards are bit for bit unchanged;
  * both kernels, and the host-layout route (memset spans + listed zero rows) and the tile route (the kernel zero-fills
    every unscored row), write byte-identical buffers, guards included;
  * the forward writes every scored log-prob, 0 for ignored rows, and nothing else;
  * grad_entropy: K1b's entropy-gradient variant on the same case leaves the rows with g_H == 0 bit-identical to
    aa_logprob_bwd's and puts the float64 tile formula with the entropy term in the others.  It runs once per case and
    mode, through the case's first route: aa_logprob_bwd_entropy is always TMA-staged (the LDG row kernel has no
    entropy variant), so there is no LDG run to compare.
K1f (the single-pass nodes) is checked against K1 -> loss kernel -> K1b on the same inputs, both into guarded tiles.
"""
import ctypes
import itertools

import pytest
import torch

from align_anything_b200 import _lib as Lb
from oracle import ref_port as O
from test_gpu_parity import assert_close_f32, assert_ulp_close, ops  # noqa: F401

pytestmark = pytest.mark.gpu

DEV = 'cuda'
IGNORE = -100
TMA, LDG = 0, 3  # aa_logprob_set_tuning_bwd variants
# bit patterns: POISON is a NaN in bf16, fp16 (0x7FA5) and fp32 (0x7FA5A5A5); SENTINEL is a finite value
POISON = {2: 0x7FA5, 4: 0x7FA5A5A5}
SENTINEL = {2: 0x3C5A, 4: 0x3C5A5A5A}
INT = {2: torch.int16, 4: torch.int32}


# ---- guarded buffers -----------------------------------------------------------------------------------------------
class Guarded:
    """A (rows, V) tile with row pitch `pitch` inside one allocation.  The guard bands before and after it hold at least
    one row and 256 bytes and keep the tile 16-byte aligned.  Tile elements start as POISON, everything else (guards,
    pad columns) as SENTINEL."""

    def __init__(self, rows, V, pitch, dtype):
        esz = torch.empty(0, dtype=dtype).element_size()
        g = max(pitch, 256 // esz)
        self.guard = (g + 15) // 16 * 16
        self.rows, self.V, self.pitch, self.esz = rows, V, pitch, esz
        self.buf = torch.empty(2 * self.guard + rows * pitch, dtype=dtype, device=DEV)
        self.bits = self.buf.view(INT[esz])
        self.bits.fill_(SENTINEL[esz])
        self.bits.as_strided((rows, V), (pitch, 1), self.guard).fill_(POISON[esz])
        self.fresh = self.bits.clone()
        self.tile = self.buf.as_strided((rows, V), (pitch, 1), self.guard)

    def outside(self):
        """bool mask over the allocation: guards and pad columns."""
        m = torch.ones(self.buf.numel(), dtype=torch.bool, device=DEV)
        m.as_strided((self.rows, self.V), (self.pitch, 1), self.guard).fill_(False)
        return m

    def row_bits(self, rows):
        return self.bits.as_strided((self.rows, self.V), (self.pitch, 1), self.guard)[rows]


def _poisoned(shape, dtype):
    t = torch.empty(shape, dtype=dtype, device=DEV)
    t.view(INT[t.element_size()]).fill_(POISON[t.element_size()])
    return t


def _status_take():
    """Read and clear the device status word."""
    from align_anything_b200 import ops as _ops

    st = _ops._device_scratch(torch.device(DEV))['status']
    v = int(st.item())
    st.zero_()
    return v


def _set_bwd_kernel(variant):
    Lb.check(Lb.lib().aa_logprob_set_tuning_bwd(variant, 0))


def _half_ulp(ref64, dtype):
    """Half an ulp of `dtype` at |ref| (float64): the rounding of the finished value into a 16-bit tile."""
    if dtype == torch.float32:
        return torch.zeros_like(ref64)
    fi = torch.finfo(dtype)
    a = ref64.abs().clamp(min=fi.tiny)
    return torch.exp2(torch.floor(torch.log2(a))) * fi.eps / 2 + fi.tiny * fi.eps / 2


# ---- the matrix ------------------------------------------------------------------------------------------------------
# (dtype, V, plan, layout, grad sources, use_ignore, samples B, rows per sample S)
#   plan:   'host'   RowPlan with a tile: run in tile mode (kernel zero-fills) AND host layout (memset spans + listed rows)
#           'device' DevicePlan from aa_tail_plan_build (tile mode), lengths that clamp to 0 included
#           'scored' RowPlan without a tile (n_tile_rows == 0): rows outside the plan keep their poison
#   layout: 'contig' | 'pitch' (logits and tile share a pitch > V) | 'mixed' (different pitches) | 'odd' (logits base
#           one element off: 2-byte aligned rows)
#   grad:   'r<dt>' grad_rows in dtype dt, 'seg' grad_seg, 's<dt>' a device grad_scale in dtype dt, joined by '+'
BF, F16, F32 = torch.bfloat16, torch.float16, torch.float32
CASES = [
    (BF, 1, 'host', 'contig', 'rbf', True, 6, 24),
    (BF, 7, 'scored', 'odd', 'seg', False, 6, 24),
    (BF, 8, 'device', 'pitch', 'rf32+sbf', False, 6, 24),
    (BF, 9, 'host', 'mixed', 'rf16+seg+sf32', False, 160, 24),  # > 3 x 132 x 4 work rows: every CTA loops
    (BF, 2048, 'scored', 'contig', 'rbf+seg', True, 4, 24),
    (BF, 2049, 'host', 'contig', 'rbf', False, 4, 24),
    (BF, 4096, 'device', 'contig', 'rbf+sf16', False, 4, 24),
    (BF, 4097, 'host', 'pitch', 'seg+sbf', False, 4, 24),
    (BF, 8192, 'host', 'odd', 'rf32', True, 3, 24),
    (BF, 8193, 'scored', 'mixed', 'rbf', False, 3, 24),
    (BF, 32064, 'host', 'contig', 'rbf+seg', False, 3, 20),
    (BF, 128257, 'host', 'contig', 'rbf', True, 3, 16),
    (BF, 128257, 'device', 'contig', 'rf32', False, 4, 12),
    (F16, 1, 'scored', 'contig', 'rf16', False, 6, 24),
    (F16, 7, 'host', 'pitch', 'rf16+sf16', True, 6, 24),
    (F16, 9, 'device', 'odd', 'seg', False, 6, 24),
    (F16, 2049, 'host', 'mixed', 'rbf', False, 4, 24),
    (F16, 4097, 'device', 'pitch', 'rf16+seg', True, 4, 24),
    (F16, 8193, 'scored', 'contig', 'rf32+sf32', False, 3, 24),
    (F16, 32064, 'host', 'contig', 'rf16', False, 3, 20),
    (F16, 128257, 'scored', 'contig', 'rf16', False, 2, 16),
    (F32, 1, 'device', 'contig', 'rf32', False, 6, 24),
    (F32, 8, 'scored', 'contig', 'rf32', False, 180, 24),  # > 3 x 132 x 4 scored rows
    (F32, 9, 'host', 'odd', 'rbf+sbf', True, 6, 24),
    (F32, 2048, 'scored', 'pitch', 'seg+sf32', False, 4, 24),
    (F32, 2049, 'host', 'contig', 'rf32', False, 4, 24),
    (F32, 4096, 'host', 'mixed', 'rf16', False, 3, 24),
    # the forward's ring / LDG switch at 128 KB rows: 32767 streams through the ring, 32768 and 32769 take the LDG
    # kernel.  32767 also has no label outside the vocabulary: the out-of-range status bit must stay clear
    (F32, 32767, 'host', 'contig', 'rf32', False, 3, 16, False),
    (F32, 32768, 'host', 'contig', 'rf32', True, 3, 16),
    (F32, 32769, 'device', 'contig', 'rf32+seg', False, 4, 16),
]
_DT = {'bf': BF, 'f16': F16, 'f32': F32}


def _case_id(c):
    return (f'{str(c[0])[6:]}-V{c[1]}-{c[2]}-{c[3]}-{c[4]}' + ('-ignore' if c[5] else '') + f'-{c[6]}x{c[7]}'
            + ('-inrange' if len(c) > 8 and not c[8] else ''))


def _pitches(layout, V, esz):
    """-> (logits pitch, logits base offset in elements, tile pitch)."""
    q = 16 // esz
    if layout == 'contig':
        return V, 0, V
    if layout == 'pitch':
        P = (V + q - 1) // q * q + q
        return P, 0, P
    if layout == 'mixed':
        return V + 3, 0, (V + q - 1) // q * q + q
    return V, 1, V  # 'odd'


def _counts(B, S):
    """Scored rows per sample: long and short gaps between them (memset spans and listed rows in the host layout),
    an empty sample, and a last sample with nothing scored, so the last zero span ends at the tile's end."""
    pat = [S - 1, S - 6, 3, 0, S // 2, 1, 7]
    c = [min(pat[i % len(pat)], S - 1) for i in range(B)]
    c[-1] = 0
    return c


class Case:
    """Inputs of one matrix case and the host-side list of its scored rows (in the plan's flat row order).
    oob = False: every label lies in [0, V) (or is ignored)."""

    def __init__(self, ops, dtype, V, plan, layout, grad, ignore, B, S, oob=True):
        gen = torch.Generator().manual_seed(V * 31 + B * 7 + S + len(plan) + len(layout) + len(grad))
        self.dtype, self.V, self.kind, self.layout, self.ignore, self.B, self.S = dtype, V, plan, layout, ignore, B, S
        esz = torch.empty(0, dtype=dtype).element_size()
        self.lpitch, self.loff, self.gpitch = _pitches(layout, V, esz)
        R = B * S
        self.R = R
        n = self.loff + R * self.lpitch
        self.lbuf = (torch.randn(n + 16, generator=gen) * 2.5).to(dtype).to(DEV)
        self.logits = self.lbuf.as_strided((R, V), (self.lpitch, 1), self.loff)
        if plan == 'device':
            lens = [[S - 1, 0, 7, -2, 3, S // 2][b % 6] for b in range(B)]  # -2 clamps to 0 (status: short sequence)
            self.lens = lens
            W = S - 1
            dl = ops.DeviceLens(torch.tensor(lens, dtype=torch.int32, device=DEV), W)
            _status_take()
            self.plan = ops.DevicePlan(dl, S, S * self.lpitch, self.lpitch, S, S, 0, -1, W)
            self.plan_status = _status_take()
            labels = torch.randint(0, V, (B, S), generator=gen)
            rows = []  # (tile row, label position, out index, segment)
            for b, r in enumerate(lens):
                r = max(0, min(r, S - 1))
                first = S - r - 1
                for j in range(min(r, W)):
                    rows.append((b * S + first + j, b * S + S - r + j, b * W + j, b))
            self.n_seg, out_shape = B, (B, W)
        else:
            counts = _counts(B, S)
            firsts = [S - c - 1 for c in counts]
            W = max(max(counts), 1)
            labels = torch.randint(0, V, (R,), generator=gen)
            self.plan = ops.RowPlan([(b * S + firsts[b]) * self.lpitch for b in range(B)],
                                    [b * S + firsts[b] for b in range(B)], [b * W for b in range(B)], counts,
                                    [b * S + firsts[b] for b in range(B)], (B, W), 0 if plan == 'scored' else R, DEV)
            rows = [(b * S + firsts[b] + j, b * S + firsts[b] + j, b * W + j, b) for b in range(B) for j in range(counts[b])]
            self.n_seg, out_shape = B, (B, W)
        self.out_shape = out_shape
        self.tile_row = torch.tensor([r[0] for r in rows], dtype=torch.int64)
        lab_pos = torch.tensor([r[1] for r in rows], dtype=torch.int64)
        self.out_idx = torch.tensor([r[2] for r in rows], dtype=torch.int64)
        self.seg = torch.tensor([r[3] for r in rows], dtype=torch.int64)
        k = len(rows)
        assert k > 8, 'every case has scored rows of each special kind'
        # labels: column 0, V - 1, inside the head / tail peel, both sides of the first 8 KB stage boundary, out of range
        # above the vocabulary (once) and below it (or ignored, twice), random elsewhere
        stage = 8192 // esz
        special = [0, V - 1, min(1, V - 1), max(V - 2, 0), stage - 1 if V > stage else None, stage if V > stage else None,
                   V + 3 if oob else None, IGNORE if (oob or ignore) else None]
        flat = labels.view(-1)
        for i in range(k):
            s = special[i % 10] if i % 10 < len(special) else None
            if s is not None and (0 <= s < V or i < 20) and not (s == V + 3 and i >= 10):
                flat[lab_pos[i]] = s
        self.labels = labels.to(DEV)
        self.y = flat[lab_pos].clone()
        self.ignored = (self.y == IGNORE) if ignore else torch.zeros(k, dtype=torch.bool)
        self.oob = ((self.y < 0) | (self.y >= V)) & ~self.ignored
        # upstream gradients: every factor exactly representable in bf16, fp16 and fp32, so the faithful reference can
        # take the product in the tile dtype
        parts = grad.split('+')
        g_rows = (torch.randn(out_shape, generator=gen).bfloat16().float() * 2)
        g_rows = torch.where(g_rows.abs() < 2 ** -8, torch.full_like(g_rows, 0.75), g_rows)
        g_rows.view(-1)[self.out_idx[8]] = 0.0       # g == 0: written as a zero row
        g_rows.view(-1)[self.out_idx[9]] = float('nan')  # NaN g: a NaN row, as in ATen
        g_seg = torch.tensor([[0.5, -2.0, 4.0, 1.0, -0.25][s % 5] for s in range(self.n_seg)])
        if not any(p.startswith('r') for p in parts) and self.seg[k - 1] != self.seg[0]:
            g_seg[self.seg[k - 1]] = 0.0  # without per-row gradients, the last scored segment has g == 0
        self.grad_rows = self.grad_seg = self.grad_scale = None
        g = torch.ones(k, dtype=torch.float64)
        for p in parts:
            if p.startswith('r'):
                self.grad_rows = g_rows.to(_DT[p[1:]]).to(DEV)
                g = g * g_rows.view(-1)[self.out_idx].double()
            elif p == 'seg':
                self.grad_seg = g_seg.float().to(DEV)
                g = g * g_seg[self.seg].double()
            else:
                self.grad_scale = torch.tensor([-0.5], dtype=_DT[p[1:]], device=DEV)
                g = g * -0.5
        self.g = torch.where(self.ignored, torch.zeros_like(g), g)  # an ignored row gets no gradient
        self.zero_g = (g == 0) | self.ignored
        self.nan_g = torch.isnan(g) & ~self.ignored
        self.scored_rows = set(self.tile_row.tolist())

    def routes(self):
        return [True, False] if self.kind == 'host' else [None]  # _ZERO_SPANS: host layout, tile mode

    def run(self, ops, mode_code, kernel, zero_spans, monkeypatch, grad_entropy=None):
        """One forward + backward into freshly poisoned buffers -> (tile guard object, out, stats, status word).
        grad_entropy (fp32, laid out like the log-probs): K1b's entropy-gradient variant, fed the float64 entropy of
        the scored rows rounded to fp32."""
        if zero_spans is not None:
            monkeypatch.setattr(ops, '_ZERO_SPANS', zero_spans)
        out_dtype = self.dtype if mode_code == Lb.MODE_FAITHFUL else torch.float32
        out = _poisoned(self.out_shape, out_dtype)
        stats = _poisoned((2, max(self.plan.n_rows, 1)), torch.float32)
        tile = Guarded(self.R, self.V, self.gpitch, self.dtype)
        ig = IGNORE if self.ignore else None
        _status_take()
        ops._launch_fwd(self.logits, self.labels, self.plan, out, stats[0], stats[1], ignore_index=ig)
        ent = None
        if grad_entropy is not None:
            from test_gpu_entropy import entropy64

            ent = torch.zeros(self.out_shape, dtype=torch.float32, device=DEV)
            ent.view(-1)[self.out_idx.to(DEV)] = entropy64(self.logits[self.tile_row.to(DEV)]).float()
        _set_bwd_kernel(kernel)
        try:
            ops._launch_bwd(self.logits, self.labels, self.plan, stats[0], stats[1], self.grad_rows, self.grad_seg,
                            self.grad_scale, tile.tile, mode_code, ignore_index=ig, grad_row_stride=self.gpitch,
                            entropy=ent, grad_entropy=grad_entropy)
        finally:
            _set_bwd_kernel(-1)
        torch.cuda.synchronize()
        return tile, out, stats, _status_take()


def _check_against_reference(case, mode_code, tile, out, stats, status):
    what = f'{_case_id((case.dtype, case.V, case.kind, case.layout, "", case.ignore, case.B, case.S))} mode {mode_code}'
    dtype, V = case.dtype, case.V
    k = case.tile_row.numel()
    idx_all = torch.arange(k)
    live = ~case.ignored & ~case.zero_g
    X = case.logits[case.tile_row.to(DEV)]  # (k, V) scored logits rows
    got = tile.tile[case.tile_row.to(DEV)]
    # 1. forward: every scored log-prob written, ignored rows exactly 0, stats = log-sum-exp, nothing else touched
    out_flat, out_bits = out.view(-1), out.view(-1).view(INT[out.element_size()])
    written = torch.zeros(out_flat.numel(), dtype=torch.bool)
    written[case.out_idx] = True
    assert bool((out_bits[written.to(DEV)] != POISON[out.element_size()]).all()), f'{what}: a log-prob was not written'
    assert bool((out_bits[~written.to(DEV)] == POISON[out.element_size()]).all()), f'{what}: write outside the scored rows'
    lp = out_flat[case.out_idx.to(DEV)].cpu()
    if case.ignored.any():
        assert bool((lp[case.ignored] == 0).all()), f'{what}: ignored rows must score 0'
        assert bool((stats[:, : k][:, case.ignored.to(DEV)] == 0).all())
    x64 = X.double()
    lse = torch.logsumexp(x64, dim=-1)
    st = (stats[0, :k] + stats[1, :k]).double()
    nz = ~case.ignored.to(DEV)
    assert bool(((st - lse).abs()[nz] <= 2e-5 * lse.abs().clamp(min=1.0)[nz]).all()), f'{what}: saved max + log-sum'
    st_bits = stats.view(torch.int32)
    assert bool((st_bits[:, k:] == POISON[4]).all()), f'{what}: stats written past the scored rows'
    assert bool((status & Lb.STATUS_LABEL_OOB) != 0) == bool(case.oob.any()), f'{what}: status {status:#x}'
    y_safe = torch.where(case.oob | case.ignored, torch.zeros_like(case.y), case.y)
    onehot = torch.zeros(k, V, dtype=torch.float64)
    onehot[idx_all, y_safe] = 1.0
    onehot[case.oob | case.ignored] = 0.0  # no one-hot term for a label outside [0, V)
    g64 = case.g.to(DEV)
    ref64 = g64[:, None] * (onehot.to(DEV) - torch.exp(x64 - lse[:, None]))
    # 2. zero rows: ignored, g == 0 and (tile / host routes) every unscored tile row
    zrows = case.tile_row[case.zero_g]
    if case.kind != 'scored':
        zrows = torch.tensor(sorted(set(range(case.R)) - set(case.tile_row[live | case.nan_g].tolist())), dtype=torch.int64)
    if zrows.numel():
        z = tile.tile[zrows.to(DEV)]
        assert bool((z == 0).all()) and not bool(torch.isnan(z).any()), f'{what}: a zero row is not zero'
    # 3. rows outside a scored-only plan, pad columns and guards: bit for bit unchanged
    keep = tile.outside()
    if case.kind == 'scored':
        outside_rows = torch.tensor(sorted(set(range(case.R)) - case.scored_rows), dtype=torch.int64)
        if outside_rows.numel():
            rb = tile.row_bits(outside_rows.to(DEV))
            assert bool((rb == POISON[tile.esz]).all()), f'{what}: a row outside the plan was written'
    assert torch.equal(tile.bits[keep], tile.fresh[keep]), f'{what}: a guard or pad sentinel changed'
    # 4. scored rows against the references
    if mode_code == Lb.MODE_F32:
        lp_ref = x64[idx_all.to(DEV), y_safe.to(DEV)] - lse
        lp_ref[(case.oob).to(DEV)] = float('nan')
        lp_ref[case.ignored.to(DEV)] = 0.0
        assert_close_f32(lp, lp_ref.float().cpu(), what=f'{what} log-probs')
        gv = got.double()
        assert torch.equal(torch.isnan(gv), torch.isnan(ref64)), f'{what}: NaN pattern of the tile'
        err = (torch.nan_to_num(gv) - torch.nan_to_num(ref64)).abs()
        tol = 2e-5 * torch.maximum(g64.abs()[:, None], ref64.abs()).nan_to_num() + _half_ulp(torch.nan_to_num(ref64), dtype)
        bad = err > tol
        assert not bool(bad.any()), f'{what}: tile max err {float(err.max()):.3e}, {int(bad.sum())} elements beyond tolerance'
        return
    # faithful: the eager ATen chain in the tile dtype (a label outside [0, V): column 0 stands in, then patched)
    leaf = X.clone().requires_grad_(True)
    ref_lp = O.token_log_probs(leaf.unsqueeze(0), y_safe.to(DEV).unsqueeze(0))[0]
    g_t = case.g.to(dtype).to(DEV)
    g_t[case.ignored.to(DEV)] = 0
    ref_lp.backward(g_t)
    ref_tile = leaf.grad.clone()
    if case.oob.any():
        lsm = torch.log_softmax(X[case.oob.to(DEV)], dim=-1)
        ref_tile[case.oob.to(DEV), 0] = (-(torch.exp(lsm[:, 0].float()) * g_t[case.oob.to(DEV)].float())).to(dtype)
    ref_lp = ref_lp.detach().clone()
    ref_lp[case.oob.to(DEV)] = float('nan')
    ref_lp[case.ignored.to(DEV)] = 0
    assert_ulp_close(lp, ref_lp, max_ulp=1, min_exact=0.97, what=f'{what} log-probs')
    assert_ulp_close(got, ref_tile, max_ulp=2, min_exact=0.97, what=f'{what} tile', tie_frac=1e-4, tie_ulp=40)


@pytest.mark.parametrize('case_args', CASES, ids=[_case_id(c) for c in CASES])
def test_backward_tile_contract(ops, case_args, monkeypatch):
    """K1 + K1b (TMA-staged and LDG) through the case's plan routes, in both modes, into poisoned guarded buffers."""
    case = Case(ops, *case_args)
    for mode_code in (Lb.MODE_FAITHFUL, Lb.MODE_F32):
        runs = []
        for kernel, route in itertools.product((TMA, LDG), case.routes()):
            runs.append(((kernel, route), case.run(ops, mode_code, kernel, route, monkeypatch)))
        (_, (tile0, out0, stats0, status0)) = runs[0]
        for key, (tile, out, stats, status) in runs[1:]:
            assert torch.equal(tile.bits, tile0.bits), f'{_case_id(case_args)} mode {mode_code}: {key} wrote a different buffer'
            assert torch.equal(out.view(INT[out.element_size()]), out0.view(INT[out0.element_size()]))
            assert torch.equal(stats.view(torch.int32), stats0.view(torch.int32)) and status == status0
        if case.kind == 'device':
            flagged = bool(case.plan_status & Lb.STATUS_SHORT_SEQUENCE)
            assert flagged == any(r < 0 for r in case.lens), 'a negative length is clamped to 0 and flagged'
        _check_against_reference(case, mode_code, tile0, out0, stats0, status0)
        _check_entropy_gradient(ops, case, mode_code, runs[0][0][1], tile0, monkeypatch)


def _check_entropy_gradient(ops, case, mode_code, route, plain, monkeypatch):
    """The grad_entropy axis: aa_logprob_bwd_entropy (always TMA-staged) on the case's rows with g_H != 0 on most
    scored rows, the g == 0 row included.  Rows with g_H == 0, the rows outside the plan, pad columns and guards are
    bit-identical to aa_logprob_bwd's buffer; the others hold test_gpu_entropy_bonus._tile64's
    g (onehot - p) - g_H p (l + H) (FAITHFUL: the rounded log-softmax) at its _close bar."""
    from test_gpu_entropy_bonus import EPS, _tile64

    k = case.tile_row.numel()
    gh = torch.tensor([0.0, 0.5, -1.25, 0.0, 2.0, -0.375])[torch.arange(k) % 6]
    gh[8] = 0.75  # g == 0: the row carries the entropy's gradient alone
    gh[case.ignored | case.oob | case.nan_g] = 0.0
    gh_rows = torch.zeros(case.out_shape, dtype=torch.float32)
    gh_rows.view(-1)[case.out_idx] = gh
    tile, out, stats, status = case.run(ops, mode_code, TMA, route, monkeypatch, grad_entropy=gh_rows.to(DEV))
    what = f'{_case_id((case.dtype, case.V, case.kind, case.layout, "", case.ignore, case.B, case.S))} mode {mode_code}'
    hot = torch.zeros(case.R, dtype=torch.bool)
    hot[case.tile_row[gh != 0]] = True
    keep = tile.outside()
    assert torch.equal(tile.bits[keep], plain.bits[keep]), f'{what}: grad_entropy changed a guard or pad column'
    cold = torch.nonzero(~hot).flatten().to(DEV)
    assert torch.equal(tile.row_bits(cold), plain.row_bits(cold)), f'{what}: a row with g_H == 0 differs from K1b'
    sel = gh != 0
    rows = case.tile_row[sel].to(DEV)
    x = case.logits[rows].float()
    y = case.y[sel].to(DEV)
    faithful = case.dtype if (mode_code == Lb.MODE_FAITHFUL and case.dtype != torch.float32) else None
    g_h = gh[sel].to(DEV) * (-0.5 if case.grad_scale is not None else 1.0)  # grad_scale multiplies g_H too
    g = case.g[sel].to(DEV)
    want = _tile64(x, y, g, g_h, faithful)
    # test_gpu_entropy_bonus._close's bar, its floor relative to the larger of the row's largest element, |g| and |g_H|
    # (a one-column row has want == 0 and p rounded from an fp32 exp)
    scale = torch.maximum(want.abs().amax(-1), torch.maximum(g.abs(), g_h.abs()).double())[:, None]
    eps = EPS[case.dtype]
    err = (tile.tile[rows].double() - want).abs()
    bad = ~(err <= eps * want.abs() + max(eps, 2e-5) * scale)
    assert not bool(bad.any()), f'{what} grad_entropy: {int(bad.sum())} elements beyond tolerance'


def test_pitched_tile_host_layout_keeps_pad_columns(ops, monkeypatch):
    """A host-layout plan on a pitched tile: the copy-engine spans clear the zero rows' V columns at the tile's pitch
    and leave the pad columns alone -- what the lm_head backward relies on for its padded d(logits) buffer."""
    case = Case(ops, BF, 1000, 'host', 'pitch', 'rbf', False, 4, 24)
    assert case.plan.n_zero_spans > 0
    tile, out, stats, status = case.run(ops, Lb.MODE_FAITHFUL, TMA, True, monkeypatch)
    _check_against_reference(case, Lb.MODE_FAITHFUL, tile, out, stats, status)
    # aa_zero_rows alone: spans at the pitch, pad columns and guards untouched
    t = Guarded(10, 33, 40, BF)
    spans = (ctypes.c_int64 * 4)(1, 2, 7, 3)
    Lb.check(Lb.lib().aa_zero_rows(t.tile.data_ptr(), Lb.dtype_code(BF), 40, 33, 10, ctypes.cast(spans, ctypes.c_void_p), 2,
                                   Lb.stream_ptr(t.buf.device)))
    want = t.fresh.clone()
    for a, n in ((1, 2), (7, 3)):
        want.as_strided((10, 33), (40, 1), t.guard)[a:a + n] = 0
    assert torch.equal(t.bits, want)


# ---- K1f: the single-pass nodes against K1 -> loss kernel -> K1b ---------------------------------------------------
def _zero_rows(tile):
    return (tile.tile.float().abs().amax(dim=-1) == 0) & ~torch.isnan(tile.tile.float()).any(dim=-1)


def _compare_tiles(a, b, what):
    """b (single pass) against a (two-pass): same zero rows, DESIGN section 4's K1f bar, guards intact in both."""
    for t in (a, b):
        keep = t.outside()
        assert torch.equal(t.bits[keep], t.fresh[keep]), f'{what}: a guard sentinel changed'
        assert not bool((t.row_bits(slice(None)) == POISON[t.esz]).any()), f'{what}: a tile element was not written'
    assert torch.equal(_zero_rows(a), _zero_rows(b)), f'{what}: the two paths disagree on which rows carry gradient'
    if a.tile.dtype == torch.float32:
        assert_close_f32(b.tile, a.tile, what=f'{what} tile')
    else:
        assert_ulp_close(b.tile, a.tile, max_ulp=2, min_exact=0.97, what=f'{what} tile', tie_frac=1e-4, tie_ulp=40)


def _device_plan(ops, lens, B, S, V):
    W = S - 1
    dl = ops.DeviceLens(torch.tensor(lens, dtype=torch.int32, device=DEV), W)
    return ops.DevicePlan(dl, S, S * V, V, S, S, 0, -1, W), W


@pytest.mark.parametrize('dtype,V', [(BF, 32064), (BF, 128257), (F32, 8200), (F32, 65537)])
def test_single_pass_actor_tile_contract(ops, dtype, V):
    """aa_logprob_actor_fused against K1 -> K5 -> K1b, both into poisoned guarded tiles: masked tokens, clipped tokens
    and samples with nothing scored become zero rows in both; rows under and over 192 KB."""
    gen = torch.Generator().manual_seed(V + 5)
    B, S = 3, 12
    lens = [S - 1, 0, 6]
    plan, W = _device_plan(ops, lens, B, S, V)
    logits = (torch.randn(B * S, V, generator=gen) * 2.5).to(dtype).to(DEV)
    ids = torch.randint(0, V, (B, S), generator=gen).to(DEV)
    mode = Lb.MODE_FAITHFUL
    lp_dtype = dtype
    old = torch.zeros((B, W), dtype=lp_dtype, device=DEV)
    stats = torch.empty((2, plan.n_rows), dtype=torch.float32, device=DEV)
    ops._launch_fwd(logits, ids, plan, old, stats[0], stats[1])
    old = (old.float() + 0.4 * torch.randn(B, W, generator=gen).to(DEV)).to(lp_dtype)
    adv = (3.0 * torch.randn(B, W, generator=gen)).to(DEV)  # large |A| x noisy old log-probs: clipped tokens occur
    mask = torch.zeros((B, W), dtype=torch.bool, device=DEV)
    for b, r in enumerate(lens):
        mask[b, :r] = True
    mask[0, 2] = mask[2, 0] = False  # masked-off tokens inside a response
    _status_take()
    # two passes: K1 -> K5 -> K1b
    lp_a = torch.zeros((B, W), dtype=lp_dtype, device=DEV)
    ops._launch_fwd(logits, ids, plan, lp_a, stats[0], stats[1])
    _, _, g_lp, _ = ops._ppo_loss_launch(lp_a, old, adv, mask, 0.2, mode, True)
    assert bool(((g_lp == 0) & mask).any()), 'no clipped token (mask on, d loss / d log-prob == 0)'
    tile_a = Guarded(B * S, V, V, dtype)
    ops._launch_bwd(logits, ids, plan, stats[0], stats[1], g_lp, None, None, tile_a.tile, mode)
    # one pass: K1f
    lp_b = torch.zeros((B, W), dtype=lp_dtype, device=DEV)
    tile_b = Guarded(B * S, V, V, dtype)
    scratch = torch.empty(plan.n_tile_rows * 6, dtype=torch.int64, device=DEV)
    sc = ops._device_scratch(torch.device(DEV))
    p = plan.ptrs()
    Lb.check(Lb.lib().aa_logprob_actor_fused(
        logits.data_ptr(), Lb.dtype_code(dtype), V, V, ids.data_ptr(), plan.n_seg, p[0], p[1], p[2], p[3], p[4],
        plan.n_tile_rows, lp_b.data_ptr(), Lb.dtype_code(lp_dtype), None, None, old.data_ptr(), old.stride(0),
        adv.data_ptr(), adv.stride(0), Lb.dtype_code(adv.dtype), mask.data_ptr(), mask.stride(0), W, 0.2, mode,
        tile_b.tile.data_ptr(), V, scratch.data_ptr(), sc['status'].data_ptr(), Lb.stream_ptr(tile_b.buf.device)))
    torch.cuda.synchronize()
    assert _status_take() == 0
    if dtype == torch.float32:
        assert_close_f32(lp_b, lp_a, what='log-probs')
    else:
        assert_ulp_close(lp_b, lp_a, max_ulp=1, min_exact=0.95, what='log-probs')
    zero = _zero_rows(tile_a)
    assert int(zero.sum()) > B * S - sum(max(r, 0) for r in lens)  # masked / clipped rows exist among the scored ones
    _compare_tiles(tile_a, tile_b, f'actor V={V}')


@pytest.mark.parametrize('dtype,V', [(BF, 32064), (BF, 128257), (F32, 8200), (F32, 65537)])
def test_single_pass_grpo_tile_contract(ops, dtype, V):
    """aa_logprob_grpo_fused against K1 -> aa_grpo_loss -> K1b, both into poisoned guarded tiles.  A completion counts up
    to and including its first eos: the rows after it, the prompt rows and the last row of each sample are zero rows in
    both; one completion has no eos at all, one ends at its first token."""
    gen = torch.Generator().manual_seed(V + 13)
    B, S, K = 4, 12, 8  # K completion rows per sample, scored by logits rows S - K - 1 .. S - 2
    eos = V - 1
    # the plan's output width is K: the log-probs, reference log-probs and d loss / d log-prob are all (B, K)
    dl = ops.DeviceLens(torch.full((B,), K, dtype=torch.int32, device=DEV), K)
    plan = ops.DevicePlan(dl, S, S * V, V, S, S, 0, -1, K)
    logits = (torch.randn(B * S, V, generator=gen) * 2.5).to(dtype).to(DEV)
    ids = torch.randint(0, V - 1, (B, S), generator=gen)  # no eos but the ones placed below
    ids[0, S - K + 3] = eos  # eos inside the completion: row_end 4
    ids[2, S - K] = eos      # eos at the first completion token: row_end 1
    ids[3, S - K + 5] = eos  # row_end 6; sample 1 has no eos: row_end K
    want_end = [4, K, 1, 6]
    ids = ids.to(DEV)
    tokens = ids[:, -K:]
    mode = Lb.MODE_FAITHFUL
    lp_dtype = dtype
    sc = ops._device_scratch(torch.device(DEV))
    stats = torch.empty((2, plan.n_rows), dtype=torch.float32, device=DEV)
    _status_take()
    # two passes: K1 -> aa_grpo_loss -> K1b
    lp_a = torch.zeros((B, K), dtype=lp_dtype, device=DEV)
    ops._launch_fwd(logits, ids, plan, lp_a, stats[0], stats[1])
    ref = (lp_a.float() + 0.3 * torch.randn(B, K, generator=gen).to(DEV)).to(lp_dtype)
    adv = torch.tensor([1.5, -0.75, 0.5, -2.0], dtype=torch.float32, device=DEV)
    g_lp = torch.zeros((B, K), dtype=lp_dtype, device=DEV)
    row_end_a = torch.empty(B, dtype=torch.int32, device=DEV)
    loss_a = torch.empty(1, dtype=torch.float32, device=DEV)
    loss_scratch = torch.empty(B + 1, dtype=torch.float32, device=DEV)
    Lb.check(Lb.lib().aa_grpo_loss(
        lp_a.data_ptr(), lp_a.stride(0), ref.data_ptr(), ref.stride(0), Lb.dtype_code(lp_dtype), adv.data_ptr(),
        tokens.data_ptr(), tokens.stride(0), eos, B, K, 0.04, mode, loss_a.data_ptr(), g_lp.data_ptr(), g_lp.stride(0),
        row_end_a.data_ptr(), loss_scratch.data_ptr(), sc['counter'][5:7].data_ptr(), Lb.stream_ptr(lp_a.device)))
    tile_a = Guarded(B * S, V, V, dtype)
    ops._launch_bwd(logits, ids, plan, stats[0], stats[1], g_lp, None, None, tile_a.tile, mode)
    # one pass: K1f
    lp_b = torch.zeros((B, K), dtype=lp_dtype, device=DEV)
    tile_b = Guarded(B * S, V, V, dtype)
    scratch = torch.empty(plan.n_tile_rows * 6, dtype=torch.int64, device=DEV)
    row_end_b = torch.empty(B, dtype=torch.int32, device=DEV)
    total = torch.empty(B + 1, dtype=torch.float32, device=DEV)
    p = plan.ptrs()
    Lb.check(Lb.lib().aa_logprob_grpo_fused(
        logits.data_ptr(), Lb.dtype_code(dtype), V, V, ids.data_ptr(), plan.n_seg, p[0], p[1], p[2], p[3], p[4],
        plan.n_tile_rows, lp_b.data_ptr(), Lb.dtype_code(lp_dtype), ref.data_ptr(), ref.stride(0), adv.data_ptr(),
        tokens.data_ptr(), tokens.stride(0), eos, K, 0.04, mode, tile_b.tile.data_ptr(), V, scratch.data_ptr(),
        row_end_b.data_ptr(), total.data_ptr(), sc['counter'][5:6].data_ptr(), sc['status'].data_ptr(),
        Lb.stream_ptr(tile_b.buf.device)))
    torch.cuda.synchronize()
    assert _status_take() == 0
    assert row_end_a.tolist() == want_end and row_end_b.tolist() == want_end
    if dtype == torch.float32:
        assert_close_f32(lp_b, lp_a, what='log-probs')
    else:
        assert_ulp_close(lp_b, lp_a, max_ulp=1, min_exact=0.95, what='log-probs')
    # the rows after each completion's eos carry no gradient; every counted row does (A != 0, KL term)
    counted = torch.zeros(B * S, dtype=torch.bool)
    for b, e in enumerate(want_end):
        counted[b * S + S - K - 1: b * S + S - K - 1 + e] = True
    assert torch.equal(_zero_rows(tile_a).cpu(), ~counted), 'two-pass zero rows: prompt, post-eos and last rows'
    _compare_tiles(tile_a, tile_b, f'grpo V={V}')


@pytest.mark.parametrize('dtype,V', [(BF, 32064), (BF, 128257), (F32, 8200), (F32, 65537)])
def test_single_pass_cross_entropy_tile_contract(ops, dtype, V):
    """aa_logprob_ce_fused against K1 (ignore_index) -> -loss_scale / n_valid -> K1b, both into poisoned guarded tiles:
    ignored positions become zero rows in both."""
    gen = torch.Generator().manual_seed(V + 9)
    B, S = 3, 10
    R = B * S
    logits = (torch.randn(R, V, generator=gen) * 2.5).to(dtype).to(DEV)
    labels = torch.randint(0, V, (R,), generator=gen)
    labels[[0, 4, 5, 6, 13, R - 1]] = IGNORE
    labels = labels.to(DEV)
    plan = ops.RowPlan([0], [0], [0], [R], [0], (B, S), R, DEV)
    n_valid = int((labels != IGNORE).sum())
    loss_scale = 0.5
    _status_take()
    # two passes
    lp_a = torch.empty((B, S), dtype=torch.float32, device=DEV)
    stats = torch.empty((2, R), dtype=torch.float32, device=DEV)
    ops._launch_fwd(logits, labels, plan, lp_a, stats[0], stats[1], ignore_index=IGNORE)
    scale = torch.tensor([-loss_scale], dtype=torch.float32) / torch.tensor([float(n_valid)], dtype=torch.float32)
    tile_a = Guarded(R, V, V, dtype)
    ops._launch_bwd(logits, labels, plan, stats[0], stats[1], None, None, scale.to(DEV), tile_a.tile, Lb.MODE_F32,
                    ignore_index=IGNORE)
    # one pass
    lp_b = torch.zeros((B, S), dtype=torch.float32, device=DEV)
    tile_b = Guarded(R, V, V, dtype)
    scratch = torch.empty(R * 6, dtype=torch.int64, device=DEV)
    coeff = torch.empty(1, dtype=torch.float32, device=DEV)
    sc = ops._device_scratch(torch.device(DEV))
    p = plan.ptrs()
    Lb.check(Lb.lib().aa_logprob_ce_fused(
        logits.data_ptr(), Lb.dtype_code(dtype), V, V, labels.data_ptr(), R, IGNORE, plan.n_seg, p[0], p[1], p[2], p[3],
        p[4], R, lp_b.data_ptr(), loss_scale, tile_b.tile.data_ptr(), V, scratch.data_ptr(), coeff.data_ptr(),
        sc['status'].data_ptr(), Lb.stream_ptr(tile_b.buf.device)))
    torch.cuda.synchronize()
    assert _status_take() == 0
    assert_close_f32(lp_b, lp_a, what='log-probs')
    assert bool((lp_b.view(-1)[labels == IGNORE] == 0).all())
    zero = _zero_rows(tile_a)
    assert torch.equal(zero.cpu(), (labels == IGNORE).cpu())
    _compare_tiles(tile_a, tile_b, f'cross-entropy V={V}')
