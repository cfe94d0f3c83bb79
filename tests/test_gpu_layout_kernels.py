"""The layout and bookkeeping kernels pinned through the C ABI on guarded buffers (run on an H100: `pytest -m gpu`).

These kernels decide which rows, positions and labels every loss reads: the device row plan of per-sample response
tails (`aa_tail_plan_build`), the rollout layout (`aa_ppo_rollout_layout`, `aa_move_padding_left`, `aa_count_nonpad`),
the tail gather and its adjoints (`aa_tail_rows` both ways, `aa_tail_scatter_scaled`), DPO's pad-stripped labels
(`aa_strip_pad_tail`), the SimPO / ORPO / KTO pair bookkeeping (`aa_pair_slices`, `aa_slice_sums`) and the hand-over
scaling of a gradient tile (`aa_scale_tile`).  A fault in one of them moves data rather than perturbing it, so every
integer result is held exactly and every float result bit for bit.

Premise.  The references below are plain Python / torch integer code on the CPU that restates the reference trainers'
own expressions: `move_padding_left`, `len(remove_pad(seq)[len(remove_pad(prompt)):])`, `strip_pad(ids)[-R:]`, the
SimPO loop's `nonzero()[0]` / `nonzero()[-1]` after its identical-pair skip, and `pad_sequence` of the tails.
`tests/test_cpu_layout_refs.py` holds them to `oracle/ref_port.py` on the same case matrix.  The shapes pass each loop
that small batches never leave: more than 256 plan segments (the block scan's carry), pad scans across several
256-token windows with the R-th non-pad token on a window boundary, rows longer than one block, several blocks per
row, and more than one grid-stride pass; the plan's strides take its int64 offsets past 2^31.  Pad ids include -1, 0
and 2^40 + 3, and the rows hold ids with the same low 32 bits as the pad, so a 32-bit compare miscounts.

Guarded buffers and fenced inputs come from `test_gpu_loss_kernels.py`.  Outputs sit mid-allocation between guard
bands and start as POISON (NaN for floats, 0x7FA5... / 0xA5 for integers); guards and pad columns hold SENTINEL.
Inputs with a row stride above their width carry a marker in their pad columns and sit between marker rows: NaN for
floats, for ids a value that is neither the pad nor an id of the rows, for masks a nonzero value.  The fences reach
past the largest out-of-contract length used, so a kernel that reads outside its row reads a marker, never outside the
allocation.  Each launch gets its own status word, which must afterwards hold exactly the predicted bits.

Float results.  `aa_slice_sums` is held bit-exact on exact operands (integers times 2^-3 whose partial sums are exact
in fp32 in any order, then the one 16-bit rounding of faithful mode), and to the summation bound / ATen on real
values.  The scatter and `aa_scale_tile` form one fp32 product and round it once, which the float64 reference
reproduces exactly on any operands.

Tail lengths.  Every tail kernel follows one rule: R = clamp(len, 0, row width), and the tail is row columns
[width - R, width - R + bound).  The gathers are checked against `pad_sequence` of the tails, and each adjoint is held
to the exact transpose of its gather through index maps (source column + 1 in every element), for lengths inside
and outside [0, bound].  R = 0 is an empty tail in every kernel, where the reference's `x[-0:]` is the whole row.
"""
import random

import pytest
import torch

from align_anything_b200 import _lib as Lb
from oracle import ref_port as O
from test_gpu_loss_kernels import (BF, CODE, DEV, F16, F32, F32MODE, F64, FAITHFUL, INT, U, Guarded, Words, _sm_count,
                                   _stream, assert_same, assert_within, exact_ints, fenced, fenced_vec, rc_ok, rnd)
from test_gpu_parity import assert_ulp_close, ops  # noqa: F401

gpu = pytest.mark.gpu
I32, I64, U8 = torch.int32, torch.int64, torch.uint8
SHORT, EMPTY, DIVERGE = Lb.STATUS_SHORT_SEQUENCE, Lb.STATUS_EMPTY_MASK, Lb.STATUS_DIVERGE_RANGE
PADS = [-1, 0, 2 ** 40 + 3]
MARK = 777_777_777_777  # the id marker of fence rows and pad columns: no pad and no id of the rows
SEED = 9090


def confuser(pad):
    """An id with the low 32 bits of `pad`: equal to it under an int32 compare."""
    return pad - 2 ** 32 if pad >= 2 ** 32 else pad + 2 ** 32


def _bits(t):
    return t.contiguous().view(INT[t.element_size()]).cpu()


def _what_differs(got, want):
    bad = (got != want).reshape(-1)
    i = int(bad.nonzero()[0]) if bool(bad.any()) else 0
    return f'{int(bad.sum())} of {want.numel()} differ, first at flat {i}: got {got.reshape(-1)[i]}, want {want.reshape(-1)[i]}'


def assert_equal_ints(got, want, what):
    got, want = got.cpu().long(), want.cpu().long()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    assert torch.equal(got, want), f'{what}: {_what_differs(got, want)}'


# ---- references (CPU, Python integers) -------------------------------------------------------------------------------
def plan_hi(seq, ltl, rsh):
    return seq + rsh if ltl <= 0 else min(seq + rsh, ltl)


def ref_plan(lens, B, seq, sb, sl, lab_stride, ltl, lsh, rsh, width, copies, cld, cod):
    """aa_tail_plan_build's table [5][S + 1] (logit_off, label_off, out_off, cum, tile_row) and whether a length was
    outside [0, hi] (clamped)."""
    S = B * copies
    hi = plan_hi(seq, ltl, rsh)
    t = [[0] * (S + 1) for _ in range(5)]
    short, cum = False, 0
    for seg in range(S):
        c, b = divmod(seg, B)
        r = lens[b]
        if not 0 <= r <= hi:
            short, r = True, max(0, min(r, hi))
        first = seq - r + rsh
        t[0][seg] = b * sb + first * sl + c * cld
        t[1][seg] = b * lab_stride + (ltl - r if ltl > 0 else 0) + lsh
        t[2][seg] = b * width + c * cod
        t[3][seg] = cum
        t[4][seg] = (c * B + b) * seq + first
        cum += max(min(r - lsh, width), 0)
    t[3][S] = cum
    return torch.tensor(t, dtype=I64), short


def ref_rollout(prompt, seq, pad):
    """moved = move_padding_left(seq), mask = moved != pad, lens = len(remove_pad(seq)[len(remove_pad(prompt)):]),
    counts = len(remove_pad(seq))."""
    moved = O.move_padding_left(seq, pad)
    lens, counts = [], []
    for b in range(seq.size(0)):
        kept = seq[b][seq[b] != pad]
        lens.append(len(kept[len(prompt[b][prompt[b] != pad]):]))
        counts.append(len(kept))
    return moved, moved != pad, torch.tensor(lens), torch.tensor(counts)


def ref_strip(row, R, pad, strip):
    """strip_pad(ids)[-R:] (strip) or ids[-R:] (plain tail) for R > 0, filled with -1 in front where the row holds
    fewer than R tokens (the kernel's answer to a shape the reference cannot form); nothing for R <= 0."""
    if R <= 0:
        return row[:0]
    kept = row[row != pad] if strip else row
    tail = kept[-R:]
    return torch.cat([torch.full((R - len(tail),), -1, dtype=I64), tail])


def ref_pairs(ids, mask, n):
    """The SimPO / ORPO / KTO loop per pair: identical id rows are skipped before the masks are read; otherwise
    `nonzero()[-1]` of an empty mask raises (EMPTY_MASK) and the range asserts fail (DIVERGE_RANGE).  -> int32 [4][n]
    (valid, diverge, end_better, end_worse: the kernel writes both ends for every pair, -1 for an empty mask row), bits."""
    out = torch.zeros(4, n, dtype=I32)
    bits = 0
    for i in range(n):
        a, b = ids[i], ids[n + i]
        nz_b, nz_w = mask[i].nonzero(), mask[n + i].nonzero()
        end_b = int(nz_b[-1]) if len(nz_b) else -1
        end_w = int(nz_w[-1]) if len(nz_w) else -1
        out[2, i], out[3, i] = end_b, end_w
        if torch.all(torch.eq(a, b)):
            continue
        d = int((a != b).nonzero()[0])
        out[0, i], out[1, i] = 1, d
        if end_b < 0 or end_w < 0:
            bits |= EMPTY
        elif not (0 <= d <= end_b and 0 <= d <= end_w):
            bits |= DIVERGE
    return out, bits


def ref_slice_sums(lp64, slices, n, rd):
    """sums[r] = sum(lp[r, diverge : end + 1]) with Python slice semantics on the (2n, W) rows, one rounding (fp32,
    then rd in faithful 16-bit mode); the sums themselves are exact on exact operands."""
    s = []
    for r in range(2 * n):
        i = r % n
        lo, end = int(slices[1, i]), int(slices[2 if r < n else 3, i])
        s.append(lp64[r, lo:end + 1].sum())
    return rnd(torch.stack(s), rd)


def tail_span(r, width, bound):
    """The tail rule: (first column, count) of the tail of a width-`width` row for length r."""
    R = max(0, min(r, width))
    return width - R, min(R, bound)


def ref_tail_gather(x, lens, bound):
    """pad_sequence([x[b][-R_b:] for b]) cut / padded to `bound` columns, under the tail rule (R = 0: empty)."""
    out = torch.zeros(x.size(0), bound, dtype=x.dtype)
    for b, r in enumerate(lens):
        off, n = tail_span(r, x.size(1), bound)
        out[b, :n] = x[b, off:off + n]
    return out


def ref_tail_scatter(g, lens, width):
    """The adjoint of ref_tail_gather: g (B, bound) placed back on the tail columns of (B, width) zero rows."""
    out = torch.zeros(g.size(0), width, dtype=g.dtype)
    for b, r in enumerate(lens):
        off, n = tail_span(r, width, g.size(1))
        out[b, off:off + n] = g[b, :n]
    return out


# ---- case matrix (shared with the CPU file) --------------------------------------------------------------------------
PLAN_B = [1, 255, 256, 257, 1000]
# seq, row stride, sample stride, label row stride, label tail length, label shift, row shift, width
PLAN_LAYOUTS = {
    'trainer': (37, 1031, 37 * 1031, 40, 40, 0, -1, 20),  # ops.device_tail_plan's form: the last seq - 1 rows
    'shift1': (64, 515, 64 * 515 + 3, 70, 0, 1, 1, 64),  # no label tail, both shifts 1
    'shift0': (33, 8, 300, 33, 33, 1, 0, 7),  # label shift 1, row shift 0, width below most lengths
    'past2^31': (32768, 152064, 32768 * 152064, 32768, 32768, 0, -1, 4096),  # b * sample_stride > 2^31 from b = 1
}


def plan_lens(B, layout, kind):
    """Per-sample lengths: inside [0, hi] (0 and hi included), or with -1, hi + 1 and the int32 extremes mixed in."""
    seq, _, _, _, ltl, _, rsh, _ = PLAN_LAYOUTS[layout]
    hi = plan_hi(seq, ltl, rsh)
    g = random.Random(B * 31 + seq)
    lens = [g.randint(0, hi) for _ in range(B)]
    lens[0] = hi
    lens[B // 2] = 0 if B > 1 else lens[B // 2]
    if kind == 'out':
        bad = [hi + 1, -1, 2 ** 31 - 1, -2 ** 31]
        for k, v in enumerate(bad[:max(1, B // 2)]):
            lens[(1 + 3 * k) % B] = v
    return lens


ROLL_L = [1, 255, 256, 257, 4097]


def id_rows(B, L, pad, seed):
    """(B, L) int64 id rows, each of a different kind: pads left, inside and right; all pad; no pad; left pads only;
    right pads only; scattered pads.  One id in ten has the pad's low 32 bits."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(5, 1000, (B, L), generator=g)
    ids[torch.rand(B, L, generator=g) < 0.1] = confuser(pad)
    for b in range(B):
        row, k = ids[b], b % 6
        if k == 0:
            a, z = L // 5, L - L // 7
            row[:a] = pad
            row[z:] = pad
            row[a + 1:z:3] = pad
        elif k == 1:
            row[:] = pad
        elif k == 3:
            row[:L // 2 + 1] = pad
        elif k == 4:
            row[L - L // 3 - 1:] = pad
        elif k == 5:
            row[torch.rand(L, generator=g) < 0.4] = pad
    return ids


STRIP_L = [1, 255, 256, 257, 600, 4097]


def strip_cases(L, pad, strip, seed):
    """Samples (ids rows, R) of two groups: 'fit' (every R within the row's tokens; no status) and 'short' (every R
    beyond them).  With strip, the R-th non-pad token from the right sits exactly on each 256-token window boundary of
    the right-to-left scan and one token either side of it."""
    g = torch.Generator().manual_seed(seed)

    def row():  # its first token is never the pad
        r = torch.randint(5, 1000, (L,), generator=g)
        r[torch.rand(L, generator=g) < 0.1] = confuser(pad)
        r[torch.rand(L, generator=g) < 0.3] = pad
        r[0] = 9
        return r

    fit, short = [], []
    if strip:
        for w in range(1, (L - 1) // 256 + 1):
            q = L - 256 * w  # the lowest position of the scan's window w - 1
            for d in (-1, 0, 1):
                if 0 <= q + d < L:
                    r = row()
                    r[q + d] = 7
                    fit.append((r, int((r[q + d:] != pad).sum())))
        r = row()
        cnt = int((r != pad).sum())
        fit += [(r, cnt), (row(), 1), (row(), 0), (row(), -2)]
        if cnt:
            fit.append((r, max(1, cnt // 2)))
        short += [(r, cnt + 3), (torch.full((L,), pad, dtype=I64), 2), (row(), L + 1)]
    else:
        fit += [(row(), 1), (row(), L), (row(), max(1, L // 2)), (row(), 0), (row(), -1)]
        short += [(row(), L + 1), (row(), L + 300)]
    return {'fit': fit, 'short': short}


PAIR_L = [2, 255, 256, 257, 1000, 4097]
PAIR_GROUPS = {'clean': 0, 'identical': 0, 'empty_mask': EMPTY, 'range_better': DIVERGE, 'range_worse': DIVERGE}


def pair_cases(L, group, seed):
    """(ids (2n, L), mask (2n, L) bool) for one group of pairs.  clean: divergence at 0, at L - 1 and inside, and an
    identical pair with full masks; identical: identical pairs with one or both mask rows empty (no status: the
    reference skips them before reading the masks); empty_mask: valid pairs with an empty mask row; range_*: the
    divergence past one row's last attended position."""
    g = torch.Generator().manual_seed(seed)
    rnd_int = lambda lo, hi: int(torch.randint(lo, hi + 1, (1,), generator=g))  # noqa: E731
    pairs = []

    def pair(div, end_b, end_w):
        a = torch.randint(5, 1000, (L,), generator=g)
        b = a.clone()
        if div is not None:
            b[div] = a[div] + 1
            b[div + 1:] = torch.randint(5, 1000, (L - div - 1,), generator=g)
        ma, mb = torch.zeros(L, dtype=torch.bool), torch.zeros(L, dtype=torch.bool)
        for m, e in ((ma, end_b), (mb, end_w)):
            if e >= 0:
                m[:e + 1] = torch.rand(e + 1, generator=g) < 0.7
                m[e] = True
        pairs.append((a, b, ma, mb))

    if group == 'clean':
        pair(0, rnd_int(0, L - 1), rnd_int(0, L - 1))
        pair(L - 1, L - 1, L - 1)
        d = rnd_int(0, L - 1)
        pair(d, rnd_int(d, L - 1), rnd_int(d, L - 1))
        pair(None, rnd_int(0, L - 1), rnd_int(0, L - 1))
    elif group == 'identical':
        pair(None, -1, rnd_int(0, L - 1))
        pair(None, rnd_int(0, L - 1), -1)
        pair(None, -1, -1)
    elif group == 'empty_mask':
        pair(0, -1, L - 1)
        pair(L - 1, L - 1, -1)
    elif group == 'range_better':
        pair(L - 1, L - 2 if L > 1 else -1, L - 1)
    else:
        pair(L - 1, L - 1, L - 2 if L > 1 else -1)
    n = len(pairs)
    ids = torch.stack([p[0] for p in pairs] + [p[1] for p in pairs])
    mask = torch.stack([p[2] for p in pairs] + [p[3] for p in pairs])
    return ids, mask, n


SS_W = [1, 127, 128, 129, 4097]
SS_N = 6


def slice_table(W, seed):
    """int32 [4][6] (valid, lo, end_better, end_worse): a full row, end = -1, lo > hi, ends past W, an invalid pair
    (the kernel sums it all the same: `valid` is for the caller), and a random range."""
    g = random.Random(seed)
    lo = [0, 0, min(W - 1, 3), 1, 0, g.randint(0, W - 1)]
    eb = [W - 1, -1, max(0, min(W - 1, 3) - 3), W + 6, W - 1, g.randint(lo[5], W - 1)]
    ew = [W - 1, W - 1, -1, W + 2, 0, g.randint(-1, W - 1)]
    valid = [1, 1, 1, 1, 0, 1]
    return torch.tensor([valid, lo, eb, ew], dtype=I32)


def slice_operands(W, seed, device='cpu'):
    """(2n, W) non-positive integers times 2^-3, |x| <= 8: 2 * 4097 * 64 units of 2^-3 bound every partial sum."""
    return exact_ints((2 * SS_N, W), 8, -3, seed, device, nonpos=True)


TAIL_W = [1, 255, 256, 257, 4097]
TAIL_B = 8


def tail_bounds(W):
    return sorted({W, (W + 1) // 2})


def tail_lens(W, bound, kind):
    """Eight lengths.  in: 0, 1, bound and values inside [0, bound]; out: -3, bound + 5 and W + 7 mixed in (the guards
    reach past W + 7)."""
    g = random.Random(W * 13 + bound)
    lens = [0, 1, bound, bound // 2] + [g.randint(0, bound) for _ in range(TAIL_B - 4)]
    if kind == 'out':
        lens[1], lens[4], lens[6] = -3, bound + 5, W + 7
    return lens


SCATTER_CASES = [(W, src) for W in TAIL_W for src in (W, W + 9)]


def scatter_lens(W, src, kind):
    g = random.Random(W * 7 + src)
    top = min(W, src)
    lens = [0, 1, top, top // 2] + [g.randint(0, top) for _ in range(TAIL_B - 4)]
    if kind == 'out':
        lens[1], lens[4], lens[6] = -3, W + 5, src + 7
    return lens


# ---- aa_tail_plan_build ----------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('layout', list(PLAN_LAYOUTS))
@pytest.mark.parametrize('copies', [1, 2])
@pytest.mark.parametrize('B', PLAN_B)
def test_tail_plan_build(ops, B, copies, layout):
    """The whole [5][S + 1] table (the cum[S] total and the zero column included) for S = B * copies segments, the
    second copy above and below the first, lengths inside and outside [0, hi], with and without a status word."""
    seq, sl, sb, lab_stride, ltl, lsh, rsh, width = PLAN_LAYOUTS[layout]
    S = B * copies
    for kind in ('in', 'out'):
        lens = plan_lens(B, layout, kind)
        ln = fenced_vec(torch.tensor(lens, dtype=I32))
        for cld in ((0,) if copies == 1 else (B * sb + 4096, -(B * sb + 4096))):
            cod = B * width
            want, short = ref_plan(lens, B, seq, sb, sl, lab_stride, ltl, lsh, rsh, width, copies, cld, cod)
            assert short == (kind == 'out')
            for with_status in (True, False):
                what = f'plan B={B} copies={copies} {layout} lens={kind} delta={cld} status={with_status}'
                table = Guarded(5, S + 1, I64)
                status = Words()
                rc_ok(Lb.lib().aa_tail_plan_build(ln.data_ptr(), B, seq, sb, sl, lab_stride, ltl, lsh, rsh, width,
                                                  copies, cld, cod, table.ptr(), status.ptr() if with_status else None,
                                                  _stream()), what)
                torch.cuda.synchronize()
                table.check(what)
                status.check([SHORT if short and with_status else 0], what + ' status')
                assert_equal_ints(table.t, want, what)


# ---- rollout layout --------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('P', ROLL_L)
@pytest.mark.parametrize('L', ROLL_L)
def test_ppo_rollout_layout(ops, L, P):
    """moved sequences, attention mask and response lengths for 7 rows of different kinds, each pad id."""
    B = 7
    for pad in PADS:
        what = f'rollout L={L} P={P} pad={pad}'
        seq64 = id_rows(B, L, pad, SEED + L)
        prompt64 = id_rows(B, P, pad, SEED + 3 * P + 1)[torch.arange(B).roll(2)]  # another kind per row
        want_moved, want_mask, want_lens, _ = ref_rollout(prompt64, seq64, pad)
        seq, prompt = fenced(seq64, L + 3, pad=MARK), fenced(prompt64, P + 2, pad=MARK)
        moved, mask, lens = Guarded(B, L, I64), Guarded(B, L, U8), Guarded(B, 1, I32)
        rc_ok(Lb.lib().aa_ppo_rollout_layout(prompt.data_ptr(), P, P + 2, seq.data_ptr(), L, L + 3, B, pad, moved.ptr(),
                                             mask.ptr(), lens.ptr(), _stream()), what)
        torch.cuda.synchronize()
        for name, buf in (('moved', moved), ('mask', mask), ('lens', lens)):
            buf.check(f'{what} {name}')
        assert_equal_ints(moved.t, want_moved, what + ' moved')
        assert_equal_ints(mask.t, want_mask, what + ' mask')
        assert_equal_ints(lens.t[:, 0], want_lens, what + ' response lens')


@gpu
@pytest.mark.parametrize('L', ROLL_L)
def test_move_padding_left_and_count_nonpad(ops, L):
    B = 7
    for pad in PADS:
        what = f'move_padding_left / count_nonpad L={L} pad={pad}'
        seq64 = id_rows(B, L, pad, SEED + 5 * L)
        want_moved, _, _, want_counts = ref_rollout(seq64[:, :1], seq64, pad)
        seq = fenced(seq64, L + 5, pad=MARK)
        out, counts = Guarded(B, L, I64), Guarded(B, 1, I32)
        rc_ok(Lb.lib().aa_move_padding_left(seq.data_ptr(), B, L, L + 5, pad, out.ptr(), _stream()), what)
        rc_ok(Lb.lib().aa_count_nonpad(seq.data_ptr(), B, L, L + 5, pad, counts.ptr(), _stream()), what)
        torch.cuda.synchronize()
        out.check(what + ' moved')
        counts.check(what + ' counts')
        assert_equal_ints(out.t, want_moved, what + ' moved')
        assert_equal_ints(counts.t[:, 0], want_counts, what + ' counts')


# ---- aa_strip_pad_tail -----------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('strip', [1, 0])
@pytest.mark.parametrize('L', STRIP_L)
def test_strip_pad_tail(ops, L, strip):
    """Labels of each sample into rows of out_stride > max R: the first R columns written, the rest left alone."""
    for pad in PADS:
        for group, samples in strip_cases(L, pad, strip, SEED + L + pad % 97).items():
            what = f'strip_pad_tail L={L} strip={strip} pad={pad} {group}'
            n = len(samples)
            ids = fenced(torch.stack([s[0] for s in samples]), L + 5, pad=MARK)
            Rs = [s[1] for s in samples]
            lens = fenced_vec(torch.tensor(Rs, dtype=I32))
            wout = max(max(Rs), 1) + 3
            out = Guarded(n, wout, I64)
            status = Words()
            rc_ok(Lb.lib().aa_strip_pad_tail(ids.data_ptr(), n, L, L + 5, pad, strip, lens.data_ptr(), out.ptr(),
                                             wout, status.ptr(), _stream()), what)
            torch.cuda.synchronize()
            status.check([SHORT if group == 'short' else 0], what + ' status')
            written = torch.arange(wout)[None, :] < torch.tensor(Rs)[:, None]
            out.check(what, written)
            for i, (row, R) in enumerate(samples):
                assert_equal_ints(out.t[i, :max(R, 0)], ref_strip(row, R, pad, strip), f'{what} sample {i} R={R}')


# ---- aa_pair_slices --------------------------------------------------------------------------------------------------
def _pair_launch(L, group, mkind):
    ids64, mask, n = pair_cases(L, group, SEED + L + len(group))
    want, bits = ref_pairs(ids64, mask, n)
    assert bits == PAIR_GROUPS[group], (group, bits)
    what = f'pair_slices L={L} {group} mask={mkind}'
    ids = fenced(ids64, L + 2, pad=MARK)
    if mkind == 'u8':
        mt = fenced(mask.to(U8) * torch.where(torch.arange(L) % 2 == 0, 1, 255).to(U8), L + 4, pad=1)
        code = Lb.MASK_U8
    else:  # nonzero int64 values whose low 32 bits are zero count as attended
        mt = fenced(mask.to(I64) * torch.where(torch.arange(L) % 2 == 0, 1, 2 ** 32), L + 4, pad=1)
        code = Lb.MASK_I64
    out = Guarded(4, n, I32)
    status = Words()
    rc_ok(Lb.lib().aa_pair_slices(ids.data_ptr(), L + 2, mt.data_ptr(), code, L + 4, n, L, out.ptr(), status.ptr(),
                                  _stream()), what)
    torch.cuda.synchronize()
    out.check(what)
    status.check([bits], what + ' status')
    assert_equal_ints(out.t, want, what)


@gpu
@pytest.mark.parametrize('mkind', ['u8', 'i64'])
@pytest.mark.parametrize('L', PAIR_L)
def test_pair_slices(ops, L, mkind):
    for group in ('clean', 'empty_mask', 'range_better', 'range_worse'):
        _pair_launch(L, group, mkind)


@gpu
@pytest.mark.parametrize('mkind', ['u8', 'i64'])
@pytest.mark.parametrize('L', PAIR_L)
def test_pair_slices_identical_pairs(ops, L, mkind):
    """Identical pairs with empty mask rows raise nothing: the reference skips them before it reads the masks."""
    _pair_launch(L, 'identical', mkind)


# ---- aa_slice_sums ---------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('W', SS_W)
def test_slice_sums(ops, W):
    slices = slice_table(W, SEED + W)
    sl = fenced_vec(slices.reshape(-1))
    lp64 = slice_operands(W, SEED + 2 * W)
    for dt in (BF, F16, F32):
        lp = fenced(lp64.to(dt), W + 3, reach=W + 8)
        for mode in (FAITHFUL, F32MODE):
            rd = dt if mode == FAITHFUL and dt != F32 else None
            what = f'slice_sums W={W} {dt} mode={mode}'
            sums = Guarded(1, 2 * SS_N, F32)
            rc_ok(Lb.lib().aa_slice_sums(lp.data_ptr(), CODE[dt], W + 3, SS_N, W, sl.data_ptr(), mode, sums.ptr(),
                                         _stream()), what)
            torch.cuda.synchronize()
            sums.check(what)
            assert_same(sums.t[0], ref_slice_sums(lp64.cpu(), slices, SS_N, rd), what)


@gpu
@pytest.mark.parametrize('W', SS_W)
def test_slice_sums_real_values(ops, W):
    """Real-valued log-probs: f32 mode within the summation bound of float64, faithful mode against ATen's sum of the
    same slice in the 16-bit dtype (<= 1 ulp)."""
    slices = slice_table(W, SEED + W)
    sl = fenced_vec(slices.reshape(-1))
    gen = torch.Generator(device=DEV).manual_seed(W)
    base = -3 * torch.rand(2 * SS_N, W, generator=gen, device=DEV, dtype=F64)
    for dt in (BF, F16, F32):
        lp = fenced(base.to(dt), W + 3, reach=W + 8)
        for mode in (FAITHFUL, F32MODE):
            what = f'slice_sums real W={W} {dt} mode={mode}'
            sums = Guarded(1, 2 * SS_N, F32)
            rc_ok(Lb.lib().aa_slice_sums(lp.data_ptr(), CODE[dt], W + 3, SS_N, W, sl.data_ptr(), mode, sums.ptr(),
                                         _stream()), what)
            torch.cuda.synchronize()
            sums.check(what)
            rows = [(r, int(slices[1, r % SS_N]), int(slices[2 if r < SS_N else 3, r % SS_N]) + 1) for r in range(2 * SS_N)]
            if mode == FAITHFUL and dt != F32:
                want = torch.stack([lp[r, lo:hi].sum() for r, lo, hi in rows])
                assert_ulp_close(sums.t[0].to(dt), want, max_ulp=1, min_exact=0.9, what=what)
            else:
                x = lp.double()
                want = torch.stack([x[r, lo:hi].sum() for r, lo, hi in rows])
                mag = torch.stack([x[r, lo:hi].abs().sum() for r, lo, hi in rows])
                assert_within(sums.t[0], want, (W * U * mag).cpu() + 1e-30, what)


# ---- aa_tail_rows ----------------------------------------------------------------------------------------------------
def _tail_rows_call(src, dt, src_stride, lens, W, bound, out, out_stride, adjoint):
    return Lb.lib().aa_tail_rows(src.data_ptr(), CODE[dt], src_stride, lens.data_ptr(), TAIL_B, W, bound, out.ptr(),
                                 out_stride, adjoint, _stream())


def _tail_rows_check(W, kind):
    gen = torch.Generator(device=DEV).manual_seed(W)
    for bound in tail_bounds(W):
        lens = tail_lens(W, bound, kind)
        ln = fenced_vec(torch.tensor(lens, dtype=I32))
        for dt in (BF, F16, F32):
            what = f'tail_rows W={W} bound={bound} lens={kind} {dt}'
            x = torch.randn(TAIL_B, W, generator=gen, device=DEV).to(dt)
            src = fenced(x, W + 5, reach=W + 8)
            out = Guarded(TAIL_B, bound, dt, pitch=bound + 3)
            rc_ok(_tail_rows_call(src, dt, W + 5, ln, W, bound, out, bound + 3, 0), what)
            g = torch.randn(TAIL_B, bound, generator=gen, device=DEV).to(dt)
            gsrc = fenced(g, bound + 2, reach=W + 8)
            back = Guarded(TAIL_B, W, dt, pitch=W + 4)
            rc_ok(_tail_rows_call(gsrc, dt, bound + 2, ln, W, bound, back, W + 4, 1), what + ' adjoint')
            torch.cuda.synchronize()
            out.check(what)
            back.check(what + ' adjoint')
            assert torch.equal(_bits(out.t), _bits(ref_tail_gather(x.cpu(), lens, bound))), what
            assert torch.equal(_bits(back.t), _bits(ref_tail_scatter(g.cpu(), lens, W))), what + ' adjoint'


@gpu
@pytest.mark.parametrize('W', TAIL_W)
def test_tail_rows(ops, W):
    """Lengths 0, 1, bound and inside [0, bound]: the gather bit-equal to pad_sequence of the tails, the scatter to
    its adjoint; pitched outputs, several blocks per row at W = 4097."""
    _tail_rows_check(W, 'in')


@gpu
@pytest.mark.parametrize('W', TAIL_W)
def test_tail_rows_out_of_contract(ops, W):
    """Lengths -3, bound + 5 and W + 7 follow the tail rule in both directions, inside row b."""
    _tail_rows_check(W, 'out')


# ---- aa_tail_scatter_scaled ------------------------------------------------------------------------------------------
SCALES = [(F32, -0.75), (BF, -0.75), (F16, 3.0), (None, None)]


def _scatter_check(W, src, kind):
    gen = torch.Generator(device=DEV).manual_seed(W + src)
    lens = scatter_lens(W, src, kind)
    ln = fenced_vec(torch.tensor(lens, dtype=I32))
    for dt in (BF, F16, F32):
        g = torch.randn(TAIL_B, W, generator=gen, device=DEV).to(dt)
        gin = fenced(g, W + 2, reach=src + 8)
        for sdt, s in SCALES:
            for ow in sorted({src, src + 1}):
                what = f'tail_scatter W={W} src={src} out_width={ow} lens={kind} {dt} scale={sdt}'
                sc = fenced_vec(torch.tensor([s], dtype=sdt)) if sdt is not None else None
                out = Guarded(TAIL_B, ow, dt, pitch=ow + 3)
                rc_ok(Lb.lib().aa_tail_scatter_scaled(gin.data_ptr(), CODE[dt], W + 2, ln.data_ptr(), TAIL_B, W, src,
                                                      Lb.ptr(sc), CODE[sdt] if sdt else 0, out.ptr(), ow + 3, ow,
                                                      _stream()), what)
                torch.cuda.synchronize()
                out.check(what)
                gs = g.cpu() if s is None else (g.cpu().double() * float(torch.tensor(s, dtype=sdt))).float().to(dt)
                want = torch.zeros(TAIL_B, ow, dtype=dt)
                want[:, :src] = ref_tail_scatter(gs, lens, src)
                assert torch.equal(_bits(out.t), _bits(want)), what


@gpu
@pytest.mark.parametrize('W,src', SCATTER_CASES)
def test_tail_scatter_scaled(ops, W, src):
    """The critic's gradient scatter: each scale dtype and none, one fp32 product rounded once, zeros elsewhere."""
    _scatter_check(W, src, 'in')


@gpu
@pytest.mark.parametrize('W,src', SCATTER_CASES)
def test_tail_scatter_scaled_out_of_contract(ops, W, src):
    _scatter_check(W, src, 'out')


# ---- the adjoints are transposes -------------------------------------------------------------------------------------
def _index_map(bits, limit):
    """Element bits holding (source column + 1), 0 for a zero fill -> source column, -1 for none; all must be < limit."""
    m = bits.long() - 1
    assert bool(((m >= -1) & (m < limit)).all()), f'an element came from outside the row: {m.max()}'
    return m


def _assert_transpose(fwd, adj, what):
    """fwd[b, k] = j  <=>  adj[b, j] = k, for every gathered k and every written j."""
    for b in range(fwd.size(0)):
        pairs_f = {(k, int(j)) for k, j in enumerate(fwd[b].tolist()) if j >= 0}
        pairs_a = {(int(k), j) for j, k in enumerate(adj[b].tolist()) if k >= 0}
        assert pairs_f == pairs_a, f'{what} row {b}: gather {sorted(pairs_f)[:6]}... adjoint {sorted(pairs_a)[:6]}...'


@gpu
@pytest.mark.parametrize('W', TAIL_W)
def test_tail_rows_adjoint_is_transpose(ops, W):
    """`aa_tail_rows` forward on rows whose elements hold their column + 1 (bit patterns of each dtype: the kernel
    copies bits) gives the gather's source map; the adjoint on rows holding k + 1 gives the scatter's.  The two maps
    are transposes of each other, for lengths inside and outside the contract."""
    for bound in tail_bounds(W):
        lens = tail_lens(W, bound, 'out')[:5] + tail_lens(W, bound, 'in')[1:4]
        ln = fenced_vec(torch.tensor(lens, dtype=I32))
        for dt in (BF, F16, F32):
            what = f'transpose tail_rows W={W} bound={bound} {dt}'
            it = INT[torch.empty(0, dtype=dt).element_size()]
            cols = (torch.arange(W, device=DEV) + 1).to(it).expand(TAIL_B, W).contiguous().view(dt)
            ks = (torch.arange(bound, device=DEV) + 1).to(it).expand(TAIL_B, bound).contiguous().view(dt)
            src, gsrc = fenced(cols, W + 5, reach=W + 8), fenced(ks, bound + 2, reach=W + 8)
            out, back = Guarded(TAIL_B, bound, dt), Guarded(TAIL_B, W, dt)
            rc_ok(_tail_rows_call(src, dt, W + 5, ln, W, bound, out, bound, 0), what)
            rc_ok(_tail_rows_call(gsrc, dt, bound + 2, ln, W, bound, back, W, 1), what + ' adjoint')
            torch.cuda.synchronize()
            out.check(what)
            back.check(what + ' adjoint')
            _assert_transpose(_index_map(_bits(out.t), W), _index_map(_bits(back.t), bound), what)


CRITIC_MAP = [(1, 1), (1, 10), (256, 256), (256, 265), (256, 4097)]


@gpu
@pytest.mark.parametrize('Wm,src', CRITIC_MAP)
def test_critic_tail_load_adjoint_is_transpose(ops, Wm, src):
    """The critic's tail load (`aa_ppo_critic_loss` with `value_tail_lens`) against `aa_tail_scatter_scaled`.  With
    returns and old values 0, clip 0 and a full mask, d loss / d value = x / (B * Wm) exactly (B * Wm a power of two), so
    raw values holding column + 1 turn the gradient into the load's source map; the scatter of g must put g[b, t] on
    exactly that column, and nothing anywhere else."""
    B = TAIL_B
    lens = [0, 1, Wm, Wm // 2, -3, Wm + 5, src + 7, src]
    ln = fenced_vec(torch.tensor(lens, dtype=I32))
    raw = fenced((torch.arange(src, device=DEV, dtype=F32) + 1).expand(B, src), src + 3, reach=src + 8)
    zeros = fenced(torch.zeros(B, Wm, device=DEV), Wm + 1)
    mask = fenced(torch.ones(B, Wm, dtype=U8), Wm + 2, pad=1)
    grad, loss, rows = Guarded(B, Wm, F32), Guarded(1, 2, F32), Guarded(B, 1, F32)
    counter = Words()
    what = f'transpose critic Wm={Wm} src={src}'
    rc_ok(Lb.lib().aa_ppo_critic_loss(raw.data_ptr(), src + 3, zeros.data_ptr(), Wm + 1, CODE[F32], zeros.data_ptr(),
                                      Wm + 1, CODE[F32], mask.data_ptr(), Wm + 2, B, Wm, 0.0, F32MODE, loss.ptr(),
                                      grad.ptr(), Wm, None, rows.ptr(), counter.ptr(), ln.data_ptr(), src, _stream()),
          what)
    g = torch.randn(B, Wm, generator=torch.Generator(device=DEV).manual_seed(Wm + src), device=DEV)
    gin = fenced(g, Wm + 2, reach=src + 8)
    out = Guarded(B, src, F32)
    rc_ok(Lb.lib().aa_tail_scatter_scaled(gin.data_ptr(), CODE[F32], Wm + 2, ln.data_ptr(), B, Wm, src, None, 0,
                                          out.ptr(), src, src, _stream()), what + ' scatter')
    torch.cuda.synchronize()
    counter.check([0], what + ' counter')
    grad.check(what + ' grad')
    out.check(what + ' scatter')
    fmap = grad.t.double().cpu() * (B * Wm)
    assert torch.equal(fmap, fmap.round()), what + ' the gradient is not an index map'
    fmap = _index_map(fmap.long(), src)
    want = torch.zeros(B, src)
    gc = g.cpu()
    for b in range(B):
        for t in range(Wm):
            if fmap[b, t] >= 0:
                assert want[b, fmap[b, t]] == 0, what + ' two positions load one column'
                want[b, fmap[b, t]] = gc[b, t]
    assert torch.equal(_bits(out.t), _bits(want)), f'{what}: scatter is not the transpose of the load'
    rule = ref_tail_gather((torch.arange(src) + 1).expand(B, src), lens, Wm) - 1
    assert_equal_ints(fmap, rule, what + ' load vs the tail rule')


# ---- aa_scale_tile ---------------------------------------------------------------------------------------------------
def _specials(dt):
    """NaN payloads (quiet, signalling, negative), infinities, signed zeros and a subnormal, as bit patterns."""
    if dt == F32:
        return [0x7FC00001, 0x7F800ABC, 0xFFC12345, 0x7F800000, 0xFF800000, 0x0, 0x80000000, 0x00000003]
    if dt == BF:
        return [0x7FC1, 0x7F81, 0xFFA5, 0x7F80, 0xFF80, 0x0, 0x8000, 0x0003]
    return [0x7E01, 0x7C11, 0xFE5A, 0x7C00, 0xFC00, 0x0, 0x8000, 0x0003]


def _scale_case(dt, n, mis, s, sdt, gen):
    esz = torch.empty(0, dtype=dt).element_size()
    it = INT[esz]
    buf = Guarded(1, mis + n + 16 // esz, dt)
    x = (torch.randn(n, generator=gen, device=DEV) * 3).to(dt)
    sp = torch.tensor(_specials(dt), dtype=torch.int64)
    sp = (sp - (1 << (8 * esz)) * (sp >= (1 << (8 * esz - 1)))).to(it).to(DEV).view(dt)
    k = min(n, sp.numel())
    if k:
        idx = torch.randperm(n, generator=torch.Generator().manual_seed(n + mis))[:k].to(DEV)
        keep = sp[:k] if s == 1.0 else sp[3:3 + k]  # a product's NaN payload is not pinned: no NaN when s != 1
        x[idx[:keep.numel()]] = keep
    buf.t[0, mis:mis + n] = x
    before = buf.bits.clone()
    sc = fenced_vec(torch.tensor([s], dtype=sdt))
    what = f'scale_tile {dt} n={n} misalign={mis} scale={s} ({sdt})'
    rc_ok(Lb.lib().aa_scale_tile(buf.ptr() + mis * esz, CODE[dt], n, sc.data_ptr(), CODE[sdt], _stream()), what)
    torch.cuda.synchronize()
    want = before.clone()
    if s != 1.0:
        prod = (x.cpu().float() * torch.tensor(s, dtype=sdt).float()).to(dt)
        want[buf.pre + mis:buf.pre + mis + n] = prod.view(it).to(DEV)
    assert torch.equal(buf.bits, want), f'{what}: {_what_differs(buf.bits.cpu(), want.cpu())}'


@gpu
@pytest.mark.parametrize('dt', [BF, F16, F32])
def test_scale_tile(ops, dt):
    """n in {0, 1, E - 1, E, E + 1, 3E + 5} at every start misalignment (the head, the body and the scalar tail);
    scale 1 leaves every bit alone, NaN payloads included; another scale equals the fp32 product rounded once to the
    tile dtype; every element outside the tile keeps its bits."""
    E = 16 // torch.empty(0, dtype=dt).element_size()
    gen = torch.Generator(device=DEV).manual_seed(E)
    sdts = [F32, BF, F16]
    for n in (0, 1, E - 1, E, E + 1, 3 * E + 5):
        for mis in range(E):
            for s in (1.0, -0.75):
                _scale_case(dt, n, mis, s, sdts[(n + mis) % 3], gen)


@gpu
@pytest.mark.parametrize('dt', [BF, F16, F32])
def test_scale_tile_grid_stride(ops, dt):
    """A body of more than 2 * 8 * SMs * 256 vectors: every thread takes more than one grid-stride pass."""
    E = 16 // torch.empty(0, dtype=dt).element_size()
    n = E * (2 * 8 * _sm_count() * 256 + 3) + E - 1
    gen = torch.Generator(device=DEV).manual_seed(n)
    for mis in (0, E - 1):
        _scale_case(dt, n, mis, 0.5 if dt == F32 else -0.75, F32, gen)
        _scale_case(dt, n, mis, 1.0, BF, gen)
