"""No GPU: the integer references of `test_gpu_layout_kernels.py` against the reference's own expressions as ported in
`oracle/ref_port.py`, on the GPU file's case matrix, and the exact-operand premise of its float cases.

If a reference here drifted from the reference trainers, the GPU file would hold the kernels to the wrong answer;
these tests pin each restatement to `ref_port` first.
"""
import pytest
import torch

from oracle import ref_port as O
from test_gpu_layout_kernels import (DIVERGE, EMPTY, PADS, PAIR_GROUPS, PAIR_L, PLAN_B, PLAN_LAYOUTS, ROLL_L, SCATTER_CASES,
                                     SEED, SS_N, SS_W, STRIP_L, TAIL_W, CRITIC_MAP, confuser, id_rows, pair_cases,
                                     plan_hi, plan_lens, ref_pairs, ref_plan, ref_rollout, ref_slice_sums, ref_strip,
                                     ref_tail_gather, ref_tail_scatter, scatter_lens, slice_operands, slice_table,
                                     strip_cases, tail_bounds, tail_lens)
from test_gpu_loss_kernels import BF, EXACT, F16, F32, sum_exact

I32, I64 = torch.int32, torch.int64


def test_rollout_refs_match_ref_port():
    """Response lengths equal ref_port.response_lengths; the mask is moved != pad; move_padding_left is a rotation
    that keeps the ids; every matrix row holds ids that an int32 compare would take for the pad."""
    for L in ROLL_L:
        for P in ROLL_L:
            for pad in PADS:
                seq = id_rows(7, L, pad, SEED + L)
                prompt = id_rows(7, P, pad, SEED + 3 * P + 1)[torch.arange(7).roll(2)]
                moved, mask, lens, counts = ref_rollout(prompt, seq, pad)
                assert lens.tolist() == O.response_lengths(prompt, seq, pad)
                assert torch.equal(mask, moved != pad)
                assert counts.tolist() == [len(O.drop_pad(s, pad)) for s in seq]
                for b in range(7):
                    assert sorted(moved[b].tolist()) == sorted(seq[b].tolist())
                    assert any(torch.equal(moved[b], seq[b].roll(k)) for k in range(L))
                kinds = {(int(n), int(c)) for n, c in zip((seq != pad).sum(1), counts)}
                assert len(kinds) > 1
                if L > 8:
                    assert bool((seq == confuser(pad)).any()), 'no id shares the pad low 32 bits'
                    assert bool((lens == 0).any()) and bool((lens > 0).any())


def test_strip_refs_match_ref_port():
    """strip: ref_strip = drop_pad(ids)[-R:] for 0 < R <= the row's tokens, and the R-th token from the right sits on
    each scan window boundary or one token either side; plain: ids[-R:]."""
    for L in STRIP_L:
        for pad in PADS:
            for strip in (1, 0):
                cases = strip_cases(L, pad, strip, SEED + L + pad % 97)
                for row, R in cases['fit']:
                    kept = O.drop_pad(row, pad) if strip else row
                    assert R <= len(kept)
                    if R > 0:
                        assert torch.equal(ref_strip(row, R, pad, strip), kept[-R:])
                    else:
                        assert ref_strip(row, R, pad, strip).numel() == 0
                for row, R in cases['short']:
                    kept = O.drop_pad(row, pad) if strip else row
                    assert R > len(kept)
                    got = ref_strip(row, R, pad, strip)
                    assert torch.equal(got[R - len(kept):], kept) and bool((got[:R - len(kept)] == -1).all())
                if strip:
                    hit = set()
                    for row, R in cases['fit']:
                        if R > 0:
                            pos = (row != pad).nonzero()[-R].item()
                            hit.add(pos)
                    for w in range(1, (L - 1) // 256 + 1):
                        q = L - 256 * w
                        assert {q - 1, q, q + 1} & set(range(L)) <= hit, (L, pad, q)


def _simpo_loop(ids, mask, n):
    """ref_port's SimPO / ORPO / KTO loop on its own: skip identical pairs, then _pair_slices (which raises)."""
    ids_b, ids_w = ids.chunk(2, dim=0)
    m_b, m_w = mask.chunk(2, dim=0)
    res, bits = {}, 0
    for i in range(n):
        if torch.all(torch.eq(ids_b[i], ids_w[i])).item():
            continue
        try:
            sl_b, sl_w, _, _ = O._pair_slices(ids_b, ids_w, m_b, m_w, i)
            res[i] = (sl_b.start, sl_b.stop - 1, sl_w.stop - 1)
        except IndexError:
            bits |= EMPTY
        except AssertionError:
            bits |= DIVERGE
    return res, bits


def test_pair_refs_match_simpo_loop():
    for L in PAIR_L:
        for group, bits_want in PAIR_GROUPS.items():
            ids, mask, n = pair_cases(L, group, SEED + L + len(group))
            for m in (mask, mask.to(torch.uint8), mask.to(I64)):
                out, bits = ref_pairs(ids, m, n)
                res, bits_loop = _simpo_loop(ids, m, n)
                assert bits == bits_loop == bits_want, (L, group, bits, bits_loop)
                assert set(res) <= {i for i in range(n) if out[0, i] == 1}
                for i, (d, eb, ew) in res.items():
                    assert (out[1, i].item(), out[2, i].item(), out[3, i].item()) == (d, eb, ew)
                for i in range(n):
                    if out[0, i] == 0:
                        assert torch.equal(ids[i], ids[n + i]) and out[1, i] == 0
            if group == 'identical':
                assert bool((out[0] == 0).all()) and bool(((out[2] < 0) | (out[3] < 0)).all())


def test_tail_refs_match_pad_sequence():
    """For 0 < R <= bound the gather is pad_sequence([x[b][-R:]]) (ref_port._tail_rows) and the scatter is its
    autograd adjoint; outside the contract the scatter is still the adjoint of the clamped gather.  R = 0 is the one
    deliberate difference: x[-0:] is the whole row, the kernels' tail is empty."""
    gen = torch.Generator().manual_seed(5)
    for W in TAIL_W:
        for bound in tail_bounds(W):
            for kind in ('in', 'out'):
                lens = tail_lens(W, bound, kind)
                x = torch.randn(len(lens), W, generator=gen, dtype=torch.float64)
                g = torch.randn(len(lens), bound, generator=gen, dtype=torch.float64)
                got = ref_tail_gather(x, lens, bound)
                if kind == 'in':
                    rows = [x[b][-r:] if r > 0 else x[b][:0] for b, r in enumerate(lens)]
                    want = O._tail_rows(rows + [torch.zeros(bound, dtype=x.dtype)])[:-1]
                    assert torch.equal(got, want)
                    assert all(r <= bound for r in lens) and 0 in lens and bound in lens
                    assert torch.equal(x[0][-0:], x[0]) and lens[0] == 0 and not bool(got[0].any())
                leaf = x.clone().requires_grad_(True)
                (ref_tail_gather(leaf, lens, bound) * g).sum().backward()
                assert torch.equal(leaf.grad, ref_tail_scatter(g, lens, W))
    for W, src in SCATTER_CASES + CRITIC_MAP:
        for kind in ('in', 'out'):
            lens = scatter_lens(W, src, kind)
            x = torch.randn(len(lens), src, generator=gen, dtype=torch.float64)
            g = torch.randn(len(lens), W, generator=gen, dtype=torch.float64)
            leaf = x.clone().requires_grad_(True)
            (ref_tail_gather(leaf, lens, W) * g).sum().backward()
            assert torch.equal(leaf.grad, ref_tail_scatter(g, lens, src))


@pytest.mark.parametrize('layout', list(PLAN_LAYOUTS))
def test_plan_refs_match_reference_slices(layout):
    """The plan table applied to flat-index tensors picks exactly the reference's rows and labels:
    logits[b, :-1][-r:] (row shift -1) or the tail of logits[b] (row shift 0) or one further, against
    ids[b, 1:][-r:]-style label tails; copies address the second tensor at its (signed) delta."""
    seq, sl, sb, lab_stride, ltl, lsh, rsh, width = PLAN_LAYOUTS[layout]
    hi = plan_hi(seq, ltl, rsh)
    for B in PLAN_B[:3]:
        for copies in (1, 2):
            lens = plan_lens(B, layout, 'out')
            for cld in ((0,) if copies == 1 else (B * sb + 4096, -(B * sb + 4096))):
                t, short = ref_plan(lens, B, seq, sb, sl, lab_stride, ltl, lsh, rsh, width, copies, cld, B * width)
                assert short
                S = B * copies
                assert t[3, S] == sum(max(min(max(0, min(r, hi)) - lsh, width), 0) for r in lens) * copies
                assert bool((t[[0, 1, 2, 4], S] == 0).all())
                for seg in range(S):
                    # a clamped length still leaves every scored row inside the tile and every label inside its row
                    c, b = divmod(seg, B)
                    r = max(0, min(lens[b], hi))
                    n = int(t[3, seg + 1] - t[3, seg])
                    assert n == max(min(r - lsh, width), 0)
                    first = (int(t[0, seg]) - b * sb - c * cld) // sl
                    assert int(t[0, seg]) == b * sb + first * sl + c * cld and 0 <= first
                    assert n == 0 or first + n <= seq  # r = 0 with row shift 1 starts one past the tile, scoring nothing
                    lab0 = int(t[1, seg]) - b * lab_stride
                    assert 0 <= lab0 and (ltl <= 0 or n == 0 or lab0 + n <= ltl)
                    assert int(t[2, seg]) == b * width + c * B * width
                    assert int(t[4, seg]) == (c * B + b) * seq + first
    if layout == 'trainer':  # against the reference's per-sample slices on real tensors
        B, V = 5, 3
        lens = [9, 1, 17, 0, 36]
        logits = torch.arange(B * seq * V).view(B, seq, V)
        ids = torch.arange(B * lab_stride).view(B, lab_stride)
        t, short = ref_plan(lens, B, seq, seq * V, V, lab_stride, ltl, lsh, rsh, width, 1, 0, B * width)
        assert not short
        for b, r in enumerate(lens):
            n = int(t[3, b + 1] - t[3, b])
            if r == 0:
                assert n == 0
                continue
            want_rows = logits[b, :-1][-r:][:width, 0]
            want_labels = ids[b, 1:][-r:][:width]
            assert n == len(want_rows)
            assert [int(t[0, b]) + j * V for j in range(n)] == want_rows.tolist()
            assert [int(t[1, b]) + j for j in range(n)] == want_labels.tolist()


def test_exact_premise():
    """slice_sums: the operands are exact in each dtype and every partial sum of a row is exact in fp32 in any order;
    the critic index map: column + 1 and its gradient image are exact in fp32."""
    for W in SS_W:
        lp = slice_operands(W, SEED + 2 * W)
        for dt in (BF, F16, F32):
            assert torch.equal(lp.to(dt).double(), lp)
        assert sum_exact(lp, 1)
        slices = slice_table(W, SEED + W)
        for rd in (None, BF, F16):
            ref_slice_sums(lp, slices, SS_N, rd)
        assert int(slices[2].max()) > W - 1 and int(slices[2].min()) == -1
    for Wm, src in CRITIC_MAP:
        assert (src + 1) <= EXACT and 8 * Wm & (8 * Wm - 1) == 0
