"""K1 forward: the ring kernel (cp.async.bulk stages, producer-resolved rows; tuning kernel digit 1) against the
vectorised-LDG kernel (digit 2).  The default picks one of them by row length, so each kernel is forced here at every
vocabulary size.  The two differ only in the order in which a row's (max, sum) partials are folded, so fp32 results
agree to summation-order noise, 16-bit results to one ulp, and everything discrete -- zeros of ignored and saturated
rows, NaN of out-of-range labels, the status word -- is identical."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = 'cuda'
RING, LDG = 1, 2  # aa_logprob_set_tuning kernel digits


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    from align_anything_b200 import ops as _ops

    return _ops


def _ordered_bits(t):
    bits = t.contiguous().view(torch.int16).to(torch.int32) & 0xFFFF
    return torch.where(bits >= 0x8000, 0x8000 - bits, bits)


def _assert_same(got, want, what):
    got, want = got.cpu(), want.cpu()
    assert got.dtype == want.dtype and got.shape == want.shape, what
    assert torch.equal(torch.isnan(got), torch.isnan(want)), f'{what}: NaN pattern differs'
    assert torch.equal(got == 0, want == 0), f'{what}: zero pattern differs'
    got, want = torch.nan_to_num(got), torch.nan_to_num(want)
    if got.dtype == torch.float32:
        err = (got - want).abs()
        tol = 2e-6 * want.abs().clamp(min=1.0)
        assert not bool((err > tol).any()), f'{what}: max err {float(err.max()):.3e}'
    else:
        d = (_ordered_bits(got) - _ordered_bits(want)).abs()
        assert int(d.max()) <= 1, f'{what}: {int(d.max())} ulp'


def _run_both(ops, fn):
    """fn() with the ring forward and with the LDG forward; the status word each run left behind."""
    from align_anything_b200 import _lib as Lb

    status = ops._device_scratch(torch.device(DEV))['status']
    outs = []
    try:
        for digit in (RING, LDG):
            Lb.check(Lb.lib().aa_logprob_set_tuning(digit, 0))
            status.zero_()
            res = fn()
            torch.cuda.synchronize()
            outs.append((res, int(status.item())))
    finally:
        Lb.check(Lb.lib().aa_logprob_set_tuning(0, 0))
        status.zero_()
    return outs


@pytest.mark.parametrize('V', [128257, 32064, 1000, 40])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
def test_ring_forward_matches_ldg_forward(ops, V, dtype):
    gen = torch.Generator().manual_seed(V + 7)
    n, Lq = 4, 24
    lens = [9, 20, 5, 17]
    # 3 spare columns: a row stride that is neither V nor a multiple of 8 elements, so every row has its own alignment
    tile = (torch.randn(n, Lq, V + 3, generator=gen) * 2.5).to(dtype).to(DEV)
    logits = tile[..., :V]
    ids = torch.randint(0, V, (n, Lq), generator=gen).to(DEV)
    logits[0, Lq - lens[0], ids[0, Lq - lens[0] + 1]] = 60.0  # saturated: the label's probability rounds to 1
    W = max(lens) - 1
    plan = ops.RowPlan([b * logits.stride(0) + (Lq - r) * logits.stride(1) for b, r in enumerate(lens)],
                       [b * Lq + (Lq - r + 1) for b, r in enumerate(lens)], [b * W for b in range(n)],
                       [r - 1 for r in lens], [0] * n, (n, W), 0, DEV)

    def launch(labels, out_dtype, ignore_index=None):
        def fn():
            out = torch.zeros((n, W), dtype=out_dtype, device=DEV)
            stat = torch.zeros((2, plan.n_rows), dtype=torch.float32, device=DEV)
            ops._launch_fwd(logits, labels, plan, out, stat[0], stat[1], ignore_index)
            return out, stat
        return fn

    ignored = ids.clone()
    ignored[:, ::3] = -100
    bad = ids.clone()
    bad[2, Lq - 2] = V + 5  # out of range: NaN and the label status bit
    cases = [('plain', launch(ids, torch.float32)), ('plain faithful', launch(ids, dtype)),
             ('ignore_index', launch(ignored, dtype, -100)), ('label out of range', launch(bad, torch.float32))]
    if dtype != torch.float32:
        cases.append(('other 16-bit out', launch(ids, torch.bfloat16 if dtype == torch.float16 else torch.float16)))
    for what, fn in cases:
        (a, st_a), (b, st_b) = _run_both(ops, fn)
        assert st_a == st_b, (what, st_a, st_b)
        _assert_same(a[0], b[0], f'{what} V={V} {dtype}')
        assert torch.equal(a[1][0].cpu(), b[1][0].cpu()), f'{what}: row max differs'
        _assert_same(a[1][1], b[1][1], f'{what} V={V} {dtype} logsum')
        if what == 'plain':
            assert float(a[0][0, 0]) == 0.0  # the saturated row scores exactly 0


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32])
def test_ring_forward_device_plan(ops, dtype):
    """A plan built on the device (aa_tail_plan_build): n_rows is an upper bound, the table holds the exact count."""
    gen = torch.Generator().manual_seed(321)
    B, Lq, V = 5, 37, 128257
    lens = [9, 1, 17, 0, 12]
    ids = torch.randint(1, V, (B, Lq), generator=gen).to(DEV)
    tile = (torch.randn(B, Lq, V, generator=gen) * 2.5).to(dtype).to(DEV)
    dl = ops.DeviceLens(torch.tensor(lens, dtype=torch.int32, device=DEV), 20)
    (a, st_a), (b, st_b) = _run_both(ops, lambda: ops.response_tail_log_probs(tile, ids, dl))
    assert st_a == st_b == 0
    _assert_same(a, b, f'device plan {dtype}')
    assert float(a[:, max(lens):].abs().max()) == 0.0
