"""FAITHFUL K5 and K1f at mask counts a 16-bit dtype cannot hold (run on an H100: `pytest -m gpu`).

The reference divides by `mask.sum(-1)` (masked_mean) or `mask.sum()` (token mean), int64 counts that ATen casts to the
dividend's dtype: with bf16 / fp16 log-probs and advantages a row of 257 bf16 tokens is divided by 256, a token-mean total
of 1501 by 1504.  The premise test records what ATen CUDA does; K5 (through the C ABI, on guard-banded buffers) and K1f
(`aa_logprob_actor_fused_obj`, dense and tail plans at V = 152064) are held bit for bit to the port on ATen CUDA and to
the float64 restatement of tests/test_cpu_faithful_counts.py on exact operands.  GRPO divides an fp32 loss by an fp32
count, exactly, and must keep doing so.
"""
from __future__ import annotations

import pytest
import torch

from align_anything_b200 import _lib as Lb
from oracle import ref_port as O
from ppo_objective_port import actor_loss as port_loss
from test_cpu_faithful_counts import (BF, CASE_IDS, CASES, CRITIC_CLIP, F16, exact_actor_case, exact_critic_case, k5_actor,
                                      k5_critic, r)
from test_gpu_loss_kernels import CODE, FAITHFUL, Guarded, Words, _k5_buffers, _stream, fenced, fenced_vec, rc_ok
from test_gpu_parity import assert_ulp_close, ops  # noqa: F401  (fixture)
from test_gpu_ppo_objective import AGG, OPTIONS, _k5

pytestmark = pytest.mark.gpu

DEV = 'cuda'
DEFAULT = (0.2, 0.2, None, 'seq-mean-token-mean')
V = 152064


def _identical(got, want, what):
    """Bit-identical values of one dtype, except that +0 equals -0 (K5 stores a masked-out gradient as +0 where
    autograd's `grad * mask` leaves -0)."""
    got, want = got.detach(), want.detach().to(got.device)
    assert got.dtype == want.dtype, (what, got.dtype, want.dtype)
    if not torch.equal(got, want):
        bad = got != want
        i = int(bad.reshape(-1).nonzero()[0])
        raise AssertionError(f'{what}: {int(bad.sum())} of {got.numel()} differ, first at {i}: got '
                             f'{float(got.reshape(-1)[i])!r}, want {float(want.reshape(-1)[i])!r}')


def _port(lp, old, adv, mask, opt):
    lo, hi, c, agg = opt
    x = lp.clone().requires_grad_(True)
    loss = port_loss(x, old, adv, mask, lo, hi, c, agg)
    loss.backward()
    return loss.detach(), x.grad


def _loss16(loss, dt):
    """The 16-bit loss K5 leaves in the low half of loss[1], as a 0-dim tensor."""
    return loss[1:2].view(dt)[:1].reshape(())


def _counts_mask(counts, W, seed):
    """(B, W) bool on the device with counts[b] masked-in tokens in row b, at random places."""
    g = torch.Generator().manual_seed(seed)
    m = torch.zeros(len(counts), W, dtype=torch.bool)
    for b, n in enumerate(counts):
        m[b, torch.randperm(W, generator=g)[:n]] = True
    return m.to(DEV)


# ---- the premise: what ATen CUDA divides by ---------------------------------------------------------------------------
def test_aten_cuda_casts_the_count_to_the_dividend_dtype(ops):
    """(1) a 16-bit (B,) tensor divided by an int64 (B,) count (masked_mean's row step), B = 1 included; (2) the token
    mean's 0-dim quotient `-(s * mask).sum() / mask.sum()`; (3) its DivBackward.  All three divide by the count rounded
    to the 16-bit dtype (on ATen CPU only (1) at B > 1 does)."""
    for dt, n in ((BF, 257), (F16, 2049)):
        assert r(-0.5 / r(n, dt), dt) != r(-0.5 / n, dt)  # the two rules differ at this count
        for B in (1, 3):
            q = torch.full((B,), -0.5, dtype=dt, device=DEV) / torch.full((B,), n, dtype=torch.int64, device=DEV)
            assert q.dtype == dt
            assert torch.equal(q.double().cpu(), r(-0.5 / r(n, dt), dt).expand(B)), f'(B,) division {dt} n={n} B={B}'
    for dt, total in ((BF, 1501), (F16, 2049)):
        want = -r(1.0 / r(total, dt), dt)
        assert want != -r(1.0 / total, dt)
        s = torch.zeros(total + 3, dtype=dt, device=DEV)
        s[0] = 1.0
        s.requires_grad_(True)
        mask = torch.ones(total + 3, dtype=torch.bool, device=DEV)
        mask[-3:] = False
        loss = -(s * mask).sum() / mask.sum()
        assert loss.dtype == dt
        assert float(loss) == float(want), f'token-mean quotient {dt} total={total}: {float(loss)!r}'
        loss.backward()
        assert torch.equal(s.grad[:total].double().cpu(), want.expand(total)), f'token-mean DivBackward {dt} total={total}'
        assert not bool(s.grad[total:].any())


# ---- K5 through the C ABI ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B', [1, 3, 129])
@pytest.mark.parametrize('dt,n', CASES, ids=CASE_IDS)
def test_k5_actor_counts_vs_port(ops, dt, n, B):
    """aa_ppo_actor_loss and aa_ppo_actor_loss_obj (every option) at lp == old and dyadic advantages, n masked-in tokens
    per row: the 16-bit loss and the gradient bit-identical to the port on ATen CUDA, and the default objective to the
    float64 restatement."""
    lp64, adv64, mask64 = exact_actor_case(B, n, dt, seed=n + B)
    lp, adv, mask = lp64.to(dt).to(DEV), adv64.to(dt).to(DEV), mask64.to(DEV)
    w_loss, _, w_grad = k5_actor(adv64, mask64, dt)
    for name, opt in [('legacy', DEFAULT), *OPTIONS.items()]:
        what = f'{name} {dt} n={n} B={B}'
        loss, grad, _ = _k5(ops, lp, lp, adv, mask, opt, 'faithful', legacy=name == 'legacy')
        want, gwant = _port(lp, lp, adv, mask, opt)
        _identical(_loss16(loss, dt), want, what + ' loss')
        assert float(loss[0]) == float(want), what + ' fp32 loss word'
        _identical(grad, gwant, what + ' grad')
        if opt[3] == 'seq-mean-token-mean' and opt[2] is None:
            assert float(want) == float(w_loss), what + ' loss vs float64'
            assert torch.equal(grad.double().cpu(), w_grad), what + ' grad vs float64'


@pytest.mark.parametrize('dt,counts', [(BF, [1501]), (BF, [500, 500, 501]), (F16, [2049]), (F16, [683, 683, 683])],
                         ids=['bfloat16-1x1501', 'bfloat16-3x500', 'float16-1x2049', 'float16-3x683'])
def test_k5_token_mean_totals_vs_port(ops, dt, counts):
    """Token-mean over a micro-batch total the dtype cannot hold (1501 -> 1504 in bf16, 2049 -> 2048 in fp16)."""
    B, W = len(counts), max(counts) + 7
    g = torch.Generator().manual_seed(sum(counts))
    lp = (-torch.randint(1, 65, (B, W), generator=g).double() / 16).to(dt).to(DEV)
    adv = (torch.randint(-32, 33, (B, W), generator=g).double() / 8).to(dt).to(DEV)
    mask = _counts_mask(counts, W, seed=B)
    for name in ('token-mean', 'all'):
        what = f'{name} {dt} counts={counts}'
        loss, grad, _ = _k5(ops, lp, lp, adv, mask, OPTIONS[name], 'faithful')
        want, gwant = _port(lp, lp, adv, mask, OPTIONS[name])
        _identical(_loss16(loss, dt), want, what + ' loss')
        _identical(grad, gwant, what + ' grad')


@pytest.mark.parametrize('dt,n', [(BF, 257), (F16, 2049)], ids=['bfloat16-257', 'float16-2049'])
def test_k5_actor_realistic_operands_vs_port(ops, dt, n):
    """Random log-probs, ratios inside and outside the clip range: within 1 ulp of the port on ATen CUDA and >= 99 %
    bit-identical (a one-ulp error in a row's coefficient moves most of that row's gradients)."""
    B, W = 3, n + 9
    g = torch.Generator().manual_seed(n)
    lp = (-torch.rand(B, W, generator=g) * 4).to(dt).to(DEV)
    old = (lp.float().cpu() + torch.randn(B, W, generator=g) * 0.3).to(dt).to(DEV)
    adv = torch.randn(B, W, generator=g).to(dt).to(DEV)
    mask = _counts_mask([n] * B, W, seed=n)
    for name, opt in (('legacy', DEFAULT), ('dual-clip', OPTIONS['dual-clip'])):
        loss, grad, _ = _k5(ops, lp, old, adv, mask, opt, 'faithful', legacy=name == 'legacy')
        want, gwant = _port(lp, old, adv, mask, opt)
        assert_ulp_close(_loss16(loss, dt).reshape(1), want.reshape(1), max_ulp=1, min_exact=0.0, what=f'{name} loss')
        assert_ulp_close(grad, gwant, max_ulp=1, min_exact=0.99, what=f'{name} {dt} n={n} grad')


@pytest.mark.parametrize('B', [1, 3, 129])
@pytest.mark.parametrize('dt,n', CASES, ids=CASE_IDS)
def test_k5_critic_counts_vs_port(ops, dt, n, B):
    """aa_ppo_critic_loss on exact operands: the 16-bit loss, the gradient and the row means bit-identical to the port
    on ATen CUDA and to the float64 restatement."""
    x64, o64, r64, mask64 = exact_critic_case(B, n, dt, seed=2 * n + B)
    W = x64.size(1)
    mask = mask64.to(DEV)
    x, old, ret = fenced(x64.to(dt), W + 2), fenced(o64.to(dt), W + 1), fenced(r64.to(dt), W + 3)
    mt = fenced(mask, W + 3, pad=True)
    grad, loss, row_mean, rows = _k5_buffers(B, W, dt, True)
    counter = Words()
    what = f'critic {dt} n={n} B={B}'
    rc_ok(Lb.lib().aa_ppo_critic_loss(x.data_ptr(), W + 2, old.data_ptr(), W + 1, CODE[dt], ret.data_ptr(), W + 3,
                                      CODE[dt], mt.data_ptr(), W + 3, B, W, CRITIC_CLIP, FAITHFUL, loss.ptr(), grad.ptr(),
                                      W + 8, row_mean.ptr(), rows.ptr(), counter.ptr(), None, 0, _stream()), what)
    torch.cuda.synchronize()
    counter.check([0], what + ' counter')
    for name, buf in (('grad', grad), ('loss', loss), ('row_mean', row_mean), ('rows', rows)):
        buf.check(f'{what} {name}')
    leaf = x.detach().clone().requires_grad_(True)
    want = O.critic_loss(leaf, old, ret, mask, CRITIC_CLIP)
    want.backward()
    _identical(_loss16(loss.t[0], dt), want, what + ' loss')
    _identical(grad.t, leaf.grad, what + ' grad')
    w_loss, w_rows, w_grad = k5_critic(x64, o64, r64, mask64, dt)
    assert float(want) == float(w_loss), what + ' loss vs float64'
    assert torch.equal(rows.t[:, 0].double().cpu(), w_rows), what + ' row means vs float64'
    assert torch.equal(grad.t.double().cpu(), w_grad), what + ' grad vs float64'


# ---- K1f through aa_logprob_actor_fused_obj ---------------------------------------------------------------------------
def _k1f_inputs(node, seed):
    """bf16 logits (B, Lq, V) whose label logits are 0 (p_y ~ 4e-6, so the tile's label column g * (1 - p_y) rounds to
    the per-token coefficient g), rows scoring 257 and 300 tokens."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    B, W = 2, 300
    if node == 'dense':
        start, Lq = 1, 1 + 300 + 6 + 1
        W = Lq - 1 - start
        mask = _counts_mask([257, 300], W, seed)
        lens = None
    else:
        start, Lq, lens = None, 303, [257, 300]
        mask = torch.arange(W, device=DEV)[None, :] < torch.tensor(lens, device=DEV)[:, None]
    logits = torch.randn(B, Lq, V, generator=gen, device=DEV).bfloat16()
    ids = torch.randint(0, V, (B, Lq), generator=gen, device=DEV)
    logits[:, :-1].scatter_(-1, ids[:, 1:, None], 0.0)
    p_y = torch.softmax(logits[:, :-1].float(), -1).gather(-1, ids[:, 1:, None])
    assert float(p_y.max()) < 1e-4
    return logits, ids, start, lens, W, mask


def _scored(node, start, lens, W, Lq):
    """(b, t) -> tile row of the token scored at lp[b, t]; None where the position is not scored."""
    if node == 'dense':
        return lambda b, t: start + t
    return lambda b, t: Lq - 1 - lens[b] + t if t < lens[b] else None


def _k1f(ops, node, logits, ids, start, lens, W, old, adv, mask, opt):
    """aa_logprob_actor_fused_obj on guard-banded log-prob and tile buffers -> (log-probs (B, W), tile (B, Lq, V))."""
    B, Lq, _ = logits.shape
    if node == 'dense':
        plan = ops._dense_actor_plan(B, Lq, start, logits.stride(0), logits.stride(1), ids.stride(0), str(logits.device))
    else:
        plan = ops.device_tail_plan(ops.as_device_lens(lens, logits.device), Lq, logits.stride(0), logits.stride(1),
                                    ids.stride(0), ids.size(1), 0, -1, W)
    lp = Guarded(B, W, BF)
    lp.t.zero_()  # tail plans leave the unscored positions as they are
    tile = Guarded(B * Lq, V, BF)
    scratch = torch.empty(plan.n_tile_rows * 6 + (plan.n_seg + 1) // 2, dtype=torch.int64, device=DEV)
    lo, hi, c, agg = opt
    p = plan.ptrs()
    Lb.check(Lb.lib().aa_logprob_actor_fused_obj(
        logits.data_ptr(), Lb.AA_BF16, logits.stride(1), V, ids.data_ptr(), plan.n_seg, p[0], p[1], p[2], p[3], p[4],
        plan.n_tile_rows, lp.ptr(), Lb.AA_BF16, None, None, old.data_ptr(), old.stride(0), adv.data_ptr(),
        adv.stride(0), CODE[adv.dtype], mask.data_ptr(), mask.stride(0), W, float(lo), float(hi), float(c or 0.0),
        AGG[agg], FAITHFUL, tile.ptr(), V, scratch.data_ptr(), ops._device_scratch(logits.device)['status'].data_ptr(),
        0.0, None, _stream()))
    torch.cuda.synchronize()
    assert lp.outside_intact(), 'a guard of the log-prob buffer was written'
    tile.check('gradient tile')
    ops.check_status()
    return lp.t.clone(), tile.t.view(B, Lq, V)


def _label_column(tile, ids, row_of, B, W):
    """tile[b, row, label] at every scored (b, t); 0 where the position is not scored."""
    out = torch.zeros(B, W, dtype=tile.dtype, device=DEV)
    for b in range(B):
        rows = [(t, row_of(b, t)) for t in range(W) if row_of(b, t) is not None]
        t_idx = torch.tensor([t for t, _ in rows], device=DEV)
        r_idx = torch.tensor([row for _, row in rows], device=DEV)
        out[b, t_idx] = tile[b, r_idx, ids[b, r_idx + 1]]
    return out


@pytest.mark.parametrize('node', ['dense', 'tail'])
def test_k1f_label_column_vs_port(ops, node):
    """The tile's label column is d loss / d lp: bit-identical to ATen's gradient of the port evaluated on K1f's own
    log-probs at lp == old (every objective; the token-mean total 557 rounds to 556 in bf16), and within 1 ulp and
    >= 99 % identical with ratios inside and outside the clip range."""
    logits, ids, start, lens, W, mask = _k1f_inputs(node, seed=257)
    B, Lq, _ = logits.shape
    row_of = _scored(node, start, lens, W, Lq)
    gen = torch.Generator().manual_seed(3)
    adv = (torch.randint(-32, 33, (B, W), generator=gen).double() / 8).to(BF).to(DEV)
    lp, _ = _k1f(ops, node, logits, ids, start, lens, W, torch.zeros(B, W, dtype=BF, device=DEV), adv, mask, DEFAULT)
    assert bool(torch.isfinite(lp).all())
    for name, opt in [('default', DEFAULT), *OPTIONS.items()]:
        lp2, tile = _k1f(ops, node, logits, ids, start, lens, W, lp, adv, mask, opt)
        _identical(lp2, lp, f'{node} {name} log-probs')
        _, gwant = _port(lp, lp, adv, mask, opt)
        _identical(_label_column(tile, ids, row_of, B, W), gwant, f'{node} {name} label column')
    old = (lp.float() + torch.randn(B, W, generator=gen).to(DEV) * 0.3).to(BF)
    _, tile = _k1f(ops, node, logits, ids, start, lens, W, old, adv, mask, DEFAULT)
    _, gwant = _port(lp, old, adv, mask, DEFAULT)
    assert_ulp_close(_label_column(tile, ids, row_of, B, W), gwant, max_ulp=1, min_exact=0.99,
                     what=f'{node} realistic label column')


# ---- GRPO: an fp32 count, divided exactly -----------------------------------------------------------------------------
EOS = 3


def _grpo_tokens(B, K, ends):
    gen = torch.Generator().manual_seed(K)
    tok = torch.randint(4, 100, (B, K), generator=gen)
    for b, e in enumerate(ends):
        tok[b, e - 1] = EOS  # counted: positions up to and including the first eos
    return tok.to(DEV)


def test_grpo_loss_exact_total(ops):
    """aa_grpo_loss with bf16 log-probs over 1501 counted tokens (1504 in bf16): the per-token loss is fp32, so the
    reference divides by the exact count; lp == ref keeps every gradient exact, bit-identical to the port."""
    B, K, ends, beta = 3, 520, [500, 500, 501], 0.04
    tok64 = _grpo_tokens(B, K, ends)
    gen = torch.Generator().manual_seed(11)
    lp64 = (-torch.rand(B, K, generator=gen) * 4).to(BF).to(DEV)
    A = fenced_vec(torch.randn(B, generator=gen).to(DEV))
    lp, rf, tok = fenced(lp64, K + 2), fenced(lp64, K + 1), fenced(tok64, K + 3, pad=EOS)
    loss, grad = Guarded(1, 1, torch.float32), Guarded(B, K, BF, pitch=K + 8)
    row_end, scratch = Guarded(B, 1, torch.int32), Guarded(1, B + 1, torch.float32)
    counter = Words(n=2)
    rc_ok(Lb.lib().aa_grpo_loss(lp.data_ptr(), K + 2, rf.data_ptr(), K + 1, CODE[BF], A.data_ptr(), tok.data_ptr(), K + 3,
                                EOS, B, K, beta, FAITHFUL, loss.ptr(), grad.ptr(), K + 8, row_end.ptr(), scratch.ptr(),
                                counter.ptr(), _stream()), 'grpo')
    torch.cuda.synchronize()
    counter.check([0, 0], 'grpo counters')
    for name, buf in (('loss', loss), ('grad', grad), ('row_end', row_end), ('scratch', scratch)):
        buf.check(f'grpo {name}')
    assert float(scratch.t[0, 0]) == 1501.0
    leaf = lp.detach().clone().requires_grad_(True)
    want = O.grpo_loss(leaf, rf, A[:, None], tok64, 0, EOS, beta)
    want.backward()
    assert want.dtype == torch.float32
    _identical(grad.t, leaf.grad, 'grpo grad')
    # fp32 sums in different orders; a divisor of 1504 would be 2e-3 off
    assert abs(float(loss.t[0, 0]) - float(want)) <= 1e-5 * abs(float(want)), (float(loss.t[0, 0]), float(want))


def test_grpo_k1f_exact_total(ops):
    """The K1f GRPO node over 1501 counted bf16 tokens: the tile's label column bit-identical to ATen's gradient of the
    port on K1f's own log-probs (ref == lp), the loss within fp32 summation error of the exact-count mean."""
    B, P, K, ends, beta = 3, 4, 520, [500, 500, 501], 0.04
    gen = torch.Generator(device=DEV).manual_seed(5)
    ids = torch.randint(4, V, (B, P + K), generator=gen, device=DEV)
    ids[:, P:] = _grpo_tokens(B, K, ends)
    logits = torch.randn(B, P + K, V, generator=gen, device=DEV).bfloat16()
    logits[:, :-1].scatter_(-1, ids[:, 1:, None], 0.0)
    adv = torch.randn(B, generator=gen, device=DEV)
    x = logits.clone().requires_grad_(True)
    _, lp, _ = ops.grpo_loss_from_logits(x, ids, K, torch.zeros(B, K, dtype=BF, device=DEV), adv, EOS, beta)
    x = logits.clone().requires_grad_(True)
    loss, lp2, row_end = ops.grpo_loss_from_logits(x, ids, K, lp, adv, EOS, beta)
    loss.backward()
    _identical(lp2, lp, 'K1f GRPO log-probs')
    assert row_end.tolist() == ends
    leaf = lp.clone().requires_grad_(True)
    want = O.grpo_loss(leaf, lp, adv[:, None], ids[:, P:], 0, EOS, beta)
    want.backward()
    rows = torch.arange(P - 1, P + K - 1, device=DEV)
    col = torch.stack([x.grad[b, rows, ids[b, rows + 1]] for b in range(B)])
    _identical(col, leaf.grad, 'K1f GRPO label column')
    assert abs(float(loss) - float(want)) <= 1e-5 * abs(float(want)), (float(loss), float(want))
    ops.check_status()
