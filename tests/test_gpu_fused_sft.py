"""The fused lm_head cross-entropy of SFT (run on an H100: `pytest -m gpu`).

* K6s `aa_linear_logits` through the C ABI, on the exact-arithmetic operands and guarded, NaN-fenced buffers of
  test_gpu_lm_head_tiles: the stored tile is bit-identical to bf16 of the float64 product, its pad columns are +0,
  nothing outside it is written; stat_max is bit-exact, stat_logsum and the log-probs within 2e-5 of float64; an
  out-of-range label gives NaN and the status bit; split and unsplit vocabulary schedules.  One real-valued case against
  the GEMM bound, with statistics that describe the stored tile.
* ops.causal_lm_loss_from_hidden against ATen's ForCausalLMLoss chain (F.linear -> .float() -> cross_entropy): the loss
  within 2e-5 relative (and against ops.causal_lm_loss on the same logits); d(hidden) and d(weight) against float64
  products of autograd's d(logits), to the GEMM bar plus the d(logits) slack of test_gpu_fused_rl.  Prompt masks, right
  padding, a sample without a valid label, a single valid row, forced chunking with a 1-row last chunk, loss_scale != 1,
  upstream scalars 0.25 and 0.3, a frozen head, a tied head, no_grad, N == 0 and a second backward.
* SupervisedTrainer with `fused_lm_head` on against off: loss, gradients, and an out-of-range label's IndexError.
"""
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from align_anything_b200 import _lib as Lb
from test_gpu_fused_rl import LM, _dlogits_slack
from test_gpu_lm_head_tiles import (BF, BM, F32, POISON, Guarded, _bound, _canon, _device_status_ptr, _fwd_operands,
                                    _half_ulp_bf16, _partial_floats, _plant_labels, _status_take, _stream, _up,
                                    poisoned_operand, schedule, vec_guard)
from test_gpu_parity import assert_close_f32, ops  # noqa: F401  (ops: fixture)

pytestmark = pytest.mark.gpu

DEV = 'cuda'
IGN = -100


# ---- K6s through the C ABI -------------------------------------------------------------------------------------------
def _run_k6s(hidden, weight, labels, mode, partial_kind, n, V, H, ld):
    out = vec_guard(n, BF if mode == Lb.MODE_FAITHFUL else F32)
    smax, slog = vec_guard(n, F32), vec_guard(n, F32)
    pf = _partial_floats(partial_kind, n)
    part = vec_guard(pf, F32) if pf else None
    tile = Guarded(n, _up(V, 256), ld, BF, tail_rows=_up(n, BM) - n)
    _status_take()
    Lb.check(Lb.lib().aa_linear_logits(
        hidden.data_ptr(), n, H, hidden.stride(0), weight.data_ptr(), V, weight.stride(0), labels.data_ptr(),
        out.ptr(), Lb.dtype_code(out.t.dtype), smax.ptr(), slog.ptr(), part.ptr() if part else None, pf, mode,
        _device_status_ptr(), tile.ptr(), ld, _stream()))
    torch.cuda.synchronize()
    return out, smax, slog, part, tile, _status_take()


# (n, H, V, partial, ld - roundup256(V))
K6S_CASES = [
    (63, 192, 257, 'wide', 0),
    (129, 320, 777, 'none', 64),
    (300, 4096, 32064, 'wide', 0),
    (2100, 256, 32064, 'wide', 64),
    (260, 4096, 128257, 'wide', 0),
]


@pytest.mark.parametrize('case', K6S_CASES, ids=[f'{c[0]}x{c[1]}x{c[2]}-{c[3]}-ld+{c[4]}' for c in K6S_CASES])
def test_k6s_exact(ops, case):
    n, H, V, partial_kind, ld_extra = case
    ld = _up(V, 256) + ld_extra
    splits, tps, _ = schedule(n, V, partial_kind != 'none', _partial_floats(partial_kind, n))
    assert (splits > 1) == (partial_kind != 'none'), 'the case must hit the schedule it names'
    oob = n != 129  # the 129-row case has in-range labels only: the status bit must stay clear
    labels = _plant_labels(n, V, splits, tps, n + V + 1, oob=oob).to(DEV)
    hidden, weight = _fwd_operands(n, H, V)
    hs, ws = (H, H) if n % 2 else (H + 8, H + 64)
    hidden, weight = poisoned_operand(hidden, hs), poisoned_operand(weight, ws)
    x64 = hidden.double() @ weight.double().T
    xr = x64.float().bfloat16()  # exact GEMM: its bf16 rounding is the reference tile bit for bit
    xr64 = xr.double()
    lab_ok = (labels >= 0) & (labels < V)
    y = torch.where(lab_ok, labels, torch.zeros_like(labels))
    m_ref = xr64.max(dim=1).values
    ls_ref = torch.logsumexp(xr64 - m_ref[:, None], dim=1)
    for mode in (Lb.MODE_FAITHFUL, Lb.MODE_F32):
        what = f'{case} mode {mode}'
        out, smax, slog, part, tile, status = _run_k6s(hidden, weight, labels, mode, partial_kind, n, V, H, ld)
        for gd in (out, smax, slog, tile):
            assert gd.outside_intact(), f'{what}: write outside an output'
            assert not bool((gd.region_bits() == POISON[gd.esz]).any()), f'{what}: an output was not written'
        if part is not None:
            assert part.outside_intact(), f'{what}: write outside partial'
        assert torch.equal(_canon(tile.t[:, :V]), _canon(xr)), f'{what}: stored logits'
        assert bool((tile.region_bits()[:, V:] == 0).all()), f'{what}: pad columns are not +0'
        assert bool(status & Lb.STATUS_LABEL_OOB) == (not bool(lab_ok.all())), f'{what}: status {status:#x}'
        assert torch.equal(smax.vec.double(), m_ref), f'{what}: stat_max'
        err = (slog.vec.double() - ls_ref).abs()
        assert bool((err <= 2e-5 * ls_ref.abs().clamp(min=1.0)).all()), f'{what}: stat_logsum {float(err.max()):.3e}'
        lp = out.vec
        assert torch.equal(torch.isnan(lp), ~lab_ok), f'{what}: NaN pattern of the log-probs'
        x_lab = xr64.gather(1, y[:, None])[:, 0]
        if mode == Lb.MODE_F32:
            ref = x_lab - m_ref - ls_ref
            e = (lp.double() - ref).abs()[lab_ok]
            assert bool((e <= 2e-5 * ref.abs().clamp(min=1.0)[lab_ok]).all()), f'{what}: log-probs {float(e.max()):.3e}'
        else:  # bf16((x_label - m) - logsum) from the kernel's own statistics
            want = ((x_lab.float() - smax.vec) - slog.vec).bfloat16()
            assert torch.equal(lp[lab_ok].view(torch.int16), want[lab_ok].view(torch.int16)), f'{what}: faithful log-probs'


def test_k6s_real_valued(ops):
    """Random operands: the stored tile within the GEMM bound of float64, and the statistics describe the stored tile
    (stat_max its row maximum bit for bit, stat_logsum and the log-probs within 2e-5 of float64 over it)."""
    n, H, V = 300, 4096, 32064
    ld = _up(V, 256)
    gen = torch.Generator().manual_seed(77)
    hidden = torch.randn(n, H, generator=gen).bfloat16().to(DEV)
    weight = (torch.randn(V, H, generator=gen) * (2.5 / H ** 0.5)).bfloat16().to(DEV)
    labels = torch.randint(0, V, (n,), generator=gen).to(DEV)
    out, smax, slog, part, tile, status = _run_k6s(hidden, weight, labels, Lb.MODE_F32, 'wide', n, V, H, ld)
    assert status == 0 and tile.outside_intact()
    ref = hidden.double() @ weight.double().T
    got = tile.t[:, :V].double()
    bar = _bound(ref, hidden.double().abs() @ weight.double().abs().T, H)
    assert bool(((got - ref).abs() <= bar).all()), f'tile: max err / bar {float(((got - ref).abs() / bar).max()):.3f}'
    m = got.max(dim=1).values
    assert torch.equal(smax.vec.double(), m)
    ls = torch.logsumexp(got - m[:, None], dim=1)
    assert bool(((slog.vec.double() - ls).abs() <= 2e-5 * ls.abs().clamp(min=1.0)).all())
    lp_ref = got.gather(1, labels[:, None])[:, 0] - m - ls
    assert bool(((out.vec.double() - lp_ref).abs() <= 2e-5 * lp_ref.abs().clamp(min=1.0)).all())


# ---- the op --------------------------------------------------------------------------------------------------------
def _labels(B, Lq, V, seed, layout='mixed'):
    """'mixed': a masked prompt, a right-padded sample, a sample without any valid label and one with a single valid
    row, in turn; 'all': every label valid."""
    gen = torch.Generator().manual_seed(seed)
    lab = torch.randint(0, V, (B, Lq), generator=gen)
    lab[:, 0] = V - 1
    if layout == 'mixed':
        for b in range(B):
            kind = b % 4
            if kind == 0:
                lab[b, :Lq // 5] = IGN  # prompt
            elif kind == 1:
                lab[b, :3] = IGN
                lab[b, Lq - Lq // 4:] = IGN  # right padding
            elif kind == 2:
                lab[b] = IGN
            else:
                keep = lab[b, Lq // 2].clone()
                lab[b] = IGN
                lab[b, Lq // 2] = keep
    return lab.to(DEV)


def _operands(B, Lq, H, V, seed):
    gen = torch.Generator().manual_seed(seed)
    hidden = torch.randn(B, Lq, H, generator=gen).bfloat16().to(DEV)
    weight = (torch.randn(V, H, generator=gen) * (2.5 / H ** 0.5)).bfloat16().to(DEV)
    return hidden, weight


def _aten_loss(logits, labels):
    """transformers ForCausalLMLoss: the upcast logits, shifted labels, mean cross-entropy over labels != -100."""
    V = logits.size(-1)
    return F.cross_entropy(logits.float()[:, :-1].reshape(-1, V), labels[:, 1:].reshape(-1), ignore_index=IGN)


def _is_pow2(x):
    return x > 0 and float(torch.tensor(x).log2().round().exp2()) == x


def _check_grads(hidden, weight, labels, dh, dw, scale, n_chunks, what):
    """d(hidden) / d(weight) of `scale` * loss against float64 products of autograd's d(logits) (loss_scale folded into
    `scale` by the caller), to the GEMM bar plus the d(logits) slack; a scalar that is not a power of two adds one
    rounding of the result (aa_scale_tile)."""
    B, Lq, H = hidden.shape
    V = weight.size(0)
    logits = F.linear(hidden, weight).requires_grad_(True)
    _aten_loss(logits, labels).backward()
    dl = logits.grad.double()  # the seed -1 / N per valid row: the backward of scale 1
    valid = torch.zeros(B, Lq, dtype=torch.bool, device=DEV)
    valid[:, :-1] = labels[:, 1:] != IGN
    n_valid = int(valid.sum())
    g_rows = valid.double() * (-1.0 / max(n_valid, 1))
    slack = _dlogits_slack(logits, dl, g_rows)
    del logits

    def bar_of(ref, bar):
        b = abs(scale) * bar
        return b + _half_ulp_bf16(abs(scale) * ref.abs() + b) if not _is_pow2(abs(scale)) else b

    w64 = weight.double()
    if dh is not None:
        ref = dl @ w64
        sp = slack @ w64.abs()
        bar = bar_of(ref, _bound(ref, dl.abs() @ w64.abs() + sp, V) + sp)
        err = (dh.double() - scale * ref).abs()
        assert bool((err <= bar).all()), f'{what} d(hidden): {int((err > bar).sum())} beyond, max err / bar {float((err / bar).max()):.3f}'
        assert bool((dh[~valid] == 0).all()), f'{what}: d(hidden) of rows that score nothing'
    if dw is not None:
        dl2, sl2, h2 = dl.view(-1, V), slack.view(-1, V), hidden.reshape(-1, H).double()
        for v0 in range(0, V, 16384):
            blk = dl2[:, v0:v0 + 16384].T
            ref = blk @ h2
            sp = sl2[:, v0:v0 + 16384].T @ h2.abs()
            bar = bar_of(ref, _bound(ref, blk.abs() @ h2.abs() + sp, B * Lq, extra_adds=2 * n_chunks) + sp)
            err = (dw[v0:v0 + 16384].double() - scale * ref).abs()
            assert bool((err <= bar).all()), \
                f'{what} d(weight) rows {v0}+: {int((err > bar).sum())} beyond, max err / bar {float((err / bar).max()):.3f}'


# (B, L, H, V, chunk_rows, loss_scale, upstream scalar, label layout)
OP_CASES = [
    (4, 40, 128, 2053, None, 1.0, 1.0, 'mixed'),
    (4, 40, 128, 32064, None, 0.5, 0.25, 'mixed'),
    (4, 40, 4096, 2053, None, 1.0, 0.3, 'mixed'),
    (4, 40, 4096, 32064, None, 2.0, 1.0, 'mixed'),
    (4, 100, 128, 2053, 128, 1.7, 1.0, 'mixed'),    # ~300 rows in chunks of 128
    (1, 258, 128, 2053, 128, 1.0, 0.3, 'all'),      # 257 rows: 128 + 128 + 1
    (4, 40, 128, 128257, None, 1.0, 1.0, 'mixed'),
    (2, 40, 4096, 128257, None, 1.0, 0.25, 'mixed'),
]


@pytest.mark.parametrize('case', OP_CASES, ids=[f'B{c[0]}-L{c[1]}-H{c[2]}-V{c[3]}-c{c[4]}-s{c[5]}-g{c[6]}' for c in OP_CASES])
def test_causal_lm_loss_from_hidden(ops, case):
    B, Lq, H, V, chunk_rows, loss_scale, up, layout = case
    hidden, weight = _operands(B, Lq, H, V, B * Lq + H + V)
    labels = _labels(B, Lq, V, Lq + V, layout)
    idx, N = ops.causal_lm_valid_rows(labels)
    n_chunks = len(ops._ce_chunks(N, V, chunk_rows))
    if chunk_rows is not None:
        assert n_chunks == -(-N // chunk_rows) and (layout != 'all' or N - (n_chunks - 1) * chunk_rows == 1)
    want = _aten_loss(F.linear(hidden, weight), labels)
    tile = ops.causal_lm_loss(F.linear(hidden, weight), labels)
    h, w = hidden.clone().requires_grad_(True), weight.clone().requires_grad_(True)
    scaled, loss = ops.causal_lm_loss_from_hidden(h, w, labels, loss_scale=loss_scale, chunk_rows=chunk_rows)
    assert loss.dtype == torch.float32 and not loss.requires_grad and scaled.requires_grad
    assert_close_f32(loss, want, what='loss against ATen')
    assert_close_f32(loss, tile, what='loss against causal_lm_loss')
    assert_close_f32(scaled, loss * loss_scale, rtol=1e-7, what='scaled loss')
    (scaled * up).backward()
    _check_grads(hidden, weight, labels, h.grad, w.grad, up * loss_scale, n_chunks, str(case))
    ops.check_status()


def test_frozen_head_no_grad_and_a_second_backward(ops):
    B, Lq, H, V = 4, 40, 128, 2053
    hidden, weight = _operands(B, Lq, H, V, 5)
    labels = _labels(B, Lq, V, 6)
    h, w = hidden.clone().requires_grad_(True), weight.clone().requires_grad_(True)
    loss = ops.causal_lm_loss_from_hidden(h, w, labels, chunk_rows=128)[0]
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match='once'):
        loss.backward()
    # frozen head (LoRA SFT): the same d(hidden), bit for bit, and no d(weight)
    h2 = hidden.clone().requires_grad_(True)
    loss2 = ops.causal_lm_loss_from_hidden(h2, weight, labels, chunk_rows=128)[0]
    loss2.backward()
    assert torch.equal(h2.grad, h.grad) and torch.equal(loss2, loss.detach())
    # no_grad, with inputs that require a gradient (a Parameter head at eval): the same loss, no graph, no gradient work
    h3, w3 = hidden.clone().requires_grad_(True), torch.nn.Parameter(weight.clone())
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        loss3, raw3 = ops.causal_lm_loss_from_hidden(h3, w3, labels, chunk_rows=128)
    torch.cuda.synchronize()
    assert not loss3.requires_grad and torch.equal(loss3, loss.detach())
    # the logits chunk (128 rows x ld) and small buffers only: no d(logits) chunk, no d(weight), no fp32 accumulator
    assert torch.cuda.max_memory_allocated() - base < 2 * 128 * _up(V, 256) * 2 + (1 << 20), 'gradient buffers under no_grad'
    assert h3.grad is None and w3.grad is None
    # frozen hidden states: d(weight) only, the same as with both
    w2 = weight.clone().requires_grad_(True)
    ops.causal_lm_loss_from_hidden(hidden, w2, labels, chunk_rows=128)[0].backward()
    assert torch.equal(w2.grad, w.grad)
    ops.check_status()


def test_tied_head_accumulates(ops):
    """The head is the input embedding: d(weight) = the head's share + the embedding's share of d(hidden rows)."""
    B, Lq, H, V = 3, 40, 128, 2053
    gen = torch.Generator().manual_seed(9)
    emb = (torch.randn(V, H, generator=gen) * 0.3).bfloat16().to(DEV)
    ids = torch.randint(0, V, (B, Lq), generator=gen).to(DEV)
    labels = _labels(B, Lq, V, 10)
    mix = torch.randn(H, H, generator=gen).bfloat16().to(DEV) * (1 / H ** 0.5)
    grads = []
    for fused in (True, False):
        w = emb.clone().requires_grad_(True)
        hidden = F.embedding(ids, w) @ mix
        if fused:
            ops.causal_lm_loss_from_hidden(hidden, w, labels)[0].backward()
        else:
            _aten_loss(F.linear(hidden, w), labels).backward()
        grads.append(w.grad.float())
    err = float((grads[0] - grads[1]).abs().max())
    assert err <= 2e-2 * float(grads[1].abs().max()), err


def test_no_valid_row_and_bad_operands(ops):
    B, Lq, H, V = 2, 16, 128, 2053
    hidden, weight = _operands(B, Lq, H, V, 11)
    labels = torch.full((B, Lq), IGN, dtype=torch.int64, device=DEV)
    labels[:, 0] = 3  # position 0 is never a target
    want = ops.causal_lm_loss(F.linear(hidden, weight), labels)
    h, w = hidden.clone().requires_grad_(True), weight.clone().requires_grad_(True)
    scaled, loss = ops.causal_lm_loss_from_hidden(h, w, labels)
    torch.testing.assert_close(loss, want, equal_nan=True, rtol=0, atol=0)
    scaled.backward()
    assert bool((h.grad == 0).all()) and bool((w.grad == 0).all())
    with pytest.raises(ValueError, match='bf16'):
        ops.causal_lm_loss_from_hidden(hidden.float(), weight.float(), labels)
    with pytest.raises(ValueError, match='divisible by 64'):
        ops.causal_lm_loss_from_hidden(hidden[..., :96], weight[:, :96], labels)


# ---- the trainer -----------------------------------------------------------------------------------------------------
def _run_sft(fused, hidden, weight, labels, chunk_rows=None):
    from align_anything_b200.trainers.text_to_text.sft import SupervisedTrainer

    h, w = hidden.clone().requires_grad_(True), weight.clone().requires_grad_(True)
    tr = SupervisedTrainer(None, LM(h, w))
    tr.fused_lm_head, tr.lm_head_chunk_rows = fused, chunk_rows
    ids = torch.where(labels == IGN, torch.zeros_like(labels), labels)
    out = tr.train_step({'input_ids': ids, 'labels': labels, 'attention_mask': torch.ones_like(labels, dtype=torch.bool)})
    return out, h.grad, w.grad


@pytest.mark.parametrize('V', [2053, 128257])
def test_sft_trainer_fused_lm_head(ops, V):
    B, Lq, H = 4, 48, 256
    hidden, weight = _operands(B, Lq, H, V, 21)
    labels = _labels(B, Lq, V, 22)
    a, b = (_run_sft(fused, hidden, weight, labels, chunk_rows=64) for fused in (False, True))
    assert set(a[0]) == set(b[0]) == {'train/loss', 'train/lr'}
    assert abs(a[0]['train/loss'] - b[0]['train/loss']) <= 5e-5 * max(1.0, abs(a[0]['train/loss'])), (a[0], b[0])
    for i, what in ((1, 'd hidden'), (2, 'd weight')):
        err = float((b[i].float() - a[i].float()).abs().max())
        assert err <= 2e-2 * float(a[i].float().abs().max()), (what, err)
    ops.check_status()


def test_sft_out_of_range_label_raises_like_the_tile_path(ops):
    B, Lq, H, V = 2, 24, 128, 2053
    hidden, weight = _operands(B, Lq, H, V, 31)
    labels = _labels(B, Lq, V, 32)
    labels[0, 10] = V + 3
    for fused in (False, True):
        with pytest.raises(IndexError):
            _run_sft(fused, hidden, weight, labels)
        assert ops.check_status() == 0  # raise_for_status reset the status word
