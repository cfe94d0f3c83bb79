"""GSPO's sequence-level ratio on the H100 (DESIGN §4.8): aa_grpo_loss_seq through the C ABI against the port
(tests/gspo_port.py) on guarded buffers, the first update's launches, rows whose ratio crosses GSPO's bounds, the
composed path of grpo_loss_from_logits without K1f, and the trainer's update loop against float64 autograd of the port,
on the fused lm_head path and at one update."""
from __future__ import annotations

from types import SimpleNamespace

import pytest
import torch

import gspo_port as port
from grpo_objective_port import completion_mask
from test_gpu_entropy import _bits
from test_gpu_grpo_objective import AGG, EOS, SGD
from test_gpu_parity import _ordered_bits, assert_ulp_close, ops  # noqa: F401  (fixture)
from test_gpu_ppo_objective import Guarded, _rel

pytestmark = pytest.mark.gpu

DEV = 'cuda'
KL = {'k1': 0, 'k2': 1, 'k3': 2}
# (clip_low, clip_high, dual_clip, loss_agg_mode, kl_estimator): each aggregation, dual-clip, each estimator, GSPO's
# published clip range
OPTIONS = {
    'token-mean': (0.2, 0.28, None, 'token-mean', 'k3'),
    'seq-mean': (0.2, 0.28, None, 'seq-mean-token-mean', 'k3'),
    'sum-norm': (0.2, 0.28, None, 'seq-mean-token-sum-norm', 'k3'),
    'dual-clip': (0.2, 0.28, 3.0, 'token-mean', 'k3'),
    'k1': (0.2, 0.28, 3.0, 'seq-mean-token-mean', 'k1'),
    'k2': (0.2, 0.28, None, 'seq-mean-token-sum-norm', 'k2'),
    'gspo': (3e-4, 4e-4, None, 'seq-mean-token-mean', 'k3'),
}


def _inputs(B, K, dtype, seed):
    """Log-probs and old log-probs on the grid of 2^-6 in [-4, 0): every lp - old is exact in each dtype and every
    order of the fp32 row sum gives the same S, so the kernel and ATen start the ratio from the same bits.  Rows are
    shifted by different amounts (w inside and outside the clip ranges), and have different lengths."""
    g = torch.Generator().manual_seed(seed)
    q = lambda t: (t * 64).round() / 64  # noqa: E731
    lp = q(-torch.rand(B, K, generator=g) * 3.9 - 0.05)
    shift = torch.tensor([0.0, 0.125, -0.125, 0.5, -0.5, 2 ** -6, -2 ** -6])[torch.arange(B) % 7].unsqueeze(-1)
    old = q((lp - shift + torch.randn(B, K, generator=g) * 0.05).clamp(-3.98, -0.02))
    ref = lp + torch.randn(B, K, generator=g) * 0.3
    adv = torch.randn(B, 1, generator=g)
    adv = torch.where(adv.abs() < 0.25, adv.sign() * 0.25 + 0.25 * (adv == 0), adv)
    adv[3], adv[B - 3] = adv[3].abs(), -adv[B - 3].abs()  # w far above 1 with A > 0, far below with A < 0: clipped
    tokens = torch.randint(2, 50, (B, K), generator=g)
    tokens[0, 5] = EOS
    tokens[2, 0] = EOS
    tokens[3, K - 1] = EOS
    return (lp.to(dtype).to(DEV), ref.to(dtype).to(DEV), old.to(dtype).to(DEV), adv.to(DEV), tokens.to(DEV))


def _seq_c_abi(lp, ref, old, adv, tokens, beta, opt, mode):
    """aa_grpo_loss_seq through the C ABI on guarded, NaN-fenced buffers -> (loss, grad, clip fractions, row_end)."""
    from align_anything_b200 import _lib as L

    B, K = lp.shape
    lo, hi, c, agg, est = opt
    mode_code = L.MODE_FAITHFUL if mode == 'faithful' else L.MODE_F32
    gl, gr, go = Guarded(lp), Guarded(ref), Guarded(old)
    gt = SimpleNamespace(view=tokens.contiguous())
    ga = Guarded(adv.view(1, B).contiguous())
    grad = Guarded(torch.zeros_like(lp))
    loss = Guarded(torch.zeros(1, 1, dtype=torch.float32, device=DEV))
    cf = Guarded(torch.zeros(1, 2, dtype=torch.float32, device=DEV))
    row_end = Guarded(torch.zeros(1, B, dtype=torch.int32, device=DEV), fill=-7)
    scratch = torch.full((1 + 4 * B,), float('nan'), dtype=torch.float32, device=DEV)
    counter = torch.zeros(2, dtype=torch.int32, device=DEV)
    L.check(L.lib().aa_grpo_loss_seq(
        gl.view.data_ptr(), gl.view.stride(0), gr.view.data_ptr(), gr.view.stride(0), go.view.data_ptr(),
        go.view.stride(0), L.dtype_code(lp.dtype), ga.view.data_ptr(), gt.view.data_ptr(), gt.view.stride(0), EOS, B, K,
        float(beta), float(lo), float(hi), float(c or 0.0), AGG[agg], KL[est], mode_code, loss.view.data_ptr(),
        grad.view.data_ptr(), grad.view.stride(0), cf.view.data_ptr(), row_end.view.data_ptr(), scratch.data_ptr(),
        counter.data_ptr(), L.stream_ptr(DEV)))
    torch.cuda.synchronize()
    for g in (gl, gr, go, ga, grad, loss, cf, row_end):
        assert g.intact(), 'a guard band was written'
    return loss.view[0, 0].clone(), grad.view.clone(), cf.view[0].clone(), row_end.view[0].clone()


def _port(lp, ref, old, adv, mask, beta, opt, cd):
    lo, hi, c, agg, est = opt
    x = lp.to(cd).clone().requires_grad_(True)
    want = port.grpo_loss(x, ref.to(cd), adv, mask, beta, old.to(cd), lo, hi, c, agg, est)
    want.backward()
    return want.detach(), x.grad


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize('mode', ['faithful', 'f32'])
@pytest.mark.parametrize('name', list(OPTIONS))
def test_grpo_loss_seq_c_abi_vs_port(ops, dtype, mode, name):
    lo, hi, c, agg, est = opt = OPTIONS[name]
    B, K = 14, 301
    lp, ref, old, adv, tokens = _inputs(B, K, dtype, seed=list(OPTIONS).index(name))
    loss, grad, cf, row_end = _seq_c_abi(lp, ref, old, adv, tokens, 0.04, opt, mode)
    mask = completion_mask(tokens, EOS)
    assert torch.equal(row_end.long(), mask.sum(-1))
    faithful = mode == 'faithful' and dtype != torch.float32
    cd = dtype if faithful else torch.float32  # the port on ATen CUDA in the dtype the kernel rounds to
    want, gwant = _port(lp, ref, old, adv, mask, 0.04, opt, cd)
    assert want.dtype == torch.float32
    torch.testing.assert_close(loss, want, rtol=2e-5, atol=1e-7)
    if dtype == torch.float32:
        torch.testing.assert_close(grad, gwant, rtol=2e-5, atol=2e-5 * float(gwant.abs().max()))
    else:  # F32 mode keeps fp32 throughout and rounds the gradient once, to the log-probs' dtype
        gw = gwant if faithful else gwant.to(dtype)
        d = (_ordered_bits(grad.cpu()) - _ordered_bits(gw.cpu())).abs()
        print(f'{name} {dtype} {mode}: {float((d == 0).double().mean()):.4f} of the gradient bit-identical')
        assert_ulp_close(grad, gw, max_ulp=1, min_exact=0.97, what=f'{name} grad')
    # every counted token of a row shares w: the fractions count clipped rows, or the tokens in them
    fc, fd = port.clip_fractions(lp.to(cd), old.to(cd), adv, mask, lo, hi, c, agg)
    assert abs(float(cf[0]) - fc) <= 1e-6, (float(cf[0]), fc)
    assert abs(float(cf[1]) - fd) <= 1e-6, (float(cf[1]), fd)
    if c is None:
        assert float(cf[1]) == 0.0
    assert 0.0 < fc < 1.0 or name == 'gspo'  # some rows clipped, some not


def test_gspo_bounds_zero_the_clipped_rows(ops):
    """Half of the rows get old log-probs shifted by a constant 2^-6 (|log w| = 2^-6, far outside [1 - 3e-4, 1 + 4e-4]),
    the other half one token shifted (|log w| = 2^-6 / n, inside): with beta = 0 the gradient is zero exactly on the
    rows the port clips, in fp32, though both bounds round to 1 in bf16."""
    B, K = 16, 257
    opt = (3e-4, 4e-4, None, 'token-mean', 'k3')
    lp, ref, _, adv, tokens = _inputs(B, K, torch.bfloat16, seed=11)
    sign = torch.where(torch.arange(B, device=DEV) % 4 < 2, 1.0, -1.0).unsqueeze(-1)
    adv[0], adv[2] = adv[0].abs(), -adv[2].abs()  # rows the clip must zero
    old = lp.float() - sign * 2 ** -6
    old[1::2, 1:] = lp.float()[1::2, 1:]
    old = old.to(torch.bfloat16)
    mask = completion_mask(tokens, EOS)
    _, grad, cf, _ = _seq_c_abi(lp, ref, old, adv, tokens, 0.0, opt, 'faithful')
    _, gwant = _port(lp, ref, old, adv, mask, 0.0, opt, torch.bfloat16)
    w = torch.exp(port.sequence_log_weights(lp, old, mask))
    outside = (w < 1 - 3e-4) | (w > 1 + 4e-4)
    assert outside[0::2].all() and not outside[1::2].any()
    zero = (gwant == 0).all(-1)
    assert zero.any() and not zero.all()
    assert torch.equal((grad == 0).all(-1), zero)
    assert_ulp_close(grad, gwant, max_ulp=1, min_exact=0.97, what='gspo bounds grad')
    fc, _ = port.clip_fractions(lp, old, adv, mask, 3e-4, 4e-4, None, 'token-mean')
    assert abs(float(cf[0]) - fc) <= 1e-6


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize('mode', ['faithful', 'f32'])
def test_first_update_is_the_token_level_objective(ops, dtype, mode):
    from align_anything_b200.ops import GrpoObjective

    lp, ref, _, adv, tokens = _inputs(5, 129, dtype, seed=7)
    for fields in ({}, dict(clip_range_ratio_high=0.28, dual_clip_ratio=3.0, loss_agg_mode='seq-mean-token-mean',
                            kl_estimator='k2')):
        outs = []
        for level in ('token', 'sequence'):
            x = lp.clone().requires_grad_(True)
            got = ops.grpo_loss(x, ref, adv, tokens, EOS, 0.04, mode=mode, return_clip_fraction=True,
                                objective=GrpoObjective(importance_sampling_level=level, **fields))
            got[0].backward()
            outs.append((got[0].detach(), x.grad, got[2]))
        (a, ga, ca), (b, gb, cb) = outs
        assert torch.equal(_bits(a), _bits(b)) and torch.equal(_bits(ga), _bits(gb)) and torch.equal(ca, cb)
        assert float(cb.abs().sum()) == 0.0


def _grpo_node(ops, logits, ids, K, ref, adv, mode, **kw):
    leaf = logits.clone().requires_grad_(True)
    out = ops.grpo_loss_from_logits(leaf, ids, K, ref, adv, EOS, 0.04, mode=mode, **kw)
    out[0].backward()
    return out, leaf.grad


@pytest.mark.parametrize('dtype,mode', [(torch.bfloat16, 'faithful'), (torch.bfloat16, 'f32'), (torch.float32, 'f32')])
def test_sequence_level_from_logits_takes_the_composed_path(ops, monkeypatch, dtype, mode):
    from align_anything_b200.ops import GrpoObjective

    V, B, Lq, K = 152064, 4, 14, 9
    torch.manual_seed(19)
    logits = (torch.randn(B, Lq, V, device=DEV) * 2.0).to(dtype)
    ids = torch.randint(2, V, (B, Lq), device=DEV)
    ids[1, Lq - K + 4] = EOS
    ids[2, Lq - K] = EOS
    adv = torch.tensor([[1.5], [-0.7], [0.4], [-2.0]], device=DEV)
    ref = ops.tail_token_log_probs(logits, ids, K, mode=mode).float()
    lp0 = ops.tail_token_log_probs(logits, ids, K, mode=mode)
    old = (lp0.float() - torch.tensor([[0.0], [0.1], [-0.002], [0.6]], device=DEV)).to(lp0.dtype)
    obj = GrpoObjective(0.2, 0.28, 3.0, 'seq-mean-token-mean', importance_sampling_level='sequence')

    def no_k1f(*a, **kw):
        raise AssertionError('K1f launched for a sequence-level objective with old log-probs')

    monkeypatch.setattr(ops, '_k1f_grpo_launch', no_k1f)
    kw = dict(objective=obj, old_per_token_logps=old, return_clip_fraction=True)
    one, gone = _grpo_node(ops, logits, ids, K, ref, adv, mode, **kw)
    # K1 -> ops.grpo_loss -> K1b on the same inputs
    leaf = logits.clone().requires_grad_(True)
    lp = ops.tail_token_log_probs(leaf, ids, K, mode=mode)
    two = ops.grpo_loss(lp, ref, adv, ids[:, -K:], EOS, 0.04, mode=mode, **kw)
    two[0].backward()
    assert torch.equal(_bits(one[0].detach()), _bits(two[0].detach()))
    assert torch.equal(_bits(one[1]), _bits(lp.detach())) and torch.equal(one[2], two[1])
    assert torch.equal(_bits(gone), _bits(leaf.grad)) and torch.equal(one[-1], two[-1])
    ops.check_status()


GSPO = dict(num_iterations=2, importance_sampling_level='sequence', clip_range_ratio_low=3e-4,
            clip_range_ratio_high=4e-4, loss_agg_mode='seq-mean-token-mean', log_clip_fraction=True)


def _run(fused, seq, P, H, V, seed, lr, **attrs):
    from test_gpu_fused_rl import LM

    from align_anything_b200.trainers.text_to_text.grpo import GRPOTrainer

    gen = torch.Generator().manual_seed(seed)
    B, Lq = seq.shape
    hid = torch.randn(B, Lq, H, generator=gen).bfloat16().to(DEV)
    hid_r = torch.randn(B, Lq, H, generator=gen).bfloat16().to(DEV)
    w = (torch.randn(V, H, generator=gen) * 0.2).bfloat16().to(DEV)
    w_r = (w.float().cpu() + torch.randn(V, H, generator=gen) * 0.02).bfloat16().to(DEV)
    rewards = torch.randn(B, generator=gen).to(DEV)
    policy = SGD(hid, w, lr)
    tr = type('GRPO', (GRPOTrainer,), attrs)(None, policy, LM(hid_r, w_r),
                                            SimpleNamespace(pad_token_id=0, eos_token_id=EOS), beta=0.04,
                                            num_generations=2)
    tr.fused_lm_head, tr.lm_head_chunk_rows = fused, 32
    out = tr.step_from_rollout(seq, P, rewards)
    return out, policy, (hid_r, w_r, rewards)


def test_gspo_two_updates_vs_float64(ops, monkeypatch):
    from test_gpu_fused_rl import _grpo_sequences

    seq = _grpo_sequences(7)
    P, H, V, seed = 16, 128, 2053, 47
    K = seq.size(1) - P
    olds = []
    real = ops.grpo_loss_from_logits

    def spy(*a, **kw):
        olds.append(kw.get('old_per_token_logps'))
        return real(*a, **kw)

    monkeypatch.setattr(ops, 'grpo_loss_from_logits', spy)
    out, policy, (hid_r, w_r, rewards) = _run(False, seq, P, H, V, seed, 0.02, mode='f32', **GSPO)
    assert set(out) == {'train/loss', 'train/reward', 'train/actor_clip_fraction'}
    assert len(policy.seen) == len(policy.grads) == 2 and olds[0] is None and olds[1] is not None
    ref = ops.tail_token_log_probs(torch.nn.functional.linear(hid_r, w_r), seq, K, mode='f32').double()
    adv = ops.group_advantages(rewards, 2).double()
    mask = completion_mask(seq[:, -K:], EOS)
    losses = []
    for u, ((h, w), (dh, dw)) in enumerate(zip(policy.seen, policy.grads)):
        hh, ww = h.double().requires_grad_(True), w.double().requires_grad_(True)
        x = torch.nn.functional.linear(h, w).double()  # the bf16 logits the trainer's model returns
        x = x + (torch.nn.functional.linear(hh, ww) - torch.nn.functional.linear(hh, ww).detach())
        lp64 = torch.log_softmax(x[:, :-1][:, -K:], -1).gather(-1, seq[:, -K:, None]).squeeze(-1)
        old = None if olds[u] is None else olds[u].double()
        loss64 = port.grpo_loss(lp64, ref, adv, mask, 0.04, old, 3e-4, 4e-4, None, 'seq-mean-token-mean')
        loss64.backward()
        losses.append(float(loss64))
        if old is not None:
            w64 = torch.exp(port.sequence_log_weights(lp64.detach(), old, mask))
            print(f'update {u + 1}: w = {[round(float(v), 6) for v in w64]}')
        _rel(dh, hh.grad, 2e-2, f'update {u + 1}: d hidden')
        _rel(dw, ww.grad, 2e-2, f'update {u + 1}: d weight')
    assert abs(out['train/loss'] - sum(losses) / 2) <= 1e-4 * max(1.0, abs(sum(losses) / 2))
    h2, w2 = policy.seen[1]
    lp2 = ops.tail_token_log_probs(torch.nn.functional.linear(h2, w2), seq, K, mode='f32').double()
    fc, _ = port.clip_fractions(lp2, olds[1].double(), adv, mask, 3e-4, 4e-4, None, 'seq-mean-token-mean')
    assert abs(out['train/actor_clip_fraction'] - fc / 2) <= 1e-6, (out, fc)  # the first update clips nothing
    ops.check_status()


def test_gspo_two_updates_fused_lm_head_vs_tile_path(ops):
    from test_gpu_fused_rl import _grpo_sequences

    seq = _grpo_sequences(8)
    a, pa, _ = _run(False, seq, 16, 128, 2053, 49, 1e-4, **GSPO)
    b, pb, _ = _run(True, seq, 16, 128, 2053, 49, 1e-4, **GSPO)
    assert set(a) == set(b)
    for k, v in a.items():
        assert abs(v - b[k]) <= 1e-2 * max(1.0, abs(v)), (k, v, b[k])
    for u in range(2):
        _rel(pb.grads[u][0], pa.grads[u][0].double(), 2e-2, f'update {u + 1}: fused d hidden')
        _rel(pb.grads[u][1], pa.grads[u][1].double(), 2e-2, f'update {u + 1}: fused d weight')
    ops.check_status()


def test_single_update_at_either_level_is_the_plain_trainer(ops):
    from test_gpu_fused_rl import _grpo_sequences

    seq = _grpo_sequences(7)
    for fused in (False, True):
        plain, p0, _ = _run(fused, seq, 16, 128, 2053, 47, 1.0)
        for level in ('token', 'sequence'):
            got, p1, _ = _run(fused, seq, 16, 128, 2053, 47, 1.0, num_iterations=1, importance_sampling_level=level)
            assert got == plain, (fused, level)
            for (a, b), (c, d) in zip(p0.grads, p1.grads):
                assert torch.equal(_bits(a), _bits(c)) and torch.equal(_bits(b), _bits(d)), (fused, level)
    ops.check_status()
