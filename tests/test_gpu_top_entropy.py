"""High-entropy token masking on the H100 (DESIGN §4.10): the exact entropy quantile against CUDA torch.quantile (and
the sort-based restatement past 2^24 values), aa_grpo_loss_topent through the C ABI against the port
(tests/top_entropy_port.py) on guarded buffers, the composed path of grpo_loss_from_logits without K1f, the trainer's
two updates against float64, the fused lm_head path against the tile path, rho = 1 bit for bit, and two ranks."""
from __future__ import annotations

import os
import subprocess
import sys
from types import SimpleNamespace

import pytest
import torch

import top_entropy_port as port
from grpo_objective_port import completion_mask
from test_gpu_entropy import _bits
from test_gpu_grpo_objective import AGG, EOS, SGD  # noqa: F401
from test_gpu_gspo import OPTIONS, _inputs
from test_gpu_parity import _ordered_bits, assert_ulp_close, ops  # noqa: F401  (fixture)
from test_gpu_ppo_objective import Guarded, _rel

pytestmark = pytest.mark.gpu

DEV = 'cuda'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KL = {'k1': 0, 'k2': 1, 'k3': 2}
RHOS = [0.0, 0.2, 0.5, 0.7, 1.0]


def _threshold(ops, ent, counted, q):
    """ops.entropy_quantile_threshold under the sync debugger: the selection makes no host sync."""
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        thr = ops.entropy_quantile_threshold(ent, counted, q)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    return thr


def _same_value(a, b):
    """Equal as values (-0.0 == +0.0), NaN == NaN."""
    a, b = float(a), float(b)
    return a == b or (a != a and b != b)


def _entropies(kind, B, K, gen):
    if kind == 'random':
        return torch.rand(B, K, generator=gen) * 5
    if kind == 'ties':
        return torch.randint(0, 7, (B, K), generator=gen).float() * 0.25
    if kind == 'signed':  # slightly negative entropies from rounding, and both zeros
        e = torch.randn(B, K, generator=gen) * 1e-6
        e[e.abs() < 3e-7] = -0.0
        e[:, ::5] = 0.0
        return e
    raise ValueError(kind)


SIZES = [(1, 1), (1, 2), (3, 17), (32, 512), (128, 8195), (4096, 4096)]


@pytest.mark.parametrize('B,K', SIZES)
@pytest.mark.parametrize('kind', ['random', 'ties', 'signed'])
def test_threshold_equals_cuda_torch_quantile(ops, kind, B, K):
    gen = torch.Generator().manual_seed(B * 7 + K)
    ent = _entropies(kind, B, K, gen).to(DEV)
    if B * K == 4096 * 4096:  # exactly 2^24 counted values: the most torch.quantile takes
        row_end = torch.full((B,), K, dtype=torch.int32, device=DEV)
    else:
        row_end = torch.randint(1, K + 1, (B,), generator=gen, dtype=torch.int32).to(DEV)
    counted = torch.arange(K, device=DEV) < row_end.unsqueeze(1)
    vals = ent[counted]
    for rho in RHOS:
        got = _threshold(ops, ent, row_end, 1.0 - rho)
        want = torch.quantile(vals, 1.0 - rho)
        assert _same_value(got[0], want), (kind, B, K, rho, float(got[0]), float(want))
    # the (B, K) mask form counts the same tokens
    got = _threshold(ops, ent, counted, 0.8)
    assert _same_value(got[0], torch.quantile(vals, 0.8))


def test_threshold_of_kernel_entropies(ops):
    torch.manual_seed(5)
    B, Lq, K, V = 16, 70, 64, 32000
    logits = (torch.randn(B, Lq, V, device=DEV) * 3).bfloat16()
    logits[:4] *= 0.01  # near-uniform rows: entropies near log V; peaked rows near 0 (some may round below 0)
    logits[4:8, :, 7] += 40
    ids = torch.randint(2, V, (B, Lq), device=DEV)
    ids[3, Lq - K + 9] = EOS
    _, ent = ops.tail_token_log_probs(logits, ids, K, return_entropy=True)
    row_end = ops.grpo_row_end(ids[:, -K:], EOS)
    mask = completion_mask(ids[:, -K:], EOS).to(DEV)
    assert torch.equal(row_end.long(), mask.sum(-1))
    for rho in RHOS:
        got = _threshold(ops, ent, row_end, 1.0 - rho)
        assert _same_value(got[0], torch.quantile(ent[mask.bool()], 1.0 - rho)), rho


def test_threshold_beyond_torch_quantile_vs_sort(ops):
    gen = torch.Generator().manual_seed(3)
    B, K = 4352, 4096  # 2^24 + 2^20 counted values: torch.quantile refuses them
    ent = (torch.randint(0, 1 << 20, (B, K), generator=gen).float() * 2 ** -18).to(DEV)
    row_end = torch.full((B,), K, dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match='too large'):
        torch.quantile(ent.reshape(-1), 0.5)
    for q in (0.0, 0.3, 0.8, 0.999, 1.0):
        got = _threshold(ops, ent, row_end, q)
        assert _same_value(got[0], port.quantile_threshold(ent.reshape(-1), q)), q


def test_threshold_nan_and_empty(ops):
    ent = torch.rand(3, 9, device=DEV)
    row_end = torch.tensor([4, 0, 9], dtype=torch.int32, device=DEV)
    ent[1, 2] = float('nan')  # not counted: no effect
    want = torch.quantile(torch.cat([ent[0, :4], ent[2]]), 0.8)
    assert _same_value(_threshold(ops, ent, row_end, 0.8)[0], want)
    ent[2, 3] = float('nan')
    assert torch.isnan(_threshold(ops, ent, row_end, 0.8)[0])
    none = torch.zeros(3, dtype=torch.int32, device=DEV)
    assert torch.isnan(_threshold(ops, ent, none, 0.8)[0])  # N == 0: NaN, nothing is kept


# ---- the masked loss through the C ABI -----------------------------------------------------------------------------
def _topent_c_abi(lp, ref, old, adv, tokens, beta, opt, mode, sequence, ent, thr):
    from align_anything_b200 import _lib as L

    B, K = lp.shape
    lo, hi, c, agg, est = opt
    mode_code = L.MODE_FAITHFUL if mode == 'faithful' else L.MODE_F32
    gl, gr, go, ge = Guarded(lp), Guarded(ref), Guarded(old), Guarded(ent)
    ga = Guarded(adv.view(1, B).contiguous())
    grad = Guarded(torch.zeros_like(lp))
    loss = Guarded(torch.zeros(1, 1, dtype=torch.float32, device=DEV))
    cf = Guarded(torch.zeros(1, 2, dtype=torch.float32, device=DEV))
    row_end = Guarded(torch.zeros(1, B, dtype=torch.int32, device=DEV), fill=-7)
    scratch = torch.full((1 + 4 * B,), float('nan'), dtype=torch.float32, device=DEV)
    counter = torch.zeros(2, dtype=torch.int32, device=DEV)
    tok = tokens.contiguous()
    L.check(L.lib().aa_grpo_loss_topent(
        gl.view.data_ptr(), gl.view.stride(0), gr.view.data_ptr(), gr.view.stride(0), go.view.data_ptr(),
        go.view.stride(0), L.dtype_code(lp.dtype), ga.view.data_ptr(), tok.data_ptr(), tok.stride(0), EOS, B, K,
        float(beta), float(lo), float(hi), float(c or 0.0), AGG[agg], KL[est], int(sequence), mode_code,
        loss.view.data_ptr(), grad.view.data_ptr(), grad.view.stride(0), cf.view.data_ptr(), ge.view.data_ptr(),
        ge.view.stride(0), thr.data_ptr(), row_end.view.data_ptr(), scratch.data_ptr(), counter.data_ptr(),
        L.stream_ptr(DEV)))
    torch.cuda.synchronize()
    for g in (gl, gr, go, ge, ga, grad, loss, cf, row_end):
        assert g.intact(), 'a guard band was written'
    return loss.view[0, 0].clone(), grad.view.clone(), cf.view[0].clone(), row_end.view[0].clone()


def _masked_entropy(B, K, seed):
    """fp32 entropies with ties at a few levels, so the threshold lands on tied values."""
    g = torch.Generator().manual_seed(seed)
    e = torch.rand(B, K, generator=g) * 3
    e[:, ::3] = torch.randint(0, 4, (B, (K + 2) // 3), generator=g).float() * 0.75
    return e.to(DEV)


@pytest.mark.parametrize('sequence', [False, True])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32])
@pytest.mark.parametrize('mode', ['faithful', 'f32'])
@pytest.mark.parametrize('name', list(OPTIONS))
def test_grpo_loss_topent_c_abi_vs_port(ops, dtype, mode, name, sequence):
    lo, hi, c, agg, est = opt = OPTIONS[name]
    B, K = 14, 301
    lp, ref, old, adv, tokens = _inputs(B, K, dtype, seed=list(OPTIONS).index(name))
    ent = _masked_entropy(B, K, seed=len(name))
    mask = completion_mask(tokens, EOS)
    thr = ops.entropy_quantile_threshold(ent, ops.grpo_row_end(tokens, EOS), 0.8)
    keep = port.entropy_keep(ent, mask, 0.2, thr=thr)
    assert 0 < int(keep.sum()) < int(mask.sum())
    loss, grad, cf, row_end = _topent_c_abi(lp, ref, old, adv, tokens, 0.04, opt, mode, sequence, ent, thr)
    assert torch.equal(row_end.long(), mask.sum(-1))
    faithful = mode == 'faithful' and dtype != torch.float32
    cd = dtype if faithful else torch.float32
    x = lp.to(cd).clone().requires_grad_(True)
    want = port.grpo_loss(x, ref.to(cd), adv, mask, 0.04, keep, old.to(cd), lo, hi, c, agg, est, sequence)
    want.backward()
    gwant = x.grad
    torch.testing.assert_close(loss, want.detach(), rtol=2e-5, atol=1e-7)
    if dtype == torch.float32:
        torch.testing.assert_close(grad, gwant, rtol=2e-5, atol=2e-5 * float(gwant.abs().max()))
    else:
        gw = gwant if faithful else gwant.to(dtype)
        d = (_ordered_bits(grad.cpu()) - _ordered_bits(gw.cpu())).abs()
        print(f'{name} {dtype} {mode} seq={sequence}: {float((d == 0).double().mean()):.4f} bit-identical')
        assert_ulp_close(grad, gw, max_ulp=1, min_exact=0.97, what=f'{name} grad')
    if not sequence:  # a masked token's gradient is the KL term's alone
        y = lp.to(cd).clone().requires_grad_(True)
        port.grpo_loss(y, ref.to(cd), adv, mask, 0.04, torch.zeros_like(keep), old.to(cd), lo, hi, c, agg, est)\
            .backward()
        off = mask.bool() & ~keep
        if dtype == torch.float32:
            torch.testing.assert_close(grad[off], y.grad[off], rtol=2e-5, atol=2e-5 * float(y.grad.abs().max()))
        else:
            assert_ulp_close(grad[off], (y.grad if faithful else y.grad.to(dtype))[off], max_ulp=1, min_exact=0.97,
                             what='masked grad')
    # the clip fractions count every counted token, kept or not: the unmasked kernel's
    base = ops.grpo_loss(lp, ref, adv, tokens, EOS, 0.04, mode=mode, old_per_token_logps=old, return_clip_fraction=True,
                         objective=ops.GrpoObjective(lo, hi, c, agg, kl_estimator=est,
                                                     importance_sampling_level='sequence' if sequence else 'token'))
    assert torch.equal(cf, base[2])


# ---- the node and the trainer ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype,mode', [(torch.bfloat16, 'faithful'), (torch.bfloat16, 'f32'), (torch.float32, 'f32')])
def test_from_logits_takes_the_composed_path(ops, monkeypatch, dtype, mode):
    V, B, Lq, K = 152064, 4, 14, 9
    torch.manual_seed(19)
    logits = (torch.randn(B, Lq, V, device=DEV) * 2.0).to(dtype)
    ids = torch.randint(2, V, (B, Lq), device=DEV)
    ids[1, Lq - K + 4] = EOS
    adv = torch.tensor([[1.5], [-0.7], [0.4], [-2.0]], device=DEV)
    ref = ops.tail_token_log_probs(logits, ids, K, mode=mode).float()
    obj = ops.GrpoObjective(0.2, 0.28, 3.0, 'seq-mean-token-mean', top_entropy_quantile=0.2)

    def no_k1f(*a, **kw):
        raise AssertionError('K1f launched under the top-entropy mask')

    monkeypatch.setattr(ops, '_k1f_grpo_launch', no_k1f)
    leaf = logits.clone().requires_grad_(True)
    one = ops.grpo_loss_from_logits(leaf, ids, K, ref, adv, EOS, 0.04, mode=mode, objective=obj, return_entropy=True,
                                    return_clip_fraction=True)
    one[0].backward()
    # K1's entropy variant -> threshold -> aa_grpo_loss_topent -> K1b, by hand
    leaf2 = logits.clone().requires_grad_(True)
    lp, ent = ops.tail_token_log_probs(leaf2, ids, K, mode=mode, return_entropy=True)
    two = ops.grpo_loss(lp, ref, adv, ids[:, -K:], EOS, 0.04, mode=mode, objective=obj, entropy=ent,
                        return_clip_fraction=True)
    two[0].backward()
    assert torch.equal(_bits(one[0].detach()), _bits(two[0].detach())) and torch.equal(one[2], two[1])
    assert torch.equal(_bits(leaf.grad), _bits(leaf2.grad)) and torch.equal(one[-1], two[2])
    assert torch.equal(_bits(one[-2]), _bits(ent))
    ops.check_status()


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


TOPENT = dict(num_iterations=2, top_entropy_quantile=0.2, clip_range_ratio_high=0.28, log_clip_fraction=True)


@pytest.mark.parametrize('level', ['token', 'sequence'])
def test_two_updates_vs_float64(ops, monkeypatch, level):
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
    out, policy, (hid_r, w_r, rewards) = _run(False, seq, P, H, V, seed, 0.02, mode='f32',
                                              importance_sampling_level=level, **TOPENT)
    assert len(policy.seen) == 2 and olds[0] is None and olds[1] is not None
    ref = ops.tail_token_log_probs(torch.nn.functional.linear(hid_r, w_r), seq, K, mode='f32').double()
    adv = ops.group_advantages(rewards, 2).double()
    mask = completion_mask(seq[:, -K:], EOS)
    losses = []
    for u, ((h, w), (dh, dw)) in enumerate(zip(policy.seen, policy.grads)):
        logits = torch.nn.functional.linear(h, w)
        _, ent = ops.tail_token_log_probs(logits, seq, K, mode='f32', return_entropy=True)  # the update's own pass
        keep = port.entropy_keep(ent, mask, 0.2)
        assert 0 < int(keep.sum()) < int(mask.sum())
        hh, ww = h.double().requires_grad_(True), w.double().requires_grad_(True)
        x = logits.double() + (torch.nn.functional.linear(hh, ww) - torch.nn.functional.linear(hh, ww).detach())
        lp64 = torch.log_softmax(x[:, :-1][:, -K:], -1).gather(-1, seq[:, -K:, None]).squeeze(-1)
        old = None if olds[u] is None else olds[u].double()
        loss64 = port.grpo_loss(lp64, ref, adv, mask, 0.04, keep, old, 0.2, 0.28, None, 'token-mean', 'k3',
                                level == 'sequence' and old is not None)
        loss64.backward()
        losses.append(float(loss64))
        _rel(dh, hh.grad, 2e-2, f'update {u + 1}: d hidden')
        _rel(dw, ww.grad, 2e-2, f'update {u + 1}: d weight')
    assert abs(out['train/loss'] - sum(losses) / 2) <= 1e-4 * max(1.0, abs(sum(losses) / 2))
    ops.check_status()


def test_two_updates_fused_lm_head_vs_tile_path(ops):
    from test_gpu_fused_rl import _grpo_sequences

    seq = _grpo_sequences(8)
    a, pa, _ = _run(False, seq, 16, 128, 2053, 49, 1e-4, **TOPENT)
    b, pb, _ = _run(True, seq, 16, 128, 2053, 49, 1e-4, **TOPENT)
    assert set(a) == set(b)
    for k, v in a.items():
        assert abs(v - b[k]) <= 1e-2 * max(1.0, abs(v)), (k, v, b[k])
    for u in range(2):
        _rel(pb.grads[u][0], pa.grads[u][0].double(), 2e-2, f'update {u + 1}: fused d hidden')
        _rel(pb.grads[u][1], pa.grads[u][1].double(), 2e-2, f'update {u + 1}: fused d weight')
    ops.check_status()


def test_rho_one_is_the_plain_trainer(ops):
    from test_gpu_fused_rl import _grpo_sequences

    seq = _grpo_sequences(7)
    for fused in (False, True):
        plain, p0, _ = _run(fused, seq, 16, 128, 2053, 47, 1.0)
        got, p1, _ = _run(fused, seq, 16, 128, 2053, 47, 1.0, top_entropy_quantile=1.0)
        assert got == plain, fused
        for (a, b), (c, d) in zip(p0.grads, p1.grads):
            assert torch.equal(_bits(a), _bits(c)) and torch.equal(_bits(b), _bits(d)), fused
    ops.check_status()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_ranks_share_one_threshold(ops):
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr',
           '127.0.0.1', '--master-port', '29543', os.path.join(ROOT, 'tests', 'dist_top_entropy.py')]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and 'TOP ENTROPY DIST OK world=2' in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
