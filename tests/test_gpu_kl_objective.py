"""KL regularisation options on the H100 (DESIGN §4.6): K4's estimator (aa_ppo_prep_kl) and GRPO's
(aa_grpo_loss_kl) through the C ABI against the port (tests/kl_objective_port.py) on guarded buffers, their defaults
against the existing entry points bit for bit, K1f's GRPO node with each estimator against the composed path, the GRPO
trainer with k1 and k2 at mu = 2 against float64 autograd of the port, and text, Multi-PPO (rloo) and image PPO (tail
layout) steps with a k2 / k3 penalty and the adaptive coefficient against float64."""
from __future__ import annotations

from types import SimpleNamespace

import pytest
import torch

import kl_objective_port as port
from grpo_objective_port import completion_mask
from test_gpu_entropy import _bits
from test_gpu_grpo_objective import EOS, OPTIONS, _grpo_node, _inputs, _rel, _run
from test_gpu_parity import assert_ulp_close, ops  # noqa: F401  (fixture)
from test_gpu_ppo_objective import Guarded

pytestmark = pytest.mark.gpu

DEV = 'cuda'
DTYPES = [torch.bfloat16, torch.float16, torch.float32]
KL = {'k1': 0, 'k2': 1, 'k3': 2}
AGG = {'seq-mean-token-mean': 0, 'token-mean': 1, 'seq-mean-token-sum-norm': 2}


# ---- K4 --------------------------------------------------------------------------------------------------------------
def _k4_inputs(B, W, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, W, generator=g) * 4
    ref = lp + torch.randn(B, W, generator=g) * 0.5
    values = torch.randn(B, W, generator=g)
    mask = torch.ones(B, W, dtype=torch.bool)
    for b in range(B):
        mask[b, W - 1 - 7 * b:] = False if b else True  # rows end at different positions
    reward = torch.randn(B, generator=g) * 3
    return (lp.to(dtype).to(DEV), ref.to(dtype).to(DEV), values.to(dtype).to(DEV), mask.to(DEV), reward.to(DEV))


class _Flat:
    """A contiguous (B, W) output between two NaN-filled guard rows (K4 writes its outputs densely)."""

    def __init__(self, B, W, dtype):
        self.buf = torch.full(((B + 2) * W,), float('nan'), dtype=dtype, device=DEV)
        self.view = self.buf[W:(B + 1) * W].view(B, W)
        self.W = W

    def intact(self) -> bool:
        return bool(torch.isnan(self.buf[:self.W]).all() and torch.isnan(self.buf[-self.W:]).all())


def _k4_c_abi(lp, ref, values, mask, reward, coeff, est, mode):
    """aa_ppo_prep_kl (est given) or aa_ppo_prep (est None) on guarded buffers -> (old_rewards, adv, ret, row_stats)."""
    from align_anything_b200 import _lib as L

    B, W = lp.shape
    faithful = mode == 'faithful'
    rew_dtype = lp.dtype if faithful else torch.float32
    adv_dtype = lp.dtype if faithful else torch.float32
    gl, gr, gv = Guarded(lp), Guarded(ref), Guarded(values)
    gm = SimpleNamespace(view=mask.contiguous())
    out = _Flat(B, W, rew_dtype)
    adv = _Flat(B, W, adv_dtype)
    ret = _Flat(B, W, adv_dtype)
    stats = _Flat(B, 8, torch.float32)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    head = (gl.view.data_ptr(), gr.view.data_ptr(), L.dtype_code(lp.dtype), gl.view.stride(0), reward.data_ptr(),
            gv.view.data_ptr(), L.dtype_code(values.dtype), gv.view.stride(0), gm.view.data_ptr(), gm.view.stride(0),
            B, W, 0, float(coeff))
    tail = (10.0, 1.0, 0.95, L.MODE_FAITHFUL if faithful else L.MODE_F32, out.view.data_ptr(), L.dtype_code(rew_dtype),
            adv.view.data_ptr(), ret.view.data_ptr(), L.dtype_code(adv_dtype), stats.view.data_ptr(), status.data_ptr(),
            L.stream_ptr(DEV))
    lib = L.lib()
    if est is None:
        L.check(lib.aa_ppo_prep(*head, *tail))
    else:
        L.check(lib.aa_ppo_prep_kl(*head, KL[est], *tail))
    torch.cuda.synchronize()
    for g in (gl, gr, gv, out, adv, ret, stats):
        assert g.intact(), 'a guard band was written'
    return out.view.clone(), adv.view.clone(), ret.view.clone(), stats.view.clone()


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('mode', ['faithful', 'f32'])
@pytest.mark.parametrize('est', list(KL))
def test_k4_estimator_c_abi_vs_port(ops, dtype, mode, est):
    lp, ref, values, mask, reward = _k4_inputs(6, 203, dtype, seed=KL[est])
    rew, adv, ret, stats = _k4_c_abi(lp, ref, values, mask, reward, 0.3, est, mode)
    faithful = mode == 'faithful' and dtype != torch.float32
    cd = dtype if faithful else torch.float32
    want = port.kl_rewards(reward, lp.to(cd), ref.to(cd), mask, 0.3, 10.0, est)
    if faithful:
        assert_ulp_close(rew, want, max_ulp=1, min_exact=0.97, what=f'{est} rewards')
    else:
        torch.testing.assert_close(rew, want, rtol=2e-5, atol=2e-5)
    # the metric lane keeps the k1 row sum under every estimator: the bits of aa_ppo_prep's
    base = _k4_c_abi(lp, ref, values, mask, reward, 0.3, None, mode)
    assert torch.equal(_bits(stats[:, 0]), _bits(base[3][:, 0])) and torch.equal(stats[:, 2], base[3][:, 2])
    if est == 'k1':  # the default estimator through the new entry point: every output bit-identical
        for a, b in zip((rew, adv, ret, stats), base):
            assert torch.equal(_bits(a), _bits(b))


def test_k4_through_ops_defaults_and_estimators(ops):
    lp, ref, values, mask, reward = _k4_inputs(5, 97, torch.bfloat16, seed=11)
    a = ops.kl_rewards_and_gae(reward, lp, ref, values, mask, 3, 0.1, 10.0, 1.0, 0.95)
    b = ops.kl_rewards_and_gae(reward, lp, ref, values, mask, 3, 0.1, 10.0, 1.0, 0.95, kl_estimator='k1')
    for x, y in zip(a, b):
        assert torch.equal(_bits(x), _bits(y))
    c = ops.kl_rewards_and_gae(reward, lp, ref, values, mask, 3, 0.1, 10.0, 1.0, 0.95, kl_estimator='k3')
    assert torch.equal(_bits(c[3][:, 0]), _bits(a[3][:, 0]))
    assert_ulp_close(c[0], port.kl_rewards(reward, lp, ref, mask, 0.1, 10.0, 'k3'), max_ulp=1, min_exact=0.97,
                     what='k3 rewards')
    with pytest.raises(ValueError, match='kl_estimator'):
        ops.kl_rewards_and_gae(reward, lp, ref, values, mask, 3, 0.1, 10.0, 1.0, 0.95, kl_estimator='abs')
    ops.check_status()


# ---- GRPO's loss kernel --------------------------------------------------------------------------------------------
def _grpo_c_abi(lp, ref, old, adv, tokens, beta, opt, est, mode):
    """aa_grpo_loss_kl (est given) or aa_grpo_loss_obj (est None) on guarded buffers -> (loss, grad, cf, row_end)."""
    from align_anything_b200 import _lib as L

    B, K = lp.shape
    lo, hi, c, agg = opt
    gl, gr = Guarded(lp), Guarded(ref)
    go = Guarded(old) if old is not None else None
    ga = Guarded(adv.view(1, B).contiguous())
    grad = Guarded(torch.zeros_like(lp))
    loss = Guarded(torch.zeros(1, 1, dtype=torch.float32, device=DEV))
    cf = Guarded(torch.zeros(1, 2, dtype=torch.float32, device=DEV))
    row_end = Guarded(torch.zeros(1, B, dtype=torch.int32, device=DEV), fill=-7)
    scratch = torch.full((1 + 4 * B,), float('nan'), dtype=torch.float32, device=DEV)
    counter = torch.zeros(2, dtype=torch.int32, device=DEV)
    tok = tokens.contiguous()
    head = (gl.view.data_ptr(), gl.view.stride(0), gr.view.data_ptr(), gr.view.stride(0),
            go.view.data_ptr() if go else None, go.view.stride(0) if go else 0, L.dtype_code(lp.dtype),
            ga.view.data_ptr(), tok.data_ptr(), tok.stride(0), EOS, B, K, float(beta), float(lo), float(hi),
            float(c or 0.0), AGG[agg])
    tail = (L.MODE_FAITHFUL if mode == 'faithful' else L.MODE_F32, loss.view.data_ptr(), grad.view.data_ptr(),
            grad.view.stride(0), cf.view.data_ptr(), row_end.view.data_ptr(), scratch.data_ptr(), counter.data_ptr(),
            L.stream_ptr(DEV))
    lib = L.lib()
    if est is None:
        L.check(lib.aa_grpo_loss_obj(*head, *tail))
    else:
        L.check(lib.aa_grpo_loss_kl(*head, KL[est], *tail))
    torch.cuda.synchronize()
    for g in (gl, gr, ga, grad, loss, cf, row_end) + ((go,) if go else ()):
        assert g.intact(), 'a guard band was written'
    return loss.view[0, 0].clone(), grad.view.clone(), cf.view[0].clone(), row_end.view[0].clone()


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('mode', ['faithful', 'f32'])
@pytest.mark.parametrize('est', list(KL))
@pytest.mark.parametrize('name', ['clip', 'all'])
def test_grpo_loss_kl_c_abi_vs_port(ops, dtype, mode, est, name):
    lo, hi, c, agg = opt = OPTIONS[name]
    B, K = 7, 301
    lp, ref, old, adv, tokens = _inputs(B, K, dtype, seed=3 + KL[est])
    loss, grad, cf, row_end = _grpo_c_abi(lp, ref, old, adv, tokens, 0.04, opt, est, mode)
    mask = completion_mask(tokens, EOS)
    assert torch.equal(row_end.long(), mask.sum(-1))
    faithful = mode == 'faithful' and dtype != torch.float32
    cd = dtype if faithful else torch.float32
    x = lp.to(cd).clone().requires_grad_(True)
    want = port.grpo_loss(x, ref.to(cd), adv, mask, 0.04, est, old.to(cd), lo, hi, c, agg)
    want.backward()
    torch.testing.assert_close(loss, want.detach(), rtol=2e-5, atol=1e-7)
    if faithful:
        assert_ulp_close(grad, x.grad, max_ulp=1, min_exact=0.97, what=f'{est} {name} grad')
    elif dtype == torch.float32:
        torch.testing.assert_close(grad, x.grad, rtol=2e-5, atol=2e-5 * float(x.grad.abs().max()))
    else:
        assert_ulp_close(grad, x.grad.to(dtype), max_ulp=1, min_exact=0.97, what=f'{est} {name} grad')
    if est == 'k3':  # the default estimator through the new entry point: the bits of aa_grpo_loss_obj
        base = _grpo_c_abi(lp, ref, old, adv, tokens, 0.04, opt, None, mode)
        for a, b in zip((loss, grad, cf, row_end), base):
            assert torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize('dtype,mode', [(torch.bfloat16, 'faithful'), (torch.bfloat16, 'f32'), (torch.float32, 'f32')])
def test_k1f_grpo_estimators_vs_composed_path(ops, monkeypatch, dtype, mode):
    from align_anything_b200.ops import GrpoObjective

    V, B, Lq, K = 152064, 4, 14, 9
    torch.manual_seed(23)
    logits = (torch.randn(B, Lq, V, device=DEV) * 2.0).to(dtype)
    ids = torch.randint(2, V, (B, Lq), device=DEV)
    ids[1, Lq - K + 4] = EOS
    adv = torch.tensor([[1.5], [-0.7], [0.4], [-2.0]], device=DEV)
    # reference log-probs a visible distance from the policy's, so every estimator's gradient term is non-trivial
    ref = (ops.tail_token_log_probs(logits, ids, K, mode=mode).float()
           + torch.randn(B, K, device=DEV) * 0.5).clamp(max=0.0)
    base, _ = _grpo_node(ops, logits, ids, K, ref, adv, mode)
    for est in ('k1', 'k2', 'k3'):
        for opts in ({}, {'clip_range_ratio_high': 0.28, 'loss_agg_mode': 'seq-mean-token-mean'}):
            for coeff in (0.0, 0.05):
                obj = GrpoObjective(kl_estimator=est, **opts)
                kw = dict(objective=obj, **({'entropy_coeff': coeff} if coeff else {}))
                one, gone = _grpo_node(ops, logits, ids, K, ref, adv, mode, **kw)
                assert torch.equal(_bits(one[1]), _bits(base[1])), f'{est}: log-probs differ'
                monkeypatch.setattr(ops, '_FUSED_GRPO', False)
                two, gtwo = _grpo_node(ops, logits, ids, K, ref, adv, mode, **kw)
                monkeypatch.setattr(ops, '_FUSED_GRPO', True)
                what = f'{est} {opts} coeff={coeff}'
                if dtype == torch.float32 or mode == 'f32':
                    scale = float(gtwo.float().abs().max())
                    assert float((gone.float() - gtwo.float()).abs().max()) <= 1e-5 * scale + 1e-12, what
                else:
                    assert_ulp_close(gone, gtwo, max_ulp=2, min_exact=0.97, what=what)
                assert float(one[0].detach()) == pytest.approx(float(two[0].detach()), rel=1e-5, abs=1e-7), what
        if est == 'k3':  # k3 with default fields is the reference's node: today's launch, the same bits
            dflt, gd = _grpo_node(ops, logits, ids, K, ref, adv, mode, objective=GrpoObjective(kl_estimator='k3'))
            plain, gp = _grpo_node(ops, logits, ids, K, ref, adv, mode)
            assert torch.equal(_bits(dflt[0].detach()), _bits(plain[0].detach())) and torch.equal(_bits(gd), _bits(gp))
    ops.check_status()


# ---- trainers -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('est', ['k1', 'k2'])
def test_grpo_two_updates_with_an_estimator_vs_float64(ops, monkeypatch, est):
    from test_gpu_fused_rl import _grpo_sequences

    seq = _grpo_sequences(7)
    P, H, V, seed = 16, 128, 2053, 53
    K = seq.size(1) - P
    olds = []
    real = ops.grpo_loss_from_logits

    def spy(*a, **kw):
        olds.append(kw.get('old_per_token_logps'))
        return real(*a, **kw)

    monkeypatch.setattr(ops, 'grpo_loss_from_logits', spy)
    out, policy, (hid_r, w_r, rewards) = _run(False, seq, P, H, V, seed, 0.3, mode='f32', num_iterations=2,
                                              kl_estimator=est)
    assert set(out) == {'train/loss', 'train/reward'}
    ref = ops.tail_token_log_probs(torch.nn.functional.linear(hid_r, w_r), seq, K, mode='f32').double()
    adv = ops.group_advantages(rewards, 2).double()
    mask = completion_mask(seq[:, -K:], EOS)
    losses = []
    for u, ((h, w), (dh, dw)) in enumerate(zip(policy.seen, policy.grads)):
        hh, ww = h.double().requires_grad_(True), w.double().requires_grad_(True)
        x = torch.nn.functional.linear(h, w).double()
        x = x + (torch.nn.functional.linear(hh, ww) - torch.nn.functional.linear(hh, ww).detach())
        lp64 = torch.log_softmax(x[:, :-1][:, -K:], -1).gather(-1, seq[:, -K:, None]).squeeze(-1)
        old = None if olds[u] is None else olds[u].double()
        loss64 = port.grpo_loss(lp64, ref, adv, mask, 0.04, est, old)
        loss64.backward()
        losses.append(float(loss64))
        _rel(dh, hh.grad, 2e-2, f'{est} update {u + 1}: d hidden')
        _rel(dw, ww.grad, 2e-2, f'{est} update {u + 1}: d weight')
    assert abs(out['train/loss'] - sum(losses) / 2) <= 1e-4 * max(1.0, abs(sum(losses) / 2))
    ops.check_status()


def _penalty_checks(out, plain, training, tensors, mask, start, est, gae):
    """The step's KL-shaped rewards, its KL metrics and (gae) its GAE advantages against float64 restatements from the
    rollout's own log-probs and values (F32 mode); the metric dict is the plain step's plus train/kl_coeff."""
    from oracle import ref_port

    assert set(out) == set(plain) | {'train/kl_coeff'} and out['train/kl_coeff'] == 0.02
    lp, ref = training['log_probs'].double(), training['ref_log_probs'].double()
    rew64 = port.kl_rewards(training['reward'].double(), lp, ref, mask, 0.02, 50.0, est)
    _rel(tensors['old_rewards'], rew64, 1e-5, f'{est} shaped rewards')
    m = mask[:, start:]
    assert abs(out['train/kl_divergence'] - port.kl_divergence_metric(lp, ref, mask, start)) <= \
        1e-5 * max(1.0, abs(out['train/kl_divergence']))
    want = float((rew64[:, start:] * m).sum(-1).mean())
    assert abs(out['train/reward_with_kl_penalty'] - want) <= 1e-5 * max(1.0, abs(want))
    if gae:
        adv64, _ = ref_port.gae_advantages_and_returns(training['reward_values'].double(), rew64, mask, start, 1.0,
                                                       0.95)
        _rel(tensors['advantages'], adv64, 1e-4, f'{est} advantages')


@pytest.mark.parametrize('trainer,est', [('text', 'k3'), ('text', 'k2'), ('multi-rloo', 'k2'), ('multi-rloo', 'k3')])
def test_text_ppo_step_with_an_estimator_vs_float64(ops, trainer, est):
    """A text or Multi-PPO (rloo) step with a k2 / k3 penalty and the adaptive coefficient, F32 mode, against float64;
    the plain step for comparison."""
    from test_gpu_fused_rl import _ppo_batch, _run_ppo

    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer as Multi
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer as Text

    cls, kw = (Text, {}) if trainer == 'text' else (Multi, {'advantage_estimator': 'rloo', 'n_samples_per_prompt': 2})
    ids = _ppo_batch(5)
    P, H, V, seed = 12, 128, 2053, 43
    plain = _run_ppo(type('PPO', (cls,), {'mode': 'f32'}), False, ids, P, H, V, seed, **kw)
    on = _run_ppo(type('PPO', (cls,), {'mode': 'f32', 'kl_estimator': est, 'kl_target': 0.01, 'kl_horizon': 64}),
                  False, ids, P, H, V, seed, **kw)
    _penalty_checks(on[1], plain[1], on[0], on[2], (ids != 0)[:, 1:], P - 1, est, gae=trainer == 'text')
    assert on[1]['train/kl_divergence'] == plain[1]['train/kl_divergence']  # the k1 metric, bit for bit
    ops.check_status()


def test_image_ppo_step_tail_layout_with_an_estimator_vs_float64(ops):
    """The image PPO trainer on the tail layout (responses of different lengths) with a k3 penalty and the adaptive
    coefficient, F32 mode, against float64."""
    from test_gpu_fused_rl import LM, Critic, Phased

    from align_anything_b200.models.reward_model import ScoreModelOutput
    from align_anything_b200.trainers.text_image_to_text.ppo import PPOTrainer

    gen = torch.Generator().manual_seed(37)
    B, Lq, H, V = 3, 40, 128, 1031
    resp = [20, 9, 28]
    seq = torch.zeros((B, Lq), dtype=torch.int64)
    for b, r in enumerate(resp):
        seq[b, Lq - r - 8:] = torch.randint(2, V, (r + 8,), generator=gen)
    ids = seq.to(DEV)
    t = lambda *shape, s=1.0: (torch.randn(*shape, generator=gen) * s)  # noqa: E731
    hid_a, hid_r, hid_new = (t(B, Lq, H).bfloat16().to(DEV) for _ in range(3))
    w_a = t(V, H, s=0.2).bfloat16().to(DEV)
    w_r = (w_a.float().cpu() + t(V, H, s=0.02)).bfloat16().to(DEV)
    reward = t(B).to(DEV)
    critic, new_critic = t(B, Lq, 1).to(DEV), t(B, Lq, 1).to(DEV)

    def run(attrs):
        h_new, w_new = hid_new.clone().requires_grad_(True), w_a.clone().requires_grad_(True)
        tr = type('PPO', (PPOTrainer,), attrs)(None, tokenizer=SimpleNamespace(pad_token_id=0))
        state = {'phase': 'rollout'}
        tr.actor_model = Phased(LM(hid_a, w_a), LM(h_new, w_new), state)
        tr.actor_reference_model = LM(hid_r, w_r)
        tr.reward_model = Critic(lambda: ScoreModelOutput(end_scores=reward.unsqueeze(-1)))
        g_critic = new_critic.clone().requires_grad_(True)
        tr.reward_critic_model = Critic(lambda: ScoreModelOutput(scores=critic if state['phase'] == 'rollout' else g_critic))
        inference, training = tr.score_rollout({'input_ids': ids, 'attention_mask': ids != 0}, resp)
        state['phase'] = 'train'
        return training, tr.rl_step(inference, training), tr.last_rl_tensors

    plain = run({'mode': 'f32'})
    on = run({'mode': 'f32', 'kl_estimator': 'k3', 'kl_target': 0.01, 'kl_horizon': 64})
    _penalty_checks(on[1], plain[1], on[0], on[2], on[0]['response_mask'], 0, 'k3', gae=True)
    assert on[1]['train/kl_divergence'] == plain[1]['train/kl_divergence']
    ops.check_status()


def test_text_ppo_step_k3_penalty_with_the_adaptive_coefficient(ops):
    """One text PPO step with a k3 penalty and the adaptive coefficient: the rewards K4 shaped against the port, the
    metric dict of one collective with train/kl_divergence still the k1 sum and train/kl_coeff the step's coefficient."""
    from test_gpu_fused_rl import _ppo_batch, _run_ppo

    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer

    cls = type('PPO', (PPOTrainer,), {'kl_estimator': 'k3', 'kl_target': 0.01, 'kl_horizon': 64})
    ids = _ppo_batch(5)
    P = 12
    training, out, tensors, _, _ = _run_ppo(cls, False, ids, P, 128, 2053, 5, kl_coeff=0.05)
    assert out['train/kl_coeff'] == 0.05
    lp, ref = training['log_probs'], training['ref_log_probs']
    mask = (ids != 0)[:, 1:]
    # the k1 row sums are rounded to bf16 as the reference's `.sum(dim=-1)` rounds them: a few bf16 ulp from float64
    assert out['train/kl_divergence'] == pytest.approx(port.kl_divergence_metric(lp, ref, mask, P - 1), rel=1e-2,
                                                       abs=1e-3)
    want = port.kl_rewards(training['reward'], lp, ref, mask, 0.05, 50.0, 'k3')
    assert_ulp_close(tensors['old_rewards'], want, max_ulp=1, min_exact=0.97, what='k3 shaped rewards')
    base = type('PPO', (PPOTrainer,), {})
    _, plain, _, _, _ = _run_ppo(base, False, ids, P, 128, 2053, 5, kl_coeff=0.05)
    assert 'train/kl_coeff' not in plain and plain['train/kl_divergence'] == out['train/kl_divergence']
    ops.check_status()
