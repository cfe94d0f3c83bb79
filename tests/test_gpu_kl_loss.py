"""The KL term in the PPO actor loss on the H100 (DESIGN §4.7): aa_ppo_actor_loss_kl through the C ABI against the port
(tests/kl_loss_port.py) on guarded buffers, K1f's actor node with the term (aa_logprob_actor_fused_kl) against the
composed path K1 -> K5 -> K1b, and text, Multi-PPO (rloo), image PPO (tail layout, with the entropy bonus), fused
lm_head and kl_coeff = 0 steps against float64 autograd of the port."""
from __future__ import annotations

import pytest
import torch

import kl_loss_port as port
from ppo_objective_port import actor_loss as objective_loss
from ppo_objective_port import masked_mean
from test_gpu_entropy import _bits
from test_gpu_parity import assert_ulp_close, ops  # noqa: F401  (fixture)
from test_gpu_ppo_objective import Guarded, _param_grads, _rel, _with

pytestmark = pytest.mark.gpu

DEV = 'cuda'
AGG = {'seq-mean-token-mean': 0, 'token-mean': 1}
KL = {'k1': 0, 'k2': 1, 'k3': 2}
COEFF = 0.1  # not a power of two: its 16-bit rounding is part of the chain


def _loss_inputs(B, W, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, W, generator=g) * 4
    old = lp + torch.randn(B, W, generator=g) * 0.5
    ref = lp + torch.randn(B, W, generator=g) * 0.5
    adv = torch.randn(B, W, generator=g)
    mask = torch.rand(B, W, generator=g) > 0.2
    mask[:, 0] = True
    mask[-1, W // 2:] = False
    return tuple(t.to(dtype).to(DEV) for t in (lp, old, ref, adv)) + (mask.to(DEV),)


def _k5_kl(lp, old, ref, adv, mask, obj, mode, coeff, est):
    """aa_ppo_actor_loss_kl on guarded buffers -> (loss fp32[2], agg(KL) fp32, grad, clip fractions)."""
    from align_anything_b200 import _lib as L

    B, W = lp.shape
    mode_code = L.MODE_FAITHFUL if mode == 'faithful' else L.MODE_F32
    gl, go, gr, ga = Guarded(lp), Guarded(old), Guarded(ref), Guarded(adv)
    gm = Guarded(mask.to(torch.uint8), fill=1)
    grad = Guarded(torch.zeros_like(lp))
    loss = Guarded(torch.zeros(1, 2, dtype=torch.float32, device=DEV))
    kl = Guarded(torch.zeros(1, 1, dtype=torch.float32, device=DEV))
    cf = Guarded(torch.zeros(1, 2, dtype=torch.float32, device=DEV))
    rows = torch.full((5 * B,), float('nan'), dtype=torch.float32, device=DEV)
    counter = torch.zeros(1, dtype=torch.int32, device=DEV)
    lo, hi, c, agg = obj
    L.check(L.lib().aa_ppo_actor_loss_kl(
        gl.view.data_ptr(), gl.view.stride(0), go.view.data_ptr(), go.view.stride(0), L.dtype_code(lp.dtype),
        ga.view.data_ptr(), ga.view.stride(0), L.dtype_code(adv.dtype), gm.view.data_ptr(), gm.view.stride(0), B, W,
        float(lo), float(hi), float(c or 0.0), AGG[agg], mode_code, gr.view.data_ptr(), gr.view.stride(0), coeff,
        KL[est], loss.view.data_ptr(), kl.view.data_ptr(), grad.view.data_ptr(), grad.view.stride(0),
        cf.view.data_ptr(), rows.data_ptr(), counter.data_ptr(), L.stream_ptr(DEV)))
    torch.cuda.synchronize()
    for g in (gl, go, gr, ga, gm, grad, loss, kl, cf):
        assert g.intact(), 'a guard band was written'
    return loss.view[0].clone(), kl.view[0, 0].clone(), grad.view.clone(), cf.view[0].clone()


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize('mode', ['faithful', 'f32'])
@pytest.mark.parametrize('agg', list(AGG))
@pytest.mark.parametrize('dual', [None, 3.0])
@pytest.mark.parametrize('est', list(KL))
def test_k5_kl_c_abi_vs_port(ops, dtype, mode, agg, dual, est):
    obj = (0.2, 0.28, dual, agg)
    B, W = 7, 301
    lp, old, ref, adv, mask = _loss_inputs(B, W, dtype, seed=KL[est] + 3 * AGG[agg])
    loss, kl, grad, cf = _k5_kl(lp, old, ref, adv, mask, obj, mode, COEFF, est)
    faithful = mode == 'faithful' and dtype != torch.float32
    cd = dtype if faithful else torch.float32  # the port on ATen CUDA in the dtype the kernel rounds to
    x = lp.to(cd).clone().requires_grad_(True)
    total = port.actor_loss(x, old.to(cd), adv.to(cd), mask, 0.2, 0.28, dual, agg, ref_log_probs=ref.to(cd),
                            kl_loss_coeff=COEFF, estimator=est)
    total.backward()
    with torch.no_grad():
        want_loss = objective_loss(lp.to(cd), old.to(cd), adv.to(cd), mask, 0.2, 0.28, dual, agg)
        want_kl = port.kl_loss(lp.to(cd), ref.to(cd), mask, est, agg)
    # the clip fractions and the clipped objective are aa_ppo_actor_loss_obj's
    from test_gpu_ppo_objective import _k5

    base = _k5(ops, lp, old, adv, mask, obj, mode)
    assert torch.equal(_bits(loss), _bits(base[0])) and torch.equal(_bits(cf), _bits(base[2]))
    what = f'{est} {agg} dual={dual}'
    if faithful:
        assert_ulp_close(loss[1:2].view(dtype)[:1].reshape(()), want_loss, max_ulp=1, min_exact=0.0, what=f'{what} loss')
        assert_ulp_close(kl.to(dtype), want_kl, max_ulp=1, min_exact=0.0, what=f'{what} agg(KL)')
        assert_ulp_close(grad, x.grad, max_ulp=1, min_exact=0.97, what=f'{what} grad')
    else:
        torch.testing.assert_close(loss[0], want_loss.float(), rtol=2e-5, atol=0.0)
        torch.testing.assert_close(kl, want_kl.float(), rtol=2e-5, atol=1e-7)
        if dtype == torch.float32:
            torch.testing.assert_close(grad, x.grad, rtol=2e-5, atol=2e-5 * float(x.grad.abs().max()))
        else:  # F32 mode keeps fp32 throughout and rounds the gradient once, to the log-probs' dtype
            assert_ulp_close(grad, x.grad.to(dtype), max_ulp=1, min_exact=0.97, what=f'{what} grad')
    assert bool((grad[~mask] == 0).all())


def test_k5_kl_exact_operands_vs_float64(ops):
    # dyadic log-probs, a ref one k1 / k2 step away, power-of-two counts and coefficient: every op of the fp32 kernel
    # is exact, so it equals float64 bit for bit
    B, W = 4, 64
    g = torch.Generator().manual_seed(5)
    lp = (-torch.randint(1, 64, (B, W), generator=g).float() / 16).to(DEV)
    ref = lp - (torch.randint(-8, 8, (B, W), generator=g).float() / 8).to(DEV)
    adv = (torch.randint(-32, 32, (B, W), generator=g).float() / 8).to(DEV)
    mask = torch.zeros(B, W, dtype=torch.bool, device=DEV)
    for b, n in enumerate((8, 8, 16, 32)):
        mask[b, :n] = True
    for est in ('k1', 'k2'):
        for agg in AGG:
            loss, kl, grad, _ = _k5_kl(lp, lp, ref, adv, mask, (0.2, 0.2, None, agg), 'faithful', 0.25, est)
            x = lp.double().clone().requires_grad_(True)
            total = port.actor_loss(x, lp.double(), adv.double(), mask, 0.2, 0.2, None, agg,
                                    ref_log_probs=ref.double(), kl_loss_coeff=0.25, estimator=est)
            total.backward()
            assert float(kl) == float(port.kl_loss(lp.double(), ref.double(), mask, est, agg)), (est, agg)
            assert torch.equal(grad.double(), x.grad), (est, agg)


# ---- K1f: the single-pass node with the term against the composed path --------------------------------------------
def _node(ops, node, logits, ids, start, lens, old, adv, mask, mode, **kw):
    leaf = logits.clone().requires_grad_(True)
    if node == 'dense':
        out = ops.dense_actor_loss(leaf, ids, start, old, adv, mask, 0.2, mode=mode, **kw)
    else:
        out = ops.tail_actor_loss(leaf, ids, lens, old, adv, mask, 0.2, mode=mode, **kw)
    out[0].backward()
    return out, leaf.grad


VARIANTS = {  # (estimator, objective fields or None, entropy_coeff)
    'k3 alone': ('k3', None, 0.0),
    'k2 all options + bonus': ('k2', (0.2, 0.28, 3.0, 'token-mean'), 0.05),
    'k1 dual-clip + bonus': ('k1', (0.2, 0.2, 3.0, 'seq-mean-token-mean'), 0.05),
}


@pytest.mark.parametrize('V', [152064, 32003])
@pytest.mark.parametrize('node', ['dense', 'tail'])
@pytest.mark.parametrize('dtype,mode', [(torch.bfloat16, 'faithful'), (torch.bfloat16, 'f32'), (torch.float32, 'f32')])
def test_k1f_kl_vs_composed_path(ops, monkeypatch, V, node, dtype, mode):
    from test_gpu_ppo_objective import _node_inputs

    monkeypatch.setattr(ops, '_FUSED_MIN_ROW_BYTES', 0)  # the short vocabulary takes the single pass too
    logits, ids, start, lens, W, mask = _node_inputs(node, dtype, V, seed=V % 97)
    B = logits.size(0)
    plain, _ = _node(ops, node, logits, ids, start, lens, torch.zeros(B, W, device=DEV), torch.zeros(B, W, device=DEV),
                     mask, mode)
    old = (plain[1].float() + torch.randn(B, W, device=DEV) * 0.3).to(plain[1].dtype)
    ref = (plain[1].float() + torch.randn(B, W, device=DEV) * 0.3).to(plain[1].dtype)
    adv = torch.randn(B, W, device=DEV).to(dtype)
    for name, (est, fields, coeff) in VARIANTS.items():
        kw = dict(entropy_coeff=coeff, return_clip_fraction=True)
        if fields is not None:
            kw['objective'] = ops.ActorObjective(*fields)
        base, gbase = _node(ops, node, logits, ids, start, lens, old, adv, mask, mode, **kw)
        kl_kw = dict(kw, ref_log_probs=ref, kl_loss_coeff=COEFF, kl_loss_estimator=est)
        one, gone = _node(ops, node, logits, ids, start, lens, old, adv, mask, mode, **kl_kw)
        again, gagain = _node(ops, node, logits, ids, start, lens, old, adv, mask, mode, **kw)
        what = f'{node} V={V} {name}'
        # the node without the term is unchanged next to it; log-probs, the clipped loss and the clip fractions are its
        assert torch.equal(_bits(gagain), _bits(gbase)) and torch.equal(_bits(again[0].detach()), _bits(base[0].detach()))
        assert torch.equal(_bits(one[1]), _bits(base[1])), f'{what}: log-probs'
        assert torch.equal(_bits(one[2][:1]), _bits(base[2][:1])), f'{what}: actor loss'
        assert torch.equal(one[-1], base[-1]), f'{what}: clip fractions'
        assert len(one) == len(base) + 1
        monkeypatch.setattr(ops, '_FUSED_ACTOR', False)
        two, gtwo = _node(ops, node, logits, ids, start, lens, old, adv, mask, mode, **kl_kw)
        monkeypatch.setattr(ops, '_FUSED_ACTOR', True)
        if dtype == torch.float32 or mode == 'f32':
            scale = float(gtwo.float().abs().max())
            assert float((gone.float() - gtwo.float()).abs().max()) <= 1e-5 * scale + 1e-12, what
        else:
            assert_ulp_close(gone, gtwo, max_ulp=2, min_exact=0.97, what=what)
        zero_rows = lambda g: (g.reshape(-1, V) == 0).all(-1)  # noqa: E731
        assert torch.equal(zero_rows(gone), zero_rows(gtwo)), what
        assert float(one[0]) == pytest.approx(float(two[0]), rel=1e-5, abs=1e-7), what
        assert float(one[-2]) == pytest.approx(float(two[-2]), rel=1e-5, abs=1e-7), what  # agg(KL)
        # the term moves the gradient
        assert not torch.equal(_bits(gone), _bits(gbase)), what
    ops.check_status()


# ---- trainers -------------------------------------------------------------------------------------------------------
def _total64(lp64, old, ref, adv, mask, est, agg='seq-mean-token-mean'):
    return port.actor_loss(lp64, old.double(), adv.double(), mask, 0.2, 0.2, None, agg, ref_log_probs=ref.double(),
                           kl_loss_coeff=COEFF, estimator=est)


def _check_step(out, plain, lp64, old, ref, adv, mask, est, agg, extra64=None):
    """The metric dict (plain's plus train/actor_kl_loss), train/actor_loss the clipped objective, train/actor_kl_loss
    agg(KL), train/kl_divergence the plain step's, all against float64; returns the float64 total for the gradients."""
    assert set(out) == set(plain) | {'train/actor_kl_loss'}
    assert out['train/kl_divergence'] == plain['train/kl_divergence']
    with torch.no_grad():
        want_loss = objective_loss(lp64, old.double(), adv.double(), mask, 0.2, 0.2, None, agg)
        want_kl = port.kl_loss(lp64, ref.double(), mask, est, agg)
    assert abs(out['train/actor_loss'] - float(want_loss)) <= 1e-4 * max(1.0, abs(float(want_loss)))
    assert abs(out['train/actor_kl_loss'] - float(want_kl)) <= 1e-4 * max(1e-2, abs(float(want_kl)))
    total = _total64(lp64, old, ref, adv, mask, est, agg)
    return total if extra64 is None else total + extra64


@pytest.mark.parametrize('trainer,est,agg,kl_coeff', [('text', 'k3', 'seq-mean-token-mean', 0.02),
                                                      ('multi-rloo', 'k2', 'token-mean', 0.02),
                                                      ('text', 'k2', 'seq-mean-token-mean', 0.0)])
def test_text_ppo_step_with_a_kl_loss_term(ops, trainer, est, agg, kl_coeff):
    from test_gpu_fused_rl import _ppo_batch, _run_ppo

    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer as Multi
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer as Text

    cls, kw = (Text, {}) if trainer == 'text' else (Multi, {'advantage_estimator': 'rloo', 'n_samples_per_prompt': 2})
    ids = _ppo_batch(5)
    P, H, V, seed = 12, 128, 2053, 43
    attrs = {'mode': 'f32'} if agg == 'seq-mean-token-mean' else {'mode': 'f32', 'loss_agg_mode': agg}
    plain = _run_ppo(_with(cls, **attrs), False, ids, P, H, V, seed, kl_coeff=kl_coeff, **kw)
    on = _run_ppo(_with(cls, kl_loss_estimator=est, kl_loss_coeff=COEFF, **attrs), False, ids, P, H, V, seed,
                  kl_coeff=kl_coeff, **kw)
    gen = torch.Generator().manual_seed(seed)  # _run_ppo's draws: hid_a, hid_r, hid_new, w_a
    B, Lq = ids.shape
    for _ in range(2):
        torch.randn(B, Lq, H, generator=gen)
    h_new = torch.randn(B, Lq, H, generator=gen).bfloat16().to(DEV)
    w = (torch.randn(V, H, generator=gen) * 0.2).bfloat16().to(DEV)
    start = P - 1
    x = torch.nn.functional.linear(h_new, w).double().requires_grad_(True)
    lp64 = torch.log_softmax(x[:, start:-1], -1).gather(-1, ids[:, start + 1:, None]).squeeze(-1)
    old, ref = on[0]['log_probs'][:, start:], on[0]['ref_log_probs'][:, start:]
    adv, mask = on[2]['advantages'], (ids != 0)[:, 1:][:, start:]
    _check_step(on[1], plain[1], lp64, old, ref, adv, mask, est, agg).backward()
    dh, dw = _param_grads(x.grad, h_new, w)
    _rel(on[3], dh, 2e-2, 'd hidden')
    _rel(on[4], dw, 2e-2, 'd weight')
    ops.check_status()


def test_text_fused_lm_head_step_with_a_kl_loss_term(ops):
    """The fused lm_head node (K6 -> K5 with the term -> K6b) against the tile path, FAITHFUL."""
    from test_gpu_fused_rl import _ppo_batch, _run_ppo

    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer

    ids = _ppo_batch(5)
    cls = _with(PPOTrainer, kl_loss_estimator='k3', kl_loss_coeff=COEFF)
    tile = _run_ppo(cls, False, ids, 12, 128, 2053, 43)
    fused = _run_ppo(cls, True, ids, 12, 128, 2053, 43)
    assert 'train/actor_kl_loss' in tile[1] and set(fused[1]) == set(tile[1])
    for k, v in tile[1].items():
        assert abs(v - fused[1][k]) <= 1e-2 * max(1.0, abs(v)), (k, v, fused[1][k])
    _rel(fused[3], tile[3].double(), 2e-2, 'fused d hidden')
    _rel(fused[4], tile[4].double(), 2e-2, 'fused d weight')
    ops.check_status()


def test_image_ppo_step_tail_layout_with_a_kl_loss_term_and_the_bonus(ops):
    """The image PPO trainer on the tail layout (responses of different lengths), k1 with the entropy bonus, F32."""
    from types import SimpleNamespace

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

    def run(cls):
        h_new, w_new = hid_new.clone().requires_grad_(True), w_a.clone().requires_grad_(True)
        tr = cls(None, tokenizer=SimpleNamespace(pad_token_id=0))
        state = {'phase': 'rollout'}
        tr.actor_model = Phased(LM(hid_a, w_a), LM(h_new, w_new), state)
        tr.actor_reference_model = LM(hid_r, w_r)
        tr.reward_model = Critic(lambda: ScoreModelOutput(end_scores=reward.unsqueeze(-1)))
        g_critic = new_critic.clone().requires_grad_(True)
        tr.reward_critic_model = Critic(lambda: ScoreModelOutput(scores=critic if state['phase'] == 'rollout' else g_critic))
        inference, training = tr.score_rollout({'input_ids': ids, 'attention_mask': ids != 0}, resp)
        state['phase'] = 'train'
        return training, tr.rl_step(inference, training), tr.last_rl_tensors, h_new.grad, w_new.grad

    c_ent = 0.01
    plain = run(_with(PPOTrainer, mode='f32', entropy_coeff=c_ent))
    on = run(_with(PPOTrainer, mode='f32', entropy_coeff=c_ent, kl_loss_estimator='k1', kl_loss_coeff=COEFF))
    x = torch.nn.functional.linear(hid_new, w_a).double().requires_grad_(True)
    W = max(resp)
    lp = torch.zeros(B, W, dtype=torch.float64, device=DEV)
    ent = torch.zeros(B, W, dtype=torch.float64, device=DEV)
    for b, r in enumerate(resp):
        lsm = torch.log_softmax(x[b, Lq - 1 - r:Lq - 1], -1)
        lp[b, :r] = lsm.gather(-1, ids[b, Lq - r:, None]).squeeze(-1)
        ent[b, :r] = -(lsm.exp() * lsm).sum(-1)
    mask = on[0]['response_mask']
    bonus = -c_ent * masked_mean(ent, mask)
    total = _check_step(on[1], plain[1], lp, on[0]['log_probs'], on[0]['ref_log_probs'], on[2]['advantages'], mask,
                        'k1', 'seq-mean-token-mean', bonus)
    total.backward()
    dh, dw = _param_grads(x.grad, hid_new, w_a)
    _rel(on[3], dh, 2e-2, 'd hidden')
    _rel(on[4], dw, 2e-2, 'd weight')
    ops.check_status()
