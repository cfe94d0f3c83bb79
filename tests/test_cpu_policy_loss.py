"""CISPO and SAPO without a GPU: the port (tests/policy_loss_port.py) against a float64 transcription of the two
papers' formulas, the gradient at ratio 1, every refusal on the host and in the C argument checks, the trainer
switches with their config precedence, Safe RLHF-V's refusal, the untouched Clip-Cov call counter and, on the
stand-in library, which entry points each path calls."""
from __future__ import annotations

import ctypes
from types import SimpleNamespace

import pytest
import torch

import policy_loss_port as port
from test_cpu_entropy import fake_reference  # noqa: F401  (fixture)
from test_cpu_plumbing import dry  # noqa: F401  (fixture)
from test_cpu_ppo_step import packed  # noqa: F401  (fixture)

MODES = ('cispo', 'sapo')
PM_KEYS = ('sapo_temperature_pos', 'sapo_temperature_neg')
K1 = ('aa_logprob_fwd', 'aa_logprob_fwd_entropy', 'aa_logprob_bwd', 'aa_logprob_bwd_entropy')
COV = ('aa_cov_moments', 'aa_cov_keys', 'aa_cov_select_hi', 'aa_cov_hist_lo', 'aa_cov_select_lo', 'aa_cov_mark',
       'aa_ppo_actor_loss_cov', 'aa_grpo_loss_cov')


def _paper(mode, lp, old, adv, eps_high=0.2, tau_pos=1.0, tau_neg=1.05):
    """The per-token objectives as the papers write them, in float64 with the gradient stop spelled out:
    CISPO  sg(min(r, 1 + eps_high)) * A * log pi ;  SAPO  f(r) * A with f(r) = sigmoid(tau (r - 1)) * 4 / tau."""
    r = torch.exp(lp - old)
    if mode == 'cispo':
        w = torch.minimum(r, torch.full_like(r, 1.0 + eps_high)).detach()
        return w * adv * lp
    tau = torch.where(adv > 0, torch.full_like(adv, tau_pos), torch.full_like(adv, tau_neg))
    return 4.0 / tau * torch.sigmoid(tau * (r - 1.0)) * adv


def _inputs(B=5, W=17, seed=0):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, W, generator=g, dtype=torch.float64) * 3
    old = lp + torch.randn(B, W, generator=g, dtype=torch.float64) * 0.4
    adv = torch.randn(B, W, generator=g, dtype=torch.float64)
    adv[0, :3] = 0.0
    mask = torch.rand(B, W, generator=g) < 0.8
    mask[:, 0] = True
    return lp, old, adv, mask


@pytest.mark.parametrize('agg', ['seq-mean-token-mean', 'token-mean'])
@pytest.mark.parametrize('mode', MODES)
def test_port_matches_the_papers(mode, agg):
    lp, old, adv, mask = _inputs()
    x = lp.clone().requires_grad_(True)
    y = lp.clone().requires_grad_(True)
    got = port.actor_loss(mode, x, old, adv, mask, agg, 0.28, 1.25, 2.0)  # temperatures exact in fp32
    s = _paper(mode, y, old, adv, 0.28, 1.25, 2.0)
    m = mask.double()
    want = -((s * m).sum(-1) / m.sum(-1)).mean() if agg == 'seq-mean-token-mean' else -(s * m).sum() / m.sum()
    got.backward()
    want.backward()
    assert torch.allclose(got, want, rtol=1e-14, atol=0)
    assert torch.allclose(x.grad, y.grad, rtol=1e-12, atol=1e-15)
    # the closed-form gradients the kernels implement: w * A (CISPO) and 4 sigma (1 - sigma) r A (SAPO)
    r = torch.exp(lp - old)
    if mode == 'cispo':
        ds = torch.clamp(r, max=1.28) * adv
    else:
        tau = torch.where(adv > 0, 1.25, 2.0).double()
        sig = torch.sigmoid(tau * (r - 1))
        ds = 4 * sig * (1 - sig) * r * adv
    coeff = -(m / m.sum(-1, keepdim=True) / m.size(0)) if agg == 'seq-mean-token-mean' else -(m / m.sum())
    assert torch.allclose(x.grad, ds * coeff, rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize('mode', MODES)
def test_gradient_at_ratio_one_is_the_vanilla_gradient(mode):
    lp, _, adv, mask = _inputs(seed=2)
    for agg in ('seq-mean-token-mean', 'token-mean'):
        x = lp.clone().requires_grad_(True)
        port.actor_loss(mode, x, lp, adv, mask, agg).backward()
        v = lp.clone().requires_grad_(True)
        s = adv * torch.exp(v - lp)  # the vanilla objective at ratio 1 (nothing clipped)
        m = mask.double()
        (-((s * m).sum(-1) / m.sum(-1)).mean() if agg == 'seq-mean-token-mean' else -(s * m).sum() / m.sum()).backward()
        assert torch.allclose(x.grad, v.grad, rtol=1e-12, atol=1e-15)
    # GRPO's first update (no old log-probs): d loss / d lp of the policy term is -A * coeff, the KL term added
    re = mask.sum(-1)
    gmask = torch.arange(lp.size(1)) < re.unsqueeze(1)
    a = lp.clone().requires_grad_(True)
    b = lp.clone().requires_grad_(True)
    ref = lp - 0.1
    port.grpo_loss(mode, a, ref, None, adv[:, 0], gmask, 0.04).backward()
    from grpo_objective_port import grpo_loss as vanilla
    vanilla(b, ref, adv[:, :1], gmask, 0.04, clipped=False).backward()
    assert torch.allclose(a.grad, b.grad, rtol=1e-12, atol=1e-15)


def test_cispo_keeps_every_gradient_and_sapo_is_smooth():
    lp = torch.tensor([[-1.0, -1.0, -1.0]], dtype=torch.float64)
    old = lp - torch.tensor([[0.0, 0.5, 3.0]], dtype=torch.float64)  # r = 1, e^0.5, e^3: the last two over 1.2
    adv = torch.tensor([[1.0, 1.0, -1.0]], dtype=torch.float64)
    mask = torch.ones(1, 3, dtype=torch.bool)
    x = lp.clone().requires_grad_(True)
    port.actor_loss('cispo', x, old, adv, mask).backward()
    assert (x.grad != 0).all()  # PPO's clip would zero the second token's gradient
    assert torch.allclose(x.grad[0, 1:], torch.tensor([-1.2, 1.2], dtype=torch.float64) / 3)
    assert port.clip_fraction('cispo', lp, old, adv, mask) == pytest.approx(2 / 3)
    assert port.clip_fraction('sapo', lp, old, adv, mask) == 0.0
    y = lp.clone().requires_grad_(True)
    port.actor_loss('sapo', y, old, adv, mask).backward()
    # the soft gate: every gradient is nonzero, and the far off-policy token's (r = e^3, A < 0) all but vanishes
    assert (y.grad.abs() > 0).all() and y.grad.abs()[0, 2] < 1e-6 * y.grad.abs()[0, 0]


def test_port_rounds_cispos_bound_in_the_log_prob_dtype():
    lp = torch.zeros(1, 2, dtype=torch.bfloat16)
    old = torch.tensor([[-0.2, -0.19]], dtype=torch.bfloat16)
    adv = torch.ones(1, 2, dtype=torch.bfloat16)
    s, over = port.policy_terms('cispo', lp + 1, old + 1, adv, 0.2)
    hi = torch.tensor(1.2).to(torch.bfloat16)
    assert (s <= hi * 1).all() and over.dtype == torch.bool
    ratio = torch.exp((lp + 1) - (old + 1))
    assert torch.equal(over, ratio > hi)


def test_objective_fields_and_refusals():
    from align_anything_b200 import ops

    assert ops.POLICY_LOSS_MODES['cispo'] == 3 and ops.POLICY_LOSS_MODES['sapo'] == 4  # include/aa_b200.h AA_PM_*
    for mode in MODES:
        for cls in (ops.ActorObjective, ops.GrpoObjective):
            o = cls(policy_loss_mode=mode)
            assert not o.is_default
            assert (o.sapo_value('sapo_temperature_pos'), o.sapo_value('sapo_temperature_neg')) == port.DEFAULT_TAU
    o = ops.ActorObjective(policy_loss_mode='cispo', clip_range_ratio_high=0.28, loss_agg_mode='token-mean')
    assert o.args(0.2)[1] == 0.28 and ops.ActorObjective(policy_loss_mode='cispo').args(0.3)[1] == 0.3
    assert ops.ActorObjective(policy_loss_mode='sapo', sapo_temperature_pos=2, sapo_temperature_neg=0.5)\
        .sapo_value('sapo_temperature_neg') == 0.5
    bad = [
        dict(policy_loss_mode='gpg'),
        dict(policy_loss_mode='cispo', dual_clip_ratio=3.0),
        dict(policy_loss_mode='sapo', dual_clip_ratio=3.0),
        dict(policy_loss_mode='cispo', clip_range_ratio_low=0.2),
        dict(policy_loss_mode='sapo', clip_range_ratio_low=0.2),
        dict(policy_loss_mode='sapo', clip_range_ratio_high=0.28),
        *[dict({k: 1.0}) for k in PM_KEYS],  # a temperature under vanilla
        *[dict(policy_loss_mode=m, **{k: 1.0}) for m in ('cispo', 'clip_cov', 'kl_cov') for k in PM_KEYS],
        *[dict(policy_loss_mode='sapo', **{k: v}) for k in PM_KEYS
          for v in (0.0, -1.0, float('inf'), float('nan'), '1', True, 1e39, 1e-50)],  # 1e39 / 1e-50: inf / 0 in fp32
        *[dict(policy_loss_mode=m, **{k: v}) for m in MODES
          for k, v in (('clip_cov_ratio', 0.1), ('clip_cov_lb', 0.0), ('clip_cov_ub', 2.0), ('kl_cov_ratio', 0.1),
                       ('ppo_kl_coef', 1.0))],
    ]
    for kw in bad:
        for cls in (ops.ActorObjective, ops.GrpoObjective):
            with pytest.raises(ValueError):
                cls(**kw)
    for kw in (dict(importance_sampling_level='sequence'), dict(top_entropy_quantile=0.5)):
        for mode in MODES:
            with pytest.raises(ValueError, match='token-level'):
                ops.GrpoObjective(policy_loss_mode=mode, **kw)


def test_switches_default_to_none_and_config_keys_win():
    from align_anything_b200.trainers.text_image_to_text.ppo import PPOTrainer as ImagePPO
    from align_anything_b200.trainers.text_to_text import grpo as G
    from align_anything_b200.trainers.text_to_text import ppo as P
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer as MultiPPO
    from align_anything_b200.trainers.text_audio_to_text.ppo import PPOTrainer as AudioPPO
    from align_anything_b200.trainers.text_video_to_text.ppo import PPOTrainer as VideoPPO

    for keys, classes in ((P.OBJECTIVE_KEYS, (P.PPOTrainer, MultiPPO, ImagePPO, AudioPPO, VideoPPO)),
                          (G.GRPO_OBJECTIVE_KEYS, (G.GRPOTrainer,))):
        for cls in classes:
            for k in PM_KEYS:
                assert k in keys and k in cls.SWITCHES and getattr(cls, k) is None
    tc = SimpleNamespace(update_iters=1, policy_loss_mode=None, sapo_temperature_pos=None)
    tr = P.PPOTrainer(SimpleNamespace(train_cfgs=tc))
    tr.policy_loss_mode, tr.sapo_temperature_pos = 'sapo', 3.0
    o = P.actor_objective_of(tr)
    assert o.policy_loss_mode == 'sapo' and o.sapo_value('sapo_temperature_pos') == 3.0
    tc.sapo_temperature_pos, tc.sapo_temperature_neg = 0.5, 0.25  # the recipe's values win over the attributes
    o = P.actor_objective_of(tr)
    assert (o.sapo_temperature_pos, o.sapo_temperature_neg) == (0.5, 0.25)
    g = G.GRPOTrainer(SimpleNamespace(train_cfgs=tc))
    g.policy_loss_mode = 'sapo'
    assert G.grpo_objective_of(g).sapo_temperature_neg == 0.25
    tc.policy_loss_mode = 'cispo'
    with pytest.raises(ValueError, match='sapo_temperature'):
        P.actor_objective_of(tr)


def test_objective_kwargs_and_the_clip_cov_counter():
    from align_anything_b200 import ops
    from align_anything_b200.trainers.text_to_text import ppo as P

    for mode in MODES:
        tr = P.PPOTrainer(SimpleNamespace(train_cfgs=SimpleNamespace(seed=42, policy_loss_mode=mode)))
        tr.log_clip_fraction = False
        for _ in range(3):
            kw = P.objective_kwargs(tr)
            assert kw['objective'].policy_loss_mode == mode and 'cov_seed' not in kw
        assert P.cov_seed_of(tr, kw['objective']) == 0
        assert getattr(tr, 'cov_calls', 0) == 0
    assert P.cov_seed_of(tr, ops.ActorObjective(policy_loss_mode='clip_cov')) == ops.cov_hash_seed(42, 0, 0)
    assert tr.cov_calls == 1


def test_install_grafts_the_switches(fake_reference):  # noqa: F811
    from align_anything_b200 import patch

    rl = {m: c for m, c in fake_reference.items() if 'ppo' in m or 'grpo' in m}
    assert rl
    try:
        patch.install(models=False)
        for modname, cls in rl.items():
            for k in PM_KEYS:
                assert k in cls.__dict__ and cls.__dict__[k] is None, (modname, k)
    finally:
        patch.uninstall()
    for modname, cls in rl.items():
        for k in PM_KEYS:
            assert k not in cls.__dict__, (modname, k)


def test_safe_rlhf_v_refuses_the_modes_and_keys():
    from align_anything_b200.trainers.text_image_to_text.saferlhf import SafeRLHFVTrainer

    t = object.__new__(SafeRLHFVTrainer)
    for k, v in (('policy_loss_mode', 'cispo'), ('policy_loss_mode', 'sapo'), ('sapo_temperature_pos', 1.0),
                 ('sapo_temperature_neg', 2.0)):
        t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(**{k: v}))
        with pytest.raises(ValueError, match='Safe RLHF-V'):
            t.rl_step({}, {})


def test_entry_points_check_their_arguments_before_cuda():
    from align_anything_b200 import _lib

    lib = _lib.lib()
    buf = (ctypes.c_int64 * 8)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def err():
        return lib.aa_last_error()

    def ppo(pm=3, hi=0.2, agg=0, tp=1.0, tn=1.05, mode=0, ref=None, klc=0.0, est=2, lp=p, B=2):
        return lib.aa_ppo_actor_loss_pm(lp, 8, p, 8, 2, p, 8, 2, p, 8, B, 8, hi, agg, pm, tp, tn, mode, ref, 8, klc, est,
                                        p, p, p, 8, None, p, p, None)

    def grpo(pm=4, hi=0.2, agg=1, est=2, tp=1.0, tn=1.05, mode=0):
        return lib.aa_grpo_loss_pm(p, 8, p, 8, None, 0, 2, p, p, 8, 1, 2, 8, 0.04, hi, agg, est, pm, tp, tn, mode, p, p,
                                   8, None, p, p, p, None)

    def actor_k1f(pm=3, hi=0.2, agg=0, tp=1.0, tn=1.05, coeff=0.0, ent=None, ref=None, klc=0.0, est=2):
        return lib.aa_logprob_actor_fused_pm(p, 0, 8, 8, p, 1, p, p, p, p, p, 8, p, 0, None, None, p, 8, p, 8, 0, p, 8,
                                             8, hi, agg, pm, tp, tn, 0, p, 8, p, None, coeff, ent, ref, klc, est, None)

    def grpo_k1f(pm=4, hi=0.2, agg=1, est=2, tp=1.0, tn=1.05, coeff=0.0, ent=None):
        return lib.aa_logprob_grpo_fused_pm(p, 0, 8, 8, p, 1, p, p, p, p, p, 8, p, 0, p, 8, None, p, p, 8, 1, 8, 0.04,
                                            hi, agg, est, pm, tp, tn, 0, p, 8, p, p, p, p, None, ent, coeff, None)

    for call, who in ((ppo, b'aa_ppo_actor_loss_pm'), (grpo, b'aa_grpo_loss_pm'),
                      (actor_k1f, b'aa_logprob_actor_fused_pm'), (grpo_k1f, b'aa_logprob_grpo_fused_pm')):
        for pm in (0, 1, 2, 5, -1):
            assert call(pm=pm) == -2 and who + b': unknown pm_mode' in err(), (who, pm)
        for tau in (0.0, -1.0, float('inf'), float('nan')):
            assert call(tp=tau) == -2 and b'tau_pos and tau_neg must be finite and > 0' in err()
            assert call(tn=tau) == -2 and b'tau_pos and tau_neg must be finite and > 0' in err()
        for hi in (-0.1, float('nan')):
            assert call(hi=hi) == -2 and b'bad objective' in err(), (who, hi)
        assert call(agg=7) == -2 and b'bad objective' in err()
    assert ppo(agg=2) == -2 and actor_k1f(agg=2) == -2  # Dr. GRPO's aggregation is GRPO's alone
    assert ppo(mode=3) == -2 and b'bad mode' in err()
    assert ppo(lp=None) == -2 and b'null pointer' in err()
    assert ppo(B=0) == -2 and b'bad sizes' in err()
    assert ppo(ref=p, klc=0.0) == -2 and b'a KL loss term needs kl_loss_coeff' in err()
    assert ppo(ref=p, klc=0.1, est=7) == -2 and b'unknown kl_estimator' in err()
    assert grpo(est=3) == -2 and b'unknown kl_estimator' in err()
    assert grpo(mode=4) == -2 and b'bad mode' in err()
    assert actor_k1f(coeff=0.1) == -2 and b'entropy_coeff needs entropy' in err()
    assert actor_k1f(coeff=float('nan'), ent=p) == -2 and b'entropy_coeff is NaN' in err()
    assert actor_k1f(ref=p, klc=-1.0) == -2 and b'kl_loss_coeff must be finite and > 0' in err()
    assert grpo_k1f(coeff=0.1) == -2 and b'entropy_coeff needs entropy' in err()
    assert grpo_k1f(est=9) == -2 and b'unknown kl_estimator' in err()
    # the Cov entry points refuse the new codes, as every code but AA_COV_CLIP / AA_COV_KL
    for cm in (3, 4):
        assert lib.aa_ppo_actor_loss_cov(p, 8, p, 8, 2, p, 8, 2, p, 8, 2, 8, 0.2, 0.2, 0, cm, 0.0, p, 8, 0, None, 8,
                                         0.0, 2, p, p, p, 8, None, p, p, None) == -2
        assert b'unknown cov_mode' in err()
        assert lib.aa_grpo_loss_cov(p, 8, p, 8, None, 0, 2, p, p, 8, 1, 2, 8, 0.04, 0.2, 0.2, 1, 2, cm, 1.0, p, 8, 0,
                                    p, p, 8, None, p, p, p, None) == -2
        assert b'unknown cov_mode' in err()


def _nodes(calls):
    """The log-prob, lm_head and loss launches of `calls` (the plan and layout helpers left out)."""
    return [c for c in calls if c.startswith(('aa_logprob', 'aa_linear', 'aa_ppo_actor', 'aa_grpo_loss', 'aa_cov'))]


def _actor_inputs(B, W):
    return torch.rand(B, W), torch.rand(B, W), torch.ones(B, W, dtype=torch.bool)


@pytest.mark.parametrize('mode', MODES)
def test_actor_nodes_take_k1f_when_it_runs(dry, mode):  # noqa: F811
    from align_anything_b200 import ops

    B, Lq, V = 2, 9, 97
    ids = torch.randint(0, V, (B, Lq))
    W = Lq - 1 - 2
    obj = ops.ActorObjective(policy_loss_mode=mode)
    # long rows: K1f's PM entry point, then K5's for the loss value; no K1 / K1b, no selection
    logits = torch.randn(B, Lq, V, dtype=torch.bfloat16, requires_grad=True)
    out = ops.dense_actor_loss(logits, ids, 2, *_actor_inputs(B, W), 0.2, objective=obj, return_clip_fraction=True)
    assert len(out) == 4
    assert dry.calls == ['aa_logprob_actor_fused_pm', 'aa_ppo_actor_loss_pm']
    dry.calls.clear()
    out[0].backward()
    assert not set(K1) & set(dry.calls) and not set(COV) & set(dry.calls)
    dry.calls.clear()
    # with a KL loss term and an entropy bonus: the same entry points
    out = ops.dense_actor_loss(logits, ids, 2, *_actor_inputs(B, W), 0.2, objective=obj, entropy_coeff=0.01,
                               ref_log_probs=torch.rand(B, W), kl_loss_coeff=0.1)
    assert len(out) == 5
    assert 'aa_logprob_actor_fused_pm' in dry.calls and 'aa_ppo_actor_loss_pm' in dry.calls
    assert not set(K1) & set(dry.calls) and not set(COV) & set(dry.calls)
    dry.calls.clear()
    # fp16: K1 -> aa_ppo_actor_loss_pm -> K1b
    logits16 = torch.randn(B, Lq, V, dtype=torch.float16, requires_grad=True)
    out = ops.dense_actor_loss(logits16, ids, 2, *_actor_inputs(B, W), 0.2, objective=obj)
    assert dry.calls == ['aa_logprob_fwd', 'aa_ppo_actor_loss_pm']
    out[0].backward()
    assert dry.calls[-1] == 'aa_logprob_bwd'
    assert not any(c.startswith('aa_logprob_actor_fused') for c in dry.calls)
    dry.calls.clear()
    # the tail layout: K1f's PM entry point too
    lens = [W, W - 2]
    ops.tail_actor_loss(logits, ids, lens, *_actor_inputs(B, W), 0.2, objective=obj)
    assert _nodes(dry.calls) == ['aa_logprob_actor_fused_pm', 'aa_ppo_actor_loss_pm']


@pytest.mark.parametrize('mode', MODES)
def test_actor_nodes_with_short_rows_compose(dry, monkeypatch, mode):  # noqa: F811
    from align_anything_b200 import ops

    monkeypatch.setattr(ops, '_FUSED_MIN_ROW_BYTES', 1 << 30)
    B, Lq, V = 2, 9, 97
    ids = torch.randint(0, V, (B, Lq))
    logits = torch.randn(B, Lq, V, dtype=torch.bfloat16, requires_grad=True)
    out = ops.dense_actor_loss(logits, ids, 2, *_actor_inputs(B, 6), 0.2, objective=ops.ActorObjective(
        policy_loss_mode=mode))
    out[0].backward()
    assert dry.calls == ['aa_logprob_fwd', 'aa_ppo_actor_loss_pm', 'aa_logprob_bwd']


@pytest.mark.parametrize('mode', MODES)
def test_grpo_nodes(dry, mode):  # noqa: F811
    from align_anything_b200 import ops

    B, Lq, V, K = 2, 9, 97, 5
    ids = torch.randint(3, V, (B, Lq))
    obj = ops.GrpoObjective(policy_loss_mode=mode)
    logits = torch.randn(B, Lq, V, dtype=torch.bfloat16, requires_grad=True)
    out = ops.grpo_loss_from_logits(logits, ids, K, torch.rand(B, K), torch.rand(B, 1), 2, 0.04, objective=obj,
                                    old_per_token_logps=torch.rand(B, K), return_clip_fraction=True)
    assert len(out) == 4
    assert _nodes(dry.calls) == ['aa_logprob_grpo_fused_pm', 'aa_grpo_loss_pm']
    dry.calls.clear()
    logits16 = torch.randn(B, Lq, V, dtype=torch.float16, requires_grad=True)
    out = ops.grpo_loss_from_logits(logits16, ids, K, torch.rand(B, K), torch.rand(B, 1), 2, 0.04, objective=obj)
    out[0].backward()
    assert _nodes(dry.calls) == ['aa_logprob_fwd', 'aa_grpo_loss_pm', 'aa_logprob_bwd']
    dry.calls.clear()
    lp = torch.rand(B, K, requires_grad=True)
    ops.grpo_loss(lp, torch.rand(B, K), torch.rand(B, 1), ids[:, -K:], 2, 0.04, objective=obj)
    assert _nodes(dry.calls) == ['aa_grpo_loss_pm']


def _grpo_trainer(dry, fused, **cfg):  # noqa: F811
    from test_cpu_top_entropy import _trainer

    return _trainer(dry, fused, **cfg)


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('fused', [False, True])
def test_grpo_updates(dry, packed, fused, mode):  # noqa: F811
    t = _grpo_trainer(dry, fused, update_iters=2, num_iterations=2, policy_loss_mode=mode, seed=3,
                      log_clip_fraction=True)
    gen = torch.Generator().manual_seed(0)
    out = t.step_from_rollout(torch.randint(3, 97, (4, 9), generator=gen), 4, torch.randn(4, generator=gen))
    assert 'train/actor_cov_fraction' not in out and 'train/actor_clip_fraction' in out
    assert dry.calls.count('aa_grpo_loss_pm') == 2 and not set(COV) & set(dry.calls)
    if fused:  # K6 -> aa_grpo_loss_pm -> K6b
        assert 'aa_linear_logprob_fwd' in dry.calls and 'aa_linear_dlogits' in dry.calls
        assert not any(c.startswith('aa_logprob_grpo_fused') for c in dry.calls)
    else:
        assert dry.calls.count('aa_logprob_grpo_fused_pm') == 2 and not set(K1) & set(dry.calls[-4:])
    assert getattr(t, 'cov_calls', 0) == 0


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('fused', [False, True])
@pytest.mark.parametrize('trainer', ['text', 'multi_rloo', 'image'])
def test_ppo_rl_step_paths(dry, packed, fused, trainer, mode):  # noqa: F811
    """One rl_step of each PPO trainer under each mode on the stand-in library: the tile path runs K1f's and K5's PM
    entry points and no K1 / K1b; fused_lm_head runs K6 -> aa_ppo_actor_loss_pm -> K6b; neither selects tokens nor
    adds a metric lane beyond the clip fraction."""
    from test_cpu_ppo_step import _ppo_trainer, _prompts, _standalone_class

    from align_anything_b200 import ops

    if fused and trainer == 'image':  # the stand-in leaves the multimodal response lengths at 0: take the full width
        layout = ops.rollout_layout

        def full(prompt_ids, sequences, pad_id):
            moved, mask, lens = layout(prompt_ids, sequences, pad_id)
            lens.dev.fill_(lens.bound)
            return moved, mask, lens

        import unittest.mock
        patcher = unittest.mock.patch.object(ops, 'rollout_layout', full)
        patcher.start()
    else:
        patcher = None
    try:
        t = _ppo_trainer(_standalone_class(trainer), trainer)
        t.fused_lm_head, t.log_entropy, t.entropy_coeff, t.log_clip_fraction = fused, False, 0.0, True
        t.policy_loss_mode = mode
        inference, training = t.rollout(_prompts())
        dry.calls.clear()
        out = t.rl_step(inference[0], training[0])
    finally:
        if patcher is not None:
            patcher.stop()
    assert 'train/actor_clip_fraction' in out and 'train/actor_cov_fraction' not in out
    assert all(isinstance(v, float) for v in out.values())
    calls = _nodes(dry.calls)
    assert calls.count('aa_ppo_actor_loss_pm') == 1 and not set(COV) & set(calls)
    assert not any(c in ('aa_ppo_actor_loss', 'aa_ppo_actor_loss_obj', 'aa_ppo_actor_loss_kl') for c in calls)
    pm = calls.index('aa_ppo_actor_loss_pm')
    if fused:  # K6 -> aa_ppo_actor_loss_pm -> K6b
        assert 'aa_linear_logprob_fwd' in calls[:pm] and 'aa_linear_dlogits' in calls[pm:]
        assert not any(c.startswith('aa_logprob_actor_fused') for c in calls)
    else:
        assert calls[pm - 1] == 'aa_logprob_actor_fused_pm' and not set(K1) & set(calls)
    assert getattr(t, 'cov_calls', 0) == 0
