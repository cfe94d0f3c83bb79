"""KL regularisation options without a GPU: the port (tests/kl_objective_port.py) against the reference's k1 reward
penalty and k3 GRPO loss and against float64 autograd, ops.GrpoObjective's estimator field, the trainers' KL switches
and their config precedence, the graft, the Safe RLHF-V refusal, the adaptive KL coefficient, the C argument checks
of the new entry points and, on the stand-in library, which entry points each path calls."""
from __future__ import annotations

import contextlib
import ctypes
from types import SimpleNamespace

import pytest
import torch

import kl_objective_port as port
from grpo_objective_port import completion_mask
from oracle import ref_port
from test_cpu_entropy import fake_reference  # noqa: F401  (fixture)
from test_cpu_plumbing import dry  # noqa: F401  (fixture)
from test_cpu_ppo_step import _PPO_MODULES, _grafted, _ppo_trainer, _prompts, _standalone_class
from test_cpu_ppo_step import full_lens, packed  # noqa: F401  (fixtures)

DTYPES = [torch.bfloat16, torch.float16, torch.float32]
ESTIMATORS = ['k1', 'k2', 'k3']


def _inputs(B=6, K=29, dtype=torch.float32, seed=0, eos=1):
    g = torch.Generator().manual_seed(seed)
    lp = (-torch.rand(B, K, generator=g) * 4).to(dtype)
    ref = (lp.float() + torch.randn(B, K, generator=g) * 0.3).to(dtype)
    adv = torch.randn(B, 1, generator=g)
    tokens = torch.randint(2, 50, (B, K), generator=g)
    for b in range(0, B, 2):
        tokens[b, 3 + 2 * b] = eos
    return lp, ref, adv, tokens


def _grad(fn, lp, *args, **kw):
    x = lp.clone().requires_grad_(True)
    loss = fn(x, *args, **kw)
    loss.backward()
    return loss.detach(), x.grad


@pytest.mark.parametrize('dtype', DTYPES)
def test_default_port_is_the_reference_penalty_and_grpo_loss(dtype):
    lp, ref, adv, tokens = _inputs(dtype=dtype)
    mask = torch.ones_like(lp, dtype=torch.bool)
    mask[1, 20:] = False
    reward = torch.randn(lp.size(0))
    want = ref_port.kl_shaped_rewards(reward, lp, ref, mask, 0.05, 10.0)
    got = port.kl_rewards(reward, lp, ref, mask, 0.05, 10.0)
    assert got.dtype == want.dtype and torch.equal(got, want)
    seq = torch.cat([torch.zeros(lp.size(0), 3, dtype=torch.int64), tokens], 1)
    want, gwant = _grad(ref_port.grpo_loss, lp, ref, adv, seq, 3, 1, 0.04)
    got, ggot = _grad(port.grpo_loss, lp, ref, adv, completion_mask(tokens, 1), 0.04)
    assert torch.equal(got, want) and torch.equal(ggot, gwant)


@pytest.mark.parametrize('est', ESTIMATORS)
def test_port_matches_float64(est):
    lp, ref, adv, tokens = _inputs(dtype=torch.float64)
    d = lp - ref
    want = {'k1': d, 'k2': 0.5 * d * d, 'k3': torch.exp(-d) + d - 1}[est]
    torch.testing.assert_close(port.kl_estimate(lp, ref, est), want, rtol=1e-14, atol=1e-14)
    mask = completion_mask(tokens, 1)

    def f64(x):
        kl = {'k1': x - ref, 'k2': 0.5 * (x - ref) ** 2, 'k3': torch.exp(ref - x) - (ref - x) - 1}[est]
        ptl = -(torch.exp(x - x.detach()) * adv - 0.04 * kl)
        return (ptl * mask).sum() / mask.sum()

    got, g = _grad(port.grpo_loss, lp, ref, adv, mask, 0.04, est)
    want, gw = _grad(f64, lp)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(g, gw, rtol=1e-12, atol=1e-12)
    # d KL / d lp: 1, lp - ref, 1 - exp(ref - lp)
    x = lp.clone().requires_grad_(True)
    port.kl_estimate(x, ref, est).sum().backward()
    dk = {'k1': torch.ones_like(d), 'k2': d, 'k3': 1 - torch.exp(-d)}[est]
    torch.testing.assert_close(x.grad, dk, rtol=1e-12, atol=1e-12)


def test_kl_metric_keeps_the_k1_definition():
    lp, ref, _, _ = _inputs(dtype=torch.float32)
    mask = torch.ones_like(lp, dtype=torch.bool)
    assert port.kl_divergence_metric(lp, ref, mask) == pytest.approx(float((lp - ref).double().sum(-1).mean()))


def test_grpo_objective_takes_the_estimator():
    from align_anything_b200 import ops

    assert ops.GrpoObjective().kl_estimator == 'k3' and ops.GrpoObjective().is_default
    assert not ops.GrpoObjective(kl_estimator='k1').is_default
    assert ops.GrpoObjective(kl_estimator='k2').args() == (0.2, 0.2, 0.0, 1)
    assert ops._grpo_objective_args(ops.GrpoObjective(kl_estimator='k2'), None, False) == (0.2, 0.2, 0.0, 1, 1)
    assert ops._grpo_objective_args(ops.GrpoObjective(), None, False) is None
    for bad in ('k4', 'abs', None, 3):
        with pytest.raises(ValueError, match='kl_estimator'):
            ops.GrpoObjective(kl_estimator=bad)
    with pytest.raises(ValueError, match='kl_estimator'):
        ops.kl_estimator_code('low_var_kl')
    assert ops.KL_ESTIMATORS == {'k1': 0, 'k2': 1, 'k3': 2}


def test_adaptive_controller_follows_the_formula():
    from align_anything_b200.trainers.text_to_text.ppo import adaptive_kl_coeff

    kls, n, target, horizon = [0.5, 12.0, 6.0, 5.9, 0.0, 100.0], 64, 6.0, 10000.0
    want = port.adaptive_kl_coeffs(0.1, kls, n, target, horizon)
    got, c = [], 0.1
    for kl in kls:
        got.append(c)
        c = adaptive_kl_coeff(c, kl, n, target, horizon)
    assert got == want
    assert want[2] == pytest.approx(0.1 * (1 - 0.2 * 64 / 1e4) * (1 + 0.2 * 64 / 1e4))


def test_kl_switches_default_off_and_config_takes_precedence():
    from align_anything_b200.trainers.text_to_text import ppo as P
    from align_anything_b200.trainers.text_to_text.grpo import GRPOTrainer

    for cls in {_standalone_class(t) for t in _PPO_MODULES}:
        for k in ('kl_estimator', 'kl_target', 'kl_horizon', 'kl_loss_coeff'):
            assert k in cls.SWITCHES, (cls, k)
        assert cls.kl_estimator is None and cls.kl_target is None and cls.kl_horizon == 10000
        assert cls.kl_loss_coeff == 0.0
    assert 'kl_estimator' in GRPOTrainer.SWITCHES and GRPOTrainer.kl_estimator == 'k3'
    t = object.__new__(P.PPOTrainer)
    t.kl_coeff = 0.05
    t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace())
    assert P.kl_estimator_of(t) == 'k1' and P.kl_controller_of(t) is None
    t.kl_estimator = 'k2'
    t.cfgs.train_cfgs.kl_estimator = 'k3'
    assert P.kl_estimator_of(t) == 'k3'
    t.cfgs.train_cfgs.kl_target, t.kl_horizon = 6.0, 500
    assert P.kl_controller_of(t) == (6.0, 500.0)
    t.cfgs.train_cfgs.kl_horizon = 2000
    assert P.kl_controller_of(t) == (6.0, 2000.0)
    for name, bad in (('kl_target', 0.0), ('kl_target', -1.0), ('kl_target', float('nan')), ('kl_horizon', 0),
                      ('kl_horizon', float('inf'))):
        u = object.__new__(P.PPOTrainer)
        u.kl_coeff, u.cfgs = 0.05, SimpleNamespace(train_cfgs=SimpleNamespace(kl_target=6.0, kl_horizon=100))
        setattr(u.cfgs.train_cfgs, name, bad)
        with pytest.raises(ValueError, match=name):
            P.kl_controller_of(u)
    t.kl_coeff = 0.0
    with pytest.raises(ValueError, match='kl_coeff'):
        P.kl_controller_of(t)
    t.cfgs.train_cfgs.kl_estimator = 'k5'
    with pytest.raises(ValueError, match='kl_estimator'):
        P.kl_estimator_of(t)


def test_install_grafts_the_kl_switches(fake_reference):  # noqa: F811
    from align_anything_b200 import patch

    keys = ('kl_estimator', 'kl_target', 'kl_horizon', 'kl_loss_coeff')
    ppo = {m: c for m, c in fake_reference.items() if 'ppo' in m}
    assert ppo
    try:
        patch.install(models=False)
        for modname, cls in ppo.items():
            for k in keys:
                assert k in cls.__dict__, (modname, k)
            assert cls.kl_horizon == 10000
    finally:
        patch.uninstall()
    for modname, cls in ppo.items():
        for k in keys:
            assert k not in cls.__dict__, (modname, k)


@pytest.mark.parametrize('key, value', [('kl_estimator', 'k3'), ('kl_target', 6.0), ('kl_horizon', 500),
                                        ('kl_loss_coeff', 0.1)])
def test_safe_rlhf_v_refuses_the_kl_switches(key, value):
    from align_anything_b200.trainers.text_image_to_text.saferlhf import SafeRLHFVTrainer, refuse_kl_switches

    t = object.__new__(SafeRLHFVTrainer)
    t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace())
    refuse_kl_switches(t)  # defaults: nothing to refuse
    t.cfgs.train_cfgs.kl_estimator = 'k1'
    refuse_kl_switches(t)
    setattr(t.cfgs.train_cfgs, key, value)
    with pytest.raises(ValueError, match='Safe RLHF-V'):
        t.rl_step({}, {})
    with pytest.raises(ValueError, match='Safe RLHF-V'):
        t.add_kl_divergence_regularization_with_cost(None, None, None, None, None)


def test_new_entry_points_check_their_arguments_before_cuda():
    from align_anything_b200 import _lib

    lib = _lib.lib()
    buf = (ctypes.c_int64 * 8)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def k4(coeff, est):
        return lib.aa_ppo_prep_kl(p, p, 2, 8, p, p, 2, 8, p, 8, 2, 8, 0, coeff, est, 10.0, 1.0, 0.95, 0, p, 2, p, p, 2,
                                  p, p, None)

    def grpo(est):
        return lib.aa_grpo_loss_kl(p, 8, p, 8, None, 0, 2, p, p, 8, 1, 2, 8, 0.04, 0.2, 0.2, 0.0, 1, est, 0, p, p, 8,
                                   None, p, p, p, None)

    def k1f(est):
        return lib.aa_logprob_grpo_fused_kl(p, 0, 64, 64, p, 2, p, p, p, p, p, 2, p, 0, p, 8, None, p, p, 8, 1, 8, 0.04,
                                            0.2, 0.2, 0.0, 1, est, 0, p, 64, p, p, p, p, p, None, 0.0, None)

    for est in (-1, 3, 7):
        assert k4(0.05, est) == -2 and b'aa_ppo_prep_kl: unknown kl_estimator' in lib.aa_last_error()
        assert grpo(est) == -2 and b'aa_grpo_loss_kl: unknown kl_estimator' in lib.aa_last_error()
        assert k1f(est) == -2 and b'aa_logprob_grpo_fused_kl: unknown kl_estimator' in lib.aa_last_error()
    for bad in (float('nan'), float('inf'), -float('inf')):
        assert k4(bad, 2) == -2 and b'kl_coeff must be finite' in lib.aa_last_error()
    rc = lib.aa_ppo_prep_kl(None, None, 2, 8, None, p, 2, 8, p, 8, 2, 8, 0, 0.05, 1, 10.0, 1.0, 0.95, 0, p, 2, p, p,
                            2, p, p, None)
    assert rc == -2 and b'GAE-only' in lib.aa_last_error()


def _run_ppo(trainer, grafted, settings, train_cfgs=None):
    with contextlib.ExitStack() as stack:
        if grafted:
            cls = stack.enter_context(_grafted())[_PPO_MODULES[trainer]].PPOTrainer
        else:
            cls = _standalone_class(trainer)
        t = _ppo_trainer(cls, trainer)
        for k, v in settings.items():
            setattr(t, k, v)
        for k, v in (train_cfgs or {}).items():
            setattr(t.cfgs.train_cfgs, k, v)
        inference, training = t.rollout(_prompts())
        outs = [t.rl_step(inference[0], training[0]) for _ in range(2)]
    return t, outs


@pytest.mark.parametrize('grafted', [False, True])
@pytest.mark.parametrize('trainer', list(_PPO_MODULES))
def test_ppo_paths_call_the_entry_points_the_switches_ask_for(dry, packed, full_lens, trainer, grafted):  # noqa: F811
    _, outs = _run_ppo(trainer, grafted, {})
    assert 'aa_ppo_prep_kl' not in dry.calls and 'aa_ppo_prep' in dry.calls
    assert 'train/kl_coeff' not in outs[0]
    dry.calls.clear()
    t, outs = _run_ppo(trainer, grafted, {'kl_estimator': 'k3', 'kl_coeff': 0.1},
                       {'kl_target': 6.0, 'kl_horizon': 100})
    assert 'aa_ppo_prep_kl' in dry.calls and 'aa_ppo_prep' not in dry.calls
    # the step's own coefficient, then the controller's update from that step's KL and its samples
    n = t.last_rl_tensors['old_rewards'].size(0)
    want = port.adaptive_kl_coeffs(0.1, [o['train/kl_divergence'] for o in outs] + [0.0], n, 6.0, 100)
    assert [o['train/kl_coeff'] for o in outs] + [t.kl_coeff] == want


@pytest.mark.parametrize('est', ['k1', 'k2', 'k3'])
@pytest.mark.parametrize('fused', [False, True])
def test_grpo_step_calls_the_kl_entry_points(dry, packed, fused, est):  # noqa: F811
    from align_anything_b200.trainers.text_to_text.grpo import GRPOTrainer
    from test_cpu_ppo_step import _LM, _Engine

    t = object.__new__(GRPOTrainer)
    t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(update_iters=1, kl_estimator=est))
    t.actor_model = _Engine(_LM(97, 64, 0, 2, 6, seed=1).bfloat16())
    t.actor_reference_model = _Engine(_LM(97, 64, 0, 2, 6, seed=2).bfloat16())
    t.tokenizer = SimpleNamespace(pad_token_id=0, eos_token_id=2)
    t.beta, t.num_generations, t.fused_lm_head = 0.04, 2, fused
    gen = torch.Generator().manual_seed(0)
    out = t.step_from_rollout(torch.randint(3, 97, (4, 9), generator=gen), 4, torch.randn(4, generator=gen))
    assert set(out) == {'train/loss', 'train/reward'}
    kl_calls = {c for c in dry.calls if c in ('aa_grpo_loss_kl', 'aa_logprob_grpo_fused_kl')}
    if est == 'k3':  # the reference's loss: today's launches
        assert not kl_calls and 'aa_grpo_loss_obj' not in dry.calls
        assert ('aa_grpo_loss' in dry.calls) or ('aa_logprob_grpo_fused' in dry.calls)
    else:
        assert kl_calls == ({'aa_grpo_loss_kl'} if fused else {'aa_grpo_loss_kl', 'aa_logprob_grpo_fused_kl'})


@pytest.mark.parametrize('grafted', [False, True])
@pytest.mark.parametrize('trainer', list(_PPO_MODULES))
def test_ppo_refuses_a_kl_loss_term_before_anything_runs(dry, packed, full_lens, trainer, grafted):  # noqa: F811
    """The KL term in the actor loss is not implemented: a non-zero kl_loss_coeff (attribute or train_cfgs key) raises
    at the top of rl_step, before K4 or any other launch; 0 runs the step."""
    for settings, cfg in (({'kl_loss_coeff': 0.1}, {}), ({}, {'kl_loss_coeff': 0.05})):
        with contextlib.ExitStack() as stack:
            if grafted:
                cls = stack.enter_context(_grafted())[_PPO_MODULES[trainer]].PPOTrainer
            else:
                cls = _standalone_class(trainer)
            t = _ppo_trainer(cls, trainer)
            for k, v in settings.items():
                setattr(t, k, v)
            for k, v in cfg.items():
                setattr(t.cfgs.train_cfgs, k, v)
            inference, training = t.rollout(_prompts())
            dry.calls.clear()
            with pytest.raises(ValueError, match='kl_loss_coeff'):
                t.rl_step(inference[0], training[0])
            assert not {'aa_ppo_prep', 'aa_ppo_prep_kl', 'aa_ppo_pack_metrics'} & set(dry.calls)
    _, outs = _run_ppo(trainer, grafted, {'kl_loss_coeff': 0.0})
    assert 'train/kl_coeff' not in outs[0]
