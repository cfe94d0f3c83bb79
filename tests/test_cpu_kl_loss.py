"""The KL term in the PPO actor loss without a GPU: the port (tests/kl_loss_port.py) against the objective port and
float64 autograd, the trainers' switch resolution (kl_loss_of) and its precedence, the graft and the Safe RLHF-V
refusal, the ops keywords, the C argument checks of aa_ppo_actor_loss_kl and aa_logprob_actor_fused_kl and, on the
stand-in library, which entry points each path calls and which metric lanes the step packs."""
from __future__ import annotations

import contextlib
import ctypes
import math
from types import SimpleNamespace

import pytest
import torch

import kl_loss_port as port
from ppo_objective_port import actor_loss as objective_loss
from test_cpu_entropy import fake_reference  # noqa: F401  (fixture)
from test_cpu_plumbing import dry  # noqa: F401  (fixture)
from test_cpu_ppo_step import _PPO_MODULES, _grafted, _ppo_trainer, _prompts, _standalone_class
from test_cpu_ppo_step import full_lens, packed  # noqa: F401  (fixtures)

ESTIMATORS = ['k1', 'k2', 'k3']
AGGS = ['seq-mean-token-mean', 'token-mean']
KL_CALLS = {'aa_ppo_actor_loss_kl', 'aa_logprob_actor_fused_kl'}


def _inputs(B=5, W=23, dtype=torch.float32, seed=0):
    g = torch.Generator().manual_seed(seed)
    lp = (-torch.rand(B, W, generator=g) * 4).to(dtype)
    old = (lp.double() + torch.randn(B, W, generator=g) * 0.4).to(dtype)
    ref = (lp.double() + torch.randn(B, W, generator=g) * 0.3).to(dtype)
    adv = torch.randn(B, W, generator=g).to(dtype)
    mask = torch.rand(B, W, generator=g) > 0.25
    mask[:, 0] = True
    return lp, old, ref, adv, mask


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize('agg', AGGS)
def test_port_without_the_term_is_the_objective_port(dtype, agg):
    lp, old, ref, adv, mask = _inputs(dtype=dtype)
    for c in (None, 3.0):
        x, y = lp.clone().requires_grad_(True), lp.clone().requires_grad_(True)
        got = port.actor_loss(x, old, adv, mask, 0.2, 0.28, c, agg, ref_log_probs=ref, kl_loss_coeff=0.0)
        want = objective_loss(y, old, adv, mask, 0.2, 0.28, c, agg)
        got.backward()
        want.backward()
        assert got.dtype == want.dtype and torch.equal(got, want) and torch.equal(x.grad, y.grad)


@pytest.mark.parametrize('est', ESTIMATORS)
@pytest.mark.parametrize('agg', AGGS)
def test_port_gradient_is_the_analytic_one_in_float64(est, agg):
    lp, old, ref, adv, mask = _inputs(dtype=torch.float64)
    coeff = 0.3
    x = lp.clone().requires_grad_(True)
    total = port.actor_loss(x, old, adv, mask, 0.2, 0.28, 3.0, agg, ref_log_probs=ref, kl_loss_coeff=coeff,
                            estimator=est)
    total.backward()
    y = lp.clone().requires_grad_(True)
    objective_loss(y, old, adv, mask, 0.2, 0.28, 3.0, agg).backward()
    d = lp - ref
    dkl = {'k1': torch.ones_like(d), 'k2': d, 'k3': 1 - torch.exp(-d)}[est]
    kl = {'k1': d, 'k2': 0.5 * d * d, 'k3': torch.exp(-d) + d - 1}[est]
    m = mask.double()
    if agg == 'token-mean':
        w = m / m.sum()
    else:
        w = m / (m.size(0) * m.sum(-1, keepdim=True))
    torch.testing.assert_close(x.grad, y.grad + coeff * w * dkl, rtol=1e-12, atol=1e-12)
    want = objective_loss(lp, old, adv, mask, 0.2, 0.28, 3.0, agg) + coeff * (w * kl).sum()
    torch.testing.assert_close(total.detach(), want, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(port.kl_loss(lp, ref, mask, est, agg), (w * kl).sum(), rtol=1e-12, atol=1e-12)


# ---- switches -------------------------------------------------------------------------------------------------------
def _bare(**cfg):
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer

    t = object.__new__(PPOTrainer)
    t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(**cfg))
    return t


def test_switch_resolution_and_precedence():
    from align_anything_b200.trainers.text_to_text import ppo as P

    for cls in {_standalone_class(t) for t in _PPO_MODULES} | {_video_class()}:
        assert 'kl_loss_estimator' in cls.SWITCHES and 'kl_loss_coeff' in cls.SWITCHES, cls
        assert cls.kl_loss_estimator is None and cls.kl_loss_coeff == 0.0
    t = _bare()
    assert P.kl_loss_of(t) is None
    t.kl_loss_estimator, t.kl_loss_coeff = 'k2', 0.1
    assert P.kl_loss_of(t) == (0.1, 'k2')
    t.cfgs.train_cfgs.kl_loss_estimator, t.cfgs.train_cfgs.kl_loss_coeff = 'k3', 0.05
    assert P.kl_loss_of(t) == (0.05, 'k3')
    t = _bare(kl_loss_coeff=0.2)
    t.kl_loss_estimator = 'k1'
    assert P.kl_loss_of(t) == (0.2, 'k1')


@pytest.mark.parametrize('settings, match', [
    ({'kl_loss_coeff': 0.1}, 'kl_loss_estimator'),                       # a coefficient alone: refused, not ignored
    ({'kl_loss_estimator': 'k3'}, 'kl_loss_coeff'),                      # the estimator with the default 0
    ({'kl_loss_estimator': 'k3', 'kl_loss_coeff': -0.1}, 'kl_loss_coeff'),
    ({'kl_loss_estimator': 'k3', 'kl_loss_coeff': math.nan}, 'kl_loss_coeff'),
    ({'kl_loss_estimator': 'k3', 'kl_loss_coeff': math.inf}, 'kl_loss_coeff'),
    ({'kl_loss_estimator': 'k3', 'kl_loss_coeff': True}, 'kl_loss_coeff'),
    ({'kl_loss_estimator': 'k3', 'kl_loss_coeff': '0.1'}, 'kl_loss_coeff'),
    ({'kl_loss_estimator': 'low_var_kl', 'kl_loss_coeff': 0.1}, 'kl_estimator'),
])
def test_invalid_switches_raise(settings, match):
    from align_anything_b200.trainers.text_to_text import ppo as P

    for where in ('attr', 'cfg'):
        t = _bare(**(settings if where == 'cfg' else {}))
        if where == 'attr':
            for k, v in settings.items():
                setattr(t, k, v)
        with pytest.raises(ValueError, match=match):
            P.kl_loss_of(t)


def _video_class():
    from align_anything_b200.trainers.text_video_to_text.ppo import PPOTrainer

    return PPOTrainer


def test_install_grafts_the_switch(fake_reference):  # noqa: F811
    from align_anything_b200 import patch

    ppo = {m: c for m, c in fake_reference.items() if 'ppo' in m}
    assert ppo
    try:
        patch.install(models=False)
        for modname, cls in ppo.items():
            assert 'kl_loss_estimator' in cls.__dict__ and cls.kl_loss_estimator is None, modname
    finally:
        patch.uninstall()
    for modname, cls in ppo.items():
        assert 'kl_loss_estimator' not in cls.__dict__, modname


def test_safe_rlhf_v_refuses_the_switch():
    from align_anything_b200.trainers.text_image_to_text.saferlhf import SafeRLHFVTrainer, refuse_kl_switches

    t = object.__new__(SafeRLHFVTrainer)
    t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace())
    refuse_kl_switches(t)
    t.cfgs.train_cfgs.kl_loss_estimator = 'k3'
    with pytest.raises(ValueError, match='Safe RLHF-V'):
        t.rl_step({}, {})


# ---- C argument checks ----------------------------------------------------------------------------------------------
def test_entry_points_check_their_arguments_before_cuda():
    from align_anything_b200 import _lib

    lib = _lib.lib()
    buf = (ctypes.c_int64 * 16)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def k5(ref, coeff, est, agg=0):
        return lib.aa_ppo_actor_loss_kl(p, 8, p, 8, 0, p, 8, 0, p, 8, 2, 8, 0.2, 0.2, 0.0, agg, 0, ref, 8, coeff, est,
                                        p, p, p, 8, None, p, p, None)

    def k1f(ref, coeff, est, agg=0):
        return lib.aa_logprob_actor_fused_kl(p, 0, 64, 64, p, 2, p, p, p, p, p, 2, p, 0, None, None, p, 8, p, 8, 0, p,
                                             8, 8, 0.2, 0.2, 0.0, agg, 0, p, 64, p, p, 0.0, None, ref, coeff, est,
                                             None)

    for name, fn in (('aa_ppo_actor_loss_kl', k5), ('aa_logprob_actor_fused_kl', k1f)):
        for est in (-1, 3, 7):
            assert fn(p, 0.1, est) == -2 and f'{name}: unknown kl_estimator'.encode() in lib.aa_last_error()
        for bad in (0.0, -0.1, math.nan, math.inf, -math.inf):
            assert fn(p, bad, 2) == -2 and b'kl_loss_coeff must be finite and > 0' in lib.aa_last_error()
        assert fn(None, 0.1, 2) == -2 and b'null ref_log_probs' in lib.aa_last_error()
        assert fn(p, 0.1, 2, agg=2) == -2 and b'bad objective' in lib.aa_last_error()
    rc = lib.aa_ppo_actor_loss_kl(p, 8, p, 8, 0, p, 8, 0, p, 8, 2, 8, 0.2, 0.2, 0.0, 0, 0, p, 8, 0.1, 2, p, None, p, 8,
                                  None, p, p, None)
    assert rc == -2 and b'kl_loss' in lib.aa_last_error()


# ---- ops keywords on the stand-in library ---------------------------------------------------------------------------
def test_ops_keywords(dry):  # noqa: F811
    from align_anything_b200 import ops

    lp, old, ref, adv, mask = _inputs()
    out = ops.actor_loss(lp, old, adv, mask, 0.2)
    assert isinstance(out, torch.Tensor) and not KL_CALLS & set(dry.calls)
    loss, kl = ops.actor_loss(lp, old, adv, mask, 0.2, ref_log_probs=ref, kl_loss_coeff=0.1, kl_loss_estimator='k2')
    assert loss.dim() == 0 and kl.dim() == 0 and dry.calls[-1] == 'aa_ppo_actor_loss_kl'
    loss, kl, cf = ops.actor_loss(lp, old, adv, mask, 0.2, return_clip_fraction=True, ref_log_probs=ref,
                                  kl_loss_coeff=0.1)
    assert cf.shape == (2,)
    for kw, match in (({'kl_loss_coeff': 0.1}, 'ref_log_probs'),
                      ({'kl_loss_coeff': 0.1, 'ref_log_probs': ref[:, 1:]}, 'ref_log_probs'),
                      ({'kl_loss_coeff': -1.0, 'ref_log_probs': ref}, 'kl_loss_coeff'),
                      ({'kl_loss_coeff': math.nan, 'ref_log_probs': ref}, 'kl_loss_coeff'),
                      ({'kl_loss_coeff': 0.1, 'ref_log_probs': ref, 'kl_loss_estimator': 'k4'}, 'kl_estimator')):
        dry.calls.clear()
        with pytest.raises(ValueError, match=match):
            ops.actor_loss(lp, old, adv, mask, 0.2, **kw)
        assert not dry.calls


# ---- trainer paths on the stand-in library --------------------------------------------------------------------------
def _run(trainer, grafted, settings, monkeypatch=None, fused_actor=True):
    from align_anything_b200 import ops

    with contextlib.ExitStack() as stack:
        cls = stack.enter_context(_grafted())[_PPO_MODULES[trainer]].PPOTrainer if grafted else _standalone_class(trainer)
        t = _ppo_trainer(cls, trainer)
        for k, v in settings.items():
            setattr(t, k, v)
        if not fused_actor:
            monkeypatch.setattr(ops, '_FUSED_ACTOR', False)
        inference, training = t.rollout(_prompts())
        return t.rl_step(inference[0], training[0])


@pytest.mark.parametrize('path', ['k1f', 'composed', 'fused_lm_head'])
@pytest.mark.parametrize('grafted', [False, True])
@pytest.mark.parametrize('trainer', list(_PPO_MODULES))
def test_paths_call_the_kl_entry_points(dry, packed, full_lens, monkeypatch, trainer, grafted, path):  # noqa: F811
    base = {'fused_lm_head': path == 'fused_lm_head'}
    out = _run(trainer, grafted, base, monkeypatch, fused_actor=path != 'composed')
    assert not KL_CALLS & set(dry.calls) and 'train/actor_kl_loss' not in out
    assert packed == [(12, (9, 10))]
    dry.calls.clear()
    packed.clear()
    on = {**base, 'kl_loss_estimator': 'k3', 'kl_loss_coeff': 0.05, 'entropy_coeff': 0.01, 'log_clip_fraction': True}
    out = _run(trainer, grafted, on, monkeypatch, fused_actor=path != 'composed')
    calls = set(dry.calls)
    assert 'aa_ppo_actor_loss_kl' in calls
    assert not {'aa_ppo_actor_loss', 'aa_ppo_actor_loss_obj'} & calls
    if path == 'k1f':
        assert 'aa_logprob_actor_fused_kl' in calls
        assert not {'aa_logprob_actor_fused', 'aa_logprob_actor_fused_entropy', 'aa_logprob_actor_fused_obj'} & calls
    else:
        assert 'aa_logprob_actor_fused_kl' not in calls
    if path == 'composed':
        assert {'aa_logprob_fwd_entropy', 'aa_logprob_bwd_entropy'} <= calls
    # the entropy bonus, the clip fraction, then agg(KL): one more AVG lane of the one packed vector
    assert set(out) >= {'train/actor_kl_loss', 'train/actor_entropy', 'train/actor_clip_fraction'}
    assert packed == [(15, (9, 10))]


@pytest.mark.parametrize('settings', [{'kl_loss_coeff': 0.1}, {'kl_loss_estimator': 'k2'},
                                      {'kl_loss_estimator': 'k2', 'kl_loss_coeff': math.nan},
                                      {'kl_loss_estimator': 'k9', 'kl_loss_coeff': 0.1}])
@pytest.mark.parametrize('trainer', ['text', 'image'])
def test_rl_step_refuses_before_any_launch(dry, packed, full_lens, trainer, settings):  # noqa: F811
    t = _ppo_trainer(_standalone_class(trainer), trainer)
    for k, v in settings.items():
        setattr(t.cfgs.train_cfgs, k, v)
    inference, training = t.rollout(_prompts())
    dry.calls.clear()
    with pytest.raises(ValueError):
        t.rl_step(inference[0], training[0])
    assert not dry.calls
