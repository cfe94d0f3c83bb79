"""Advantage whitening without a GPU: the port (tests/whiten_port.py) against float64 masked_whiten, the
`whiten_advantages` switch, its config precedence and the graft, Safe RLHF-V's refusal, the argument checks of
ops.whiten_advantages and of the three C entry points and, on the stand-in library, which launches rollout() and
rl_step make with the switch on and off."""
from __future__ import annotations

import contextlib
import ctypes
from types import SimpleNamespace

import pytest
import torch

import whiten_port as port
from test_cpu_entropy import fake_reference  # noqa: F401  (fixture)
from test_cpu_plumbing import _saferlhf_trainer, dry  # noqa: F401  (fixture)
from test_cpu_ppo_step import MULTI, _PPO_MODULES, _grafted, _ppo_trainer, _prompts, _standalone_class, full_lens, packed  # noqa: F401

TRAINERS = ['text', 'multi_gae', 'multi_reinforce', 'multi_rloo', 'multi_group_norm', 'image', 'audio']
WHITEN_CALLS = {'aa_whiten_moments', 'aa_whiten_reduce', 'aa_whiten_apply'}
K4_CALLS = {'aa_ppo_prep', 'aa_ppo_prep_kl', 'aa_ppo_returns'}


def _rollout(widths=(23, 7, 40), rows=(3, 1, 4), dtype=torch.float32, seed=0, loc=0.7, scale=1.9):
    """Micro-batches of different shapes, one all-masked-out row, masked-out NaNs (never read)."""
    g = torch.Generator().manual_seed(seed)
    advs, masks = [], []
    for B, W in zip(rows, widths):
        a = (torch.randn(B, W, generator=g, dtype=torch.float64) * scale + loc)
        m = torch.rand(B, W, generator=g) < 0.7
        a[~m] = float('nan')
        advs.append(a.to(dtype))
        masks.append(m)
    masks[0][1] = False
    return advs, masks


def _masked_whiten64(values, mask):
    """TRL's masked_whiten(values, mask, shift_mean=True) in float64 (masked_mean, masked_var with Bessel's correction),
    with the masked-out positions written as 0."""
    mask = mask.double()
    mean = (values * mask).sum() / mask.sum()
    variance = (((values - mean) ** 2) * mask).sum() / mask.sum()
    variance = variance * (mask.sum() / (mask.sum() - 1))
    whitened = (values - mean) * torch.rsqrt(variance + 1e-8)
    return torch.where(mask.bool(), whitened, torch.zeros_like(whitened))


@pytest.mark.parametrize('loc, scale', [(0.7, 1.9), (-3e3, 2.5), (0.0, 1e-5)])
def test_port_matches_float64_masked_whiten_over_the_rollout(loc, scale):
    advs, masks = _rollout(loc=loc, scale=scale)
    got = port.whiten(advs, masks)
    flat = torch.cat([a.double().flatten() for a in advs])
    want = _masked_whiten64(torch.nan_to_num(flat), torch.cat([m.flatten() for m in masks]))
    got_flat = torch.cat([g.double().flatten() for g in got])
    assert all(g.dtype == torch.float32 for g in got)
    # fp32 rounding of mean and rstd and of the two fp32 operations: a few fp32 ulps of |A - mean| * rstd, plus the
    # rounding of the fp32 mean, |mean| * 2^-24, carried through rstd
    n, mean, var = port.statistics(advs, masks)
    rstd = (var + 1e-8) ** -0.5
    tol = 4 * 2.0 ** -24 * (want.abs() + abs(mean) * rstd)
    assert bool(((got_flat - want).abs() <= tol).all()), float(((got_flat - want).abs() - tol).max())
    for g, m in zip(got, masks):
        assert torch.equal(g[~m], torch.zeros_like(g[~m]))  # masked-out positions (NaN on the way in): exactly 0


def test_port_rounds_once_to_the_advantages_dtype():
    for dtype in (torch.bfloat16, torch.float16):
        advs, masks = _rollout(dtype=dtype, seed=3)
        got = port.whiten(advs, masks)
        n, mean, var = port.statistics(advs, masks)
        mean32 = torch.tensor(mean).float()
        rstd32 = torch.rsqrt(torch.tensor(var, dtype=torch.float64) + 1e-8).float()
        for g, a, m in zip(got, advs, masks):
            assert g.dtype == dtype
            want = ((a.float() - mean32) * rstd32).to(dtype)
            assert torch.equal(g[m], want[m])


def test_port_leaves_fewer_than_two_tokens_unchanged():
    a = torch.tensor([[1.5, 2.0, -3.0]])
    for m in (torch.tensor([[False, True, False]]), torch.zeros(1, 3, dtype=torch.bool)):
        assert torch.equal(port.whiten([a], [m])[0], a)


# ---- the switch -----------------------------------------------------------------------------------------------------
def _video_class():
    from align_anything_b200.trainers.text_video_to_text.ppo import PPOTrainer

    return PPOTrainer


def test_switch_defaults_off_and_the_config_key_wins():
    from align_anything_b200.trainers.text_to_text import ppo as P

    for cls in {_standalone_class(t) for t in _PPO_MODULES} | {_video_class()}:
        assert cls.whiten_advantages is False and 'whiten_advantages' in cls.SWITCHES, cls
    t = object.__new__(P.PPOTrainer)
    t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace())
    assert P.whiten_advantages_of(t) is False
    t.whiten_advantages = True
    assert P.whiten_advantages_of(t) is True
    t.cfgs.train_cfgs.whiten_advantages = False  # the recipe's value wins over the attribute
    assert P.whiten_advantages_of(t) is False
    t.whiten_advantages, t.cfgs.train_cfgs.whiten_advantages = False, True
    assert P.whiten_advantages_of(t) is True
    t.cfgs.train_cfgs.whiten_advantages = None  # unset: the attribute
    assert P.whiten_advantages_of(t) is False


@pytest.mark.parametrize('bad', [1, 0, 'true', 'False', 1.0, [True]])
def test_non_bool_values_are_refused(bad):
    from align_anything_b200.trainers.text_to_text import ppo as P

    for where in ('attr', 'cfg'):
        t = object.__new__(P.PPOTrainer)
        t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(**({'whiten_advantages': bad} if where == 'cfg' else {})))
        if where == 'attr':
            t.whiten_advantages = bad
        with pytest.raises(ValueError, match='whiten_advantages'):
            P.whiten_advantages_of(t)


def test_install_grafts_the_switch(fake_reference):  # noqa: F811
    from align_anything_b200 import patch

    ppo = {m: c for m, c in fake_reference.items() if 'ppo' in m}
    assert ppo
    try:
        patch.install(models=False)
        for modname, cls in ppo.items():
            assert cls.__dict__.get('whiten_advantages') is False, modname
    finally:
        patch.uninstall()
    for modname, cls in ppo.items():
        assert 'whiten_advantages' not in cls.__dict__, modname


def test_safe_rlhf_v_refuses_the_switch(dry):  # noqa: F811
    from align_anything_b200.trainers.text_image_to_text.saferlhf import refuse_whitening

    t = _saferlhf_trainer()
    refuse_whitening(t)
    inference, training = t.rollout(t.prompt_only_dataloader[0])
    for where in ('attr', 'cfg'):
        t = _saferlhf_trainer()
        if where == 'attr':
            t.whiten_advantages = True
        else:
            t.cfgs.train_cfgs.whiten_advantages = True
        dry.calls.clear()
        with pytest.raises(ValueError, match='Safe RLHF-V'):
            t.rollout(t.prompt_only_dataloader[0])
        with pytest.raises(ValueError, match='Safe RLHF-V'):
            t.rl_step(inference[0], training[0])
        assert not dry.calls


# ---- argument checks ------------------------------------------------------------------------------------------------
def test_ops_refuses_bad_arguments_before_any_launch(dry):  # noqa: F811
    from align_anything_b200 import ops

    a, m = torch.zeros(2, 5), torch.ones(2, 5, dtype=torch.bool)
    for advs, masks, match in (([], [], 'at least one'), ([a, a], [m], 'one mask per'),
                               ([a], [m[:, 1:]], 'matching'), ([a[0]], [m[0]], 'matching'),
                               ([a.long()], [m], 'bf16 / fp16 / fp32'), ([a[:, :0]], [m[:, :0]], 'non-empty')):
        with pytest.raises(ValueError, match=match):
            ops.whiten_advantages(advs, masks)
    assert not dry.calls


def test_ops_refuses_cpu_tensors():
    from align_anything_b200 import ops

    with pytest.raises(ValueError, match='H100'):
        ops.whiten_advantages([torch.zeros(2, 5)], [torch.ones(2, 5, dtype=torch.bool)])


def test_entry_points_check_their_arguments_before_cuda():
    from align_anything_b200 import _lib

    lib = _lib.lib()
    buf = (ctypes.c_int64 * 16)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def moments(adv=p, dt=2, sa=8, mask=p, sm=8, B=2, W=8, out=p, k=0, K=1):
        return lib.aa_whiten_moments(adv, dt, sa, mask, sm, B, W, out, k, K, None)

    def apply(adv=p, dt=2, sa=8, mask=p, sm=8, B=2, W=8, total=p, status=p):
        return lib.aa_whiten_apply(adv, dt, sa, mask, sm, B, W, total, status, None)

    for name, fn in (('aa_whiten_moments', moments), ('aa_whiten_apply', apply)):
        for kw in ({'adv': None}, {'mask': None}, {'out': None} if fn is moments else {'total': None},
                   {} if fn is moments else {'status': None}):
            if kw:
                assert fn(**kw) == -2 and f'{name}: null pointer'.encode() in lib.aa_last_error(), (name, kw)
        for dt in (-1, 3, 7):
            assert fn(dt=dt) == -1 and f'{name}: bad dtype'.encode() in lib.aa_last_error()
        for kw in ({'B': 0}, {'W': 0}, {'B': -1}, {'W': -3}):
            assert fn(**kw) == -2 and f'{name}: bad sizes'.encode() in lib.aa_last_error(), (name, kw)
        for kw in ({'sa': 7}, {'sm': 4}):
            assert fn(**kw) == -2 and b'row strides must be >= W' in lib.aa_last_error(), (name, kw)
    assert moments(B=65536, W=32768, sa=32768, sm=32768) == -2 and b'bad sizes' in lib.aa_last_error()
    for k, K in ((1, 1), (-1, 2), (3, 2), (0, 0)):
        assert moments(k=k, K=K) == -2 and b'aa_whiten_moments: slot k=' in lib.aa_last_error(), (k, K)
    assert lib.aa_whiten_reduce(None, 1, p, None) == -2 and b'aa_whiten_reduce: null pointer' in lib.aa_last_error()
    assert lib.aa_whiten_reduce(p, 1, None, None) == -2
    assert lib.aa_whiten_reduce(p, 0, p, None) == -2 and b'aa_whiten_reduce: bad slot count' in lib.aa_last_error()


# ---- launches on the stand-in library -------------------------------------------------------------------------------
def _trainer(trainer, grafted, stack, whiten):
    module = MULTI if trainer.startswith('multi') else _PPO_MODULES[trainer]
    cls = stack.enter_context(_grafted())[module].PPOTrainer if grafted else _standalone_class(
        'multi_gae' if trainer.startswith('multi') else trainer)
    t = _ppo_trainer(cls, trainer)
    if whiten is not None:
        t.cfgs.train_cfgs.whiten_advantages = whiten
    return t


def _micro_batches(trainer):
    return 1 if trainer == 'image' else 2  # 4 prompts, per_device_train_batch_size 2; the image trainer scores at once


@pytest.mark.parametrize('grafted', [False, True])
@pytest.mark.parametrize('trainer', TRAINERS)
def test_switch_on_whitens_in_the_rollout_and_rl_step_reuses_it(dry, packed, full_lens, trainer, grafted):  # noqa: F811
    K = _micro_batches(trainer)
    group = trainer.startswith('multi') and trainer != 'multi_gae'
    with contextlib.ExitStack() as stack:
        t = _trainer(trainer, grafted, stack, True)
        inference, training = t.rollout(_prompts())
        assert len(training) == K
        assert dry.calls.count('aa_ppo_prep') == K and dry.calls.count('aa_ppo_returns') == (K if group else 0)
        assert [c for c in dry.calls if c in WHITEN_CALLS] == ['aa_whiten_moments'] * K + ['aa_whiten_reduce'] + \
            ['aa_whiten_apply'] * K
        assert dry.calls.index('aa_whiten_moments') > max(i for i, c in enumerate(dry.calls) if c in K4_CALLS)
        for tb in training:
            assert {'old_rewards', 'advantages', 'returns', 'row_stats'} <= set(tb)
        for _ in range(2):  # update_iters = 2: the stored tensors again, no K4 / K4r and no whitening
            dry.calls.clear()
            out = t.rl_step(inference[0], training[0])
            assert not (K4_CALLS | WHITEN_CALLS) & set(dry.calls)
            assert 'aa_ppo_pack_metrics' in dry.calls and 'train/reward_advantage' in out
            assert t.last_rl_tensors['advantages'] is training[0]['advantages']
            assert t.last_rl_tensors['returns'] is training[0]['returns']


@pytest.mark.parametrize('whiten', [None, False])
@pytest.mark.parametrize('trainer', TRAINERS)
def test_switch_off_makes_todays_calls(dry, packed, full_lens, trainer, whiten):  # noqa: F811
    group = trainer.startswith('multi') and trainer != 'multi_gae'
    with contextlib.ExitStack() as stack:
        t = _trainer(trainer, False, stack, whiten)
        inference, training = t.rollout(_prompts())
        assert not (K4_CALLS | WHITEN_CALLS) & set(dry.calls)
        assert not {'old_rewards', 'advantages', 'returns', 'row_stats'} & set(training[0])
        dry.calls.clear()
        t.rl_step(inference[0], training[0])
    assert dry.calls.count('aa_ppo_prep') == 1 and dry.calls.count('aa_ppo_returns') == (1 if group else 0)
    assert not WHITEN_CALLS & set(dry.calls)
    assert set(t.last_rl_tensors) == {'old_rewards', 'advantages', 'returns'}


def test_rollout_whitens_with_the_rollout_time_kl_coeff_and_estimator(dry, packed, full_lens, monkeypatch):  # noqa: F811
    from align_anything_b200 import ops

    seen = []
    real = ops.kl_rewards_and_gae

    def spy(*a, **kw):
        seen.append((a[6], kw.get('kl_estimator', 'k1')))
        return real(*a, **kw)

    monkeypatch.setattr(ops, 'kl_rewards_and_gae', spy)
    with contextlib.ExitStack() as stack:
        t = _trainer('text', False, stack, True)
        t.kl_estimator, t.kl_target, t.kl_coeff = 'k3', 0.01, 0.05
        inference, training = t.rollout(_prompts())
        assert seen == [(0.05, 'k3')] * 2 and dry.calls.count('aa_ppo_prep_kl') == 2
        t.kl_coeff = 0.5  # what an adaptive update between steps does: the stored tensors keep the rollout's
        dry.calls.clear()
        t.rl_step(inference[0], training[0])
        assert seen == [(0.05, 'k3')] * 2 and not K4_CALLS & set(dry.calls)
