"""PPO actor objective options without a GPU: the port (tests/ppo_objective_port.py) against the reference's actor loss
and float64 autograd, ops.ActorObjective's checks, the config precedence of the switches, the graft of the switches
and the argument checks of the new C entry points."""
from __future__ import annotations

import ctypes
import dataclasses
import types

import pytest
import torch

from oracle import ref_port
from ppo_objective_port import actor_loss as port_loss
from ppo_objective_port import clip_fractions
from test_cpu_entropy import fake_reference  # noqa: F401  (fixture)

DTYPES = [torch.bfloat16, torch.float16, torch.float32]


def _inputs(B=4, W=37, dtype=torch.float32, seed=0):
    g = torch.Generator().manual_seed(seed)
    lp = (-torch.rand(B, W, generator=g) * 4).to(dtype)
    old = (lp.float() + torch.randn(B, W, generator=g) * 0.4).to(dtype)
    adv = torch.randn(B, W, generator=g).to(dtype)
    mask = torch.rand(B, W, generator=g) > 0.25
    mask[:, 0] = True
    return lp, old, adv, mask


def _grad(fn, lp, *args, **kw):
    x = lp.clone().requires_grad_(True)
    loss = fn(x, *args, **kw)
    loss.backward()
    return loss.detach(), x.grad


@pytest.mark.parametrize('dtype', DTYPES)
def test_default_port_is_the_reference_actor_loss(dtype):
    lp, old, adv, mask = _inputs(dtype=dtype)
    want, gwant = _grad(ref_port.actor_loss, lp, old, adv, mask, 0.2)
    got, ggot = _grad(port_loss, lp, old, adv, mask, 0.2, 0.2)
    assert got.dtype == want.dtype
    assert torch.equal(got, want)
    assert torch.equal(ggot, gwant)


def _f64(lp, old, adv, mask, lo, hi, c, agg):
    """The objective in float64 autograd, written independently of the port (explicit branch selection)."""
    x = lp.double().clone().requires_grad_(True)
    r = torch.exp(x - old.double())
    a = adv.double()
    s = torch.minimum(a * r, a * torch.clamp(r, 1.0 - lo, 1.0 + hi))
    if c is not None:
        s = torch.where(a < 0, torch.maximum(s, c * a), s)
    m = mask.double()
    loss = -((s * m).sum(-1) / m.sum(-1)).mean() if agg == 'seq-mean-token-mean' else -(s * m).sum() / m.sum()
    loss.backward()
    return loss.detach(), x.grad


OPTIONS = [
    (0.2, 0.2, None, 'seq-mean-token-mean'),
    (0.2, 0.28, None, 'seq-mean-token-mean'),
    (0.2, 0.2, 3.0, 'seq-mean-token-mean'),
    (0.2, 0.2, None, 'token-mean'),
    (0.2, 0.28, 3.0, 'token-mean'),
]


@pytest.mark.parametrize('opt', OPTIONS, ids=lambda o: f'{o[0]}-{o[1]}-{o[2]}-{o[3]}')
def test_port_matches_float64_autograd_on_random_inputs(opt):
    lo, hi, c, agg = opt
    lp, old, adv, mask = _inputs(B=6, W=53, dtype=torch.float64, seed=3)
    got, ggot = _grad(port_loss, lp, old, adv, mask, lo, hi, c, agg)
    want, gwant = _f64(lp, old, adv, mask, lo, hi, c, agg)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(ggot, gwant, rtol=1e-12, atol=1e-14)


def test_port_ties_split_the_gradient_like_autograd():
    # float64 operands, ratios exactly at the bounds, s1 == s2 inside the range and c * A == min(s1, s2)
    lo, hi, c = 0.25, 0.5, 2.0
    ratio = torch.tensor([[0.75, 1.5, 1.0, 4.0, 0.125, 1.25]], dtype=torch.float64)
    adv = torch.tensor([[1.0, -1.0, 0.5, -0.5, -2.0, 0.0]], dtype=torch.float64)
    old = torch.zeros_like(ratio)
    lp = torch.log(ratio)
    lp = torch.where(ratio == 1.0, torch.zeros_like(lp), lp)
    mask = torch.ones_like(ratio, dtype=torch.bool)
    # token 3: r = 4 clamps to 1.5, A = -0.5: min(-2, -0.75) = -2 == c * A? no: c * A = -1 -> dual wins
    # token 4: r = 0.125, A = -2: s1 = -0.25, s2 = -1.5 -> min -1.5; c * A = -4 -> min wins
    for agg in ('seq-mean-token-mean', 'token-mean'):
        got, ggot = _grad(port_loss, lp, old, adv, mask, lo, hi, c, agg)
        want, gwant = _f64(lp, old, adv, mask, lo, hi, c, agg)
        torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-14)
        torch.testing.assert_close(ggot, gwant, rtol=1e-12, atol=1e-14)
    # a tie of c * A with min(s1, s2): A = -1, r = 2 (clamped to 1.5), c = 2: min(-2, -1.5) = -2 == c * A
    lp2 = torch.log(torch.tensor([[2.0]], dtype=torch.float64))
    a2 = torch.tensor([[-1.0]], dtype=torch.float64)
    _, g = _grad(port_loss, lp2, torch.zeros_like(lp2), a2, torch.ones_like(a2, dtype=torch.bool), lo, hi, c)
    # d(-max(s, cA))/ds = -1/2 on the tie; ds/dlp = A * r = -2  ->  +1
    assert float(g) == 1.0
    _, gw = _f64(lp2, torch.zeros_like(lp2), a2, torch.ones_like(a2, dtype=torch.bool), lo, hi, c, 'seq-mean-token-mean')
    assert float(gw) == 1.0


def test_clip_fractions_count_the_branches():
    lo, hi, c = 0.2, 0.2, 2.0
    ratio = torch.tensor([[1.5, 0.5, 1.0, 3.0], [1.0, 1.0, 0.1, 1.0]], dtype=torch.float64)
    adv = torch.tensor([[1.0, -1.0, 1.0, -1.0], [1.0, 1.0, -1.0, -1.0]], dtype=torch.float64)
    mask = torch.tensor([[True, True, True, True], [True, True, True, False]])
    lp = torch.log(ratio)
    # row 0: token 0 clipped (A > 0, r > 1.2), token 1 clipped (A < 0, r < 0.8: -0.8 < -0.5), token 3 unclipped
    # (min(-3, -1.2) = -3) and c * A = -2 wins; row 1: token 2: r = 0.1, A = -1: s1 = -0.1, s2 = -0.8 -> clipped,
    # c * A = -2 loses
    fc, fd = clip_fractions(lp, torch.zeros_like(lp), adv, mask, lo, hi, c, 'token-mean')
    assert fc == 3 / 7 and fd == 1 / 3
    fc, fd = clip_fractions(lp, torch.zeros_like(lp), adv, mask, lo, hi, c, 'seq-mean-token-mean')
    assert fc == pytest.approx((2 / 4 + 1 / 3) / 2) and fd == pytest.approx((1 / 4) / (2 / 4 + 1 / 3))


def test_actor_objective_checks_its_fields():
    from align_anything_b200.ops import ActorObjective

    assert ActorObjective().is_default
    assert ActorObjective().args(0.2) == (0.2, 0.2, 0.0, 0)
    assert ActorObjective(0.2, 0.28, 3.0, 'token-mean').args(0.1) == (0.2, 0.28, 3.0, 1)
    assert not ActorObjective(clip_range_ratio_high=0.28).is_default
    for bad in (dict(clip_range_ratio_low=1.0), dict(clip_range_ratio_low=-0.1), dict(clip_range_ratio_low=float('nan')),
                dict(clip_range_ratio_high=-0.01), dict(dual_clip_ratio=1.0), dict(dual_clip_ratio=0.5),
                dict(dual_clip_ratio=float('inf')), dict(loss_agg_mode='seq-mean-token-sum')):
        with pytest.raises(ValueError):
            ActorObjective(**bad)
    with pytest.raises(ValueError):
        ActorObjective(clip_range_ratio_high=0.3).args(1.5)  # the trainer's clip range fills the low bound
    with pytest.raises(dataclasses.FrozenInstanceError):
        ActorObjective().dual_clip_ratio = 2.0


def test_objective_switches_default_off_on_every_ppo_trainer():
    from align_anything_b200.trainers.text_audio_to_text.ppo import PPOTrainer as Audio
    from align_anything_b200.trainers.text_image_to_text.ppo import PPOTrainer as Image
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer as Multi
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer, actor_objective_of, objective_kwargs
    from align_anything_b200.trainers.text_video_to_text.ppo import PPOTrainer as Video

    for cls in (PPOTrainer, Multi, Image, Audio, Video):
        for key in ('clip_range_ratio_low', 'clip_range_ratio_high', 'dual_clip_ratio', 'loss_agg_mode'):
            assert getattr(cls, key) is None, (cls, key)
        assert cls.log_clip_fraction is False
        tr = types.SimpleNamespace(cfgs=None, **{k: getattr(cls, k) for k in (
            'clip_range_ratio_low', 'clip_range_ratio_high', 'dual_clip_ratio', 'loss_agg_mode', 'log_clip_fraction')})
        assert actor_objective_of(tr) is None and objective_kwargs(tr) == {}


def test_config_keys_take_precedence_over_the_attributes():
    from align_anything_b200.ops import ActorObjective
    from align_anything_b200.trainers.text_to_text.ppo import actor_objective_of, entropy_coeff_of

    tr = types.SimpleNamespace(clip_range_ratio_low=None, clip_range_ratio_high=0.28, dual_clip_ratio=None,
                               loss_agg_mode=None, entropy_coeff=0.0, cfgs=None)
    assert actor_objective_of(tr) == ActorObjective(clip_range_ratio_high=0.28)
    tc = types.SimpleNamespace(clip_range_ratio_low=None, clip_range_ratio_high=None, dual_clip_ratio=3.0,
                               loss_agg_mode='token-mean', entropy_coeff=None)
    tr.cfgs = types.SimpleNamespace(train_cfgs=tc)
    assert actor_objective_of(tr) == ActorObjective(clip_range_ratio_high=0.28, dual_clip_ratio=3.0,
                                                    loss_agg_mode='token-mean')
    tc.clip_range_ratio_high = 0.3  # the recipe's value wins over the attribute
    assert actor_objective_of(tr).clip_range_ratio_high == 0.3
    tc.dual_clip_ratio = 0.5
    with pytest.raises(ValueError):
        actor_objective_of(tr)
    assert entropy_coeff_of(tr) == 0.0  # the entropy coefficient keeps its rule


def test_install_sets_and_uninstall_restores_the_objective_switches(fake_reference):  # noqa: F811
    from align_anything_b200 import patch

    keys = ('clip_range_ratio_low', 'clip_range_ratio_high', 'dual_clip_ratio', 'loss_agg_mode', 'log_clip_fraction')
    ppo = {m: c for m, c in fake_reference.items() if 'ppo' in m}
    assert ppo
    try:
        patch.install(models=False)
        for modname, cls in ppo.items():
            for k in keys:
                assert k in cls.__dict__, (modname, k)
            assert cls.dual_clip_ratio is None and cls.log_clip_fraction is False
    finally:
        patch.uninstall()
    for modname, cls in ppo.items():
        for k in keys:
            assert k not in cls.__dict__, (modname, k)


def test_new_entry_points_check_the_objective_before_cuda():
    from align_anything_b200 import _lib

    lib = _lib.lib()
    buf = (ctypes.c_int64 * 8)()
    ptr = ctypes.cast(buf, ctypes.c_void_p)

    def k5(lo, hi, c, agg, mode=0):
        return lib.aa_ppo_actor_loss_obj(ptr, 8, ptr, 8, 2, ptr, 8, 2, ptr, 8, 2, 8, lo, hi, c, agg, mode, ptr, ptr, 8,
                                         None, ptr, ptr, None)

    def k1f(lo, hi, c, agg):
        return lib.aa_logprob_actor_fused_obj(ptr, 0, 64, 64, ptr, 1, ptr, ptr, ptr, ptr, ptr, 2, ptr, 0, None, None, ptr,
                                              8, ptr, 8, 2, ptr, 8, 8, lo, hi, c, agg, 0, ptr, 64, ptr, ptr, 0.0, None,
                                              None)

    for fn, name in ((k5, b'aa_ppo_actor_loss_obj'), (k1f, b'aa_logprob_actor_fused_obj')):
        for bad in ((1.0, 0.2, 0.0, 0), (-0.1, 0.2, 0.0, 0), (0.2, -0.1, 0.0, 0), (0.2, 0.2, 1.0, 0), (0.2, 0.2, 0.5, 0),
                    (0.2, 0.2, 0.0, 2), (float('nan'), 0.2, 0.0, 0), (0.2, 0.2, float('nan'), 0)):
            rc = fn(*bad)
            assert rc == -2 and name + b': bad objective' in lib.aa_last_error(), bad
    assert k5(0.2, 0.2, 0.0, 0, mode=7) == -2 and b'bad mode' in lib.aa_last_error()
    rc = lib.aa_logprob_actor_fused_obj(ptr, 0, 64, 64, ptr, 1, ptr, ptr, ptr, ptr, ptr, 2, ptr, 0, None, None, ptr, 8,
                                        ptr, 8, 2, ptr, 8, 8, 0.2, 0.28, 3.0, 1, 0, ptr, 64, ptr, ptr, float('nan'), ptr,
                                        None)
    assert rc == -2 and b'entropy_coeff is NaN' in lib.aa_last_error()
