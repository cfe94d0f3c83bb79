"""GRPO objective options without a GPU: the port (tests/grpo_objective_port.py) against the reference's loss and float64
autograd, ops.GrpoObjective's checks, the switches and their config precedence, the update loop's bookkeeping, the
graft of the switches and the argument checks of the new C entry points."""
from __future__ import annotations

import ctypes
import dataclasses
import types

import pytest
import torch

from grpo_objective_port import clip_fractions, completion_mask, group_advantages
from grpo_objective_port import grpo_loss as port_loss
from oracle import ref_port
from test_cpu_entropy import fake_reference  # noqa: F401  (fixture)

DTYPES = [torch.bfloat16, torch.float16, torch.float32]


def _inputs(B=6, K=29, dtype=torch.float32, seed=0, eos=1):
    g = torch.Generator().manual_seed(seed)
    lp = (-torch.rand(B, K, generator=g) * 4).to(dtype)
    ref = (lp.float() + torch.randn(B, K, generator=g) * 0.3).to(dtype)
    old = (lp.float() + torch.randn(B, K, generator=g) * 0.4).to(dtype)
    adv = torch.randn(B, 1, generator=g)
    tokens = torch.randint(2, 50, (B, K), generator=g)
    for b in range(0, B, 2):  # every other row ends early
        tokens[b, 3 + 2 * b] = eos
    return lp, ref, old, adv, tokens


def _grad(fn, lp, *args, **kw):
    x = lp.clone().requires_grad_(True)
    loss = fn(x, *args, **kw)
    loss.backward()
    return loss.detach(), x.grad


@pytest.mark.parametrize('dtype', DTYPES)
def test_default_port_is_the_reference_loss(dtype):
    lp, ref, _, adv, tokens = _inputs(dtype=dtype)
    prompt = torch.zeros(lp.size(0), 3, dtype=torch.int64)
    seq = torch.cat([prompt, tokens], 1)
    want, gwant = _grad(ref_port.grpo_loss, lp, ref, adv, seq, 3, 1, 0.04)
    got, ggot = _grad(port_loss, lp, ref, adv, completion_mask(tokens, 1), 0.04)
    assert got.dtype == want.dtype
    assert torch.equal(got, want)
    assert torch.equal(ggot, gwant)


def test_default_port_group_advantages_are_the_reference():
    r = torch.randn(12, generator=torch.Generator().manual_seed(1))
    assert torch.equal(group_advantages(r, 4), ref_port.grpo_group_advantages(r, 3, 4))
    torch.testing.assert_close(group_advantages(r, 4, scale=False).view(3, 4),
                               r.view(3, 4) - r.view(3, 4).mean(1, keepdim=True), rtol=0, atol=0)


def _f64(lp, ref, old, adv, mask, beta, lo, hi, c, agg):
    """The objective in float64 autograd, written independently of the port."""
    x = lp.double().clone().requires_grad_(True)
    o = x.detach() if old is None else old.double()
    r = torch.exp(x - o)
    a = adv.double().expand_as(r)
    s = torch.minimum(a * r, a * torch.clamp(r, 1.0 - lo, 1.0 + hi))
    if c is not None:
        s = torch.where(a < 0, torch.maximum(s, c * a), s)
    d = ref.double() - x
    ptl = -(s - beta * (torch.exp(d) - d - 1))
    m = mask.double()
    if agg == 'token-mean':
        loss = (ptl * m).sum() / m.sum()
    elif agg == 'seq-mean-token-mean':
        loss = ((ptl * m).sum(-1) / m.sum(-1)).mean()
    else:
        loss = (ptl * m).sum() / (m.size(0) * m.size(1))
    loss.backward()
    return loss.detach(), x.grad


OPTIONS = [
    (0.2, 0.2, None, 'token-mean'),
    (0.2, 0.28, None, 'token-mean'),
    (0.2, 0.2, 3.0, 'token-mean'),
    (0.2, 0.2, None, 'seq-mean-token-mean'),
    (0.2, 0.2, None, 'seq-mean-token-sum-norm'),
    (0.2, 0.28, 3.0, 'seq-mean-token-mean'),
]


@pytest.mark.parametrize('with_old', [False, True])
@pytest.mark.parametrize('opt', OPTIONS, ids=lambda o: f'{o[0]}-{o[1]}-{o[2]}-{o[3]}')
def test_port_matches_float64_autograd(opt, with_old):
    lo, hi, c, agg = opt
    lp, ref, old, adv, tokens = _inputs(B=8, K=41, dtype=torch.float64, seed=3)
    mask = completion_mask(tokens, 1)
    o = old if with_old else None
    got, ggot = _grad(port_loss, lp, ref, adv, mask, 0.04, o, lo, hi, c, agg)
    want, gwant = _f64(lp, ref, o, adv, mask, 0.04, lo, hi, c, agg)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(ggot, gwant, rtol=1e-12, atol=1e-14)


def test_first_update_ratio_is_one_and_matches_the_reference_gradient():
    # own log-probs as `old`: nothing is clipped and, in float64, the clipped form gives the reference's loss
    lp, ref, _, adv, tokens = _inputs(dtype=torch.float64, seed=5)
    mask = completion_mask(tokens, 1)
    want, gwant = _grad(port_loss, lp, ref, adv, mask, 0.04)
    got, ggot = _grad(port_loss, lp, ref, adv, mask, 0.04, None, 0.2, 0.28, 3.0, 'token-mean')
    torch.testing.assert_close(got, want, rtol=1e-14, atol=0)
    torch.testing.assert_close(ggot, gwant, rtol=1e-14, atol=0)
    assert clip_fractions(lp, None, adv, mask, 0.2, 0.28, 3.0) == (0.0, 0.0)


def test_clip_fractions_under_each_aggregation():
    ratio = torch.tensor([[1.5, 0.5, 1.0, 1.0], [1.0, 1.0, 0.1, 1.0]], dtype=torch.float64)
    adv = torch.tensor([[1.0], [-1.0]], dtype=torch.float64)
    mask = torch.tensor([[1, 1, 1, 0], [1, 1, 1, 1]])
    lp = torch.log(ratio)
    # row 0 (A = 1): token 0 clipped; row 1 (A = -1): token 2 (r = 0.1 < 0.8) clipped, c * A = -2 never wins
    fc, fd = clip_fractions(lp, torch.zeros_like(lp), adv, mask, 0.2, 0.2, 2.0, 'token-mean')
    assert fc == 2 / 7 and fd == 0.0
    assert clip_fractions(lp, torch.zeros_like(lp), adv, mask, 0.2, 0.2, 2.0, 'seq-mean-token-sum-norm') == (fc, fd)
    fc, _ = clip_fractions(lp, torch.zeros_like(lp), adv, mask, 0.2, 0.2, 2.0, 'seq-mean-token-mean')
    assert fc == pytest.approx((1 / 3 + 1 / 4) / 2)


def test_grpo_objective_checks_its_fields():
    from align_anything_b200.ops import ActorObjective, GrpoObjective

    assert GrpoObjective().is_default and GrpoObjective().loss_agg_mode == 'token-mean'
    assert GrpoObjective().args() == (0.2, 0.2, 0.0, 1)
    assert GrpoObjective(0.2, 0.28, 3.0, 'seq-mean-token-sum-norm').args() == (0.2, 0.28, 3.0, 2)
    assert GrpoObjective(loss_agg_mode='seq-mean-token-mean', clip_range_ratio=0.1).args() == (0.1, 0.1, 0.0, 0)
    assert not GrpoObjective(loss_agg_mode='seq-mean-token-mean').is_default
    assert not GrpoObjective(clip_range_ratio_high=0.28).is_default
    for bad in (dict(clip_range_ratio_low=1.0), dict(clip_range_ratio_low=float('nan')), dict(clip_range_ratio_high=-0.1),
                dict(dual_clip_ratio=1.0), dict(dual_clip_ratio=float('inf')), dict(loss_agg_mode='seq-sum'),
                dict(clip_range_ratio=1.0), dict(clip_range_ratio=-0.5)):
        with pytest.raises(ValueError):
            GrpoObjective(**bad)
    # the PPO objective keeps its two modes
    with pytest.raises(ValueError):
        ActorObjective(loss_agg_mode='seq-mean-token-sum-norm')
    assert ActorObjective().args(0.2) == (0.2, 0.2, 0.0, 0)
    with pytest.raises(dataclasses.FrozenInstanceError):
        GrpoObjective().clip_range_ratio = 0.3


def test_switches_default_to_the_reference_and_config_keys_win():
    from align_anything_b200.ops import GrpoObjective
    from align_anything_b200.trainers.text_to_text import grpo as G

    cls = G.GRPOTrainer
    assert (cls.num_iterations, cls.clip_range_ratio, cls.clip_range_ratio_low, cls.clip_range_ratio_high,
            cls.dual_clip_ratio, cls.loss_agg_mode, cls.scale_rewards, cls.log_clip_fraction) == \
        (1, 0.2, None, None, None, 'token-mean', True, False)
    tr = G.GRPOTrainer()
    assert G.grpo_objective_of(tr) is None and G.num_iterations_of(tr) == 1
    tc = types.SimpleNamespace(num_iterations=None, clip_range_ratio=None, clip_range_ratio_low=None,
                               clip_range_ratio_high=0.28, dual_clip_ratio=None, loss_agg_mode=None, update_iters=1)
    tr = G.GRPOTrainer(types.SimpleNamespace(train_cfgs=tc))
    assert G.grpo_objective_of(tr) == GrpoObjective(clip_range_ratio_high=0.28)
    tc.clip_range_ratio_high, tc.num_iterations, tc.update_iters = None, 2, 2
    assert G.num_iterations_of(tr) == 2
    assert G.grpo_objective_of(tr) == GrpoObjective()  # mu > 1: the clipped ratio even with default fields
    tc.loss_agg_mode = 'seq-mean-token-sum-norm'
    assert G.grpo_objective_of(tr).loss_agg_mode == 'seq-mean-token-sum-norm'
    tr.num_iterations = 3  # the recipe's value wins over the attribute
    assert G.num_iterations_of(tr) == 2
    tc.dual_clip_ratio = 0.5
    with pytest.raises(ValueError):
        G.grpo_objective_of(tr)


def test_num_iterations_is_checked_against_update_iters():
    from align_anything_b200.trainers.text_to_text import grpo as G

    tc = types.SimpleNamespace(update_iters=1, num_iterations=None)
    tr = G.GRPOTrainer(types.SimpleNamespace(train_cfgs=tc))
    assert G.num_iterations_of(tr) == 1
    tr.num_iterations = 4
    with pytest.raises(ValueError, match='update_iters'):
        G.num_iterations_of(tr)
    tc.update_iters = 4
    assert G.num_iterations_of(tr) == 4
    for bad in (0, -1, 1.5, True):
        tr.num_iterations = bad
        with pytest.raises(ValueError):
            G.num_iterations_of(tr)


class _Engine:
    def __init__(self, calls):
        self.calls = calls

    def __call__(self, **kw):
        self.calls.append('forward')
        return types.SimpleNamespace(logits=None)

    def zero_grad(self):
        self.calls.append('zero_grad')

    def backward(self, loss):
        self.calls.append(('backward', float(loss.detach())))

    def step(self):
        self.calls.append('step')


def _fake_step(monkeypatch, mu, **attrs):
    """One step_from_rollout with CPU stand-ins for the device work: -> (output, engine calls, loss calls, packs)."""
    from align_anything_b200.trainers.text_to_text import grpo as G

    packed, seen, calls = [], [], []
    monkeypatch.setattr(G, 'all_reduce_packed', lambda stats, max_lanes=(): packed.append(stats.clone()) or stats)
    monkeypatch.setattr(G.ops, 'group_advantages',
                        lambda r, n, scale=True: seen.append(('adv', scale)) or r.view(-1, 1))
    monkeypatch.setattr(G.ops, 'status_lane', lambda dev: torch.zeros(1))
    monkeypatch.setattr(G.ops, 'raise_for_status', lambda v, dev: int(v))

    def fake_loss(logits, seq, K, ref, adv, eos, beta, mode=None, return_entropy=False, **kw):
        i = len([s for s in seen if s[0] == 'loss'])
        seen.append(('loss', kw))
        loss = torch.tensor(0.25 * (i + 1), requires_grad=True) * 1
        lp = torch.full((seq.size(0), K), -float(i + 1))
        out = (loss, lp, torch.full((seq.size(0),), K, dtype=torch.int32))
        return out + (torch.tensor([0.125 * (i + 1), 0.5]),) if kw.get('return_clip_fraction') else out

    monkeypatch.setattr(G.ops, 'grpo_loss_from_logits', fake_loss)
    tr = G.GRPOTrainer(None, _Engine(calls), _Engine(calls), types.SimpleNamespace(pad_token_id=0, eos_token_id=1),
                       beta=0.1, num_generations=2)
    tr.num_iterations = mu
    for k, v in attrs.items():
        setattr(tr, k, v)
    n_ref = []
    tr._get_per_token_logps = lambda *a, **k: n_ref.append(1) or torch.zeros(2, 3)
    out = tr.step_from_rollout(torch.ones(2, 5, dtype=torch.int64), 2, torch.tensor([1.0, 2.0]))
    return out, calls, seen, packed, n_ref


def test_update_loop_bookkeeping(monkeypatch):
    out, calls, seen, packed, n_ref = _fake_step(monkeypatch, 3, log_clip_fraction=True, dual_clip_ratio=3.0)
    assert len(n_ref) == 1  # the reference model is scored once per rollout
    assert [c for c in calls if c == 'step'] == ['step'] * 3
    assert [c[1] for c in calls if isinstance(c, tuple)] == [0.25, 0.5, 0.75]
    assert calls == ['forward', 'zero_grad', ('backward', 0.25), 'step'] + \
        ['forward', 'zero_grad', ('backward', 0.5), 'step'] + ['forward', 'zero_grad', ('backward', 0.75), 'step']
    losses = [s[1] for s in seen if s[0] == 'loss']
    assert [s for s in seen if s[0] == 'adv'] == [('adv', True)]
    assert 'old_per_token_logps' not in losses[0]  # the first update: the ratio is 1
    for kw in losses[1:]:  # updates 2..mu: the first update's log-probs
        assert torch.equal(kw['old_per_token_logps'], torch.full((2, 3), -1.0))
    assert all(kw['objective'].dual_clip_ratio == 3.0 and kw['return_clip_fraction'] for kw in losses)
    assert len(packed) == 1  # one collective, one sync per rollout
    assert out['train/loss'] == pytest.approx(0.5)
    assert out['train/actor_clip_fraction'] == pytest.approx(0.25)
    assert out['train/actor_dual_clip_fraction'] == pytest.approx(0.5)
    assert packed[0].numel() == 5


def test_single_update_with_default_switches_is_todays_step(monkeypatch):
    out, calls, seen, packed, _ = _fake_step(monkeypatch, 1)
    assert set(out) == {'train/loss', 'train/reward'} and out['train/loss'] == 0.25
    assert [s[1] for s in seen if s[0] == 'loss'] == [{}]  # no objective keyword reaches the loss
    assert packed[0].numel() == 3 and calls.count('step') == 1


def test_scale_rewards_switch_reaches_the_advantages(monkeypatch):
    _, _, seen, _, _ = _fake_step(monkeypatch, 1, scale_rewards=False, loss_agg_mode='seq-mean-token-sum-norm')
    assert [s for s in seen if s[0] == 'adv'] == [('adv', False)]
    kw = [s[1] for s in seen if s[0] == 'loss'][0]
    assert kw['objective'].loss_agg_mode == 'seq-mean-token-sum-norm'


def test_update_iters_mismatch_raises_before_the_first_pass(monkeypatch):
    with pytest.raises(ValueError, match='update_iters'):
        from align_anything_b200.trainers.text_to_text import grpo as G

        calls = []
        tr = G.GRPOTrainer(types.SimpleNamespace(train_cfgs=types.SimpleNamespace(update_iters=1, num_iterations=2)),
                           _Engine(calls), _Engine(calls), types.SimpleNamespace(pad_token_id=0, eos_token_id=1))
        try:
            tr.step_from_rollout(torch.ones(2, 5, dtype=torch.int64), 2, torch.tensor([1.0, 2.0]))
        finally:
            assert calls == []


def test_install_sets_and_uninstall_restores_the_grpo_switches(fake_reference):  # noqa: F811
    from align_anything_b200 import patch

    keys = ('num_iterations', 'clip_range_ratio', 'clip_range_ratio_low', 'clip_range_ratio_high', 'dual_clip_ratio',
            'loss_agg_mode', 'scale_rewards', 'log_clip_fraction')
    grpo = {m: c for m, c in fake_reference.items() if 'grpo' in m}
    assert grpo
    try:
        patch.install(models=False)
        for modname, cls in grpo.items():
            for k in keys:
                assert k in cls.__dict__, (modname, k)
            assert cls.num_iterations == 1 and cls.loss_agg_mode == 'token-mean' and cls.scale_rewards is True
    finally:
        patch.uninstall()
    for modname, cls in grpo.items():
        for k in keys:
            assert k not in cls.__dict__, (modname, k)


def test_new_entry_points_check_the_objective_before_cuda():
    from align_anything_b200 import _lib

    lib = _lib.lib()
    buf = (ctypes.c_int64 * 8)()
    ptr = ctypes.cast(buf, ctypes.c_void_p)

    def loss(lo, hi, c, agg, mode=0):
        return lib.aa_grpo_loss_obj(ptr, 8, ptr, 8, None, 0, 2, ptr, ptr, 8, 1, 2, 8, 0.04, lo, hi, c, agg, mode, ptr,
                                    ptr, 8, None, ptr, ptr, ptr, None)

    def k1f(lo, hi, c, agg, coeff=0.0, ent=None):
        return lib.aa_logprob_grpo_fused_obj(ptr, 0, 64, 64, ptr, 1, ptr, ptr, ptr, ptr, ptr, 2, ptr, 0, ptr, 8, None,
                                             ptr, ptr, 8, 1, 8, 0.04, lo, hi, c, agg, 0, ptr, 64, ptr, ptr, ptr, ptr,
                                             ptr, ent, coeff, None)

    for fn, name in ((loss, b'aa_grpo_loss_obj'), (k1f, b'aa_logprob_grpo_fused_obj')):
        for bad in ((1.0, 0.2, 0.0, 1), (-0.1, 0.2, 0.0, 1), (0.2, -0.1, 0.0, 1), (0.2, 0.2, 1.0, 1), (0.2, 0.2, 0.5, 1),
                    (0.2, 0.2, 0.0, 3), (0.2, 0.2, 0.0, -1), (float('nan'), 0.2, 0.0, 1), (0.2, 0.2, float('nan'), 1)):
            rc = fn(*bad)
            assert rc == -2 and name + b': bad objective' in lib.aa_last_error(), bad
    assert loss(0.2, 0.2, 0.0, 2, mode=7) == -2 and b'bad mode' in lib.aa_last_error()
    assert k1f(0.2, 0.28, 3.0, 2, coeff=float('nan'), ent=ptr) == -2 and b'entropy_coeff is NaN' in lib.aa_last_error()
    assert k1f(0.2, 0.28, 3.0, 2, coeff=0.01) == -2 and b'needs entropy' in lib.aa_last_error()
    assert lib.aa_group_advantages_centered(None, 1, 4, ptr, None) == -2
    # the PPO entry points still refuse GRPO's third aggregation
    rc = lib.aa_ppo_actor_loss_obj(ptr, 8, ptr, 8, 2, ptr, 8, 2, ptr, 8, 2, 8, 0.2, 0.2, 0.0, 2, 0, ptr, ptr, 8, None,
                                   ptr, ptr, None)
    assert rc == -2 and b'bad objective' in lib.aa_last_error()
