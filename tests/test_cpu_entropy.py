"""Policy entropy without a GPU: the merge rule the kernels use, restated in Python against float64, the `log_entropy`
switch that patch.install() puts on the trainer classes, and the metric key's absence when the switch is off."""
from __future__ import annotations

import math
import random
import sys
import types

import numpy as np
import pytest


def _fold(xs):
    """(m, s, t) of a run of logits: m = max, s = sum e^{x - m}, t = sum e^{x - m} (x - m) (-inf adds nothing)."""
    fin = [x for x in xs if x != -math.inf]
    if not fin:
        return -math.inf, 0.0, 0.0
    m = max(fin)
    s = sum(math.exp(x - m) for x in fin)
    t = sum(math.exp(x - m) * (x - m) for x in fin)
    return m, s, t


def _merge(a, b):
    """The kernels' rule (logprob_math.cuh ent_rescale / lse_merge_t, K6's split merge): moving a partial from its
    maximum m to m' scales it by alpha = e^{m - m'} and t' = alpha (t + (m - m') s)."""
    (m1, s1, t1), (m2, s2, t2) = a, b
    mn = max(m1, m2)
    if mn == -math.inf:
        return mn, 0.0, 0.0

    def move(m, s, t):
        if m == -math.inf:
            return 0.0, 0.0
        al = math.exp(m - mn)
        return al * s, al * (t + (m - mn) * s)

    sa, ta = move(m1, s1, t1)
    sb, tb = move(m2, s2, t2)
    return mn, sa + sb, ta + tb


def _entropy(m, s, t):
    return math.log(s) - t / s if s > 0 else math.nan


def _entropy64(xs):
    x = np.asarray(xs, dtype=np.float64)
    fin = x[np.isfinite(x)]
    if fin.size == 0:
        return math.nan
    lp = fin - (fin.max() + np.log(np.exp(fin - fin.max()).sum()))
    return float(-(np.exp(lp) * lp).sum())


@pytest.mark.parametrize('seed', range(8))
def test_merge_rule_matches_float64(seed):
    rng = random.Random(seed)
    V = rng.choice([7, 100, 1000, 5003])
    xs = [rng.gauss(0, rng.choice([0.1, 1, 5, 20])) for _ in range(V)]
    for _ in range(V // 10):
        xs[rng.randrange(V)] = -math.inf
    # random split points, merged in a random tree order (as the thread / warp / split merges do)
    cuts = sorted(rng.sample(range(1, V), min(V - 1, rng.randint(1, 12))))
    parts = [_fold(xs[a:b]) for a, b in zip([0] + cuts, cuts + [V])]
    while len(parts) > 1:
        i = rng.randrange(len(parts) - 1)
        parts[i:i + 2] = [_merge(parts[i], parts[i + 1])]
    got = _entropy(*parts[0])
    assert abs(got - _entropy64(xs)) <= 1e-9 * max(1.0, abs(got)), (got, _entropy64(xs))


def test_merge_rule_edge_rows():
    assert math.isnan(_entropy(*_merge(_fold([-math.inf] * 3), _fold([-math.inf]))))  # all -inf: NaN
    uni = _merge(_fold([2.0] * 40), _fold([2.0] * 60))
    assert abs(_entropy(*uni) - math.log(100)) < 1e-12  # uniform: log V
    one = _merge(_fold([50.0]), _fold([0.0] * 9))
    assert 0 <= _entropy(*one) < 1e-18  # near one-hot: ~0
    assert _merge(_fold([]), _fold([1.0, 2.0])) == _fold([1.0, 2.0])  # an empty partial changes nothing


# ---- the switch ---------------------------------------------------------------------------------------------------------
_CLASSES = {
    'align_anything.trainers.text_to_text.ppo': 'PPOTrainer',
    'align_anything.trainers.text_image_to_text.ppo': 'PPOTrainer',
    'align_anything.trainers.text_audio_to_text.ppo': 'PPOTrainer',
    'align_anything.trainers.text_video_to_text.ppo': 'PPOTrainer',
    'align_anything.trainers.text_to_text.multi_ppo': 'PPOTrainer',
    'align_anything.trainers.text_to_text.grpo': 'GRPOTrainer',
}


@pytest.fixture
def fake_reference(monkeypatch):
    """Just enough of an importable `align_anything` for patch.install(): the tools module and the PPO / GRPO classes."""
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        monkeypatch.setitem(sys.modules, name, m)
        return m

    for name in ('align_anything', 'align_anything.utils', 'align_anything.trainers', 'align_anything.trainers.text_to_text',
                 'align_anything.trainers.text_image_to_text', 'align_anything.trainers.text_audio_to_text',
                 'align_anything.trainers.text_video_to_text'):
        mod(name)
    mod('align_anything.utils.tools', gather_log_probabilities=lambda *a: None, masked_mean=lambda *a: None,
        move_padding_left=lambda *a: None)
    classes = {}
    for modname, clsname in _CLASSES.items():
        cls = type(clsname, (), {'rl_step': lambda self: 'reference', 'train_step': lambda self: 'reference'})
        mod(modname, **{clsname: cls})
        classes[modname] = cls
    return classes


def test_install_sets_and_uninstall_restores_log_entropy(fake_reference):
    from align_anything_b200 import patch

    try:
        patch.install(models=False)
        for modname, cls in fake_reference.items():
            assert cls.__dict__.get('log_entropy', 'missing') is False, modname
    finally:
        patch.uninstall()
    for modname, cls in fake_reference.items():
        assert 'log_entropy' not in cls.__dict__, modname
        assert cls.rl_step(None) == 'reference'


def test_log_entropy_defaults_off():
    from align_anything_b200.trainers.text_audio_to_text.ppo import PPOTrainer as Audio
    from align_anything_b200.trainers.text_image_to_text.ppo import PPOTrainer as Image
    from align_anything_b200.trainers.text_to_text.grpo import GRPOTrainer
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer as Multi
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer as Text
    from align_anything_b200.trainers.text_video_to_text.ppo import PPOTrainer as Video

    for cls in (Text, Multi, Image, Audio, Video, GRPOTrainer):
        assert cls.log_entropy is False, cls


def test_metric_key_absent_when_off(monkeypatch):
    """GRPO's step with the switch off packs and returns exactly what it did before (no entropy lane, no key); the
    device work is replaced by CPU stand-ins so that only the bookkeeping runs."""
    import torch

    from align_anything_b200.trainers.text_to_text import grpo as G

    packed = []

    def fake_reduce(stats, max_lanes=()):
        packed.append(stats.clone())
        return stats

    monkeypatch.setattr(G, 'all_reduce_packed', fake_reduce)
    monkeypatch.setattr(G.ops, 'group_advantages', lambda r, n: r.view(-1, 1))
    monkeypatch.setattr(G.ops, 'status_lane', lambda dev: torch.zeros(1))
    monkeypatch.setattr(G.ops, 'raise_for_status', lambda v, dev: int(v))
    loss = torch.tensor(0.5, requires_grad=True)
    seen = {}

    def fake_loss(logits, seq, K, ref, adv, eos, beta, mode=None, return_entropy=False):
        seen['return_entropy'] = return_entropy
        return loss * 1, torch.zeros(seq.size(0), K), torch.full((seq.size(0),), K, dtype=torch.int32)

    monkeypatch.setattr(G.ops, 'grpo_loss_from_logits', fake_loss)

    class Model:
        def __call__(self, **kw):
            return types.SimpleNamespace(logits=None)

        def zero_grad(self):
            pass

        def backward(self, loss):
            pass

        def step(self):
            pass

    tr = G.GRPOTrainer(None, Model(), Model(), types.SimpleNamespace(pad_token_id=0, eos_token_id=1), beta=0.1,
                       num_generations=2)
    tr._get_per_token_logps = lambda *a, **k: torch.zeros(2, 3)
    out = tr.step_from_rollout(torch.ones(2, 5, dtype=torch.int64), 2, torch.tensor([1.0, 2.0]))
    assert set(out) == {'train/loss', 'train/reward'}
    assert seen['return_entropy'] is False
    assert packed[0].numel() == 3
