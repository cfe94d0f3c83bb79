"""Entropy bonus without a GPU: the gradient-tile formula the kernels implement against float64 autograd, the
`entropy_coeff` switch that patch.install() puts on the trainer classes, the config key's precedence and the argument
checks of the new C entry points."""
from __future__ import annotations

import ctypes
import types

import numpy as np
import pytest
import torch

from test_cpu_entropy import fake_reference  # noqa: F401  (fixture)


def _tile(x: np.ndarray, y: int, g: float, g_h: float) -> np.ndarray:
    """The kernels' tile in float64: g (onehot_y - p) - g_H p (l + H), a -inf logit's l clamped as in the kernels."""
    m = x.max()
    s = np.exp(x - m).sum()
    lp = (x - m) - np.log(s)
    p = np.exp(lp)
    lc = np.maximum(lp, -3.0e38)
    h = -(p * lc).sum()
    onehot = np.zeros_like(x)
    onehot[y] = 1.0
    return g * (onehot - p) - g_h * p * (lc + h)


def _autograd(x: np.ndarray, y: int, g: float, g_h: float) -> np.ndarray:
    t = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    lsm = torch.log_softmax(t, -1)
    p = lsm.exp()
    ent = -(p * torch.where(torch.isinf(lsm), torch.zeros_like(lsm), lsm)).sum()
    (g * lsm[y] + g_h * ent).backward()
    return t.grad.numpy()


def _rows(V: int, seed: int):
    r = np.random.default_rng(seed)
    yield 'random', r.normal(0.0, 3.0, V)
    one = r.normal(0.0, 0.5, V)
    one[r.integers(V)] += 40.0
    yield 'near one-hot', one
    yield 'uniform', np.full(V, 0.25)
    half = r.normal(0.0, 2.0, V)
    half[r.permutation(V)[: V // 2]] = -np.inf
    yield 'half -inf', half


@pytest.mark.parametrize('V', [7, 257, 4001])
@pytest.mark.parametrize('g,g_h', [(1.0, 0.0), (-0.3, 0.7), (0.0, -1.5), (2.0, 1e-3)])
def test_tile_formula_matches_float64_autograd(V, g, g_h):
    for name, x in _rows(V, V):
        y = int(np.argmax(np.where(np.isinf(x), -1e300, x))) if name == 'half -inf' else V // 3
        got = _tile(x, y, g, g_h)
        want = _autograd(x, y, g, g_h)
        assert np.all(np.isfinite(got)), name
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-13 * (1.0 + abs(g) + abs(g_h)), err_msg=name)
        if name == 'half -inf':
            assert np.all(got[np.isinf(x)] == 0.0)


def test_install_sets_and_uninstall_restores_entropy_coeff(fake_reference):  # noqa: F811
    from align_anything_b200 import patch

    try:
        patch.install(models=False)
        for modname, cls in fake_reference.items():
            assert cls.__dict__.get('entropy_coeff', 'missing') == 0.0, modname
    finally:
        patch.uninstall()
    for modname, cls in fake_reference.items():
        assert 'entropy_coeff' not in cls.__dict__, modname


def test_entropy_coeff_defaults_off_on_every_trainer():
    from align_anything_b200.trainers.text_audio_to_text.ppo import PPOTrainer as Audio
    from align_anything_b200.trainers.text_image_to_text.ppo import PPOTrainer as Image
    from align_anything_b200.trainers.text_to_text.grpo import GRPOTrainer
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer as Multi
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer
    from align_anything_b200.trainers.text_video_to_text.ppo import PPOTrainer as Video

    for cls in (PPOTrainer, Multi, Image, Audio, Video, GRPOTrainer):
        assert cls.entropy_coeff == 0.0, cls


def test_config_key_takes_precedence_over_the_attribute():
    from align_anything_b200.trainers.text_to_text.ppo import entropy_coeff_of

    tr = types.SimpleNamespace(entropy_coeff=0.25, cfgs=None)
    assert entropy_coeff_of(tr) == 0.25
    tr.cfgs = types.SimpleNamespace(train_cfgs=types.SimpleNamespace(entropy_coeff=None))
    assert entropy_coeff_of(tr) == 0.25  # None: not set in the recipe
    tr.cfgs.train_cfgs.entropy_coeff = 0.01
    assert entropy_coeff_of(tr) == 0.01
    tr.cfgs.train_cfgs.entropy_coeff = 0
    assert entropy_coeff_of(tr) == 0.0


def test_new_entry_points_check_arguments_before_cuda():
    from align_anything_b200 import _lib

    lib = _lib.lib()
    rc = lib.aa_logprob_bwd_entropy(None, 0, 0, 64, None, 0, 0, 1, 1, None, None, None, None, None, None, None, None, 0,
                                    None, None, 0, None, None, 2, None, 64, 0, None, 0, None, 0, None)
    assert rc == -2 and b'aa_logprob_bwd_entropy' in lib.aa_last_error()  # no entropy / grad_entropy / scratch
    buf = (ctypes.c_int64 * 8)()
    ptr = ctypes.cast(buf, ctypes.c_void_p)
    rc = lib.aa_logprob_bwd_entropy(ptr, 0, 64, 64, ptr, 0, 0, 1, 1, ptr, ptr, ptr, ptr, ptr, ptr, ptr, None, 2,
                                    None, None, 2, ptr, ptr, 9, ptr, 64, 0, None, 0, ptr, 0, None)
    assert rc == -1 and b'grad_entropy dtype' in lib.aa_last_error()  # AA_ERR_DTYPE
    rc = lib.aa_logprob_bwd_entropy(ptr, 0, 64, -1, ptr, 0, 0, 1, 1, ptr, ptr, ptr, ptr, ptr, ptr, ptr, None, 2,
                                    None, None, 2, ptr, ptr, 2, ptr, 64, 0, None, 0, ptr, 0, None)
    assert rc == -2 and b'bad sizes' in lib.aa_last_error()
    args = [ptr, 0, 64, 64, ptr, 1, ptr, ptr, ptr, ptr, ptr, 2, ptr, 0, None, None, ptr, 8, ptr, 8, 2, ptr, 8, 8,
            0.2, 0, ptr, 64, ptr, ptr]
    rc = lib.aa_logprob_actor_fused_entropy(*args, 0.1, None, None)
    assert rc == -2 and b'null entropy' in lib.aa_last_error()
    rc = lib.aa_logprob_actor_fused_entropy(*args, float('nan'), ptr, None)
    assert rc == -2 and b'NaN' in lib.aa_last_error()
    bad = list(args)
    bad[3] = 0  # V = 0
    rc = lib.aa_logprob_actor_fused_entropy(*bad, 0.1, ptr, None)
    assert rc == -2 and b'aa_logprob_actor_fused_entropy: bad sizes' in lib.aa_last_error()
    gargs = [ptr, 0, 64, 64, ptr, 1, ptr, ptr, ptr, ptr, ptr, 2, ptr, 0, ptr, 8, ptr, ptr, 8, 2, 8, 0.04, 0, ptr, 64,
             ptr, ptr, ptr, ptr, ptr]
    rc = lib.aa_logprob_grpo_fused_entropy_grad(*gargs, None, 0.1, None)
    assert rc == -2 and b'null entropy' in lib.aa_last_error()
    gargs[20] = 0  # K = 0
    rc = lib.aa_logprob_grpo_fused_entropy_grad(*gargs, ptr, 0.1, None)
    assert rc == -2 and b'aa_logprob_grpo_fused_entropy_grad: bad sizes' in lib.aa_last_error()
    largs = [ptr, 4, 64, 64, ptr, 100, 64, ptr, ptr, ptr, ptr, 2]
    rc = lib.aa_linear_dlogits_entropy(*largs, None, None, 2, ptr, 256, 0, None)
    assert rc == -2 and b'entropy and grad_entropy' in lib.aa_last_error()
    rc = lib.aa_linear_dlogits_entropy(*largs, ptr, ptr, 7, ptr, 256, 0, None)
    assert rc == -1 and b'grad_entropy dtype' in lib.aa_last_error()
    rc = lib.aa_linear_dlogits_entropy(*largs, ptr, ptr, 2, ptr, 64, 0, None)  # ld < ceil(V / 256) * 256
    assert rc == -3 and b'aa_linear_dlogits_entropy: ld' in lib.aa_last_error()
