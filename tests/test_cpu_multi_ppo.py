"""Multi-PPO without a GPU: the port of the reference's estimators against the goldens the reference produced (bit for
bit) and against an independent float64 statement, the argument errors of aa_ppo_returns / ops.estimator_returns, and
a dry run of the patched Multi-PPO train loop on a stand-in module tree (calls, graft list, metric dict)."""
import ctypes
import sys
import types

import numpy as np
import pytest
import torch

import fake_reference_tree as fake
import multi_ppo_port as P
from test_cpu_plumbing import _trainer, dry  # noqa: F401  (`dry` is a fixture)

MULTI = 'align_anything.trainers.text_to_text.multi_ppo'


# ---- the port against the reference's goldens --------------------------------------------------------------------
@pytest.mark.parametrize('dname', ['bf16', 'f32'])
def test_port_matches_reference_estimators(golden, dname):
    g = golden('multi_ppo')['estimators'][dname]
    mask, start = g['mask'], g['start']
    assert len(g['cases']) == 5 * 3 * 2
    for key, c in g['cases'].items():
        adv, ret = P.advantages_and_returns(g['values'], c['rewards'], mask, start, c['estimator'], c['n'], c['gamma'])
        assert torch.equal(adv, c['advantages']) and torch.equal(ret, c['returns']), key
        assert adv.dtype == c['advantages'].dtype and ret.dtype == c['returns'].dtype, key
        if c['estimator'] == 'gae':
            continue
        # rewards dtype, not promoted with the values dtype (unlike GAE); masked positions are exactly zero
        assert ret.dtype == c['rewards'].dtype, key
        assert not bool(ret[~mask[:, start:]].any()), key
        want = P.returns_f64(c['rewards'], mask, start, c['estimator'], c['n'], c['gamma'])
        tol = 1e-5 if dname == 'f32' else 6e-2
        assert np.allclose(ret.double().numpy(), want, rtol=tol, atol=tol), key


def test_group_quirk_and_constant_group(golden):
    """SURVEY H9: a group is n consecutive flat elements of the (B, W) token rewards, across row boundaries; a
    constant group normalises to 0 / 1e-9 = 0, not NaN."""
    g = golden('multi_ppo')['estimators']['f32']
    W = g['mask'].size(1)
    for n in (2, 3, 4):
        assert W % n != 0  # so that groups straddle rows
        c = g['cases'][f'group_norm_n{n}_g1.0']
        assert not bool(torch.isnan(c['returns']).any())
        g0 = (g['start'] + 1 + n - 1) // n * n
        assert bool((c['rewards'].view(-1)[g0:g0 + n] == 0.5).all())
    # the reference's rloo differs from a per-prompt leave-one-out on the same rewards
    c = g['cases']['rloo_n2_g1.0']
    m = g['mask']
    r = c['rewards'] * m
    per_prompt = r.view(-1, 2, W)
    loo = per_prompt - (per_prompt.sum(1, keepdim=True) - per_prompt) / 1
    ret_pp = P.cumulative_returns(loo.view_as(r), m, g['start'], 1.0) * m[:, g['start']:]
    assert not torch.equal(ret_pp, c['returns'])


@pytest.mark.parametrize('dname', ['bf16', 'f32'])
def test_port_matches_reference_rl_step(golden, dname):
    c = golden('multi_ppo')['rl_step'][dname]
    roll = {'log_probs': c['log_probs'], 'ref_log_probs': c['ref_log_probs'], 'reward': c['end_scores'].squeeze(-1),
            'reward_values': c['critic_scores'].squeeze(-1)[:, :-1]}
    for est in P.ESTIMATORS:
        w = c[est]
        leaf = c['new_actor_logits'].clone().requires_grad_(True)
        cleaf = c['new_critic_scores'].clone().requires_grad_(True)
        got = P.rl_step(roll, leaf, cleaf, c['input_ids'], c['attention_mask'], c['start'], est, c['n'])
        got['actor_loss'].backward()
        got['reward_critic_loss'].backward()
        for k in ('old_rewards', 'advantages', 'returns'):
            assert torch.equal(got['_' + k], w[k]), (est, k)
        assert torch.allclose(leaf.grad.float(), w['grad_actor_logits'].float(), rtol=1e-2, atol=1e-6), est
        assert torch.allclose(cleaf.grad, w['grad_critic_scores'], rtol=1e-5, atol=1e-8), est
        for k, v in w['metrics'].items():
            assert abs(float(got[k].detach()) - float(v)) <= 1e-3 * max(1.0, abs(float(v))), (est, k)


# ---- argument errors ---------------------------------------------------------------------------------------------
def test_returns_argument_errors_need_no_gpu():
    from align_anything_b200 import _lib

    lib = _lib.lib()
    buf = (ctypes.c_int64 * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def call(B=4, W=10, start=3, est=1, n=2, rew=p, adv=p, ret=None, rs=10, ms=10, dt=0):
        return lib.aa_ppo_returns(rew, dt, rs, p, ms, B, W, start, est, n, 1.0, 0, 1, adv, ret if ret is not None else
                                  ctypes.c_void_p(p.value + 8), dt, None, None)

    assert call(W=10, start=10) == -2 and b'bad sizes' in lib.aa_last_error()
    assert call(rew=None) == -2 and b'null or aliased' in lib.aa_last_error()
    assert call(ret=p) == -2 and b'null or aliased' in lib.aa_last_error()
    assert call(rs=9) == -2 and b'row strides' in lib.aa_last_error()
    assert call(est=4) == -2 and b'unknown estimator' in lib.aa_last_error()
    assert call(est=3, n=1) == -2 and b'n > 1' in lib.aa_last_error()
    assert call(B=3, W=5, start=1, rs=5, ms=5, est=2, n=2) == -2 and b'not a multiple' in lib.aa_last_error()
    assert call(dt=7) == -1 and b'bad dtype' in lib.aa_last_error()
    assert call(est=0, n=0) == -2  # reinforce takes n >= 1


def test_ops_raise_like_the_reference_before_any_launch():
    from align_anything_b200 import ops

    r = torch.zeros(3, 5)
    m = torch.ones(3, 5, dtype=torch.bool)
    with pytest.raises(ValueError, match='Unknown estimator: ppo'):
        ops.estimator_returns(r, m, 1, 'ppo', 2, 1.0)
    with pytest.raises(ValueError, match='requires n_samples_per_prompt > 1'):
        ops.estimator_returns(r, m, 1, 'group_norm', 1, 1.0)
    with pytest.raises(RuntimeError, match=r"shape '\[-1, 2\]' is invalid for input of size 15"):
        ops.estimator_returns(r, m, 1, 'rloo', 2, 1.0)
    with pytest.raises(RuntimeError, match='no CPU fallback'):  # reinforce needs no grouping: it reaches the launch
        ops.estimator_returns(r, m, 1, 'reinforce', 2, 1.0)


def test_trainer_init_reads_the_estimator():
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer

    cfgs = types.SimpleNamespace(train_cfgs=types.SimpleNamespace(advantage_estimator='rloo', n_samples_per_prompt=3))
    t = PPOTrainer(cfgs)
    assert (t.advantage_estimator, t.n_samples_per_prompt) == ('rloo', 3)
    cfgs.train_cfgs.n_samples_per_prompt = 1
    with pytest.raises(AssertionError, match='rloo requires n_samples_per_prompt > 1'):
        PPOTrainer(cfgs)
    cfgs.train_cfgs.advantage_estimator = 'reinforce'
    assert PPOTrainer(cfgs).n_samples_per_prompt == 1


# ---- the patched train loop --------------------------------------------------------------------------------------
class _MultiPPOTrainer(fake._TextPPOTrainer):
    """Shape of trainers/text_to_text/multi_ppo.py:PPOTrainer: the text trainer's methods plus cumulative_returns."""

    cumulative_returns = fake._not_grafted('cumulative_returns')


def _install_multi(mods):
    m = types.ModuleType(MULTI)
    m.PPOTrainer = type('PPOTrainer', (_MultiPPOTrainer,), {'__module__': MULTI})
    for fn in ('gather_log_probabilities', 'masked_mean'):
        setattr(m, fn, getattr(mods['align_anything.utils.tools'], fn))
    sys.modules[MULTI] = m
    mods['align_anything.trainers.text_to_text'].multi_ppo = m
    return m


@pytest.mark.parametrize('estimator', P.ESTIMATORS)
def test_patched_multi_ppo_train_loop_dry_run(dry, estimator):  # noqa: F811
    from align_anything_b200 import patch

    with fake.installed() as mods:
        saved = sys.modules.get(MULTI)
        m = _install_multi(mods)
        try:
            done = patch.install()
            try:
                t = _trainer(m.PPOTrainer)
                t.advantage_estimator, t.n_samples_per_prompt = estimator, 2
                inference, training = t.rollout(t.prompt_only_dataloader[0])
                t.train()
            finally:
                patch.uninstall()
        finally:
            if saved is None:
                sys.modules.pop(MULTI, None)
            else:
                sys.modules[MULTI] = saved
    want = {f'PPOTrainer.{n}' for n in ('rollout', 'get_advantages_and_returns', 'cumulative_returns', 'rl_step',
                                        'actor_loss_fn', 'critic_loss_fn', 'add_kl_divergence_regularization',
                                        'ptx_step')}
    assert want <= set(done[MULTI]), want - set(done[MULTI])
    assert 'PPOTrainer.actor_step' not in done[MULTI]  # generate + mask stay the reference's
    assert 'PPOTrainer.cumulative_returns' not in done['align_anything.trainers.text_to_text.ppo']
    # rollout: every prompt repeated n times (micro-batch of 2 prompts -> 4 samples), action_mask added
    assert [b['input_ids'].size(0) for b in inference] == [4, 4]
    assert torch.equal(inference[0]['input_ids'][0, :5], inference[0]['input_ids'][1, :5])
    assert all(torch.equal(tb['action_mask'], ib['attention_mask'][:, 1:].bool()) for ib, tb in zip(inference, training))
    assert t.global_step == 2 and t.actor_model.steps == t.reward_critic_model.steps == 2
    records = t.logger.writer.records  # the tensorboard-style writer asserts scalars only
    keys = {k for k, _, _ in records if not k.endswith('/step')}
    assert keys == {'train/actor_loss', 'train/reward_critic_loss', 'train/reward', 'train/reward_with_kl_penalty',
                    'train/reward_advantage', 'train/reward_return', 'train/reward_value', 'train/kl_divergence',
                    'train/actor_lr', 'train/reward_critic_lr', 'train/mean_generated_length',
                    'train/max_generated_length'}
    assert {'aa_ppo_prep', 'aa_logprob_actor_fused', 'aa_ppo_critic_loss', 'aa_ppo_pack_metrics'} <= set(dry.calls)
    assert 'aa_logprob_bwd' not in dry.calls
    assert ('aa_ppo_returns' in dry.calls) == (estimator != 'gae')
