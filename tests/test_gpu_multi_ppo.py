"""Multi-PPO on the H100 (`pytest -m gpu`): K4r (ops.estimator_returns) and the grafted rl_step against
  * STRICT: the reference's estimator code (tests/multi_ppo_port.py) executed with torch's CUDA kernels on the same
    device tensors -- faithful mode: every element within 1 ulp and >= 97 % bit-identical, masked positions exactly
    zero; 'f32' mode: within 2e-5 relative of the port on fp32-upcast rewards;
  * GOLDEN: the fixtures the unmodified reference produced on CPU (tests/golden/make_golden_multi_ppo.py).
With 'gae' the Multi-PPO step must be bit-identical to the text PPO step on the same inputs."""
from types import SimpleNamespace

import pytest
import torch

import multi_ppo_port as P
from test_gpu_parity import _cuda, assert_close_f32, assert_loose, assert_ulp_close, ops  # noqa: F401

pytestmark = pytest.mark.gpu

DEV = 'cuda'
GROUP = ('reinforce', 'rloo', 'reinforce_baseline', 'group_norm')


def _rollout_like(B, W, dtype, gen):
    """K4-style token rewards (small KL terms, the sequence reward at the last attended position) and a mask with left
    pads inside the prompt, right pads after the response and a few holes."""
    start = W // 4
    mask = torch.zeros(B, W, dtype=torch.bool)
    for b in range(B):
        left = int(torch.randint(0, max(1, start // 2), (1,), generator=gen))
        resp = int(torch.randint(1, W - start + 1, (1,), generator=gen))
        mask[b, left:start + resp] = True
    holes = torch.rand(B, W, generator=gen) < 0.02
    mask &= ~holes
    mask[:, start] = True  # no empty row
    r = 0.02 * torch.randn(B, W, generator=gen)
    end = W - 1 - mask.flip(-1).int().argmax(-1)
    r[torch.arange(B), end] += torch.randn(B, generator=gen)
    return r.to(dtype), mask, start


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize('n', [2, 3, 4, 8])
@pytest.mark.parametrize('W', [37, 1000, 4097])
def test_estimators_vs_eager_cuda(ops, W, n, dtype):
    gen = torch.Generator().manual_seed(W * 31 + n)
    B = 24 if n == 3 else 32
    r, mask, start = _rollout_like(B, W, dtype, gen)
    r, mask = r.to(DEV), mask.to(DEV)
    gamma = 1.0 if n % 2 == 0 else 0.99
    off = ~mask[:, start:]
    for est in GROUP:
        adv, ret = ops.estimator_returns(r, mask, start, est, n, gamma)
        w_adv, w_ret = P.advantages_and_returns(torch.zeros_like(r), r, mask, start, est, n, gamma)
        assert adv.dtype == ret.dtype == dtype
        assert_ulp_close(adv, w_adv, max_ulp=1, min_exact=0.97, what=f'{est} adv')
        assert_ulp_close(ret, w_ret, max_ulp=1, min_exact=0.97, what=f'{est} ret')
        # masks and zeros are exact; fp16 group_norm: 1e-9 rounds to 0 in fp16, so a constant group is 0 / 0 = NaN and
        # the reference's returns carry it (the NaN pattern is compared above)
        assert not bool((ret[off].nan_to_num() != 0).any()) and not bool((adv[off].nan_to_num() != 0).any()), est
        if not (dtype == torch.float16 and est == 'group_norm'):
            assert not bool(torch.isnan(ret).any()), est
        if dtype != torch.float32:
            adv32, ret32 = ops.estimator_returns(r, mask, start, est, n, gamma, mode='f32')
            _, w32 = P.advantages_and_returns(torch.zeros_like(r, dtype=torch.float32), r.float(), mask, start, est, n, gamma)
            assert ret32.dtype == torch.float32
            assert_close_f32(ret32, w32, what=f'{est} f32 mode')
            assert torch.equal(adv32, ret32)


def test_cumulative_returns_and_row_stats(ops):
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer

    gen = torch.Generator().manual_seed(5)
    r, mask, start = _rollout_like(8, 300, torch.bfloat16, gen)
    r, mask = r.to(DEV), mask.to(DEV)
    tr = PPOTrainer(None, advantage_estimator='reinforce', n_samples_per_prompt=1)
    tr.gamma = 0.99
    assert_ulp_close(tr.cumulative_returns(r, mask, start), P.cumulative_returns(r, mask, start, 0.99),
                     min_exact=0.97, what='cumulative_returns (not masked afterwards)')
    assert_ulp_close(tr.cumulative_returns(r, None, start), P.cumulative_returns(r, None, start, 0.99),
                     min_exact=0.97, what='cumulative_returns without a mask')
    rs = torch.full((8, 8), 7.0, device=DEV)
    adv, ret = ops.estimator_returns(r, mask, start, 'group_norm', 4, 1.0, row_stats=rs)
    m = mask[:, start:]
    want = (ret.float() * m).sum(-1) / m.sum(-1)
    assert torch.allclose(rs[:, 3], want, rtol=1e-5, atol=1e-6) and torch.equal(rs[:, 3], rs[:, 4])
    assert bool((rs[:, [0, 1, 2, 5, 6, 7]] == 7.0).all())  # the other lanes are K4's and stay untouched


@pytest.mark.parametrize('dname', ['bf16', 'f32'])
def test_estimators_golden(ops, golden, dname):
    g = {k: _cuda(v) for k, v in golden('multi_ppo')['estimators'][dname].items() if k != 'cases'}
    cases = golden('multi_ppo')['estimators'][dname]['cases']
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer

    for key, c in cases.items():
        tr = PPOTrainer(None, advantage_estimator=c['estimator'], n_samples_per_prompt=c['n'], gamma=c['gamma'])
        adv, ret = tr.get_advantages_and_returns(g['values'], c['rewards'].to(DEV), g['mask'], g['start'])
        assert_loose(adv, c['advantages'], what=f'{key} adv golden')
        assert_loose(ret, c['returns'], what=f'{key} ret golden')
        w_adv, w_ret = P.advantages_and_returns(g['values'], c['rewards'].to(DEV), g['mask'], g['start'], c['estimator'],
                                                c['n'], c['gamma'])
        assert_ulp_close(adv, w_adv, min_exact=0.97, what=f'{key} adv vs eager CUDA')
        assert_ulp_close(ret, w_ret, min_exact=0.97, what=f'{key} ret vs eager CUDA')
        if c['estimator'] != 'gae':  # K4 -> K4r from the log-probs, as rl_step runs it
            rew, _, _, _ = ops.kl_rewards_and_gae(g['reward'], g['log_probs'], g['ref_log_probs'], g['values'], g['mask'],
                                                  g['start'], 0.02, 50.0, c['gamma'], 0.95)
            if c['estimator'] == 'group_norm':
                n = c['n']
                g0 = (g['start'] + 1 + n - 1) // n * n
                rew.view(-1)[g0:g0 + n] = 0.5
            assert_loose(rew, c['rewards'], what=f'{key} K4 rewards golden')


class _Engine:
    def __init__(self, fn):
        self.fn = fn
        self.optimizer = SimpleNamespace(param_groups=[{'lr': 2e-6}])

    def __call__(self, **kw):
        return self.fn()

    def backward(self, loss):
        loss.backward()

    def step(self):
        pass


def _run_step(cls, c, est=None):
    from align_anything_b200.models.reward_model import ScoreModelOutput

    new_actor = c['new_actor_logits'].clone().requires_grad_(True)
    new_critic = c['new_critic_scores'].clone().requires_grad_(True)
    state = {'phase': 'rollout'}
    actor = _Engine(lambda: SimpleNamespace(logits=c['actor_logits'] if state['phase'] == 'rollout' else new_actor))
    ref = _Engine(lambda: SimpleNamespace(logits=c['ref_logits']))
    rm = _Engine(lambda: ScoreModelOutput(end_scores=c['end_scores']))
    critic = _Engine(lambda: ScoreModelOutput(scores=c['critic_scores'] if state['phase'] == 'rollout' else new_critic))
    kw = {} if est is None else {'advantage_estimator': est, 'n_samples_per_prompt': c['n']}
    tr = cls(None, actor, ref, rm, critic, SimpleNamespace(pad_token_id=0), **kw)
    inference, training = tr.score_rollout({'input_ids': c['input_ids'], 'attention_mask': c['attention_mask']},
                                           prompt_len=c['start'] + 1)
    state['phase'] = 'train'
    out = tr.rl_step(inference, training)
    return tr, out, new_actor.grad, new_critic.grad


@pytest.mark.parametrize('dname', ['bf16', 'f32'])
def test_rl_step_golden(ops, golden, dname):
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer

    c = {k: _cuda(v) if not isinstance(v, dict) else v for k, v in golden('multi_ppo')['rl_step'][dname].items()}
    roll_ref = P.O.ppo_text_rollout_scoring(c['actor_logits'], c['ref_logits'], c['input_ids'], c['end_scores'],
                                            c['critic_scores'])
    for est in P.ESTIMATORS:
        w = {k: _cuda(v) if torch.is_tensor(v) else v for k, v in c[est].items()}
        tr, out, g_actor, g_critic = _run_step(PPOTrainer, c, est)
        leaf = c['new_actor_logits'].clone().requires_grad_(True)
        cleaf = c['new_critic_scores'].clone().requires_grad_(True)
        want = P.rl_step(roll_ref, leaf, cleaf, c['input_ids'], c['attention_mask'], c['start'], est, c['n'])
        want['actor_loss'].backward()
        want['reward_critic_loss'].backward()
        for k in ('old_rewards', 'advantages', 'returns'):
            assert_ulp_close(tr.last_rl_tensors[k], want['_' + k], what=f'{est} {k} vs eager CUDA')
        assert_ulp_close(g_actor, leaf.grad, min_exact=0.97, what=f'{est} actor logits grad')
        assert_ulp_close(g_critic, cleaf.grad, min_exact=0.9, what=f'{est} critic scores grad')
        for k in w['metrics']:
            got, v = out['train/' + k], float(want[k].detach())
            assert abs(got - v) <= 8e-3 * max(1.0, abs(v)), (est, k, got, v)
        # the CPU golden's 16-bit log-probs differ from the CUDA kernels' (module docstring of test_gpu_parity.py) and
        # the KL-shaped rewards inherit that, so the golden step is held strictly in fp32, like the text PPO step
        if dname == 'f32':
            for k in ('old_rewards', 'advantages', 'returns'):
                assert_close_f32(tr.last_rl_tensors[k], w[k], what=f'{est} {k} golden')
            assert_close_f32(g_actor, w['grad_actor_logits'], what=f'{est} actor grad golden')
            assert_close_f32(g_critic, w['grad_critic_scores'], what=f'{est} critic grad golden')
            for k, v in w['metrics'].items():
                assert abs(out['train/' + k] - float(v)) <= 1e-4 * max(1.0, abs(float(v))), (est, k)
        assert all(isinstance(v, float) for v in out.values())


@pytest.mark.parametrize('dname', ['bf16', 'f32'])
def test_gae_step_is_the_text_ppo_step(ops, golden, dname):
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer as Multi
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer as Text

    c = {k: _cuda(v) if not isinstance(v, dict) else v for k, v in golden('multi_ppo')['rl_step'][dname].items()}
    tm, om, gam, gcm = _run_step(Multi, c, 'gae')
    tt, ot, gat, gct = _run_step(Text, c)
    assert om == ot
    for k in ('old_rewards', 'advantages', 'returns'):
        assert torch.equal(tm.last_rl_tensors[k], tt.last_rl_tensors[k]), k
    assert torch.equal(gam, gat) and torch.equal(gcm, gct)
