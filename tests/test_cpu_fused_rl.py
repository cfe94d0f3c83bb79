"""The fused lm_head switch of the text RL trainers (text PPO, Multi-PPO, GRPO) without a GPU:
  * the graft: patch.install() puts `fused_lm_head = False` / `lm_head_chunk_rows = None` on the reference-shaped text
    PPO, Multi-PPO and GRPO classes, does not list them among the grafted methods, and uninstall() takes them away;
  * the refusals: with the switch on, every trainer raises ops.lm_head_weight's error for a ZeRO-3 placeholder weight,
    a biased head and a soft-capped / logit-scaled head before any model forward and before any kernel launch;
  * a dry run (the C ABI replaced by a signature-checking stand-in, see test_cpu_plumbing) of each fused step: the
    lm_head entry points are called, the logits-tile ones are not, and the gradient reaches the hidden states and the
    lm_head weight."""
import contextlib
import sys
import types
from types import SimpleNamespace

import pytest
import torch

import fake_reference_tree as fake
from test_cpu_plumbing import dry  # noqa: F401  (fixture)

_EXTRA = ('align_anything.trainers.text_to_text.multi_ppo', 'align_anything.trainers.text_to_text.grpo')


class _RefGRPOTrainer:
    """Shape of trainers/text_to_text/grpo.py:GRPOTrainer: the two methods the graft replaces."""

    _get_per_token_logps = fake._not_grafted('_get_per_token_logps')
    train_step = fake._not_grafted('train_step')


@contextlib.contextmanager
def _tree():
    """fake_reference_tree plus the Multi-PPO and GRPO modules."""
    saved = {n: sys.modules.get(n) for n in _EXTRA}
    with fake.installed() as mods:
        t2t = mods['align_anything.trainers.text_to_text']
        for n in _EXTRA:
            m = types.ModuleType(n)
            mods[n] = sys.modules[n] = m
            setattr(t2t, n.rpartition('.')[2], m)
        mods[_EXTRA[0]].PPOTrainer = type('PPOTrainer', (fake._TextPPOTrainer,), {'__module__': _EXTRA[0]})
        mods[_EXTRA[1]].GRPOTrainer = type('GRPOTrainer', (_RefGRPOTrainer,), {'__module__': _EXTRA[1]})
        try:
            yield mods
        finally:
            for n, old in saved.items():
                if old is None:
                    sys.modules.pop(n, None)
                else:
                    sys.modules[n] = old


def test_install_sets_and_uninstall_removes_the_switch():
    from align_anything_b200 import patch

    with _tree() as mods:
        classes = [mods['align_anything.trainers.text_to_text.ppo'].PPOTrainer, mods[_EXTRA[0]].PPOTrainer,
                   mods[_EXTRA[1]].GRPOTrainer]
        for cls in classes:
            assert not hasattr(cls, 'fused_lm_head') and not hasattr(cls, 'lm_head_chunk_rows')
        done = patch.install()
        try:
            for cls in classes:
                assert cls.__dict__['fused_lm_head'] is False and cls.__dict__['lm_head_chunk_rows'] is None, cls
            listed = [x for names in done.values() for x in names]
            assert not any('fused_lm_head' in x or 'lm_head_chunk_rows' in x for x in listed), listed
            assert 'GRPOTrainer._get_per_token_logps' in done[_EXTRA[1]]
        finally:
            patch.uninstall()
        for cls in classes:
            assert not hasattr(cls, 'fused_lm_head') and not hasattr(cls, 'lm_head_chunk_rows'), cls
            assert 'rl_step' not in cls.__dict__ or cls.__dict__['rl_step'].__name__ == 'rl_step'


# ---- refusals before anything runs -------------------------------------------------------------------------------------
class _NoKernels:
    def __getattr__(self, name):
        raise AssertionError(f'kernel entry point {name} reached')


class _Head(torch.nn.Module):
    def __init__(self, kind):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.randn(11, 8))
        self.bias = torch.nn.Parameter(torch.zeros(11)) if kind == 'bias' else None
        if kind == 'zero3':
            self.weight.ds_id = 7  # what DeepSpeed ZeRO-3 puts on a partitioned parameter


class _RefusedModel:
    """An engine whose forward must never run; its module has one of the heads lm_head_weight refuses."""

    def __init__(self, kind):
        self.module = SimpleNamespace(get_output_embeddings=lambda: _Head(kind),
                                      config=SimpleNamespace(final_logit_softcapping=30.0 if kind == 'softcap' else None,
                                                             logit_scale=0.25 if kind == 'scale' else None))

    def __call__(self, *a, **k):
        raise AssertionError('model forward reached')


_REFUSALS = {'zero3': 'ZeRO-3', 'bias': 'bias-free', 'softcap': 'final_logit_softcapping', 'scale': 'logit_scale'}


@pytest.fixture
def no_kernels(monkeypatch):
    from align_anything_b200 import _lib

    monkeypatch.setattr(_lib, 'lib', lambda: _NoKernels())
    monkeypatch.setattr(_lib, 'require_cuda', lambda *t: None)


def _rl_batches(B=2, Lq=6):
    ids = torch.randint(3, 11, (B, Lq))
    w = Lq - 1
    inference = {'input_ids': ids, 'attention_mask': torch.ones(B, Lq, dtype=torch.bool)}
    training = {'prompt_idx': 2, 'log_probs': torch.zeros(B, w), 'ref_log_probs': torch.zeros(B, w),
                'reward': torch.zeros(B), 'reward_values': torch.zeros(B, w)}
    return inference, training


@pytest.mark.parametrize('kind', list(_REFUSALS))
@pytest.mark.parametrize('step', ['ppo_rollout', 'ppo_rl_step', 'multi_ppo_gae', 'multi_ppo_rloo', 'grpo'])
def test_refusals_come_before_any_forward_or_kernel(no_kernels, step, kind):
    from align_anything_b200.trainers.text_to_text.grpo import GRPOTrainer
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer as MultiPPO
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer

    bad = _RefusedModel(kind)
    never = _RefusedModel('none')
    if step == 'grpo':
        tr = GRPOTrainer(None, bad, never, SimpleNamespace(pad_token_id=0, eos_token_id=2), beta=0.04, num_generations=2)
        tr.fused_lm_head = True
        run = lambda: tr.step_from_rollout(torch.randint(3, 11, (4, 7)), 3, torch.zeros(4))
    else:
        if step.startswith('multi_ppo'):
            tr = MultiPPO(None, bad, never, never, never, SimpleNamespace(pad_token_id=0),
                          advantage_estimator=step.rpartition('_')[2], n_samples_per_prompt=2)
        else:
            tr = PPOTrainer(None, bad, never, never, never, SimpleNamespace(pad_token_id=0))
        tr.fused_lm_head = True
        inference, training = _rl_batches()
        run = (lambda: tr.score_rollout(inference, 3)) if step == 'ppo_rollout' else (lambda: tr.rl_step(inference, training))
    with pytest.raises(RuntimeError, match=_REFUSALS[kind]):
        run()
    if step in ('ppo_rollout', 'grpo'):  # the reference model's head is checked too
        tr.actor_model, tr.actor_reference_model = never, bad
        with pytest.raises(RuntimeError, match=_REFUSALS[kind]):
            run()


# ---- dry run of the fused steps ----------------------------------------------------------------------------------------
class _HiddenLM:
    """A causal-LM-shaped module that hands out fixed last hidden states; its forward must be asked for them."""

    def __init__(self, hidden, weight):
        self.hidden, self.weight = hidden, weight
        self.module = self
        self.calls = []
        self.optimizer = SimpleNamespace(param_groups=[{'lr': 1e-6}])

    def __call__(self, output_hidden_states=False, logits_to_keep=0, **kw):
        assert output_hidden_states and logits_to_keep == 1, 'the fused path must not ask for a logits tile'
        self.calls.append(sorted(kw))
        return SimpleNamespace(hidden_states=(None, self.hidden), logits=None)

    def get_output_embeddings(self):
        return SimpleNamespace(weight=self.weight)

    def backward(self, loss):
        loss.backward()

    def step(self):
        pass

    def zero_grad(self):
        pass


class _Scores:
    def __init__(self, make):
        self.make = make
        self.optimizer = SimpleNamespace(param_groups=[{'lr': 1e-6}])

    def __call__(self, **kw):
        return self.make()

    def backward(self, loss):
        loss.backward()

    def step(self):
        pass


_TILE_ENTRIES = {'aa_logprob_fwd', 'aa_logprob_bwd', 'aa_logprob_actor_fused', 'aa_logprob_grpo_fused'}
_LM_HEAD_ENTRIES = {'aa_linear_logprob_fwd', 'aa_linear_dlogits', 'aa_linear_dhidden', 'aa_linear_dweight'}


@pytest.mark.parametrize('trainer', ['ppo', 'multi_ppo_gae', 'multi_ppo_reinforce', 'multi_ppo_group_norm'])
def test_fused_ppo_dry_run(dry, trainer):
    from align_anything_b200.models.reward_model import ScoreModelOutput
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer as MultiPPO
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer

    B, Lq, H, V = 4, 9, 64, 97
    ids = torch.randint(3, V, (B, Lq))
    hid = torch.randn(B, Lq, H).bfloat16().requires_grad_(True)
    w = torch.randn(V, H).bfloat16().requires_grad_(True)
    actor, ref = _HiddenLM(hid, w), _HiddenLM(hid.detach(), w.detach())
    critic = torch.randn(B, Lq, 1).requires_grad_(True)
    reward_model = _Scores(lambda: ScoreModelOutput(end_scores=torch.randn(B, 1)))
    critic_model = _Scores(lambda: ScoreModelOutput(scores=critic))
    if trainer == 'ppo':
        tr = PPOTrainer(None, actor, ref, reward_model, critic_model, SimpleNamespace(pad_token_id=0))
    else:
        tr = MultiPPO(None, actor, ref, reward_model, critic_model, SimpleNamespace(pad_token_id=0),
                      advantage_estimator=trainer.partition('ppo_')[2], n_samples_per_prompt=2)
    tr.fused_lm_head = True
    inference, training = tr.score_rollout({'input_ids': ids, 'attention_mask': ids != 0}, 4)
    assert training['log_probs'].shape == training['ref_log_probs'].shape == (B, Lq - 1)
    assert training['log_probs'].dtype == torch.bfloat16
    dry.calls.clear()
    out = tr.rl_step(inference, training)
    assert all(isinstance(v, float) for v in out.values())
    assert _LM_HEAD_ENTRIES <= set(dry.calls) and not (_TILE_ENTRIES & set(dry.calls)), dry.calls
    assert 'aa_ppo_actor_loss' in dry.calls and dry.calls.count('aa_ppo_pack_metrics') == 1
    assert actor.calls[-1] == ['attention_mask', 'input_ids', 'use_cache']
    assert hid.grad is not None and hid.grad.shape == hid.shape and w.grad is not None and w.grad.shape == w.shape


def test_fused_grpo_dry_run(dry):
    from align_anything_b200.trainers.text_to_text.grpo import GRPOTrainer

    B, Lq, H, V, P = 4, 10, 64, 97, 4
    seq = torch.randint(3, V, (B, Lq))
    hid = torch.randn(B, Lq, H).bfloat16().requires_grad_(True)
    w = torch.randn(V, H).bfloat16().requires_grad_(True)
    actor, ref = _HiddenLM(hid, w), _HiddenLM(hid.detach(), w.detach())
    tr = GRPOTrainer(None, actor, ref, SimpleNamespace(pad_token_id=0, eos_token_id=2), beta=0.04, num_generations=2)
    tr.fused_lm_head = True
    out = tr.step_from_rollout(seq, P, torch.randn(B))
    assert set(out) == {'train/loss', 'train/reward'} and all(isinstance(v, float) for v in out.values())
    assert {'aa_group_advantages', 'aa_grpo_loss'} | _LM_HEAD_ENTRIES <= set(dry.calls)
    assert not (_TILE_ENTRIES & set(dry.calls)), dry.calls
    assert hid.grad is not None and w.grad is not None
