"""The PPO and GRPO steps over their switches, without a GPU (the C ABI replaced by the signature-checking stand-in of
test_cpu_plumbing).  For the text, Multi-PPO ('gae' and 'rloo'), image and audio PPO trainers, each run standalone and
grafted onto the reference-shaped classes, and for every combination of `fused_lm_head`, `log_entropy`,
`entropy_coeff`, the actor objective and `log_clip_fraction`, rollout + rl_step returns exactly the metric keys the
switches call for and hands ONE packed vector to the collective: ppo_pack_metrics' 12 lanes (the entropy in the spare
lane 11), then the entropy bonus, then the clip fraction(s), with lanes 9 and 10 MAX-reduced.  GRPO's step_from_rollout
is pinned the same way over `log_entropy`, the bonus, the clip fractions and dual-clip."""
import contextlib
import importlib
import sys
import types
from types import SimpleNamespace

import pytest
import torch

import fake_reference_tree as fake
from test_cpu_plumbing import dry  # noqa: F401  (fixture)

MULTI = 'align_anything.trainers.text_to_text.multi_ppo'
GRPO = 'align_anything.trainers.text_to_text.grpo'
_PPO_MODULES = {'text': 'align_anything.trainers.text_to_text.ppo', 'multi_gae': MULTI, 'multi_rloo': MULTI,
                'image': 'align_anything.trainers.text_image_to_text.ppo',
                'audio': 'align_anything.trainers.text_audio_to_text.ppo'}
_OBJECTIVE = {'clip_range_ratio_low': 0.2, 'clip_range_ratio_high': 0.28, 'dual_clip_ratio': 3.0,
              'loss_agg_mode': 'token-mean'}
_PPO_KEYS = {'train/actor_loss', 'train/reward_critic_loss', 'train/reward', 'train/reward_with_kl_penalty',
             'train/reward_advantage', 'train/reward_return', 'train/reward_value', 'train/kl_divergence',
             'train/mean_generated_length', 'train/max_generated_length', 'train/actor_lr', 'train/reward_critic_lr'}


class _LM(fake.TinyLM):
    """TinyLM that also hands out its last hidden states (`output_hidden_states=True`) and its lm_head."""

    def forward(self, input_ids=None, attention_mask=None, use_cache=None, logits_to_keep=0, output_hidden_states=False,
                **kw):
        if output_hidden_states:
            return SimpleNamespace(logits=None, hidden_states=(self.emb[input_ids],))
        return super().forward(input_ids, attention_mask, use_cache, logits_to_keep, **kw)

    def get_output_embeddings(self):
        return SimpleNamespace(weight=self.head)


class _Engine(fake.Engine):
    def zero_grad(self):
        self.optimizer.zero_grad(set_to_none=True)


class _RefGRPOTrainer:
    """Shape of trainers/text_to_text/grpo.py:GRPOTrainer: the two methods the graft replaces."""

    _get_per_token_logps = fake._not_grafted('_get_per_token_logps')
    train_step = fake._not_grafted('train_step')


class _RefMultiPPOTrainer(fake._TextPPOTrainer):
    cumulative_returns = fake._not_grafted('cumulative_returns')


@contextlib.contextmanager
def _grafted():
    """fake_reference_tree plus the Multi-PPO and GRPO modules, with patch.install() in effect."""
    from align_anything_b200 import patch

    saved = {n: sys.modules.get(n) for n in (MULTI, GRPO)}
    with fake.installed() as mods:
        for n, cls, name in ((MULTI, _RefMultiPPOTrainer, 'PPOTrainer'), (GRPO, _RefGRPOTrainer, 'GRPOTrainer')):
            m = mods[n] = sys.modules[n] = types.ModuleType(n)
            setattr(m, name, type(name, (cls,), {'__module__': n}))
            setattr(mods['align_anything.trainers.text_to_text'], n.rpartition('.')[2], m)
        patch.install()
        try:
            yield mods
        finally:
            patch.uninstall()
            for n, old in saved.items():
                if old is None:
                    sys.modules.pop(n, None)
                else:
                    sys.modules[n] = old


@pytest.fixture
def packed(monkeypatch):
    """Every vector the trainer modules hand to all_reduce_packed: (length, max_lanes)."""
    calls = []

    def record(stats, max_lanes=(), group=None):
        calls.append((stats.numel(), tuple(max_lanes)))
        return stats

    for name in ('text_to_text.ppo', 'text_to_text.multi_ppo', 'text_image_to_text.ppo', 'text_to_text.grpo'):
        mod = importlib.import_module(f'align_anything_b200.trainers.{name}')
        monkeypatch.setattr(mod, 'all_reduce_packed', record, raising=False)
    return calls


@pytest.fixture
def full_lens(monkeypatch):
    """The stand-in library leaves the multimodal response lengths at 0, which the fused lm_head path refuses: every
    response takes the whole generated width instead."""
    from align_anything_b200 import ops

    layout = ops.rollout_layout

    def full(prompt_ids, sequences, pad_id):
        moved, mask, lens = layout(prompt_ids, sequences, pad_id)
        lens.dev.fill_(lens.bound)
        return moved, mask, lens

    monkeypatch.setattr(ops, 'rollout_layout', full)


def _standalone_class(trainer):
    from align_anything_b200.trainers.text_audio_to_text.ppo import PPOTrainer as Audio
    from align_anything_b200.trainers.text_image_to_text.ppo import PPOTrainer as Image
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer as Multi
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer as Text

    return {'text': Text, 'multi_gae': Multi, 'multi_rloo': Multi, 'image': Image, 'audio': Audio}[trainer]


def _ppo_trainer(cls, trainer):
    t = object.__new__(cls)
    t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(per_device_train_batch_size=2, update_iters=1))
    t.tokenizer = t.reward_tokenizer = SimpleNamespace(pad_token_id=0, eos_token_id=2)
    t.generation_config = None
    t.infer_batch = t.reward_infer_batch = lambda batch: {k: v for k, v in batch.items() if k != 'meta_info'}
    t.actor_model = _Engine(_LM(97, 64, 0, 2, 6, seed=1).bfloat16())
    t.actor_reference_model = _Engine(_LM(97, 64, 0, 2, 6, seed=2).bfloat16())
    t.reward_model = _Engine(fake.TinyScoreModel(97, 16, seed=3).bfloat16())
    t.reward_critic_model = _Engine(fake.TinyScoreModel(97, 16, seed=4).bfloat16())
    t.kl_coeff, t.clip_range_ratio, t.clip_range_score, t.clip_range_value = 0.02, 0.2, 50.0, 5.0
    t.gamma, t.gae_lambda, t.ptx_coeff = 1.0, 0.95, 16.0
    t.train_mode_calls = []
    if trainer.startswith('multi'):
        t.advantage_estimator, t.n_samples_per_prompt = trainer.partition('_')[2], 2
    return t


def _prompts():
    ids = torch.randint(3, 97, (4, 5), generator=torch.Generator().manual_seed(0))
    ids[1, :2] = 0
    return {'input_ids': ids, 'attention_mask': ids != 0}


def _ppo_expect(log_entropy, coeff, objective, log_cf):
    keys, n = set(_PPO_KEYS), 12
    if log_entropy:
        keys.add('train/entropy')
    if coeff:
        keys.add('train/actor_entropy')
        n += 1
    if log_cf:
        keys.add('train/actor_clip_fraction')
        n += 1
        if objective:
            keys.add('train/actor_dual_clip_fraction')
            n += 1
    return keys, n


@pytest.mark.parametrize('log_cf', [False, True])
@pytest.mark.parametrize('objective', [False, True])
@pytest.mark.parametrize('coeff', [0.0, 0.01])
@pytest.mark.parametrize('log_entropy', [False, True])
@pytest.mark.parametrize('fused', [False, True])
@pytest.mark.parametrize('grafted', [False, True])
@pytest.mark.parametrize('trainer', list(_PPO_MODULES))
def test_ppo_rl_step_metrics_and_packed_lanes(dry, packed, full_lens, trainer, grafted, fused, log_entropy,  # noqa: F811
                                             coeff, objective, log_cf):
    with contextlib.ExitStack() as stack:
        if grafted:
            mods = stack.enter_context(_grafted())
            cls = mods[_PPO_MODULES[trainer]].PPOTrainer
        else:
            cls = _standalone_class(trainer)
        t = _ppo_trainer(cls, trainer)
        t.fused_lm_head, t.log_entropy, t.entropy_coeff, t.log_clip_fraction = fused, log_entropy, coeff, log_cf
        for k, v in (_OBJECTIVE if objective else {}).items():
            setattr(t, k, v)
        inference, training = t.rollout(_prompts())
        assert packed == []
        out = t.rl_step(inference[0], training[0])
    keys, n = _ppo_expect(log_entropy, coeff, objective, log_cf)
    assert set(out) == keys
    assert all(isinstance(v, float) for v in out.values())
    assert packed == [(n, (9, 10))]
    assert set(t.last_rl_tensors) == {'old_rewards', 'advantages', 'returns'}
    assert dry.calls.count('aa_ppo_pack_metrics') == 1
    assert ('aa_ppo_returns' in dry.calls) == (trainer == 'multi_rloo')


@pytest.mark.parametrize('dual', [False, True])
@pytest.mark.parametrize('log_cf', [False, True])
@pytest.mark.parametrize('coeff', [0.0, 0.01])
@pytest.mark.parametrize('log_entropy', [False, True])
@pytest.mark.parametrize('fused', [False, True])
@pytest.mark.parametrize('grafted', [False, True])
def test_grpo_step_metrics_and_packed_lanes(dry, packed, grafted, fused, log_entropy, coeff, log_cf, dual):  # noqa: F811
    from align_anything_b200.trainers.text_to_text.grpo import GRPOTrainer

    with contextlib.ExitStack() as stack:
        cls = stack.enter_context(_grafted())[GRPO].GRPOTrainer if grafted else GRPOTrainer
        t = object.__new__(cls)
        t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(update_iters=1))
        t.actor_model = _Engine(_LM(97, 64, 0, 2, 6, seed=1).bfloat16())
        t.actor_reference_model = _Engine(_LM(97, 64, 0, 2, 6, seed=2).bfloat16())
        t.tokenizer = SimpleNamespace(pad_token_id=0, eos_token_id=2)
        t.beta, t.num_generations = 0.04, 2
        t.fused_lm_head, t.log_entropy, t.entropy_coeff, t.log_clip_fraction = fused, log_entropy, coeff, log_cf
        if dual:
            t.dual_clip_ratio = 3.0
        gen = torch.Generator().manual_seed(0)
        out = t.step_from_rollout(torch.randint(3, 97, (4, 9), generator=gen), 4, torch.randn(4, generator=gen))
    keys, n = {'train/loss', 'train/reward'}, 3
    for on, key in ((log_entropy, 'train/entropy'), (coeff, 'train/actor_entropy'),
                    (log_cf, 'train/actor_clip_fraction'), (log_cf and dual, 'train/actor_dual_clip_fraction')):
        if on:
            keys.add(key)
            n += 1
    assert set(out) == keys
    assert all(isinstance(v, float) for v in out.values())
    assert packed == [(n, (2,))]
