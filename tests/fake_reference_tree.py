"""TEST INFRASTRUCTURE ONLY -- a stand-in `align_anything` module tree, so that the graft can be tested without the
reference's sources.  It has the reference's module paths, class names and method names for the PPO recipes, with

  * the methods `align_anything_b200.patch.install()` is expected to REPLACE written as `raise AssertionError` bodies
    (so a test that runs the loop proves the graft took), and
  * the methods the graft is expected to LEAVE ALONE restated minimally from the reference: the `train()` loop
    (trainers/text_to_text/ppo.py:410-460: rollout -> rl_step -> Logger.log per micro-batch), `reward_model_step`
    (:224-242), the text trainer's `actor_step` (:209-222), `set_train` (trainers/base/rl_trainer.py:274-286) and
    `Logger.log` (utils/logger.py:129-138) with a tensorboard-style writer whose `add_scalar` accepts scalars only.

Nothing here is product code, and nothing here computes a loss."""
from __future__ import annotations

import contextlib
import copy
import sys
import types

import torch

_NAMES = [
    'align_anything', 'align_anything.utils', 'align_anything.utils.tools', 'align_anything.trainers',
    'align_anything.trainers.text_to_text', 'align_anything.trainers.text_to_text.ppo',
    'align_anything.trainers.text_image_to_text', 'align_anything.trainers.text_image_to_text.ppo',
    'align_anything.trainers.text_audio_to_text', 'align_anything.trainers.text_audio_to_text.ppo',
]


def _not_grafted(name):
    def fn(*a, **k):
        raise AssertionError(f'{name} was not replaced by align_anything_b200.patch.install()')

    fn.__name__ = name
    return fn


class ScalarOnlyWriter:
    """torch.utils.tensorboard.SummaryWriter.add_scalar asserts 'scalar should be 0D'; wandb would histogram tensors."""

    def __init__(self):
        self.records = []

    def add_scalar(self, key, value, global_step=None):
        assert isinstance(value, (int, float)) and not isinstance(value, bool), (key, type(value))
        self.records.append((key, float(value), global_step))


class Logger:
    """utils/logger.py:129-138, log_type == 'tensorboard'."""

    def __init__(self):
        self.writer = ScalarOnlyWriter()

    def log(self, metrics, step):
        tags = {key.rpartition('/')[0] for key in metrics}
        metrics = {**{f'{tag}/step': step for tag in tags}, **metrics}
        for key, value in metrics.items():
            self.writer.add_scalar(key, value, global_step=step)

    def print(self, *a, **k):
        pass


class _TextPPOTrainer:
    """Shape of trainers/text_to_text/ppo.py:PPOTrainer."""

    def actor_step(self, mini_prompt_only_batch):  # :209-222 -- NOT replaced for the text trainer
        infer_batch = self.infer_batch(mini_prompt_only_batch)
        actor_batch = copy.deepcopy(infer_batch)
        sequences = self.actor_model.module.generate(**infer_batch, generation_config=self.generation_config,
                                                     synced_gpus=True, do_sample=True)
        actor_batch['input_ids'] = sequences
        actor_batch['attention_mask'] = sequences.not_equal(self.tokenizer.pad_token_id)
        return actor_batch

    def reward_model_step(self, actor_batch):  # :224-242 (same tokenizer) -- NOT replaced
        reward_batch = copy.deepcopy(actor_batch)
        reward_batch['reward'] = self.reward_model(**self.reward_infer_batch(reward_batch)).end_scores.squeeze(dim=-1)
        scores = self.reward_critic_model(**self.reward_infer_batch(actor_batch)).scores
        reward_batch['reward_values'] = scores.squeeze(dim=-1)[:, :-1]
        return reward_batch

    def set_train(self, mode=True):  # trainers/base/rl_trainer.py:274-286
        self.train_mode_calls.append(mode)
        for m in (self.actor_model, self.reward_critic_model):
            (m.train if mode else m.eval)()

    rollout = _not_grafted('rollout')
    actor_loss_fn = _not_grafted('actor_loss_fn')
    critic_loss_fn = _not_grafted('critic_loss_fn')
    add_kl_divergence_regularization = _not_grafted('add_kl_divergence_regularization')
    get_advantages_and_returns = _not_grafted('get_advantages_and_returns')
    rl_step = _not_grafted('rl_step')
    ptx_step = _not_grafted('ptx_step')

    def train(self):  # :410-460, one epoch, no ptx / eval / save
        infos = []
        for prompt_only_batch in self.prompt_only_dataloader:
            inference_batches, training_batches = self.rollout(prompt_only_batch)
            for _ in range(self.cfgs.train_cfgs.update_iters):
                for inference_batch, training_batch in zip(inference_batches, training_batches):
                    rl_info = self.rl_step(inference_batch, training_batch)
                    self.logger.log(rl_info, step=self.global_step)
                    self.global_step += 1
                    infos.append(f'(reward {rl_info["train/reward"]:.4f})')  # the progress-bar f-string of :451-454
        return infos


class _MMPPOTrainer(_TextPPOTrainer):
    """Shape of trainers/text_image_to_text/ppo.py:PPOTrainer (subclass of the text trainer, :90)."""

    actor_step = _not_grafted('actor_step')  # :174-204 -- replaced (per-sample .tolist() bookkeeping)
    rollout = _not_grafted('rollout')
    rl_step = _not_grafted('rl_step')


class _AudioPPOTrainer(_TextPPOTrainer):
    """Shape of trainers/text_audio_to_text/ppo.py:PPOTrainer."""

    actor_step = _not_grafted('actor_step')
    rollout = _not_grafted('rollout')
    rl_step = _not_grafted('rl_step')


@contextlib.contextmanager
def installed():
    """Put the stand-in tree into sys.modules (saving whatever was there) for the duration of the block."""
    saved = {n: sys.modules.get(n) for n in _NAMES}
    mods = {}
    for n in _NAMES:
        m = types.ModuleType(n)
        m.__path__ = []
        mods[n] = m
    tools = mods['align_anything.utils.tools']
    for fn in ('gather_log_probabilities', 'masked_mean', 'move_padding_left'):
        setattr(tools, fn, _not_grafted(fn))
    for modname, cls in (('align_anything.trainers.text_to_text.ppo', _TextPPOTrainer),
                         ('align_anything.trainers.text_image_to_text.ppo', _MMPPOTrainer),
                         ('align_anything.trainers.text_audio_to_text.ppo', _AudioPPOTrainer)):
        m = mods[modname]
        # fresh subclasses so that patching never leaks between tests
        m.PPOTrainer = type('PPOTrainer', (cls,), {'__module__': modname})
        for fn in ('gather_log_probabilities', 'masked_mean'):  # `from align_anything.utils.tools import ...`
            setattr(m, fn, getattr(tools, fn))
    mods['align_anything.trainers.text_image_to_text.ppo'].move_padding_left = tools.move_padding_left
    for n, m in mods.items():
        sys.modules[n] = m
        parent, _, child = n.rpartition('.')
        if parent:
            setattr(mods[parent], child, m)
    try:
        yield mods
    finally:
        for n, old in saved.items():
            if old is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = old


class TinyLM(torch.nn.Module):
    """Embedding -> linear head: a causal-LM-shaped module (`.logits`, `generate`, `logits_to_keep`)."""

    def __init__(self, vocab, hidden, pad_id, eos_id, max_new_tokens, seed):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.emb = torch.nn.Parameter(torch.randn(vocab, hidden, generator=g) * 0.5)
        self.head = torch.nn.Parameter(torch.randn(vocab, hidden, generator=g) * 0.3)
        self.pad_id, self.eos_id, self.max_new_tokens, self.vocab = pad_id, eos_id, max_new_tokens, vocab
        self.gen = torch.Generator().manual_seed(seed + 1)

    def forward(self, input_ids=None, attention_mask=None, use_cache=None, logits_to_keep=0, **kw):
        h = self.emb[input_ids]
        if isinstance(logits_to_keep, int) and logits_to_keep > 0:
            h = h[:, -logits_to_keep:]
        return types.SimpleNamespace(logits=h @ self.head.t())

    @torch.no_grad()
    def generate(self, input_ids=None, attention_mask=None, generation_config=None, synced_gpus=None, do_sample=None, **kw):
        B = input_ids.size(0)
        out = torch.full((B, self.max_new_tokens), self.pad_id, dtype=torch.int64)
        n_new = torch.randint(2, self.max_new_tokens + 1, (B,), generator=self.gen)
        n_new[0] = self.max_new_tokens
        for b in range(B):
            n = int(n_new[b])
            out[b, :n - 1] = torch.randint(3, self.vocab, (n - 1,), generator=self.gen)
            out[b, n - 1] = self.eos_id
        return torch.cat([input_ids, out.to(input_ids.device)], dim=1)


class TinyScoreModel(torch.nn.Module):
    """Backbone + scalar head returning the ScoreModelOutput of the grafted Accustomed*RewardModel.forward."""

    def __init__(self, vocab, hidden, seed, end_mode='mask'):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.emb = torch.nn.Parameter(torch.randn(vocab, hidden, generator=g) * 0.5)
        self.score_head = torch.nn.Linear(hidden, 1, bias=False)
        with torch.no_grad():
            self.score_head.weight.copy_(torch.randn(1, hidden, generator=g) * 0.2)
        self.end_mode = end_mode

    def forward(self, input_ids=None, attention_mask=None, **kw):
        from align_anything_b200.models.reward_model import score_model_outputs

        return score_model_outputs(self.emb[input_ids], self.score_head.weight, attention_mask, self.end_mode)


class Engine:
    """DeepSpeed-engine-shaped wrapper: __call__, .module, backward, step, optimizer.param_groups, train / eval."""

    def __init__(self, module, lr=1e-3):
        self.module = module
        self.optimizer = torch.optim.SGD(module.parameters(), lr=lr)
        self.training = True
        self.steps = 0

    def __call__(self, *a, **k):
        return self.module(*a, **k)

    def backward(self, loss):
        loss.backward()

    def step(self):
        self.optimizer.step()
        self.optimizer.zero_grad(set_to_none=True)
        self.steps += 1

    def train(self):
        self.training = True

    def eval(self):
        self.training = False
