"""Drop-in test of the graft under the reference's own `train()` loop (VERDICT r1, task 1): `patch.install()` on a
reference-shaped module tree (tests/fake_reference_tree.py: the reference's sources are not needed), then
`train()` = rollout -> rl_step -> Logger.log per micro-batch with fake engines and a fake `generate`.  What is
asserted: the grafted `rollout` / `actor_step` / `rl_step` are ours, the text trainer's `actor_step` and every
`reward_model_step` stay the tree's own, every value that reaches the tensorboard-style writer is a Python scalar,
the key set is the reference's (trainers/text_to_text/ppo.py:385-398), and the numbers are finite and consistent with
the generated lengths."""
import math
from types import SimpleNamespace

import pytest
import torch

import fake_reference_tree as fake  # tests/ is on sys.path (pytest rootdir conftest)

pytestmark = pytest.mark.gpu

DEV = 'cuda'

REFERENCE_KEYS = {
    'train/actor_loss', 'train/reward_critic_loss', 'train/reward', 'train/reward_with_kl_penalty',
    'train/reward_advantage', 'train/reward_return', 'train/reward_value', 'train/kl_divergence', 'train/actor_lr',
    'train/reward_critic_lr', 'train/mean_generated_length', 'train/max_generated_length',
}


def _make_trainer(cls, dtype, micro_batch, n_prompts=4, prompt_len=9, max_new=12, vocab=311, hidden=32, pad=0, eos=2):
    t = object.__new__(cls)  # like the reference: the graft never sees our __init__
    t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(per_device_train_batch_size=micro_batch, update_iters=1))
    t.tokenizer = SimpleNamespace(pad_token_id=pad, eos_token_id=eos)
    t.reward_tokenizer = t.tokenizer
    t.generation_config = None
    t.infer_batch = lambda batch: {k: v for k, v in batch.items() if k != 'meta_info'}
    t.reward_infer_batch = t.infer_batch
    mk = lambda m: fake.Engine(m.to(DEV).to(dtype))
    t.actor_model = mk(fake.TinyLM(vocab, hidden, pad, eos, max_new, seed=1))
    t.actor_reference_model = mk(fake.TinyLM(vocab, hidden, pad, eos, max_new, seed=2))
    t.reward_model = mk(fake.TinyScoreModel(vocab, hidden, seed=3))
    t.reward_critic_model = mk(fake.TinyScoreModel(vocab, hidden, seed=4))
    t.kl_coeff, t.clip_range_ratio, t.clip_range_score, t.clip_range_value = 0.02, 0.2, 50.0, 5.0
    t.gamma, t.gae_lambda, t.ptx_coeff = 1.0, 0.95, 16.0
    t.logger = fake.Logger()
    t.global_step = 0
    t.train_mode_calls = []
    gen = torch.Generator().manual_seed(11)
    batches = []
    for _ in range(2):
        ids = torch.randint(3, vocab, (n_prompts, prompt_len), generator=gen)
        for b in range(n_prompts):  # left padding of different lengths, as PromptOnlyDataset's collator makes it
            ids[b, :b % 3] = pad
        batches.append({'input_ids': ids.to(DEV), 'attention_mask': (ids != pad).to(DEV)})
    t.prompt_only_dataloader = batches
    return t


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32])
@pytest.mark.parametrize('modality', ['text', 'image', 'audio'])
def test_patched_train_loop_logs_scalars_only(modality, dtype):
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    from align_anything_b200 import patch
    from align_anything_b200.trainers.text_audio_to_text.ppo import PPOTrainer as OurAudio
    from align_anything_b200.trainers.text_image_to_text.ppo import PPOTrainer as OurMM
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer as OurText

    modname = {'text': 'text_to_text', 'image': 'text_image_to_text', 'audio': 'text_audio_to_text'}[modality]
    with fake.installed() as mods:
        cls = mods[f'align_anything.trainers.{modname}.ppo'].PPOTrainer
        tree_actor_step = cls.actor_step
        tree_reward_step = cls.reward_model_step
        done = patch.install()
        try:
            ours = {'text': OurText, 'image': OurMM, 'audio': OurAudio}[modality]
            assert f'PPOTrainer.rollout' in done[f'align_anything.trainers.{modname}.ppo']
            assert cls.rollout is ours.rollout and cls.rl_step is ours.rl_step
            assert cls.reward_model_step is tree_reward_step  # a7: the reference's method runs the patched RM forward
            if modality == 'text':
                assert cls.actor_step is tree_actor_step  # generate + mask: nothing to replace
            else:
                assert cls.actor_step is OurMM.actor_step
                assert cls.micro_batched_rollout is (modality == 'audio')
            micro = 2
            t = _make_trainer(cls, dtype, micro_batch=micro)
            infos = t.train()
        finally:
            patch.uninstall()
    n_prompts = 4
    per_batch = 1 if modality == 'image' else n_prompts // micro  # TI2T: one rollout batch (:206-269)
    assert t.global_step == 2 * per_batch == len(infos)
    assert t.train_mode_calls == [False, True] * 2
    assert t.actor_model.steps == t.reward_critic_model.steps == t.global_step
    records = t.logger.writer.records
    keys = {k for k, _, _ in records}
    assert keys == REFERENCE_KEYS | {'train/step'}, keys ^ (REFERENCE_KEYS | {'train/step'})
    assert all(math.isfinite(v) for _, v, _ in records), [r for r in records if not math.isfinite(r[1])]
    by_key = {}
    for k, v, step in records:
        by_key.setdefault(k, []).append(v)
    # generated lengths: the fake generate always gives sample 0 of a generate call the full 12 new tokens
    assert all(2 <= v <= 12 for v in by_key['train/mean_generated_length'])
    assert all(v == 12.0 for v in by_key['train/max_generated_length'])
    assert all(v >= 0 for v in by_key['train/reward_critic_loss'])
    assert by_key['train/step'] == list(range(t.global_step))
