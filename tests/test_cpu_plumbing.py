"""CPU dry run of the Python layer above the C ABI (no kernel runs, no numbers are checked): `_lib.lib()` is replaced by
a stand-in that validates every call against the declared ctypes signature (argument count, pointer / integer / float
kinds) and returns 0, `require_cuda` is disabled and `torch.empty` zero-fills, so every trainer path can be driven end
to end on CPU tensors.  What this pins: the host logic -- argument marshalling for every entry point on the DPO / PPO /
lm_head paths, autograd wiring of the fused nodes, the graft (patch.install on a reference-shaped tree), dict keys,
scalar-only metric dicts -- i.e. everything that would otherwise only fail on the GPU."""
import ctypes
import math
import sys
from types import SimpleNamespace

import pytest
import torch

import fake_reference_tree as fake


class _FakeLib:
    def __init__(self, sigs):
        self.calls = []
        for name, (res, args) in sigs.items():
            setattr(self, name, self._make(name, args))

    def _make(self, name, argtypes):
        def fn(*args):
            assert len(args) == len(argtypes), f'{name}: {len(args)} arguments, the C ABI declares {len(argtypes)}'
            for i, (a, t) in enumerate(zip(args, argtypes)):
                if t is ctypes.c_void_p:
                    assert a is None or isinstance(a, int) or isinstance(a, ctypes.c_void_p), (name, i, type(a))
                elif t in (ctypes.c_int, ctypes.c_int32, ctypes.c_int64, ctypes.c_uint32):
                    assert isinstance(a, int) and not isinstance(a, bool), (name, i, type(a), a)
                elif t is ctypes.c_float:
                    assert isinstance(a, (int, float)), (name, i, type(a))
                else:  # POINTER(struct / int32): None, byref(...) or a ctypes pointer
                    assert a is None or 'CArgObject' in type(a).__name__ or isinstance(a, ctypes._Pointer), (name, i, type(a))
            self.calls.append(name)
            return 0

        return fn

    def aa_abi_version(self):
        return 3

    def aa_last_error(self):
        return b''


def _install_dry(setattr_):
    """Swap the stand-in library in through `setattr_` (monkeypatch.setattr, or the builtin in a subprocess)."""
    from align_anything_b200 import _lib, ops

    lib = _FakeLib(_lib._SIGS)
    setattr_(_lib, 'lib', lambda: lib)
    setattr_(_lib, 'require_cuda', lambda *t: None)
    setattr_(_lib, 'stream_ptr', lambda device=None: 0)
    setattr_(torch, 'empty', torch.zeros)  # outputs the kernels would have written: zeros (status word = 0)
    setattr_(ops, '_scratch', {})
    setattr_(ops, '_device_scratch', lambda device: ops._scratch.setdefault('cpu', {
        'status': torch.zeros(1, dtype=torch.int32), 'counter': torch.zeros(8, dtype=torch.int32)}))
    return lib


@pytest.fixture
def dry(monkeypatch):
    from align_anything_b200 import ops

    lib = _install_dry(monkeypatch.setattr)
    monkeypatch.setattr(ops, '_FUSED_MIN_ROW_BYTES', 0)  # the toy vocabularies here would take the two-pass path: drive K1f's calls
    ops._lens_tensor.cache_clear()
    ops._tail_plan.cache_clear()
    ops._dense_plan.cache_clear()
    yield lib
    ops._lens_tensor.cache_clear()
    ops._tail_plan.cache_clear()
    ops._dense_plan.cache_clear()


def _trainer(cls, micro=2):
    t = object.__new__(cls)
    t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(per_device_train_batch_size=micro, update_iters=1))
    t.tokenizer = SimpleNamespace(pad_token_id=0, eos_token_id=2)
    t.reward_tokenizer = t.tokenizer
    t.generation_config = None
    t.infer_batch = lambda batch: {k: v for k, v in batch.items() if k != 'meta_info'}
    t.reward_infer_batch = t.infer_batch
    mk = lambda m: fake.Engine(m.bfloat16())
    t.actor_model = mk(fake.TinyLM(97, 16, 0, 2, 6, seed=1))
    t.actor_reference_model = mk(fake.TinyLM(97, 16, 0, 2, 6, seed=2))
    t.reward_model = mk(fake.TinyScoreModel(97, 16, seed=3))
    t.reward_critic_model = mk(fake.TinyScoreModel(97, 16, seed=4))
    t.kl_coeff, t.clip_range_ratio, t.clip_range_score, t.clip_range_value = 0.02, 0.2, 50.0, 5.0
    t.gamma, t.gae_lambda, t.ptx_coeff = 1.0, 0.95, 16.0
    t.logger = fake.Logger()
    t.global_step = 0
    t.train_mode_calls = []
    ids = torch.randint(3, 97, (4, 5))
    ids[1, :2] = 0
    t.prompt_only_dataloader = [{'input_ids': ids, 'attention_mask': ids != 0}]
    return t


@pytest.mark.parametrize('modality', ['text', 'image', 'audio'])
def test_patched_ppo_train_loop_dry_run(dry, modality):
    from align_anything_b200 import patch

    modname = {'text': 'text_to_text', 'image': 'text_image_to_text', 'audio': 'text_audio_to_text'}[modality]
    with fake.installed() as mods:
        cls = mods[f'align_anything.trainers.{modname}.ppo'].PPOTrainer
        patch.install()
        try:
            t = _trainer(cls)
            t.train()
        finally:
            patch.uninstall()
    assert t.global_step == (1 if modality == 'image' else 2)
    keys = {k for k, _, _ in t.logger.writer.records}
    assert {'train/actor_loss', 'train/reward_critic_loss', 'train/kl_divergence', 'train/max_generated_length'} <= keys
    assert t.actor_model.steps == t.reward_critic_model.steps == t.global_step
    # the actor node is the single-pass K1f in every modality: no separate K1b launch
    expect = {'aa_ppo_prep', 'aa_logprob_fwd', 'aa_ppo_actor_loss', 'aa_ppo_critic_loss', 'aa_score_head_fwd',
              'aa_score_head_bwd', 'aa_ppo_pack_metrics', 'aa_logprob_actor_fused', 'aa_scale_tile'}
    if modality != 'text':
        expect |= {'aa_ppo_rollout_layout', 'aa_tail_plan_build', 'aa_tail_scatter_scaled', 'aa_tail_rows'}
    assert 'aa_logprob_bwd' not in dry.calls
    assert expect <= set(dry.calls), expect - set(dry.calls)
    assert 'aa_move_padding_left' not in dry.calls and 'aa_count_nonpad' not in dry.calls  # one layout launch instead


@pytest.mark.parametrize('modality', ['text', 'image', 'audio'])
@pytest.mark.parametrize('fused_head', [False, True])
def test_dpo_train_step_dry_run(dry, modality, fused_head):
    from align_anything_b200.trainers.text_audio_to_text.dpo import DPOTrainer as A
    from align_anything_b200.trainers.text_image_to_text.dpo import DPOTrainer as I
    from align_anything_b200.trainers.text_to_text.dpo import DPOTrainer as T

    cls = {'text': T, 'image': I, 'audio': A}[modality]
    V, H, L_, B = 101, 64, 12, 2
    ids = torch.randint(2, V - 1, (2 * B, L_))
    lens = [5, 7, 4, 6]
    leaf = torch.randn(2 * B, L_, V).bfloat16().requires_grad_(True)
    ref = torch.randn(2 * B, L_, V).bfloat16()
    hid = torch.randn(2 * B, L_, H).bfloat16().requires_grad_(True)
    w = torch.randn(V, H).bfloat16().requires_grad_(True)

    class Eng:
        def __init__(self, logits, hidden, weight):
            self.module = self
            self.o = SimpleNamespace(logits=logits, hidden_states=(hidden,))
            self.w = weight
            self.optimizer = SimpleNamespace(param_groups=[{'lr': 1e-6}])

        def __call__(self, **kw):
            return self.o

        def get_output_embeddings(self):
            return SimpleNamespace(weight=self.w)

        def backward(self, loss):
            loss.backward()

        def step(self):
            pass

    tr = cls(SimpleNamespace(train_cfgs=SimpleNamespace(scale_coeff=0.1)), Eng(leaf, hid, w), Eng(ref, hid.detach(), w.detach()),
             SimpleNamespace(pad_token_id=V - 1))
    tr.fused_lm_head = fused_head
    out = tr.train_step({'input_ids': ids, 'attention_mask': ids != V - 1, 'meta_info': {'response_lens': lens}})
    assert set(out) == {'train/loss', 'train/reward', 'train/better_sample_reward', 'train/worse_sample_reward',
                        'train/reward_accuracy', 'train/reward_margin', 'train/lr'}
    assert all(isinstance(v, float) for v in out.values())
    if fused_head:
        assert {'aa_linear_logprob_fwd', 'aa_linear_dlogits', 'aa_linear_dhidden', 'aa_linear_dweight', 'aa_dpo_loss'} <= set(dry.calls)
        assert hid.grad is not None and w.grad is not None and hid.grad.shape == hid.shape and w.grad.shape == w.shape
    else:
        assert {'aa_strip_pad_tail', 'aa_logprob_fwd', 'aa_dpo_loss', 'aa_logprob_bwd'} <= set(dry.calls)
        assert leaf.grad is not None and leaf.grad.shape == leaf.shape


def test_sibling_trainers_dry_run(dry):
    """SFT / RM / GRPO steps: the status lane rides in each metric vector, every returned value is a float."""
    from align_anything_b200.models.reward_model import score_model_outputs
    from align_anything_b200.trainers.text_to_text.grpo import GRPOTrainer
    from align_anything_b200.trainers.text_to_text.rm import RMTrainer
    from align_anything_b200.trainers.text_to_text.sft import SupervisedTrainer

    V, L_ = 53, 9

    class Eng:
        def __init__(self, fn):
            self.fn, self.module = fn, SimpleNamespace(parameters=lambda: iter([torch.zeros(1)]))
            self.optimizer = SimpleNamespace(param_groups=[{'lr': 1e-6}])

        def __call__(self, **kw):
            return self.fn()

        def backward(self, loss):
            loss.backward()

        def step(self):
            pass

        def zero_grad(self):
            pass

        def train(self):
            pass

    logits = torch.randn(2, L_, V).bfloat16().requires_grad_(True)
    labels = torch.randint(0, V, (2, L_))
    out = SupervisedTrainer(None, Eng(lambda: SimpleNamespace(logits=logits))).train_step(
        {'input_ids': labels, 'labels': labels, 'attention_mask': torch.ones_like(labels)})
    assert isinstance(out['train/loss'], float)
    assert 'aa_logprob_ce_fused' in dry.calls and 'aa_nll_mean' in dry.calls  # the single-pass cross-entropy node
    hidden = torch.randn(4, L_, 16).bfloat16().requires_grad_(True)
    wt = torch.randn(1, 16).bfloat16().requires_grad_(True)
    mask = torch.ones(4, L_, dtype=torch.bool)
    rm = RMTrainer(SimpleNamespace(train_cfgs=SimpleNamespace(regularization=0.01)),
                   Eng(lambda: score_model_outputs(hidden, wt, mask, 'mask', True)))
    out = rm.train_step({'input_ids': torch.randint(0, V, (4, L_)), 'attention_mask': mask})
    assert isinstance(out['train/loss'], float) and isinstance(out['train/accuracy'], float)
    g = GRPOTrainer(None, Eng(lambda: SimpleNamespace(logits=torch.randn(4, L_, V).bfloat16().requires_grad_(True))),
                    Eng(lambda: SimpleNamespace(logits=torch.randn(4, L_, V).bfloat16())),
                    SimpleNamespace(pad_token_id=0, eos_token_id=2), beta=0.04, num_generations=2)
    out = g.step_from_rollout(torch.randint(3, V, (4, L_)), 4, torch.randn(4))
    assert isinstance(out['train/loss'], float) and isinstance(out['train/reward'], float)
    assert 'aa_logprob_grpo_fused' in dry.calls and 'aa_grpo_loss' in dry.calls  # the single-pass GRPO node


def _saferlhf_trainer():
    import copy

    from align_anything_b200.trainers.text_image_to_text.saferlhf import SafeRLHFVTrainer

    t = _trainer(SafeRLHFVTrainer)
    t.mode = None
    t.cost_model = fake.Engine(fake.TinyScoreModel(97, 16, seed=5).bfloat16())
    t.cost_critic_model = fake.Engine(fake.TinyScoreModel(97, 16, seed=6).bfloat16())
    t.log_lambda = torch.nn.Parameter(torch.tensor(0.1))
    t.log_lambda_optimizer = torch.optim.SGD([t.log_lambda], lr=0.1)
    t.log_lambda_max, t.threshold, t.episode_costs, t.lambda_update_delay_steps = 5.0, 0.0, [0.3, -0.1], 0

    def cost_model_step(actor_batch):  # the reference's own method (saferlhf.py:321-341), restated for the harness
        cost_batch = copy.copy(actor_batch)
        cost_batch['cost'] = t.cost_model(**t.reward_infer_batch(cost_batch)).end_scores.squeeze(dim=-1)
        cost_batch['cost_values'] = t.cost_critic_model(**t.reward_infer_batch(actor_batch)).scores.squeeze(dim=-1)[:, :-1]
        return cost_batch

    t.cost_model_step = cost_model_step
    t.set_train = lambda mode=True: None
    return t


def test_saferlhf_rollout_and_rl_step_dry_run(dry):
    """Safe RLHF-V: actor_step -> score_rollout (reward + cost) -> rl_step, scalar-only dict with the 16 + 5 keys."""
    t = _saferlhf_trainer()
    inference, training = t.rollout(t.prompt_only_dataloader[0])
    assert len(inference) == len(training) == 1 and {'cost', 'cost_values', 'response_lens', 'response_mask'} <= set(training[0])
    out = t.rl_step(inference[0], training[0])
    assert all(isinstance(v, float) for v in out.values()), {k: type(v) for k, v in out.items()}
    assert {'train/cost_critic_loss', 'train/lambda', 'train/cost_value', 'train/actor_loss'} <= set(out)
    assert t.cost_critic_model.steps == 1 and set(t.last_rl_tensors) >= {'old_costs', 'cost_advantages'}


def test_short_rows_take_the_two_pass_calls(dry, monkeypatch):
    """With the default ops._FUSED_MIN_ROW_BYTES the toy vocabulary (97 tokens) is far too short for K1f: the text PPO
    rl_step must then call K1 -> K5 -> K1b (aa_logprob_fwd, aa_ppo_actor_loss, aa_logprob_bwd) and never the single-pass entry."""
    from align_anything_b200 import ops, patch

    monkeypatch.setattr(ops, '_FUSED_MIN_ROW_BYTES', 192 * 1024)
    with fake.installed() as mods:
        cls = mods['align_anything.trainers.text_to_text.ppo'].PPOTrainer
        patch.install()
        try:
            t = _trainer(cls)
            t.train()
        finally:
            patch.uninstall()
    assert 'aa_logprob_actor_fused' not in dry.calls
    assert {'aa_logprob_fwd', 'aa_ppo_actor_loss', 'aa_logprob_bwd'} <= set(dry.calls)


@pytest.mark.parametrize('min_row_bytes', [0, 192 * 1024])
def test_saferlhf_actor_node_picks_its_path(dry, monkeypatch, min_row_bytes):
    """SafeRLHF-V's rl_step hands the Lagrangian-mixed advantages to ops.tail_actor_loss and lets ops pick the path:
    the single-pass K1f once the rows are long enough, K1 -> K5 -> K1b on the toy vocabulary's 194-byte rows at the
    default threshold."""
    from align_anything_b200 import ops

    monkeypatch.setattr(ops, '_FUSED_MIN_ROW_BYTES', min_row_bytes)
    t = _saferlhf_trainer()
    inference, training = t.rollout(t.prompt_only_dataloader[0])
    dry.calls.clear()
    t.rl_step(inference[0], training[0])
    if min_row_bytes == 0:
        assert 'aa_logprob_actor_fused' in dry.calls and 'aa_logprob_bwd' not in dry.calls
    else:
        assert 'aa_logprob_actor_fused' not in dry.calls
        assert {'aa_logprob_fwd', 'aa_ppo_actor_loss', 'aa_logprob_bwd'} <= set(dry.calls)


_RETIRED_SWITCHES = {  # environment variables that once chose between duplicate paths, at their non-default values
    'AA_B200_REROUTE_BASE': '0', 'AA_B200_K6': '0', 'AA_B200_K6B': '0', 'AA_B200_ZERO_SPANS': '0',
    'AA_B200_FUSED_ACTOR': '0', 'AA_B200_FUSED_F16': '1', 'AA_B200_FUSED_MIN_ROW_BYTES': '0',
    'AA_B200_FUSED_GRPO': '0', 'AA_B200_FUSED_CE': '0', 'AA_B200_DUAL_K1': '0',
}

_ENV_WORKER = r'''
import sys
sys.path[:0] = sys.argv[1:]
import torch
import test_cpu_plumbing as T
from align_anything_b200 import ops
knobs = (ops._K6B, ops._ZERO_SPANS, ops._FUSED_ACTOR, ops._FUSED_GRPO, ops._FUSED_CE, ops._FUSED_F16, ops._FUSED_MIN_ROW_BYTES)
assert knobs == (True, True, True, True, True, False, 192 * 1024), knobs
lib = T._install_dry(setattr)
B, K, V = 2, 6, 98304  # 192 KB bf16 rows: long enough for the single-pass nodes
gen = torch.Generator().manual_seed(0)
logits = torch.randn(B, K, V, generator=gen).bfloat16().requires_grad_(True)
ids = torch.randint(0, V, (B, K + 2), generator=gen)
W = 3
loss, _, _ = ops.tail_actor_loss(logits, ids, [W, 2], torch.zeros(B, W), torch.randn(B, W, generator=gen),
                                 torch.ones(B, W, dtype=torch.bool), 0.2)
loss.backward()
assert 'aa_logprob_actor_fused' in lib.calls and 'aa_logprob_fwd' not in lib.calls, lib.calls
lib.calls.clear()
ops.causal_lm_loss(logits, torch.randint(0, V, (B, K), generator=gen)).backward()
assert 'aa_logprob_ce_fused' in lib.calls and 'aa_logprob_fwd' not in lib.calls, lib.calls
print('ok')
'''


def test_retired_switches_do_not_change_paths(tmp_path):
    """The paths are chosen from the input alone: with every retired switch set, ops still starts from its defaults and
    a long-row tile still reaches the single-pass actor and cross-entropy entry points."""
    import os
    import subprocess

    tests = os.path.dirname(os.path.abspath(__file__))
    script = tmp_path / 'worker.py'
    script.write_text(_ENV_WORKER)
    r = subprocess.run([sys.executable, str(script), os.path.dirname(tests), tests], env=dict(os.environ, **_RETIRED_SWITCHES),
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip().endswith('ok'), r.stdout + r.stderr
