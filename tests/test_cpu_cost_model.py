"""The cost-model loss without a GPU: the ATen port against the goldens the reference produced (bit for bit, value and
dtype) and against a float64 restatement, the argument errors of aa_cost_pair_loss / ops.cost_pair_loss, and a dry
run of the graft on a stand-in tree of the reference's RM / cost-model trainer modules."""
import contextlib
import ctypes
import sys
import types
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import cost_model_port as P
import fake_reference_tree as fake
from test_cpu_plumbing import dry  # noqa: F401  (`dry` is a fixture)


# ---- the port against the reference's goldens --------------------------------------------------------------------
def test_port_matches_reference_goldens(golden):
    cases = golden('cost_model')['cases']
    assert len(cases) == 3 * 2 * 5 * 2 * 2
    for key, c in cases.items():
        leaf = c['end_scores'].clone().requires_grad_(True)
        got = P.cm_loss(leaf, c['better'], c['worse'], c['scale_coeff'], c['regularization'])
        got['loss'].backward()
        assert got['loss'].dtype == c['loss_dtype'], key
        assert torch.equal(got['loss'].detach(), c['loss']), key
        assert torch.equal(got['accuracy'], c['accuracy']), key
        assert torch.equal(leaf.grad, c['grad']), key
        want, want_grad = P.cm_loss_f64(c['end_scores'], c['better'], c['worse'], c['scale_coeff'], c['regularization'])
        tol = 1e-5 if c['end_scores'].dtype == torch.float32 else 3e-2
        assert abs(float(c['loss']) - want) <= tol * max(1.0, abs(want)), key
        g = c['grad'].double().reshape(-1).numpy()
        assert np.allclose(g, want_grad, rtol=tol, atol=tol * np.abs(want_grad).max()), key


def test_sign_dtypes_decide_the_arithmetic(golden):
    """int / bool signs keep bf16 end scores in bf16; a float in either list makes that term, and the loss, fp32."""
    cases = golden('cost_model')['cases']
    for kind, want in (('int', torch.bfloat16), ('bool', torch.bfloat16), ('float', torch.float32),
                       ('mixed', torch.float32), ('int_float', torch.float32)):
        for B in (1, 4, 7):
            assert cases[f'B{B}_bf16_{kind}_s1_r0.001']['loss_dtype'] == want, (kind, B)
            assert cases[f'B{B}_f32_{kind}_s1_r0.001']['loss_dtype'] == torch.float32, (kind, B)
    c = cases['B4_bf16_int_s1_r0.0']
    assert c['better'][0] == 0 and c['grad'].dtype == torch.bfloat16
    # the tie and the saturated rows are in the grid
    h, lo = c['end_scores'].float().reshape(-1).chunk(2)
    assert h[0] == lo[0] and abs(float(h[1] - lo[1])) >= 30 and abs(float(h[2] - lo[2])) >= 30


def test_audio_rm_golden_is_the_rm_loss(golden):
    for key, c in golden('cost_model')['audio_rm'].items():
        leaf = c['end_scores'].clone().requires_grad_(True)
        got = P.rm_loss(leaf, c['regularization'])
        got['loss'].backward()
        assert torch.equal(got['loss'].detach(), c['loss']) and got['loss'].dtype == c['loss_dtype'], key
        assert torch.equal(leaf.grad, c['grad']), key


# ---- argument errors ---------------------------------------------------------------------------------------------
def test_cost_pair_loss_argument_errors_need_no_gpu():
    from align_anything_b200 import _lib

    lib = _lib.lib()
    buf = (ctypes.c_int64 * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def call(n=4, scores=p, sd=0, sb=p, bd=0, sw=p, wd=0, mode=0, loss=p, stats=p):
        return lib.aa_cost_pair_loss(scores, sd, sb, bd, sw, wd, n, 1.0, 0.001, mode, loss, stats, None, None)

    assert call(n=0) == -2 and b'bad sizes' in lib.aa_last_error()
    assert call(n=-3) == -2 and b'bad sizes' in lib.aa_last_error()
    for kw in ({'scores': None}, {'sb': None}, {'sw': None}, {'loss': None}, {'stats': None}):
        assert call(**kw) == -2 and b'null pointer' in lib.aa_last_error(), kw
    assert call(sd=7) == -1 and b'bad dtype' in lib.aa_last_error()
    assert call(sd=0, bd=1) == -1 and b'bad sign dtype' in lib.aa_last_error()  # bf16 scores, f16 signs
    assert call(sd=2, wd=0) == -1 and b'bad sign dtype' in lib.aa_last_error()  # fp32 scores, bf16 signs
    assert call(mode=2) == -2 and b'bad mode' in lib.aa_last_error()


def test_ops_raise_on_the_host_before_any_launch():
    from align_anything_b200 import ops

    with pytest.raises(ValueError, match='2B values'):
        ops.cost_pair_loss(torch.zeros(5, 1), [1, 1], [1, 1], 1, 0.001)
    with pytest.raises(RuntimeError, match='is_better_safe holds 3 values for 2 pairs'):
        ops.cost_pair_loss(torch.zeros(4, 1), [1, -1, 0], [1, 1], 1, 0.001)
    with pytest.raises(RuntimeError, match='is_worse_safe holds 1 values for 2 pairs'):  # the reference would broadcast
        ops.cost_pair_loss(torch.zeros(4, 1), [1, -1], [1], 1, 0.001)
    with pytest.raises(RuntimeError, match='no CPU fallback'):  # valid arguments reach the launch
        ops.cost_pair_loss(torch.zeros(4, 1), [1, -1], [0.5, 1], 1, 0.001)


def test_missing_safety_fields_raise_the_reference_keyerror(golden, dry):  # noqa: F811
    from align_anything_b200.trainers.text_to_text.cost_model import CMTrainer

    missing = golden('cost_model')['missing_safety_fields']
    calls = []
    t = CMTrainer(SimpleNamespace(train_cfgs=SimpleNamespace(scale_coeff=1, regularization=0.001)),
                  lambda **kw: calls.append(kw))
    batch = {'input_ids': torch.zeros(4, 3, dtype=torch.int64), 'meta_info': {'better_response': ['a', 'b']}}
    with pytest.raises(KeyError) as e:
        t.loss(batch)
    assert e.value.args[0] == missing == 'is_better_safe'
    assert calls == [] and dry.calls == []  # neither the model nor a kernel ran


# ---- the graft on a stand-in tree --------------------------------------------------------------------------------
RM_MODS = {
    'text': 'align_anything.trainers.text_to_text.rm',
    'audio': 'align_anything.trainers.text_audio_to_text.rm',
    'video': 'align_anything.trainers.text_video_to_text.rm',
}
CM_MODS = {
    'text': 'align_anything.trainers.text_to_text.cost_model',
    'image': 'align_anything.trainers.text_image_to_text.cost_model',
}


@contextlib.contextmanager
def _rm_cm_tree():
    """The reference's class shapes: the text RMTrainer / CMTrainer own loss + train_step; the audio and video
    RMTrainers override loss only (text_audio_to_text/rm.py:67-102); the image CMTrainer overrides neither."""
    names = [*RM_MODS.values(), *CM_MODS.values()]
    saved = {n: sys.modules.get(n) for n in names}
    mods = {n: types.ModuleType(n) for n in names}
    text_rm = type('RMTrainer', (), {'__module__': RM_MODS['text'], 'loss': fake._not_grafted('RMTrainer.loss'),
                                     'train_step': fake._not_grafted('RMTrainer.train_step')})
    mods[RM_MODS['text']].RMTrainer = text_rm
    for m in ('audio', 'video'):
        mods[RM_MODS[m]].RMtextTrainer = text_rm
        mods[RM_MODS[m]].RMTrainer = type('RMTrainer', (text_rm,), {'__module__': RM_MODS[m],
                                                                    'loss': fake._not_grafted(f'{m} RMTrainer.loss')})
    text_cm = type('CMTrainer', (), {'__module__': CM_MODS['text'], 'loss': fake._not_grafted('CMTrainer.loss'),
                                     'train_step': fake._not_grafted('CMTrainer.train_step')})
    mods[CM_MODS['text']].CMTrainer = text_cm
    mods[CM_MODS['image']].CMtextTrainer = text_cm
    mods[CM_MODS['image']].CMTrainer = type('CMTrainer', (text_cm,), {'__module__': CM_MODS['image']})
    sys.modules.update(mods)
    try:
        yield mods
    finally:
        for n, old in saved.items():
            if old is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = old


class _Engine:
    def __init__(self, fn):
        self.fn = fn
        self.optimizer = SimpleNamespace(param_groups=[{'lr': 3e-5}])

    def __call__(self, **kw):
        return self.fn(kw)

    def backward(self, loss):
        loss.backward()

    def step(self):
        pass


def _trainer(cls, cfgs):
    """object.__new__ a stand-in trainer with the attributes the reference's __init__ sets and the loss reads."""
    from align_anything_b200.models.reward_model import score_model_outputs

    t = object.__new__(cls)
    t.cfgs = cfgs
    t.scale_coeff = cfgs.train_cfgs.scale_coeff
    t.infer_batch = lambda b: {k: v for k, v in b.items() if k != 'meta_info'}
    hidden = torch.randn(4, 5, 16).bfloat16().requires_grad_(True)
    wt = torch.randn(1, 16).bfloat16().requires_grad_(True)
    t.model = _Engine(lambda kw: score_model_outputs(hidden, wt, kw['attention_mask'], 'mask', True))
    return t, hidden, wt


def test_graft_dry_run(dry):  # noqa: F811
    from align_anything_b200 import patch
    from align_anything_b200.trainers.text_to_text.cost_model import CMTrainer as MirrorCM
    from align_anything_b200.trainers.text_to_text.rm import RMTrainer as MirrorRM

    cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(scale_coeff=1, regularization=0.001))
    batch = {'input_ids': torch.zeros(4, 5, dtype=torch.int64), 'attention_mask': torch.ones(4, 5, dtype=torch.bool),
             'meta_info': {'is_better_safe': [-1, 0], 'is_worse_safe': [1.0, -2.5]}}
    with fake.installed(), _rm_cm_tree() as mods:
        audio = mods[RM_MODS['audio']].RMTrainer
        image_cm = mods[CM_MODS['image']].CMTrainer
        originals = {cls: dict(cls.__dict__) for cls in (audio, image_cm, mods[RM_MODS['text']].RMTrainer,
                                                         mods[CM_MODS['text']].CMTrainer, mods[RM_MODS['video']].RMTrainer)}
        done = patch.install()
        try:
            for modname, cls in (*((m, 'RMTrainer') for m in RM_MODS.values()), (CM_MODS['text'], 'CMTrainer')):
                assert set(done[modname]) == {f'{cls}.loss', f'{cls}.train_step'}, modname
            assert CM_MODS['image'] not in done  # it inherits both from the text trainer
            assert image_cm.loss is MirrorCM.loss and image_cm.train_step is MirrorRM.train_step
            assert audio.loss is MirrorRM.loss and audio.train_step is MirrorRM.train_step

            t, hidden, wt = _trainer(audio, cfgs)
            out = t.train_step(batch)  # the reference's own loss here would not return '_stats': KeyError
            assert set(out) == {'train/loss', 'train/accuracy', 'train/lr'}
            assert all(isinstance(v, float) for v in out.values())
            assert 'aa_rm_pair_loss' in dry.calls and 'aa_cost_pair_loss' not in dry.calls

            t, hidden, wt = _trainer(image_cm, cfgs)
            res = t.loss(batch)
            assert {'loss', 'accuracy', 'higher_end_reward', 'lower_end_reward', 'higher_rewards', 'lower_rewards',
                    '_stats'} == set(res)
            assert res['loss'].dtype == torch.float32  # a float sign list: the loss is fp32
            out = t.train_step(batch)
            assert set(out) == {'train/loss', 'train/accuracy', 'train/lr'} and out['train/lr'] == 3e-5
            assert all(isinstance(v, float) for v in out.values())
            assert 'aa_cost_pair_loss' in dry.calls and 'aa_score_head_bwd' in dry.calls
            assert hidden.grad is not None and wt.grad is not None
        finally:
            patch.uninstall()
        for cls, d in originals.items():
            assert dict(cls.__dict__) == d, cls
