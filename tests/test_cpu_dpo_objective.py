"""DPO objective options without a GPU: the port (tests/dpo_objective_port.py) against the reference's loss and float64
autograd, ops.DpoObjective's checks, the switches and their config precedence, the graft of the switches, the argument
checks of aa_dpo_loss_obj, and a dry run of train_step on the CPU stand-in library for every modality and head path."""
from __future__ import annotations

import ctypes
import dataclasses
import sys
import types
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from dpo_objective_port import dpo_loss as port_loss
from oracle import ref_port
from test_cpu_plumbing import dry  # noqa: F401  (fixture)

DTYPES = [torch.bfloat16, torch.float16, torch.float32]
LOSS_TYPES = ['sigmoid', 'robust', 'hinge', 'ipo', 'sppo_hard', 'nca_pair', 'apo_zero', 'apo_down']


def _inputs(B=5, W=13, dtype=torch.float32, seed=0):
    g = torch.Generator().manual_seed(seed)
    pol = (-torch.rand(2 * B, W, generator=g) * 3).to(dtype)
    ref = (pol.float() + torch.randn(2 * B, W, generator=g) * 0.5).to(dtype)
    lens = [int(x) for x in torch.randint(2, W + 2, (2 * B,), generator=g)]
    for r, n in enumerate(lens):  # right padding with 0, as the log-prob kernels leave it
        pol[r, n - 1:] = 0
        ref[r, n - 1:] = 0
    ids = torch.randint(0, 50, (2 * B, 7), generator=g)
    ids[B + 1] = ids[1]  # pair 1 is an identical pair
    return pol, ref, ids, lens


def _grad(fn, pol, *args, **kw):
    x = pol.clone().requires_grad_(True)
    out = fn(x, *args, **kw)
    out['loss'].backward()
    return out, x.grad


@pytest.mark.parametrize('skip', [False, True])
@pytest.mark.parametrize('dtype', DTYPES)
def test_default_port_is_the_reference_loss(dtype, skip):
    pol, ref, ids, lens = _inputs(dtype=dtype)
    want, gwant = _grad(ref_port.dpo_loss, pol, ref, 0.1, ids, skip)
    got, ggot = _grad(port_loss, pol, ref, 0.1, ids, skip, response_lens=lens)
    assert set(got) == set(want)
    for k in want:
        assert got[k].dtype == want[k].dtype and torch.equal(got[k], want[k]), k
    assert torch.equal(ggot, gwant)


def _f64(pol, ref, beta, keep, lens, loss_type, eps, alpha, ref_free):
    """The objective in float64 autograd, vectorised over the pairs and written independently of the port."""
    x = pol.double().clone().requires_grad_(True)
    B = x.size(0) // 2
    s = x.sum(1)
    r = torch.zeros_like(s) if ref_free else ref.double().sum(1)
    n = torch.tensor(lens, dtype=torch.float64) - 1
    if loss_type == 'ipo':
        s, r = s / n, r / n
    a, b = (s[:B] - r[:B])[keep], (s[B:] - r[B:])[keep]
    h, c = a - b, 1 / (2 * beta)
    ls, sg = F.logsigmoid, torch.sigmoid
    per = {
        'sigmoid': lambda: -(1 - eps) * ls(beta * h) - eps * ls(-beta * h),
        'robust': lambda: (-(1 - eps) * ls(beta * h) + eps * ls(-beta * h)) / (1 - 2 * eps),
        'hinge': lambda: torch.relu(1 - beta * h),
        'ipo': lambda: (h - c) ** 2,
        'sppo_hard': lambda: (a - c) ** 2 + (b + c) ** 2,
        'nca_pair': lambda: -ls(beta * a) - 0.5 * ls(-beta * a) - 0.5 * ls(-beta * b),
        'apo_zero': lambda: (1 - sg(beta * a)) + sg(beta * b),
        'apo_down': lambda: sg(beta * a) + (1 - sg(beta * h)),
    }[loss_type]()
    loss = per.mean()
    nll = None
    if alpha > 0:
        nll = -x.sum(1)[:B][keep].sum() / n[:B][keep].sum()
        loss = loss + alpha * nll
    loss.backward()
    return loss.detach(), x.grad, nll


OPTIONS = [(t, 0.0, 0.0, False) for t in LOSS_TYPES] + [
    ('sigmoid', 0.1, 0.0, False), ('robust', 0.2, 0.0, False), ('sigmoid', 0.0, 1.0, False), ('ipo', 0.0, 0.5, False),
    ('sigmoid', 0.0, 0.0, True), ('apo_down', 0.0, 1.0, True), ('robust', 0.1, 0.3, True)]


@pytest.mark.parametrize('skip', [False, True])
@pytest.mark.parametrize('opt', OPTIONS, ids=lambda o: '-'.join(map(str, o)))
def test_port_matches_float64_autograd(opt, skip):
    loss_type, eps, alpha, ref_free = opt
    pol, ref, ids, lens = _inputs(B=6, W=17, dtype=torch.float64, seed=3)
    keep = torch.ones(6, dtype=torch.bool)
    if skip:
        keep[1] = False
    got, ggot = _grad(port_loss, pol, ref, 0.1, ids, skip, loss_type, eps, alpha, ref_free, lens)
    want, gwant, nll = _f64(pol, ref, 0.1, keep, lens, loss_type, eps, alpha, ref_free)
    torch.testing.assert_close(got['loss'], want, rtol=1e-12, atol=1e-14)
    mask = pol != 0  # the padding carries no gradient in the trainers (the log-prob kernels never write it)
    torch.testing.assert_close(ggot * mask, gwant * mask, rtol=1e-12, atol=1e-14)
    if alpha > 0:
        torch.testing.assert_close(got['nll_loss'], nll.detach(), rtol=1e-12, atol=1e-14)
    else:
        assert 'nll_loss' not in got
    # the metrics keep the reference's definitions whatever the loss type
    base = ref_port.dpo_loss(pol, torch.zeros_like(ref) if ref_free else ref, 0.1, ids, skip)
    for k in ('reward', 'better_sample_reward', 'worse_sample_reward', 'reward_accuracy', 'reward_margin'):
        assert torch.equal(got[k], base[k]), k


def test_reference_free_is_zero_reference():
    pol, ref, ids, lens = _inputs(dtype=torch.bfloat16, seed=7)
    a, ga = _grad(port_loss, pol, ref, 0.1, loss_type='ipo', reference_free=True, response_lens=lens)
    b, gb = _grad(port_loss, pol, torch.zeros_like(ref), 0.1, loss_type='ipo', response_lens=lens)
    assert torch.equal(a['loss'], b['loss']) and torch.equal(ga, gb)


def test_dpo_objective_checks_its_fields():
    from align_anything_b200.ops import DpoObjective

    assert DpoObjective().is_default and DpoObjective(loss_type='sigmoid', rpo_alpha=0.0).is_default
    for kw in (dict(loss_type='ipo'), dict(label_smoothing=0.1), dict(rpo_alpha=1.0), dict(reference_free=True),
               dict(loss_type='robust', label_smoothing=0.3)):
        assert not DpoObjective(**kw).is_default, kw
    assert DpoObjective(loss_type='ipo').needs_counts and DpoObjective(rpo_alpha=0.5).needs_counts
    assert not DpoObjective(loss_type='hinge', reference_free=True).needs_counts
    for bad in (dict(loss_type='bco_pair'), dict(loss_type='IPO'), dict(label_smoothing=0.5),
                dict(label_smoothing=-0.1), dict(label_smoothing=float('nan')), dict(loss_type='ipo', label_smoothing=0.1),
                dict(loss_type='hinge', label_smoothing=0.2), dict(rpo_alpha=-1.0), dict(rpo_alpha=float('inf')),
                dict(rpo_alpha=float('nan')), dict(reference_free=1)):
        with pytest.raises(ValueError):
            DpoObjective(**bad)
    with pytest.raises(dataclasses.FrozenInstanceError):
        DpoObjective().loss_type = 'ipo'


def test_counts_are_checked_on_the_host():
    from align_anything_b200 import ops

    obj = ops.DpoObjective(loss_type='ipo')
    with pytest.raises(ValueError, match='R_i - 1'):
        ops._dpo_counts(obj, [3, 1, 4, 5], 'cpu')
    with pytest.raises(ValueError, match='response_lens'):
        ops._dpo_counts(obj, None, 'cpu')
    with pytest.raises(ValueError, match='chosen responses'):
        ops._dpo_counts(ops.DpoObjective(rpo_alpha=1.0), [1, 1, 4, 5], 'cpu')
    assert ops._dpo_counts(ops.DpoObjective(loss_type='hinge'), None, 'cpu') is None
    assert ops._dpo_counts(ops.DpoObjective(rpo_alpha=1.0), [1, 2, 4, 5], 'cpu').tolist() == [0, 1, 3, 4]


def test_switches_default_to_the_reference_and_config_keys_win():
    from align_anything_b200.ops import DpoObjective
    from align_anything_b200.trainers.text_audio_to_text.dpo import DPOTrainer as A
    from align_anything_b200.trainers.text_to_text import dpo as D
    from align_anything_b200.trainers.text_video_to_text.dpo import DPOTrainer as V

    for cls in (D.DPOTrainer, A, V):
        assert (cls.loss_type, cls.label_smoothing, cls.rpo_alpha, cls.reference_free) == (None,) * 4
    tr = D.DPOTrainer(None, None, None, None)
    assert D.dpo_objective_of(tr) is None
    tr.loss_type, tr.rpo_alpha = 'ipo', 0.5
    assert D.dpo_objective_of(tr) == DpoObjective(loss_type='ipo', rpo_alpha=0.5)
    tc = types.SimpleNamespace(loss_type='robust', label_smoothing=0.1, rpo_alpha=None, reference_free=None)
    tr = A(types.SimpleNamespace(train_cfgs=tc), None, None, None)
    tr.loss_type = 'hinge'  # the recipe's value wins over the attribute
    assert D.dpo_objective_of(tr) == DpoObjective(loss_type='robust', label_smoothing=0.1)
    tc.loss_type = 'hinge'
    with pytest.raises(ValueError):  # label smoothing with hinge
        D.dpo_objective_of(tr)


_DPO_MODULES = {
    'align_anything.trainers.text_to_text.dpo': 'DPOTrainer',
    'align_anything.trainers.text_image_to_text.dpo': 'DPOTrainer',
    'align_anything.trainers.text_audio_to_text.dpo': 'DPOTrainer',
    'align_anything.trainers.text_video_to_text.dpo': 'DPOTrainer',
}
_KEYS = ('loss_type', 'label_smoothing', 'rpo_alpha', 'reference_free')


@pytest.fixture
def fake_dpo_reference(monkeypatch):
    """Just enough of an importable `align_anything` for patch.install(): the tools module and the four DPO classes."""
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
    for modname, clsname in _DPO_MODULES.items():
        cls = type(clsname, (), {'loss': lambda self: 'reference', 'train_step': lambda self: 'reference',
                                 'compute_log_probs': lambda self: 'reference'})
        mod(modname, **{clsname: cls})
        classes[modname] = cls
    return classes


def test_install_sets_and_uninstall_restores_the_dpo_switches(fake_dpo_reference):
    from align_anything_b200 import patch
    from align_anything_b200.trainers.text_to_text.dpo import DPOTrainer

    try:
        patch.install(models=False)
        for modname, cls in fake_dpo_reference.items():
            for k in _KEYS:
                assert k in cls.__dict__ and cls.__dict__[k] is None, (modname, k)
            assert cls.loss is DPOTrainer.loss
    finally:
        patch.uninstall()
    for modname, cls in fake_dpo_reference.items():
        for k in _KEYS:
            assert k not in cls.__dict__, (modname, k)
        assert cls.loss(None) == 'reference'


def test_simpo_orpo_kto_keep_their_own_loss():
    from align_anything_b200.trainers.text_to_text.dpo import DPOTrainer
    from align_anything_b200.trainers.text_to_text.kto import KTOTrainer
    from align_anything_b200.trainers.text_to_text.orpo import ORPOTrainer
    from align_anything_b200.trainers.text_to_text.simpo import SimPOTrainer

    for cls in (SimPOTrainer, ORPOTrainer, KTOTrainer):
        assert cls.loss is not DPOTrainer.loss and cls.train_step is not DPOTrainer.train_step


def test_entry_point_checks_its_arguments_before_cuda():
    from align_anything_b200 import _lib

    lib = _lib.lib()
    buf = (ctypes.c_int64 * 64)()
    ptr = ctypes.cast(buf, ctypes.c_void_p)

    def call(loss_type=0, eps=0.0, alpha=0.0, counts=ptr, beta=0.1, dtype=0, mode=0, grad_seg=ptr, n_pairs=2):
        return lib.aa_dpo_loss_obj(ptr, ptr, dtype, n_pairs, 4, 4, beta, mode, loss_type, eps, alpha, counts, None, 0, 0,
                                   ptr, grad_seg, ptr, ptr, None, None)

    cases = [
        (dict(loss_type=8), b'bad objective: loss_type'), (dict(loss_type=-1), b'bad objective: loss_type'),
        (dict(eps=0.5), b'label_smoothing'), (dict(eps=-0.1), b'label_smoothing'), (dict(eps=float('nan')), b'label_smoothing'),
        (dict(loss_type=2, eps=0.1), b'label_smoothing'), (dict(loss_type=3, eps=0.1), b'label_smoothing'),
        (dict(alpha=-1.0), b'rpo_alpha'), (dict(alpha=float('inf')), b'rpo_alpha'), (dict(alpha=float('nan')), b'rpo_alpha'),
        (dict(loss_type=3, counts=None), b'needs the row counts'), (dict(alpha=0.5, counts=None), b'needs the row counts'),
        (dict(loss_type=3, beta=0.0), b'needs scale_coeff > 0'), (dict(loss_type=4, beta=-0.1), b'needs scale_coeff > 0'),
        (dict(dtype=5), b'bad dtype'), (dict(mode=3), b'bad mode'), (dict(grad_seg=None), b'null pointer'),
        (dict(n_pairs=0), b'bad sizes'),
    ]
    for kw, msg in cases:
        rc = call(**kw)
        assert rc in (-1, -2), kw
        err = lib.aa_last_error()
        assert err.startswith(b'aa_dpo_loss_obj') and msg in err, (kw, err)


# ---- dry run of train_step on the stand-in library ----------------------------------------------------------------
class _Eng:
    def __init__(self, logits, hidden, weight, calls):
        self.module = self
        self.o = SimpleNamespace(logits=logits, hidden_states=(hidden,))
        self.w = weight
        self.calls = calls
        self.optimizer = SimpleNamespace(param_groups=[{'lr': 1e-6}])

    def __call__(self, **kw):
        self.calls.append('forward')
        return self.o

    def get_output_embeddings(self):
        return SimpleNamespace(weight=self.w)

    def backward(self, loss):
        loss.backward()

    def step(self):
        pass


@pytest.mark.parametrize('objective', ['default', 'ipo-rpo', 'reference_free', 'robust-cfg'])
@pytest.mark.parametrize('fused_head', [False, True])
@pytest.mark.parametrize('modality', ['text', 'image', 'audio', 'video'])
def test_dpo_train_step_dry_run(dry, modality, fused_head, objective):  # noqa: F811
    from align_anything_b200.trainers.text_audio_to_text.dpo import DPOTrainer as A
    from align_anything_b200.trainers.text_image_to_text.dpo import DPOTrainer as I
    from align_anything_b200.trainers.text_to_text.dpo import DPOTrainer as T
    from align_anything_b200.trainers.text_video_to_text.dpo import DPOTrainer as Vd

    cls = {'text': T, 'image': I, 'audio': A, 'video': Vd}[modality]
    V, H, L_, B = 101, 64, 12, 2
    ids = torch.randint(2, V - 1, (2 * B, L_))
    lens = [5, 7, 4, 6]
    leaf = torch.randn(2 * B, L_, V).bfloat16().requires_grad_(True)
    ref = torch.randn(2 * B, L_, V).bfloat16()
    hid = torch.randn(2 * B, L_, H).bfloat16().requires_grad_(True)
    w = torch.randn(V, H).bfloat16().requires_grad_(True)
    pol_calls, ref_calls = [], []
    tc = SimpleNamespace(scale_coeff=0.1)
    if objective == 'robust-cfg':
        tc.loss_type, tc.label_smoothing = 'robust', 0.1
    tr = cls(SimpleNamespace(train_cfgs=tc), _Eng(leaf, hid, w, pol_calls), _Eng(ref, hid.detach(), w.detach(), ref_calls),
             SimpleNamespace(pad_token_id=V - 1))
    tr.fused_lm_head = fused_head
    if objective == 'ipo-rpo':
        tr.loss_type, tr.rpo_alpha = 'ipo', 1.0
    elif objective == 'reference_free':
        tr.reference_free = True
    out = tr.train_step({'input_ids': ids, 'attention_mask': ids != V - 1, 'meta_info': {'response_lens': lens}})
    keys = {'train/loss', 'train/reward', 'train/better_sample_reward', 'train/worse_sample_reward',
            'train/reward_accuracy', 'train/reward_margin', 'train/lr'}
    assert set(out) == (keys | {'train/nll_loss'} if objective == 'ipo-rpo' else keys)
    assert all(isinstance(v, float) for v in out.values())
    calls = dry.calls
    if objective == 'default':
        assert 'aa_dpo_loss' in calls and 'aa_dpo_loss_obj' not in calls
    else:
        assert calls.count('aa_dpo_loss_obj') == 1 and 'aa_dpo_loss' not in calls
    if objective == 'reference_free':
        assert ref_calls == []  # the reference engine is never called
    else:
        assert ref_calls == ['forward']
    if fused_head:
        fwd = [c for c in calls if c.startswith('aa_linear_logprob_fwd')]
        assert len(fwd) == (1 if objective == 'reference_free' else 2), calls
        assert {'aa_linear_dlogits', 'aa_linear_dhidden', 'aa_linear_dweight'} <= set(calls)
        assert hid.grad is not None and w.grad is not None
    else:
        assert calls.count('aa_logprob_fwd') == (1 if objective == 'reference_free' else 2), calls
        assert calls.count('aa_logprob_bwd') == 1
        assert leaf.grad is not None and leaf.grad.shape == leaf.shape
