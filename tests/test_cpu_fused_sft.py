"""The fused lm_head switch of the SFT trainers without a GPU:
  * the graft: patch.install() puts `fused_lm_head = False` / `lm_head_chunk_rows = None` on the reference-shaped text,
    image and audio SFT classes, lists only the grafted methods, and uninstall() takes the attributes away;
  * the refusals: with the switch on, SupervisedTrainer raises ops.lm_head_weight's error for a ZeRO-3 placeholder
    weight, a biased head and a soft-capped / logit-scaled head before the valid-row index, any model forward and any
    kernel launch;
  * the valid-row index and the row chunks of ops.causal_lm_loss_from_hidden, restated in Python;
  * a dry run (the C ABI replaced by a signature-checking stand-in, see test_cpu_plumbing) of the fused step: per chunk
    K6s -> K1b -> d(hidden) -> d(weight), no logits-tile entry point, no d(weight) launch for a frozen head."""
import contextlib
import sys
import types
from types import SimpleNamespace

import pytest
import torch

import fake_reference_tree as fake
from test_cpu_plumbing import dry  # noqa: F401  (fixture)

_SFT = ('align_anything.trainers.text_to_text.sft', 'align_anything.trainers.text_image_to_text.sft',
        'align_anything.trainers.text_audio_to_text.sft')


class _RefSupervisedTrainer:
    """Shape of trainers/text_to_text/sft.py:SupervisedTrainer: the two methods the graft replaces."""

    loss = fake._not_grafted('loss')
    train_step = fake._not_grafted('train_step')


@contextlib.contextmanager
def _tree():
    """fake_reference_tree plus the three SFT modules (the image and audio trainers subclass the text one)."""
    saved = {n: sys.modules.get(n) for n in _SFT}
    with fake.installed() as mods:
        base = None
        for n in _SFT:
            m = types.ModuleType(n)
            parent, _, child = n.rpartition('.')
            mods[n] = sys.modules[n] = m
            setattr(mods[parent], child, m)
            m.SupervisedTrainer = type('SupervisedTrainer', (base or _RefSupervisedTrainer,), {'__module__': n})
            base = base or m.SupervisedTrainer
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
        classes = [mods[n].SupervisedTrainer for n in _SFT]
        for cls in classes:
            assert 'fused_lm_head' not in cls.__dict__ and 'lm_head_chunk_rows' not in cls.__dict__
        done = patch.install()
        try:
            for n, cls in zip(_SFT, classes):
                assert cls.__dict__['fused_lm_head'] is False and cls.__dict__['lm_head_chunk_rows'] is None, cls
                assert done[n] == ['SupervisedTrainer.loss', 'SupervisedTrainer.train_step'], done[n]
            listed = [x for names in done.values() for x in names]
            assert not any('fused_lm_head' in x or 'lm_head_chunk_rows' in x for x in listed), listed
        finally:
            patch.uninstall()
        for cls in classes:
            assert 'fused_lm_head' not in cls.__dict__ and 'lm_head_chunk_rows' not in cls.__dict__, cls
            assert not hasattr(cls, 'fused_lm_head') and cls.__dict__.get('loss', cls.loss).__name__ == 'loss'


# ---- refusals before anything runs -------------------------------------------------------------------------------------
class _NoKernels:
    def __getattr__(self, name):
        raise AssertionError(f'kernel entry point {name} reached')


class _Head(torch.nn.Module):
    def __init__(self, kind):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.randn(11, 64))
        self.bias = torch.nn.Parameter(torch.zeros(11)) if kind == 'bias' else None
        if kind == 'zero3':
            self.weight.ds_id = 7  # what DeepSpeed ZeRO-3 puts on a partitioned parameter


class _CountingEngine:
    """An engine that counts its forwards; its module has one of the heads lm_head_weight refuses."""

    def __init__(self, kind):
        self.forwards = 0
        self.module = SimpleNamespace(get_output_embeddings=lambda: _Head(kind),
                                      config=SimpleNamespace(final_logit_softcapping=30.0 if kind == 'softcap' else None,
                                                             logit_scale=0.25 if kind == 'scale' else None))

    def __call__(self, *a, **k):
        self.forwards += 1
        raise AssertionError('model forward reached')


_REFUSALS = {'zero3': 'ZeRO-3', 'bias': 'bias-free', 'softcap': 'final_logit_softcapping', 'scale': 'logit_scale'}


@pytest.mark.parametrize('kind', list(_REFUSALS))
def test_refusals_come_before_the_index_any_forward_or_kernel(monkeypatch, kind):
    from align_anything_b200 import _lib, ops
    from align_anything_b200.trainers.text_to_text.sft import SupervisedTrainer

    monkeypatch.setattr(_lib, 'lib', lambda: _NoKernels())
    monkeypatch.setattr(_lib, 'require_cuda', lambda *t: None)
    index_calls = []
    monkeypatch.setattr(ops, 'causal_lm_valid_rows', lambda *a, **k: index_calls.append(a))
    eng = _CountingEngine(kind)
    tr = SupervisedTrainer(None, eng)
    tr.fused_lm_head = True
    labels = torch.randint(0, 11, (2, 6))
    with pytest.raises(RuntimeError, match=_REFUSALS[kind]):
        tr.train_step({'input_ids': labels, 'labels': labels, 'attention_mask': torch.ones_like(labels)})
    assert eng.forwards == 0 and not index_calls


# ---- the index and the chunks, restated -------------------------------------------------------------------------------
def test_valid_rows_restated():
    from align_anything_b200 import ops

    gen = torch.Generator().manual_seed(3)
    for ign in (-100, 0):
        lab = torch.randint(-1, 9, (5, 13), generator=gen)
        lab[lab == -1] = ign
        lab[2] = ign  # a sample without a valid label
        lab[3] = ign
        lab[3, 7] = 4  # a single valid row (position 6)
        idx, n = ops.causal_lm_valid_rows(lab, ign)
        want = [b * 13 + t for b in range(5) for t in range(12) if int(lab[b, t + 1]) != ign]
        assert idx.tolist() == want and n == len(want) and idx.dtype == torch.int64
        assert 3 * 13 + 6 in want and not any(2 * 13 <= r < 3 * 13 for r in want)


@pytest.mark.parametrize('N, V, chunk_rows, want', [
    (0, 2053, None, []),
    (300, 2053, 128, [128, 128, 44]),
    (257, 2053, 128, [128, 128, 1]),
    (100, 2053, None, [100]),
    (16376, 128257, None, [4096, 4096, 4096, 4088]),
    (8000, 128257, None, [4096, 3904]),
    (9000, 128257, 8192, [4608, 4392]),
])
def test_chunks_restated(N, V, chunk_rows, want):
    """Default: (1 GB // (ld * 2 bytes)) rows rounded down to 128 (4096 at V = 128257, ld = 128512: the logits and
    d(logits) buffers of a chunk take 2 x 1.05 GB); then ceil(N / chunk) equal chunks of whole 256-row tiles."""
    from align_anything_b200 import ops

    chunks = ops._ce_chunks(N, V, chunk_rows)
    assert [n for _, n in chunks] == want
    assert [r0 for r0, _ in chunks] == [sum(want[:i]) for i in range(len(want))]
    ld = (V + 255) // 256 * 256
    if chunk_rows is None and want:
        assert max(want) * ld * 2 <= 1 << 30


# ---- dry run of the fused step ----------------------------------------------------------------------------------------
class _HiddenLM:
    """A causal-LM-shaped engine that hands out fixed last hidden states; its forward must be asked for them."""

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


_FUSED_ORDER = ('aa_linear_logits', 'aa_logprob_bwd', 'aa_linear_dhidden', 'aa_linear_dweight')
_NOT_HERE = {'aa_logprob_fwd', 'aa_logprob_ce_fused', 'aa_linear_logprob_fwd', 'aa_linear_dlogits'}


@pytest.mark.parametrize('frozen_head', [False, True])
def test_fused_sft_dry_run(dry, frozen_head):
    from align_anything_b200.trainers.text_to_text.sft import SupervisedTrainer

    B, Lq, H, V = 3, 6, 64, 97
    labels = torch.randint(0, V, (B, Lq))
    labels[0, :2] = -100
    labels[2, 4:] = -100  # N = 4 + 5 + 3 = 12 rows: chunks of 4
    hid = torch.randn(B, Lq, H).bfloat16().requires_grad_(True)
    w = torch.randn(V, H).bfloat16().requires_grad_(not frozen_head)
    eng = _HiddenLM(hid, w)
    tr = SupervisedTrainer(None, eng)
    tr.fused_lm_head, tr.lm_head_chunk_rows = True, 4
    out = tr.train_step({'input_ids': labels.clamp(min=0), 'labels': labels, 'attention_mask': torch.ones_like(labels)})
    assert set(out) == {'train/loss', 'train/lr'} and isinstance(out['train/loss'], float)
    assert eng.calls == [['attention_mask', 'input_ids']]
    seq = [c for c in dry.calls if c in _FUSED_ORDER]
    per_chunk = [c for c in _FUSED_ORDER if not (frozen_head and c == 'aa_linear_dweight')]
    assert seq == per_chunk * 3, dry.calls
    assert not (_NOT_HERE & set(dry.calls)), dry.calls
    assert dry.calls.count('aa_nll_mean') == 1 and dry.calls.index('aa_nll_mean') > dry.calls.index(seq[-1])
    assert dry.calls.count('aa_scale_tile') == (1 if frozen_head else 2)  # the backward: one per gradient
    assert hid.grad is not None and hid.grad.shape == hid.shape
    assert (w.grad is None) == frozen_head


def test_no_grad_loss_launches_no_gradient_work(dry):
    """SupervisedTrainer.loss under torch.no_grad (the reference's eval) with a Parameter head and hidden states that
    require a gradient: K6s and the loss only -- needs_input_grad follows requires_grad, not the grad mode."""
    from align_anything_b200.trainers.text_to_text.sft import SupervisedTrainer

    B, Lq, H, V = 3, 6, 64, 97
    labels = torch.randint(0, V, (B, Lq))
    hid = torch.randn(B, Lq, H).bfloat16().requires_grad_(True)
    w = torch.nn.Parameter(torch.randn(V, H).bfloat16())
    tr = SupervisedTrainer(None, _HiddenLM(hid, w))
    tr.fused_lm_head, tr.lm_head_chunk_rows = True, 4
    with torch.no_grad():
        loss = tr.loss({'input_ids': labels, 'labels': labels, 'attention_mask': torch.ones_like(labels)})['loss']
    assert not loss.requires_grad
    assert dry.calls == ['aa_linear_logits'] * 4 + ['aa_nll_mean'], dry.calls
