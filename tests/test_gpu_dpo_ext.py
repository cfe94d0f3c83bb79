"""The further DPO objectives on an H100 (`pytest -m gpu`): aa_dpo_loss_ext on guarded buffers against the port
(tests/dpo_ext_port.py) for every new type, f-divergence, reference-free and skipped-pair case, the default new fields
against aa_dpo_loss_obj, the gradient tile of dpo_fused_loss against float64 autograd, the fused lm_head node against
the tile path, and train_step of the text, image and audio trainers against float64.

Operands.  The log-probs are multiples of 1/8 in [-8, 0]: every partial sum of a row is exact in fp32, so the four
sequence sums are the same in K2 and in ATen whatever the order, and what is compared is the objective's arithmetic.
FAITHFUL against the port on ATen CUDA: within 1 ulp and >= 97 % bit-identical; F32 against the port in float64: 2e-5
(DESIGN section 4.3)."""
import math

import pytest
import torch

from align_anything_b200 import _lib as Lb
from dpo_ext_port import dpo_loss as port_loss
from dpo_ext_port import exp_cap
from oracle import ref_port as O
from test_gpu_loss_kernels import Guarded, Words, _p, _stream, assert_same, fenced, rc_ok
from test_gpu_parity import assert_close_f32, assert_ulp_close, ops  # noqa: F401

DEV = 'cuda'
gpu = pytest.mark.gpu
BF, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
CODE = {BF: Lb.AA_BF16, F16: Lb.AA_F16, F32: Lb.AA_F32}
TYPES = {'sigmoid': 0, 'robust': 1, 'hinge': 2, 'ipo': 3, 'sppo_hard': 4, 'nca_pair': 5, 'apo_zero': 6, 'apo_down': 7,
         'exo_pair': 8, 'discopop': 9, 'aot': 10, 'aot_pair': 11}
FDIV = {'reverse_kl': 0, 'js_divergence': 1, 'alpha_divergence': 2}
BETA = 0.1
B, W, L_IDS = 96, 31, 9


def _operands(seed, ties=False, nb=B):
    g = torch.Generator().manual_seed(seed)
    pol = -torch.randint(0, 65, (2 * nb, W), generator=g).double() / 8
    ref = -torch.randint(0, 65, (2 * nb, W), generator=g).double() / 8
    lens = torch.randint(2, W + 2, (2 * nb,), generator=g)
    ids = torch.randint(0, 1000, (2 * nb, L_IDS), generator=g)
    same = torch.rand(nb, generator=g) < 0.2
    ids[nb:][same] = ids[:nb][same]
    if ties:  # every fourth pair repeats pair 0's chosen rows: equal keys, ordered by the pair index alone
        pol[4:nb:4], ref[4:nb:4] = pol[0], ref[0]
    return pol, ref, lens, ids


def _launch(pol, ref, dt, mode, opt, counts, ids, stride, fn='aa_dpo_loss_ext'):
    loss_type, eps, alpha, fdiv, coef, tau = opt
    nb = pol.size(0) // 2
    per_pair, grad_seg = Guarded(5, nb, F32), Guarded(1, 2 * nb, F32)
    stats = Guarded(1, 9 if alpha > 0 else 8, F32)
    counter, status = Words(), Words(value=6)
    head = (_p(pol), Lb.ptr(ref), CODE[dt], nb, W, stride, BETA, mode, TYPES[loss_type], eps, alpha)
    tail = (Lb.ptr(counts), Lb.ptr(ids), L_IDS, L_IDS + 3 if ids is not None else 0, per_pair.ptr(), grad_seg.ptr(),
            stats.ptr(), counter.ptr(), status.ptr(), _stream())
    if fn == 'aa_dpo_loss_ext':
        e = eps or 1e-3  # EXO's constants, formed in double as ops forms them
        rc_ok(Lb.lib().aa_dpo_loss_ext(*head, FDIV[fdiv], coef, tau, math.log(1 - e), math.log(e), *tail), fn)
    else:
        rc_ok(Lb.lib().aa_dpo_loss_obj(*head, *tail), fn)
    torch.cuda.synchronize()
    for buf, what in ((per_pair, 'per_pair'), (grad_seg, 'grad_seg'), (stats, 'stats')):
        buf.check(what)
    counter.check([0], 'counter')
    status.check([6], 'status')
    assert float(stats.t[0, 7]) == 6.0
    return per_pair.t, grad_seg.t[0], stats.t[0]


# (loss_type, label_smoothing, rpo_alpha, f_divergence_type, f_alpha_divergence_coef, discopop_tau).  The alpha
# divergence's clamp holds for some pairs of these operands; a coefficient >= 1 keeps its h finite in fp32.
OPTS = [('sigmoid', 0.0, 0.0, 'js_divergence', 1.0, 0.05), ('robust', 0.25, 0.5, 'js_divergence', 1.0, 0.05),
        ('hinge', 0.0, 0.0, 'js_divergence', 1.0, 0.05), ('sigmoid', 0.0, 0.5, 'alpha_divergence', 1.0, 0.05),
        ('robust', 0.125, 0.0, 'alpha_divergence', 1.5, 0.05), ('hinge', 0.0, 0.0, 'alpha_divergence', 2.0, 0.05),
        ('exo_pair', 0.0, 0.0, 'reverse_kl', 1.0, 0.05), ('exo_pair', 0.25, 0.5, 'reverse_kl', 1.0, 0.05),
        ('exo_pair', 0.1, 0.0, 'reverse_kl', 1.0, 0.05),  # 0.1 has no exact fp32 copy: EXO's constants from the double
        ('exo_pair', 0.0, 0.0, 'js_divergence', 1.0, 0.05), ('exo_pair', 0.125, 0.0, 'alpha_divergence', 1.5, 0.05),
        ('discopop', 0.0, 0.0, 'reverse_kl', 1.0, 0.05), ('discopop', 0.0, 1.0, 'reverse_kl', 1.0, 0.5),
        ('aot', 0.0, 0.0, 'reverse_kl', 1.0, 0.05), ('aot', 0.25, 0.5, 'reverse_kl', 1.0, 0.05),
        ('aot_pair', 0.0, 0.0, 'reverse_kl', 1.0, 0.05), ('aot_pair', 0.125, 1.0, 'reverse_kl', 1.0, 0.05)]
CASES = [o + (rf, skip) for o in OPTS for rf, skip in ((False, False), (True, True), (False, True))]


@gpu
@pytest.mark.parametrize('case', CASES, ids=lambda c: '-'.join(map(str, c)))
def test_dpo_loss_ext_against_the_port(ops, case):
    loss_type, eps, alpha, fdiv, coef, tau, ref_free, skip = case
    opt = case[:6]
    seed = sum(map(ord, loss_type + fdiv)) + int(100 * eps + 10 * alpha) + ref_free + 2 * skip
    pol64, ref64, lens, ids64 = _operands(seed, ties=loss_type.startswith('aot'))
    counts = fenced((lens - 1).to(torch.int32).reshape(1, -1), pad=-7)[0]
    kw = dict(loss_type=loss_type, label_smoothing=eps, rpo_alpha=alpha, reference_free=ref_free,
              response_lens=lens.tolist(), f_divergence_type=fdiv, f_alpha_divergence_coef=coef, discopop_tau=tau)
    keep = ~(ids64[:B] == ids64[B:]).all(1) if skip else torch.ones(B, dtype=torch.bool)
    for dt in (BF, F16, F32):
        stride = W + 5
        pol, ref = fenced(pol64.to(dt), stride), fenced(ref64.to(dt), stride)
        ids = fenced(ids64, L_IDS + 3) if skip else None
        for mode in (Lb.MODE_FAITHFUL, Lb.MODE_F32):
            what = f'{case} {dt} mode={mode}'
            pp, gs, st = _launch(pol, None if ref_free else ref, dt, mode, opt, counts, ids, stride)
            pdt = dt if mode == Lb.MODE_FAITHFUL else F64
            leaf = pol64.to(DEV).to(pdt).requires_grad_(True)
            want = port_loss(leaf, ref64.to(DEV).to(pdt), BETA, ids64.to(DEV), skip, cap=exp_cap(dt), **kw)
            want['loss'].backward()
            gwant = leaf.grad[:, 0]
            cmp_dt = dt if mode == Lb.MODE_FAITHFUL else F32

            def close(got, w, what_, min_exact=0.97):
                assert_ulp_close(got.to(cmp_dt), w.detach().to(cmp_dt), max_ulp=1, min_exact=min_exact, what=what_)

            close(st[:1], want['loss'].reshape(1), what + ' loss', 0.0)
            close(gs, gwant, what + ' grad_seg')
            close(pp[3], gwant[:B], what + ' per_pair g')
            k = keep.to(DEV)
            close(pp[1][k], want['better_sample_reward'], what + ' better')
            close(pp[2][k], want['worse_sample_reward'], what + ' worse')
            assert_same(pp[4].bool(), k, what + ' valid')
            assert float(st[6]) == float(keep.sum())
            close(st[1:4], torch.stack([want['reward'].mean(), want['better_sample_reward'].mean(),
                                        want['worse_sample_reward'].mean()]), what + ' metric means', 0.0)
            assert float(st[4]) == pytest.approx(float(want['reward_accuracy']), abs=1e-6)
            if alpha > 0:
                close(st[8:9], want['nll_loss'].reshape(1), what + ' nll', 0.0)


@gpu
@pytest.mark.parametrize('nb', [300, 1024])
@pytest.mark.parametrize('loss_type', ['aot', 'aot_pair'])
def test_aot_sort_over_many_pairs_against_the_port(ops, loss_type, nb):
    """More pairs than the last block has threads (several passes of each strided loop), up to AA_DPO_AOT_MAX_PAIRS."""
    pol64, ref64, lens, ids64 = _operands(nb, ties=True, nb=nb)
    keep = ~(ids64[:nb] == ids64[nb:]).all(1)
    opt = (loss_type, 0.125, 0.5, 'reverse_kl', 1.0, 0.05)
    counts = (lens - 1).to(torch.int32).to(DEV)
    for dt, mode in ((BF, Lb.MODE_FAITHFUL), (F32, Lb.MODE_F32)):
        pol, ref = fenced(pol64.to(dt), W), fenced(ref64.to(dt), W)
        pp, gs, st = _launch(pol, ref, dt, mode, opt, counts, fenced(ids64, L_IDS + 3), W)
        pdt = dt if mode == Lb.MODE_FAITHFUL else F64
        leaf = pol64.to(DEV).to(pdt).requires_grad_(True)
        want = port_loss(leaf, ref64.to(DEV).to(pdt), BETA, ids64.to(DEV), True, loss_type=loss_type,
                         label_smoothing=0.125, rpo_alpha=0.5, response_lens=lens.tolist())
        want['loss'].backward()
        gwant = leaf.grad[:, 0]
        what = f'{loss_type} nb={nb} {dt}'
        assert float(st[6]) == float(keep.sum())
        assert_ulp_close(st[:1].to(dt), want['loss'].detach().reshape(1).to(dt), max_ulp=1, min_exact=0.0,
                         what=what + ' loss')
        assert_ulp_close(gs.to(dt), gwant.to(dt), max_ulp=1, min_exact=0.97, what=what + ' grad_seg')


@gpu
@pytest.mark.parametrize('loss_type', list(TYPES)[:8])
def test_default_new_fields_are_aa_dpo_loss_obj_bit_for_bit(ops, loss_type):
    pol64, ref64, lens, ids64 = _operands(11)
    pol64 = pol64 + torch.rand(pol64.shape, generator=torch.Generator().manual_seed(3)).double() / 3  # inexact sums too
    counts = (lens - 1).to(torch.int32).to(DEV)
    eps = 0.1 if loss_type in ('sigmoid', 'robust') else 0.0
    for dt in (BF, F16, F32):
        pol, ref = fenced(pol64.to(dt), W), fenced(ref64.to(dt), W)
        for skip in (False, True):
            ids = fenced(ids64, L_IDS + 3) if skip else None
            for mode in (Lb.MODE_FAITHFUL, Lb.MODE_F32):
                opt = (loss_type, eps, 0.5, 'reverse_kl', 1.0, 0.05)
                a = _launch(pol, ref, dt, mode, opt, counts, ids, W)
                b = _launch(pol, ref, dt, mode, opt, counts, ids, W, fn='aa_dpo_loss_obj')
                for x, y, what in zip(a, b, ('per_pair', 'grad_seg', 'stats')):
                    assert torch.equal(x.view(torch.int32), y.view(torch.int32)), f'{loss_type} {dt} {mode} {skip} {what}'


# ---- the nodes ---------------------------------------------------------------------------------------------------
def _f64_tile(logits, ref_logits, ids, lens, pad, obj, strip=True, skip=False, cap=None):
    leaf = logits.detach().double().requires_grad_(True)
    lp = O.dpo_sequence_log_probs(leaf, ids, lens, pad, strip)
    rlp = O.dpo_sequence_log_probs(ref_logits.double(), ids, lens, pad, strip)
    out = port_loss(lp, rlp, BETA, ids, skip, obj.loss_type, obj.label_smoothing, obj.rpo_alpha, obj.reference_free, lens,
                    obj.f_divergence_type, obj.f_alpha_divergence_coef, obj.discopop_tau, cap)
    out['loss'].backward()
    return out, leaf.grad


def _near(got, want, what, rtol=1e-4):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    tol = rtol * want.abs() + 1e-6 * float(want.abs().max())
    bad = (got - want).abs() > tol
    assert not bool(bad.any()), f'{what}: {int(bad.sum())} beyond the bar, max err {float((got - want).abs().max()):.3e}'


@gpu
@pytest.mark.parametrize('obj_kw', [dict(f_divergence_type='js_divergence', rpo_alpha=1.0), dict(loss_type='aot'),
                                    dict(f_divergence_type='alpha_divergence', f_alpha_divergence_coef=2.0)], ids=str)
def test_fused_loss_gradient_tile_against_float64(ops, obj_kw):
    obj = ops.DpoObjective(**obj_kw)
    V, L_, pad = 128257, 24, 0
    g = torch.Generator().manual_seed(17)
    logits = (torch.randn(8, L_, V, generator=g) * 2).float()
    ref_logits = (torch.randn(8, L_, V, generator=g) * 2).float()
    ids = torch.randint(1, V, (8, L_), generator=g)
    ids[0, :3] = pad
    lens = [9, 17, 12, 20, 15, 7, 22, 11]
    want, gwant = _f64_tile(logits, ref_logits, ids, lens, pad, obj, cap=exp_cap(F32))
    leaf = logits.to(DEV).requires_grad_(True)
    out = ops.dpo_fused_loss(leaf, None if obj.reference_free else ref_logits.to(DEV), ids.to(DEV), lens, pad, BETA,
                             mode='f32', objective=obj)
    out['loss'].backward()
    _near(out['loss'].reshape(1), want['loss'].reshape(1), f'{obj} loss')
    _near(leaf.grad, gwant, f'{obj} d logits')
    if obj.rpo_alpha > 0:
        _near(out['nll_loss'].reshape(1), want['nll_loss'].reshape(1), f'{obj} nll')


@gpu
@pytest.mark.parametrize('obj_kw', [dict(loss_type='exo_pair', f_divergence_type='js_divergence', rpo_alpha=0.5),
                                    dict(loss_type='aot_pair', reference_free=True)], ids=str)
def test_fused_lm_head_node_against_the_tile_path(ops, obj_kw):
    obj = ops.DpoObjective(**obj_kw)
    V, H, L_, pad = 4096, 128, 20, 0
    g = torch.Generator().manual_seed(23)
    hid = (torch.randn(4, L_, H, generator=g) / 4).bfloat16().to(DEV)
    w = (torch.randn(V, H, generator=g) / 4).bfloat16().to(DEV)
    ref_hid = (hid.float() + torch.randn(4, L_, H, generator=g).to(DEV) / 20).bfloat16()
    ids = torch.randint(1, V, (4, L_), generator=g).to(DEV)
    lens = [8, 15, 11, 19]
    h1 = hid.clone().requires_grad_(True)
    lp = ops.sequence_log_probs_from_hidden(h1, w, ids, lens, pad)
    rlp = None if obj.reference_free else ops.sequence_log_probs_from_hidden(ref_hid, w, ids, lens, pad)
    a = ops.dpo_loss_from_log_probs(lp, rlp, BETA, objective=obj, response_lens=lens)
    a['loss'].backward()
    h2 = hid.clone().requires_grad_(True)
    b = ops.dpo_fused_loss(h2 @ w.t(), None if obj.reference_free else ref_hid @ w.t(), ids, lens, pad, BETA,
                           objective=obj)
    b['loss'].backward()
    assert abs(float(a['loss']) - float(b['loss'])) <= 2e-2 * max(1.0, abs(float(b['loss'])))
    for k in ('better_sample_reward', 'worse_sample_reward'):
        assert torch.allclose(a[k].float(), b[k].float(), rtol=2e-2, atol=2e-2), k
    err = (h1.grad.float() - h2.grad.float()).norm() / h2.grad.float().norm().clamp(min=1e-30)
    assert float(err) <= 3e-2, float(err)


@gpu
@pytest.mark.parametrize('modality', ['text', 'image', 'audio'])
def test_train_step_with_one_option_against_float64(ops, modality):
    from types import SimpleNamespace

    from align_anything_b200.trainers.text_audio_to_text.dpo import DPOTrainer as A
    from align_anything_b200.trainers.text_image_to_text.dpo import DPOTrainer as I
    from align_anything_b200.trainers.text_to_text.dpo import DPOTrainer as T

    cls, opt = {'text': (T, dict(loss_type='aot_pair', label_smoothing=0.1)),
                'image': (I, dict(f_divergence_type='js_divergence')),
                'audio': (A, dict(loss_type='discopop', discopop_tau=0.1))}[modality]
    V, L_, pad = 32003, 16, 32002
    g = torch.Generator().manual_seed(29)
    logits = torch.randn(6, L_, V, generator=g)
    ref_logits = torch.randn(6, L_, V, generator=g)
    ids = torch.randint(0, V - 1, (6, L_), generator=g)
    ids[4] = ids[1]  # pair 1 is identical: the audio trainer drops it from the loss
    lens = [7, 12, 9, 10, 12, 5]
    leaf = logits.to(DEV).requires_grad_(True)

    class Eng:
        def __init__(self, x):
            self.module = self
            self.x = x
            self.optimizer = SimpleNamespace(param_groups=[{'lr': 1e-6}])

        def __call__(self, **kw):
            return SimpleNamespace(logits=self.x)

        def backward(self, loss):
            loss.backward()

        def step(self):
            pass

    tr = cls(SimpleNamespace(train_cfgs=SimpleNamespace(scale_coeff=BETA, **opt)), Eng(leaf), Eng(ref_logits.to(DEV)),
             SimpleNamespace(pad_token_id=pad))
    tr.mode = 'f32'
    out = tr.train_step({'input_ids': ids.to(DEV), 'meta_info': {'response_lens': lens}})
    obj = ops.DpoObjective(**opt)
    want, gwant = _f64_tile(logits, ref_logits, ids, lens, pad, obj, strip=modality != 'audio', skip=modality == 'audio',
                            cap=exp_cap(F32))
    assert out['train/loss'] == pytest.approx(float(want['loss']), rel=1e-4, abs=1e-6)
    assert out['train/better_sample_reward'] == pytest.approx(float(want['better_sample_reward'].mean()), rel=1e-4, abs=1e-6)
    assert 'train/nll_loss' not in out
    _near(leaf.grad, gwant, f'{modality} d logits')
