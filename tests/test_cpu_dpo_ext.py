"""The further DPO objectives (f-divergences, exo_pair, discopop, aot, aot_pair) without a GPU: the port
(tests/dpo_ext_port.py) against float64 autograd, ops.DpoObjective's new checks, the new switches and their config
precedence, their graft, the argument checks of aa_dpo_loss_ext, and which entry points a train_step calls on the CPU
stand-in library for every modality and head path."""
from __future__ import annotations

import ctypes
import math
import types
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from dpo_ext_port import dpo_loss as port_loss
from dpo_ext_port import exp_cap
from dpo_objective_port import dpo_loss as objective_loss
from oracle import ref_port
from test_cpu_dpo_objective import _Eng, _grad, _inputs, fake_dpo_reference  # noqa: F401  (fixture)
from test_cpu_plumbing import dry  # noqa: F401  (fixture)

NEW_KEYS = ('f_divergence_type', 'f_alpha_divergence_coef', 'discopop_tau')


def _sorted(v: torch.Tensor) -> torch.Tensor:
    """v sorted ascending by (NaN last, value, index): the stable order, written without torch.sort."""
    x = v.detach().tolist()
    order = sorted(range(len(x)), key=lambda j: (math.isnan(x[j]), 0.0 if math.isnan(x[j]) else x[j], j))
    return v[torch.tensor(order, dtype=torch.long)]


def _f64(pol, ref, beta, keep, lens, opt, cap):
    """The objective in float64 autograd, vectorised over the pairs and written independently of the port."""
    loss_type, eps, alpha, ref_free, fdiv, coef, tau = opt
    x = pol.double().clone().requires_grad_(True)
    B = x.size(0) // 2
    s = x.sum(1)
    r = torch.zeros_like(s) if ref_free else ref.double().sum(1)
    a, b = (s[:B] - r[:B])[keep], (s[B:] - r[B:])[keep]
    ls, sg = F.logsigmoid, torch.sigmoid
    if loss_type in ('aot', 'aot_pair'):
        k1, k2 = (a, b) if loss_type == 'aot_pair' else ((s[:B] - s[B:])[keep], (r[:B] - r[B:])[keep])
        z = beta * (_sorted(k1) - _sorted(k2))
        per = -(1 - eps) * ls(z) - eps * ls(-z)
    else:
        if fdiv == 'js_divergence':
            h = (a - b) - (F.softplus(a) - F.softplus(b))
        elif fdiv == 'alpha_divergence':
            h = (torch.exp((-coef * b).clamp(max=cap)) - torch.exp((-coef * a).clamp(max=cap))) / coef
        else:
            h = a - b
        z = beta * h
        e = eps if eps > 0 else 1e-3
        per = {
            'sigmoid': lambda: -(1 - eps) * ls(z) - eps * ls(-z),
            'robust': lambda: (-(1 - eps) * ls(z) + eps * ls(-z)) / (1 - 2 * eps),
            'hinge': lambda: torch.relu(1 - z),
            'exo_pair': lambda: sg(z) * (ls(z) - math.log(1 - e)) + sg(-z) * (ls(-z) - math.log(e)),
            'discopop': lambda: -ls(z) * (1 - sg(z / tau)) + torch.exp(-z) * sg(z / tau),
        }[loss_type]()
    loss = per.mean()
    if alpha > 0:
        n = torch.tensor(lens, dtype=torch.float64) - 1
        loss = loss + alpha * (-x.sum(1)[:B][keep].sum() / n[:B][keep].sum())
    loss.backward()
    return loss.detach(), x.grad


# (loss_type, label_smoothing, rpo_alpha, reference_free, f_divergence_type, f_alpha_divergence_coef, discopop_tau)
OPTIONS = [
    ('sigmoid', 0.0, 0.0, False, 'js_divergence', 1.0, 0.05), ('robust', 0.2, 0.0, False, 'js_divergence', 1.0, 0.05),
    ('hinge', 0.0, 0.5, False, 'alpha_divergence', 0.5, 0.05), ('sigmoid', 0.1, 0.0, True, 'alpha_divergence', 1.0, 0.05),
    ('exo_pair', 0.0, 0.0, False, 'reverse_kl', 1.0, 0.05), ('exo_pair', 0.25, 1.0, False, 'js_divergence', 1.0, 0.05),
    ('exo_pair', 0.1, 0.0, True, 'alpha_divergence', 2.0, 0.05), ('discopop', 0.0, 0.0, False, 'reverse_kl', 1.0, 0.05),
    ('discopop', 0.0, 0.5, True, 'reverse_kl', 1.0, 0.3), ('aot', 0.0, 0.0, False, 'reverse_kl', 1.0, 0.05),
    ('aot', 0.2, 1.0, True, 'reverse_kl', 1.0, 0.05), ('aot_pair', 0.0, 0.0, False, 'reverse_kl', 1.0, 0.05),
    ('aot_pair', 0.1, 0.5, True, 'reverse_kl', 1.0, 0.05),
]


def _kw(opt, lens):
    loss_type, eps, alpha, ref_free, fdiv, coef, tau = opt
    return dict(loss_type=loss_type, label_smoothing=eps, rpo_alpha=alpha, reference_free=ref_free, response_lens=lens,
                f_divergence_type=fdiv, f_alpha_divergence_coef=coef, discopop_tau=tau)


@pytest.mark.parametrize('ties', [False, True])
@pytest.mark.parametrize('skip', [False, True])
@pytest.mark.parametrize('opt', OPTIONS, ids=lambda o: '-'.join(map(str, o)))
def test_port_matches_float64_autograd(opt, skip, ties):
    pol, ref, ids, lens = _inputs(B=6, W=17, dtype=torch.float64, seed=3)
    if ties:  # pairs 2, 3 and 5 share every ratio and key (exact in float64): only the pair index orders them
        for i in (3, 5):
            for r in (i, 6 + i):
                pol[r], ref[r], lens[r] = pol[r - i + 2], ref[r - i + 2], lens[r - i + 2]
    keep = torch.ones(6, dtype=torch.bool)
    if skip:
        keep[1] = False
    cap = 1.5 if opt[4] == 'alpha_divergence' else exp_cap(torch.float64)  # a low cap: the clamp holds for some pairs
    got, ggot = _grad(port_loss, pol, ref, 0.1, ids, skip, **_kw(opt, lens), cap=cap)
    want, gwant = _f64(pol, ref, 0.1, keep, lens, opt, cap)
    torch.testing.assert_close(got['loss'], want, rtol=1e-12, atol=1e-14)
    mask = pol != 0  # the padding carries no gradient in the trainers (the log-prob kernels never write it)
    torch.testing.assert_close(ggot * mask, gwant * mask, rtol=1e-12, atol=1e-14)
    # the metrics keep the reference's definitions (unsorted, unweighted ratios) whatever the objective
    base = ref_port.dpo_loss(pol, torch.zeros_like(ref) if opt[3] else ref, 0.1, ids, skip)
    for k in ('reward', 'better_sample_reward', 'worse_sample_reward', 'reward_accuracy', 'reward_margin'):
        assert torch.equal(got[k], base[k]), k


def test_alpha_divergence_clamp_stops_the_gradient():
    pol, ref, ids, lens = _inputs(B=4, W=9, dtype=torch.float64, seed=5)
    opt = ('sigmoid', 0.0, 0.0, True, 'alpha_divergence', 1.0, 0.05)
    _, g = _grad(port_loss, pol, ref, 0.1, **_kw(opt, lens), cap=-1e9)  # every exponent clamped: no gradient at all
    assert torch.count_nonzero(g) == 0


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
def test_default_new_fields_are_the_objective_port(dtype):
    pol, ref, ids, lens = _inputs(dtype=dtype)
    for kw in (dict(), dict(loss_type='ipo', rpo_alpha=0.5), dict(loss_type='robust', label_smoothing=0.1)):
        a, ga = _grad(port_loss, pol, ref, 0.1, ids, True, response_lens=lens, **kw)
        b, gb = _grad(objective_loss, pol, ref, 0.1, ids, True, response_lens=lens, **kw)
        assert all(torch.equal(a[k], b[k]) for k in b) and torch.equal(ga, gb)


def test_exp_cap_is_trls():
    assert exp_cap(torch.bfloat16) == 88.7189 and exp_cap(torch.float32) == 88.7228
    assert exp_cap(torch.float16) == 11.0898


def test_dpo_objective_checks_its_new_fields():
    from align_anything_b200.ops import DpoObjective

    d = DpoObjective()
    assert (d.f_divergence_type, d.f_alpha_divergence_coef, d.discopop_tau) == ('reverse_kl', 1.0, 0.05)
    assert d.is_default and not d.needs_ext
    assert not DpoObjective(loss_type='ipo').needs_ext
    for kw in (dict(f_divergence_type='js_divergence'), dict(f_divergence_type='alpha_divergence'),
               dict(f_divergence_type='alpha_divergence', f_alpha_divergence_coef=0.5), dict(loss_type='exo_pair'),
               dict(loss_type='discopop'), dict(loss_type='discopop', discopop_tau=0.1), dict(loss_type='aot'),
               dict(loss_type='aot_pair', label_smoothing=0.2), dict(loss_type='exo_pair', label_smoothing=0.3),
               dict(loss_type='hinge', f_divergence_type='js_divergence'), dict(loss_type='aot', reference_free=True)):
        o = DpoObjective(**kw)
        assert o.needs_ext and not o.is_default, kw
    assert DpoObjective(loss_type='aot', rpo_alpha=1.0).needs_counts
    for bad in (dict(loss_type='bco_pair'), dict(f_divergence_type='kl'), dict(f_divergence_type='JS_DIVERGENCE'),
                dict(loss_type='ipo', f_divergence_type='js_divergence'),
                dict(loss_type='aot', f_divergence_type='alpha_divergence'),
                dict(loss_type='discopop', f_divergence_type='js_divergence'),
                dict(f_alpha_divergence_coef=0.5), dict(f_divergence_type='js_divergence', f_alpha_divergence_coef=2.0),
                dict(f_divergence_type='alpha_divergence', f_alpha_divergence_coef=0.0),
                dict(f_divergence_type='alpha_divergence', f_alpha_divergence_coef=-1.0),
                dict(f_divergence_type='alpha_divergence', f_alpha_divergence_coef=float('inf')),
                dict(f_divergence_type='alpha_divergence', f_alpha_divergence_coef=float('nan')),
                dict(discopop_tau=0.1), dict(loss_type='aot', discopop_tau=0.1), dict(loss_type='discopop', discopop_tau=0.0),
                dict(loss_type='discopop', discopop_tau=float('nan')), dict(loss_type='discopop', label_smoothing=0.1),
                dict(loss_type='aot', label_smoothing=0.5), dict(loss_type='exo_pair', label_smoothing=-0.1)):
        with pytest.raises(ValueError):
            DpoObjective(**bad)


def test_aot_pair_cap_is_checked_on_the_host(dry):  # noqa: F811
    from align_anything_b200 import ops

    n = 2 * (ops.DPO_AOT_MAX_PAIRS + 1)
    lp = torch.zeros(n, 3)
    with pytest.raises(ValueError, match='sorts at most'):
        ops.dpo_loss_from_log_probs(lp, lp, 0.1, objective=ops.DpoObjective(loss_type='aot'))
    ops.dpo_loss_from_log_probs(lp, lp, 0.1, objective=ops.DpoObjective(loss_type='exo_pair'))
    assert dry.calls == ['aa_dpo_loss_ext']


def test_new_switches_default_to_unset_and_config_keys_win():
    from align_anything_b200.ops import DpoObjective
    from align_anything_b200.trainers.text_audio_to_text.dpo import DPOTrainer as A
    from align_anything_b200.trainers.text_image_to_text.dpo import DPOTrainer as I
    from align_anything_b200.trainers.text_to_text import dpo as D
    from align_anything_b200.trainers.text_video_to_text.dpo import DPOTrainer as V

    for cls in (D.DPOTrainer, A, I, V):
        assert all(getattr(cls, k) is None for k in NEW_KEYS) and set(NEW_KEYS) <= set(cls.SWITCHES)
    assert set(NEW_KEYS) <= set(D.DPO_OBJECTIVE_KEYS)
    tr = D.DPOTrainer(None, None, None, None)
    tr.loss_type, tr.f_divergence_type = 'exo_pair', 'js_divergence'
    assert D.dpo_objective_of(tr) == DpoObjective(loss_type='exo_pair', f_divergence_type='js_divergence')
    tc = types.SimpleNamespace(loss_type='discopop', discopop_tau=0.2, f_divergence_type=None)
    tr = A(types.SimpleNamespace(train_cfgs=tc), None, None, None)
    tr.discopop_tau = 0.7  # the recipe's value wins over the attribute
    assert D.dpo_objective_of(tr) == DpoObjective(loss_type='discopop', discopop_tau=0.2)
    tc.f_divergence_type = 'alpha_divergence'
    with pytest.raises(ValueError):  # an f-divergence with discopop
        D.dpo_objective_of(tr)


def test_install_sets_and_uninstall_restores_the_new_switches(fake_dpo_reference):  # noqa: F811
    from align_anything_b200 import patch

    try:
        patch.install(models=False)
        for modname, cls in fake_dpo_reference.items():
            for k in NEW_KEYS:
                assert k in cls.__dict__ and cls.__dict__[k] is None, (modname, k)
    finally:
        patch.uninstall()
    for modname, cls in fake_dpo_reference.items():
        for k in NEW_KEYS:
            assert k not in cls.__dict__, (modname, k)


def test_entry_point_checks_its_arguments_before_cuda():
    from align_anything_b200 import _lib

    lib = _lib.lib()
    buf = (ctypes.c_int64 * 64)()
    ptr = ctypes.cast(buf, ctypes.c_void_p)

    def call(loss_type=0, eps=0.0, alpha=0.0, fdiv=0, coef=1.0, tau=0.05, c1=math.log(1 - 1e-3), c2=math.log(1e-3),
             counts=ptr, beta=0.1, dtype=0, mode=0, grad_seg=ptr, n_pairs=2):
        return lib.aa_dpo_loss_ext(ptr, ptr, dtype, n_pairs, 4, 4, beta, mode, loss_type, eps, alpha, fdiv, coef, tau,
                                   c1, c2, counts, None, 0, 0, ptr, grad_seg, ptr, ptr, None, None)

    cases = [
        (dict(loss_type=12), b'bad objective: loss_type'), (dict(loss_type=-1), b'bad objective: loss_type'),
        (dict(fdiv=3), b'bad objective: f_divergence'), (dict(fdiv=-1), b'bad objective: f_divergence'),
        (dict(fdiv=1, loss_type=3), b'f_divergence 1 with loss_type 3'), (dict(fdiv=2, loss_type=9), b'f_divergence'),
        (dict(fdiv=1, loss_type=10), b'f_divergence'), (dict(coef=0.5), b'f_alpha_coef'),
        (dict(fdiv=2, coef=0.0), b'f_alpha_coef'), (dict(fdiv=2, coef=float('inf')), b'f_alpha_coef'),
        (dict(tau=0.1), b'discopop_tau'), (dict(loss_type=9, tau=0.0), b'discopop_tau'),
        (dict(loss_type=9, tau=float('nan')), b'discopop_tau'), (dict(loss_type=9, eps=0.1), b'label_smoothing'),
        (dict(loss_type=8, eps=0.5), b'label_smoothing'), (dict(loss_type=2, eps=0.1), b'label_smoothing'),
        (dict(alpha=-1.0), b'rpo_alpha'), (dict(loss_type=3, counts=None), b'needs the row counts'),
        (dict(loss_type=3, beta=0.0), b'needs scale_coeff > 0'), (dict(loss_type=10, n_pairs=1025), b'sorts at most'),
        (dict(loss_type=11, n_pairs=1025), b'sorts at most'), (dict(dtype=5), b'bad dtype'), (dict(mode=3), b'bad mode'),
        (dict(grad_seg=None), b'null pointer'), (dict(n_pairs=0), b'bad sizes'),
        (dict(loss_type=8, c1=0.0), b"EXO's log"), (dict(loss_type=8, c2=float('-inf')), b"EXO's log"),
        (dict(loss_type=8, c2=float('nan')), b"EXO's log"),
    ]
    for kw, msg in cases:
        rc = call(**kw)
        assert rc in (-1, -2), kw
        err = lib.aa_last_error()
        assert err.startswith(b'aa_dpo_loss_ext') and msg in err, (kw, err)
    # aa_dpo_loss_obj still refuses the new types
    assert lib.aa_dpo_loss_obj(ptr, ptr, 0, 2, 4, 4, 0.1, 0, 8, 0.0, 0.0, ptr, None, 0, 0, ptr, ptr, ptr, ptr, None,
                               None) in (-1, -2)
    assert b'bad objective: loss_type' in lib.aa_last_error()


@pytest.mark.parametrize('objective', ['js-exo', 'aot-cfg', 'alpha-hinge-free', 'ipo'])
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
    if objective == 'aot-cfg':
        tc.loss_type, tc.label_smoothing, tc.rpo_alpha = 'aot', 0.1, 1.0
    tr = cls(SimpleNamespace(train_cfgs=tc), _Eng(leaf, hid, w, pol_calls), _Eng(ref, hid.detach(), w.detach(), ref_calls),
             SimpleNamespace(pad_token_id=V - 1))
    tr.fused_lm_head = fused_head
    if objective == 'js-exo':
        tr.loss_type, tr.f_divergence_type = 'exo_pair', 'js_divergence'
    elif objective == 'alpha-hinge-free':
        tr.loss_type, tr.f_divergence_type, tr.f_alpha_divergence_coef, tr.reference_free = \
            'hinge', 'alpha_divergence', 0.5, True
    elif objective == 'ipo':
        tr.loss_type = 'ipo'
    out = tr.train_step({'input_ids': ids, 'attention_mask': ids != V - 1, 'meta_info': {'response_lens': lens}})
    keys = {'train/loss', 'train/reward', 'train/better_sample_reward', 'train/worse_sample_reward',
            'train/reward_accuracy', 'train/reward_margin', 'train/lr'}
    assert set(out) == (keys | {'train/nll_loss'} if objective == 'aot-cfg' else keys)
    calls = dry.calls
    if objective == 'ipo':  # a type aa_dpo_loss_obj has: today's entry point
        assert calls.count('aa_dpo_loss_obj') == 1 and 'aa_dpo_loss_ext' not in calls
    else:
        assert calls.count('aa_dpo_loss_ext') == 1 and 'aa_dpo_loss_obj' not in calls and 'aa_dpo_loss' not in calls
    free = objective == 'alpha-hinge-free'
    assert ref_calls == ([] if free else ['forward'])
    if fused_head:
        assert len([c for c in calls if c.startswith('aa_linear_logprob_fwd')]) == (1 if free else 2), calls
        assert {'aa_linear_dlogits', 'aa_linear_dhidden', 'aa_linear_dweight'} <= set(calls)
        assert hid.grad is not None and w.grad is not None
    else:
        assert calls.count('aa_logprob_fwd') == (1 if free else 2), calls
        assert calls.count('aa_logprob_bwd') == 1
        assert leaf.grad is not None and leaf.grad.shape == leaf.shape


def test_use_weighting_is_refused_not_ignored():
    from align_anything_b200.trainers.text_audio_to_text.dpo import DPOTrainer as A
    from align_anything_b200.trainers.text_to_text import dpo as D

    tc = types.SimpleNamespace(use_weighting=True)
    with pytest.raises(ValueError, match='use_weighting'):
        D.dpo_objective_of(A(types.SimpleNamespace(train_cfgs=tc), None, None, None))
    tr = D.DPOTrainer(None, None, None, None)
    tr.use_weighting = True
    with pytest.raises(ValueError, match='use_weighting'):
        D.dpo_objective_of(tr)
    tc.use_weighting = False  # TRL's default: the reference's loss
    assert D.dpo_objective_of(D.DPOTrainer(types.SimpleNamespace(train_cfgs=tc), None, None, None)) is None


def test_exo_constants_are_formed_from_the_python_value(dry):  # noqa: F811
    from align_anything_b200 import ops

    seen = []
    fn = dry.aa_dpo_loss_ext
    dry.aa_dpo_loss_ext = lambda *a: seen.append(a[14:16]) or fn(*a)
    lp = torch.zeros(4, 3)
    for eps, e in ((0.1, 0.1), (0.0, 1e-3)):
        ops.dpo_loss_from_log_probs(lp, lp, 0.1, objective=ops.DpoObjective(loss_type='exo_pair', label_smoothing=eps))
        assert seen[-1] == (math.log(1 - e), math.log(e))
