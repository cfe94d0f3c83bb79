"""Clip-Cov and KL-Cov without a GPU: the port (tests/cov_port.py) against a direct transcription of verl's
expressions, the selection counts at int()'s edges, the key order (ties, -0.0, NaN), every refusal, the trainer
switches with their config precedence and the graft, the C argument checks of the new entry points and, on the
stand-in library, which entry points the nodes call."""
from __future__ import annotations

import ctypes
from types import SimpleNamespace

import pytest
import torch

import cov_port as port
from test_cpu_entropy import fake_reference  # noqa: F401  (fixture)
from test_cpu_plumbing import dry  # noqa: F401  (fixture)
from test_cpu_ppo_step import packed  # noqa: F401  (fixture)

COV_KEYS = ('policy_loss_mode', 'clip_cov_ratio', 'clip_cov_lb', 'clip_cov_ub', 'kl_cov_ratio', 'ppo_kl_coef')
SELECTION = ['aa_cov_moments', 'aa_cov_keys', 'aa_cov_select_hi', 'aa_cov_hist_lo', 'aa_cov_select_lo', 'aa_cov_mark']


def _verl_agg(loss_mat, mask, agg):
    if agg == 'token-mean':
        return (loss_mat * mask).sum() / mask.sum()
    return ((loss_mat * mask).sum(-1) / mask.sum(-1)).mean()


def _verl_clip_cov(old, lp, adv, mask, sel, lo, hi, agg):
    """verl's compute_policy_loss_clip_cov after its draw: corr = 0 on the drawn tokens."""
    ratio = torch.exp(lp - old)
    pg1 = -adv * ratio
    pg2 = -adv * torch.clamp(ratio, 1 - lo, 1 + hi)
    corr = torch.ones_like(adv)
    corr[sel] = 0
    return _verl_agg(torch.maximum(pg1, pg2) * corr, mask, agg)


def _verl_kl_cov(old, lp, adv, mask, sel, coef, agg):
    """verl's compute_policy_loss_kl_cov after its top-k: the chosen tokens take pg_losses_kl."""
    d = lp - old
    ratio = torch.exp(d)
    pg = -adv * ratio
    pg_kl = -adv * ratio + coef * d.abs()
    pg = torch.where(sel, pg_kl, pg)
    return _verl_agg(pg, mask, agg)


def _inputs(B=5, W=17, seed=0):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, W, generator=g, dtype=torch.float64) * 3
    old = lp + torch.randn(B, W, generator=g, dtype=torch.float64) * 0.3
    adv = torch.randn(B, W, generator=g, dtype=torch.float64)
    mask = torch.rand(B, W, generator=g) < 0.8
    mask[:, 0] = True
    sel = (torch.rand(B, W, generator=g) < 0.2) & mask
    return lp, old, adv, mask, sel


@pytest.mark.parametrize('agg', ['seq-mean-token-mean', 'token-mean'])
@pytest.mark.parametrize('mode', ['clip_cov', 'kl_cov'])
def test_port_matches_verl_transcription(mode, agg):
    lp, old, adv, mask, sel = _inputs()
    x = lp.clone().requires_grad_(True)
    y = lp.clone().requires_grad_(True)
    got = port.ppo_loss(mode, x, old, adv, mask, sel, agg, 0.2, 0.28, 0.7)
    want = (_verl_clip_cov(old, y, adv, mask, sel, 0.2, 0.28, agg) if mode == 'clip_cov' else
            _verl_kl_cov(old, y, adv, mask, sel, 0.7, agg))
    got.backward()
    want.backward()
    assert torch.allclose(got, want, rtol=1e-14, atol=0)
    assert torch.allclose(x.grad, y.grad, rtol=1e-12, atol=1e-15)
    if mode == 'clip_cov':
        assert (x.grad[sel] == 0).all()


def test_kl_cov_on_the_first_update_changes_nothing():
    lp, _, adv, mask, sel = _inputs(seed=3)
    a = lp.clone().requires_grad_(True)
    b = lp.clone().requires_grad_(True)
    port.grpo_loss('kl_cov', a, lp * 0.9, None, adv[:, 0], mask, sel, 0.04).backward()
    port.grpo_loss('kl_cov', b, lp * 0.9, None, adv[:, 0], mask, torch.zeros_like(sel), 0.04).backward()
    assert torch.equal(a.grad, b.grad)


@pytest.mark.parametrize('ratio,n,k', [(2e-4, 0, 0), (2e-4, 1, 1), (2e-4, 4999, 1), (2e-4, 10000, 2),
                                       (2e-4, 14999, 2), (0.29, 100, 28), (0.3, 10, 3), (0.7, 10, 7), (1.0, 7, 7),
                                       (0.1, 30, 3), (0.57, 100, 56)])
def test_select_count_at_int_edges(ratio, n, k):
    # the product in double as Python forms it: 0.29 * 100 = 28.999999999999996 and 0.57 * 100 = 56.99999999999999
    assert port.n_select(ratio, n) == k == (0 if n == 0 else max(int(ratio * n), 1))


def test_key_order_ties_signed_zero_and_nan():
    x = torch.tensor([1.0, -0.0, 0.0, float('nan'), float('inf'), -float('inf'), -1.0, 1.0, float('nan')])
    keys = port.order_key(x)
    assert keys[1] == keys[2] and keys[3] == keys[8] and keys[3] > keys[4] > keys[0] > keys[2] > keys[6] > keys[5]
    every = torch.ones_like(x, dtype=torch.bool)
    assert port.top_k(keys, every, 3).nonzero().squeeze(1).tolist() == [3, 4, 8]
    assert port.top_k(keys, every, 5).nonzero().squeeze(1).tolist() == [0, 3, 4, 7, 8]  # 1.0 ties: both taken
    assert port.top_k(keys, every, 4).nonzero().squeeze(1).tolist() == [0, 3, 4, 8]  # ... the smaller index first
    zeros = torch.tensor([[0.0, -0.0], [-0.0, 0.0]])
    assert port.top_k(port.order_key(zeros), torch.ones(2, 2, dtype=torch.bool), 3).tolist() == [[True, True],
                                                                                                  [True, False]]


def test_clip_cov_hash_is_a_bijection_and_seeded():
    t = torch.arange(1 << 16, dtype=torch.int64)
    for s in (0, port.hash_seed(0, 0, 1), port.hash_seed(7, 3, 11)):
        assert port.fmix32(t ^ s).unique().numel() == t.numel()
    from align_anything_b200 import ops

    for seed, rank, call in ((0, 0, 0), (42, 1, 5), (2 ** 40 + 3, 7, 2 ** 33)):
        assert ops.cov_hash_seed(seed, rank, call) == port.hash_seed(seed & port.U32, rank, call & port.U32)
    assert port.hash_seed(1, 0, 0) != port.hash_seed(1, 0, 1) != port.hash_seed(1, 1, 0)


def test_objective_fields_and_refusals():
    from align_anything_b200 import ops

    assert ops.ActorObjective().is_default and ops.ActorObjective(policy_loss_mode='vanilla').is_default
    assert ops.GrpoObjective(policy_loss_mode='vanilla').is_default
    for mode in ('clip_cov', 'kl_cov'):
        assert not ops.ActorObjective(policy_loss_mode=mode).is_default
        assert not ops.GrpoObjective(policy_loss_mode=mode).is_default
    o = ops.ActorObjective(policy_loss_mode='clip_cov', clip_range_ratio_high=0.28)
    assert [o.cov_value(k) for k in port.DEFAULTS] == list(port.DEFAULTS.values())
    bad = [
        dict(policy_loss_mode='gpg'),
        *[dict({k: v}) for k, v in (('clip_cov_ratio', 0.1), ('clip_cov_lb', 0.0), ('clip_cov_ub', 2.0),
                                    ('kl_cov_ratio', 0.1), ('ppo_kl_coef', 1.0))],  # a key under vanilla
        dict(policy_loss_mode='clip_cov', dual_clip_ratio=3.0),
        dict(policy_loss_mode='kl_cov', dual_clip_ratio=3.0),
        dict(policy_loss_mode='kl_cov', clip_range_ratio_low=0.2),
        dict(policy_loss_mode='kl_cov', clip_range_ratio_high=0.28),
        *[dict(policy_loss_mode='clip_cov', clip_cov_ratio=r) for r in (0.0, -1e-4, 1.5, float('nan'))],
        *[dict(policy_loss_mode='kl_cov', kl_cov_ratio=r) for r in (0.0, 1.01, float('inf'))],
        dict(policy_loss_mode='clip_cov', clip_cov_lb=5.0),  # lb == ub
        dict(policy_loss_mode='clip_cov', clip_cov_lb=-float('inf')),
        dict(policy_loss_mode='clip_cov', clip_cov_ub=float('nan')),
        dict(policy_loss_mode='kl_cov', ppo_kl_coef=-0.1),
        dict(policy_loss_mode='kl_cov', ppo_kl_coef=float('inf')),
        dict(policy_loss_mode='kl_cov', ppo_kl_coef='1'),
        dict(policy_loss_mode='kl_cov', kl_cov_ratio=True),
    ]
    for kw in bad:
        for cls in (ops.ActorObjective, ops.GrpoObjective):
            with pytest.raises(ValueError):
                cls(**kw)
    for kw in (dict(importance_sampling_level='sequence'), dict(top_entropy_quantile=0.5)):
        for mode in ('clip_cov', 'kl_cov'):
            with pytest.raises(ValueError, match='token-level'):
                ops.GrpoObjective(policy_loss_mode=mode, **kw)
    assert ops.ActorObjective(policy_loss_mode='kl_cov', ppo_kl_coef=0.0).cov_value('ppo_kl_coef') == 0.0


def test_switches_default_to_vanilla_and_config_keys_win():
    from align_anything_b200.trainers.text_to_text import grpo as G
    from align_anything_b200.trainers.text_to_text import ppo as P

    for keys, cls in ((P.OBJECTIVE_KEYS, P.PPOTrainer), (G.GRPO_OBJECTIVE_KEYS, G.GRPOTrainer)):
        for k in COV_KEYS:
            assert k in keys and k in cls.SWITCHES and getattr(cls, k) is None
    assert P.actor_objective_of(P.PPOTrainer()) is None
    tc = SimpleNamespace(update_iters=1, policy_loss_mode=None)
    tr = P.PPOTrainer(SimpleNamespace(train_cfgs=tc))
    assert P.actor_objective_of(tr) is None
    tr.policy_loss_mode = 'kl_cov'
    assert P.actor_objective_of(tr).policy_loss_mode == 'kl_cov'
    tc.policy_loss_mode, tc.clip_cov_ratio = 'clip_cov', 0.01  # the recipe's values win over the attributes
    o = P.actor_objective_of(tr)
    assert o.policy_loss_mode == 'clip_cov' and o.clip_cov_ratio == 0.01
    g = G.GRPOTrainer(SimpleNamespace(train_cfgs=tc))
    assert G.grpo_objective_of(g).policy_loss_mode == 'clip_cov'
    tc.policy_loss_mode = 'vanilla'
    with pytest.raises(ValueError, match='clip_cov_ratio'):
        P.actor_objective_of(tr)


def test_clip_cov_counter_and_seed():
    from align_anything_b200 import ops
    from align_anything_b200.trainers.text_to_text import ppo as P

    tr = P.PPOTrainer(SimpleNamespace(train_cfgs=SimpleNamespace(seed=42, policy_loss_mode='clip_cov')))
    o = P.actor_objective_of(tr)
    assert [P.cov_seed_of(tr, o) for _ in range(3)] == [ops.cov_hash_seed(42, 0, n) for n in range(3)]
    assert tr.cov_calls == 3
    assert P.cov_seed_of(tr, ops.ActorObjective(policy_loss_mode='kl_cov')) == 0 and tr.cov_calls == 3
    bare = P.PPOTrainer()
    assert P.cov_seed_of(bare, o) == ops.cov_hash_seed(0, 0, 0)


def test_install_grafts_the_switches(fake_reference):  # noqa: F811
    from align_anything_b200 import patch

    rl = {m: c for m, c in fake_reference.items() if 'ppo' in m or 'grpo' in m}
    assert rl
    try:
        patch.install(models=False)
        for modname, cls in rl.items():
            for k in COV_KEYS:
                assert k in cls.__dict__ and cls.__dict__[k] is None, (modname, k)
    finally:
        patch.uninstall()
    for modname, cls in rl.items():
        for k in COV_KEYS:
            assert k not in cls.__dict__, (modname, k)


def test_entry_points_check_their_arguments_before_cuda():
    from align_anything_b200 import _lib

    lib = _lib.lib()
    buf = (ctypes.c_int64 * 8)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def err():
        return lib.aa_last_error()

    def moments(lp=p, ls=8, dt=2, adv=p, ast=8, adt=2, mask=p, ms=8, re=None, B=2, W=8, state=p):
        return lib.aa_cov_moments(lp, ls, dt, adv, ast, adt, mask, ms, re, B, W, state, None)

    assert moments(lp=None) == -2 and b'aa_cov_moments: null pointer' in err()
    assert moments(state=None) == -2 and b'null state' in err()
    assert moments(re=p) == -2 and b'give exactly one of row_end and mask' in err()
    assert moments(mask=None) == -2 and b'give exactly one' in err()
    assert moments(B=0) == -2 and b'bad sizes' in err()
    assert moments(B=1 << 16, W=1 << 16) == -2 and b'bad sizes' in err()
    assert moments(ls=7) == -2 and b'row strides must be >= W' in err()
    assert moments(ms=7) == -2 and moments(ast=7) == -2
    assert moments(dt=5) == -1 and b'bad dtype' in err()
    assert moments(mask=None, re=p, adt=0) == -1 and b'per-row advantages are fp32' in err()

    def keys(cm=1, old=p, os_=8, lo=0.2, hi=0.2, lb=1.0, ub=5.0, mode=0, k=p):
        return lib.aa_cov_keys(cm, p, 8, old, os_, 2, p, 8, 2, p, 8, None, 2, 8, lo, hi, lb, ub, 0, mode, p, k, p, p,
                               None)

    assert keys(cm=0) == -2 and b'aa_cov_keys: unknown cov_mode 0' in err()
    assert keys(cm=3) == -2
    assert keys(k=None) == -2 and b'aa_cov_keys: null pointer' in err()
    assert keys(mode=5) == -2 and b'aa_cov_keys: bad mode' in err()
    assert keys(os_=7) == -2 and b'old_stride' in err()
    for bad in (dict(lo=1.0), dict(hi=-0.1), dict(lb=5.0), dict(lb=float('nan')), dict(ub=float('inf'))):
        assert keys(**bad) == -2 and b'bad Clip-Cov arguments' in err()
    for r in (0.0, -1.0, 1.5, float('nan')):
        assert lib.aa_cov_select_hi(p, ctypes.byref(ctypes.c_double(r)), p, None) == -2 and \
            b'aa_cov_select_hi: ratio must lie in (0, 1]' in err()
    assert lib.aa_cov_select_hi(None, ctypes.byref(ctypes.c_double(0.5)), p, None) == -2
    assert lib.aa_cov_select_hi(p, None, p, None) == -2 and b'aa_cov_select_hi: null pointer' in err()
    assert lib.aa_cov_hist_lo(p, p, 0, p, p, None) == -2 and b'aa_cov_hist_lo: bad size' in err()
    assert lib.aa_cov_hist_lo(p, None, 8, p, p, None) == -2 and b'aa_cov_hist_lo: null pointer' in err()
    assert lib.aa_cov_select_lo(p, p, None, None) == -2 and b'aa_cov_select_lo: null pointer' in err()
    assert lib.aa_cov_mark(p, p, 2, 8, p, p, None, 8, None) == -2 and b'aa_cov_mark: null pointer' in err()
    assert lib.aa_cov_mark(p, p, 2, 8, p, p, p, 7, None) == -2 and b'aa_cov_mark: bad sizes' in err()

    def ppo(cm=1, coef=0.0, sel=p, ss=8, ref=None, klc=0.0, est=2, lo=0.2, agg=0, mode=0):
        return lib.aa_ppo_actor_loss_cov(p, 8, p, 8, 2, p, 8, 2, p, 8, 2, 8, lo, 0.2, agg, cm, coef, sel, ss, mode, ref,
                                         8, klc, est, p, p, p, 8, None, p, p, None)

    assert ppo(cm=0) == -2 and b'aa_ppo_actor_loss_cov: unknown cov_mode' in err()
    assert ppo(coef=-1.0) == -2 and b'cov_coef must be finite and >= 0' in err()
    assert ppo(coef=float('inf')) == -2
    assert ppo(sel=None) == -2 and b'null pointer' in err()
    assert ppo(ss=7) == -2 and b'sel_stride' in err()
    assert ppo(lo=1.0) == -2 and b'bad objective' in err()
    assert ppo(agg=2) == -2 and b'bad objective' in err()
    assert ppo(mode=3) == -2 and b'bad mode' in err()
    assert ppo(ref=p, klc=0.0) == -2 and b'a KL loss term needs kl_loss_coeff' in err()
    assert ppo(ref=p, klc=0.1, est=7) == -2 and b'unknown kl_estimator' in err()

    def grpo(cm=2, coef=1.0, sel=p, ss=8, lo=0.2, est=2, mode=0):
        return lib.aa_grpo_loss_cov(p, 8, p, 8, None, 0, 2, p, p, 8, 1, 2, 8, 0.04, lo, 0.2, 1, est, cm, coef, sel, ss,
                                    mode, p, p, 8, None, p, p, p, None)

    assert grpo(cm=7) == -2 and b'aa_grpo_loss_cov: unknown cov_mode' in err()
    assert grpo(coef=float('nan')) == -2 and b'cov_coef must be finite' in err()
    assert grpo(sel=None) == -2 and grpo(ss=7) == -2 and b'sel must be given' in err()
    assert grpo(lo=1.0) == -2 and b'aa_grpo_loss_cov: bad objective' in err()
    assert grpo(est=3) == -2 and b'unknown kl_estimator' in err()
    assert grpo(mode=4) == -2 and b'bad mode' in err()


def test_cov_token_selection_checks_before_any_launch(dry):  # noqa: F811
    from align_anything_b200 import ops

    lp, adv = torch.rand(2, 5), torch.rand(2, 5)
    mask, re = torch.ones(2, 5, dtype=torch.bool), torch.tensor([3, 5], dtype=torch.int32)
    for bad in (dict(policy_loss_mode='vanilla'), dict(policy_loss_mode='gpg'), dict(log_probs=lp.double()),
                dict(log_probs=lp[0]), dict(log_probs=torch.empty(0, 5)), dict(advantages=adv[:, :4]),
                dict(mask_or_row_end=re.float()), dict(mask_or_row_end=torch.ones(3, dtype=torch.int32)),
                dict(mask_or_row_end=re.bool()), dict(old_log_probs=lp[:, :4]), dict(clip_cov_ratio=0.0),
                dict(clip_range_ratio_low=1.0), dict(kl_cov_ratio=2.0)):
        kw = {**dict(log_probs=lp, advantages=adv, mask_or_row_end=mask, policy_loss_mode='clip_cov'), **bad}
        if 'kl_cov_ratio' in bad:
            kw['policy_loss_mode'] = 'kl_cov'
        with pytest.raises(ValueError):
            ops.cov_token_selection(**kw)
    with pytest.raises(ValueError, match='one advantage per row'):
        ops.cov_token_selection(lp, adv, re, 'kl_cov')
    assert dry.calls == []
    sel = ops.cov_token_selection(lp, adv, mask, 'kl_cov')
    assert sel.shape == (2, 5) and sel.dtype == torch.uint8 and dry.calls == SELECTION
    dry.calls.clear()
    sel, share = ops.cov_token_selection(lp, adv[:, 0], re, 'clip_cov', return_share=True)
    assert share.shape == (1,) and dry.calls == SELECTION


@pytest.mark.parametrize('mode', ['clip_cov', 'kl_cov'])
def test_nodes_take_the_composed_path(dry, mode):  # noqa: F811
    from align_anything_b200 import ops

    B, Lq, V = 2, 9, 97
    logits = torch.randn(B, Lq, V, requires_grad=True)
    ids = torch.randint(0, V, (B, Lq))
    W = Lq - 1 - 2
    obj = ops.ActorObjective(policy_loss_mode=mode)
    out = ops.dense_actor_loss(logits, ids, 2, torch.rand(B, W), torch.rand(B, W), torch.ones(B, W, dtype=torch.bool),
                               0.2, objective=obj, cov_seed=5)
    assert len(out) == 4 and out[-1].shape == (1,)
    assert not any(c.startswith('aa_logprob_actor_fused') for c in dry.calls)
    assert dry.calls[-7:] == SELECTION + ['aa_ppo_actor_loss_cov']
    dry.calls.clear()
    plain = ops.dense_actor_loss(logits, ids, 2, torch.rand(B, W), torch.rand(B, W),
                                 torch.ones(B, W, dtype=torch.bool), 0.2, objective=ops.ActorObjective())
    assert len(plain) == 3 and not set(SELECTION) & set(dry.calls)
    dry.calls.clear()
    lp, ref, adv, tok = torch.rand(2, 5), torch.rand(2, 5), torch.rand(2, 1), torch.randint(3, 9, (2, 5))
    out = ops.grpo_loss(lp, ref, adv, tok, 2, 0.04, objective=ops.GrpoObjective(policy_loss_mode=mode), cov_seed=1,
                        return_clip_fraction=True)
    assert len(out) == 4 and dry.calls[-8:] == ['aa_grpo_row_end', *SELECTION, 'aa_grpo_loss_cov']


def _grpo_trainer(dry, fused, **cfg):  # noqa: F811
    from test_cpu_top_entropy import _trainer

    return _trainer(dry, fused, **cfg)


@pytest.mark.parametrize('mode', ['clip_cov', 'kl_cov'])
@pytest.mark.parametrize('fused', [False, True])
def test_grpo_updates_select_and_never_run_k1f(dry, packed, fused, mode):  # noqa: F811
    t = _grpo_trainer(dry, fused, update_iters=2, num_iterations=2, policy_loss_mode=mode, seed=3)
    gen = torch.Generator().manual_seed(0)
    out = t.step_from_rollout(torch.randint(3, 97, (4, 9), generator=gen), 4, torch.randn(4, generator=gen))
    assert 'train/actor_cov_fraction' in out
    assert dry.calls.count('aa_grpo_loss_cov') == 2 and dry.calls.count('aa_cov_mark') == 2
    assert not any(c.startswith('aa_logprob_grpo_fused') for c in dry.calls)
    assert getattr(t, 'cov_calls', 0) == (2 if mode == 'clip_cov' else 0)


@pytest.mark.parametrize('fused', [False, True])
def test_grpo_vanilla_makes_todays_calls(dry, packed, fused):  # noqa: F811
    runs = []
    for cfg in ({}, {'policy_loss_mode': 'vanilla'}, {'policy_loss_mode': None}):
        dry.calls.clear()
        t = _grpo_trainer(dry, fused, update_iters=1, **cfg)
        gen = torch.Generator().manual_seed(0)
        out = t.step_from_rollout(torch.randint(3, 97, (4, 9), generator=gen), 4, torch.randn(4, generator=gen))
        assert 'train/actor_cov_fraction' not in out
        runs.append(list(dry.calls))
    assert runs[0] == runs[1] == runs[2] and not set(SELECTION) & set(runs[0])


def test_safe_rlhf_v_refuses_the_switches():
    from align_anything_b200.trainers.text_image_to_text.saferlhf import SafeRLHFVTrainer, refuse_cov_switches

    t = object.__new__(SafeRLHFVTrainer)
    t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(policy_loss_mode='vanilla'))
    refuse_cov_switches(t)
    for k, v in (('policy_loss_mode', 'kl_cov'), ('clip_cov_ratio', 0.1), ('ppo_kl_coef', 0.5)):
        t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(**{k: v}))
        with pytest.raises(ValueError, match='Safe RLHF-V'):
            t.rl_step({}, {})
