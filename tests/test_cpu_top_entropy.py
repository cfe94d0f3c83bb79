"""High-entropy token masking without a GPU: the port (tests/top_entropy_port.py) against float64 autograd, its
sort-based threshold against torch.quantile, ops.GrpoObjective's top_entropy_quantile field, the trainer switch, its
config precedence and the graft, the C argument checks of the new entry points and, on the stand-in library, which
entry points each update calls."""
from __future__ import annotations

import ctypes
from types import SimpleNamespace

import pytest
import torch

import top_entropy_port as port
from grpo_objective_port import completion_mask
from test_cpu_entropy import fake_reference  # noqa: F401  (fixture)
from test_cpu_plumbing import dry  # noqa: F401  (fixture)
from test_cpu_ppo_step import packed  # noqa: F401  (fixture)

AGGS = ['token-mean', 'seq-mean-token-mean', 'seq-mean-token-sum-norm']
ESTIMATORS = ['k1', 'k2', 'k3']


def _inputs(B=6, K=23, seed=0):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, K, generator=g, dtype=torch.float64) * 4
    ref = lp + torch.randn(B, K, generator=g, dtype=torch.float64) * 0.3
    shift = torch.tensor([0.0, 0.1, -0.1, 0.5, -0.5, 0.05], dtype=torch.float64)[:B].unsqueeze(-1)
    old = lp - shift + torch.randn(B, K, generator=g, dtype=torch.float64) * 0.2
    adv = torch.tensor([[1.3], [-0.8], [0.6], [-1.7], [2.1], [-0.4]], dtype=torch.float64)[:B]
    ent = (torch.rand(B, K, generator=g) * 3 - 0.01).float()  # the kernels' entropy is fp32
    tokens = torch.randint(2, 50, (B, K), generator=g)
    tokens[0, 4] = 1
    tokens[2, 0] = 1
    tokens[3, 11] = 1
    return lp, ref, old, adv, ent, tokens


def _f64(x, ref, old, adv, mask, keep, beta, lo, hi, c, agg, est, sequence):
    """The masked objective written row by row over each row's counted tokens (slices, not masks)."""
    B, K = x.shape
    rows, n_all = [], mask.sum()
    for i in range(B):
        n = int(mask[i].sum())
        a = adv[i, 0]
        if sequence:
            w = torch.exp((x[i, :n] - old[i, :n]).sum() / n).expand(n)
        else:
            w = torch.exp(x[i, :n] - (x[i, :n].detach() if old is None else old[i, :n]))
        s = torch.minimum(a * w, a * w.clamp(1 - lo, 1 + hi))
        if c is not None and a < 0:
            s = torch.maximum(s, c * a)
        s = torch.where(keep[i, :n], s, torch.zeros_like(s))
        d = x[i, :n] - ref[i, :n]
        kl = {'k1': d, 'k2': 0.5 * d * d, 'k3': torch.exp(-d) + d - 1}[est]
        rows.append(-(s - beta * kl))
    if agg == 'token-mean':
        return torch.cat(rows).sum() / n_all
    if agg == 'seq-mean-token-mean':
        return torch.stack([r.mean() for r in rows]).mean()
    return torch.cat(rows).sum() / (B * K)


@pytest.mark.parametrize('sequence', [False, True])
@pytest.mark.parametrize('est', ESTIMATORS)
@pytest.mark.parametrize('dual', [None, 3.0])
@pytest.mark.parametrize('agg', AGGS)
def test_port_matches_float64_autograd(agg, dual, est, sequence):
    lp, ref, old, adv, ent, tokens = _inputs()
    mask = completion_mask(tokens, 1)
    keep = port.entropy_keep(ent, mask, 0.3)
    assert 0 < int(keep.sum()) < int(mask.sum())
    x = lp.clone().requires_grad_(True)
    got = port.grpo_loss(x, ref, adv, mask, 0.04, keep, old, 0.2, 0.28, dual, agg, est, sequence)
    got.backward()
    y = lp.clone().requires_grad_(True)
    want = _f64(y, ref, old, adv, mask, keep, 0.04, 0.2, 0.28, dual, agg, est, sequence)
    want.backward()
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(x.grad, y.grad, rtol=1e-12, atol=1e-12)
    assert torch.equal(x.grad[mask == 0], torch.zeros_like(x.grad[mask == 0]))


@pytest.mark.parametrize('agg', AGGS)
def test_masked_tokens_carry_the_kl_gradient_alone(agg):
    from kl_objective_port import kl_estimate

    lp, ref, old, adv, ent, tokens = _inputs(seed=3)
    mask = completion_mask(tokens, 1)
    keep = port.entropy_keep(ent, mask, 0.2)
    x = lp.clone().requires_grad_(True)
    port.grpo_loss(x, ref, adv, mask, 0.04, keep, old, 0.2, 0.28, 3.0, agg, 'k3').backward()
    y = lp.clone().requires_grad_(True)
    m = mask.double()
    kl = 0.04 * kl_estimate(y, ref, 'k3') * m
    n = {'token-mean': m.sum(), 'sum-norm': float(lp.numel())}.get(agg.replace('seq-mean-token-', ''), None)
    if agg == 'seq-mean-token-mean':
        (kl.sum(-1) / m.sum(-1)).mean().backward()
    else:
        (kl.sum() / (m.sum() if agg == 'token-mean' else n)).backward()
    off = mask.bool() & ~keep
    assert off.any()
    torch.testing.assert_close(x.grad[off], y.grad[off], rtol=1e-12, atol=1e-15)


def test_rho_one_keeps_every_counted_token():
    lp, ref, old, adv, ent, tokens = _inputs(seed=5)
    mask = completion_mask(tokens, 1)
    keep = port.entropy_keep(ent, mask, 1.0)
    assert torch.equal(keep, mask.bool())


VALUES = {
    'random': lambda g: torch.rand(1000, generator=g) * 4,
    'ties': lambda g: torch.randint(0, 5, (777,), generator=g).float() * 0.5,
    'all-equal': lambda g: torch.full((64,), 0.625),
    'one': lambda g: torch.tensor([1.75]),
    'two': lambda g: torch.tensor([3.0, -1.0]),
    'negative': lambda g: torch.randn(501, generator=g) * 1e-6,
    'signed-zeros': lambda g: torch.tensor([0.0, -0.0, -0.0, 0.0, 1e-7, -1e-7, -0.0]),
    'wide': lambda g: torch.cat([torch.rand(300, generator=g) * 1e30, -torch.rand(300, generator=g) * 1e-30]),
}


@pytest.mark.parametrize('rho', [0.0, 0.2, 0.5, 1.0])
@pytest.mark.parametrize('name', list(VALUES))
def test_sort_threshold_equals_torch_quantile(name, rho):
    v = VALUES[name](torch.Generator().manual_seed(len(name)))
    got = port.quantile_threshold(v, 1.0 - rho)
    want = torch.quantile(v, 1.0 - rho)
    assert got.dtype == torch.float32 and float(got) == float(want), (float(got), float(want))


def test_sort_threshold_at_rho_zero_is_the_maximum_and_keeps_its_ties():
    v = torch.tensor([[0.5, 2.0, 2.0, 1.0, 2.0]])
    keep = port.entropy_keep(v, torch.ones_like(v, dtype=torch.int64), 0.0)
    assert keep.tolist() == [[False, True, True, False, True]]


def test_sort_threshold_nan_and_empty():
    v = torch.tensor([0.5, float('nan'), 1.0])
    assert torch.isnan(port.quantile_threshold(v, 0.8)) and torch.isnan(torch.quantile(v, 0.8))
    assert torch.isnan(port.quantile_threshold(torch.empty(0), 0.8))
    ent = torch.rand(2, 3)
    assert not port.entropy_keep(ent, torch.zeros(2, 3, dtype=torch.int64), 0.5).any()  # N == 0: keep nothing
    assert not port.entropy_keep(torch.full((1, 3), float('nan')), torch.ones(1, 3), 0.5).any()


def test_sort_threshold_rounds_the_rank_in_fp32():
    # fl32(0.3) * (10^7 - 1) = 2999999.75 in fp32: v[2999999] = 0, v[3000000] = 1, weight 0.75
    v = torch.zeros(10 ** 7)
    v[3 * 10 ** 6:] = 1.0
    assert float(torch.quantile(v, 0.3)) == 0.75 == float(port.quantile_threshold(v, 0.3))


def test_grpo_objective_takes_top_entropy_quantile():
    from align_anything_b200 import ops

    assert ops.GrpoObjective().top_entropy_quantile == 1.0 and ops.GrpoObjective().is_default
    assert ops.GrpoObjective(top_entropy_quantile=1).is_default
    for rho in (0.0, 0.2, 0.999):
        o = ops.GrpoObjective(top_entropy_quantile=rho)
        assert not o.is_default and ops._top_entropy(o)
        # the clipped objective's arguments at default fields (the reference form is not used under the mask)
        assert ops._grpo_objective_args(o, None, False) == ops._grpo_objective_args(ops.GrpoObjective(), None, True)
    assert not ops._top_entropy(None) and not ops._top_entropy(ops.GrpoObjective())
    for bad in (-0.1, 1.5, float('nan'), float('inf'), '0.2', None, True):
        with pytest.raises(ValueError, match='top_entropy_quantile'):
            ops.GrpoObjective(top_entropy_quantile=bad)


def test_switch_defaults_to_one_and_config_key_wins():
    from align_anything_b200.ops import GrpoObjective
    from align_anything_b200.trainers.text_to_text import grpo as G

    assert G.GRPOTrainer.top_entropy_quantile == 1.0
    assert 'top_entropy_quantile' in G.GRPO_OBJECTIVE_KEYS and 'top_entropy_quantile' in G.GRPOTrainer.SWITCHES
    assert G.grpo_objective_of(G.GRPOTrainer()) is None
    tc = SimpleNamespace(update_iters=1, top_entropy_quantile=None)
    tr = G.GRPOTrainer(SimpleNamespace(train_cfgs=tc))
    assert G.grpo_objective_of(tr) is None
    tr.top_entropy_quantile = 0.2
    assert G.grpo_objective_of(tr) == GrpoObjective(top_entropy_quantile=0.2)
    tc.top_entropy_quantile = 0.5  # the recipe's value wins over the attribute
    assert G.grpo_objective_of(tr).top_entropy_quantile == 0.5
    tc.top_entropy_quantile = 1.0
    assert G.grpo_objective_of(tr) is None
    for bad in (1.01, -0.5):
        tc.top_entropy_quantile = bad
        with pytest.raises(ValueError, match='top_entropy_quantile'):
            G.grpo_objective_of(tr)


def test_out_of_range_switch_is_refused_before_anything_runs(dry):  # noqa: F811
    from align_anything_b200.trainers.text_to_text import grpo as G

    t = object.__new__(G.GRPOTrainer)
    t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(update_iters=1, top_entropy_quantile=2.0))
    t.fused_lm_head = False
    with pytest.raises(ValueError, match='top_entropy_quantile'):
        t.step_from_rollout(torch.randint(3, 97, (4, 9)), 4, torch.randn(4))
    assert dry.calls == []


def test_install_grafts_the_switch(fake_reference):  # noqa: F811
    from align_anything_b200 import patch

    grpo = {m: c for m, c in fake_reference.items() if 'grpo' in m}
    assert grpo
    try:
        patch.install(models=False)
        for modname, cls in grpo.items():
            assert cls.__dict__.get('top_entropy_quantile') == 1.0, modname
    finally:
        patch.uninstall()
    for modname, cls in grpo.items():
        assert 'top_entropy_quantile' not in cls.__dict__, modname


def test_entry_points_check_their_arguments_before_cuda():
    from align_anything_b200 import _lib

    lib = _lib.lib()
    buf = (ctypes.c_int64 * 8)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def topent(old=p, seq=0, ent=p, es=8, thr=p, lo=0.2, est=2, mode=0):
        return lib.aa_grpo_loss_topent(p, 8, p, 8, old, 8, 2, p, p, 8, 1, 2, 8, 0.04, lo, 0.2, 0.0, 1, est, seq, mode,
                                       p, p, 8, None, ent, es, thr, p, p, p, None)

    def err():
        return lib.aa_last_error()

    assert topent(seq=2) == -2 and b'aa_grpo_loss_topent: sequence must be 0 or 1' in err()
    assert topent(ent=None) == -2 and b'aa_grpo_loss_topent: the top-entropy mask needs entropy' in err()
    assert topent(thr=None) == -2 and b'the top-entropy mask needs entropy' in err()
    assert topent(es=7) == -2 and b'the top-entropy mask needs entropy (row stride >= K)' in err()
    assert topent(old=None, seq=1) == -2 and b'needs old_log_probs' in err()
    assert topent(lo=1.0) == -2 and b'aa_grpo_loss_topent: bad objective' in err()
    assert topent(est=3) == -2 and b'aa_grpo_loss_topent: unknown kl_estimator' in err()
    assert topent(mode=5) == -2 and b'aa_grpo_loss_topent: bad mode' in err()

    assert lib.aa_grpo_row_end(None, 8, 1, 2, 8, p, p, p, None) == -2 and b'aa_grpo_row_end: bad arguments' in err()
    assert lib.aa_grpo_row_end(p, 8, 1, 0, 8, p, p, p, None) == -2
    for name in ('aa_entropy_hist_hi', 'aa_entropy_hist_lo'):
        fn = getattr(lib, name)
        extra = (p,) if name.endswith('lo') else ()

        def call(ent=p, es=8, re=p, mask=None, ms=0, B=2, K=8, hist=p):
            return fn(ent, es, re, mask, ms, B, K, *extra, hist, None)

        assert call(ent=None) == -2 and f'{name}: null pointer'.encode() in err()
        assert call(hist=None) == -2 and f'{name}: null pointer'.encode() in err()
        assert call(re=None) == -2 and b'give exactly one of row_end and mask' in err()
        assert call(mask=p, ms=8) == -2 and b'give exactly one of row_end and mask' in err()
        assert call(B=0) == -2 and b'bad sizes' in err()
        assert call(B=1 << 16, K=1 << 16) == -2 and b'bad sizes' in err()
        assert call(es=7) == -2 and b'row strides must be >= K' in err()
        assert call(re=None, mask=p, ms=4) == -2 and b'row strides must be >= K' in err()
    assert lib.aa_entropy_hist_lo(p, 8, p, None, 0, 2, 8, None, p, None) == -2
    for q in (-0.01, 1.01, float('nan')):
        assert lib.aa_entropy_select_hi(p, q, p, None) == -2 and b'aa_entropy_select_hi: q must lie in [0, 1]' in err()
    assert lib.aa_entropy_select_hi(None, 0.5, p, None) == -2
    assert lib.aa_entropy_select_lo(p, p, None, None) == -2 and b'aa_entropy_select_lo: null pointer' in err()


def test_entropy_quantile_threshold_checks_before_any_launch(dry):  # noqa: F811
    from align_anything_b200 import ops

    ent = torch.rand(2, 5)
    re = torch.tensor([3, 5], dtype=torch.int32)
    for bad in (dict(q=-0.1), dict(q=1.5), dict(q=True), dict(q='0.5'), dict(entropy=ent.double()),
                dict(entropy=ent[0]), dict(entropy=torch.empty(0, 5)), dict(row_end_or_mask=re.float()),
                dict(row_end_or_mask=torch.ones(3, dtype=torch.int32)), dict(row_end_or_mask=torch.ones(2, 4)),
                dict(row_end_or_mask=re.bool())):
        kw = {**dict(entropy=ent, row_end_or_mask=re, q=0.5), **bad}
        with pytest.raises(ValueError, match='entropy_quantile_threshold'):
            ops.entropy_quantile_threshold(**kw)
    assert dry.calls == []
    thr = ops.entropy_quantile_threshold(ent, re, 0.8)
    assert thr.shape == (1,) and thr.dtype == torch.float32
    assert dry.calls == ['aa_entropy_hist_hi', 'aa_entropy_select_hi', 'aa_entropy_hist_lo', 'aa_entropy_select_lo']
    dry.calls.clear()
    ops.entropy_quantile_threshold(ent, torch.ones(2, 5, dtype=torch.bool), 0.8)
    assert len(dry.calls) == 4


def test_grpo_loss_needs_the_entropy_under_the_mask(dry):  # noqa: F811
    from align_anything_b200 import ops

    lp, ref = torch.rand(2, 5), torch.rand(2, 5)
    adv, tok = torch.rand(2, 1), torch.randint(3, 9, (2, 5))
    obj = ops.GrpoObjective(top_entropy_quantile=0.2)
    with pytest.raises(ValueError, match='top_entropy_quantile < 1 needs the policy entropy'):
        ops.grpo_loss(lp, ref, adv, tok, 2, 0.04, objective=obj)
    assert 'aa_grpo_loss_topent' not in dry.calls
    ops.grpo_loss(lp, ref, adv, tok, 2, 0.04, objective=obj, entropy=torch.rand(2, 5))
    assert dry.calls[-6:] == ['aa_grpo_row_end', 'aa_entropy_hist_hi', 'aa_entropy_select_hi', 'aa_entropy_hist_lo',
                              'aa_entropy_select_lo', 'aa_grpo_loss_topent']


def _trainer(dry, fused, **cfg):
    from align_anything_b200.trainers.text_to_text import grpo as G
    from test_cpu_ppo_step import _LM, _Engine

    t = object.__new__(G.GRPOTrainer)
    t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(**cfg))
    t.actor_model = _Engine(_LM(97, 64, 0, 2, 6, seed=1).bfloat16())
    t.actor_reference_model = _Engine(_LM(97, 64, 0, 2, 6, seed=2).bfloat16())
    t.tokenizer = SimpleNamespace(pad_token_id=0, eos_token_id=2)
    t.beta, t.num_generations, t.fused_lm_head = 0.04, 2, fused
    return t


@pytest.mark.parametrize('fused', [False, True])
def test_rho_one_makes_todays_calls(dry, packed, fused):  # noqa: F811
    runs = []
    for cfg in ({}, {'top_entropy_quantile': 1.0}, {'top_entropy_quantile': None}):
        dry.calls.clear()
        t = _trainer(dry, fused, update_iters=1, **cfg)
        gen = torch.Generator().manual_seed(0)
        t.step_from_rollout(torch.randint(3, 97, (4, 9), generator=gen), 4, torch.randn(4, generator=gen))
        runs.append(list(dry.calls))
    assert runs[0] == runs[1] == runs[2] and 'aa_grpo_loss' in runs[0]
    assert fused or 'aa_logprob_grpo_fused' in runs[0]
    assert not {'aa_grpo_loss_topent', 'aa_entropy_hist_hi', 'aa_grpo_row_end'} & set(runs[0])


@pytest.mark.parametrize('level', ['token', 'sequence'])
@pytest.mark.parametrize('fused', [False, True])
def test_rho_below_one_calls_the_selection_and_never_k1f(dry, packed, monkeypatch, fused, level):  # noqa: F811
    """mu = 2: every update takes its own threshold from its own policy pass, then the masked loss."""
    from align_anything_b200.trainers.text_to_text import grpo as G

    per_update = []
    real = G.policy_update

    def spy(*a, **kw):
        start = len(dry.calls)
        out = real(*a, **kw)
        per_update.append(list(dry.calls[start:]))
        return out

    monkeypatch.setattr(G, 'policy_update', spy)
    t = _trainer(dry, fused, update_iters=2, num_iterations=2, top_entropy_quantile=0.2,
                 importance_sampling_level=level)
    gen = torch.Generator().manual_seed(0)
    t.step_from_rollout(torch.randint(3, 97, (4, 9), generator=gen), 4, torch.randn(4, generator=gen))
    assert len(per_update) == 2
    k1f = {'aa_logprob_grpo_fused', 'aa_logprob_grpo_fused_obj', 'aa_logprob_grpo_fused_kl',
           'aa_logprob_grpo_fused_entropy', 'aa_logprob_grpo_fused_entropy_grad'}
    sel = ['aa_grpo_row_end', 'aa_entropy_hist_hi', 'aa_entropy_select_hi', 'aa_entropy_hist_lo',
           'aa_entropy_select_lo', 'aa_grpo_loss_topent']
    for calls in per_update:
        assert not set(calls) & k1f
        assert not {'aa_grpo_loss', 'aa_grpo_loss_obj', 'aa_grpo_loss_kl', 'aa_grpo_loss_seq'} & set(calls)
        assert [c for c in calls if c in sel] == sel
        if not fused:  # K1's entropy variant before the selection, K1b's after the loss
            assert calls.index('aa_logprob_fwd_entropy') < calls.index('aa_grpo_row_end')
            assert any(c.startswith('aa_logprob_bwd') for c in calls[calls.index('aa_grpo_loss_topent'):])
