"""GSPO's sequence-level ratio without a GPU: the port (tests/gspo_port.py) against float64 autograd and at its rounding
points, ops.GrpoObjective's importance_sampling_level field, the trainer switch, its config precedence and the graft,
the C argument checks of aa_grpo_loss_seq and, on the stand-in library, which entry points each update calls."""
from __future__ import annotations

import ctypes
from types import SimpleNamespace

import pytest
import torch

import gspo_port as port
from grpo_objective_port import completion_mask
from test_cpu_entropy import fake_reference  # noqa: F401  (fixture)
from test_cpu_plumbing import dry  # noqa: F401  (fixture)
from test_cpu_ppo_step import packed  # noqa: F401  (fixture)

AGGS = ['token-mean', 'seq-mean-token-mean', 'seq-mean-token-sum-norm']
ESTIMATORS = ['k1', 'k2', 'k3']


def _inputs(B=6, K=23, seed=0):
    """float64 log-probs with per-row log-ratio means spread inside and outside [1 - 0.2, 1 + 0.28], rows of different
    lengths (one of a single token), advantages of both signs."""
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, K, generator=g, dtype=torch.float64) * 4
    ref = lp + torch.randn(B, K, generator=g, dtype=torch.float64) * 0.3
    shift = torch.tensor([0.0, 0.1, -0.1, 0.5, -0.5, 0.05], dtype=torch.float64)[:B].unsqueeze(-1)
    old = lp - shift + torch.randn(B, K, generator=g, dtype=torch.float64) * 0.02
    adv = torch.tensor([[1.3], [-0.8], [0.6], [-1.7], [2.1], [-0.4]], dtype=torch.float64)[:B]
    tokens = torch.randint(2, 50, (B, K), generator=g)
    tokens[0, 4] = 1
    tokens[2, 0] = 1
    tokens[3, 11] = 1
    return lp, ref, old, adv, tokens


def _f64(x, ref, old, adv, mask, beta, lo, hi, c, agg, est):
    """The objective written row by row, over each row's counted tokens (slices, not masks)."""
    B, K = x.shape
    rows, n_all = [], mask.sum()
    for i in range(B):
        n = int(mask[i].sum())
        a = adv[i, 0]
        w = torch.exp((x[i, :n] - old[i, :n]).sum() / n)
        s = torch.minimum(a * w, a * w.clamp(1 - lo, 1 + hi))
        if c is not None and a < 0:
            s = torch.maximum(s, c * a)
        d = x[i, :n] - ref[i, :n]
        kl = {'k1': d, 'k2': 0.5 * d * d, 'k3': torch.exp(-d) + d - 1}[est]
        rows.append(-(s - beta * kl))
    if agg == 'token-mean':
        return torch.cat(rows).sum() / n_all
    if agg == 'seq-mean-token-mean':
        return torch.stack([r.mean() for r in rows]).mean()
    return torch.cat(rows).sum() / (B * K)


@pytest.mark.parametrize('est', ESTIMATORS)
@pytest.mark.parametrize('dual', [None, 3.0])
@pytest.mark.parametrize('agg', AGGS)
def test_port_matches_float64_autograd(agg, dual, est):
    lp, ref, old, adv, tokens = _inputs()
    mask = completion_mask(tokens, 1)
    assert mask.dtype == torch.int64 and sorted(mask.sum(-1).tolist())[:2] == [1, 5]
    x = lp.clone().requires_grad_(True)
    got = port.grpo_loss(x, ref, adv, mask, 0.04, old, 0.2, 0.28, dual, agg, est)
    got.backward()
    y = lp.clone().requires_grad_(True)
    want = _f64(y, ref, old, adv, mask, 0.04, 0.2, 0.28, dual, agg, est)
    want.backward()
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(x.grad, y.grad, rtol=1e-12, atol=1e-12)
    assert torch.equal(x.grad[mask == 0], torch.zeros_like(x.grad[mask == 0]))


def test_without_old_log_probs_the_port_is_the_token_level_objective():
    from kl_objective_port import grpo_loss as token_loss

    lp, ref, _, adv, tokens = _inputs()
    mask = completion_mask(tokens, 1)
    for agg in AGGS:
        x, y = lp.clone().requires_grad_(True), lp.clone().requires_grad_(True)
        a = port.grpo_loss(x, ref, adv, mask, 0.04, None, 0.2, 0.28, 3.0, agg)
        b = token_loss(y, ref, adv, mask, 0.04, 'k3', None, 0.2, 0.28, 3.0, agg)
        a.backward()
        b.backward()
        assert float(a.detach()) == float(b.detach())
        torch.testing.assert_close(x.grad, y.grad, rtol=1e-12, atol=1e-14)


def _gspo_rows(dtype):
    """bf16 / fp16 rows of 8 counted tokens whose summed log-ratio D sits on token 0 (lp = -0.375, old = lp - D), so
    log_w = D / 8 exactly: 2^-12 lies inside [1 - 3e-4, 1 + 4e-4] on both sides, 2^-11 outside."""
    D = torch.tensor([2.0 ** -9, -2.0 ** -9, 2.0 ** -8, -2.0 ** -8], dtype=torch.float64)
    lp = torch.full((4, 10), -0.375, dtype=dtype)
    old = lp.clone()
    old[:, 0] = (lp[:, 0].double() - D).to(dtype)
    assert torch.equal(lp[:, 0].double() - old[:, 0].double(), D)
    mask = torch.zeros(4, 10, dtype=torch.int64)
    mask[:, :8] = 1
    return lp, old, mask, D / 8


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16])
@pytest.mark.parametrize('sign', [1.0, -1.0])
def test_port_clips_in_fp32_at_gspo_bounds(dtype, sign):
    lp, old, mask, log_w = _gspo_rows(dtype)
    lo, hi = 3e-4, 4e-4
    # in the log-prob dtype both bounds (and w itself) would round to 1
    assert float(torch.tensor(1 - lo).to(torch.bfloat16)) == 1.0 == float(torch.tensor(1 + hi).to(torch.bfloat16))
    got = port.sequence_log_weights(lp, old, mask)
    assert got.dtype == torch.float32 and torch.equal(got.double(), log_w)
    w = torch.exp(log_w)
    outside = (w < 1 - lo) | (w > 1 + hi)
    assert outside.tolist() == [False, False, True, True]
    adv = torch.full((4, 1), sign)
    x = lp.clone().requires_grad_(True)
    loss = port.grpo_loss(x, lp.clone(), adv, mask, 0.0, old, lo, hi)
    loss.backward()
    assert x.grad.dtype == dtype
    g = x.grad.float()
    # the clipped branch carries no gradient: zero exactly where fp32 clips (the branch the minimum takes)
    clipped = (outside & ((sign > 0) == (w > 1))).tolist()
    for i, c in enumerate(clipped):
        assert bool((g[i, :8] == 0).all()) == c, (i, g[i])
        if not c:  # every counted token of the row gets the same coefficient
            assert bool((g[i, :8] == g[i, 0]).all())
    fc, _ = port.clip_fractions(lp, old, adv, mask, lo, hi, agg='seq-mean-token-mean')
    assert fc == sum(clipped) / 4


def test_port_rounds_the_row_sum_once_to_the_log_prob_dtype():
    # 0.25 + 2^-10 is a bf16 tie between 0.25 and 0.25 + 2^-9: the row sum rounds to even, 0.25
    lp = torch.tensor([[-0.5, -0.0625, -0.375]], dtype=torch.bfloat16)
    old = torch.tensor([[-0.75, -0.0625 - 2.0 ** -10, -0.375]], dtype=torch.bfloat16)
    assert float(old[0, 1]) == -0.0625 - 2.0 ** -10
    mask = torch.ones(1, 3, dtype=torch.int64)
    got = port.sequence_log_weights(lp, old, mask)
    assert got.dtype == torch.float32 and float(got) == float(torch.tensor(0.25) / torch.tensor(3.0))


def test_grpo_objective_takes_the_level():
    from align_anything_b200 import ops

    assert ops.GrpoObjective().importance_sampling_level == 'token' and ops.GrpoObjective().is_default
    seq = ops.GrpoObjective(importance_sampling_level='sequence')
    assert not seq.is_default and seq.sequence_level and not ops.GrpoObjective().sequence_level
    assert ops.IMPORTANCE_SAMPLING_LEVELS == ('token', 'sequence')
    for bad in ('Sequence', 'seq', 'tokens', None, 1):
        with pytest.raises(ValueError, match='importance_sampling_level'):
            ops.GrpoObjective(importance_sampling_level=bad)
    # without old log-probs w = 1: the token-level objective and its launches (None: the reference loss)
    assert ops._grpo_objective_args(seq, None, False) is None
    assert ops._grpo_objective_args(seq, None, True) == ops._grpo_objective_args(ops.GrpoObjective(), None, True)
    s2 = ops.GrpoObjective(0.2, 0.28, 3.0, 'seq-mean-token-mean', kl_estimator='k1', importance_sampling_level='sequence')
    old = torch.zeros(2, 3)
    assert ops._grpo_objective_args(s2, None, False) == (0.2, 0.28, 3.0, 0, 0)
    assert ops._grpo_objective_args(s2, old, False) == (0.2, 0.28, 3.0, 0, 0)
    assert ops._sequence_level(s2, old) and not ops._sequence_level(s2, None)
    assert not ops._sequence_level(ops.GrpoObjective(), old) and not ops._sequence_level(None, old)


def test_switch_defaults_to_token_and_config_key_wins():
    from align_anything_b200.ops import GrpoObjective
    from align_anything_b200.trainers.text_to_text import grpo as G

    assert G.GRPOTrainer.importance_sampling_level == 'token'
    assert 'importance_sampling_level' in G.GRPO_OBJECTIVE_KEYS and 'importance_sampling_level' in G.GRPOTrainer.SWITCHES
    tr = G.GRPOTrainer()
    assert G.grpo_objective_of(tr) is None
    tc = SimpleNamespace(update_iters=2, num_iterations=2, importance_sampling_level=None)
    tr = G.GRPOTrainer(SimpleNamespace(train_cfgs=tc))
    assert G.grpo_objective_of(tr) == GrpoObjective()
    tr.importance_sampling_level = 'sequence'
    assert G.grpo_objective_of(tr) == GrpoObjective(importance_sampling_level='sequence')
    tr.importance_sampling_level = 'token'
    tc.importance_sampling_level = 'sequence'  # the recipe's value wins over the attribute
    assert G.grpo_objective_of(tr).importance_sampling_level == 'sequence'
    tc.importance_sampling_level = 'group'
    with pytest.raises(ValueError, match='importance_sampling_level'):
        G.grpo_objective_of(tr)


def test_install_grafts_the_level_switch(fake_reference):  # noqa: F811
    from align_anything_b200 import patch

    grpo = {m: c for m, c in fake_reference.items() if 'grpo' in m}
    assert grpo
    try:
        patch.install(models=False)
        for modname, cls in grpo.items():
            assert cls.__dict__.get('importance_sampling_level') == 'token', modname
    finally:
        patch.uninstall()
    for modname, cls in grpo.items():
        assert 'importance_sampling_level' not in cls.__dict__, modname


def test_aa_grpo_loss_seq_checks_its_arguments_before_cuda():
    from align_anything_b200 import _lib

    lib = _lib.lib()
    buf = (ctypes.c_int64 * 8)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def seq(old, lo=0.2, hi=0.2, c=0.0, agg=1, est=2, mode=0):
        return lib.aa_grpo_loss_seq(p, 8, p, 8, old, 8, 2, p, p, 8, 1, 2, 8, 0.04, lo, hi, c, agg, est, mode, p, p, 8,
                                    None, p, p, p, None)

    assert seq(None) == -2 and b'aa_grpo_loss_seq: the sequence-level ratio needs old_log_probs' in lib.aa_last_error()
    for bad in ((1.0, 0.2, 0.0, 1), (-0.1, 0.2, 0.0, 1), (0.2, 0.2, 0.5, 1), (0.2, 0.2, 0.0, 3),
                (float('nan'), 0.2, 0.0, 1)):
        assert seq(p, *bad) == -2 and b'aa_grpo_loss_seq: bad objective' in lib.aa_last_error(), bad
    for est in (-1, 3):
        assert seq(p, est=est) == -2 and b'aa_grpo_loss_seq: unknown kl_estimator' in lib.aa_last_error()
    assert seq(p, mode=5) == -2 and b'aa_grpo_loss_seq: bad mode' in lib.aa_last_error()
    rc = lib.aa_grpo_loss_seq(None, 8, p, 8, p, 8, 2, p, p, 8, 1, 2, 8, 0.04, 0.2, 0.2, 0.0, 1, 2, 0, p, p, 8, None, p,
                              p, p, None)
    assert rc == -2 and b'aa_grpo_loss_seq: bad arguments' in lib.aa_last_error()


@pytest.mark.parametrize('fused', [False, True])
@pytest.mark.parametrize('level', ['token', 'sequence'])
def test_updates_call_the_entry_points_the_level_asks_for(dry, packed, monkeypatch, fused, level):  # noqa: F811
    """mu = 2: update 1 (no old log-probs) runs the token-level launches at either level; update 2 at sequence level
    runs aa_grpo_loss_seq on the composed path and never K1f."""
    from align_anything_b200.trainers.text_to_text import grpo as G
    from test_cpu_ppo_step import _LM, _Engine

    per_update = []
    real = G.policy_update

    def spy(*a, **kw):
        start = len(dry.calls)
        out = real(*a, **kw)
        per_update.append(set(dry.calls[start:]))
        return out

    monkeypatch.setattr(G, 'policy_update', spy)
    t = object.__new__(G.GRPOTrainer)
    t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(update_iters=2, num_iterations=2,
                                                        importance_sampling_level=level))
    t.actor_model = _Engine(_LM(97, 64, 0, 2, 6, seed=1).bfloat16())
    t.actor_reference_model = _Engine(_LM(97, 64, 0, 2, 6, seed=2).bfloat16())
    t.tokenizer = SimpleNamespace(pad_token_id=0, eos_token_id=2)
    t.beta, t.num_generations, t.fused_lm_head = 0.04, 2, fused
    gen = torch.Generator().manual_seed(0)
    t.step_from_rollout(torch.randint(3, 97, (4, 9), generator=gen), 4, torch.randn(4, generator=gen))
    assert len(per_update) == 2
    k1f = {'aa_logprob_grpo_fused', 'aa_logprob_grpo_fused_obj', 'aa_logprob_grpo_fused_kl'}
    first, second = per_update
    # w = 1: the token-level objective at its default fields, so today's launches at either level
    assert 'aa_grpo_loss_seq' not in first and 'aa_grpo_loss_obj' not in first
    assert 'aa_grpo_loss' in first and (fused or 'aa_logprob_grpo_fused' in first)
    if level == 'token':
        assert 'aa_grpo_loss_seq' not in second and 'aa_grpo_loss_obj' in second
        assert fused or 'aa_logprob_grpo_fused_obj' in second
    else:
        assert 'aa_grpo_loss_seq' in second and not (second & k1f)
        assert not {'aa_grpo_loss', 'aa_grpo_loss_obj', 'aa_grpo_loss_kl'} & second
        assert fused or {'aa_logprob_fwd', 'aa_logprob_bwd'} <= second


def test_single_update_at_sequence_level_runs_todays_launches(dry, packed):  # noqa: F811
    from align_anything_b200.trainers.text_to_text import grpo as G
    from test_cpu_ppo_step import _LM, _Engine

    runs = []
    for level in ('token', 'sequence'):
        dry.calls.clear()
        t = object.__new__(G.GRPOTrainer)
        t.cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(update_iters=1, importance_sampling_level=level))
        t.actor_model = _Engine(_LM(97, 64, 0, 2, 6, seed=1).bfloat16())
        t.actor_reference_model = _Engine(_LM(97, 64, 0, 2, 6, seed=2).bfloat16())
        t.tokenizer = SimpleNamespace(pad_token_id=0, eos_token_id=2)
        t.beta, t.num_generations, t.fused_lm_head = 0.04, 2, False
        gen = torch.Generator().manual_seed(0)
        t.step_from_rollout(torch.randint(3, 97, (4, 9), generator=gen), 4, torch.randn(4, generator=gen))
        runs.append(list(dry.calls))
    assert runs[0] == runs[1] and 'aa_logprob_grpo_fused' in runs[0] and 'aa_grpo_loss' in runs[0]
