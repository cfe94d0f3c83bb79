"""Policy entropy from the log-prob kernels (H100).

* K1's entropy variant (aa_logprob_fwd_entropy) against a float64 oracle on guard-banded, poisoned buffers, for bf16 /
  fp16 / fp32 logits, both K1 kernels (bulk-copy ring for short rows, LDG for long ones), dense, tail and two-copy row
  plans, near one-hot, uniform, partly -inf and all -inf rows, ignored and unscored rows;
* K6's (aa_linear_logprob_fwd_entropy) against float64 with and without the split-vocabulary merge;
* the GRPO single pass (aa_logprob_grpo_fused_entropy) against float64;
* bit-identity: log-probs, statistics, loss and gradient tiles of each entropy launch equal the plain launch's;
* the trainers' `log_entropy` switch: `train/entropy` against a float64 recompute, every other key unchanged, and the
  fused lm_head path against the logits-tile path.
"""
from __future__ import annotations

from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from test_gpu_fused_rl import LM, Critic, Phased, _grpo_sequences, _ppo_batch, _run_grpo, _run_ppo
from test_gpu_parity import ops  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOL = 1e-4  # absolute, per row
POISON = float('nan')
GUARD = 64


def entropy64(x: torch.Tensor) -> torch.Tensor:
    """-(softmax * log_softmax).sum(-1) in float64 with 0 * log 0 = 0 (a -inf logit adds nothing); a row of -inf only
    is NaN, as the plain torch expression gives."""
    x = x.double()
    lp = x - torch.logsumexp(x, -1, keepdim=True)
    p = lp.exp()
    h = -torch.where(p > 0, p * lp, torch.zeros_like(p)).sum(-1)
    return torch.where(torch.isinf(x).all(-1) & (x < 0).all(-1), torch.full_like(h, float('nan')), h)


def _logits(B, L, V, dtype, seed):
    """Random rows plus the edge cases: near one-hot, uniform, half -inf, all -inf."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(B, L, V, generator=gen) * 3.0
    x[0, 0] = 0.0
    x[0, 0, 7] = 40.0                    # H ~ V * 40 e^-40: 0 to fp32 precision
    x[0, 1] = 1.5                        # uniform: H = log V
    x[0, 2, ::2] = float('-inf')         # half the vocabulary masked
    if L > 3:
        x[0, 3] = float('-inf')          # nothing left: NaN
    return x.to(dtype).to(DEV)


def _bits(t):
    """The raw bits (NaN == NaN): bit-identity checks on outputs that hold the NaN of an all -inf row."""
    return t.contiguous().view({2: torch.int16, 4: torch.int32}[t.element_size()])


def _same(a, b):
    return a.dtype == b.dtype and torch.equal(_bits(a), _bits(b))


def _check(got, want, what):
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan), f'{what}: NaN pattern'
    err = (got.double() - want)[~nan].abs()
    assert float(err.max()) <= TOL, f'{what}: max abs error {float(err.max()):.3e}'


DTYPES = [torch.bfloat16, torch.float16, torch.float32]
VOCABS = [32001, 128257, 152064]


@pytest.mark.parametrize('V', VOCABS)
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'f16', 'f32'])
def test_k1_entropy_dense_guarded(ops, dtype, V):
    """Direct ABI launch on poisoned buffers with guard bands: every scored row is written, ignored rows get exactly 0,
    rows at or past n_entropy and the guards are left alone; log-probs and statistics equal aa_logprob_fwd's."""
    from align_anything_b200 import _lib as L

    B, Lr = 2, 6
    x = _logits(B, Lr, V, dtype, seed=V % 97)
    labels = torch.randint(0, V, (B, Lr), generator=torch.Generator().manual_seed(3)).to(DEV)
    labels[1, 2] = -100  # ignored
    n = B * Lr
    plan = ops._dense_plan(B, Lr, Lr * V, V, Lr, 0, Lr, n, DEV)
    p = plan.ptrs()
    lib, st = L.lib(), L.stream_ptr(x.device)
    runs = {}
    for with_ent in (False, True):
        out = torch.full((n + 2 * GUARD,), POISON, dtype=torch.float32, device=DEV)
        stats = torch.full((2, n + 2 * GUARD), POISON, dtype=torch.float32, device=DEV)
        ent = torch.full((n + 2 * GUARD,), POISON, dtype=torch.float32, device=DEV)
        n_ent = n - Lr // 2  # the last rows are not the caller's: they must stay untouched
        args = (x.data_ptr(), L.dtype_code(dtype), V, V, labels.data_ptr(), -100, 1, plan.n_seg, plan.n_rows,
                p[0], p[1], p[2], p[3], out[GUARD:].data_ptr(), L.AA_F32, stats[0, GUARD:].data_ptr(),
                stats[1, GUARD:].data_ptr(), None)
        if with_ent:
            L.check(lib.aa_logprob_fwd_entropy(*args, ent[GUARD:].data_ptr(), n_ent, st))
        else:
            L.check(lib.aa_logprob_fwd(*args, st))
        runs[with_ent] = (out, stats, ent, n_ent)
    (o0, s0, _, _), (o1, s1, e1, n_ent) = runs[False], runs[True]
    assert torch.equal(o0.view(torch.int32), o1.view(torch.int32)), 'log-probs differ with the entropy on'
    assert torch.equal(s0.view(torch.int32), s1.view(torch.int32)), 'statistics differ with the entropy on'
    assert bool(torch.isnan(e1[:GUARD]).all() and torch.isnan(e1[GUARD + n_ent:]).all()), 'guard / foreign rows written'
    got = e1[GUARD:GUARD + n_ent]
    want = entropy64(x.view(n, V).float().cpu())[:n_ent].to(DEV)
    ign = torch.zeros(n, dtype=torch.bool)
    ign[1 * Lr + 2] = True
    ign = ign[:n_ent].to(DEV)
    assert bool((got[ign] == 0).all()), 'ignored row entropy must be exactly 0'
    _check(got[~ign], want[~ign], f'K1 dense {dtype} V={V}')


@pytest.mark.parametrize('V', VOCABS)
@pytest.mark.parametrize('dtype', DTYPES, ids=['bf16', 'f16', 'f32'])
def test_k1_entropy_plans(ops, dtype, V):
    """gather (dense view `[:, :-1]`, with a gradient: bit-identical tile too), tail_token_log_probs (tail plan, unscored
    rows exactly 0 in the padded layout) and the two-copy pair (actor entropy only)."""
    B, Lq = 2, 7
    x = _logits(B, Lq, V, dtype, seed=11 + V % 13)
    ids = torch.randint(0, V, (B, Lq), generator=torch.Generator().manual_seed(5)).to(DEV)
    ref = entropy64(x.float().cpu()).to(DEV)  # (B, Lq): entropy of every position's row

    # dense, through autograd: same log-probs and same gradient tile with and without the entropy
    xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    lp0 = ops.gather_log_probabilities(xa[:, :-1], ids[:, 1:])
    lp1, ent = ops.gather_log_probabilities_with_entropy(xb[:, :-1], ids[:, 1:])
    assert not ent.requires_grad and ent.dtype == torch.float32
    assert _same(lp0, lp1)
    g = torch.randn(lp0.shape, generator=torch.Generator().manual_seed(9)).to(DEV).to(lp0.dtype)
    g[0, 3] = 0  # the all -inf row: its gradient is NaN, keep it out of the comparison
    lp0.backward(g)
    lp1.backward(g)
    assert torch.equal(xa.grad.view(-1).view(torch.uint8), xb.grad.view(-1).view(torch.uint8)), 'gradient tile differs'
    _check(ent, ref[:, :-1], f'gather {dtype} V={V}')

    # tail plan: the last K positions' predictions
    K = 4
    lpt, ent_t = ops.tail_token_log_probs(x, ids, K, return_entropy=True)
    assert _same(lpt, ops.tail_token_log_probs(x, ids, K))
    _check(ent_t, ref[:, -K - 1:-1], f'tail {dtype} V={V}')

    # two copies in one launch, per-sample response lengths (unscored padding must be exactly 0)
    y = _logits(B, Lq, V, dtype, seed=23)
    lens = [3, 5]
    a0, b0 = ops.response_tail_log_probs_pair(x, y, ids, lens)
    a1, b1, ent_p = ops.response_tail_log_probs_pair_with_entropy(x, y, ids, lens)
    assert _same(a0, a1) and _same(b0, b1)
    W = max(lens)
    for b, r in enumerate(lens):
        _check(ent_p[b, :r], ref[b, Lq - 1 - r:Lq - 1], f'pair {dtype} V={V} sample {b}')
        assert bool((ent_p[b, r:W] == 0).all()), 'unscored padding must be exactly 0'
    ops.check_status()


def _k6_operands(N, H, V, seed):
    """Small-integer operands: every product and partial sum is exact in fp32, so the float64 oracle sees the kernel's
    logits bit for bit (before the bf16 rounding both apply)."""
    gen = torch.Generator().manual_seed(seed)
    h = torch.randint(-3, 4, (N, H), generator=gen).float()
    w = torch.randint(-2, 3, (V, H), generator=gen).float() / 8
    lab = torch.randint(0, V, (N,), generator=gen)
    return h.bfloat16().to(DEV), w.bfloat16().to(DEV), lab.to(DEV)


@pytest.mark.parametrize('split', [False, True], ids=['one-split', 'v-splits'])
@pytest.mark.parametrize('N', [130, 1100])
def test_k6_entropy(ops, N, split):
    """K6 against float64 on exact operands, FAITHFUL (bf16-rounded logits) and F32; with `partial` the vocabulary is split
    across CTAs (few row tiles) and merged by the second launch, without it one CTA sweeps the whole vocabulary."""
    from align_anything_b200 import _lib as L

    H, V = 128, 32001
    h, w, lab = _k6_operands(N, H, V, seed=N)
    logits = h.double().cpu() @ w.double().cpu().t()
    lib, st = L.lib(), L.stream_ptr(h.device)
    for mode in (L.MODE_FAITHFUL, L.MODE_F32):
        x = logits.to(torch.bfloat16).double() if mode == L.MODE_FAITHFUL else logits
        want = entropy64(x).to(DEV)
        res = {}
        for with_ent in (False, True):
            out = torch.full((N,), POISON, dtype=torch.float32, device=DEV)
            stats = torch.full((2, N), POISON, dtype=torch.float32, device=DEV)
            ent = torch.full((N + 2 * GUARD,), POISON, dtype=torch.float32, device=DEV)
            part = torch.empty(4 * 132 * 128, dtype=torch.float32, device=DEV) if split else None
            args = (h.data_ptr(), N, H, H, w.data_ptr(), V, H, lab.data_ptr(), out.data_ptr(), L.AA_F32,
                    stats[0].data_ptr(), stats[1].data_ptr(), L.ptr(part), 0 if part is None else part.numel(), mode, None)
            if with_ent:
                L.check(lib.aa_linear_logprob_fwd_entropy(*args, ent[GUARD:].data_ptr(), st))
            else:
                L.check(lib.aa_linear_logprob_fwd(*args, st))
            res[with_ent] = (out, stats, ent)
        assert torch.equal(res[False][0].view(torch.int32), res[True][0].view(torch.int32)), 'K6 log-probs differ'
        assert torch.equal(res[False][1].view(torch.int32), res[True][1].view(torch.int32)), 'K6 statistics differ'
        ent = res[True][2]
        assert bool(torch.isnan(ent[:GUARD]).all() and torch.isnan(ent[GUARD + N:]).all()), 'guards written'
        _check(ent[GUARD:GUARD + N], want, f'K6 N={N} split={split} mode={mode}')


def test_k6_entropy_through_ops(ops):
    """fused_linear_token_log_probs / linear_token_log_probs (K6 forward inside the autograd node, and the library-GEMM
    path around K1) return the same log-probs and gradients with the entropy on."""
    N, H, V = 300, 128, 2053
    h, w, lab = _k6_operands(N, H, V, seed=3)
    want = entropy64((h.double().cpu() @ w.double().cpu().t()).to(torch.bfloat16).double()).to(DEV)
    lp0, st0 = ops.fused_linear_token_log_probs(h, w, lab, return_stats=True)
    lp1, st1, ent = ops.fused_linear_token_log_probs(h, w, lab, return_stats=True, return_entropy=True)
    assert torch.equal(lp0, lp1) and torch.equal(st0, st1)
    _check(ent, want, 'fused_linear_token_log_probs')
    for head_dtype in (torch.bfloat16, torch.float16):  # tensor-core path, then library GEMMs around K1
        ha, wa = (t.to(head_dtype).clone().requires_grad_(True) for t in (h, w))
        hb, wb = (t.to(head_dtype).clone().requires_grad_(True) for t in (h, w))
        l0 = ops.linear_token_log_probs(ha, wa, lab, chunk_rows=128)
        l1, e1 = ops.linear_token_log_probs(hb, wb, lab, chunk_rows=128, return_entropy=True)
        assert torch.equal(l0, l1) and not e1.requires_grad
        l0.float().sum().backward()
        l1.float().sum().backward()
        assert torch.equal(ha.grad, hb.grad) and torch.equal(wa.grad, wb.grad)
        x = (h.double().cpu() @ w.double().cpu().t()).to(head_dtype).double()
        _check(e1, entropy64(x).to(DEV), f'linear_token_log_probs {head_dtype}')


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32], ids=['bf16', 'f32'])
def test_grpo_fused_entropy(ops, dtype):
    """K1f (GRPO): loss, log-probs, counted tokens and the gradient tile are bit-identical with the entropy on; the
    entropy of every completion row matches float64."""
    B, Lq, K, V = 4, 12, 6, 128257
    x = _logits(B, Lq, V, dtype, seed=77)
    x[0, 3] = 0.25  # the single pass rows stay finite (the all -inf case is K1's above)
    ids = torch.randint(2, V, (B, Lq), generator=torch.Generator().manual_seed(8)).to(DEV)
    ids[1, Lq - K + 2] = 1  # an eos inside one completion
    ref_lp = (torch.randn(B, K, generator=torch.Generator().manual_seed(2)) - 10).to(DEV)
    adv = torch.randn(B, 1, generator=torch.Generator().manual_seed(4)).to(DEV)
    assert ops._single_pass_ok(x, ops._FUSED_GRPO, True), 'these rows must take the single pass'
    xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    loss0, lp0, re0 = ops.grpo_loss_from_logits(xa, ids, K, ref_lp, adv, 1, 0.04)
    loss1, lp1, re1, ent = ops.grpo_loss_from_logits(xb, ids, K, ref_lp, adv, 1, 0.04, return_entropy=True)
    assert torch.equal(loss0, loss1) and torch.equal(lp0, lp1) and torch.equal(re0, re1)
    loss0.backward()
    loss1.backward()
    assert torch.equal(xa.grad.view(torch.uint8), xb.grad.view(torch.uint8)), 'gradient tile differs'
    _check(ent, entropy64(x.float().cpu()).to(DEV)[:, -K - 1:-1], f'GRPO K1f {dtype}')
    ops.check_status()


# ---- trainers ---------------------------------------------------------------------------------------------------------
def _with_entropy(cls):
    return type(cls.__name__, (cls,), {'log_entropy': True})


def _actor_entropy(hid, w):
    """float64 entropy of every position of the rollout actor's logits, F.linear(hidden, weight) as the tile path sees
    them (the fused path rounds its own fp32 accumulators: within an ulp of these)."""
    return entropy64(F.linear(hid.to(DEV), w.to(DEV)).cpu()).to(DEV)


def _ppo_entropy_ref(ids, hid, w, start):
    """train/entropy of the text trainers: per-row sum over the rl_step mask from `start` on, mean over rows."""
    ent = _actor_entropy(hid, w)[:, :-1]
    mask = (ids != 0)[:, 1:].double()
    return float((ent[:, start:] * mask[:, start:]).sum(-1).mean())


def _check_trainer(off, on, want, fused, what):
    assert set(on) == set(off) | {'train/entropy'} and 'train/entropy' not in off, what
    for k, v in off.items():
        assert on[k] == v, (what, k, v, on[k])
    assert abs(on['train/entropy'] - want) <= TOL * max(1.0, abs(want)) * 10, (what, on['train/entropy'], want)


@pytest.mark.parametrize('trainer', ['text', 'multi-gae', 'multi-rloo'])
def test_text_ppo_log_entropy(ops, trainer):
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer as Multi
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer as Text

    cls, kw = (Text, {}) if trainer == 'text' else (Multi, {'advantage_estimator': trainer.split('-')[1],
                                                             'n_samples_per_prompt': 2})
    ids = _ppo_batch(5)
    P, H, V, seed = 12, 128, 2053, 41
    got = {}
    for fused in (False, True):
        off = _run_ppo(cls, fused, ids, P, H, V, seed, **kw)
        on = _run_ppo(_with_entropy(cls), fused, ids, P, H, V, seed, **kw)
        gen = torch.Generator().manual_seed(seed)  # _run_ppo's first draws: the rollout actor's hidden states, weight
        hid_a = (torch.randn(ids.size(0), ids.size(1), H, generator=gen)).bfloat16()
        for _ in range(2):
            torch.randn(ids.size(0), ids.size(1), H, generator=gen)
        w_a = (torch.randn(V, H, generator=gen) * 0.2).bfloat16()
        want = _ppo_entropy_ref(ids, hid_a, w_a, P - 1)
        assert torch.equal(on[0]['log_probs'], off[0]['log_probs'])
        _check_trainer(off[1], on[1], want, fused, f'{trainer} fused={fused}')
        got[fused] = on[1]['train/entropy']
    assert abs(got[True] - got[False]) <= TOL * max(1.0, abs(got[False])) * 10, got
    ops.check_status()


def test_image_ppo_log_entropy(ops):
    from align_anything_b200.models.reward_model import ScoreModelOutput
    from align_anything_b200.trainers.text_image_to_text.ppo import PPOTrainer

    gen = torch.Generator().manual_seed(31)
    B, Lq, H, V = 3, 40, 128, 1031
    resp = [20, 9, 28]
    seq = torch.zeros((B, Lq), dtype=torch.int64)
    for b, r in enumerate(resp):
        seq[b, Lq - r - 8:] = torch.randint(2, V, (r + 8,), generator=gen)
    ids = seq.to(DEV)
    t = lambda *shape, s=1.0: (torch.randn(*shape, generator=gen) * s)
    hid_a, hid_r, hid_new = (t(B, Lq, H).bfloat16().to(DEV) for _ in range(3))
    w_a = t(V, H, s=0.2).bfloat16().to(DEV)
    w_r = (w_a.float().cpu() + t(V, H, s=0.02)).bfloat16().to(DEV)
    reward = t(B).to(DEV)
    critic, new_critic = t(B, Lq, 1).to(DEV), t(B, Lq, 1).to(DEV)

    def run(cls, fused):
        h_new, w_new = hid_new.clone().requires_grad_(True), w_a.clone().requires_grad_(True)
        tr = cls(None, tokenizer=SimpleNamespace(pad_token_id=0))
        tr.fused_lm_head, tr.lm_head_chunk_rows = fused, 32
        state = {'phase': 'rollout'}
        tr.actor_model = Phased(LM(hid_a, w_a), LM(h_new, w_new), state)
        tr.actor_reference_model = LM(hid_r, w_r)
        tr.reward_model = Critic(lambda: ScoreModelOutput(end_scores=reward.unsqueeze(-1)))
        g_critic = new_critic.clone().requires_grad_(True)
        tr.reward_critic_model = Critic(lambda: ScoreModelOutput(scores=critic if state['phase'] == 'rollout' else g_critic))
        inference, training = tr.score_rollout({'input_ids': ids, 'attention_mask': ids != 0}, resp)
        state['phase'] = 'train'
        return training, tr.rl_step(inference, training)

    ent_all = _actor_entropy(hid_a, w_a)
    got = {}
    for fused in (False, True):
        tr_off, off = run(PPOTrainer, fused)
        tr_on, on = run(_with_entropy(PPOTrainer), fused)
        tails = torch.zeros(B, max(resp), dtype=torch.float64, device=DEV)
        for b, r in enumerate(resp):
            tails[b, :r] = ent_all[b, Lq - 1 - r:Lq - 1]
        want = float((tails * tr_on['response_mask']).sum(-1).mean())
        _check_trainer(off, on, want, fused, f'image fused={fused}')
        got[fused] = on['train/entropy']
    assert abs(got[True] - got[False]) <= TOL * max(1.0, abs(got[False])) * 10, got
    ops.check_status()


def test_grpo_log_entropy(ops, monkeypatch):
    from align_anything_b200.trainers.text_to_text.grpo import GRPOTrainer

    seq = _grpo_sequences(7)
    P, H, V, seed = 16, 128, 2053, 47
    got = {}
    for fused in (False, True):
        off = _run_grpo(fused, seq, P, H, V, seed)[0]
        monkeypatch.setattr(GRPOTrainer, 'log_entropy', True)
        on = _run_grpo(fused, seq, P, H, V, seed)[0]
        monkeypatch.setattr(GRPOTrainer, 'log_entropy', False)
        gen = torch.Generator().manual_seed(seed)
        hid = torch.randn(seq.size(0), seq.size(1), H, generator=gen).bfloat16()
        torch.randn(seq.size(0), seq.size(1), H, generator=gen)
        w = (torch.randn(V, H, generator=gen) * 0.2).bfloat16()
        K = seq.size(1) - P
        ent = _actor_entropy(hid, w)[:, -K - 1:-1].cpu()
        tok = seq[:, -K:].cpu()
        first_eos = torch.where((tok == 1).any(1), (tok == 1).int().argmax(1) + 1, torch.full((tok.size(0),), K))
        mask = (torch.arange(K) < first_eos.unsqueeze(1)).double()
        want = float((ent * mask).sum() / mask.sum())
        _check_trainer(off, on, want, fused, f'grpo fused={fused}')
        got[fused] = on['train/entropy']
    assert abs(got[True] - got[False]) <= TOL * max(1.0, abs(got[False])) * 10, got
    ops.check_status()
