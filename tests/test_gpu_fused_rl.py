"""The fused lm_head path of the text RL trainers (run on an H100: `pytest -m gpu`).

* ops.dense_log_probs_from_hidden against `token_log_probs(F.linear(hidden, weight)[:, :-1], ids[:, 1:])[:, start:]`
  on ATen CUDA kernels: faithful bf16 within 2 ulp and >= 95 % bit-identical (the bar of K6 in the DPO path), f32 mode
  within 2e-5; with a gradient, d(hidden) and d(weight) against float64 products of autograd's d(logits) tile, to the
  GEMM bar of test_gpu_lm_head_tiles plus what may separate the two d(logits) tiles (_dlogits_slack).
* The text PPO, Multi-PPO (all five estimators) and GRPO trainers with `fused_lm_head = True` against the same trainer
  fed `F.linear(hidden, weight)` logits: rollout log-probs (full width, prompt and pad positions included), every
  rl_step metric, last_rl_tensors, the GRPO loss and reward, d(hidden) and d(weight).
* An out-of-range label raises the same exception class with the switch on as with it off.
"""
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from oracle import ref_port as O
from test_gpu_lm_head_tiles import _bound, _half_ulp_bf16
from test_gpu_parity import assert_close_f32, assert_ulp_close, ops  # noqa: F401  (ops: fixture)

pytestmark = pytest.mark.gpu

DEV = 'cuda'


def _operands(B, Lq, H, V, seed):
    gen = torch.Generator().manual_seed(seed)
    hidden = torch.randn(B, Lq, H, generator=gen).bfloat16().to(DEV)
    weight = (torch.randn(V, H, generator=gen) * (2.5 / H ** 0.5)).bfloat16().to(DEV)
    ids = torch.randint(0, V, (B, Lq), generator=gen).to(DEV)
    ids[0, -1], ids[-1, 1] = V - 1, 0
    return hidden, weight, ids


def _ulp_bf16(a64):
    """One bf16 ulp at |a| (float64), taken one percent above |a| so that a neighbour in the next binade is covered."""
    return 2.0 * _half_ulp_bf16(a64.abs() * 1.01)


def _dlogits_slack(logits, dl, g_rows):
    """Per element, how far K6b's d(logits) may lie from ATen's `dl`.  Both tiles are g * (onehot - p) with
    p = exp(bf16((bf16(x) - max) - logsum)); the exact one-hot term is shared.  The two GEMMs accumulate in fp32 in
    different orders, so every bf16(x) may differ by one ulp of x; the row's log-sum-exp then moves by up to
    s = sum_u p_u * ulp(x_u), and the rounded log-softmax ls by ulp(x) + s plus one ulp of ls; exp (ex2.approx of
    ls * log2(e) on our side) adds < 2^-18 relative; rounding the result to bf16 one ulp of d(logits).  So
    |delta| <= |g| * p * (exp(ulp(x) + s + ulp(ls)) - 1 + 2^-18) + ulp(d(logits))."""
    x = logits.detach().double()
    ls = torch.log_softmax(logits.detach(), dim=-1).double()  # ATen's bf16 log-softmax: what its backward re-reads
    p, ux = torch.exp(ls), _ulp_bf16(x)
    shift = 1.01 * (p * ux).sum(-1, keepdim=True)
    return g_rows.abs()[..., None] * p * (torch.expm1(ux + shift + _ulp_bf16(ls)) + 2.0 ** -18) \
        + _ulp_bf16(dl.abs()) * (g_rows != 0)[..., None]


# (B, L, H, V, start)
OP_CASES = [
    (3, 40, 128, 2053, 0), (3, 40, 128, 2053, 17), (3, 40, 128, 2053, 38),
    (2, 24, 4096, 1031, 0), (2, 24, 4096, 1031, 11), (2, 24, 4096, 1031, 22),
    (2, 40, 4096, 128257, 9),
]


@pytest.mark.parametrize('case', OP_CASES, ids=[f'B{c[0]}-L{c[1]}-H{c[2]}-V{c[3]}-start{c[4]}' for c in OP_CASES])
def test_dense_log_probs_from_hidden(ops, case):
    B, Lq, H, V, start = case
    hidden, weight, ids = _operands(B, Lq, H, V, B * Lq + H + V + start)
    W = Lq - 1 - start
    # forward, both modes, no gradient (K6)
    want = O.token_log_probs(F.linear(hidden, weight)[:, :-1], ids[:, 1:])[:, start:]
    with torch.no_grad():
        got = ops.dense_log_probs_from_hidden(hidden, weight, ids, start)
    assert got.shape == (B, W) and got.dtype == want.dtype == torch.bfloat16
    assert_ulp_close(got, want, max_ulp=2, min_exact=0.95, what='faithful log-probs')
    want32 = O.token_log_probs(F.linear(hidden.float(), weight.float())[:, :-1], ids[:, 1:])[:, start:]
    with torch.no_grad():
        got32 = ops.dense_log_probs_from_hidden(hidden, weight, ids, start, mode='f32')
    assert got32.dtype == torch.float32
    assert_close_f32(got32, want32, what='f32 log-probs')
    # with a gradient (K6 + K6b + d(hidden) + d(weight)): the same log-probs, and the gradients of autograd's chain
    gen = torch.Generator().manual_seed(start + 1)
    g = torch.randn(B, W, generator=gen).bfloat16().to(DEV)
    h, w = hidden.clone().requires_grad_(True), weight.clone().requires_grad_(True)
    lp = ops.dense_log_probs_from_hidden(h, w, ids, start)
    assert_ulp_close(lp.detach(), want, max_ulp=2, min_exact=0.95, what='log-probs with a gradient')
    lp.backward(g)
    logits = F.linear(hidden, weight).requires_grad_(True)
    O.token_log_probs(logits[:, :-1], ids[:, 1:])[:, start:].backward(g)
    dl = logits.grad.double()  # (B, L, V); rows outside [start, L - 1) are zero
    g_rows = torch.zeros(B, Lq, dtype=torch.float64, device=DEV)
    g_rows[:, start:Lq - 1] = g.double()
    slack = _dlogits_slack(logits, dl, g_rows)  # zero on unscored rows
    del logits
    # the GEMM bar of test_gpu_lm_head_tiles (_bound, over |d(logits)| widened by the slack) plus the slack carried
    # through the GEMM
    ref = dl @ weight.double()
    slack_prod = slack @ weight.double().abs()
    bar = _bound(ref, dl.abs() @ weight.double().abs() + slack_prod, V) + slack_prod
    err = (h.grad.double() - ref).abs()
    assert bool((err <= bar).all()), f'd(hidden): {int((err > bar).sum())} beyond the bar, max err / bar {float((err / bar).max()):.3f}'
    assert bool((h.grad[:, :start] == 0).all() and (h.grad[:, Lq - 1:] == 0).all()), 'd(hidden) of unscored rows'
    del ref, bar, err
    dl2, sl2, h2 = dl.view(-1, V), slack.view(-1, V), hidden.reshape(-1, H).double()
    for v0 in range(0, V, 16384):  # vocabulary blocks: float64 (V, H) temporaries would take 4 GB each at V = 128257
        blk = dl2[:, v0:v0 + 16384].T
        ref = blk @ h2
        slack_prod = sl2[:, v0:v0 + 16384].T @ h2.abs()
        bar = _bound(ref, blk.abs() @ h2.abs() + slack_prod, Lq * B) + slack_prod
        err = (w.grad[v0:v0 + 16384].double() - ref).abs()
        assert bool((err <= bar).all()), \
            f'd(weight) rows {v0}+: {int((err > bar).sum())} beyond the bar, max err / bar {float((err / bar).max()):.3f}'
    ops.check_status()


# ---- the trainers, fused against the same trainer fed F.linear logits ---------------------------------------------------
class LM:
    """A causal LM reduced to its last hidden states and its lm_head: the fused path asks for the hidden states, the
    default path gets F.linear(hidden, weight)."""

    def __init__(self, hidden, weight):
        self.hidden, self.weight = hidden, weight
        self.optimizer = SimpleNamespace(param_groups=[{'lr': 1e-6}])

    def __call__(self, output_hidden_states=False, logits_to_keep=0, **kw):
        if output_hidden_states:
            assert logits_to_keep == 1
            return SimpleNamespace(hidden_states=(None, self.hidden), logits=None)
        return SimpleNamespace(logits=F.linear(self.hidden, self.weight))

    def get_output_embeddings(self):
        return SimpleNamespace(weight=self.weight)

    def backward(self, loss):
        loss.backward()

    def step(self):
        pass

    def zero_grad(self):
        pass


class Critic:
    def __init__(self, fn):
        self.fn = fn
        self.optimizer = SimpleNamespace(param_groups=[{'lr': 1e-6}])

    def __call__(self, **kw):
        return self.fn()

    def backward(self, loss):
        loss.backward()

    def step(self):
        pass


class Phased:
    """The actor engine: the rollout model while scoring, the trained one in rl_step."""

    def __init__(self, roll, train, state):
        self.roll, self.train_lm, self.state = roll, train, state
        self.optimizer = SimpleNamespace(param_groups=[{'lr': 1e-6}])

    def _cur(self):
        return self.roll if self.state['phase'] == 'rollout' else self.train_lm

    def __call__(self, **kw):
        return self._cur()(**kw)

    def get_output_embeddings(self):
        return self._cur().get_output_embeddings()

    def backward(self, loss):
        loss.backward()

    def step(self):
        pass


def _ppo_batch(seed, B=4, Lq=40, P=12, V=2053, pad=0):
    """Left-padded prompts of P tokens, right-padded responses."""
    gen = torch.Generator().manual_seed(seed)
    ids = torch.full((B, Lq), pad, dtype=torch.int64)
    for b in range(B):
        p = P - 3 * b  # prompt tokens of sample b (left pad before them)
        r = Lq - P - 5 * b  # response tokens (right pad after them)
        ids[b, P - p:P] = torch.randint(2, V, (p,), generator=gen)
        ids[b, P:P + r] = torch.randint(2, V, (r,), generator=gen)
    return ids.to(DEV)


def _run_ppo(cls, fused, ids, P, H, V, seed, **kw):
    from align_anything_b200.models.reward_model import ScoreModelOutput

    gen = torch.Generator().manual_seed(seed)
    B, Lq = ids.shape
    t = lambda *shape, s=1.0: (torch.randn(*shape, generator=gen) * s)
    hid_a, hid_r, hid_new = (t(B, Lq, H).bfloat16().to(DEV) for _ in range(3))
    w_a = t(V, H, s=0.2).bfloat16().to(DEV)
    w_r = (w_a.float().cpu() + t(V, H, s=0.02)).bfloat16().to(DEV)
    reward = t(B).to(DEV)
    critic, new_critic = t(B, Lq, 1).to(DEV), t(B, Lq, 1).to(DEV)
    h_new, w_new = hid_new.clone().requires_grad_(True), w_a.clone().requires_grad_(True)
    tr = cls(None, tokenizer=SimpleNamespace(pad_token_id=0), **kw)
    tr.fused_lm_head, tr.lm_head_chunk_rows = fused, 32
    state = {'phase': 'rollout'}
    tr.actor_model = Phased(LM(hid_a, w_a), LM(h_new, w_new), state)
    tr.actor_reference_model = LM(hid_r, w_r)
    tr.reward_model = Critic(lambda: ScoreModelOutput(end_scores=reward.unsqueeze(-1)))
    g_critic = new_critic.clone().requires_grad_(True)
    tr.reward_critic_model = Critic(lambda: ScoreModelOutput(scores=critic if state['phase'] == 'rollout' else g_critic))
    inference, training = tr.score_rollout({'input_ids': ids, 'attention_mask': ids != 0}, P)
    state['phase'] = 'train'
    out = tr.rl_step(inference, training)
    return training, out, tr.last_rl_tensors, h_new.grad, w_new.grad


def _close(got, want, rel, what):
    err = float((got.float() - want.float()).abs().max())
    scale = max(1.0, float(want.float().abs().max()))
    assert err <= rel * scale, (what, err, scale)


def _compare_ppo(a, b):
    for k in ('log_probs', 'ref_log_probs'):  # the full (B, L - 1) width, prompt and pad positions included
        assert_ulp_close(b[0][k], a[0][k], max_ulp=2, min_exact=0.95, what=f'rollout {k}')
    assert set(a[1]) == set(b[1])
    for k, v in a[1].items():
        assert abs(v - b[1][k]) <= 1e-2 * max(1.0, abs(v)), (k, v, b[1][k])
    for k, v in a[2].items():
        _close(b[2][k], v, 2e-2, k)
    _close(b[3], a[3], 2e-2, 'd hidden')
    _close(b[4], a[4], 2e-2, 'd weight')


def test_text_ppo_fused_lm_head(ops):
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer

    ids = _ppo_batch(5)
    res = {fused: _run_ppo(PPOTrainer, fused, ids, 12, 128, 2053, 41) for fused in (False, True)}
    _compare_ppo(res[False], res[True])
    ops.check_status()


@pytest.mark.parametrize('estimator', ['gae', 'reinforce', 'rloo', 'reinforce_baseline', 'group_norm'])
def test_multi_ppo_fused_lm_head(ops, estimator):
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer

    ids = _ppo_batch(6)
    res = {fused: _run_ppo(PPOTrainer, fused, ids, 12, 128, 2053, 43, advantage_estimator=estimator,
                           n_samples_per_prompt=2) for fused in (False, True)}
    _compare_ppo(res[False], res[True])
    ops.check_status()


def _grpo_sequences(seed, B=4, Lq=40, P=16, V=2053, pad=0, eos=1):
    """Completions of K = Lq - P tokens: two end at an eos inside the completion (pad after it), two never do."""
    gen = torch.Generator().manual_seed(seed)
    seq = torch.randint(2, V, (B, Lq), generator=gen)
    seq[0, :3] = pad  # a left-padded prompt
    seq[1, P + 5] = eos
    seq[1, P + 6:] = pad
    seq[2, P] = eos  # eos as the first completion token
    seq[2, P + 1:] = pad
    return seq.to(DEV)


def _run_grpo(fused, seq, P, H, V, seed):
    from align_anything_b200.trainers.text_to_text.grpo import GRPOTrainer

    gen = torch.Generator().manual_seed(seed)
    B, Lq = seq.shape
    hid = torch.randn(B, Lq, H, generator=gen).bfloat16().to(DEV)
    hid_r = torch.randn(B, Lq, H, generator=gen).bfloat16().to(DEV)
    w = (torch.randn(V, H, generator=gen) * 0.2).bfloat16().to(DEV)
    w_r = (w.float().cpu() + torch.randn(V, H, generator=gen) * 0.02).bfloat16().to(DEV)
    rewards = torch.randn(B, generator=gen).to(DEV)
    h, wt = hid.clone().requires_grad_(True), w.clone().requires_grad_(True)
    tr = GRPOTrainer(None, LM(h, wt), LM(hid_r, w_r), SimpleNamespace(pad_token_id=0, eos_token_id=1), beta=0.04,
                     num_generations=2)
    tr.fused_lm_head, tr.lm_head_chunk_rows = fused, 32
    out = tr.step_from_rollout(seq, P, rewards)
    return out, h.grad, wt.grad


def test_grpo_fused_lm_head(ops):
    seq = _grpo_sequences(7)
    a, b = (_run_grpo(fused, seq, 16, 128, 2053, 47) for fused in (False, True))
    assert set(a[0]) == set(b[0]) == {'train/loss', 'train/reward'}
    assert b[0]['train/reward'] == a[0]['train/reward']
    assert abs(a[0]['train/loss'] - b[0]['train/loss']) <= 1e-2 * max(1.0, abs(a[0]['train/loss'])), (a[0], b[0])
    _close(b[1], a[1], 2e-2, 'd hidden')
    _close(b[2], a[2], 2e-2, 'd weight')
    assert bool((b[1][:, :15] == 0).all()), 'd(hidden) of prompt rows'
    ops.check_status()


@pytest.mark.parametrize('trainer', ['ppo', 'grpo'])
def test_out_of_range_label_raises_like_the_tile_path(ops, trainer):
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer

    V = 2053
    errors = {}
    for fused in (False, True):
        with pytest.raises(Exception) as info:
            if trainer == 'ppo':
                ids = _ppo_batch(8)
                ids[1, 20] = V  # a response token outside the vocabulary
                _run_ppo(PPOTrainer, fused, ids, 12, 128, V, 49)
            else:
                seq = _grpo_sequences(9)
                seq[3, 30] = V + 7
                _run_grpo(fused, seq, 16, 128, V, 51)
        errors[fused] = info.type
    assert errors[True] is errors[False] is IndexError, errors
    assert ops.check_status() == 0  # raise_for_status reset the status word
