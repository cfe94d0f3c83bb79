"""Advantage whitening on the H100 (DESIGN §4.9): aa_whiten_moments / aa_whiten_reduce / aa_whiten_apply through the C
ABI against the port (tests/whiten_port.py, float64 statistics) on guarded, poisoned buffers, the determinism of two
runs, the n < 2 status bit, whitening text PPO, Multi-PPO 'reinforce' (REINFORCE++) and image PPO rollouts followed by
an rl_step, the fused lm_head path against the tile path, and two ranks against one whitening of both ranks' data."""
from __future__ import annotations

import os
import subprocess
import sys
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

import whiten_port as port
from test_gpu_fused_rl import LM, Phased
from test_gpu_parity import ops  # noqa: F401  (fixture)
from test_gpu_ppo_objective import Guarded

pytestmark = pytest.mark.gpu

DEV = 'cuda'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.bfloat16, torch.float16, torch.float32]
SHAPES = {'K1': [(32, 512)], 'K3-ragged': [(4, 37), (1, 300), (7, 129)]}


def _ulps(got: torch.Tensor, want: torch.Tensor) -> torch.Tensor:
    """|got - want| in units in the last place of their (common) dtype; +0 and -0 are 0 apart."""
    assert got.dtype == want.dtype and got.shape == want.shape
    ib, mag = (torch.int32, 0x7FFFFFFF) if got.dtype == torch.float32 else (torch.int16, 0x7FFF)

    def ordered(t):
        b = t.contiguous().view(ib).to(torch.int64)
        return torch.where(b < 0, -(b & mag), b)

    return (ordered(got) - ordered(want)).abs()


def _inputs(shapes, dtype, seed, loc=0.3, scale=1.7):
    """Micro-batches of the given shapes: about 70 % of each mask on, one all-masked-out row, the masked-out
    advantages poisoned with NaN (the kernels never read them)."""
    g = torch.Generator().manual_seed(seed)
    advs, masks = [], []
    for B, W in shapes:
        a = torch.randn(B, W, generator=g, dtype=torch.float64) * scale + loc
        m = torch.rand(B, W, generator=g) < 0.7
        a[~m] = float('nan')
        advs.append(a.to(dtype).to(DEV))
        masks.append(m.to(DEV))
    masks[-1][0] = False
    return advs, masks


def _c_abi(advs, masks):
    """The three entry points on guarded buffers (NaN guard bands around the advantages, guard bands of 1 = 'on'
    around the masks) -> (whitened advantages, moments (K, 3), total (3,), status word)."""
    from align_anything_b200 import _lib as L

    lib, stream = L.lib(), L.stream_ptr(DEV)
    K = len(advs)
    ga = [Guarded(a) for a in advs]
    gm = [Guarded(m.to(torch.uint8), fill=1) for m in masks]
    moments = torch.full((K, 3), float('nan'), dtype=torch.float64, device=DEV)
    total = torch.full((3,), float('nan'), dtype=torch.float64, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    for k, (a, m) in enumerate(zip(ga, gm)):
        B, W = a.view.shape
        L.check(lib.aa_whiten_moments(a.view.data_ptr(), L.dtype_code(a.view.dtype), a.view.stride(0), m.view.data_ptr(),
                                      m.view.stride(0), B, W, moments.data_ptr(), k, K, stream))
    L.check(lib.aa_whiten_reduce(moments.data_ptr(), K, total.data_ptr(), stream))
    for a, m in zip(ga, gm):
        B, W = a.view.shape
        L.check(lib.aa_whiten_apply(a.view.data_ptr(), L.dtype_code(a.view.dtype), a.view.stride(0), m.view.data_ptr(),
                                    m.view.stride(0), B, W, total.data_ptr(), status.data_ptr(), stream))
    torch.cuda.synchronize()
    for g in ga + gm:
        assert g.intact(), 'a guard band was written'
    return [a.view.clone() for a in ga], moments.cpu(), total.cpu(), int(status)


@pytest.mark.parametrize('spread', ['unit', 'mean>>std'])
@pytest.mark.parametrize('shapes', list(SHAPES))
@pytest.mark.parametrize('dtype', DTYPES)
def test_c_abi_vs_port(ops, dtype, shapes, spread):
    loc, scale = (0.3, 1.7) if spread == 'unit' else (1e3, 1.0)
    advs, masks = _inputs(SHAPES[shapes], dtype, seed=len(shapes) + DTYPES.index(dtype), loc=loc, scale=scale)
    got, moments, total, status = _c_abi(advs, masks)
    assert status == 0
    counts = [float(m.sum()) for m in masks]
    assert moments[:, 0].tolist() == counts and float(total[0]) == sum(counts)  # exact counts, slot by slot
    n, mean, var = port.statistics(advs, masks)
    assert abs(float(total[1]) / n - mean) <= 1e-12 * max(1.0, abs(mean))
    k_var = (float(total[2]) - float(total[1]) * (float(total[1]) / n)) / (n - 1)
    assert abs(k_var - var) <= 1e-9 * var, (k_var, var)
    want = port.whiten(advs, masks)
    exact = 0
    for g, w, m in zip(got, want, masks):
        assert torch.equal(g[~m], torch.zeros_like(g[~m]))  # masked-out (NaN-poisoned) positions: 0
        d = _ulps(g, w)
        assert int(d.max()) <= 1, f'{int(d.max())} ulps'  # within one rounding of the output dtype
        exact += int((d == 0).sum())
    assert exact >= 0.99 * sum(g.numel() for g in got), exact


@pytest.mark.parametrize('dtype', DTYPES)
def test_two_runs_are_bit_identical(ops, dtype):
    advs, masks = _inputs([(8, 1000), (3, 77), (16, 512)], dtype, seed=11)
    a = ops.whiten_advantages([x.clone() for x in advs], masks)
    b = ops.whiten_advantages([x.clone() for x in advs], masks)
    c_a, mo_a, t_a, _ = _c_abi(advs, masks)
    c_b, mo_b, t_b, _ = _c_abi(advs, masks)
    for x, y, u, v in zip(a, b, c_a, c_b):
        assert torch.equal(_ulps(x, y), torch.zeros_like(x, dtype=torch.int64))
        assert torch.equal(_ulps(u, v), torch.zeros_like(u, dtype=torch.int64))
        assert torch.equal(_ulps(x, u), torch.zeros_like(x, dtype=torch.int64))  # ops makes the C ABI's launches
    assert torch.equal(mo_a.view(torch.int64), mo_b.view(torch.int64))
    assert torch.equal(t_a.view(torch.int64), t_b.view(torch.int64))
    ops.check_status()


@pytest.mark.parametrize('on', [0, 1])
def test_fewer_than_two_tokens_set_the_status_bit_and_write_nothing(ops, on):
    from align_anything_b200 import _lib as L

    advs, masks = _inputs([(2, 40), (3, 9)], torch.bfloat16, seed=5)
    masks = [torch.zeros_like(m) for m in masks]
    masks[1][2, 4] = bool(on)
    before = [a.clone() for a in advs]
    got, _, total, status = _c_abi(advs, masks)
    assert status == L.STATUS_WHITEN_COUNT and float(total[0]) == on
    for g, b in zip(got, before):
        assert torch.equal(_ulps(g, b), torch.zeros_like(g, dtype=torch.int64))  # NaN poison included: untouched
    out = ops.whiten_advantages(advs, masks)
    with pytest.raises(ValueError, match='at least 2 masked tokens'):
        ops.check_status()
    assert all(torch.equal(o.view(torch.int16), b.view(torch.int16)) for o, b in zip(out, before))
    ops.check_status()  # the word was reset


# ---- trainers -------------------------------------------------------------------------------------------------------
class _TokLM(LM):
    """hidden = emb[input_ids]: a micro-batch of the rollout sees exactly the rows the whole batch would."""

    def __init__(self, emb, weight):
        super().__init__(None, weight)
        self.emb = emb

    def __call__(self, input_ids=None, output_hidden_states=False, logits_to_keep=0, **kw):
        self.hidden = self.emb[input_ids]
        return super().__call__(output_hidden_states=output_hidden_states, logits_to_keep=logits_to_keep)


class _Scorer:
    """Reward model / critic: end_scores and scores as functions of the tokens; `train` carries the gradient."""

    def __init__(self, table, train, state):
        self.table, self.train_table, self.state = table, train, state
        self.optimizer = SimpleNamespace(param_groups=[{'lr': 1e-6}])

    def __call__(self, input_ids=None, **kw):
        from align_anything_b200.models.reward_model import ScoreModelOutput

        t = self.table if self.state['phase'] == 'rollout' else self.train_table
        s = t[input_ids]
        return ScoreModelOutput(scores=s.unsqueeze(-1), end_scores=s.sum(-1, keepdim=True) * 0.1)

    def backward(self, loss):
        loss.backward()

    def step(self):
        pass


def _ids(B, Lq=40, P=12, V=2053, seed=3):
    """Left-padded prompts of P tokens, right-padded responses of different lengths."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros((B, Lq), dtype=torch.int64)
    for b in range(B):
        p, r = P - (b % 3) * 2, Lq - P - (b * 7) % 19
        ids[b, P - p:P] = torch.randint(2, V, (p,), generator=g)
        ids[b, P:P + r] = torch.randint(2, V, (r,), generator=g)
    return ids.to(DEV)


def _text_trainer(cls, ids, P, micro, whiten, fused=False, V=2053, H=128, **kw):
    """A text PPO / Multi-PPO trainer whose actor_step hands out the rows of `ids` in order."""
    g = torch.Generator().manual_seed(17)
    r = lambda *s, k=1.0: torch.randn(*s, generator=g) * k  # noqa: E731
    emb = r(V, H).bfloat16().to(DEV)
    w_a = r(V, H, k=0.2)
    w_ref, w_new = (w_a + r(V, H, k=0.02)).bfloat16().to(DEV), (w_a + r(V, H, k=0.01)).bfloat16().to(DEV)
    table = r(V)
    new_table = (table + r(V, k=0.1)).to(DEV).requires_grad_(True)
    cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(per_device_train_batch_size=micro, whiten_advantages=whiten))
    tr = cls(cfgs, tokenizer=SimpleNamespace(pad_token_id=0), **kw)
    tr.fused_lm_head, tr.lm_head_chunk_rows = fused, 32
    state = {'phase': 'rollout'}
    tr.actor_model = Phased(_TokLM(emb, w_a.bfloat16().to(DEV)), _TokLM(emb, w_new.requires_grad_(True)), state)
    tr.actor_reference_model = _TokLM(emb, w_ref)
    tr.reward_model = _Scorer(table.to(DEV), table.to(DEV), state)
    tr.reward_critic_model = _Scorer(table.to(DEV) * 0.5, new_table, state)
    row = [0]

    def actor_step(mini):
        n = mini['input_ids'].size(0)
        seq = ids[row[0]:row[0] + n]
        row[0] += n
        return {'input_ids': seq, 'attention_mask': seq != 0}

    tr.actor_step = actor_step
    prompts = {'input_ids': ids[:, :P], 'attention_mask': ids[:, :P] != 0}
    return tr, prompts, state, emb, w_new


def _expected(tr, training, inference, returns_of=None):
    """Each micro-batch's K4 (+ K4r) again with the switch off, and the port's whitening of all of them."""
    from align_anything_b200 import ops

    plain, masks = [], []
    for t, i in zip(training, inference):
        mask = i['attention_mask'][:, 1:]
        out = list(ops.kl_rewards_and_gae(t['reward'], t['log_probs'], t['ref_log_probs'], t['reward_values'], mask,
                                          t['prompt_idx'], tr.kl_coeff, tr.clip_range_score, tr.gamma, tr.gae_lambda))
        if returns_of is not None:
            out[1], out[2] = returns_of(out[0], mask, t['prompt_idx'], out[3])
        plain.append(out)
        masks.append(mask[:, t['prompt_idx']:])
    return plain, masks, port.whiten([p[1] for p in plain], masks)


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(_ulps(a, b), torch.zeros_like(a, dtype=torch.int64))


def _check_rollout(training, plain, want):
    for t, p, w in zip(training, plain, want):
        for k, v in zip(('old_rewards', 'returns', 'row_stats'), (p[0], p[2], p[3])):
            assert _same(t[k], v), k  # unwhitened returns, pre-whitening row sums: K4's (K4r's) bits
        assert int(_ulps(t['advantages'], w).max()) <= 1


def _check_step(tr, out, training, inference, emb, w_new):
    """rl_step on micro-batch 0 consumed the whitened advantages: its actor loss against float64, its advantage
    metric the pre-whitening row mean."""
    from oracle import ref_port as O

    t, i = training[0], inference[0]
    assert tr.last_rl_tensors['advantages'] is t['advantages'] and tr.last_rl_tensors['returns'] is t['returns']
    start, ids = t['prompt_idx'], i['input_ids']
    mask = i['attention_mask'][:, 1:][:, start:]
    logits = F.linear(emb[ids].double(), w_new.detach().double())[:, :-1]
    lp64 = torch.log_softmax(logits, -1).gather(-1, ids[:, 1:].unsqueeze(-1)).squeeze(-1)[:, start:]
    want = float(O.actor_loss(lp64, t['log_probs'][:, start:].double(), t['advantages'].double(), mask, 0.2))
    assert abs(out['train/actor_loss'] - want) <= 1e-2 * max(1.0, abs(want)), (out['train/actor_loss'], want)
    adv_metric = float(t['row_stats'][:, 3].mean())
    assert abs(out['train/reward_advantage'] - adv_metric) <= 1e-6 * max(1.0, abs(adv_metric))


@pytest.mark.parametrize('fused', [False, True])
def test_text_ppo_rollout_and_step_vs_port(ops, fused):
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer

    ids, P = _ids(6), 12
    tr, prompts, state, emb, w_new = _text_trainer(PPOTrainer, ids, P, 2, True, fused=fused)
    inference, training = tr.rollout(prompts)
    assert len(training) == 3
    plain, masks, want = _expected(tr, training, inference)
    _check_rollout(training, plain, want)
    state['phase'] = 'train'
    out = tr.rl_step(inference[0], training[0])
    _check_step(tr, out, training, inference, emb, w_new)
    ops.check_status()


def test_multi_ppo_reinforce_plus_plus_vs_port(ops):
    """REINFORCE++: Multi-PPO's 'reinforce' returns of the KL-shaped rewards, whitened over the rollout."""
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer, estimator_returns_of

    ids, P = _ids(8, seed=9), 12
    tr, prompts, state, emb, w_new = _text_trainer(PPOTrainer, ids, P, 1, True, advantage_estimator='reinforce',
                                                   n_samples_per_prompt=2)
    prompts = {k: v[::2] for k, v in prompts.items()}  # 4 prompts, 2 samples each (the rows of `ids` in order)
    inference, training = tr.rollout(prompts)
    assert len(training) == 4
    plain, masks, want = _expected(tr, training, inference, estimator_returns_of(tr))
    _check_rollout(training, plain, want)
    state['phase'] = 'train'
    out = tr.rl_step(inference[0], training[0])
    _check_step(tr, out, training, inference, emb, w_new)
    ops.check_status()


def test_fused_lm_head_rollout_equals_the_tile_path(ops):
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer

    ids, P = _ids(6, seed=21), 12
    runs = []
    for fused in (False, True):
        tr, prompts, state, _, _ = _text_trainer(PPOTrainer, ids, P, 3, True, fused=fused)
        inference, training = tr.rollout(prompts)
        state['phase'] = 'train'
        runs.append((training, tr.rl_step(inference[0], training[0])))
    for a, b in zip(runs[0][0], runs[1][0]):
        scale = max(1.0, float(a['advantages'].abs().max()))
        assert float((a['advantages'] - b['advantages']).abs().max()) <= 2e-2 * scale
    for k, v in runs[0][1].items():
        assert abs(v - runs[1][1][k]) <= 1e-2 * max(1.0, abs(v)), (k, v, runs[1][1][k])
    ops.check_status()


def test_image_ppo_tail_layout_rollout_and_step(ops):
    """The multimodal trainer on the tail layout (responses of different lengths): response_mask is the mask."""
    from test_gpu_fused_rl import Critic

    from align_anything_b200.models.reward_model import ScoreModelOutput
    from align_anything_b200.trainers.text_image_to_text.ppo import PPOTrainer

    gen = torch.Generator().manual_seed(37)
    B, Lq, H, V = 3, 40, 128, 1031
    resp = [20, 9, 28]
    seq = torch.zeros((B, Lq), dtype=torch.int64)
    for b, r in enumerate(resp):
        seq[b, Lq - r - 8:] = torch.randint(2, V, (r + 8,), generator=gen)
    ids = seq.to(DEV)
    t = lambda *shape, s=1.0: (torch.randn(*shape, generator=gen) * s)  # noqa: E731
    hid_a, hid_r, hid_new = (t(B, Lq, H).bfloat16().to(DEV) for _ in range(3))
    w_a = t(V, H, s=0.2).bfloat16().to(DEV)
    w_r = (w_a.float().cpu() + t(V, H, s=0.02)).bfloat16().to(DEV)
    reward = t(B).to(DEV)
    critic, new_critic = t(B, Lq, 1).to(DEV), t(B, Lq, 1).to(DEV)

    def run(whiten):
        from align_anything_b200 import ops as O

        h_new, w_new = hid_new.clone().requires_grad_(True), w_a.clone().requires_grad_(True)
        cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(whiten_advantages=whiten))
        tr = PPOTrainer(cfgs, tokenizer=SimpleNamespace(pad_token_id=0))
        state = {'phase': 'rollout'}
        tr.actor_model = Phased(LM(hid_a, w_a), LM(h_new, w_new), state)
        tr.actor_reference_model = LM(hid_r, w_r)
        tr.reward_model = Critic(lambda: ScoreModelOutput(end_scores=reward.unsqueeze(-1)))
        g_critic = new_critic.clone().requires_grad_(True)
        tr.reward_critic_model = Critic(lambda: ScoreModelOutput(scores=critic if state['phase'] == 'rollout' else g_critic))
        tr.actor_step = lambda mini: ({'input_ids': ids, 'attention_mask': ids != 0}, O.as_device_lens(resp, DEV))
        inference, training = tr.rollout({'input_ids': ids[:, :12], 'attention_mask': ids[:, :12] != 0})
        state['phase'] = 'train'
        return training[0], tr.rl_step(inference[0], training[0]), tr.last_rl_tensors

    plain = run(False)
    on = run(True)
    mask = on[0]['response_mask']
    assert torch.equal(mask, plain[0]['response_mask']) and [int(x) for x in mask.sum(-1)] == resp
    want = port.whiten([plain[2]['advantages']], [mask])[0]
    assert int(_ulps(on[2]['advantages'], want).max()) <= 1
    assert on[2]['advantages'] is on[0]['advantages']
    for k in ('old_rewards', 'returns'):
        assert _same(on[2][k], plain[2][k]), k
    assert set(on[1]) == set(plain[1])
    for k in ('train/reward_advantage', 'train/reward_return', 'train/kl_divergence', 'train/reward_with_kl_penalty'):
        assert on[1][k] == plain[1][k], k  # the pre-whitening metrics, bit for bit
    ops.check_status()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_ranks_whiten_as_one(ops):
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr',
           '127.0.0.1', '--master-port', '29541', os.path.join(ROOT, 'tests', 'dist_whiten.py')]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and 'WHITEN DIST OK world=2' in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
