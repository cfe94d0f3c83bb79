"""Entropy bonus on the H100: K1b's entropy-gradient variant through ops against a float64 oracle of the stated tile
formula (FAITHFUL rounding included), bit-identity of rows with g_H = 0 and of the log-probs, the actor / GRPO nodes
with entropy_coeff != 0 -- single pass (K1f) and composed path against each other and against float64 autograd of the
regularised objective, in the production configuration (16-bit FAITHFUL, V = 152064) too --, K1f and K6b through the
C ABI on poisoned, guard-banded buffers, the lm_head node's d(hidden) / d(weight), and one step of the text, Multi-PPO,
image PPO and GRPO trainers on both the logits-tile and the fused lm_head path (parameter gradients and
train/actor_entropy against float64; coefficient 0 bit-identical to a trainer without the switch)."""
from __future__ import annotations

import pytest
import torch

from test_gpu_entropy import _bits, _logits, entropy64
from test_gpu_parity import ops  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

DEV = 'cuda'
EPS = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -23}


def _tile64(x, y, g, g_h, faithful_dtype=None):
    """g (onehot_y - p) - g_H p (l + H) in float64; with faithful_dtype p and l come from the log-softmax rounded to
    that dtype (what K1b re-reads), H from the unrounded row.  Rows of -inf only are skipped by the callers."""
    x = x.double()
    lp = x - torch.logsumexp(x, -1, keepdim=True)
    h = entropy64(x)
    if faithful_dtype is not None:
        lp = lp.to(faithful_dtype).double()
    p = lp.exp()
    lc = torch.clamp(lp, min=-3.0e38)
    onehot = torch.nn.functional.one_hot(y, x.size(-1)).double()
    return g.double()[..., None] * (onehot - p) - g_h.double()[..., None] * p * (lc + h[..., None])


def _close(got, want, dtype, what):
    """One unit in the last place of the tile dtype plus a floor relative to the row's largest element: that ulp for
    a 16-bit tile, 2e-5 for fp32 (fp32 arithmetic with the hardware exp2, the floor the K1b tile tests use)."""
    got = got.double()
    scale = want.abs().amax(-1, keepdim=True)
    tol = EPS[dtype] * want.abs() + max(EPS[dtype], 2e-5) * scale + 1e-30
    err = (got - want).abs()
    bad = err > tol
    assert not bool(bad.any()), (f'{what}: {int(bad.sum())} elements beyond tolerance, max error / row scale '
                                 f'{float((err / scale.clamp_min(1e-30)).max()):.3e}')


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize('V', [32001, 128257, 152064])
@pytest.mark.parametrize('mode', ['faithful', 'f32'])
def test_k1b_entropy_gradient_vs_float64(ops, dtype, V, mode):
    if dtype == torch.float32 and mode == 'faithful':
        pytest.skip('fp32 logits have no rounding point: FAITHFUL is F32 mode')
    B, L = 2, 5
    x = _logits(B, L + 1, V, dtype, seed=V)
    x[0, 3] = 0.5  # no all -inf row here: its gradient is NaN by definition
    gen = torch.Generator().manual_seed(1)
    labels = torch.randint(0, V, (B, L), generator=gen).to(DEV)
    w = torch.randn(B, L, generator=gen).to(DEV)
    wh = torch.randn(B, L, generator=gen).to(DEV)
    wh[1, 2] = 0.0  # a row without an entropy gradient
    leaf = x.clone().requires_grad_(True)
    lp, ent = ops.gather_log_probabilities_with_entropy(leaf[:, :-1], labels, mode=mode, entropy_grad=True)
    assert ent.requires_grad
    ((lp.float() * w).sum() + (ent * wh).sum()).backward()
    grad = leaf.grad
    assert torch.equal(grad[:, -1], torch.zeros_like(grad[:, -1]))  # the unscored row of the base tile
    faithful = dtype if (mode == 'faithful' and dtype != torch.float32) else None
    want = _tile64(x[:, :-1].float(), labels, w, wh, faithful)
    _close(grad[:, :-1], want, dtype, f'{dtype} V={V} {mode}')
    # rows with g_H == 0: the plain K1b's bits; log-probs bit-identical to the plain gather
    plain = x.clone().requires_grad_(True)
    lp0 = ops.gather_log_probabilities(plain[:, :-1], labels, mode=mode)
    (lp0.float() * w).sum().backward()
    assert torch.equal(_bits(lp0.detach()), _bits(lp.detach()))
    assert torch.equal(_bits(plain.grad[1, 2]), _bits(grad[1, 2]))


def test_unused_entropy_runs_the_plain_backward(ops):
    x = _logits(2, 4, 32001, torch.bfloat16, seed=3)
    x[0, 3] = 0.5
    labels = torch.randint(0, 32001, (2, 4), device=DEV)
    a, b = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    lp, _ = ops.gather_log_probabilities_with_entropy(a, labels, entropy_grad=True)
    lp.float().sum().backward()
    ops.gather_log_probabilities(b, labels).float().sum().backward()
    assert torch.equal(_bits(a.grad), _bits(b.grad))


def _actor64(x, ids, start, old, adv, mask, clip, c):
    """-masked_mean(min(A r, A clip(r))) - c masked_mean(H) in float64 autograd."""
    x = x.double().detach().requires_grad_(True)
    lsm = torch.log_softmax(x[:, start:-1], -1)
    lp = lsm.gather(-1, ids[:, start + 1:, None]).squeeze(-1)
    r = torch.exp(lp - old.double())
    a = adv.double()
    obj = torch.minimum(a * r, a * torch.clamp(r, 1 - clip, 1 + clip))
    m = mask.double()
    mm = lambda t: ((t * m).sum(-1) / m.sum(-1)).mean()  # noqa: E731
    p = lsm.exp()
    h = -(p * lsm).sum(-1)
    loss = -mm(obj) - c * mm(h)
    loss.backward()
    return loss.detach(), mm(h).detach(), x.grad


@pytest.mark.parametrize('V', [32064, 152064])  # composed path / K1f
def test_dense_actor_loss_with_bonus(ops, V):
    torch.manual_seed(V)
    B, Lq, start, c = 3, 9, 3, 0.05
    W = Lq - 1 - start
    x = (torch.randn(B, Lq, V) * 2.0).to(DEV)
    ids = torch.randint(0, V, (B, Lq), device=DEV)
    old = (torch.randn(B, W) * 0.1 - 8.0).to(DEV)
    adv = torch.randn(B, W, device=DEV)
    mask = torch.ones(B, W, dtype=torch.bool, device=DEV)
    mask[1, -2:] = False
    with torch.no_grad():  # old log-probs near the new ones, so that the ratio lands inside and outside the clip range
        lp_now = ops.gather_log_probabilities(x[:, start:-1], ids[:, start + 1:], mode='f32')
        old = lp_now + torch.randn(B, W, device=DEV) * 0.2
    leaf = x.clone().requires_grad_(True)
    out = ops.dense_actor_loss(leaf, ids, start, old, adv, mask, 0.2, mode='f32', entropy_coeff=c)
    assert len(out) == 4 and not out[3].requires_grad
    out[0].backward()
    loss64, h64, g64 = _actor64(x, ids, start, old, adv, mask, 0.2, c)
    assert abs(float(out[0]) - float(loss64)) <= 1e-4 * max(1.0, abs(float(loss64)))
    assert abs(float(out[3]) - float(h64)) <= 1e-4
    # the third output is the actor loss without the bonus
    assert abs(float(out[2].float().reshape(-1)[0]) - float(loss64 + c * h64)) <= 1e-4 * max(1.0, abs(float(loss64)))
    _close(leaf.grad, g64, torch.float32, f'dense actor V={V}')
    # the composed path (K1 entropy -> K5 + masked_mean -> K1b entropy) gives the single pass's tile
    leaf2 = x.clone().requires_grad_(True)
    lp2, ent2 = ops.gather_log_probabilities_with_entropy(leaf2[:, start:-1], ids[:, start + 1:], mode='f32',
                                                          entropy_grad=True)
    (ops.actor_loss(lp2, old, adv, mask, 0.2, mode='f32') - c * ops.masked_mean(ent2, mask)).backward()
    _close(leaf2.grad, leaf.grad.double(), torch.float32, f'single pass vs composed V={V}')
    # coefficient 0: the same outputs and tile as the node without the switch
    a, b = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    o0 = ops.dense_actor_loss(a, ids, start, old, adv, mask, 0.2, mode='f32', entropy_coeff=0.0)
    o1 = ops.dense_actor_loss(b, ids, start, old, adv, mask, 0.2, mode='f32')
    assert len(o0) == len(o1) == 3
    o0[0].backward()
    o1[0].backward()
    assert torch.equal(_bits(a.grad), _bits(b.grad)) and torch.equal(_bits(o0[1]), _bits(o1[1]))


def _grpo64(x, ids, K, ref, adv, eos, beta, c):
    x = x.double().detach().requires_grad_(True)
    lsm = torch.log_softmax(x[:, :-1][:, -K:], -1)
    tok = ids[:, -K:]
    lp = lsm.gather(-1, tok[..., None]).squeeze(-1)
    is_eos = tok == eos
    first = torch.where(is_eos.any(1), is_eos.int().argmax(1), torch.full_like(is_eos.int().argmax(1), K))
    mask = (torch.arange(K, device=x.device)[None] <= first[:, None]).double()
    d = ref.double() - lp
    kl = torch.exp(d) - d - 1
    ptl = -(torch.exp(lp - lp.detach()) * adv.double().reshape(-1, 1) - beta * kl)
    h = -(lsm.exp() * lsm).sum(-1)
    loss = (ptl * mask).sum() / mask.sum() - c * (h * mask).sum() / mask.sum()
    loss.backward()
    return loss.detach(), ((h * mask).sum() / mask.sum()).detach(), x.grad


@pytest.mark.parametrize('V', [32064, 152064])
def test_grpo_loss_with_bonus(ops, V):
    torch.manual_seed(V + 1)
    B, L, K, eos, beta, c = 4, 10, 6, 5, 0.04, 0.1
    x = (torch.randn(B, L, V) * 2.0).to(DEV)
    ids = torch.randint(6, V, (B, L), device=DEV)
    ids[1, -3] = eos
    with torch.no_grad():
        ref = ops.tail_token_log_probs(x, ids, K, mode='f32') + torch.randn(B, K, device=DEV) * 0.1
    adv = torch.randn(B, 1, device=DEV)
    leaf = x.clone().requires_grad_(True)
    out = ops.grpo_loss_from_logits(leaf, ids, K, ref, adv, eos, beta, mode='f32', entropy_coeff=c)
    assert len(out) == 5
    out[0].backward()
    loss64, h64, g64 = _grpo64(x, ids, K, ref, adv, eos, beta, c)
    assert abs(float(out[0]) - float(loss64)) <= 1e-4 * max(1.0, abs(float(loss64)))
    assert abs(float(out[3]) - float(h64)) <= 1e-4
    _close(leaf.grad, g64, torch.float32, f'grpo V={V}')


# ---- trainers (the logits-tile path; the small models of test_gpu_fused_rl) -------------------------------------------
def _with_coeff(cls, c, mode=None):
    attrs = {'entropy_coeff': c}
    if mode is not None:
        attrs['mode'] = mode
    return type(cls.__name__, (cls,), attrs)


def _param_grads(dlogits64, h, w):
    """d(hidden), d(weight) of logits = F.linear(h, w) for a float64 d(logits)."""
    return dlogits64 @ w.double(), torch.einsum('blv,blh->vh', dlogits64, h.double())


def _rel(got, want, rel, what):
    err = float((got.double() - want).abs().max())
    scale = max(1e-12, float(want.abs().max()))
    assert err <= rel * scale, (what, err, scale)


@pytest.mark.parametrize('trainer', ['text', 'multi-rloo'])
def test_text_ppo_entropy_bonus(ops, trainer):
    from test_gpu_fused_rl import _ppo_batch, _run_ppo

    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer as Multi
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer as Text

    cls, kw = (Text, {}) if trainer == 'text' else (Multi, {'advantage_estimator': 'rloo', 'n_samples_per_prompt': 2})
    ids = _ppo_batch(5)
    P, H, V, seed, c = 12, 128, 2053, 41, 0.05
    plain = _run_ppo(cls, False, ids, P, H, V, seed, **kw)
    zero = _run_ppo(_with_coeff(cls, 0.0), False, ids, P, H, V, seed, **kw)
    assert zero[1] == plain[1]  # keys and values
    assert torch.equal(_bits(zero[3]), _bits(plain[3])) and torch.equal(_bits(zero[4]), _bits(plain[4]))
    # against float64 in F32 mode: the rollout and trained models of these tests are independent draws, so most ratios
    # lie far outside the clip range, where FAITHFUL's bf16 rounding of lp - old moves A * ratio by percents
    plain = _run_ppo(_with_coeff(cls, 0.0, 'f32'), False, ids, P, H, V, seed, **kw)
    on = _run_ppo(_with_coeff(cls, c, 'f32'), False, ids, P, H, V, seed, **kw)
    assert set(on[1]) == set(plain[1]) | {'train/actor_entropy'}
    assert on[1]['train/actor_loss'] == plain[1]['train/actor_loss']  # the loss without the bonus
    # float64 recompute of the regularised objective on the trained model's logits (as the tile path sees them)
    gen = torch.Generator().manual_seed(seed)  # _run_ppo's draws: hid_a, hid_r, hid_new, w_a
    B, Lq = ids.shape
    for _ in range(2):
        torch.randn(B, Lq, H, generator=gen)
    h_new = torch.randn(B, Lq, H, generator=gen).bfloat16().to(DEV)
    w = (torch.randn(V, H, generator=gen) * 0.2).bfloat16().to(DEV)
    start = P - 1
    x = torch.nn.functional.linear(h_new, w)
    old = on[0]['log_probs'][:, start:]
    adv = on[2]['advantages']
    mask = (ids != 0)[:, 1:][:, start:]
    loss64, h64, g64 = _actor64(x.float(), ids, start, old, adv, mask, 0.2, c)
    assert abs(on[1]['train/actor_entropy'] - float(h64)) <= 1e-4 * max(1.0, abs(float(h64)))
    dh, dw = _param_grads(g64, h_new, w)
    _rel(on[3], dh, 2e-2, 'd hidden')
    _rel(on[4], dw, 2e-2, 'd weight')
    # the fused lm_head path (K6's entropy variant, K6b's entropy epilogue) against the tile path in the default FAITHFUL
    # mode, where both see bf16-rounded logits, within the fused-vs-tile tolerance of test_gpu_fused_rl
    tile = _run_ppo(_with_coeff(cls, c), False, ids, P, H, V, seed, **kw)
    fused = _run_ppo(_with_coeff(cls, c), True, ids, P, H, V, seed, **kw)
    assert set(fused[1]) == set(tile[1])
    for k, v in tile[1].items():
        assert abs(v - fused[1][k]) <= 1e-2 * max(1.0, abs(v)), (k, v, fused[1][k])
    _rel(fused[3], tile[3].double(), 2e-2, 'fused d hidden')
    _rel(fused[4], tile[4].double(), 2e-2, 'fused d weight')
    ops.check_status()


def test_grpo_entropy_bonus(ops, monkeypatch):
    from test_gpu_fused_rl import _grpo_sequences, _run_grpo

    from align_anything_b200.trainers.text_to_text.grpo import GRPOTrainer

    seq = _grpo_sequences(7)
    P, H, V, seed, c = 16, 128, 2053, 47, 0.05
    plain = _run_grpo(False, seq, P, H, V, seed)
    monkeypatch.setattr(GRPOTrainer, 'entropy_coeff', 0.0)
    zero = _run_grpo(False, seq, P, H, V, seed)
    assert zero[0] == plain[0]
    assert torch.equal(_bits(zero[1]), _bits(plain[1])) and torch.equal(_bits(zero[2]), _bits(plain[2]))
    monkeypatch.setattr(GRPOTrainer, 'entropy_coeff', c)
    on = _run_grpo(False, seq, P, H, V, seed)
    assert set(on[0]) == set(plain[0]) | {'train/actor_entropy'}
    assert on[0]['train/loss'] == plain[0]['train/loss']  # GRPO's loss, without the bonus
    gen = torch.Generator().manual_seed(seed)  # _run_grpo's draws: hid, hid_r, w, w_r, rewards
    B, Lq = seq.shape
    hid = torch.randn(B, Lq, H, generator=gen).bfloat16().to(DEV)
    hid_r = torch.randn(B, Lq, H, generator=gen).bfloat16().to(DEV)
    w = (torch.randn(V, H, generator=gen) * 0.2).bfloat16()
    w_r = (w.float() + torch.randn(V, H, generator=gen) * 0.02).bfloat16().to(DEV)
    w = w.to(DEV)
    rewards = torch.randn(B, generator=gen).to(DEV)
    K = Lq - P
    ref = ops.tail_token_log_probs(torch.nn.functional.linear(hid_r, w_r), seq, K).float()
    adv = ops.group_advantages(rewards, 2).float()
    x = torch.nn.functional.linear(hid, w)
    _, h64, g64 = _grpo64(x.float(), seq, K, ref, adv, 1, 0.04, c)
    assert abs(on[0]['train/actor_entropy'] - float(h64)) <= 1e-4 * max(1.0, abs(float(h64)))
    dh, dw = _param_grads(g64, hid, w)
    _rel(on[1], dh, 2e-2, 'd hidden')
    _rel(on[2], dw, 2e-2, 'd weight')
    fused = _run_grpo(True, seq, P, H, V, seed)
    assert set(fused[0]) == set(on[0])
    for k, v in on[0].items():
        assert abs(v - fused[0][k]) <= 1e-2 * max(1.0, abs(v)), (k, v, fused[0][k])
    _rel(fused[1], dh, 2e-2, 'fused d hidden')
    _rel(fused[2], dw, 2e-2, 'fused d weight')
    ops.check_status()


def test_image_ppo_entropy_bonus(ops):
    from align_anything_b200.models.reward_model import ScoreModelOutput
    from align_anything_b200.trainers.text_image_to_text.ppo import PPOTrainer
    from test_gpu_fused_rl import LM, Critic, Phased
    from types import SimpleNamespace

    gen = torch.Generator().manual_seed(31)
    B, Lq, H, V, c = 3, 40, 128, 1031, 0.05
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

    def run(cls, fused=False):
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
        return training, tr.rl_step(inference, training), tr.last_rl_tensors, h_new.grad, w_new.grad

    plain, zero, on = run(PPOTrainer), run(_with_coeff(PPOTrainer, 0.0)), run(_with_coeff(PPOTrainer, c))
    assert zero[1] == plain[1]
    assert torch.equal(_bits(zero[3]), _bits(plain[3])) and torch.equal(_bits(zero[4]), _bits(plain[4]))
    assert set(on[1]) == set(plain[1]) | {'train/actor_entropy'}
    assert on[1]['train/actor_loss'] == plain[1]['train/actor_loss']
    # float64: the actor loss and the bonus over the response tails, through the tail rows of the logits
    x = torch.nn.functional.linear(hid_new, w_a).double().requires_grad_(True)
    W = max(resp)
    lp = torch.zeros(B, W, dtype=torch.float64, device=DEV)
    ent = torch.zeros(B, W, dtype=torch.float64, device=DEV)
    for b, r in enumerate(resp):
        lsm = torch.log_softmax(x[b, Lq - 1 - r:Lq - 1], -1)
        lp[b, :r] = lsm.gather(-1, ids[b, Lq - r:, None]).squeeze(-1)
        ent[b, :r] = -(lsm.exp() * lsm).sum(-1)
    m = on[0]['response_mask'].double()
    mm = lambda v: ((v * m).sum(-1) / m.sum(-1)).mean()  # noqa: E731
    ratio = torch.exp(lp - on[0]['log_probs'].double())
    a = on[2]['advantages'].double()
    obj = torch.minimum(a * ratio, a * torch.clamp(ratio, 0.8, 1.2))
    (-mm(obj) - c * mm(ent)).backward()
    assert abs(on[1]['train/actor_entropy'] - float(mm(ent))) <= 1e-4 * max(1.0, abs(float(mm(ent))))
    dh, dw = _param_grads(x.grad, hid_new, w_a)
    _rel(on[3], dh, 2e-2, 'd hidden')
    _rel(on[4], dw, 2e-2, 'd weight')
    fused = run(_with_coeff(PPOTrainer, c), True)
    assert set(fused[1]) == set(on[1])
    for k, v in on[1].items():
        assert abs(v - fused[1][k]) <= 1e-2 * max(1.0, abs(v)), (k, v, fused[1][k])
    _rel(fused[3], dh, 2e-2, 'fused d hidden')
    _rel(fused[4], dw, 2e-2, 'fused d weight')
    ops.check_status()


# ---- K1f in the production configuration: 16-bit logits, FAITHFUL, V = 152064 --------------------------------------
def _oracle_rows(x_rows, labels, g, g_h, dtype, mode):
    """_tile64 for the scored rows (R, V), the per-token g being the loss kernel's d loss / d log-prob."""
    faithful = dtype if (mode == 'faithful' and dtype != torch.float32) else None
    return _tile64(x_rows.float(), labels, g.float(), g_h.float(), faithful)


@pytest.mark.parametrize('node', ['dense', 'tail', 'grpo'])
@pytest.mark.parametrize('dtype,mode', [(torch.bfloat16, 'faithful'), (torch.bfloat16, 'f32'), (torch.float32, 'f32')])
def test_single_pass_bonus_production_config(ops, node, dtype, mode):
    """K1f's entropy-gradient instantiations against the float64 oracle of the tile formula (FAITHFUL rounding
    included); the per-token g is the loss kernel's own gradient of the log-probs the pass wrote.  Log-probs and the
    loss value are bit-identical to the plain single pass."""
    torch.manual_seed(11)
    V, c = 152064, 0.05
    assert ops._single_pass_ok(torch.empty(1, 1, V, dtype=dtype, device=DEV))
    B, Lq = 3, 10
    x = (torch.randn(B, Lq, V, device=DEV) * 2.0).to(dtype)
    x[0, 4, ::3] = float('-inf')  # masked vocabulary entries in a scored row
    ids = torch.randint(2, V, (B, Lq), device=DEV)
    lp_dtype = dtype if mode == 'faithful' else torch.float32
    if node == 'grpo':
        K, eos = 6, 1
        ids[1, -3] = eos
        with torch.no_grad():
            ref = (ops.tail_token_log_probs(x, ids, K, mode=mode).float()
                   + torch.randn(B, K, device=DEV) * 0.1).to(lp_dtype)
        adv = torch.randn(B, 1, device=DEV)
        run = lambda leaf, cf: ops.grpo_loss_from_logits(leaf, ids, K, ref, adv, eos, 0.04, mode=mode,  # noqa: E731
                                                          **({'entropy_coeff': cf} if cf else {}))
        rows = (slice(None), slice(Lq - 1 - K, Lq - 1))
        labels = ids[:, -K:]
    else:
        start = 3
        W = Lq - 1 - start
        lens = [W, W - 2, W - 4]
        mask = torch.zeros(B, W, dtype=torch.bool, device=DEV)
        for b, r in enumerate(lens):
            mask[b, :r] = True
        mask[2, 0] = False
        adv = torch.randn(B, W, device=DEV)
        with torch.no_grad():
            old = (ops.gather_log_probabilities(x[:, start:-1], ids[:, start + 1:], mode=mode).float()
                   + torch.randn(B, W, device=DEV) * 0.2).to(lp_dtype)
        if node == 'dense':
            run = lambda leaf, cf: ops.dense_actor_loss(leaf, ids, start, old, adv, mask, 0.2, mode=mode,  # noqa: E731
                                                        **({'entropy_coeff': cf} if cf else {}))
            rows = (slice(None), slice(start, Lq - 1))
            labels = ids[:, start + 1:]
        else:  # tail plan: every sample scores its last W rows (right-aligned responses of one length)
            lens_t = [W] * B
            run = lambda leaf, cf: ops.tail_actor_loss(leaf, ids, lens_t, old, adv, mask, 0.2, mode=mode,  # noqa: E731
                                                       **({'entropy_coeff': cf} if cf else {}))
            rows = (slice(None), slice(Lq - 1 - W, Lq - 1))
            labels = ids[:, -W:]
    a, b = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    on, off = run(a, c), run(b, 0.0)
    on[0].backward()
    off[0].backward()
    assert torch.equal(_bits(on[1]), _bits(off[1])), 'log-probs'
    assert not on[1].requires_grad and not any(t.requires_grad for t in on[2:]), 'only the loss is differentiable'
    if node == 'grpo':
        assert torch.equal(_bits(on[4].reshape(1)), _bits(off[0].detach().reshape(1))), 'GRPO loss without the bonus'
        row_end = on[2]
        m = (torch.arange(K, device=DEV)[None] < row_end[:, None])
        lp_leaf = on[1].clone().float().requires_grad_(True)
        loss, _ = ops.grpo_loss(lp_leaf.to(lp_dtype), ref, adv, ids[:, -K:], eos, 0.04, mode=mode)
        loss.backward()
        g_h = m.float() * (-c / m.sum().float())
    else:
        assert torch.equal(_bits(on[2].float().reshape(-1)[:1]), _bits(off[2].float().reshape(-1)[:1])), 'actor loss'
        lp_leaf = on[1].clone().requires_grad_(True)
        ops.actor_loss(lp_leaf, old, adv, mask, 0.2, mode=mode).backward()
        m = mask
        g_h = torch.where(m, -c / (B * m.sum(-1, keepdim=True).float()), 0.0)
    g = lp_leaf.grad
    want = _oracle_rows(x[rows], labels, g, g_h, dtype, mode)
    _close(a.grad[rows], want, dtype, f'{node} {dtype} {mode}')
    # rows outside the scored range are zero; fully masked tokens keep the plain (zero) rows bit for bit
    outside = torch.ones(Lq, dtype=torch.bool, device=DEV)
    outside[rows[1]] = False
    assert not bool(a.grad[:, outside].any())
    off_rows = ~m.bool()
    assert torch.equal(_bits(a.grad[rows][off_rows]), _bits(b.grad[rows][off_rows]))


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
def test_k1f_actor_entropy_c_abi_guarded(ops, dtype):
    """aa_logprob_actor_fused_entropy through the C ABI on poisoned, guard-banded log-prob / entropy / tile buffers:
    with coefficient 0 the tile, log-probs and statistics are bit-identical to aa_logprob_actor_fused; with a
    coefficient the tile matches the float64 oracle; the guards stay untouched."""
    from align_anything_b200 import _lib as L

    torch.manual_seed(5)
    V, B, Lq, start, G = 152064, 2, 7, 2, 64
    W = Lq - 1 - start
    mode = 'faithful'
    mode_code = ops._mode_code(mode, dtype)
    x = (torch.randn(B, Lq, V, device=DEV) * 2.0).to(dtype)
    ids = torch.randint(2, V, (B, Lq), device=DEV)
    lp_dtype = dtype if mode_code == L.MODE_FAITHFUL else torch.float32
    old = (torch.randn(B, W, device=DEV) * 0.3 - 11.0).to(lp_dtype)
    adv = torch.randn(B, W, device=DEV)
    mask = torch.ones(B, W, dtype=torch.bool, device=DEV)
    mask[1, -1] = False
    plan = ops._dense_actor_plan(B, Lq, start, x.stride(0), x.stride(1), ids.stride(0), str(x.device))
    p = plan.ptrs()
    nan16 = {torch.bfloat16: 0x7FA5, torch.float16: 0x7E55}

    def guarded(n, dt, fill):
        t = torch.empty(n + 2 * G, dtype=dt, device=DEV)
        if dt == torch.float32:
            t.view(torch.int32).fill_(0x7FA5A5A5)
        else:
            t.view(torch.int16).fill_(nan16[dt])
        if fill is not None:
            t[G:G + n] = fill
        return t

    def launch(entry, coeff):
        grad = guarded(B * Lq * V, dtype, None)
        lp = guarded(B * W, lp_dtype, 0.0)
        ent = guarded(B * W, torch.float32, 0.0)
        stats = guarded(2 * B * W, torch.float32, None)
        scratch = torch.empty(plan.n_tile_rows * 6 + B, dtype=torch.int64, device=DEV)
        args = [x.data_ptr(), L.dtype_code(dtype), x.stride(1), V, ids.data_ptr(), plan.n_seg, p[0], p[1], p[2], p[3],
                p[4], plan.n_tile_rows, lp[G:].data_ptr(), L.dtype_code(lp_dtype), stats[G:].data_ptr(),
                stats[G + B * W:].data_ptr(), old.data_ptr(), old.stride(0), adv.data_ptr(), adv.stride(0),
                L.dtype_code(adv.dtype), mask.data_ptr(), mask.stride(0), W, 0.2, mode_code, grad[G:].data_ptr(), V,
                scratch.data_ptr(), ops._device_scratch(x.device)['status'].data_ptr()]
        if entry == 'plain':
            L.check(L.lib().aa_logprob_actor_fused(*args, L.stream_ptr(x.device)))
        else:
            L.check(L.lib().aa_logprob_actor_fused_entropy(*args, coeff, ent[G:].data_ptr(), L.stream_ptr(x.device)))
        torch.cuda.synchronize()
        for buf, n in ((grad, B * Lq * V), (lp, B * W), (ent, B * W), (stats, 2 * B * W)):
            assert torch.equal(_bits(buf[:G]), _bits(guarded(0, buf.dtype, None)[:G])), 'front guard'
            assert torch.equal(_bits(buf[G + n:]), _bits(guarded(0, buf.dtype, None)[:G])), 'back guard'
        return grad[G:G + B * Lq * V].view(B, Lq, V), lp[G:G + B * W].view(B, W), ent[G:G + B * W].view(B, W), \
            stats[G:G + 2 * B * W]

    g0, lp0, _, st0 = launch('plain', 0.0)
    gz, lpz, entz, stz = launch('entropy', 0.0)
    assert torch.equal(_bits(g0), _bits(gz)) and torch.equal(_bits(lp0), _bits(lpz)) and torch.equal(_bits(st0), _bits(stz))
    want_h = entropy64(x[:, start:-1].float())
    assert float((entz.double() - want_h).abs().max()) <= 1e-4
    c = 0.05
    gc, lpc, entc, _ = launch('entropy', c)
    assert torch.equal(_bits(lpc), _bits(lp0)) and torch.equal(_bits(entc), _bits(entz))
    lp_leaf = lpc.clone().requires_grad_(True)
    ops.actor_loss(lp_leaf, old, adv, mask, 0.2, mode=mode).backward()
    g_h = torch.where(mask, -c / (B * mask.sum(-1, keepdim=True).float()), 0.0)
    want = _oracle_rows(x[:, start:-1], ids[:, start + 1:], lp_leaf.grad, g_h, dtype, mode)
    _close(gc[:, start:-1], want, dtype, f'K1f C ABI {dtype}')
    assert not bool(gc[:, :start].any()) and not bool(gc[:, -1].any())


# ---- K6b: the entropy epilogue, and the lm_head node's d(hidden) / d(weight) ------------------------------------------
@pytest.mark.parametrize('mode', ['faithful', 'f32'])
@pytest.mark.parametrize('N,H,V', [(300, 128, 32001), (200, 256, 128257)])
def test_k6b_entropy_epilogue_vs_float64(ops, mode, N, H, V):
    """aa_linear_dlogits_entropy on a poisoned, guard-banded d(logits) buffer against the float64 oracle of the tile
    formula on the bf16 logits (FAITHFUL: the rounded log-softmax); pad columns zero, guards untouched, rows with
    g_H == 0 bit-identical to aa_linear_dlogits."""
    from align_anything_b200 import _lib as L

    gen = torch.Generator(device=DEV).manual_seed(N + V)
    # exact operands: small integers times 2^-6, so every fp32 accumulation is exact and K6 / cuBLAS / float64 agree on
    # the logits bit for bit (the oracle then sees the kernel's logits, not a differently summed copy)
    h = torch.randint(-2, 3, (N, H), generator=gen, device=DEV).bfloat16()
    w = (torch.randint(-8, 9, (V, H), generator=gen, device=DEV).float() * 2.0 ** -6).bfloat16()
    lab = torch.randint(0, V, (N,), generator=gen, device=DEV)
    out, stats, ent = ops.fused_linear_token_log_probs(h, w, lab, mode=mode, return_stats=True, return_entropy=True)
    g = torch.randn(N, generator=gen, device=DEV)
    g_h = torch.randn(N, generator=gen, device=DEV)
    g_h[::7] = 0.0
    ld, G = (V + 255) // 256 * 256, 256
    mode_code = ops._mode_code(mode, torch.bfloat16)
    st = L.stream_ptr(torch.device(DEV))

    def run(with_entropy):
        buf = torch.empty(N * ld + 2 * G, dtype=torch.bfloat16, device=DEV)
        buf.view(torch.int16).fill_(0x7FA5)
        head = (h.data_ptr(), N, H, h.stride(0), w.data_ptr(), V, w.stride(0), lab.data_ptr(), stats[0].data_ptr(),
                stats[1].data_ptr(), g.data_ptr(), L.AA_F32)
        if with_entropy:
            L.check(L.lib().aa_linear_dlogits_entropy(*head, ent.data_ptr(), g_h.data_ptr(), L.AA_F32, buf[G:].data_ptr(),
                                                      ld, mode_code, st))
        else:
            L.check(L.lib().aa_linear_dlogits(*head, buf[G:].data_ptr(), ld, mode_code, st))
        torch.cuda.synchronize()
        assert bool((buf[:G].view(torch.int16) == 0x7FA5).all()) and bool((buf[G + N * ld:].view(torch.int16) == 0x7FA5).all())
        return buf[G:G + N * ld].view(N, ld)

    d, d0 = run(True), run(False)
    assert not bool(d[:, V:].float().any())
    logits = torch.nn.functional.linear(h, w)  # the bf16 logits nn.Linear returns (FAITHFUL's rounding point)
    x = logits.float() if mode == 'faithful' else (h.double() @ w.double().t())
    want = _tile64(x[None], lab[None], g[None], g_h[None], torch.bfloat16 if mode == 'faithful' else None)[0]
    _close(d[:, :V], want, torch.bfloat16, f'K6b {mode} {V}')
    zero_rows = g_h == 0
    assert torch.equal(_bits(d[zero_rows]), _bits(d0[zero_rows]))


@pytest.mark.parametrize('path', ['k6', 'library'])
def test_lm_head_entropy_grad_vs_float64(ops, path):
    """linear_token_log_probs(return_entropy=True, entropy_grad=True): d(hidden) and d(weight) of
    sum(w_lp * lp) + sum(w_h * H) against float64 autograd of the same objective on the bf16 logits (F32 mode)."""
    torch.manual_seed(3)
    N, H, V = 384, 256, 32001
    dt = torch.bfloat16 if path == 'k6' else torch.float32  # fp32 operands take the library-GEMM path around K1 / K1b
    hid = torch.randn(N, H, device=DEV).to(dt).requires_grad_(True)
    w = (torch.randn(V, H, device=DEV) * (2.0 / H ** 0.5)).to(dt).requires_grad_(True)
    lab = torch.randint(0, V, (N,), device=DEV)
    wl, wh = torch.randn(N, device=DEV), torch.randn(N, device=DEV)
    lp, ent = ops.linear_token_log_probs(hid, w, lab, chunk_rows=128, mode='f32', return_entropy=True, entropy_grad=True)
    assert ent.requires_grad
    ((lp.float() * wl).sum() + (ent * wh).sum()).backward()
    h64 = hid.detach().double().requires_grad_(True)
    w64 = w.detach().double().requires_grad_(True)
    lsm = torch.log_softmax(h64 @ w64.t(), -1)
    e64 = -(lsm.exp() * lsm).sum(-1)
    ((lsm.gather(-1, lab[:, None]).squeeze(-1) * wl.double()).sum() + (e64 * wh.double()).sum()).backward()
    assert float((ent.double() - e64.detach()).abs().max()) <= 1e-3
    _rel(hid.grad, h64.grad, 2e-2, 'd hidden')
    _rel(w.grad, w64.grad, 2e-2, 'd weight')
