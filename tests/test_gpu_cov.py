"""Clip-Cov and KL-Cov on the H100: the device selection against the port (tests/cov_port.py) bit for bit, the PPO
and GRPO losses and gradients against float64 autograd of the port on NaN-guarded buffers, the composed dense node
against the same, run-to-run bits, and one rl_step / step_from_rollout of each trainer with each mode."""
from __future__ import annotations

from types import SimpleNamespace

import pytest
import torch

import cov_port as port
from grpo_objective_port import completion_mask
from test_gpu_entropy import _bits
from test_gpu_parity import ops  # noqa: F401  (fixture)
from test_gpu_ppo_objective import Guarded, _rel

pytestmark = pytest.mark.gpu
DEV = 'cuda'
MODES = ['clip_cov', 'kl_cov']
EOS = 2


def _data(B, W, dtype, seed, kind='random'):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, W, generator=g) * 4
    adv = torch.randn(B, W, generator=g) * 2
    if kind == 'ties':  # few distinct values: many equal covariances, and +-0 among them
        lp = -torch.randint(0, 3, (B, W), generator=g).float()
        adv = torch.randint(-1, 2, (B, W), generator=g).float()
    old = lp + torch.randn(B, W, generator=g) * 0.3
    mask = torch.rand(B, W, generator=g) < 0.8
    mask[0, :] = True
    return (lp.to(dtype).to(DEV), old.to(dtype).to(DEV), adv.to(DEV), mask.to(DEV))


def _device_means(lp, adv, mask, row_end):
    """aa_cov_moments' fp32 means, read from its state words."""
    from align_anything_b200 import _lib as L

    B, W = lp.shape
    state = torch.zeros(16, dtype=torch.int32, device=DEV)
    m = mask.to(torch.uint8).contiguous() if mask is not None else None
    L.check(L.lib().aa_cov_moments(lp.data_ptr(), lp.stride(0), L.dtype_code(lp.dtype), adv.data_ptr(),
                                   adv.stride(0) if m is not None else 0, L.dtype_code(adv.dtype), L.ptr(m),
                                   m.stride(0) if m is not None else 0, L.ptr(row_end), B, W, state.data_ptr(),
                                   L.stream_ptr(lp.device)))
    return state[7:9].view(torch.float32).cpu()


def _ulps(a, b):
    return abs(int(a.view(torch.int32)) - int(b.view(torch.int32)))


@pytest.mark.parametrize('ratio', [2e-4, 0.05, 0.3])
@pytest.mark.parametrize('kind', ['random', 'ties'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('layout', ['mask', 'row_end'])
@pytest.mark.parametrize('mode', MODES)
def test_selection_equals_port(ops, mode, layout, dtype, kind, ratio):
    B, W = 32, 512
    lp, old, adv, mask = _data(B, W, dtype, 11, kind)
    if layout == 'row_end':
        g = torch.Generator().manual_seed(5)
        row_end = torch.randint(0, W + 1, (B,), generator=g).to(torch.int32).to(DEV)
        adv = adv[:, 0].contiguous()
        counted = torch.arange(W, device=DEV) < row_end.unsqueeze(1)
        a_full, sel_arg, m_arg = adv.view(-1, 1).expand(B, W), row_end, None
    else:
        counted, a_full, sel_arg, m_arg, row_end = mask, adv, mask, mask, None
    seed = port.hash_seed(7, 0, 3)
    kw = dict(clip_cov_ratio=ratio, clip_cov_lb=-1.0 if kind == 'ties' else 1.0, kl_cov_ratio=ratio)
    kw = {k: v for k, v in kw.items() if (k == 'kl_cov_ratio') == (mode == 'kl_cov')}
    sel, share = ops.cov_token_selection(lp, adv, sel_arg, mode, old_log_probs=old, clip_range_ratio_low=0.2,
                                         clip_range_ratio_high=0.28, seed=seed, return_share=True, mode='f32', **kw)
    ma, ml = _device_means(lp, adv, m_arg, row_end)
    wa, wl = port.means(lp.cpu(), a_full.cpu(), counted.cpu())
    assert _ulps(ma, wa) <= 1 and _ulps(ml, wl) <= 1, (ma, wa, ml, wl)
    cov = port.covariance(lp, a_full, ma.to(DEV), ml.to(DEV))
    if mode == 'kl_cov':
        want = port.kl_cov_select(cov, counted, ratio)
    else:
        clip = port.clipped(lp.float(), old.float(), a_full, 0.2, 0.28)
        want = port.clip_cov_select(cov, counted, clip, ratio, kw['clip_cov_lb'], 5.0, seed)
    assert torch.equal(sel.bool(), want), (int(sel.sum()), int(want.sum()))
    n = int(counted.sum())
    k = int(want.sum())
    assert k <= port.n_select(ratio, n) and (mode == 'clip_cov' or k == port.n_select(ratio, n))
    assert float(share) == pytest.approx(k / n if n else 0.0, rel=1e-6)
    again = ops.cov_token_selection(lp, adv, sel_arg, mode, old_log_probs=old, clip_range_ratio_low=0.2,
                                    clip_range_ratio_high=0.28, seed=seed, mode='f32', **kw)
    assert torch.equal(again, sel)
    ops.check_status()


def test_selection_order_of_signed_zero_and_nan(ops):
    """KL-Cov's key: NaN above +inf, -0.0 == +0.0 (ties to the smaller flat index)."""
    lp = torch.tensor([[-1.0, -2.0, -3.0, -1.0, -2.0, -3.0]], device=DEV)
    adv = torch.tensor([[0.0, float('nan'), 1.0, 0.0, -1.0, 5.0]], device=DEV)
    mask = torch.ones_like(lp, dtype=torch.bool)
    mask[0, 1] = False  # the NaN advantage is not counted: the means stay finite
    lp2, adv2 = lp.clone(), adv.clone()
    lp2[0, 1], adv2[0, 1], mask[0, 1] = float('nan'), 1.0, True  # a counted NaN log-prob: NaN means, NaN covariances
    sel = ops.cov_token_selection(lp2, adv2, mask, 'kl_cov', kl_cov_ratio=0.5)
    assert int(sel.sum()) == 3 and sel[0, :3].bool().all()  # all NaN: the first three by index
    m = torch.tensor([[True, False, True, True, True, True]], device=DEV)
    a = torch.tensor([[1.0, 0.0, 1.0, 1.0, 1.0, 1.0]], device=DEV)  # A == mean A: every cov is +-0
    sel = ops.cov_token_selection(lp, a, m, 'kl_cov', kl_cov_ratio=0.4)
    assert sel.tolist() == [[1, 0, 1, 0, 0, 0]]
    ops.check_status()


def _guarded(*ts):
    return [Guarded(t) for t in ts]


@pytest.mark.parametrize('agg', ['seq-mean-token-mean', 'token-mean'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('mode', MODES)
def test_ppo_loss_and_grad_vs_port(ops, mode, dtype, agg):
    B, W = 16, 200
    lp, old, adv, mask = _data(B, W, dtype, 23)
    g_lp, g_old, g_adv = _guarded(lp, old, adv)
    x = g_lp.view.detach().requires_grad_(True)  # the guarded view itself: the kernels read it through its stride
    kw = {'clip_cov_ratio': 0.1, 'clip_range_ratio_low': 0.2, 'clip_range_ratio_high': 0.28} if mode == 'clip_cov' \
        else {'kl_cov_ratio': 0.1, 'ppo_kl_coef': 0.5}
    obj = ops.ActorObjective(policy_loss_mode=mode, loss_agg_mode=agg, **kw)
    seed = port.hash_seed(1, 0, 0)
    loss, share = ops.actor_loss(x, g_old.view, g_adv.view, mask, 0.2, mode='f32', objective=obj, cov_seed=seed)
    loss.backward()
    sel_kw = {k: v for k, v in kw.items() if k != 'ppo_kl_coef'}
    sel = ops.cov_token_selection(lp, adv, mask, mode, old_log_probs=old, seed=seed, mode='f32', **sel_kw).bool()
    assert 0 < int(sel.sum()) and float(share) == pytest.approx(int(sel.sum()) / int(mask.sum()), rel=1e-6)
    lp64 = lp.double().requires_grad_(True)
    want = port.ppo_loss(mode, lp64, old.double(), adv.double(), mask, sel, agg, 0.2, 0.28, 0.5)
    want.backward()
    assert abs(float(loss) - float(want)) <= 1e-5 * max(1.0, abs(float(want)))
    _rel(x.grad, lp64.grad, 1e-5 if dtype == torch.float32 else 2e-2, 'd loss / d lp')
    if mode == 'clip_cov':
        assert (x.grad[sel] == 0).all()
    assert g_lp.intact() and g_old.intact() and g_adv.intact()
    ops.check_status()


@pytest.mark.parametrize('agg', ['token-mean', 'seq-mean-token-mean', 'seq-mean-token-sum-norm'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('first', [True, False])
@pytest.mark.parametrize('mode', MODES)
def test_grpo_loss_and_grad_vs_port(ops, mode, first, dtype, agg):
    B, K = 8, 96
    g = torch.Generator().manual_seed(3)
    lp, old, _, _ = _data(B, K, dtype, 31)
    ref = (lp.float().cpu() + torch.randn(B, K, generator=g) * 0.1).to(dtype).to(DEV)
    tok = torch.randint(3, 50, (B, K), generator=g)
    tok[1, 40], tok[5, 3] = EOS, EOS
    tok = tok.to(DEV)
    adv = torch.randn(B, 1, generator=g).to(DEV)
    obj = ops.GrpoObjective(policy_loss_mode=mode, loss_agg_mode=agg,
                            **({'clip_cov_ratio': 0.1, 'clip_cov_lb': -5.0} if mode == 'clip_cov' else
                               {'kl_cov_ratio': 0.1, 'ppo_kl_coef': 0.7}))
    g_lp = Guarded(lp)
    x = g_lp.view.detach().requires_grad_(True)
    kw = {} if first else {'old_per_token_logps': old}
    loss, row_end, share = ops.grpo_loss(x, ref, adv, tok, EOS, 0.04, mode='f32', objective=obj, cov_seed=9, **kw)
    loss.backward()
    mask = completion_mask(tok, EOS)
    assert torch.equal(torch.arange(K, device=DEV) < row_end.unsqueeze(1), mask.bool())
    sel = ops.cov_token_selection(lp, adv, row_end, mode, old_log_probs=None if first else old, seed=9, mode='f32',
                                  clip_range_ratio_low=0.2, clip_range_ratio_high=0.2,
                                  **({'clip_cov_ratio': 0.1, 'clip_cov_lb': -5.0} if mode == 'clip_cov' else
                                     {'kl_cov_ratio': 0.1})).bool()
    assert int(sel.sum()) > 0
    lp64 = lp.double().requires_grad_(True)
    want = port.grpo_loss(mode, lp64, ref.double(), None if first else old.double(), adv.double(), mask, sel, 0.04,
                          agg, 0.2, 0.2, 0.7)
    want.backward()
    assert abs(float(loss) - float(want)) <= 1e-5 * max(1.0, abs(float(want)))
    _rel(x.grad, lp64.grad, 1e-5 if dtype == torch.float32 else 2e-2, 'd loss / d lp')
    assert g_lp.intact()
    ops.check_status()


@pytest.mark.parametrize('mode', MODES)
def test_dense_node_vs_port_and_run_to_run_bits(ops, mode):
    """The composed node (K1 -> selection -> K5 Cov -> K1b) against float64 autograd through log_softmax."""
    g = torch.Generator().manual_seed(8)
    B, Lq, V, start = 4, 70, 1031, 10
    logits = (torch.randn(B, Lq, V, generator=g) * 2).to(DEV)
    ids = torch.randint(0, V, (B, Lq), generator=g).to(DEV)
    W = Lq - 1 - start
    old = (-torch.rand(B, W, generator=g) * 6).to(DEV)
    adv = torch.randn(B, W, generator=g).to(DEV)
    mask = (torch.rand(B, W, generator=g) < 0.9).to(DEV)
    obj = ops.ActorObjective(policy_loss_mode=mode, **({'clip_cov_ratio': 0.05, 'clip_cov_lb': -1e3,
                                                        'clip_cov_ub': 1e3} if mode == 'clip_cov' else
                                                       {'kl_cov_ratio': 0.05}))
    runs = []
    for _ in range(2):
        x = logits.clone().requires_grad_(True)
        out = ops.dense_actor_loss(x, ids, start, old, adv, mask, 0.2, mode='f32', objective=obj, cov_seed=4)
        out[0].backward()
        runs.append((out[0].detach(), x.grad, out[-1]))
    assert torch.equal(_bits(runs[0][0]), _bits(runs[1][0])) and torch.equal(_bits(runs[0][1]), _bits(runs[1][1]))
    lp = ops.gather_log_probabilities(logits[:, start:-1], ids[:, start + 1:], mode='f32')  # the node's own K1
    sel = ops.cov_token_selection(lp, adv, mask, mode, old_log_probs=old, seed=4, mode='f32',
                                  **({'clip_cov_ratio': 0.05, 'clip_cov_lb': -1e3, 'clip_cov_ub': 1e3}
                                     if mode == 'clip_cov' else {'kl_cov_ratio': 0.05})).bool()
    assert int(sel.sum()) == max(int(0.05 * int(mask.sum())), 1)
    x64 = logits.double().requires_grad_(True)
    lp64 = torch.log_softmax(x64[:, start:-1], -1).gather(-1, ids[:, start + 1:, None]).squeeze(-1)
    want = port.ppo_loss(mode, lp64, old.double(), adv.double(), mask, sel)
    want.backward()
    assert abs(float(runs[0][0]) - float(want)) <= 1e-4 * max(1.0, abs(float(want)))
    _rel(runs[0][1][:, start:-1], x64.grad[:, start:-1], 1e-4, 'd loss / d logits')
    assert float(runs[0][2]) == pytest.approx(int(sel.sum()) / int(mask.sum()), rel=1e-6)
    ops.check_status()


def test_vanilla_is_todays_node(ops):
    lp, old, adv, mask = _data(8, 64, torch.float32, 2)
    outs = []
    for obj in (None, ops.ActorObjective(policy_loss_mode='vanilla')):
        x = lp.clone().requires_grad_(True)
        loss = ops.actor_loss(x, old, adv, mask, 0.2, objective=obj)
        loss.backward()
        outs.append((loss.detach(), x.grad))
    assert torch.equal(_bits(outs[0][0]), _bits(outs[1][0])) and torch.equal(_bits(outs[0][1]), _bits(outs[1][1]))
    ops.check_status()


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('trainer', ['ppo', 'multi_ppo'])
def test_text_trainers_report_the_cov_fraction(ops, trainer, mode):
    from test_gpu_whiten import _ids, _text_trainer

    if trainer == 'ppo':
        from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer
        kw = {}
    else:
        from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer
        kw = {'advantage_estimator': 'reinforce', 'n_samples_per_prompt': 2}
    ids, P = _ids(4, seed=13), 12
    tr, prompts, state, _, _ = _text_trainer(PPOTrainer, ids, P, 2, False, **kw)
    tr.cfgs.train_cfgs.policy_loss_mode = mode
    tr.cfgs.train_cfgs.seed = 42
    if mode == 'clip_cov':  # every unclipped token eligible: the tiny rollout selects one
        tr.cfgs.train_cfgs.clip_cov_lb, tr.cfgs.train_cfgs.clip_cov_ub = -1e3, 1e3
    if trainer == 'multi_ppo':
        prompts = {k: v[::2] for k, v in prompts.items()}
    inference, training = tr.rollout(prompts)
    state['phase'] = 'train'
    out = tr.rl_step(inference[0], training[0])
    assert 0.0 < out['train/actor_cov_fraction'] <= 1.0
    assert getattr(tr, 'cov_calls', 0) == (1 if mode == 'clip_cov' else 0)
    ops.check_status()


@pytest.mark.parametrize('mode', MODES)
def test_image_trainer_reports_the_cov_fraction(ops, mode):
    from test_gpu_fused_rl import LM, Critic, Phased

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
    critic, new_critic = t(B, Lq, 1).to(DEV), t(B, Lq, 1).to(DEV).requires_grad_(True)
    bounds = {'clip_cov_lb': -1e3, 'clip_cov_ub': 1e3} if mode == 'clip_cov' else {}
    tr = PPOTrainer(SimpleNamespace(train_cfgs=SimpleNamespace(policy_loss_mode=mode, **bounds)),
                    tokenizer=SimpleNamespace(pad_token_id=0))
    state = {'phase': 'rollout'}
    tr.actor_model = Phased(LM(hid_a, w_a), LM(hid_new.clone().requires_grad_(True), w_a.clone().requires_grad_(True)),
                            state)
    tr.actor_reference_model = LM(hid_r, w_r)
    tr.reward_model = Critic(lambda: ScoreModelOutput(end_scores=reward.unsqueeze(-1)))
    tr.reward_critic_model = Critic(lambda: ScoreModelOutput(scores=critic if state['phase'] == 'rollout' else new_critic))
    tr.actor_step = lambda mini: ({'input_ids': ids, 'attention_mask': ids != 0}, ops.as_device_lens(resp, DEV))
    inference, training = tr.rollout({'input_ids': ids[:, :12], 'attention_mask': ids[:, :12] != 0})
    state['phase'] = 'train'
    out = tr.rl_step(inference[0], training[0])
    assert out['train/actor_cov_fraction'] == pytest.approx(1 / sum(resp), rel=1e-6)
    ops.check_status()


@pytest.mark.parametrize('mode', MODES)
def test_grpo_two_updates_report_the_cov_fraction_and_paths_agree(ops, mode):
    from test_gpu_fused_rl import _grpo_sequences
    from test_gpu_top_entropy import _run

    seq = _grpo_sequences(7)
    cfg = dict(num_iterations=2, policy_loss_mode=mode, log_clip_fraction=True,
               **({'clip_cov_ratio': 0.2, 'clip_cov_lb': -100.0, 'clip_cov_ub': 100.0} if mode == 'clip_cov' else
                  {'kl_cov_ratio': 0.2}))
    a, pa, _ = _run(False, seq, 16, 128, 2053, 49, 1e-4, **cfg)
    b, pb, _ = _run(True, seq, 16, 128, 2053, 49, 1e-4, **cfg)
    assert 0.0 < a['train/actor_cov_fraction'] <= 0.2 * (1 + 1e-6)  # int(0.2 * N) / N, the fp32 mean of two updates
    assert set(a) == set(b)
    for k, v in a.items():
        assert abs(v - b[k]) <= 1e-2 * max(1.0, abs(v)), (k, v, b[k])
    for u in range(2):
        _rel(pb.grads[u][0], pa.grads[u][0].double(), 2e-2, f'update {u + 1}: fused d hidden')
        _rel(pb.grads[u][1], pa.grads[u][1].double(), 2e-2, f'update {u + 1}: fused d weight')
    ops.check_status()
