"""PPO actor objective options on the GPU: clip-higher, dual-clip and token-mean aggregation in K5 (through the C ABI, on
guard-banded buffers), in K1f (dense and tail-plan nodes at V = 152064), in the fused lm_head node and in one step of the
text, Multi-PPO and image PPO trainers, held to tests/ppo_objective_port.py and to float64 autograd.  With every option at
its default the outputs are bit-identical to today's launches."""
from __future__ import annotations

import pytest
import torch

from ppo_objective_port import actor_loss as port_loss
from ppo_objective_port import clip_fractions
from test_gpu_entropy import _bits
from test_gpu_parity import assert_ulp_close, ops  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

DEV = 'cuda'
AGG = {'seq-mean-token-mean': 0, 'token-mean': 1}
# (clip_low, clip_high, dual_clip, loss_agg_mode): each option alone, then all together
OPTIONS = {
    'clip-higher': (0.2, 0.28, None, 'seq-mean-token-mean'),
    'dual-clip': (0.2, 0.2, 3.0, 'seq-mean-token-mean'),
    'token-mean': (0.2, 0.2, None, 'token-mean'),
    'all': (0.2, 0.28, 3.0, 'token-mean'),
}


def _objective(opt):
    from align_anything_b200.ops import ActorObjective

    lo, hi, c, agg = opt
    return ActorObjective(lo, hi, c, agg)


def _loss_inputs(B, W, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, W, generator=g) * 4
    old = lp + torch.randn(B, W, generator=g) * 0.5  # ratios inside and far outside the clip ranges
    adv = torch.randn(B, W, generator=g)
    mask = torch.rand(B, W, generator=g) > 0.2
    mask[:, 0] = True
    mask[-1, W // 2:] = False
    return lp.to(dtype).to(DEV), old.to(dtype).to(DEV), adv.to(dtype).to(DEV), mask.to(DEV)


class Guarded:
    """A (B, W) tensor inside a NaN-filled (B + 2, W + 2 * pad) buffer: the kernel sees the interior through its row
    stride; `intact()` checks that nothing outside it was written."""

    def __init__(self, t: torch.Tensor, pad: int = 16, fill=float('nan')):
        B, W = t.shape
        self.buf = torch.full((B + 2, W + 2 * pad), fill, dtype=t.dtype, device=t.device)
        self.view = self.buf[1:B + 1, pad:pad + W]
        self.view.copy_(t)
        self.ref = self.buf.clone()
        self.pad = pad

    def intact(self) -> bool:
        keep = torch.ones_like(self.buf, dtype=torch.bool)
        keep[1:-1, self.pad:-self.pad] = False
        got, want = self.buf[keep], self.ref[keep]
        return torch.equal(got, want) if got.element_size() == 1 else torch.equal(_bits(got), _bits(want))


def _k5(ops, lp, old, adv, mask, obj, mode, legacy=False):
    """K5 through the C ABI on guarded buffers -> (loss fp32[2], grad, clip fractions)."""
    from align_anything_b200 import _lib as L

    B, W = lp.shape
    mode_code = L.MODE_FAITHFUL if mode == 'faithful' else L.MODE_F32
    gl, go, ga = Guarded(lp), Guarded(old), Guarded(adv)
    gm = Guarded(mask.to(torch.uint8), fill=1)
    grad = Guarded(torch.zeros_like(lp))
    loss = Guarded(torch.zeros(1, 2, dtype=torch.float32, device=DEV))
    cf = Guarded(torch.zeros(1, 2, dtype=torch.float32, device=DEV))
    rows = torch.full((4 * B,), float('nan'), dtype=torch.float32, device=DEV)
    counter = torch.zeros(1, dtype=torch.int32, device=DEV)
    lib = L.lib()
    common = (gl.view.data_ptr(), gl.view.stride(0), go.view.data_ptr(), go.view.stride(0), L.dtype_code(lp.dtype),
              ga.view.data_ptr(), ga.view.stride(0), L.dtype_code(adv.dtype), gm.view.data_ptr(), gm.view.stride(0), B, W)
    if legacy:
        L.check(lib.aa_ppo_actor_loss(*common, float(obj[0]), mode_code, loss.view.data_ptr(), grad.view.data_ptr(),
                                      grad.view.stride(0), rows.data_ptr(), counter.data_ptr(), L.stream_ptr(DEV)))
    else:
        lo, hi, c, agg = obj
        L.check(lib.aa_ppo_actor_loss_obj(*common, float(lo), float(hi), float(c or 0.0), AGG[agg], mode_code,
                                          loss.view.data_ptr(), grad.view.data_ptr(), grad.view.stride(0),
                                          cf.view.data_ptr(), rows.data_ptr(), counter.data_ptr(), L.stream_ptr(DEV)))
    torch.cuda.synchronize()
    for g in (gl, go, ga, gm, grad, loss, cf):
        assert g.intact(), 'a guard band was written'
    return loss.view[0].clone(), grad.view.clone(), cf.view[0].clone()


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize('mode', ['faithful', 'f32'])
@pytest.mark.parametrize('name', list(OPTIONS))
def test_k5_objective_c_abi_vs_port(ops, dtype, mode, name):
    lo, hi, c, agg = opt = OPTIONS[name]
    B, W = 7, 301
    lp, old, adv, mask = _loss_inputs(B, W, dtype, seed=list(OPTIONS).index(name))
    loss, grad, cf = _k5(ops, lp, old, adv, mask, opt, mode)
    faithful = mode == 'faithful' and dtype != torch.float32
    cd = dtype if faithful else torch.float32  # the port on ATen CUDA in the dtype the kernel rounds to
    x = lp.to(cd).clone().requires_grad_(True)
    want = port_loss(x, old.to(cd), adv.to(cd), mask, lo, hi, c, agg)
    want.backward()
    if faithful:
        got16 = loss[1:2].view(dtype)[:1] if dtype != torch.float32 else loss[:1]
        assert_ulp_close(got16.reshape(()), want.detach(), max_ulp=1, min_exact=0.0, what=f'{name} loss')
        assert_ulp_close(grad, x.grad, max_ulp=1, min_exact=0.97, what=f'{name} grad')
    else:
        torch.testing.assert_close(loss[0], want.detach().float(), rtol=2e-5, atol=0.0)
        if dtype == torch.float32:
            torch.testing.assert_close(grad, x.grad, rtol=2e-5, atol=2e-5 * float(x.grad.abs().max()))
        else:  # F32 mode keeps fp32 throughout and rounds the gradient once, to the log-probs' dtype
            assert_ulp_close(grad, x.grad.to(dtype), max_ulp=1, min_exact=0.97, what=f'{name} grad')
    # the port's counts on its own ratios: a ratio one ulp away from ATen's (the kernel's expf) can sit exactly on a
    # clip bound, so one token may change sides
    fc, fd = clip_fractions(lp.to(cd), old.to(cd), adv.to(cd), mask, lo, hi, c, agg)
    n = float(mask.sum())
    assert abs(float(cf[0]) - fc) <= 1.0 / n + 1e-6, (float(cf[0]), fc)
    assert abs(float(cf[1]) - fd) <= 1.0 / float(((adv < 0) & mask).sum()) + 1e-6, (float(cf[1]), fd)
    if c is None:
        assert float(cf[1]) == 0.0


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize('mode', ['faithful', 'f32'])
def test_k5_default_objective_is_the_legacy_entry_point(ops, dtype, mode):
    lp, old, adv, mask = _loss_inputs(5, 129, dtype, seed=7)
    a = _k5(ops, lp, old, adv, mask, (0.2, 0.2, None, 'seq-mean-token-mean'), mode)
    b = _k5(ops, lp, old, adv, mask, (0.2, 0.2, None, 'seq-mean-token-mean'), mode, legacy=True)
    assert torch.equal(_bits(a[0]), _bits(b[0])) and torch.equal(_bits(a[1]), _bits(b[1]))


def test_k5_exact_operands_vs_float64(ops):
    # exact operands: lp == old (r = exp(0) = 1, the s1 == s2 tie on every token), dyadic advantages, row mask counts
    # and their total powers of two: every op of the fp32 kernel is exact, so it equals float64 bit for bit
    B, W = 4, 64
    g = torch.Generator().manual_seed(5)
    lp = (-torch.randint(1, 64, (B, W), generator=g).float() / 16).to(DEV)
    adv = (torch.randint(-32, 32, (B, W), generator=g).float() / 8).to(DEV)
    mask = torch.zeros(B, W, dtype=torch.bool, device=DEV)
    for b, n in enumerate((8, 8, 16, 32)):
        mask[b, :n] = True
    for opt in OPTIONS.values():
        lo, hi, c, agg = opt
        for dtype in (torch.float32,):
            loss, grad, _ = _k5(ops, lp.to(dtype), lp.to(dtype), adv.to(dtype), mask, opt, 'faithful')
            x = lp.double().clone().requires_grad_(True)
            want = port_loss(x, lp.double(), adv.double(), mask, lo, hi, c, agg)
            want.backward()
            assert float(loss[0]) == float(want.detach()), (opt, dtype)
            assert torch.equal(grad.double(), x.grad), (opt, dtype)


# ---- K1f: the single-pass node against the composed path with the same objective --------------------------------------
def _node(ops, node, logits, ids, start, lens, old, adv, mask, mode, **kw):
    leaf = logits.clone().requires_grad_(True)
    if node == 'dense':
        out = ops.dense_actor_loss(leaf, ids, start, old, adv, mask, 0.2, mode=mode, **kw)
    else:
        out = ops.tail_actor_loss(leaf, ids, lens, old, adv, mask, 0.2, mode=mode, **kw)
    out[0].backward()
    return out, leaf.grad


def _node_inputs(node, dtype, V, seed):
    torch.manual_seed(seed)
    B, Lq = 4, 12
    logits = (torch.randn(B, Lq, V, device=DEV) * 2.0).to(dtype)
    ids = torch.randint(0, V, (B, Lq), device=DEV)
    if node == 'dense':
        start, lens = 3, None
        W = Lq - 1 - start
        mask = torch.ones(B, W, dtype=torch.bool, device=DEV)
        mask[1, -3:] = False
    else:
        start, lens = None, [8, 3, 11, 6]
        W = max(lens)
        mask = torch.arange(W, device=DEV)[None, :] < torch.tensor(lens, device=DEV)[:, None]
    return logits, ids, start, lens, W, mask


@pytest.mark.parametrize('node', ['dense', 'tail'])
@pytest.mark.parametrize('dtype,mode', [(torch.bfloat16, 'faithful'), (torch.bfloat16, 'f32'), (torch.float32, 'f32')])
def test_k1f_objective_vs_composed_path(ops, monkeypatch, node, dtype, mode):
    V = 152064
    logits, ids, start, lens, W, mask = _node_inputs(node, dtype, V, seed=11)
    B = logits.size(0)
    # old log-probs near the new ones: ratios inside and outside the clip ranges
    plain, _ = _node(ops, node, logits, ids, start, lens, torch.zeros(B, W, device=DEV), torch.zeros(B, W, device=DEV),
                     mask, mode)
    old = (plain[1].float() + torch.randn(B, W, device=DEV) * 0.3).to(plain[1].dtype)
    adv = torch.randn(B, W, device=DEV).to(dtype)
    base, gbase = _node(ops, node, logits, ids, start, lens, old, adv, mask, mode)
    # default fields: the very launches (and bits) of the node without the switch
    dflt, gdflt = _node(ops, node, logits, ids, start, lens, old, adv, mask, mode,
                        objective=_objective((None, None, None, 'seq-mean-token-mean')))
    assert len(dflt) == len(base)
    assert torch.equal(_bits(gdflt), _bits(gbase)) and torch.equal(_bits(dflt[1]), _bits(base[1]))
    # the loss (the fp32[2] buffer's second word holds the 16-bit loss in its low half only)
    assert torch.equal(_bits(dflt[0].detach()), _bits(base[0].detach())) and torch.equal(_bits(dflt[2][:1]), _bits(base[2][:1]))
    for name, opt in OPTIONS.items():
        obj = _objective(opt)
        for coeff in ((0.0, 0.05) if obj.token_mean else (0.0,)):
            kw = dict(objective=obj, return_clip_fraction=True, entropy_coeff=coeff)
            one, gone = _node(ops, node, logits, ids, start, lens, old, adv, mask, mode, **kw)
            assert torch.equal(_bits(one[1]), _bits(base[1])), f'{name}: log-probs differ from the default single pass'
            monkeypatch.setattr(ops, '_FUSED_ACTOR', False)
            two, gtwo = _node(ops, node, logits, ids, start, lens, old, adv, mask, mode, **kw)
            monkeypatch.setattr(ops, '_FUSED_ACTOR', True)
            what = f'{node} {name} coeff={coeff}'
            if dtype == torch.float32 or mode == 'f32':
                scale = float(gtwo.float().abs().max())
                assert float((gone.float() - gtwo.float()).abs().max()) <= 1e-5 * scale + 1e-12, what
            else:
                assert_ulp_close(gone, gtwo, max_ulp=2, min_exact=0.97, what=what)
            zero_rows = lambda g: (g.reshape(-1, V) == 0).all(-1)  # noqa: E731
            assert torch.equal(zero_rows(gone), zero_rows(gtwo)), what
            assert float(one[0]) == pytest.approx(float(two[0]), rel=1e-5, abs=1e-7), what
            assert torch.equal(one[-1], two[-1]), what  # the clip fractions (K5 on the same log-probs)
    ops.check_status()


def test_k1f_default_objective_with_entropy_is_the_legacy_launch(ops):
    logits, ids, start, lens, W, mask = _node_inputs('dense', torch.bfloat16, 152064, seed=13)
    B = logits.size(0)
    old = torch.full((B, W), -11.0, device=DEV)
    adv = torch.randn(B, W, device=DEV)
    a, ga = _node(ops, 'dense', logits, ids, start, lens, old, adv, mask, None, entropy_coeff=0.05)
    b, gb = _node(ops, 'dense', logits, ids, start, lens, old, adv, mask, None, entropy_coeff=0.05,
                  objective=_objective((None, None, None, 'seq-mean-token-mean')))
    assert torch.equal(_bits(ga), _bits(gb)) and torch.equal(_bits(a[0]), _bits(b[0]))


# ---- trainers -------------------------------------------------------------------------------------------------------
def _with(cls, **attrs):
    return type(cls.__name__, (cls,), attrs)


ALL_ON = dict(clip_range_ratio_low=0.2, clip_range_ratio_high=0.28, dual_clip_ratio=3.0, loss_agg_mode='token-mean',
              log_clip_fraction=True)


def _objective64(lp, old, adv, mask, lo=0.2, hi=0.28, c=3.0, agg='token-mean'):
    """The objective in float64 (lp: float64 with grad)."""
    return port_loss(lp, old.double(), adv.double(), mask.double(), lo, hi, c, agg)


def _param_grads(dlogits64, h, w):
    return dlogits64 @ w.double(), torch.einsum('blv,blh->vh', dlogits64, h.double())


def _rel(got, want, rel, what):
    err = float((got.double() - want).abs().max())
    scale = max(1e-12, float(want.abs().max()))
    assert err <= rel * scale, (what, err, scale)


def _check_lanes(out, lp64, old, adv, mask):
    fc, fd = clip_fractions(lp64.detach(), old.double(), adv.double(), mask, 0.2, 0.28, 3.0, 'token-mean')
    n = float(mask.sum())
    assert abs(out['train/actor_clip_fraction'] - fc) <= 2.0 / n, (out['train/actor_clip_fraction'], fc)
    n_neg = max(1.0, float(((adv < 0) & mask).sum()))
    assert abs(out['train/actor_dual_clip_fraction'] - fd) <= 2.0 / n_neg, (out['train/actor_dual_clip_fraction'], fd)


@pytest.mark.parametrize('trainer', ['text', 'multi-rloo'])
def test_text_ppo_objective_step(ops, trainer):
    from test_gpu_fused_rl import _ppo_batch, _run_ppo

    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer as Multi
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer as Text

    cls, kw = (Text, {}) if trainer == 'text' else (Multi, {'advantage_estimator': 'rloo', 'n_samples_per_prompt': 2})
    ids = _ppo_batch(5)
    P, H, V, seed = 12, 128, 2053, 43
    plain = _run_ppo(cls, False, ids, P, H, V, seed, **kw)
    dflt = _run_ppo(_with(cls, loss_agg_mode='seq-mean-token-mean'), False, ids, P, H, V, seed, **kw)
    assert dflt[1] == plain[1]  # keys and values
    assert torch.equal(_bits(dflt[3]), _bits(plain[3])) and torch.equal(_bits(dflt[4]), _bits(plain[4]))
    on = _run_ppo(_with(cls, mode='f32', **ALL_ON), False, ids, P, H, V, seed, **kw)
    assert set(on[1]) == set(plain[1]) | {'train/actor_clip_fraction', 'train/actor_dual_clip_fraction'}
    gen = torch.Generator().manual_seed(seed)  # _run_ppo's draws: hid_a, hid_r, hid_new, w_a
    B, Lq = ids.shape
    for _ in range(2):
        torch.randn(B, Lq, H, generator=gen)
    h_new = torch.randn(B, Lq, H, generator=gen).bfloat16().to(DEV)
    w = (torch.randn(V, H, generator=gen) * 0.2).bfloat16().to(DEV)
    start = P - 1
    x = torch.nn.functional.linear(h_new, w).double().requires_grad_(True)
    lp64 = torch.log_softmax(x[:, start:-1], -1).gather(-1, ids[:, start + 1:, None]).squeeze(-1)
    old, adv = on[0]['log_probs'][:, start:], on[2]['advantages']
    mask = (ids != 0)[:, 1:][:, start:]
    loss64 = _objective64(lp64, old, adv, mask)
    loss64.backward()
    assert abs(on[1]['train/actor_loss'] - float(loss64)) <= 1e-4 * max(1.0, abs(float(loss64)))
    _check_lanes(on[1], lp64, old, adv, mask)
    dh, dw = _param_grads(x.grad, h_new, w)
    _rel(on[3], dh, 2e-2, 'd hidden')
    _rel(on[4], dw, 2e-2, 'd weight')
    # the fused lm_head node (K6 -> K5 with the objective -> K6b) against the tile path, FAITHFUL
    tile = _run_ppo(_with(cls, **ALL_ON), False, ids, P, H, V, seed, **kw)
    fused = _run_ppo(_with(cls, **ALL_ON), True, ids, P, H, V, seed, **kw)
    assert set(fused[1]) == set(tile[1])
    for k, v in tile[1].items():
        assert abs(v - fused[1][k]) <= 1e-2 * max(1.0, abs(v)), (k, v, fused[1][k])
    _rel(fused[3], tile[3].double(), 2e-2, 'fused d hidden')
    _rel(fused[4], tile[4].double(), 2e-2, 'fused d weight')
    ops.check_status()


def test_image_ppo_objective_step(ops):
    from types import SimpleNamespace

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

    plain, dflt = run(PPOTrainer), run(_with(PPOTrainer, loss_agg_mode='seq-mean-token-mean'))
    assert dflt[1] == plain[1]
    assert torch.equal(_bits(dflt[3]), _bits(plain[3])) and torch.equal(_bits(dflt[4]), _bits(plain[4]))
    on = run(_with(PPOTrainer, mode='f32', **ALL_ON))
    assert set(on[1]) == set(plain[1]) | {'train/actor_clip_fraction', 'train/actor_dual_clip_fraction'}
    x = torch.nn.functional.linear(hid_new, w_a).double().requires_grad_(True)
    W = max(resp)
    lp = torch.zeros(B, W, dtype=torch.float64, device=DEV)
    for b, r in enumerate(resp):
        lsm = torch.log_softmax(x[b, Lq - 1 - r:Lq - 1], -1)
        lp[b, :r] = lsm.gather(-1, ids[b, Lq - r:, None]).squeeze(-1)
    mask = on[0]['response_mask']
    loss64 = _objective64(lp, on[0]['log_probs'], on[2]['advantages'], mask)
    loss64.backward()
    assert abs(on[1]['train/actor_loss'] - float(loss64)) <= 1e-4 * max(1.0, abs(float(loss64)))
    _check_lanes(on[1], lp, on[0]['log_probs'], on[2]['advantages'], mask)
    dh, dw = _param_grads(x.grad, hid_new, w_a)
    _rel(on[3], dh, 2e-2, 'd hidden')
    _rel(on[4], dw, 2e-2, 'd weight')
    tile, fused = run(_with(PPOTrainer, **ALL_ON)), run(_with(PPOTrainer, **ALL_ON), True)
    assert set(fused[1]) == set(tile[1])
    for k, v in tile[1].items():
        assert abs(v - fused[1][k]) <= 1e-2 * max(1.0, abs(v)), (k, v, fused[1][k])
    _rel(fused[3], tile[3].double(), 2e-2, 'fused d hidden')
    _rel(fused[4], tile[4].double(), 2e-2, 'fused d weight')
    ops.check_status()
