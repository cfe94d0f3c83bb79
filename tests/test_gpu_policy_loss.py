"""CISPO and SAPO on the H100: aa_ppo_actor_loss_pm and aa_grpo_loss_pm through the C ABI on NaN-guarded buffers
against the port (tests/policy_loss_port.py) on ATen CUDA in the kernels' dtypes, K1f's PM nodes against the composed
path with the same mode, one rl_step of text PPO, Multi-PPO and image PPO and a two-update GRPO step per mode against
float64 autograd of the port, and the fused lm_head path against the tile path in each trainer."""
from __future__ import annotations

import pytest
import torch

import policy_loss_port as port
from grpo_objective_port import completion_mask
from test_gpu_entropy import _bits
from test_gpu_parity import assert_ulp_close, ops  # noqa: F401  (fixture)
from test_gpu_ppo_objective import Guarded, _rel

pytestmark = pytest.mark.gpu
DEV = 'cuda'
MODES = ['cispo', 'sapo']
AGG = {'seq-mean-token-mean': 0, 'token-mean': 1, 'seq-mean-token-sum-norm': 2}
CODE = {'cispo': 3, 'sapo': 4}
EPS_HI, TAU = 0.28, (1.0, 1.05)
EOS = 2


def _ulps(a, b):
    """Per-element distance in units in the last place of the (16- or 32-bit) dtype; NaN == NaN is 0."""
    bits = {2: torch.int16, 4: torch.int32}[a.element_size()]
    top = {2: 0x7fff, 4: 0x7fffffff}[a.element_size()]

    def ordered(t):
        i = t.contiguous().view(bits).long()
        return torch.where(i < 0, -(i & top), i)

    d = (ordered(a) - ordered(b)).abs()
    both_nan = torch.isnan(a) & torch.isnan(b)
    return torch.where(both_nan, torch.zeros_like(d), d)


def _close(got, want, faithful: bool, what):
    """FAITHFUL: within 1 ulp of the dtype and at least 97 % bit-identical; F32: within 2e-5 of the largest value."""
    assert got.dtype == want.dtype, what
    assert torch.equal(torch.isnan(got), torch.isnan(want)), what
    if faithful:
        u = _ulps(got, want)
        assert int(u.max()) <= 1, (what, int(u.max()))
        assert float((u == 0).double().mean()) >= 0.97, (what, float((u == 0).double().mean()))
    else:
        ok = ~torch.isnan(want)
        _rel(got[ok], want[ok].double(), 2e-5, what)


def _data(B, W, dtype, adv_dtype, seed):
    """Log-probs with ratios on both sides of 1 + EPS_HI, exactly at it and far beyond (a saturated sigmoid; an
    overflowing ratio in fp16), zero advantages, and a mask with every row counted."""
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, W, generator=g) * 3
    old = lp + torch.randn(B, W, generator=g) * 0.4
    adv = torch.randn(B, W, generator=g) * 2
    adv[:, 1] = 0.0
    mask = torch.rand(B, W, generator=g) < 0.8
    mask[:, :6] = True
    lp, old = lp.to(dtype), old.to(dtype)
    old[:, 2] = lp[:, 2]  # ratio 1
    hi = torch.tensor(1 + EPS_HI).to(dtype)
    old[:, 3] = (lp[:, 3].float() - torch.log(hi.float())).to(dtype)  # at or next to the bound
    old[:, 4] = lp[:, 4] - 12  # far beyond: sigma saturates
    old[:, 5] = lp[:, 5] + 12  # far below
    return lp.to(DEV), old.to(DEV), adv.to(adv_dtype).to(DEV), mask.to(DEV)


def _k5_pm(lp, old, adv, mask, mode, agg, faithful, kl=None):
    from align_anything_b200 import _lib as L

    B, W = lp.shape
    gl, go, ga = Guarded(lp), Guarded(old), Guarded(adv)
    gm = Guarded(mask.to(torch.uint8), fill=1)
    grad = Guarded(torch.zeros_like(lp))
    loss = Guarded(torch.zeros(1, 2, dtype=torch.float32, device=DEV))
    cf = Guarded(torch.zeros(1, 2, dtype=torch.float32, device=DEV))
    klo = Guarded(torch.zeros(1, 1, dtype=torch.float32, device=DEV))
    gr = Guarded(kl[0]) if kl is not None else None
    rows = torch.full((5 * B,), float('nan'), dtype=torch.float32, device=DEV)
    counter = torch.zeros(1, dtype=torch.int32, device=DEV)
    L.check(L.lib().aa_ppo_actor_loss_pm(
        gl.view.data_ptr(), gl.view.stride(0), go.view.data_ptr(), go.view.stride(0), L.dtype_code(lp.dtype),
        ga.view.data_ptr(), ga.view.stride(0), L.dtype_code(adv.dtype), gm.view.data_ptr(), gm.view.stride(0), B, W,
        EPS_HI, AGG[agg], CODE[mode], *TAU, L.MODE_FAITHFUL if faithful else L.MODE_F32,
        gr.view.data_ptr() if gr else None, gr.view.stride(0) if gr else 0, kl[1] if kl else 0.0, kl[2] if kl else 0,
        loss.view.data_ptr(), klo.view.data_ptr() if kl else None, grad.view.data_ptr(), grad.view.stride(0),
        cf.view.data_ptr(), rows.data_ptr(), counter.data_ptr(), L.stream_ptr(DEV)))
    torch.cuda.synchronize()
    for g in (gl, go, ga, gm, grad, loss, cf, klo) + ((gr,) if gr else ()):
        assert g.intact()
    return loss.view[0], grad.view, cf.view[0], klo.view[0, 0]


@pytest.mark.parametrize('kl', [None, 'k3', 'k2'])
@pytest.mark.parametrize('agg', ['seq-mean-token-mean', 'token-mean'])
@pytest.mark.parametrize('dtypes', [(torch.bfloat16, torch.bfloat16), (torch.float16, torch.float16),
                                    (torch.bfloat16, torch.float32), (torch.float32, torch.float32)])
@pytest.mark.parametrize('faithful', [True, False])
@pytest.mark.parametrize('mode', MODES)
def test_ppo_actor_loss_pm_against_the_port(ops, mode, faithful, dtypes, agg, kl):  # noqa: F811
    dtype, adv_dtype = dtypes
    B, W = 16, 300
    lp, old, adv, mask = _data(B, W, dtype, adv_dtype, seed=B + W)
    ref = (lp.float() - 0.05 * torch.randn(B, W, device=DEV)).to(dtype) if kl else None
    if not faithful:  # F32 mode reads and writes fp32 log-probs (the composed path's K1 writes them so)
        lp, old, ref = lp.float(), old.float(), ref.float() if kl else None
    loss, grad, cf, kl_out = _k5_pm(lp, old, adv, mask, mode, agg, faithful,
                                    (ref, 0.3, ops.KL_ESTIMATORS[kl]) if kl else None)
    cast = (lambda t: t) if faithful else (lambda t: t.float())
    x = cast(lp).clone().requires_grad_(True)
    if kl:
        want_loss, want_kl, total = port.actor_loss_kl(mode, x, cast(old), cast(adv), mask, agg, EPS_HI, *TAU,
                                                       cast(ref), 0.3, kl)
    else:
        want_loss = total = port.actor_loss(mode, x, cast(old), cast(adv), mask, agg, EPS_HI, *TAU)
    total.backward()
    _close(grad if faithful else grad.float(), x.grad, faithful, 'grad')
    want = want_loss.detach().float()
    assert abs(float(loss[0]) - float(want)) <= 4e-3 * max(1.0, abs(float(want))), (float(loss[0]), float(want))
    if faithful and want_loss.dtype != torch.float32:  # the 16-bit copy of the loss, as the port's 0-dim tensor
        got16 = loss[1:2].view(want_loss.dtype)[0]
        assert int(_ulps(got16.reshape(1), want_loss.detach().reshape(1))) <= 1
    if kl:
        assert abs(float(kl_out) - float(want_kl.detach())) <= 1e-2 * max(1e-3, abs(float(want_kl)))
    want_cf = port.clip_fraction(mode, lp, old, adv, mask, agg, EPS_HI) if faithful else \
        port.clip_fraction(mode, lp.float(), old.float(), adv.float(), mask, agg, EPS_HI)
    assert abs(float(cf[0]) - want_cf) <= 1e-6 and float(cf[1]) == 0.0


def _grpo_pm(lp, ref, old, adv, tok, mode, agg, est, faithful):
    from align_anything_b200 import _lib as L

    B, K = lp.shape
    gl, gr = Guarded(lp), Guarded(ref)
    go = Guarded(old) if old is not None else None
    grad = Guarded(torch.zeros_like(lp))
    loss = torch.zeros(1, dtype=torch.float32, device=DEV)
    cf = torch.zeros(2, dtype=torch.float32, device=DEV)
    row_end = torch.zeros(B, dtype=torch.int32, device=DEV)
    scratch = torch.full((1 + 4 * B,), float('nan'), dtype=torch.float32, device=DEV)
    counter = torch.zeros(2, dtype=torch.int32, device=DEV)
    L.check(L.lib().aa_grpo_loss_pm(
        gl.view.data_ptr(), gl.view.stride(0), gr.view.data_ptr(), gr.view.stride(0),
        go.view.data_ptr() if go else None, go.view.stride(0) if go else 0, L.dtype_code(lp.dtype), adv.data_ptr(),
        tok.data_ptr(), tok.stride(0), EOS, B, K, 0.04, EPS_HI, AGG[agg], est, CODE[mode], *TAU,
        L.MODE_FAITHFUL if faithful else L.MODE_F32, loss.data_ptr(), grad.view.data_ptr(), grad.view.stride(0),
        cf.data_ptr(), row_end.data_ptr(), scratch.data_ptr(), counter.data_ptr(), L.stream_ptr(DEV)))
    torch.cuda.synchronize()
    for g in (gl, gr, grad) + ((go,) if go else ()):
        assert g.intact()
    return loss[0], grad.view, cf


@pytest.mark.parametrize('est', ['k1', 'k3'])
@pytest.mark.parametrize('agg', ['token-mean', 'seq-mean-token-mean', 'seq-mean-token-sum-norm'])
@pytest.mark.parametrize('update', ['first', 'later'])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize('faithful', [True, False])
@pytest.mark.parametrize('mode', MODES)
def test_grpo_loss_pm_against_the_port(ops, mode, faithful, dtype, update, agg, est):  # noqa: F811
    B, K = 12, 257
    lp, old, _, _ = _data(B, K, dtype, torch.float32, seed=K + B)
    g = torch.Generator().manual_seed(5)
    adv = torch.randn(B, generator=g).to(DEV)
    adv[0] = 0.0
    ref = (lp.float() + 0.1 * torch.randn(B, K, device=DEV)).to(dtype)
    tok = torch.randint(3, 50, (B, K), generator=g)
    tok[1, 7], tok[2, 100] = EOS, EOS
    tok = tok.to(DEV)
    old = old if update == 'later' else None
    if not faithful:  # F32 mode reads and writes fp32 log-probs
        lp, ref, old = lp.float(), ref.float(), old.float() if old is not None else None
    loss, grad, cf = _grpo_pm(lp, ref, old, adv, tok, mode, agg, ops.KL_ESTIMATORS[est], faithful)
    cast = (lambda t: t) if faithful else (lambda t: t.float())
    x = cast(lp).clone().requires_grad_(True)
    mask = completion_mask(tok, EOS).bool()
    want = port.grpo_loss(mode, x, cast(ref), cast(old) if old is not None else None, adv, mask, 0.04, agg, EPS_HI,
                          *TAU, est)
    want.backward()
    want = want.detach()
    _close(grad if faithful else grad.float(), x.grad, faithful, 'grad')
    assert abs(float(loss) - float(want)) <= 1e-5 * max(1.0, abs(float(want))), (float(loss), float(want))


def _v_logits(B, Lq, V, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(B, Lq, V, device=DEV, generator=g) * 2).to(dtype)


@pytest.mark.parametrize('layout', ['dense', 'tail'])
@pytest.mark.parametrize('extras', ['plain', 'entropy+kl'])
@pytest.mark.parametrize('mode', MODES)
def test_k1f_actor_node_against_the_composed_path(ops, monkeypatch, mode, extras, layout):  # noqa: F811
    B, Lq, V, start = 4, 40, 152064, 8
    W = Lq - 1 - start
    logits = _v_logits(B, Lq, V, torch.bfloat16, 1)
    ids = torch.randint(0, V, (B, Lq), device=DEV)
    g = torch.Generator().manual_seed(3)
    old = (-torch.rand(B, W, generator=g) * 12).to(DEV)
    adv = torch.randn(B, W, generator=g).to(DEV)
    mask = (torch.rand(B, W, generator=g) < 0.8).to(DEV)
    mask[:, 0] = True
    obj = ops.ActorObjective(policy_loss_mode=mode, loss_agg_mode='token-mean' if extras != 'plain' else
                             'seq-mean-token-mean')
    kw = dict(objective=obj)
    if extras != 'plain':
        kw.update(entropy_coeff=0.01, ref_log_probs=old - 0.1, kl_loss_coeff=0.2, kl_loss_estimator='k3')
    lens = [W, W - 3, W, 5]

    def run(fused, objective=obj):
        monkeypatch.setattr(ops, '_FUSED_ACTOR', fused)
        x = logits.clone().requires_grad_(True)
        k = {**kw, 'objective': objective}
        if layout == 'dense':
            out = ops.dense_actor_loss(x, ids, start, old, adv, mask, 0.2, **k)
        else:
            out = ops.tail_actor_loss(x, ids, lens, old, adv, mask, 0.2, **k)
        out[0].backward()
        torch.cuda.synchronize()
        return out, x.grad

    (f_out, f_grad), (c_out, c_grad) = run(True), run(False)
    u = _ulps(f_grad, c_grad)
    assert int(u.max()) <= 2, int(u.max())
    assert torch.equal((f_grad == 0).all(-1), (c_grad == 0).all(-1))  # the same zero rows
    assert torch.equal(_bits(f_out[1]), _bits(c_out[1]))
    assert abs(float(f_out[0]) - float(c_out[0])) <= 1e-6 * max(1.0, abs(float(c_out[0])))
    v_out, _ = run(True, None if extras == 'plain' else ops.ActorObjective(loss_agg_mode='token-mean'))
    assert torch.equal(_bits(f_out[1]), _bits(v_out[1]))  # the log-probs are today's single pass's, bit for bit


@pytest.mark.parametrize('entropy_coeff', [0.0, 0.01])
@pytest.mark.parametrize('mode', MODES)
def test_k1f_grpo_node_against_the_composed_path(ops, monkeypatch, mode, entropy_coeff):  # noqa: F811
    B, Lq, V, K = 4, 48, 152064, 32
    logits = _v_logits(B, Lq, V, torch.bfloat16, 2)
    ids = torch.randint(3, 1000, (B, Lq), device=DEV)
    ids[1, -10] = EOS
    g = torch.Generator().manual_seed(4)
    adv = torch.randn(B, 1, generator=g).to(DEV)
    obj = ops.GrpoObjective(policy_loss_mode=mode)
    # the reference and old log-probs near the policy's: K1's and K1f's log-probs may differ by an ulp, which a KL
    # term far from 0 would magnify; log-ratios in {0, +-0.1, +-0.6} keep every ratio away from CISPO's bound
    lp0 = ops.tail_token_log_probs(logits, ids, K)
    ref = (lp0.float() + 0.05 * torch.randn(B, K, generator=g).to(DEV)).to(torch.bfloat16)
    shift = torch.tensor([0.0, 0.1, -0.1, 0.6, -0.6])[torch.randint(0, 5, (B, K), generator=g)].to(DEV)
    old = (lp0.float() - shift).to(torch.bfloat16)

    def run(fused, objective=obj):
        monkeypatch.setattr(ops, '_FUSED_GRPO', fused)
        x = logits.clone().requires_grad_(True)
        out = ops.grpo_loss_from_logits(x, ids, K, ref, adv, EOS, 0.04, entropy_coeff=entropy_coeff,
                                        objective=objective, old_per_token_logps=old, return_clip_fraction=True)
        out[0].backward()
        torch.cuda.synchronize()
        return out, x.grad

    (f_out, f_grad), (c_out, c_grad) = run(True), run(False)
    # K1f against K1b's softmax gradient at V = 152064: the project's tile tolerance, a 1e-4 share of elements up to 40
    # ulps where the rounded log-softmax sits at a 16-bit tie (test_gpu_parity.assert_ulp_close)
    assert_ulp_close(f_grad, c_grad, max_ulp=2, min_exact=0.97, what=f'{mode} grpo tile', tie_frac=1e-4, tie_ulp=40)
    assert torch.equal((f_grad == 0).all(-1), (c_grad == 0).all(-1))
    assert torch.equal(_bits(f_out[1]), _bits(c_out[1]))
    assert abs(float(f_out[0]) - float(c_out[0])) <= 1e-6 * max(1.0, abs(float(c_out[0])))
    assert torch.equal(f_out[-1], c_out[-1])
    v_out, _ = run(True, ops.GrpoObjective())
    assert torch.equal(_bits(f_out[1]), _bits(v_out[1]))


# ---- the trainers ------------------------------------------------------------------------------------------------
def _ppo_attrs(mode, f32):
    """Each mode with its options: CISPO at a clip-higher bound and token-mean, SAPO at other temperatures and the
    reference's seq-mean-token-mean; the clip fractions logged."""
    attrs = dict(policy_loss_mode=mode, log_clip_fraction=True, **({'mode': 'f32'} if f32 else {}))
    if mode == 'cispo':
        attrs.update(clip_range_ratio_high=EPS_HI, loss_agg_mode='token-mean')
    else:
        attrs.update(sapo_temperature_pos=0.5, sapo_temperature_neg=2.0)
    return attrs


def _ppo64(mode, lp64, old, adv, mask):
    """The float64 port with _ppo_attrs' options -> (loss, clip fraction)."""
    agg = 'token-mean' if mode == 'cispo' else 'seq-mean-token-mean'
    tau = (1.0, 1.05) if mode == 'cispo' else (0.5, 2.0)
    loss = port.actor_loss(mode, lp64, old.double(), adv.double(), mask, agg, EPS_HI, *tau)
    return loss, port.clip_fraction(mode, lp64.detach(), old.double(), adv.double(), mask, agg, EPS_HI)


def _run_image(cls, fused):
    from types import SimpleNamespace

    from test_gpu_fused_rl import LM, Critic, Phased

    from align_anything_b200.models.reward_model import ScoreModelOutput

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
    out = tr.rl_step(inference, training)
    return (training, out, tr.last_rl_tensors, h_new.grad, w_new.grad), (ids, resp, hid_new, w_a, Lq)


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('trainer', ['text', 'multi-rloo', 'image'])
def test_ppo_rl_step_against_float64_and_fused_lm_head(ops, trainer, mode):  # noqa: F811
    """One rl_step per trainer and mode in F32 mode against float64 autograd of the port through log_softmax (the
    loss, the clip fraction, d hidden and d weight), then the fused lm_head path (K6 -> aa_ppo_actor_loss_pm -> K6b)
    against the tile path in FAITHFUL mode.  The rollout and the trained policy have different hidden states, so the
    ratios spread far on both sides of 1 + EPS_HI."""
    from test_gpu_fused_rl import _ppo_batch, _run_ppo
    from test_gpu_ppo_objective import _param_grads, _with

    from align_anything_b200.trainers.text_image_to_text.ppo import PPOTrainer as Image
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer as Multi
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer as Text

    if trainer == 'image':
        run = lambda attrs, fused: _run_image(_with(Image, **attrs), fused)  # noqa: E731
    else:
        cls, kw = (Text, {}) if trainer == 'text' else (Multi, {'advantage_estimator': 'rloo', 'n_samples_per_prompt': 2})
        ids = _ppo_batch(5)
        P, H, V, seed = 12, 128, 2053, 43

        def run(attrs, fused):
            got = _run_ppo(_with(cls, **attrs), fused, ids, P, H, V, seed, **kw)
            gen = torch.Generator().manual_seed(seed)  # _run_ppo's draws: hid_a, hid_r, hid_new, w_a
            B, Lq = ids.shape
            for _ in range(2):
                torch.randn(B, Lq, H, generator=gen)
            h_new = torch.randn(B, Lq, H, generator=gen).bfloat16().to(DEV)
            w = (torch.randn(V, H, generator=gen) * 0.2).bfloat16().to(DEV)
            return got, (ids, P, h_new, w, Lq)

    on, (ids, lay, h_new, w, Lq) = run(_ppo_attrs(mode, True), False)
    assert 'train/actor_clip_fraction' in on[1] and 'train/actor_cov_fraction' not in on[1]
    x = torch.nn.functional.linear(h_new, w).double().requires_grad_(True)
    if trainer == 'image':
        resp = lay
        lp64 = torch.zeros(len(resp), max(resp), dtype=torch.float64, device=DEV)
        for b, r in enumerate(resp):
            lsm = torch.log_softmax(x[b, Lq - 1 - r:Lq - 1], -1)
            lp64[b, :r] = lsm.gather(-1, ids[b, Lq - r:, None]).squeeze(-1)
        old, mask = on[0]['log_probs'], on[0]['response_mask']
    else:
        start = lay - 1
        lp64 = torch.log_softmax(x[:, start:-1], -1).gather(-1, ids[:, start + 1:, None]).squeeze(-1)
        old, mask = on[0]['log_probs'][:, start:], (ids != 0)[:, 1:][:, start:]
    adv = on[2]['advantages']
    loss64, cf64 = _ppo64(mode, lp64, old, adv, mask)
    loss64.backward()
    r = torch.exp(lp64.detach() - old.double())[mask.bool()]
    assert bool((r > 1 + EPS_HI).any()) and bool((r < 1).any())  # both sides of CISPO's bound and of SAPO's centre
    assert abs(on[1]['train/actor_loss'] - float(loss64)) <= 1e-4 * max(1.0, abs(float(loss64)))
    assert abs(on[1]['train/actor_clip_fraction'] - cf64) <= 2.0 / float(mask.sum())
    if mode == 'cispo':
        assert cf64 > 0.0
    dh, dw = _param_grads(x.grad, h_new, w)
    _rel(on[3], dh, 2e-2, 'd hidden')
    _rel(on[4], dw, 2e-2, 'd weight')
    (tile, _), (fused, _) = run(_ppo_attrs(mode, False), False), run(_ppo_attrs(mode, False), True)
    assert set(fused[1]) == set(tile[1])
    for k, v in tile[1].items():
        assert abs(v - fused[1][k]) <= 1e-2 * max(1.0, abs(v)), (k, v, fused[1][k])
    _rel(fused[3], tile[3].double(), 2e-2, 'fused d hidden')
    _rel(fused[4], tile[4].double(), 2e-2, 'fused d weight')
    ops.check_status()


SHIFT = torch.tensor([0.0, 0.1, -0.1, 0.6, -0.6])  # log-ratios of update 2: 1.82 and 0.55 lie beyond both bounds


def _shift_old(monkeypatch, ops, olds):  # noqa: F811
    """Update 2's old log-probs moved by SHIFT (a fixed draw per token) before they reach either GRPO node, and every
    old the nodes see recorded; the composed node's inner grpo_loss call receives the tensor already moved."""
    moved = set()

    def wrap(real):
        def spy(*a, **kw):
            old = kw.get('old_per_token_logps')
            if old is not None and id(old) not in moved:
                g = torch.Generator().manual_seed(11)
                s = SHIFT[torch.randint(0, len(SHIFT), tuple(old.shape), generator=g)].to(old.device)
                old = (old.float() - s).to(old.dtype)
                moved.add(id(old))
                kw['old_per_token_logps'] = old
                olds.append(old)
            elif 'old_per_token_logps' in kw or old is None:
                if old is None and not any(o is None for o in olds):
                    olds.append(None)
            return real(*a, **kw)
        return spy

    monkeypatch.setattr(ops, 'grpo_loss_from_logits', wrap(ops.grpo_loss_from_logits))
    monkeypatch.setattr(ops, 'grpo_loss', wrap(ops.grpo_loss))


def _grpo_attrs(mode):
    attrs = dict(num_iterations=2, policy_loss_mode=mode, log_clip_fraction=True)
    if mode == 'cispo':
        attrs['clip_range_ratio_high'] = EPS_HI
    else:
        attrs.update(sapo_temperature_pos=0.5, sapo_temperature_neg=2.0)
    return attrs


@pytest.mark.parametrize('mode', MODES)
def test_grpo_two_updates_against_float64(ops, monkeypatch, mode):  # noqa: F811
    """A GRPOTrainer step with num_iterations = 2 in F32 mode: update 1 at ratio 1, update 2 with its old log-probs
    moved so that ratios cross 1 + EPS_HI on both sides; each update's loss, d hidden and d weight against float64
    autograd of the port on the parameters that update saw."""
    from test_gpu_fused_rl import _grpo_sequences
    from test_gpu_grpo_objective import EOS as EOS_T
    from test_gpu_top_entropy import _run

    seq = _grpo_sequences(7)
    P, H, V, seed = 16, 128, 2053, 47
    K = seq.size(1) - P
    olds = []
    _shift_old(monkeypatch, ops, olds)
    out, policy, (hid_r, w_r, rewards) = _run(False, seq, P, H, V, seed, 0.02, mode='f32', **_grpo_attrs(mode))
    assert len(policy.seen) == 2 and len(olds) == 2 and olds[0] is None and olds[1] is not None
    ref = ops.tail_token_log_probs(torch.nn.functional.linear(hid_r, w_r), seq, K, mode='f32').double()
    adv = ops.group_advantages(rewards, 2).double()
    mask = completion_mask(seq[:, -K:], EOS_T).bool()
    tau = (1.0, 1.05) if mode == 'cispo' else (0.5, 2.0)
    losses, fracs = [], []
    for u, ((h, w), (dh, dw)) in enumerate(zip(policy.seen, policy.grads)):
        logits = torch.nn.functional.linear(h, w)
        hh, ww = h.double().requires_grad_(True), w.double().requires_grad_(True)
        x = logits.double() + (torch.nn.functional.linear(hh, ww) - torch.nn.functional.linear(hh, ww).detach())
        lp64 = torch.log_softmax(x[:, :-1][:, -K:], -1).gather(-1, seq[:, -K:, None]).squeeze(-1)
        old = None if olds[u] is None else olds[u].double()
        if old is not None:
            r = torch.exp(lp64.detach() - old)[mask]
            assert bool((r > 1 + EPS_HI).any()) and bool((r < 1 - EPS_HI).any())
        loss64 = port.grpo_loss(mode, lp64, ref, old, adv, mask, 0.04, 'token-mean', EPS_HI, *tau)
        loss64.backward()
        losses.append(float(loss64))
        a = adv.reshape(-1, 1).expand(-1, K)
        fracs.append(port.clip_fraction(mode, lp64.detach(), lp64.detach() if old is None else old, a, mask,
                                        'token-mean', EPS_HI))
        _rel(dh, hh.grad, 2e-2, f'update {u + 1}: d hidden')
        _rel(dw, ww.grad, 2e-2, f'update {u + 1}: d weight')
    assert abs(out['train/loss'] - sum(losses) / 2) <= 1e-4 * max(1.0, abs(sum(losses) / 2))
    assert abs(out['train/actor_clip_fraction'] - sum(fracs) / 2) <= 2.0 / float(mask.sum())
    assert 'train/actor_cov_fraction' not in out
    if mode == 'cispo':
        assert fracs[1] > 0.0
    ops.check_status()


@pytest.mark.parametrize('mode', MODES)
def test_grpo_two_updates_fused_lm_head_vs_tile_path(ops, monkeypatch, mode):  # noqa: F811
    """The same GRPOTrainer step on the fused lm_head path (K6 -> aa_grpo_loss_pm -> K6b) and on the tile path, with
    update 2's old log-probs moved as above, FAITHFUL: the metrics and both updates' parameter gradients agree."""
    from test_gpu_fused_rl import _grpo_sequences
    from test_gpu_top_entropy import _run

    seq = _grpo_sequences(8)
    runs = []
    for fused in (False, True):
        olds = []
        with monkeypatch.context() as m:
            _shift_old(m, ops, olds)
            runs.append(_run(fused, seq, 16, 128, 2053, 49, 1e-4, **_grpo_attrs(mode)))
        assert len(olds) == 2 and olds[1] is not None
    (a, pa, _), (b, pb, _) = runs
    assert set(a) == set(b)
    for k, v in a.items():
        assert abs(v - b[k]) <= 1e-2 * max(1.0, abs(v)), (k, v, b[k])
    for u in range(2):
        _rel(pb.grads[u][0], pa.grads[u][0].double(), 2e-2, f'update {u + 1}: fused d hidden')
        _rel(pb.grads[u][1], pa.grads[u][1].double(), 2e-2, f'update {u + 1}: fused d weight')
    ops.check_status()
