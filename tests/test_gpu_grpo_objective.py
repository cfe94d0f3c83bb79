"""GRPO objective options on the H100 (DESIGN §4.4): aa_grpo_loss_obj through the C ABI against the port
(tests/grpo_objective_port.py) on guarded buffers, its default fields against aa_grpo_loss, the clip fractions, the
centred advantages, K1f's GRPO node against the composed path with the same objective, and the trainer's update loop
against float64 autograd of the port."""
from __future__ import annotations

from types import SimpleNamespace

import pytest
import torch

from grpo_objective_port import clip_fractions, completion_mask
from grpo_objective_port import grpo_loss as port_loss
from test_gpu_entropy import _bits
from test_gpu_parity import assert_ulp_close, ops  # noqa: F401  (fixture)
from test_gpu_ppo_objective import Guarded, _rel

pytestmark = pytest.mark.gpu

DEV = 'cuda'
AGG = {'seq-mean-token-mean': 0, 'token-mean': 1, 'seq-mean-token-sum-norm': 2}
# (clip_low, clip_high, dual_clip, loss_agg_mode): each option alone, then all together
OPTIONS = {
    'clip': (0.2, 0.2, None, 'token-mean'),
    'clip-higher': (0.2, 0.28, None, 'token-mean'),
    'dual-clip': (0.2, 0.2, 3.0, 'token-mean'),
    'seq-mean': (0.2, 0.2, None, 'seq-mean-token-mean'),
    'sum-norm': (0.2, 0.2, None, 'seq-mean-token-sum-norm'),
    'all': (0.2, 0.28, 3.0, 'seq-mean-token-mean'),
}
EOS = 1


def _objective(opt):
    from align_anything_b200.ops import GrpoObjective

    lo, hi, c, agg = opt
    return GrpoObjective(lo, hi, c, agg)


def _inputs(B, K, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, K, generator=g) * 4
    ref = lp + torch.randn(B, K, generator=g) * 0.3
    old = lp + torch.randn(B, K, generator=g) * 0.5  # ratios inside and far outside the clip ranges
    adv = torch.randn(B, 1, generator=g)
    adv = torch.where(adv.abs() < 0.25, adv.sign() * 0.25 + 0.25 * (adv == 0), adv)  # no 16-bit subnormal products
    tokens = torch.randint(2, 50, (B, K), generator=g)
    tokens[0, 5] = EOS
    tokens[2, 0] = EOS
    tokens[3, K - 1] = EOS
    return (lp.to(dtype).to(DEV), ref.to(dtype).to(DEV), old.to(dtype).to(DEV), adv.to(DEV), tokens.to(DEV))


def _loss_c_abi(lp, ref, old, adv, tokens, beta, obj, mode, legacy=False):
    """aa_grpo_loss_obj (or aa_grpo_loss) through the C ABI on guarded buffers -> (loss, grad, clip fractions, row_end)."""
    from align_anything_b200 import _lib as L

    B, K = lp.shape
    mode_code = L.MODE_FAITHFUL if mode == 'faithful' else L.MODE_F32
    gl, gr = Guarded(lp), Guarded(ref)
    gt = SimpleNamespace(view=tokens.contiguous())  # int64: read only
    go = Guarded(old) if old is not None else None
    ga = Guarded(adv.view(1, B).contiguous())
    grad = Guarded(torch.zeros_like(lp))
    loss = Guarded(torch.zeros(1, 1, dtype=torch.float32, device=DEV))
    cf = Guarded(torch.zeros(1, 2, dtype=torch.float32, device=DEV))
    row_end = Guarded(torch.zeros(1, B, dtype=torch.int32, device=DEV), fill=-7)
    scratch = torch.full((1 + 4 * B,), float('nan'), dtype=torch.float32, device=DEV)
    counter = torch.zeros(2, dtype=torch.int32, device=DEV)
    lib = L.lib()
    if legacy:
        L.check(lib.aa_grpo_loss(gl.view.data_ptr(), gl.view.stride(0), gr.view.data_ptr(), gr.view.stride(0),
                                 L.dtype_code(lp.dtype), ga.view.data_ptr(), gt.view.data_ptr(), gt.view.stride(0), EOS,
                                 B, K, float(beta), mode_code, loss.view.data_ptr(), grad.view.data_ptr(),
                                 grad.view.stride(0), row_end.view.data_ptr(), scratch.data_ptr(), counter.data_ptr(),
                                 L.stream_ptr(DEV)))
    else:
        lo, hi, c, agg = obj
        L.check(lib.aa_grpo_loss_obj(gl.view.data_ptr(), gl.view.stride(0), gr.view.data_ptr(), gr.view.stride(0),
                                     go.view.data_ptr() if go else None, go.view.stride(0) if go else 0,
                                     L.dtype_code(lp.dtype), ga.view.data_ptr(), gt.view.data_ptr(), gt.view.stride(0),
                                     EOS, B, K, float(beta), float(lo), float(hi), float(c or 0.0), AGG[agg], mode_code,
                                     loss.view.data_ptr(), grad.view.data_ptr(), grad.view.stride(0), cf.view.data_ptr(),
                                     row_end.view.data_ptr(), scratch.data_ptr(), counter.data_ptr(), L.stream_ptr(DEV)))
    torch.cuda.synchronize()
    for g in (gl, gr, ga, grad, loss, cf, row_end) + ((go,) if go else ()):
        assert g.intact(), 'a guard band was written'
    return loss.view[0, 0].clone(), grad.view.clone(), cf.view[0].clone(), row_end.view[0].clone()


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize('mode', ['faithful', 'f32'])
@pytest.mark.parametrize('name', list(OPTIONS))
def test_grpo_loss_obj_c_abi_vs_port(ops, dtype, mode, name):
    lo, hi, c, agg = opt = OPTIONS[name]
    B, K = 7, 301
    lp, ref, old, adv, tokens = _inputs(B, K, dtype, seed=list(OPTIONS).index(name))
    loss, grad, cf, row_end = _loss_c_abi(lp, ref, old, adv, tokens, 0.04, opt, mode)
    mask = completion_mask(tokens, EOS)
    assert torch.equal(row_end.long(), mask.sum(-1))
    faithful = mode == 'faithful' and dtype != torch.float32
    cd = dtype if faithful else torch.float32  # the port on ATen CUDA in the dtype the kernel rounds to
    x = lp.to(cd).clone().requires_grad_(True)
    want = port_loss(x, ref.to(cd), adv, mask, 0.04, old.to(cd), lo, hi, c, agg)
    want.backward()
    assert want.dtype == torch.float32
    torch.testing.assert_close(loss, want.detach(), rtol=2e-5, atol=1e-7)
    if faithful:
        assert_ulp_close(grad, x.grad, max_ulp=1, min_exact=0.97, what=f'{name} grad')
    elif dtype == torch.float32:
        torch.testing.assert_close(grad, x.grad, rtol=2e-5, atol=2e-5 * float(x.grad.abs().max()))
    else:  # F32 mode keeps fp32 throughout and rounds the gradient once, to the log-probs' dtype
        assert_ulp_close(grad, x.grad.to(dtype), max_ulp=1, min_exact=0.97, what=f'{name} grad')
    # the port's counts on its own ratios: one token may sit on a clip bound and change sides
    fc, fd = clip_fractions(lp.to(cd), old.to(cd), adv, mask, lo, hi, c, agg)
    n = float(mask.sum()) if agg != 'seq-mean-token-mean' else float(mask.sum(-1).min())
    assert abs(float(cf[0]) - fc) <= 1.0 / n + 1e-6, (float(cf[0]), fc)
    n_neg = float(((adv < 0) & mask.bool()).sum())
    assert abs(float(cf[1]) - fd) <= 1.0 / max(n_neg, 1.0) + 1e-6, (float(cf[1]), fd)
    if c is None:
        assert float(cf[1]) == 0.0


@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize('mode', ['faithful', 'f32'])
def test_grpo_loss_obj_first_update_and_default_fields(ops, dtype, mode):
    lp, ref, _, adv, tokens = _inputs(5, 129, dtype, seed=7)
    # default fields with the log-probs as their own old log-probs: the bits of aa_grpo_loss
    a = _loss_c_abi(lp, ref, None, adv, tokens, 0.04, (0.2, 0.2, None, 'token-mean'), mode)
    b = _loss_c_abi(lp, ref, None, adv, tokens, 0.04, None, mode, legacy=True)
    assert torch.equal(_bits(a[0]), _bits(b[0])) and torch.equal(_bits(a[1]), _bits(b[1]))
    assert torch.equal(a[3], b[3]) and torch.equal(a[2], torch.zeros_like(a[2]))  # ratio 1: nothing clipped
    # ... and through ops: default fields and no old log-probs run today's launch
    x = lp.clone().requires_grad_(True)
    want, _ = ops.grpo_loss(x, ref, adv, tokens, EOS, 0.04, mode=mode)
    want.backward()
    y = lp.clone().requires_grad_(True)
    from align_anything_b200.ops import GrpoObjective

    got, _ = ops.grpo_loss(y, ref, adv, tokens, EOS, 0.04, mode=mode, objective=GrpoObjective())
    got.backward()
    assert torch.equal(_bits(got.detach()), _bits(want.detach())) and torch.equal(_bits(y.grad), _bits(x.grad))


def test_centred_advantages_vs_float64(ops):
    g = torch.Generator().manual_seed(3)
    r = (torch.randn(40 * 6, generator=g) * 3 + 1).to(DEV)
    got = ops.group_advantages(r, 6, scale=False)
    r64 = r.double().view(40, 6)
    want = (r64 - r64.mean(1, keepdim=True)).view(-1, 1)
    assert float((got.double() - want).abs().max()) <= 4e-6 * float(r64.abs().max())
    torch.testing.assert_close(ops.group_advantages(r, 6), ops.group_advantages(r, 6, scale=True), rtol=0, atol=0)


# ---- K1f's GRPO node against the composed path with the same objective ---------------------------------------------
def _grpo_node(ops, logits, ids, K, ref, adv, mode, **kw):
    leaf = logits.clone().requires_grad_(True)
    out = ops.grpo_loss_from_logits(leaf, ids, K, ref, adv, EOS, 0.04, mode=mode, **kw)
    out[0].backward()
    return out, leaf.grad


@pytest.mark.parametrize('dtype,mode', [(torch.bfloat16, 'faithful'), (torch.bfloat16, 'f32'), (torch.float32, 'f32')])
def test_k1f_grpo_objective_vs_composed_path(ops, monkeypatch, dtype, mode):
    V, B, Lq, K = 152064, 4, 14, 9
    torch.manual_seed(17)
    logits = (torch.randn(B, Lq, V, device=DEV) * 2.0).to(dtype)
    ids = torch.randint(2, V, (B, Lq), device=DEV)
    ids[1, Lq - K + 4] = EOS  # a completion that ends early
    ids[2, Lq - K] = EOS  # ... and one that ends at its first token
    adv = torch.tensor([[1.5], [-0.7], [0.4], [-2.0]], device=DEV)
    ref = ops.tail_token_log_probs(logits, ids, K, mode=mode).float()
    base, gbase = _grpo_node(ops, logits, ids, K, ref, adv, mode)
    # old log-probs at designed distances from the new ones: log-ratios in {0, ±0.1, ±0.6} put every ratio well inside
    # or well outside the clip ranges, so the two paths' log-probs (a few ulp apart) clip the same tokens
    shift = torch.tensor([0.0, 0.1, -0.1, 0.6, -0.6], device=DEV)[torch.randint(0, 5, (B, K), device=DEV)]
    old = (base[1].float() - shift).to(base[1].dtype)
    for name, opt in OPTIONS.items():
        obj = _objective(opt)
        for coeff in ((0.0, 0.05) if name in ('all', 'sum-norm') else (0.0,)):
            kw = dict(objective=obj, old_per_token_logps=old, return_clip_fraction=True,
                      **({'entropy_coeff': coeff} if coeff else {}))
            one, gone = _grpo_node(ops, logits, ids, K, ref, adv, mode, **kw)
            assert torch.equal(_bits(one[1]), _bits(base[1])), f'{name}: log-probs differ from the default single pass'
            assert torch.equal(one[2], base[2])
            monkeypatch.setattr(ops, '_FUSED_GRPO', False)
            two, gtwo = _grpo_node(ops, logits, ids, K, ref, adv, mode, **kw)
            monkeypatch.setattr(ops, '_FUSED_GRPO', True)
            what = f'{name} coeff={coeff}'
            if dtype == torch.float32 or mode == 'f32':
                scale = float(gtwo.float().abs().max())
                assert float((gone.float() - gtwo.float()).abs().max()) <= 1e-5 * scale + 1e-12, what
            else:
                assert_ulp_close(gone, gtwo, max_ulp=2, min_exact=0.97, what=what)
            zero_rows = lambda g: (g.reshape(-1, V) == 0).all(-1)  # noqa: E731
            assert torch.equal(zero_rows(gone), zero_rows(gtwo)), what
            assert float(one[0].detach()) == pytest.approx(float(two[0].detach()), rel=1e-5, abs=1e-7), what
            assert torch.allclose(one[-1], two[-1], atol=1e-6), what  # clip fractions
            if coeff:
                assert float(one[3]) == pytest.approx(float(two[3]), rel=1e-5), what  # the entropy term
                assert float(one[4]) == pytest.approx(float(two[4]), rel=1e-5, abs=1e-7), what  # the loss without it
    # the first update (no old log-probs): the log-probs themselves, every ratio 1, nothing clipped
    first, gfirst = _grpo_node(ops, logits, ids, K, ref, adv, mode, objective=_objective(OPTIONS['all']),
                               return_clip_fraction=True)
    assert torch.equal(_bits(first[1]), _bits(base[1])) and float(first[-1].abs().sum()) == 0.0
    ops.check_status()


# ---- the trainer's update loop --------------------------------------------------------------------------------------
class SGD:
    """A causal LM reduced to its last hidden states and lm_head whose engine takes plain SGD steps; records the
    parameters each forward saw and the gradients each step took."""

    def __init__(self, hidden, weight, lr):
        self.h, self.w, self.lr = hidden.clone().requires_grad_(True), weight.clone().requires_grad_(True), lr
        self.seen, self.grads = [], []

    def __call__(self, output_hidden_states=False, logits_to_keep=0, **kw):
        self.seen.append((self.h.detach().clone(), self.w.detach().clone()))
        if output_hidden_states:
            return SimpleNamespace(hidden_states=(None, self.h), logits=None)
        return SimpleNamespace(logits=torch.nn.functional.linear(self.h, self.w))

    def get_output_embeddings(self):
        return SimpleNamespace(weight=self.w)

    def zero_grad(self):
        self.h.grad = self.w.grad = None

    def backward(self, loss):
        loss.backward()

    def step(self):
        self.grads.append((self.h.grad.clone(), self.w.grad.clone()))
        with torch.no_grad():
            self.h -= self.lr * self.h.grad
            self.w -= self.lr * self.w.grad


ALL_ON = dict(num_iterations=2, clip_range_ratio_low=0.2, clip_range_ratio_high=0.28, dual_clip_ratio=3.0,
              loss_agg_mode='seq-mean-token-sum-norm', scale_rewards=False, log_clip_fraction=True)


def _run(fused, seq, P, H, V, seed, lr, **attrs):
    from test_gpu_fused_rl import LM

    from align_anything_b200.trainers.text_to_text.grpo import GRPOTrainer

    gen = torch.Generator().manual_seed(seed)
    B, Lq = seq.shape
    hid = torch.randn(B, Lq, H, generator=gen).bfloat16().to(DEV)
    hid_r = torch.randn(B, Lq, H, generator=gen).bfloat16().to(DEV)
    w = (torch.randn(V, H, generator=gen) * 0.2).bfloat16().to(DEV)
    w_r = (w.float().cpu() + torch.randn(V, H, generator=gen) * 0.02).bfloat16().to(DEV)
    rewards = torch.randn(B, generator=gen).to(DEV)
    policy = SGD(hid, w, lr)
    tr = type('GRPO', (GRPOTrainer,), attrs)(None, policy, LM(hid_r, w_r),
                                            SimpleNamespace(pad_token_id=0, eos_token_id=EOS), beta=0.04,
                                            num_generations=2)
    tr.fused_lm_head, tr.lm_head_chunk_rows = fused, 32
    out = tr.step_from_rollout(seq, P, rewards)
    return out, policy, (hid_r, w_r, rewards)


def test_grpo_two_updates_with_every_option_vs_float64(ops, monkeypatch):
    from test_gpu_fused_rl import _grpo_sequences

    seq = _grpo_sequences(7)
    P, H, V, seed = 16, 128, 2053, 47
    K = seq.size(1) - P
    olds = []
    real = ops.grpo_loss_from_logits

    def spy(*a, **kw):
        olds.append(kw.get('old_per_token_logps'))
        return real(*a, **kw)

    monkeypatch.setattr(ops, 'grpo_loss_from_logits', spy)
    out, policy, (hid_r, w_r, rewards) = _run(False, seq, P, H, V, seed, 0.3, mode='f32', **ALL_ON)
    assert set(out) == {'train/loss', 'train/reward', 'train/actor_clip_fraction', 'train/actor_dual_clip_fraction'}
    assert len(policy.seen) == len(policy.grads) == 2 and olds[0] is None and olds[1] is not None
    ref = ops.tail_token_log_probs(torch.nn.functional.linear(hid_r, w_r), seq, K, mode='f32').double()
    adv = ops.group_advantages(rewards, 2, scale=False).double()
    mask = completion_mask(seq[:, -K:], EOS)
    losses = []
    for u, ((h, w), (dh, dw)) in enumerate(zip(policy.seen, policy.grads)):
        hh, ww = h.double().requires_grad_(True), w.double().requires_grad_(True)
        x = torch.nn.functional.linear(h, w).double()  # the bf16 logits the trainer's model returns
        x = x + (torch.nn.functional.linear(hh, ww) - torch.nn.functional.linear(hh, ww).detach())
        lp64 = torch.log_softmax(x[:, :-1][:, -K:], -1).gather(-1, seq[:, -K:, None]).squeeze(-1)
        old = None if olds[u] is None else olds[u].double()
        loss64 = port_loss(lp64, ref, adv, mask, 0.04, old, 0.2, 0.28, 3.0, 'seq-mean-token-sum-norm', clipped=True)
        loss64.backward()
        losses.append(float(loss64))
        _rel(dh, hh.grad, 2e-2, f'update {u + 1}: d hidden')
        _rel(dw, ww.grad, 2e-2, f'update {u + 1}: d weight')
    assert abs(out['train/loss'] - sum(losses) / 2) <= 1e-4 * max(1.0, abs(sum(losses) / 2))
    h2, w2 = policy.seen[1]
    lp2 = ops.tail_token_log_probs(torch.nn.functional.linear(h2, w2), seq, K, mode='f32').double()
    fc, fd = clip_fractions(lp2, olds[1].double(), adv, mask, 0.2, 0.28, 3.0, 'seq-mean-token-sum-norm')
    n = float(mask.sum())
    assert abs(out['train/actor_clip_fraction'] - fc / 2) <= 2.0 / n, (out, fc)  # the first update clips nothing
    ops.check_status()


def test_grpo_two_updates_fused_lm_head_vs_tile_path(ops):
    from test_gpu_fused_rl import _grpo_sequences

    seq = _grpo_sequences(8)
    a, pa, _ = _run(False, seq, 16, 128, 2053, 49, 1e-4, **ALL_ON)
    b, pb, _ = _run(True, seq, 16, 128, 2053, 49, 1e-4, **ALL_ON)
    assert set(a) == set(b)
    for k, v in a.items():
        assert abs(v - b[k]) <= 1e-2 * max(1.0, abs(v)), (k, v, b[k])
    for u in range(2):
        _rel(pb.grads[u][0], pa.grads[u][0].double(), 2e-2, f'update {u + 1}: fused d hidden')
        _rel(pb.grads[u][1], pa.grads[u][1].double(), 2e-2, f'update {u + 1}: fused d weight')
    ops.check_status()


def test_single_update_with_default_switches_is_the_plain_trainer(ops):
    from test_gpu_fused_rl import _grpo_sequences

    seq = _grpo_sequences(7)
    for fused in (False, True):
        plain, p0, _ = _run(fused, seq, 16, 128, 2053, 47, 1.0)
        dflt, p1, _ = _run(fused, seq, 16, 128, 2053, 47, 1.0, num_iterations=1, clip_range_ratio=0.2,
                           loss_agg_mode='token-mean', scale_rewards=True, log_clip_fraction=False)
        assert dflt == plain
        for (a, b), (c, d) in zip(p0.grads, p1.grads):
            assert torch.equal(_bits(a), _bits(c)) and torch.equal(_bits(b), _bits(d))
    ops.check_status()
