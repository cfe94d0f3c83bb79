"""The cost-model loss on the H100 (`pytest -m gpu`): aa_cost_pair_loss (ops.cost_pair_loss) and the grafted trainers
against
  * STRICT: the reference's loss (tests/cost_model_port.py) executed with torch's CUDA kernels on the same device
    tensors -- fp32 within 1e-5 relative; 16-bit faithful mode: loss and gradient within 1 ulp and >= 97 % of the
    gradient elements bit-identical over the grid; 'f32' mode: within 2e-5 relative of the port on fp32-upcast scores;
    the loss dtype is the reference's in every mode;
  * GOLDEN: the fixtures the unmodified reference produced on CPU (tests/golden/make_golden_cost_model.py), loosely
    for 16-bit values (ATen's CPU divides by the count where its CUDA kernels multiply by the reciprocal)."""
from types import SimpleNamespace

import pytest
import torch

import cost_model_port as P
import fake_reference_tree as fake
from oracle import ref_port as O
from test_cpu_cost_model import RM_MODS, _rm_cm_tree
from test_gpu_parity import _ordered_bits, assert_close_f32, assert_loose, assert_ulp_close, ops  # noqa: F401

pytestmark = pytest.mark.gpu

DEV = 'cuda'
KINDS = ('int', 'float', 'bool', 'mixed', 'int_float')


def _signs(kind, B, gen):
    ints = [int(v) for v in torch.randint(-3, 4, (B,), generator=gen)]
    floats = [round(float(v), 3) for v in torch.rand(B, generator=gen) * 6 - 3]
    bools = [bool(v) for v in torch.randint(0, 2, (B,), generator=gen)]
    ints2 = [int(v) for v in torch.randint(-3, 4, (B,), generator=gen)]
    if kind == 'int':
        return ints, ints2
    if kind == 'float':
        return floats, list(reversed(floats))
    if kind == 'bool':
        return bools, [not v for v in bools]
    if kind == 'mixed':  # ints and floats in one list
        return ints[:-1] + [1.5], [-2] + floats[1:]
    return ints, floats


def _scores(B, dtype, gen):
    h, lo = torch.randn(B, generator=gen) * 3, torch.randn(B, generator=gen) * 3
    if B >= 3:
        lo[0] = h[0]  # tie
        h[1], lo[1] = 35.0, -2.0  # saturated logsigmoid
        h[2], lo[2] = -4.0, 31.5
    return torch.cat([h, lo]).unsqueeze(-1).to(dtype).to(DEV)


def _ulp_diff(got, want):
    return (_ordered_bits(got.detach().cpu()) - _ordered_bits(want.detach().cpu())).abs()


@pytest.mark.parametrize('B', [1, 3, 64, 1000])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
def test_kernel_matches_the_reference_on_cuda(ops, B, dtype):
    gen = torch.Generator().manual_seed(1000 + B)
    exact = total = 0
    for kind in KINDS:
        for scale, reg in ((1, 0.001), (0.5, 0.0)):
            end = _scores(B, dtype, gen)
            b, w = _signs(kind, B, gen)
            what = f'B={B} {dtype} {kind} scale={scale} reg={reg}'
            ref = end.clone().requires_grad_(True)
            want = P.cm_loss(ref, b, w, scale, reg)
            want['loss'].backward()
            mine = end.clone().requires_grad_(True)
            got = ops.cost_pair_loss(mine, b, w, scale, reg)
            got['loss'].backward()
            assert got['loss'].dtype == want['loss'].dtype, what
            assert float(got['accuracy']) == float(want['accuracy']), what
            assert float(got['_stats'][0]) == float(got['loss']), what
            if dtype == torch.float32:
                assert_close_f32(got['loss'], want['loss'], rtol=1e-5, what=what)
                assert_close_f32(mine.grad, ref.grad, rtol=1e-5, what=what)
            else:
                lg, lw = got['loss'].detach(), want['loss'].detach()
                if lw.dtype == torch.float32:  # a float sign list: fp32 sums of 16-bit-rounded terms
                    assert abs(float(lg) - float(lw)) <= torch.finfo(dtype).eps * max(1.0, abs(float(lw))), what
                else:
                    assert int(_ulp_diff(lg.view(1), lw.view(1)).max()) <= 1, what
                d = _ulp_diff(mine.grad, ref.grad)
                assert int(d.max()) <= 1, (what, int(d.max()))
                exact += int((d == 0).sum())
                total += d.numel()
            # f32 mode: fp32 throughout, against the reference on upcast scores; the loss keeps the reference's dtype
            up = end.float().clone().requires_grad_(True)
            want32 = P.cm_loss(up, b, w, scale, reg)
            want32['loss'].backward()
            mine32 = end.clone().requires_grad_(True)
            got32 = ops.cost_pair_loss(mine32, b, w, scale, reg, mode='f32')
            got32['loss'].backward()
            assert got32['loss'].dtype == want['loss'].dtype, what
            assert_close_f32(got32['_stats'][0], want32['loss'], rtol=2e-5, what=f'f32 mode {what}')
            assert torch.equal(got32['loss'], got32['_stats'][0].to(got32['loss'].dtype)), what
            assert mine32.grad.dtype == dtype
            if dtype == torch.float32:
                assert_close_f32(mine32.grad, up.grad, rtol=2e-5, what=f'f32 mode grad {what}')
            else:
                assert int(_ulp_diff(mine32.grad, up.grad.to(dtype)).max()) <= 1, what
    if total:
        assert exact / total >= 0.97, f'{dtype} B={B}: only {exact / total:.4f} of the gradient bit-identical'


def test_goldens(ops, golden):
    g = golden('cost_model')
    for key, c in g['cases'].items():
        leaf = c['end_scores'].to(DEV).requires_grad_(True)
        got = ops.cost_pair_loss(leaf, c['better'], c['worse'], c['scale_coeff'], c['regularization'])
        got['loss'].backward()
        assert got['loss'].dtype == c['loss_dtype'], key
        assert float(got['accuracy']) == float(c['accuracy']), key
        assert_loose(got['loss'].view(1), c['loss'].view(1), what=key)
        assert_loose(leaf.grad, c['grad'], what=key)
    for key, c in g['audio_rm'].items():
        if c['end_scores'].dtype != torch.float32:
            continue  # ops.rm_pair_loss upcasts 16-bit end scores (DESIGN.md section 4): the reference stays in bf16
        res = ops.rm_pair_loss(c['end_scores'].to(DEV), c['regularization'])
        assert_close_f32(res['loss'], c['loss'], rtol=1e-5, what=key)


class _Engine:
    optimizer = SimpleNamespace(param_groups=[{'lr': 2e-5}])

    def __init__(self, fn):
        self.fn = fn

    def __call__(self, **kw):
        return self.fn(kw)

    def backward(self, loss):
        loss.backward()

    def step(self):
        pass


@pytest.mark.parametrize('end_mode,upcast', [('mask', True), ('last', True), ('last', False)])
@pytest.mark.parametrize('reg', [0.0, 0.001])
def test_cm_trainer_through_the_score_head(ops, end_mode, upcast, reg):
    """Grafted CMTrainer.loss + backward through K3 down to the hidden states and the score-head weight, against the
    reference's ops on the GPU: Llama-style ('mask', upcast), LLaVA-style ('last') and Qwen2-VL-style (bf16 head)."""
    from align_anything_b200.models.reward_model import score_model_outputs
    from align_anything_b200.trainers.text_to_text.cost_model import CMTrainer

    gen = torch.Generator().manual_seed(53)
    B, Lq, H = 5, 23, 256
    h = torch.randn(2 * B, Lq, H, generator=gen).bfloat16().to(DEV)
    wt = (0.05 * torch.randn(1, H, generator=gen)).bfloat16().to(DEV)
    mask = torch.ones(2 * B, Lq, dtype=torch.bool, device=DEV)
    mask[0, :4] = False
    mask[3, 18:] = False
    meta = {'is_better_safe': [-1, 0, 2, -3, 1], 'is_worse_safe': [1.0, -0.5, 0, 2, -1]}
    hr, wr = h.clone().requires_grad_(True), wt.clone().requires_grad_(True)
    so = O.score_head(hr, wr, mask, end_mode, upcast)
    want = P.cm_loss(so['end_scores'], meta['is_better_safe'], meta['is_worse_safe'], 1, reg)
    want['loss'].backward()

    hg, wg = h.clone().requires_grad_(True), wt.clone().requires_grad_(True)
    tr = CMTrainer(SimpleNamespace(train_cfgs=SimpleNamespace(scale_coeff=1, regularization=reg)),
                   _Engine(lambda kw: score_model_outputs(hg, wg, kw['attention_mask'], end_mode, upcast)))
    batch = {'input_ids': torch.zeros(2 * B, Lq, dtype=torch.int64, device=DEV), 'attention_mask': mask,
             'meta_info': meta}
    got = tr.loss(batch)
    assert got['loss'].dtype == want['loss'].dtype
    assert_close_f32(got['loss'], want['loss'], rtol=1e-5, what='cm loss')
    assert float(got['accuracy']) == float(want['accuracy'])
    assert torch.equal(got['higher_end_reward'], want['higher_end_reward'].detach())
    got['loss'].backward()
    assert_ulp_close(hg.grad, hr.grad, max_ulp=1, min_exact=0.97, what='cm dh')
    assert_ulp_close(wg.grad, wr.grad, max_ulp=1, min_exact=0.8, what='cm dw')
    m = tr.train_step(batch)
    assert set(m) == {'train/loss', 'train/accuracy', 'train/lr'} and m['train/lr'] == 2e-5
    assert abs(m['train/loss'] - float(want['loss'])) <= 1e-5 * max(1.0, abs(float(want['loss'])))
    assert m['train/accuracy'] == float(want['accuracy'])


def test_grafted_audio_rm_matches_the_text_mirror(ops):
    from align_anything_b200 import patch
    from align_anything_b200.models.reward_model import score_model_outputs
    from align_anything_b200.trainers.text_to_text.rm import RMTrainer

    gen = torch.Generator().manual_seed(61)
    h = torch.randn(8, 17, 128, generator=gen).bfloat16().to(DEV)
    wt = (0.05 * torch.randn(1, 128, generator=gen)).bfloat16().to(DEV)
    mask = torch.ones(8, 17, dtype=torch.bool, device=DEV)
    mask[2, 11:] = False
    cfgs = SimpleNamespace(train_cfgs=SimpleNamespace(regularization=0.001))
    batch = {'input_ids': torch.zeros(8, 17, dtype=torch.int64, device=DEV), 'attention_mask': mask}
    runs = []
    with fake.installed(), _rm_cm_tree() as mods:
        patch.install()
        try:
            for cls in (mods[RM_MODS['audio']].RMTrainer, RMTrainer):
                hg, wg = h.clone().requires_grad_(True), wt.clone().requires_grad_(True)
                t = object.__new__(cls)
                RMTrainer.__init__(t, cfgs, _Engine(lambda kw: score_model_outputs(hg, wg, kw['attention_mask'])))
                res = t.loss(batch)
                res['loss'].backward()
                runs.append((res['loss'].detach(), float(res['accuracy']), hg.grad, wg.grad, t.train_step(batch)))
        finally:
            patch.uninstall()
    (la, aa, ha, wa, sa), (lt, at, ht, wt_, st) = runs
    assert torch.equal(la, lt) and aa == at and torch.equal(ha, ht) and torch.equal(wa, wt_)
    assert set(sa) == {'train/loss', 'train/accuracy', 'train/lr'} and sa == st
