"""Clip-Cov and KL-Cov pinned at the trainers' rounding and at rollout scale (run on an H100: `pytest -m gpu`).

1. The six selection entry points (aa_cov_moments .. aa_cov_mark) through the C ABI on guard-banded buffers, bit for bit
   against a stable-sort top-k on the CPU fed the kernel's own fp32 means: the mask, the state words (E, k, T, need)
   and the share, at shapes that take every grid-stride and row-scan path, in both layouts and all three dtypes, at
   the key and count edges, and with Clip-Cov's eligibility in the `faithful` 16-bit rounding.
2. aa_ppo_actor_loss_cov and aa_grpo_loss_cov on guard-banded buffers with a hand-made selection, against
   tests/cov_port.py on ATen CUDA in the kernel's dtype, at realistic operands and at the counts a 16-bit dtype cannot
   hold; and the last-block counter K5's entry points share, re-armed after every call.
3. The composed nodes (dense, tail, GRPO) in `faithful` bf16 with every option on, against float64 autograd.
"""
from __future__ import annotations

import ctypes
from types import SimpleNamespace

import pytest
import torch

import cov_port as port
from grpo_objective_port import clip_fractions as grpo_clip_fractions
from grpo_objective_port import completion_mask
from kl_loss_port import kl_loss
from ppo_objective_port import actor_loss as obj_loss
from ppo_objective_port import clip_fractions
from test_cpu_faithful_counts import BF, CASE_IDS, CASES, F16, exact_actor_case, k5_actor, mean_rounds_alike
from test_cpu_cov_pin import TOKEN_MEAN_CASES, TOKEN_MEAN_IDS, token_mean_case
from test_gpu_faithful_counts import _identical, _loss16
from test_gpu_entropy import _bits
from test_gpu_loss_kernels import Words, fenced
from test_gpu_parity import assert_ulp_close, ops  # noqa: F401  (fixture)
from test_gpu_ppo_objective import Guarded, _rel

pytestmark = pytest.mark.gpu
DEV = 'cuda'
F32 = torch.float32
DTYPES = [F32, BF, F16]
MODES = ['clip_cov', 'kl_cov']
COV = {'clip_cov': 1, 'kl_cov': 2}  # include/aa_b200.h AA_COV_*
AGG = {'seq-mean-token-mean': 0, 'token-mean': 1, 'seq-mean-token-sum-norm': 2}
EST = {'k1': 0, 'k2': 1, 'k3': 2}
S32, S8 = 0x3C5A5A5A, 0x5A  # guard sentinels of the int32 and byte buffers
NAN = float('nan')


def _lib():
    from align_anything_b200 import _lib as L

    return L


def _mode_code(mode):
    L = _lib()
    return L.MODE_FAITHFUL if mode == 'faithful' else L.MODE_F32


def _vec(t, fill):
    """A 1-D tensor as the interior of a guarded (1, n) buffer."""
    return Guarded(t.reshape(1, -1), fill=fill)


# ---- 1. the selection through the C ABI -------------------------------------------------------------------------------
def _select(lp, adv, mask, row_end, cov_mode, ratio, mode, old, lo, hi, lb, ub, seed):
    """The six entry points on guarded buffers -> (sel (B, W) uint8, state int64 (16,), share fp32 0-dim)."""
    L = _lib()
    lib, st = L.lib(), L.stream_ptr(torch.device(DEV))
    B, W = lp.shape
    gl = Guarded(lp)
    go = Guarded(old) if old is not None else None
    if mask is not None:
        ga, gm, gr = Guarded(adv), Guarded(mask.to(torch.uint8), fill=1), None
        rows_adv = (ga.view.data_ptr(), ga.view.stride(0), L.dtype_code(adv.dtype), gm.view.data_ptr(),
                    gm.view.stride(0), None)
    else:
        ga, gm, gr = _vec(adv.float(), NAN), None, _vec(row_end.to(torch.int32), -7)
        rows_adv = (ga.view.data_ptr(), 0, L.AA_F32, None, 0, gr.view.data_ptr())
    state = _vec(torch.full((16,), S32, dtype=torch.int32, device=DEV), S32)
    keys = _vec(torch.full((B * W,), S32, dtype=torch.int32, device=DEV), S32)
    elig = _vec(torch.full((B * W,), S8, dtype=torch.uint8, device=DEV), S8)
    hist = _vec(torch.full((1 << 16,), S32, dtype=torch.int32, device=DEV), S32)
    ties = _vec(torch.full((B,), S32, dtype=torch.int32, device=DEV), S32)
    share = _vec(torch.full((1,), NAN, device=DEV), NAN)
    sel = Guarded(torch.full((B, W), S8, dtype=torch.uint8, device=DEV), fill=S8)  # row stride W + 32
    sp = state.view.data_ptr()
    rows = (gl.view.data_ptr(), gl.view.stride(0), L.dtype_code(lp.dtype), rows_adv[0], rows_adv[1], rows_adv[2],
            rows_adv[3], rows_adv[4], rows_adv[5], B, W)
    guarded = (('lp', gl), ('old', go), ('adv', ga), ('mask', gm), ('row_end', gr), ('state', state), ('keys', keys),
               ('elig', elig), ('hist', hist), ('ties', ties), ('share', share), ('sel', sel))

    def call(who, rc):  # every guard band intact after each entry point, not only after the last
        L.check(rc)
        torch.cuda.synchronize()
        for name, g in guarded:
            assert g is None or g.intact(), f'{who} wrote a guard band of {name}'

    call('aa_cov_moments', lib.aa_cov_moments(*rows, sp, st))
    call('aa_cov_keys', lib.aa_cov_keys(COV[cov_mode], rows[0], rows[1], go.view.data_ptr() if go else None,
                                        go.view.stride(0) if go else 0, *rows[2:], lo, hi, lb, ub, seed & 0xffffffff,
                                        _mode_code(mode), sp, keys.view.data_ptr(), elig.view.data_ptr(),
                                        hist.view.data_ptr(), st))
    call('aa_cov_select_hi', lib.aa_cov_select_hi(hist.view.data_ptr(), ctypes.byref(ctypes.c_double(ratio)), sp, st))
    call('aa_cov_hist_lo', lib.aa_cov_hist_lo(keys.view.data_ptr(), elig.view.data_ptr(), B * W, sp,
                                              hist.view.data_ptr(), st))
    call('aa_cov_select_lo', lib.aa_cov_select_lo(hist.view.data_ptr(), sp, share.view.data_ptr(), st))
    call('aa_cov_mark', lib.aa_cov_mark(keys.view.data_ptr(), elig.view.data_ptr(), B, W, sp, ties.view.data_ptr(),
                                        sel.view.data_ptr(), sel.view.stride(0), st))
    return sel.view.clone(), state.view[0].clone().cpu(), share.view[0, 0].clone()


def _ulps(a, b):
    if torch.isnan(a) and torch.isnan(b):
        return 0
    return abs(int(a.view(torch.int32)) - int(b.view(torch.int32)))


def _check_selection(lp, adv, counted, cov_mode, ratio, mode='faithful', old=None, row_end=None, lo=0.2, hi=0.28,
                     lb=1.0, ub=5.0, seed=0, poison=True):
    """Runs the selection twice and holds it to the reference.  counted (B, W) bool; with row_end the advantages are
    fp32 (B,) and counted must be t < row_end.  poison: uncounted log-probs, old log-probs and advantages are NaN.
    Clip-Cov: tokens whose clip decision one fp32 ulp of exp could flip get old = lp first (cov_port.clear_clip_band
    in the rounding the kernel uses), so that no case depends on ATen's exp agreeing with the kernel's expf there.
    -> (sel, state) of the first run."""
    B, W = lp.shape
    if poison:
        lp = torch.where(counted, lp, torch.full_like(lp, NAN))
        old = torch.where(counted, old, torch.full_like(old, NAN)) if old is not None else None
        if row_end is None:
            adv = torch.where(counted, adv, torch.full_like(adv, NAN))
    if cov_mode == 'clip_cov' and old is not None:
        faithful = mode == 'faithful'
        a = adv if row_end is None else adv.float().view(-1, 1).expand(B, W)
        cd, ad = (lp.dtype, a.dtype) if faithful else (F32, F32)
        old = port.clear_clip_band(lp.to(cd), old.to(cd), a.to(ad), lo, hi).to(lp.dtype)
    mask = counted if row_end is None else None
    args = (lp, adv, mask, row_end, cov_mode, ratio, mode, old, lo, hi, lb, ub, seed)
    sel, raw, share = _select(*args)
    state = raw.long() & 0xffffffff
    n = int(counted.sum())
    assert int(state[0]) == n, ('N', int(state[0]), n)
    ma, ml = raw[7:9].view(torch.float32)
    a_full = adv if row_end is None else adv.float().view(-1, 1).expand(B, W)
    if n:
        wa, wl = port.means(lp.cpu(), a_full.cpu(), counted.cpu())
        assert _ulps(ma, wa) <= 1 and _ulps(ml, wl) <= 1, ('means', float(ma), float(wa), float(ml), float(wl))
    cov = port.covariance(lp, a_full, ma.to(DEV), ml.to(DEV))
    if cov_mode == 'kl_cov':
        keys, eligible = port.order_key(cov), counted
    else:
        faithful = mode == 'faithful'
        cd = lp.dtype if faithful else F32
        ad = (a_full.dtype if faithful else F32) if row_end is None else F32
        o = (old if old is not None else lp).to(cd)
        clipped = port.clipped(lp.to(cd), o, a_full.to(ad), lo, hi)
        eligible = counted & ~clipped & (cov > lb) & (cov < ub)
        t = torch.arange(B * W, dtype=torch.int64, device=DEV).view(B, W)
        keys = port.fmix32(t ^ (seed & 0xffffffff))
    keys, eligible = keys.cpu(), eligible.cpu()
    E, k, T, need = port.state_words(keys, eligible, ratio, n)
    want = port.top_k(keys, eligible, k)
    got = sel.bool().cpu()
    assert torch.equal(got, want), ('selection', int(got.sum()), int(want.sum()), int((got != want).sum()))
    assert (int(state[1]), int(state[2]), int(state[5]), int(state[6])) == (E, k, T, need), \
        ('state words (E, k, T, need)', state[[1, 2, 5, 6]].tolist(), (E, k, T, need))
    want_share = torch.tensor(k / n if n else 0.0, dtype=F32)
    assert float(share) == float(want_share), ('share', float(share), float(want_share))
    sel2, state2, share2 = _select(*args)
    assert torch.equal(sel2, sel) and torch.equal(state2, raw) and _bits(share2).item() == _bits(share).item(), \
        'run to run'
    return sel, state


def _operands(B, W, lp_dtype, adv_dtype, seed, layout, p_counted=0.8):
    """(lp, old, adv, counted, row_end) on the device: lp in [-4, 0], old within ~0.3 of it (ratios on both sides of
    the clip range), advantages N(0, 2); the mask layout counts ~p_counted of the tokens, the row_end layout a random
    prefix of each row (an empty row included when B > 1)."""
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, W, generator=g) * 4
    old = lp + torch.randn(B, W, generator=g) * 0.3
    if layout == 'mask':
        adv = (torch.randn(B, W, generator=g) * 2).to(adv_dtype)
        counted = torch.rand(B, W, generator=g) < p_counted
        counted[0, 0] = True
        row_end = None
    else:
        adv = torch.randn(B, generator=g)
        row_end = torch.randint(0, W + 1, (B,), generator=g).to(torch.int32)
        row_end[0] = max(1, int(row_end[0]))
        if B > 1:
            row_end[-1] = 0
        counted = torch.arange(W)[None, :] < row_end[:, None].long()
        row_end = row_end.to(DEV)
    return lp.to(lp_dtype).to(DEV), old.to(lp_dtype).to(DEV), adv.to(DEV), counted.to(DEV), row_end


SHAPES = [(1, 1), (1, 31), (3, 257), (300, 700), (520, 1031)]


def _shape_cases():
    """Every shape in both layouts and both modes, the log-prob and advantage dtypes rotated over the cases (each
    shape sees all three log-prob dtypes, the mask layout every advantage dtype)."""
    out = []
    i = 0
    for B, W in SHAPES:
        for cov_mode in MODES:
            for layout in ('mask', 'row_end'):
                out.append(pytest.param(B, W, cov_mode, layout, DTYPES[i % 3], DTYPES[(i // 3) % 3],
                                        'f32' if i % 4 == 3 else 'faithful',
                                        id=f'{B}x{W}-{cov_mode}-{layout}-{i}'))
                i += 1
    return out


@pytest.mark.parametrize('B,W,cov_mode,layout,lp_dt,adv_dt,mode', _shape_cases())
def test_selection_shapes_layouts_dtypes(ops, B, W, cov_mode, layout, lp_dt, adv_dt, mode):
    """(300, 700): B > 256 rows (cov_mark_kernel's scan of the earlier rows' ties takes a second stride) and W > 256,
    neither a multiple of 32.  (520, 1031): 536 120 tokens, more than cov_grid's 262 144 a pass, so the grid-stride
    loops of cov_keys_kernel and cov_hist_lo_kernel take a second pass.  Every operand is strided (row stride W + 32)."""
    lp, old, adv, counted, row_end = _operands(B, W, lp_dt, adv_dt, seed=B * 7 + W, layout=layout)
    for ratio in (0.3, 0.05):
        _check_selection(lp, adv, counted, cov_mode, ratio, mode, old=old, row_end=row_end, lb=-1.0, ub=1.0,
                         seed=port.hash_seed(7, 0, B))


@pytest.mark.parametrize('adv_dt', DTYPES)
@pytest.mark.parametrize('lp_dt', DTYPES)
def test_selection_dtype_pairs(ops, lp_dt, adv_dt):
    """Each log-prob dtype with each advantage dtype in the mask layout, both modes, both roundings."""
    lp, old, adv, counted, _ = _operands(300, 700, lp_dt, adv_dt, seed=3, layout='mask')
    for cov_mode in MODES:
        for mode in ('faithful', 'f32'):
            _check_selection(lp, adv, counted, cov_mode, 0.1, mode, old=old, lb=-0.5, ub=2.0, seed=99)


@pytest.mark.parametrize('B,W', [(300, 700), (520, 1031)])
@pytest.mark.parametrize('layout', ['mask', 'row_end'])
def test_kl_cov_ties_across_every_row(ops, layout, B, W):
    """Every log-prob equal: every counted covariance is (A - mean A) * 0, +0 or -0, one key after the fold.  k < E, so
    `need` < the tie group, and the group spans every row: the first k counted tokens by flat index are taken, which
    needs the tie count of every earlier row (rows past 256 included) and -0 equal to +0."""
    lp, _, adv, counted, row_end = _operands(B, W, F32, F32, seed=B, layout=layout, p_counted=0.9)
    lp = torch.full_like(lp, -1.5)
    n = int(counted.sum())
    for ratio in (0.29, 0.5, 0.9, 0.999):
        sel, state = _check_selection(lp, adv, counted, 'kl_cov', ratio, row_end=row_end)
        k = port.n_select(ratio, n)
        assert int(state[6]) == k < int(state[1]) == n  # need == k < E: the cut falls inside the tie group
        first = torch.nonzero(counted.reshape(-1).cpu()).squeeze(1)[:k]
        assert bool(sel.reshape(-1).cpu()[first].all())
    a_full = adv if row_end is None else adv.view(-1, 1).expand(B, W)
    cov = port.covariance(lp, a_full, *(t.to(DEV) for t in port.means(lp.cpu(), a_full.cpu(), counted.cpu())))
    assert bool((cov == 0)[counted].all())
    neg = torch.signbit(cov)
    assert bool((neg & counted).any()) and bool((~neg & counted).any())  # both -0 and +0 among the ties


def test_kl_cov_keys_equal_in_the_high_half(ops):
    """Covariances in [1, 1 + 2^-7): every key has the same high 16 bits, so the threshold is found in the low half
    alone; each value appears twice (ties there too).  Pairs (lp -1, A v) and (lp -3, A -v) keep both means exact
    (0 and -2), so cov = v exactly."""
    B, W = 64, 96
    g = torch.Generator().manual_seed(1)
    v = 1.0 + torch.randint(0, 1 << 16, (B, W // 2), generator=g).double() * 2.0 ** -23
    lp = torch.stack([torch.full_like(v, -1.0), torch.full_like(v, -3.0)], -1).reshape(B, W)
    adv = torch.stack([v, -v], -1).reshape(B, W)
    counted = torch.ones(B, W, dtype=torch.bool)
    for lp_dt in (F32, BF, F16):
        for ratio in (0.1, 0.37, 0.8):
            sel, state = _check_selection(lp.to(lp_dt).to(DEV), adv.float().to(DEV), counted.to(DEV), 'kl_cov', ratio)
            assert int(state[5]) >> 16 == port.order_key(torch.tensor([1.0]))[0].item() >> 16


@pytest.mark.parametrize('cov_mode', MODES)
def test_selection_count_edges(ops, cov_mode):
    """k = 1 (int(ratio * N) == 0), k = E (ratio 1), ratio 0.29 at N = 100 (int(28.999...) = 28)."""
    lp, old, adv, counted, _ = _operands(1, 100, F32, F32, seed=5, layout='mask', p_counted=1.0)
    kw = dict(old=old, lb=-1e3, ub=1e3)
    for ratio, k in ((1e-9, 1), (0.29, 28), (1.0, None)):
        _, state = _check_selection(lp, adv, counted, cov_mode, ratio, **kw)
        if k is not None:
            assert int(state[2]) == k
        else:
            assert int(state[2]) == int(state[1])  # every eligible token
    lp, old, adv, counted, _ = _operands(37, 211, BF, BF, seed=6, layout='mask')
    _check_selection(lp, adv, counted, cov_mode, 1.0, old=old, lb=-1e3, ub=1e3)


def test_clip_cov_few_or_no_eligible(ops):
    """E < k (a narrow covariance window), E = 0 with N > 0 (a window no covariance reaches), and N = 0 in both layouts
    (an empty mask, every row_end 0): k = 0, T = 0xffffffff, need = 0, share 0 and an all-zero selection."""
    lp, old, adv, counted, _ = _operands(40, 300, F32, F32, seed=8, layout='mask')
    _, state = _check_selection(lp, adv, counted, 'clip_cov', 0.5, old=old, lb=0.0, ub=0.01)
    assert 0 < int(state[1]) < port.n_select(0.5, int(counted.sum())) and int(state[2]) == int(state[1])
    _, state = _check_selection(lp, adv, counted, 'clip_cov', 0.5, old=old, lb=1e29, ub=1e30)
    assert int(state[0]) > 0 and state[[1, 2, 6]].tolist() == [0, 0, 0] and int(state[5]) == 0xffffffff
    for cov_mode in MODES:
        sel, state = _check_selection(lp, adv, torch.zeros_like(counted), cov_mode, 0.5, old=old)
        assert state[[0, 1, 2]].tolist() == [0, 0, 0] and not bool(sel.any())
        lp2, old2, adv2, counted2, row_end = _operands(40, 300, F32, F32, seed=8, layout='row_end')
        sel, state = _check_selection(lp2, adv2, torch.zeros_like(counted2), cov_mode, 0.5, old=old2,
                                      row_end=torch.zeros_like(row_end))
        assert state[[0, 1, 2]].tolist() == [0, 0, 0] and not bool(sel.any())


@pytest.mark.parametrize('what', ['nan', 'inf'])
def test_kl_cov_nan_and_inf_covariances(ops, what):
    """A counted NaN log-prob: NaN means and every key 0xffffffff (ties to the smaller flat index).  A counted -inf
    log-prob: the mean is -inf, the covariances +-inf, and NaN where both factors meet (NaN above +inf)."""
    lp, _, adv, counted, _ = _operands(20, 333, F32, F32, seed=9, layout='mask')
    lp = lp.clone()
    lp[3, 5] = NAN if what == 'nan' else -float('inf')
    counted[3, 5] = True
    if what == 'inf':
        lp[7, :40] = -float('inf')
        counted[7, :40] = True
    for ratio in (0.01, 0.4):
        _check_selection(lp, adv, counted, 'kl_cov', ratio)
    _, state = _check_selection(lp, adv, counted, 'clip_cov', 0.4, old=lp)  # no covariance inside (1, 5): E = 0
    assert int(state[1]) == 0 and int(state[0]) == int(counted.sum())


@pytest.mark.parametrize('seed', [0, 0xffffffff])
def test_clip_cov_hash_seed_edges(ops, seed):
    lp, old, adv, counted, _ = _operands(260, 301, BF, F32, seed=10, layout='mask')
    for ratio in (0.01, 0.5):
        _check_selection(lp, adv, counted, 'clip_cov', ratio, old=old, lb=-2.0, ub=2.0, seed=seed)


@pytest.mark.parametrize('layout', ['mask', 'row_end'])
@pytest.mark.parametrize('dt', [BF, F16])
def test_clip_cov_eligibility_in_the_faithful_rounding(ops, dt, layout):
    """Clip-Cov's eligible tokens under `faithful` 16-bit log-probs are those the clip predicate of cov_port, on ATen
    CUDA in the dtype, leaves unclipped: the clip bounds and the ratio round to the log-probs' dtype, the products to
    the promoted one.  At ratio 1 every eligible token is selected, so the selection is the eligibility itself.
    Tokens whose predicate one fp32 ulp of exp could flip get old = lp (cov_port.clear_clip_band); explicit r = 1,
    A = 0 tokens tie the two branches and stay unclipped.  The test asserts that its operands hold tokens the fp32
    ratio would classify differently, so a selection that rounds the ratio in fp32 fails here."""
    B, W, lo, hi = 96, 1000, 0.2, 0.28
    lp, old, adv, counted, row_end = _operands(B, W, dt, dt, seed=12, layout=layout)
    a_full = adv if layout == 'mask' else adv.view(-1, 1).expand(B, W)
    if layout == 'mask':
        adv = adv.clone()
        adv[:, ::17] = 0.0
        old = torch.where(torch.arange(W, device=DEV) % 17 == 0, lp, old)
        a_full = adv
    old = port.clear_clip_band(lp, old, a_full, lo, hi)
    assert bool(port.stable_clip(lp, old, a_full, lo, hi).all())
    ad = a_full.dtype if layout == 'mask' else F32
    in_dt = port.clipped(lp, old, a_full.to(ad), lo, hi)
    # the same predicate with the ratio and the bounds in fp32 and the products still rounded to the promoted dtype
    r32 = torch.exp(lp.float() - old.float())
    a32 = a_full.float()
    in_f32 = (a32 * torch.clamp(r32, 1 - lo, 1 + hi)).to(ad) < (a32 * r32).to(ad)
    assert int(((in_dt != in_f32) & counted).sum()) >= 3, 'no token tells the two roundings apart'
    for ratio in (1.0, 0.5):
        _check_selection(lp, adv, counted, 'clip_cov', ratio, old=old, row_end=row_end, lo=lo, hi=hi, lb=-1e3,
                         ub=1e3, seed=21)


@pytest.mark.parametrize('cov_mode', MODES)
def test_selection_near_2_pow_24_tokens(ops, cov_mode):
    """4096 x 4096 bf16 log-probs, faithful: 64 grid-stride passes, 4096 rows of tie counts."""
    lp, old, adv, counted, _ = _operands(4096, 4096, BF, BF, seed=13, layout='mask')
    _check_selection(lp, adv, counted, cov_mode, 2e-4 if cov_mode == 'kl_cov' else 0.3, old=old, lb=-1.0, ub=1.0,
                     seed=77)


# ---- 2. the Cov loss entry points through the C ABI -------------------------------------------------------------------
def _k5_cov(lp, old, adv, mask, sel, cov_mode, lo, hi, agg, coef, mode, ref=None, kl_coeff=0.0, est='k3',
            counter=None):
    """aa_ppo_actor_loss_cov on guarded buffers (sel's stride gap holds 1s) -> (loss fp32[2], agg(KL) or None, grad,
    clip fractions fp32[2]); the counter must read 0 afterwards."""
    L = _lib()
    B, W = lp.shape
    gl, go, ga = Guarded(lp), Guarded(old), Guarded(adv)
    gm, gs = Guarded(mask.to(torch.uint8), fill=1), Guarded(sel.to(torch.uint8), fill=1)
    gref = Guarded(ref) if ref is not None else None
    grad = Guarded(torch.zeros_like(lp))
    loss, klo, cf = (Guarded(torch.zeros(1, n, device=DEV)) for n in (2, 1, 2))
    rows = torch.full((5 * B,), NAN, device=DEV)
    counter = Words() if counter is None else counter
    L.check(L.lib().aa_ppo_actor_loss_cov(
        gl.view.data_ptr(), gl.view.stride(0), go.view.data_ptr(), go.view.stride(0), L.dtype_code(lp.dtype),
        ga.view.data_ptr(), ga.view.stride(0), L.dtype_code(adv.dtype), gm.view.data_ptr(), gm.view.stride(0), B, W,
        lo, hi, AGG[agg], COV[cov_mode], coef, gs.view.data_ptr(), gs.view.stride(0), _mode_code(mode),
        gref.view.data_ptr() if gref else None, gref.view.stride(0) if gref else 0, kl_coeff, EST[est],
        loss.view.data_ptr(), klo.view.data_ptr() if gref else None, grad.view.data_ptr(), grad.view.stride(0),
        cf.view.data_ptr(), rows.data_ptr(), counter.ptr(), L.stream_ptr(torch.device(DEV))))
    torch.cuda.synchronize()
    for g in (gl, go, ga, gm, gs, gref, grad, loss, klo, cf):
        assert g is None or g.intact(), 'a guard band was written'
    assert counter.values() == [0], 'the counter was not re-armed'
    return loss.view[0].clone(), (klo.view[0, 0].clone() if gref else None), grad.view.clone(), cf.view[0].clone()


def _realistic(B, W, dt, seed):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, W, generator=g) * 4
    old = lp + torch.randn(B, W, generator=g) * 0.3
    ref = lp + torch.randn(B, W, generator=g) * 0.1
    adv = torch.randn(B, W, generator=g)
    mask = torch.rand(B, W, generator=g) < 0.8
    mask[:, 0] = True
    sel = torch.rand(B, W, generator=g) < 0.1  # on counted and uncounted tokens alike
    return tuple(t.to(dt).to(DEV) for t in (lp, old, ref, adv)) + (mask.to(DEV), sel.to(DEV))


def _cf_tol(mask, agg):
    """One token's weight in a clip fraction."""
    m = mask.double()
    if agg == 'token-mean':
        return 1.0 / float(m.sum()) + 1e-6
    return float((1.0 / (m.size(0) * m.sum(-1).clamp(min=1))).max()) + 1e-6


PPO_CASES = [(mode_, agg, kl) for mode_ in MODES for agg in ('seq-mean-token-mean', 'token-mean')
             for kl in (None, 'k1', 'k2', 'k3')]


@pytest.mark.parametrize('shape', [(1, 64), (7, 301), (1024, 1024)], ids=['1x64', '7x301', '1024x1024'])
@pytest.mark.parametrize('mode', ['faithful', 'f32'])
@pytest.mark.parametrize('dt', DTYPES)
def test_ppo_cov_loss_vs_port(ops, dt, mode, shape):
    """Every aggregation, KL loss term off and k1 / k2 / k3, both Cov modes: the loss, agg(KL) and the gradient within 1
    ulp of the port on ATen CUDA in the dtype (>= 97 % of the gradient bit-identical), the clip fractions within one
    token (0 under KL-Cov), and Clip-Cov's selected tokens without a gradient."""
    B, W = shape
    lp, old, ref, adv, mask, sel = _realistic(B, W, dt, seed=B + W)
    cases = PPO_CASES if B * W < 1 << 20 else [('clip_cov', 'token-mean', 'k3'), ('kl_cov', 'seq-mean-token-mean', 'k2')]
    faithful = mode == 'faithful' and dt != F32
    cd = dt if faithful else F32
    eff = sel & mask
    for cov_mode, agg, kl in cases:
        what = f'{cov_mode} {agg} kl={kl} {dt} {mode} {B}x{W}'
        lo, hi, coef, kc = 0.2, 0.28, (0.7 if cov_mode == 'kl_cov' else 0.0), 0.1
        loss, klo, grad, cf = _k5_cov(lp, old, adv, mask, sel, cov_mode, lo, hi, agg, coef, mode,
                                      ref=ref if kl else None, kl_coeff=kc if kl else 0.0, est=kl or 'k3')
        x = lp.to(cd).clone().requires_grad_(True)
        if kl:
            want, kl_want, total = port.ppo_loss_kl(cov_mode, x, old.to(cd), adv.to(cd), mask, eff, agg, lo, hi, coef,
                                                   ref.to(cd), kc, kl)
        else:
            want = total = port.ppo_loss(cov_mode, x, old.to(cd), adv.to(cd), mask, eff, agg, lo, hi, coef)
        total.backward()
        kl_want = kl_want.detach() if kl else None
        if faithful:
            assert_ulp_close(_loss16(loss, dt).reshape(1), want.detach().reshape(1), max_ulp=1, min_exact=0.0,
                             what=what + ' loss')
            assert_ulp_close(grad, x.grad, max_ulp=1, min_exact=0.97, what=what + ' grad')
        else:
            torch.testing.assert_close(loss[0], want.detach().float(), rtol=2e-5, atol=1e-7)
            if dt == F32:
                torch.testing.assert_close(grad, x.grad, rtol=2e-5, atol=2e-5 * float(x.grad.abs().max()))
            else:
                assert_ulp_close(grad, x.grad.to(dt), max_ulp=1, min_exact=0.97, what=what + ' grad')
        if kl:
            eps = {BF: 2.0 ** -7, F16: 2.0 ** -10, F32: 2e-5}[cd]
            assert abs(float(klo) - float(kl_want)) <= eps * abs(float(kl_want)) + 1e-7, (what, float(klo),
                                                                                           float(kl_want))
        if cov_mode == 'clip_cov':
            if not kl:
                assert not bool(grad[eff].any()), what + ': a selected token has a gradient'
            fc, _ = clip_fractions(lp.to(cd), old.to(cd), adv.to(cd), mask, lo, hi, None, agg)
            assert abs(float(cf[0]) - fc) <= _cf_tol(mask, agg), (what, float(cf[0]), fc)
            assert float(cf[1]) == 0.0
        else:
            assert cf.tolist() == [0.0, 0.0], what + ': KL-Cov clips nothing'
    ops.check_status()


GRPO_CASES = [(mode_, agg, est, first) for mode_ in MODES for agg in AGG for est in EST for first in (True, False)
              if (est == 'k3' or agg == 'token-mean')]
EOS = 2


def _grpo_cov(lp, ref, old, adv, tok, sel, cov_mode, lo, hi, agg, est, beta, coef, mode, counter=None):
    """aa_grpo_loss_cov on guarded buffers -> (loss, grad, clip fractions, row_end, counted total)."""
    L = _lib()
    B, K = lp.shape
    gl, gr = Guarded(lp), Guarded(ref)
    go = Guarded(old) if old is not None else None
    ga, gs = _vec(adv.float(), NAN), Guarded(sel.to(torch.uint8), fill=1)
    tk = fenced(tok, K + 3, pad=EOS)
    loss, cf = Guarded(torch.zeros(1, 1, device=DEV)), Guarded(torch.zeros(1, 2, device=DEV))
    grad = Guarded(torch.zeros_like(lp))
    row_end = _vec(torch.zeros(B, dtype=torch.int32, device=DEV), -7)
    scratch = torch.full((1 + 4 * B,), NAN, device=DEV)
    counter = Words(n=2) if counter is None else counter
    L.check(L.lib().aa_grpo_loss_cov(
        gl.view.data_ptr(), gl.view.stride(0), gr.view.data_ptr(), gr.view.stride(0),
        go.view.data_ptr() if go else None, go.view.stride(0) if go else 0, L.dtype_code(lp.dtype),
        ga.view.data_ptr(), tk.data_ptr(), tk.stride(0), EOS, B, K, beta, lo, hi, AGG[agg], EST[est], COV[cov_mode],
        coef, gs.view.data_ptr(), gs.view.stride(0), _mode_code(mode), loss.view.data_ptr(), grad.view.data_ptr(),
        grad.view.stride(0), cf.view.data_ptr(), row_end.view.data_ptr(), scratch.data_ptr(), counter.ptr(),
        L.stream_ptr(torch.device(DEV))))
    torch.cuda.synchronize()
    for g in (gl, gr, go, ga, gs, loss, cf, grad, row_end):
        assert g is None or g.intact(), 'a guard band was written'
    assert counter.values() == [0, 0], 'the counters were not re-armed'
    return loss.view[0, 0].clone(), grad.view.clone(), cf.view[0].clone(), row_end.view[0].clone(), float(scratch[0])


def _grpo_operands(B, K, dt, seed):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, K, generator=g) * 4
    old = lp + torch.randn(B, K, generator=g) * 0.3
    ref = lp + torch.randn(B, K, generator=g) * 0.1
    tok = torch.randint(3, 50, (B, K), generator=g)
    for b in range(B):
        if b % 3 != 2:  # a third of the rows run to the end without an eos
            tok[b, int(torch.randint(0, K, (1,), generator=g))] = EOS
    adv = torch.randn(B, generator=g)
    sel = torch.rand(B, K, generator=g) < 0.1  # past row_end too
    return (lp.to(dt).to(DEV), old.to(dt).to(DEV), ref.to(dt).to(DEV), adv.to(DEV), tok.to(DEV), sel.to(DEV))


@pytest.mark.parametrize('shape', [(1, 64), (9, 173), (1024, 1024)], ids=['1x64', '9x173', '1024x1024'])
@pytest.mark.parametrize('mode', ['faithful', 'f32'])
@pytest.mark.parametrize('dt', DTYPES)
def test_grpo_cov_loss_vs_port(ops, dt, mode, shape):
    """Every aggregation (with k3), k1 / k2 / k3 (token-mean), first and later updates, both Cov modes: the fp32 loss
    to fp32 summation error, the gradient within 1 ulp (>= 97 % bit-identical) of the port on ATen CUDA in the dtype,
    the clip fractions within one token (0 under KL-Cov and on the first update)."""
    B, K = shape
    lp, old, ref, adv, tok, sel = _grpo_operands(B, K, dt, seed=B * K)
    mask = completion_mask(tok, EOS).bool()
    eff = sel & mask
    cases = GRPO_CASES if B * K < 1 << 20 else [('clip_cov', 'token-mean', 'k1', False),
                                                ('kl_cov', 'seq-mean-token-mean', 'k3', False)]
    faithful = mode == 'faithful' and dt != F32
    cd = dt if faithful else F32
    for cov_mode, agg, est, first in cases:
        what = f'{cov_mode} {agg} {est} first={first} {dt} {mode} {B}x{K}'
        lo, hi, beta, coef = 0.2, 0.28, 0.04, (0.7 if cov_mode == 'kl_cov' else 0.0)
        loss, grad, cf, row_end, total = _grpo_cov(lp, ref, None if first else old, adv, tok, sel, cov_mode, lo, hi,
                                                   agg, est, beta, coef, mode)
        assert torch.equal(torch.arange(K, device=DEV) < row_end.unsqueeze(1), mask), what + ' row_end'
        assert total == float(mask.sum()), what + ' the fp32 count'
        x = lp.to(cd).clone().requires_grad_(True)
        want = port.grpo_loss(cov_mode, x, ref.to(cd), None if first else old.to(cd), adv.float(), mask, eff, beta,
                              agg, lo, hi, coef, estimator=est)
        want.backward()
        assert want.dtype == F32
        assert abs(float(loss) - float(want)) <= 1e-5 * max(1e-3, abs(float(want))), (what, float(loss), float(want))
        if dt == F32:
            torch.testing.assert_close(grad, x.grad, rtol=2e-5, atol=2e-5 * float(x.grad.abs().max()))
        else:
            assert_ulp_close(grad, x.grad.to(dt), max_ulp=1, min_exact=0.97, what=what + ' grad')
        if cov_mode == 'clip_cov' and not first:
            fc, _ = grpo_clip_fractions(lp.to(cd), old.to(cd), adv.float().view(-1, 1), mask, lo, hi, None, agg)
            assert abs(float(cf[0]) - fc) <= _cf_tol(mask, 'seq-mean-token-mean' if agg == 'seq-mean-token-mean'
                                                     else 'token-mean'), (what, float(cf[0]), fc)
        else:
            assert float(cf[0]) == 0.0, what
        assert float(cf[1]) == 0.0
    ops.check_status()


def _exact_sel(adv64, mask64, dt, seed):
    """A selection under which the Clip-Cov loss at lp == old (the masked mean of adv * ~sel) does not depend on the fp32
    summation order (test_cpu_faithful_counts.mean_rounds_alike)."""
    for s in range(seed, seed + 50):
        g = torch.Generator().manual_seed(s)
        sel = torch.rand(adv64.shape, generator=g) < 0.05
        if mean_rounds_alike(k5_actor(adv64 * ~sel, mask64, dt)[1], dt):
            return sel
    raise AssertionError('no selection keeps the loss exact')


@pytest.mark.parametrize('cov_mode', MODES)
@pytest.mark.parametrize('dt,n', CASES, ids=CASE_IDS)
def test_ppo_cov_exact_counts_vs_port(ops, dt, n, cov_mode):
    """lp == old and dyadic advantages at the counts a 16-bit dtype cannot hold: the 16-bit loss and the gradient
    bit-identical to the port on ATen CUDA (which divides by the count rounded to the dtype), and Clip-Cov's loss to the
    float64 restatement of the objective without its selected terms.  Under KL-Cov the selected tokens keep the
    unselected gradient (d = 0, sign(0) = 0)."""
    B = 3
    lp64, adv64, mask64 = exact_actor_case(B, n, dt, seed=n + B)
    sel = _exact_sel(adv64, mask64, dt, seed=n)
    lp, adv, mask, seld = lp64.to(dt).to(DEV), adv64.to(dt).to(DEV), mask64.to(DEV), sel.to(DEV)
    for agg in ('seq-mean-token-mean', 'token-mean'):
        what = f'{cov_mode} {agg} {dt} n={n}'
        coef = 0.5 if cov_mode == 'kl_cov' else 0.0
        loss, _, grad, _ = _k5_cov(lp, lp, adv, mask, seld, cov_mode, 0.2, 0.2, agg, coef, 'faithful')
        x = lp.clone().requires_grad_(True)
        want = port.ppo_loss(cov_mode, x, lp, adv, mask, seld & mask, agg, 0.2, 0.2, coef)
        want.backward()
        _identical(_loss16(loss, dt), want, what + ' loss')
        assert float(loss[0]) == float(want), what + ' fp32 loss word'
        _identical(grad, x.grad, what + ' grad')
        plain, _, gplain, _ = _k5_cov(lp, lp, adv, mask, torch.zeros_like(seld), cov_mode, 0.2, 0.2, agg, coef,
                                      'faithful')
        if cov_mode == 'kl_cov':
            _identical(grad, gplain, what + ' KL-Cov at d = 0 is the unselected gradient')
            _identical(_loss16(loss, dt), _loss16(plain, dt), what + ' KL-Cov loss at d = 0')
        elif agg == 'seq-mean-token-mean':
            w_loss, _, _ = k5_actor(adv64 * ~sel, mask64, dt)
            assert float(want) == float(w_loss), what + ' loss vs float64'
            assert not bool(grad[seld & mask].any())


@pytest.mark.parametrize('cov_mode', MODES)
@pytest.mark.parametrize('dt,counts', TOKEN_MEAN_CASES, ids=TOKEN_MEAN_IDS)
def test_ppo_cov_token_mean_totals_vs_port(ops, dt, counts, cov_mode):
    """Token-mean over a total the dtype cannot hold (1501 -> 1504 in bf16, 2049 -> 2048 in fp16), bit for bit, on
    test_cpu_cov_pin.token_mean_case's operands (whose exactness that file checks)."""
    lp64, adv64, mask64, sel64 = token_mean_case(counts)
    lp, adv = lp64.to(dt).to(DEV), adv64.to(dt).to(DEV)
    mask, sel = mask64.to(DEV), sel64.to(DEV)
    coef = 0.5 if cov_mode == 'kl_cov' else 0.0
    loss, _, grad, _ = _k5_cov(lp, lp, adv, mask, sel, cov_mode, 0.2, 0.28, 'token-mean', coef, 'faithful')
    x = lp.clone().requires_grad_(True)
    want = port.ppo_loss(cov_mode, x, lp, adv, mask, sel & mask, 'token-mean', 0.2, 0.28, coef)
    want.backward()
    _identical(_loss16(loss, dt), want, f'{cov_mode} {dt} {counts} loss')
    _identical(grad, x.grad, f'{cov_mode} {dt} {counts} grad')


@pytest.mark.parametrize('cov_mode', MODES)
def test_grpo_cov_exact_total(ops, cov_mode):
    """bf16 log-probs over 1501 counted tokens (1504 in bf16), lp == old == ref: the fp32 per-token loss is divided by
    the exact fp32 count, the gradient bit-identical to the port."""
    B, K = 3, 520
    tok = torch.randint(4, 100, (B, K), generator=torch.Generator().manual_seed(K))
    for b, e in enumerate((500, 500, 501)):
        tok[b, e - 1] = EOS
    tok = tok.to(DEV)
    g = torch.Generator().manual_seed(11)
    lp = (-torch.rand(B, K, generator=g) * 4).to(BF).to(DEV)
    adv = torch.randn(B, generator=g).to(DEV)
    sel = (torch.rand(B, K, generator=g) < 0.1).to(DEV)
    mask = completion_mask(tok, EOS).bool()
    coef = 0.5 if cov_mode == 'kl_cov' else 0.0
    loss, grad, _, _, total = _grpo_cov(lp, lp, lp, adv, tok, sel, cov_mode, 0.2, 0.2, 'token-mean', 'k3', 0.04, coef,
                                        'faithful')
    assert total == 1501.0
    x = lp.clone().requires_grad_(True)
    want = port.grpo_loss(cov_mode, x, lp, lp, adv, mask, sel & mask, 0.04, 'token-mean', 0.2, 0.2, coef,
                          estimator='k3')
    want.backward()
    _identical(grad, x.grad, f'{cov_mode} grpo grad')
    # fp32 sums in different orders; a divisor of 1504 would be 2e-3 off
    assert abs(float(loss) - float(want)) <= 1e-5 * abs(float(want)), (float(loss), float(want))


def test_k5_counter_rearms_across_the_cov_entry_points(ops):
    """The largest Cov grid here (4500 blocks), then one block, then aa_ppo_actor_loss_obj and aa_ppo_actor_loss, all on
    one counter word: every result right, the counter 0 after each call."""
    L = _lib()
    counter = Words()
    for B in (4500, 1):
        lp, old, _, adv, mask, sel = _realistic(B, 31, F32, seed=B)
        for cov_mode in MODES:
            loss, _, grad, _ = _k5_cov(lp, old, adv, mask, sel, cov_mode, 0.2, 0.28, 'seq-mean-token-mean',
                                       0.7 if cov_mode == 'kl_cov' else 0.0, 'f32', counter=counter)
            x = lp.clone().requires_grad_(True)
            want = port.ppo_loss(cov_mode, x, old, adv, mask, sel & mask, 'seq-mean-token-mean', 0.2, 0.28,
                                 0.7 if cov_mode == 'kl_cov' else 0.0)
            want.backward()
            torch.testing.assert_close(loss[0], want.detach(), rtol=2e-5, atol=1e-7)
            torch.testing.assert_close(grad, x.grad, rtol=2e-5, atol=2e-5 * float(x.grad.abs().max()))
    lp, old, _, adv, mask, _ = _realistic(3, 31, F32, seed=3)
    lib, st = L.lib(), L.stream_ptr(torch.device(DEV))
    for legacy in (False, True):
        loss = torch.full((2,), NAN, device=DEV)
        grad = torch.zeros_like(lp)
        rows = torch.full((4 * 3,), NAN, device=DEV)
        m8 = mask.to(torch.uint8)
        common = (lp.data_ptr(), 31, old.data_ptr(), 31, L.AA_F32, adv.data_ptr(), 31, L.AA_F32, m8.data_ptr(), 31, 3,
                  31)
        if legacy:
            L.check(lib.aa_ppo_actor_loss(*common, 0.2, L.MODE_F32, loss.data_ptr(), grad.data_ptr(), 31,
                                          rows.data_ptr(), counter.ptr(), st))
        else:
            L.check(lib.aa_ppo_actor_loss_obj(*common, 0.2, 0.2, 0.0, 0, L.MODE_F32, loss.data_ptr(), grad.data_ptr(),
                                              31, None, rows.data_ptr(), counter.ptr(), st))
        torch.cuda.synchronize()
        assert counter.values() == [0]
        want = obj_loss(lp, old, adv, mask, 0.2, 0.2)
        torch.testing.assert_close(loss[0], want, rtol=2e-5, atol=1e-7)


# ---- 3. the composed nodes in the trainers' mode ----------------------------------------------------------------------
V = 32000


def _cov_objective(ops, mode, grpo=False):
    cls = ops.GrpoObjective if grpo else ops.ActorObjective
    if mode == 'clip_cov':
        return cls(policy_loss_mode=mode, clip_cov_ratio=0.05, clip_cov_lb=-1e3, clip_cov_ub=1e3)
    return cls(policy_loss_mode=mode, kl_cov_ratio=0.05, ppo_kl_coef=0.5)


def _sel_kw(mode):
    return ({'clip_cov_ratio': 0.05, 'clip_cov_lb': -1e3, 'clip_cov_ub': 1e3} if mode == 'clip_cov' else
            {'kl_cov_ratio': 0.05})


def _off_the_bounds(lp, old, lo=0.2, hi=0.2, ulps=4):
    """old = lp on tokens whose ratio lies within `ulps` bf16 ulps of a clip bound: there bf16 rounding alone decides
    the side, and a float64 reference would clip a token the kernel (and the bf16 reference) leaves unclipped."""
    r = torch.exp(lp.double() - old.double())
    near = torch.zeros_like(r, dtype=torch.bool)
    for b in (1 - lo, 1 + hi):
        near |= (r - b).abs() <= ulps * 2.0 ** -8 * b
    return torch.where(near, lp.to(old.dtype), old)


def _at(lp64, lp):
    """float64 log-probs that take the kernel's values but differentiate through log_softmax: the float64 reference
    of the loss is then evaluated where the kernel evaluated it."""
    return lp64 + (lp.double() - lp64).detach()


@pytest.mark.parametrize('node', ['dense', 'tail'])
@pytest.mark.parametrize('mode', MODES)
def test_composed_actor_node_bf16(ops, mode, node):
    """K1 -> selection -> K5 Cov -> K1b in faithful bf16 at V = 32000, with an entropy bonus, a k3 KL loss term and the
    clip fractions: outputs (loss, log-probs, loss for the metrics, entropy mean, agg(KL), share, clip fractions).
    float64 autograd through log_softmax, evaluated at the node's own bf16 log-probs with the node's selection.
    Tolerances: the objective rounds each op to bf16 (8 significant bits, 2^-9 relative each), so the loss and agg(KL)
    sit within 1e-2 relative of float64 and the bf16 logit gradient within 2e-2 of its largest entry; the entropy is
    fp32 arithmetic on the same logits (1e-4)."""
    g = torch.Generator().manual_seed(21)
    B, Lq, coeff, kc = 3, 48, 0.01, 0.1
    logits = (torch.randn(B, Lq, V, generator=g) * 2).to(BF).to(DEV)
    ids = torch.randint(0, V, (B, Lq), generator=g).to(DEV)
    if node == 'dense':
        start, lens = 6, None
        W = Lq - 1 - start
        mask = (torch.rand(B, W, generator=g) < 0.9).to(DEV)
        mask[:, 0] = True
        rows = [list(range(start, Lq - 1))] * B
    else:
        start, lens = None, [30, 12, 41]
        W = max(lens)
        mask = (torch.arange(W)[None, :] < torch.tensor(lens)[:, None]).to(DEV)
        rows = [list(range(Lq - 1 - n, Lq - 1)) + [0] * (W - n) for n in lens]

    def run(old, adv, ref, **kw):
        x = logits.clone().requires_grad_(True)
        if node == 'dense':
            out = ops.dense_actor_loss(x, ids, start, old, adv, mask, 0.2, **kw)
        else:
            out = ops.tail_actor_loss(x, ids, lens, old, adv, mask, 0.2, **kw)
        return x, out

    z = torch.zeros(B, W, device=DEV)
    _, plain = run(z, z, z)
    base = plain[1].float().masked_fill(~mask, -1.0)
    old = _off_the_bounds(base.to(BF), (base + torch.randn(B, W, generator=g).to(DEV) * 0.2).to(BF))
    ref = (base + torch.randn(B, W, generator=g).to(DEV) * 0.1).to(BF)
    adv = torch.randn(B, W, generator=g).to(DEV)
    x, out = run(old, adv, ref, entropy_coeff=coeff, objective=_cov_objective(ops, mode), return_clip_fraction=True,
                 ref_log_probs=ref, kl_loss_coeff=kc, kl_loss_estimator='k3', cov_seed=4)
    assert len(out) == 7
    out[0].backward()
    lp = out[1].masked_fill(~mask, -1.0)  # the tail plan leaves its unscored positions as they were
    sel = ops.cov_token_selection(out[1], adv, mask, mode, old_log_probs=old, seed=4, **_sel_kw(mode)).bool()
    n = int(mask.sum())
    assert int(sel.sum()) == (port.n_select(0.05, n) if mode == 'kl_cov' else int(sel.sum())) and int(sel.sum()) > 0
    assert float(out[5]) == float(torch.tensor(int(sel.sum()) / n, dtype=F32)), 'share'
    x64 = logits.double().requires_grad_(True)
    r_idx = torch.tensor(rows, device=DEV)
    t64 = x64[torch.arange(B, device=DEV)[:, None], r_idx]  # (B, W, V): the tile row scoring each lp[b, t]
    lsm = torch.log_softmax(t64, -1)
    lab = ids.gather(1, (r_idx + 1).clamp(max=Lq - 1))
    lp64 = _at(lsm.gather(-1, lab[..., None]).squeeze(-1), lp)
    ent64 = -(lsm.exp() * lsm).sum(-1)
    m = mask.double()
    mm = lambda v: ((v * m).sum(-1) / m.sum(-1)).mean()  # noqa: E731
    pg = port.ppo_loss(mode, lp64, old.double(), adv.double(), mask, sel, 'seq-mean-token-mean', 0.2, 0.2,
                       0.5 if mode == 'kl_cov' else 1.0)
    d = ref.double() - lp64
    kl64 = mm(torch.exp(d) - d - 1)
    want = pg - coeff * mm(ent64) + kc * kl64
    want.backward()
    assert abs(float(out[0]) - float(want)) <= 1e-2 * max(1.0, abs(float(want))), ('loss', float(out[0]), float(want))
    assert abs(float(out[2].reshape(-1)[0]) - float(pg)) <= 1e-2 * max(1.0, abs(float(pg))), 'loss without the terms'
    assert abs(float(out[3]) - float(mm(ent64))) <= 1e-4 * float(mm(ent64)), ('entropy mean', float(out[3]))
    # k3 of a small d in bf16 is mostly rounding (exp(d) near 1 keeps 8 bits): agg(KL) is held to the bf16 port
    kl16 = kl_loss(lp, ref, mask, 'k3')
    assert abs(float(out[4]) - float(kl16)) <= 2.0 ** -7 * abs(float(kl16)), ('agg(KL)', float(out[4]), float(kl16))
    if mode == 'clip_cov':
        fc, _ = clip_fractions(lp, old, adv, mask, 0.2, 0.2)
        assert abs(float(out[6][0]) - fc) <= _cf_tol(mask, 'seq-mean-token-mean'), ('clip fraction', out[6], fc)
    else:
        assert out[6].tolist() == [0.0, 0.0]
    _rel(x.grad, x64.grad, 2e-2, f'{node} {mode} d loss / d logits')
    ops.check_status()


@pytest.mark.parametrize('mode', MODES)
def test_grpo_node_second_update_bf16(ops, mode):
    """grpo_loss_from_logits in faithful bf16 with old log-probs and beta * k3 KL: against float64 autograd at the
    node's own log-probs and selection (tolerances as the actor nodes')."""
    g = torch.Generator().manual_seed(22)
    B, P, K, beta = 4, 5, 40, 0.04
    logits = (torch.randn(B, P + K, V, generator=g) * 2).to(BF).to(DEV)
    ids = torch.randint(3, V, (B, P + K), generator=g)
    ids[0, P + 20], ids[2, P + 7] = EOS, EOS
    ids = ids.to(DEV)
    adv = torch.randn(B, generator=g).to(DEV)
    _, lp0, _ = ops.grpo_loss_from_logits(logits.clone(), ids, K, torch.zeros(B, K, dtype=BF, device=DEV), adv, EOS,
                                          beta)
    old = _off_the_bounds(lp0, (lp0.float() + torch.randn(B, K, generator=g).to(DEV) * 0.2).to(BF))
    ref = (lp0.float() + torch.randn(B, K, generator=g).to(DEV) * 0.1).to(BF)
    x = logits.clone().requires_grad_(True)
    out = ops.grpo_loss_from_logits(x, ids, K, ref, adv, EOS, beta, objective=_cov_objective(ops, mode, grpo=True),
                                    old_per_token_logps=old, return_clip_fraction=True, cov_seed=9)
    assert len(out) == 5
    loss, lp, row_end, share, cf = out
    loss.backward()
    mask = completion_mask(ids[:, -K:], EOS).bool()
    assert torch.equal(torch.arange(K, device=DEV) < row_end.unsqueeze(1), mask)
    sel = ops.cov_token_selection(lp, adv, row_end, mode, old_log_probs=old, seed=9, **_sel_kw(mode)).bool()
    assert int(sel.sum()) > 0
    assert float(share) == float(torch.tensor(int(sel.sum()) / int(mask.sum()), dtype=F32))
    x64 = logits.double().requires_grad_(True)
    lsm = torch.log_softmax(x64[:, P - 1:-1], -1)
    lp64 = _at(lsm.gather(-1, ids[:, P:, None]).squeeze(-1), lp)
    want = port.grpo_loss(mode, lp64, ref.double(), old.double(), adv.double(), mask, sel, beta, 'token-mean', 0.2,
                          0.2, 0.5 if mode == 'kl_cov' else 1.0, estimator='k3')
    want.backward()
    assert abs(float(loss) - float(want)) <= 1e-2 * max(1.0, abs(float(want))), (float(loss), float(want))
    if mode == 'clip_cov':
        fc, _ = grpo_clip_fractions(lp, old, adv.view(-1, 1), mask, 0.2, 0.2)
        assert abs(float(cf[0]) - fc) <= _cf_tol(mask, 'token-mean'), (cf, fc)
    else:
        assert cf.tolist() == [0.0, 0.0]
    _rel(x.grad, x64.grad, 2e-2, f'grpo {mode} d loss / d logits')
    ops.check_status()


@pytest.mark.parametrize('mode', MODES)
def test_image_ppo_fused_lm_head_step_vs_float64(ops, mode):
    """One rl_step of the image PPO trainer on the fused lm_head path (K6 -> selection -> K5 Cov -> K6b and the two
    backward GEMMs), in faithful bf16 with a 10 % selection: the actor's d hidden and d weight against float64 autograd
    through F.linear and log_softmax, evaluated at the step's own bf16 log-probs (K6 on the same hidden states and
    weight) with the selection ops.cov_token_selection takes from them.  Ratios within 4 bf16 ulps of a clip bound get
    old = lp before the step, so that bf16 rounding alone decides no token's clip side.  Tolerances: bf16 log-probs,
    ratios and per-token gradients (2^-9 relative each) and a bf16 gradient through bf16 GEMMs: 2e-2 of the largest
    entry of each gradient; the actor loss within 1e-2."""
    from test_gpu_fused_rl import LM, Critic, Phased

    from align_anything_b200.models.reward_model import ScoreModelOutput
    from align_anything_b200.trainers.text_image_to_text.ppo import PPOTrainer
    from align_anything_b200.trainers.text_to_text.ppo import actor_objective_of

    gen = torch.Generator().manual_seed(37)
    B, Lq, H, Vh = 3, 40, 128, 1031
    resp = [20, 9, 28]
    seq = torch.zeros((B, Lq), dtype=torch.int64)
    for b, n in enumerate(resp):
        seq[b, Lq - n - 8:] = torch.randint(2, Vh, (n + 8,), generator=gen)
    ids = seq.to(DEV)
    t = lambda *shape, s=1.0: (torch.randn(*shape, generator=gen) * s)  # noqa: E731
    hid_a, hid_r, hid_new = (t(B, Lq, H).bfloat16().to(DEV) for _ in range(3))
    hid_new = (hid_a.float() + 0.3 * hid_new.float()).bfloat16()  # the trained policy near the rollout's
    w_a = t(Vh, H, s=0.2).bfloat16().to(DEV)
    w_r = (w_a.float().cpu() + t(Vh, H, s=0.02)).bfloat16().to(DEV)
    reward = t(B).to(DEV)
    critic, new_critic = t(B, Lq, 1).to(DEV), t(B, Lq, 1).to(DEV).requires_grad_(True)
    keys = ({'clip_cov_ratio': 0.1, 'clip_cov_lb': -1e3, 'clip_cov_ub': 1e3} if mode == 'clip_cov' else
            {'kl_cov_ratio': 0.1, 'ppo_kl_coef': 0.5})
    tr = PPOTrainer(SimpleNamespace(train_cfgs=SimpleNamespace(policy_loss_mode=mode, seed=42, **keys)),
                    tokenizer=SimpleNamespace(pad_token_id=0))
    tr.fused_lm_head, tr.lm_head_chunk_rows = True, 32
    state = {'phase': 'rollout'}
    h_new, w_new = hid_new.clone().requires_grad_(True), w_a.clone().requires_grad_(True)
    tr.actor_model = Phased(LM(hid_a, w_a), LM(h_new, w_new), state)
    tr.actor_reference_model = LM(hid_r, w_r)
    tr.reward_model = Critic(lambda: ScoreModelOutput(end_scores=reward.unsqueeze(-1)))
    tr.reward_critic_model = Critic(lambda: ScoreModelOutput(scores=critic if state['phase'] == 'rollout' else new_critic))
    inference, training = tr.score_rollout({'input_ids': ids, 'attention_mask': ids != 0}, resp)
    mask = training['response_mask']
    # the step's own log-probs: the same op on the same operands as the fused node
    lp = ops.tail_log_probs_from_hidden(hid_new.clone().requires_grad_(True), w_a.clone().requires_grad_(True), ids,
                                        resp, chunk_rows=32, mode=tr.mode).detach()
    old = torch.where(mask, _off_the_bounds(lp, training['log_probs']), training['log_probs'])
    training['log_probs'] = old
    state['phase'] = 'train'
    out = tr.rl_step(inference, training)
    adv = tr.last_rl_tensors['advantages']
    objective = actor_objective_of(tr)
    lo, hi, _, _ = objective.args(tr.clip_range_ratio)
    agg = objective.loss_agg_mode
    sel = ops.cov_token_selection(lp, adv, mask, mode, old_log_probs=old, clip_range_ratio_low=lo,
                                  clip_range_ratio_high=hi, seed=ops.cov_hash_seed(42, 0, 0),
                                  **{k: v for k, v in keys.items() if k != 'ppo_kl_coef'}).bool()
    n = int(mask.sum())
    k = int(sel.sum())
    assert k > 1 and (mode == 'clip_cov' or k == port.n_select(0.1, n))
    assert out['train/actor_cov_fraction'] == pytest.approx(k / n, rel=1e-6)
    h64, w64 = hid_new.double().requires_grad_(True), w_a.double().requires_grad_(True)
    x = torch.nn.functional.linear(h64, w64)
    W = max(resp)
    lp64 = torch.zeros(B, W, dtype=torch.float64, device=DEV)
    for b, r in enumerate(resp):
        lsm = torch.log_softmax(x[b, Lq - 1 - r:Lq - 1], -1)
        lp64[b, :r] = lsm.gather(-1, ids[b, Lq - r:, None]).squeeze(-1)
    want = port.ppo_loss(mode, _at(lp64, lp), old.double(), adv.double(), mask, sel, agg, lo, hi,
                         keys.get('ppo_kl_coef', 1.0))
    want.backward()
    assert abs(out['train/actor_loss'] - float(want)) <= 1e-2 * max(1.0, abs(float(want))), (out['train/actor_loss'],
                                                                                            float(want))
    _rel(h_new.grad, h64.grad, 2e-2, f'{mode} fused d hidden')
    _rel(w_new.grad, w64.grad, 2e-2, f'{mode} fused d weight')
    ops.check_status()
