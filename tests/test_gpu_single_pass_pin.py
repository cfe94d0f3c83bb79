"""K1f (csrc/logprob_fused.cu), every entry point through the C ABI, against float64 on guard-banded buffers (run on an
H100: `pytest -m gpu`).

The cases and their geometry are tests/test_cpu_single_pass_pin.py's CASES: every (T, FAITHFUL, ENT, EGRAD, PM)
instantiation, production and crossover vocabularies, ring-stage edges, tiny vocabularies, work lists shorter than
the grid, around multiples of it and over three rounds, Z = 0 and Z >> scored, phase-mismatched logits / tile pairs,
head peels, pitched tiles, every row plan.

Every output lives between SENTINEL guard bands and starts as POISON: the gradient tile (Guarded, pad columns
included), the log-probs, the entropy, stat_max / stat_logsum, GRPO's row_end / total and the row scratch, which is
allocated at exactly the size include/aa_b200.h documents for the entry point.  After each launch every guard is
bit for bit unchanged, every element the contract writes holds no POISON and every element it does not write still
does.

References are plain float64 of the same logits (no other kernel):
  * log-probs: F32 mode within DESIGN section 4's fp32 bar, FAITHFUL within 1 ulp of the output dtype; stat_max is the
    row max, stat_max + stat_logsum the log-sum-exp (2e-5); the entropy within 1e-4 (test_gpu_entropy's bar);
  * g = d loss / d log-prob from the ports (ppo_objective_port, kl_loss_port, policy_loss_port, kl_objective_port,
    oracle.ref_port.grpo_loss) evaluated on the kernel's OWN log-probs -- in float64 for F32 mode, in eager ATen at the
    kernel's dtypes for FAITHFUL (the ports round where the kernels round); g_H from the aggregation's count;
  * the tile: test_gpu_entropy_bonus._tile64's g (onehot - p) - g_H p (l + H) (FAITHFUL: the rounded log-softmax) at
    _close's bar, plus G_ERR (below) times |onehot - p|; rows that carry no gradient (unscored, masked-off or after a
    completion's eos, g == 0 without g_H) are exactly 0;
  * the g each row's tile implies, -tile_k / p_k - g_H (l_k + H) averaged over the row's columns k != label (the
    tile's rounding errors average out), within a quarter ulp of the port's g in FAITHFUL with 16-bit log-probs -- the
    kernel's g is a 16-bit number there, so a one-ulp slip in a rounding of the coefficient chain shows -- and within
    G_ERR otherwise;
  * the work list: record s of the row scratch holds the tile row slot_order (the prep kernel's order, restated in
    tests/test_cpu_single_pass_pin.py) puts at s, and the zero-row mark exactly on the rows without a log-prob.
"""
from __future__ import annotations

import pytest
import torch

import kl_loss_port
import kl_objective_port
import policy_loss_port
import ppo_objective_port
from align_anything_b200 import _lib as Lb
from oracle import ref_port as O
from test_cpu_single_pass_pin import CASE_IDS, CASES, ENTRIES, IGNORE, entropy_grad_rows, entry_flags, slot_order
from test_gpu_entropy import entropy64
from test_gpu_entropy_bonus import EPS, _tile64
from test_gpu_logprob_tiles import INT, POISON, SENTINEL, Guarded, _half_ulp, _status_take
from test_gpu_parity import assert_close_f32, ops  # noqa: F401

pytestmark = pytest.mark.gpu

DEV = 'cuda'
TORCH_DT = {'bf16': torch.bfloat16, 'f16': torch.float16, 'f32': torch.float32}
AGG = {'seq-mean-token-mean': 0, 'token-mean': 1, 'seq-mean-token-sum-norm': 2}
EST = {'k1': 0, 'k2': 1, 'k3': 2}
PM = {'cispo': 3, 'sapo': 4}  # AA_PM_*
TAU = (1.0, 1.05)
BETA = 0.04
LOSS_SCALE = 0.5
# log-ratios lp - old placed on purpose: both sides of 1 - 0.2, 1 + 0.2, 1 + 0.28 and the dual-clip factor 3, each at
# least 0.03 away from the bound in log space -- more than the 16-bit rounding of lp, old and lp - old can move it
DELTAS = (-0.5, -0.3, -0.12, 0.0, 0.1, 0.215, 0.4, 1.4)
ADVS = (1.5, -0.75, 2.0, -1.25, 0.5, -2.0)
# G_ERR: how far the kernel's fp32 g may sit from the port's.  FAITHFUL with a 16-bit log-prob dtype: one unit in the
# last place of that dtype (the port rounds where the kernel rounds; only exp's last fp32 bit can move a rounding).
# Otherwise (fp32 arithmetic against float64): 2^-16 relative plus 2^-20 of the case's largest |g| (the k3 KL term
# subtracts two terms of g's size).
G_REL_F32, G_FLOOR_F32 = 2.0 ** -16, 2.0 ** -20
# the implied-g check's allowance for the error all columns of a row share (measured on the H100: up to 8e-5 of the
# row's factor with 16-bit tiles); with a quarter ulp it stays under half an ulp of a 16-bit g, so a one-ulp slip in g
# fails
BIAS = 2.0 ** -11


class _Tile(Guarded):
    """Guarded with the tile starting `shift` elements past a 16-byte boundary."""

    def __init__(self, rows, V, pitch, dtype, shift):
        super().__init__(rows, V, pitch, dtype)
        if shift:
            self.guard += shift
            self.bits.fill_(SENTINEL[self.esz])
            self.bits.as_strided((rows, V), (pitch, 1), self.guard).fill_(POISON[self.esz])
            self.fresh = self.bits.clone()
            self.tile = self.buf.as_strided((rows, V), (pitch, 1), self.guard)


class _Band:
    """n elements between 64-element SENTINEL guard bands (256 bytes for 4-byte elements: the interior stays 16-byte
    aligned); the interior starts as POISON."""
    G = 64

    def __init__(self, n, dtype):
        self.n = n
        self.buf = torch.empty(n + 2 * self.G, dtype=dtype, device=DEV)
        esz = self.buf.element_size()
        self.bits = self.buf.view(INT[esz])
        self.bits.fill_(SENTINEL[esz])
        self.bits[self.G:self.G + n].fill_(POISON[esz])
        self.poison = POISON[esz]
        self.fresh = self.bits.clone()
        self.t = self.buf[self.G:self.G + n]

    def ptr(self):
        return self.t.data_ptr()

    def check(self, what, written=None, guards_only=False):
        """Guards unchanged; `written` (bool over the interior, None: all): no POISON there, POISON elsewhere."""
        G, n = self.G, self.n
        assert torch.equal(self.bits[:G], self.fresh[:G]) and torch.equal(self.bits[G + n:], self.fresh[G + n:]), \
            f'{what}: a guard changed'
        if guards_only:
            return
        inner = self.bits[G:G + n]
        if written is None:
            written = torch.ones(n, dtype=torch.bool, device=DEV)
        assert not bool((inner[written] == self.poison).any()), f'{what}: an element was not written'
        assert bool((inner[~written] == self.poison).all()), f'{what}: an element outside the contract was written'


def _scratch_bytes(name, n_tile, n_seg):
    """include/aa_b200.h: 48 bytes per tile row, plus 4 bytes per segment (_entropy, _obj) or 8 (_kl, _pm)."""
    per_seg = {'aa_logprob_actor_fused_entropy': 4, 'aa_logprob_actor_fused_obj': 4, 'aa_logprob_actor_fused_kl': 8,
               'aa_logprob_actor_fused_pm': 8}.get(name, 0)
    return 48 * n_tile + per_seg * n_seg


class Run:
    """One case's inputs (built deterministically), the launch and its outputs."""

    def __init__(self, ops, case):
        self.case = c = case
        dt = self.dt = TORCH_DT[c.dt]
        self.faithful = c.mode == 'faithful'
        self.lp_dt = dt if (self.faithful and c.kind != 1) else torch.float32
        V, rows = c.V, c.rows()
        self.rows = rows
        k = len(rows)
        lpitch, loff, gpitch, gshift = c.pitches()
        gen = torch.Generator().manual_seed(sum(map(ord, c.id)))
        R = c.n_tile
        x = (torch.randn(loff + R * lpitch + 16, generator=gen) * 2.0).to(DEV)
        X = x.as_strided((R, V), (lpitch, 1), loff)
        # labels: edge columns from the case, random elsewhere; GRPO's eos only where the case puts it
        labels = torch.randint(0, V, c.label_shape(), generator=gen)
        flat = labels.view(-1)
        eos = c.eos_id()
        if c.kind >= 2:
            flat[flat == eos] = (eos + 1) % V
        for i, y in c.special_labels().items():
            flat[rows[i].lab] = y
        if c.kind >= 2:
            flat[flat == eos] = (eos + 1) % V
            for b, e in enumerate(c.eos):
                if e >= 0:
                    flat[b * c.K + e] = eos
        for i in c.ignored():
            flat[i] = IGNORE
        self.y = torch.tensor([int(flat[r.lab]) for r in rows], dtype=torch.int64)
        self.ignored = self.y == IGNORE
        self.oob = ((self.y < 0) | (self.y >= V)) & ~self.ignored
        tr = torch.tensor([r.tile_row for r in rows], dtype=torch.int64, device=DEV)
        self.tile_rows = tr
        y_safe = torch.where(self.oob | self.ignored, torch.zeros_like(self.y), self.y).to(DEV)
        self.y_safe = y_safe
        # the label's logit lifted to the row's log-sum-exp + u, u in [-1, 2): log-probs in [-1.4, -0.1], where a 16-bit
        # log-prob has the resolution DELTAS needs; a few rows with a -inf logit every fifth column
        with torch.no_grad():
            Xs = X[tr]
            ninf = torch.tensor([i % 13 == 4 for i in range(k)], device=DEV) & (V > 5)
            Xs[ninf, ::5] = float('-inf')
            lse = torch.logsumexp(Xs.double(), -1)
            u = torch.rand(k, generator=gen).to(DEV) * 3.0 - 1.0
            lifted = (lse + u).float()
            live = (~(self.oob | self.ignored)).to(DEV)
            Xs[torch.arange(k, device=DEV)[live], y_safe[live]] = lifted[live]
            X[tr] = Xs
        self.lbuf = x.to(dt)
        self.logits = self.lbuf.as_strided((R, V), (lpitch, 1), loff)
        self.labels = labels.to(DEV)
        self.lpitch, self.loff, self.gpitch, self.gshift = lpitch, loff, gpitch, gshift
        # float64 log-probs of the rounded logits (the old log-probs are placed around them)
        X64 = self.logits[tr].double()
        lse64 = torch.logsumexp(X64, -1)
        self.lse64 = lse64
        self.lp64 = X64.gather(-1, y_safe[:, None]).squeeze(-1) - lse64
        self.lp64[self.oob.to(DEV)] = float('nan')
        n_seg, W = c.n_seg, c.W
        self.seg = torch.tensor([r.seg for r in rows], dtype=torch.int64, device=DEV)
        self.jj = torch.tensor([r.j for r in rows], dtype=torch.int64, device=DEV)
        self.out = torch.tensor([r.out for r in rows], dtype=torch.int64, device=DEV)
        self.on = torch.tensor([c.on(r) for r in rows], dtype=torch.bool, device=DEV)
        n_out = c.B * c.S if c.kind == 1 else n_seg * W
        self.n_out = n_out
        delta = torch.tensor([DELTAS[(r.seg * 3 + r.j) % len(DELTAS)] for r in rows], dtype=torch.float64, device=DEV)
        lp_guess = torch.nan_to_num(self.lp64, nan=-1.0)
        # plans
        if c.plan == 'dense':
            self.plan = ops._dense_actor_plan(c.B, c.S, c.start, c.S * lpitch, lpitch, c.S, DEV)
        elif c.plan in ('tail', 'grpo'):
            lens = c.lens if c.plan == 'tail' else (c.K,) * c.B
            self.plan = ops._tail_plan(tuple(lens), c.S, c.S * lpitch, lpitch, W, 0, c.shift, W, DEV)
        elif c.plan == 'device':
            dl = ops.DeviceLens(torch.tensor(c.lens, dtype=torch.int32, device=DEV), W)
            self.plan = ops.DevicePlan(dl, c.S, c.S * lpitch, lpitch, c.S, c.S, 0, -1, W)
        else:
            self.plan = ops.RowPlan([0], [0], [0], [R], [0], (c.B, c.S), R, DEV)
        assert self.plan.n_seg == n_seg and self.plan.n_tile_rows == R
        # loss inputs
        if c.kind == 0:
            oldb = torch.randn(n_seg, W + 5, generator=gen).to(DEV) - 1.0
            oldb[self.seg, self.jj] = (lp_guess - delta).float()
            self.old = oldb.to(self.lp_dt)[:, :W]
            advb = torch.randn(n_seg, W + 3, generator=gen).to(DEV)
            advb[self.seg, self.jj] = torch.tensor([ADVS[(r.seg + 2 * r.j) % len(ADVS)] for r in rows], device=DEV)
            self.adv = advb.to(TORCH_DT[c.adv])[:, :W]
            maskb = torch.zeros(n_seg, W + 2, dtype=torch.bool, device=DEV)
            maskb[self.seg, self.jj] = self.on
            self.mask = maskb[:, :W]
            self.ref = (lp_guess + 0.3 * torch.randn(k, generator=gen, dtype=torch.float64).to(DEV))
            refb = torch.zeros(n_seg * W, dtype=torch.float64, device=DEV)
            refb[self.out] = self.ref
            self.ref = refb.view(n_seg, W).to(self.lp_dt)  # laid out like the log-probs
        elif c.kind >= 2:
            refb = torch.zeros(n_seg, W + 3, dtype=torch.float64, device=DEV)
            refb[self.seg, self.jj] = lp_guess + 0.3 * torch.randn(k, generator=gen, dtype=torch.float64).to(DEV)
            self.ref = refb.to(self.lp_dt)[:, :W]  # row stride K + 3: read at seg * ref_stride + j
            self.adv = torch.tensor([ADVS[b % len(ADVS)] for b in range(c.B)], dtype=torch.float32, device=DEV)
            polb = torch.zeros(n_seg * W, dtype=torch.float64, device=DEV)
            polb[self.out] = lp_guess - delta
            self.old_pol = polb.view(n_seg, W).to(self.lp_dt) if c.opts.get('old_pol') else None
            self.tokens = self.labels
            self.counted = torch.zeros(n_seg, W, dtype=torch.bool, device=DEV)
            for b, e in enumerate(c.row_end()):
                self.counted[b, :e] = True

    def launch(self, ops):
        c, o = self.case, self.case.opts
        name, kind, _ = ENTRIES[c.entry]
        k = len(self.rows)
        tile = self.tile = _Tile(c.n_tile, c.V, self.gpitch, self.dt, self.gshift)
        self.lp = _Band(self.n_out, self.lp_dt)
        self.ent = _Band(self.n_out, torch.float32) if 'ent' in o else None
        self.smax, self.slog = _Band(max(k, 1), torch.float32), _Band(max(k, 1), torch.float32)
        self.scratch = _Band(_scratch_bytes(name, c.n_tile, c.n_seg) // 4, torch.int32)
        sc = ops._device_scratch(torch.device(DEV))
        status = sc['status'].data_ptr()
        st = Lb.stream_ptr(torch.device(DEV))
        lib = Lb.lib()
        fn = getattr(lib, name)
        p = self.plan.ptrs()
        logits = self.lbuf.data_ptr() + self.loff * self.lbuf.element_size()
        mode = Lb.MODE_FAITHFUL if c.mode == 'faithful' else Lb.MODE_F32
        head = [logits, Lb.dtype_code(self.dt), self.lpitch, c.V, self.labels.data_ptr()]
        plan = [c.n_seg, p[0], p[1], p[2], p[3], p[4], c.n_tile]
        grad = [tile.tile.data_ptr(), self.gpitch, self.scratch.ptr()]
        coeff = float(o.get('ent') or 0.0)
        ent = self.ent.ptr() if self.ent is not None else None
        agg = AGG[o.get('agg', 'seq-mean-token-mean')]
        lo, hi, dual = o.get('lo', 0.2), o.get('hi', 0.2), o.get('dual', 0.0)
        est, kl_c = EST[o['kl'][0]] if 'kl' in o else EST['k3'], o['kl'][1] if 'kl' in o else 0.0
        _status_take()
        if kind == 0:
            a = head + plan + [self.lp.ptr(), Lb.dtype_code(self.lp_dt), self.smax.ptr(), self.slog.ptr(),
                               self.old.data_ptr(), self.old.stride(0), self.adv.data_ptr(), self.adv.stride(0),
                               Lb.dtype_code(self.adv.dtype), self.mask.data_ptr(), self.mask.stride(0), c.W]
            ref = self.ref.data_ptr() if 'kl' in o else None
            if name == 'aa_logprob_actor_fused':
                rc = fn(*a, 0.2, mode, *grad, status, st)
            elif name == 'aa_logprob_actor_fused_entropy':
                rc = fn(*a, 0.2, mode, *grad, status, coeff, ent, st)
            elif name == 'aa_logprob_actor_fused_obj':
                rc = fn(*a, lo, hi, dual, agg, mode, *grad, status, coeff, ent, st)
            elif name == 'aa_logprob_actor_fused_kl':
                rc = fn(*a, lo, hi, dual, agg, mode, *grad, status, coeff, ent, ref, kl_c, est, st)
            else:
                rc = fn(*a, hi, agg, PM[o['pm']], *TAU, mode, *grad, status, coeff, ent, ref, kl_c, est, st)
        elif kind == 1:
            self.coeff = _Band(1, torch.float32)
            rc = fn(*head, c.B * c.S, IGNORE, *plan, self.lp.ptr(), LOSS_SCALE, *grad, self.coeff.ptr(), status, st)
        else:
            self.row_end, self.total = _Band(c.B, torch.int32), _Band(1, torch.float32)
            counter = torch.zeros(1, dtype=torch.int32, device=DEV)
            a = head + plan + [self.lp.ptr(), Lb.dtype_code(self.lp_dt), self.ref.data_ptr(), self.ref.stride(0)]
            tok = [self.tokens.data_ptr(), self.tokens.stride(0), c.eos_id(), c.K]
            tail = [self.row_end.ptr(), self.total.ptr(), counter.data_ptr(), status]
            pol = self.old_pol.data_ptr() if self.old_pol is not None else None
            beta = kl_c if 'kl' in o else BETA
            if name == 'aa_logprob_grpo_fused':
                rc = fn(*a, self.adv.data_ptr(), *tok, beta, mode, *grad, *tail, st)
            elif name == 'aa_logprob_grpo_fused_entropy':
                rc = fn(*a, self.adv.data_ptr(), *tok, beta, mode, *grad, *tail, ent, st)
            elif name == 'aa_logprob_grpo_fused_entropy_grad':
                rc = fn(*a, self.adv.data_ptr(), *tok, beta, mode, *grad, *tail, ent, coeff, st)
            elif name == 'aa_logprob_grpo_fused_obj':
                rc = fn(*a, pol, self.adv.data_ptr(), *tok, beta, lo, hi, dual, agg, mode, *grad, *tail, ent, coeff, st)
            elif name == 'aa_logprob_grpo_fused_kl':
                rc = fn(*a, pol, self.adv.data_ptr(), *tok, beta, lo, hi, dual, agg, est, mode, *grad, *tail, ent,
                        coeff, st)
            else:
                rc = fn(*a, pol, self.adv.data_ptr(), *tok, beta, hi, agg, est, PM[o['pm']], *TAU, mode, *grad, *tail,
                        ent, coeff, st)
        Lb.check(rc)
        torch.cuda.synchronize()
        self.status = _status_take()

    # ---- the reference g = d loss / d log-prob, from the ports on the kernel's log-probs ----
    def g_ref(self, lp_k):
        """-> (g, g_H) float64 per scored row."""
        c, o = self.case, self.case.opts
        k = len(self.rows)
        if c.kind == 1:
            n_valid = int((~self.ignored).sum())
            g = torch.where(self.ignored.to(DEV), 0.0, -LOSS_SCALE / n_valid).double()
            return g, torch.zeros(k, dtype=torch.float64, device=DEV)
        cast = (lambda t: t) if self.faithful else (lambda t: t.double())
        lp_in = torch.zeros(c.n_seg * c.W, dtype=self.lp_dt, device=DEV)
        lp_in[self.out] = torch.nan_to_num(lp_k, nan=0.0).to(self.lp_dt)  # a NaN log-prob sits on a row without g
        lp = cast(lp_in.view(c.n_seg, c.W)).detach().requires_grad_(True)
        agg = o.get('agg', 'seq-mean-token-mean')
        lo, hi, dual = o.get('lo', 0.2), o.get('hi', 0.2), o.get('dual')
        if c.kind == 0:
            old, adv, mask, ref = cast(self.old), cast(self.adv), self.mask, cast(self.ref)
            if 'pm' in o:
                if 'kl' in o:
                    loss = policy_loss_port.actor_loss_kl(o['pm'], lp, old, adv, mask, agg, hi, *TAU, ref, o['kl'][1],
                                                          o['kl'][0])[2]
                else:
                    loss = policy_loss_port.actor_loss(o['pm'], lp, old, adv, mask, agg, hi, *TAU)
            elif 'kl' in o:
                loss = kl_loss_port.actor_loss(lp, old, adv, mask, lo, hi, dual, agg, ref, o['kl'][1], o['kl'][0])
            else:
                loss = ppo_objective_port.actor_loss(lp, old, adv, mask, lo, hi, dual, agg)
            counted = self.mask
        else:
            ref, adv = cast(self.ref), cast(self.adv).view(-1, 1)
            counted = self.counted
            beta = o['kl'][1] if 'kl' in o else BETA
            est = o['kl'][0] if 'kl' in o else 'k3'
            pol = cast(self.old_pol) if self.old_pol is not None else None
            if c.kind == 2:
                loss = O.grpo_loss(lp, ref, adv, self.tokens, 0, c.eos_id(), beta)
            elif 'pm' in o:
                loss = policy_loss_port.grpo_loss(o['pm'], lp, ref, pol, adv, counted, beta, agg, hi, *TAU, est)
            else:
                loss = kl_objective_port.grpo_loss(lp, ref, adv, counted, beta, est, pol, lo, hi, dual, agg)
        loss.backward()
        g = lp.grad.double()[self.seg, self.jj]
        ent, egrad, _ = entry_flags(c.entry)
        if egrad and o.get('ent'):
            gh = entropy_grad_rows(0 if c.kind == 0 else 2, agg, counted, o['ent'])[self.seg, self.jj]
        else:
            gh = torch.zeros(k, dtype=torch.float64, device=DEV)
        on = self.on if c.kind == 0 else counted[self.seg, self.jj]
        return torch.where(on, g, 0.0), torch.where(on, gh, 0.0)


def _check_tile(run, g, gh, g_err, g_tight, what):
    c, tile = run.case, run.tile
    dt, V = run.dt, c.V
    keep = tile.outside()
    assert torch.equal(tile.bits[keep], tile.fresh[keep]), f'{what}: a guard or pad sentinel changed'
    assert not bool((tile.row_bits(slice(None)) == POISON[tile.esz]).any()), f'{what}: a tile element was not written'
    scored = torch.zeros(c.n_tile, dtype=torch.bool, device=DEV)
    scored[run.tile_rows] = True
    zero = tile.tile[~scored]
    assert bool((zero == 0).all()), f'{what}: an unscored tile row is not zero'
    dead = (g == 0) & (gh == 0)
    if bool(dead.any()):
        assert bool((tile.tile[run.tile_rows[dead]] == 0).all()), f'{what}: a row without gradient is not zero'
    live = torch.nonzero(~dead).flatten()
    fdt = dt if (run.faithful and dt != torch.float32 and c.kind != 1) else None
    oob = run.oob.to(DEV)
    for s in range(0, live.numel(), 32):
        i = live[s:s + 32]
        x = run.logits[run.tile_rows[i]].float()
        want = _tile64(x, run.y_safe[i], g[i], gh[i], fdt)
        lp = x.double() - torch.logsumexp(x.double(), -1, keepdim=True)
        if fdt is not None:
            lp = lp.to(fdt).double()
        onehot = torch.nn.functional.one_hot(run.y_safe[i], V).double()
        onehot[oob[i]] = 0.0
        want[oob[i], 0] -= g[i][oob[i]]  # no one-hot term for a label outside [0, V)
        got = tile.tile[run.tile_rows[i]].double()
        # test_gpu_entropy_bonus._close's bar, plus the error allowed in g times |onehot - p|
        # the floor is relative to the larger of the row's largest element and |g|, |g_H| (a one-column row: want == 0)
        scale = torch.maximum(want.abs().amax(-1), torch.maximum(g[i].abs(), gh[i].abs()))[:, None]
        tol = EPS[dt] * want.abs() + max(EPS[dt], 2e-5) * scale + 1e-30 + g_err[i][:, None] * (onehot - lp.exp()).abs()
        err = (got - want).abs()
        bad = ~(err <= tol)
        assert not bool(bad.any()), (f'{what}: {int(bad.sum())} tile elements beyond tolerance in rows '
                                     f'{run.tile_rows[i][bad.any(-1)].tolist()[:8]}, max err / row scale '
                                     f'{float((err / scale.clamp_min(1e-30)).max()):.3e}')
        # the g the row implies: each column k != label gives -tile_k / p_k - g_H (l_k + H) up to the tile's rounding
        # (relative EPS, symmetric), so their mean sits within 6 sigma of the kernel's g, plus BIAS of the row's factor
        # |g| + |g_H| mean |l + H| for what every column shares (the kernel's fp32 max, log-sum and H).  Columns whose
        # tile value is 16-bit subnormal or 0 and -inf logits are left out.  Checked: rows with at least 64 usable
        # columns whose g is at least the entropy term |g_H| mean |l + H| (the check is about g's rounding; rows the
        # entropy term dominates are held by the element-wise bar above)
        lc = torch.clamp(lp, min=-3.0e38) + entropy64(x)[:, None]
        use = (onehot == 0) & (lp.exp() > 0) & (got.abs() >= torch.finfo(dt).tiny) & torch.isfinite(got)
        use[torch.arange(use.size(0), device=DEV), run.y_safe[i]] = False
        n = use.sum(-1)
        gk = torch.where(use, -got / lp.exp().clamp_min(1e-300) - gh[i][:, None] * lc, 0.0)
        g_imp = gk.sum(-1) / n.clamp_min(1)
        lca = torch.where(use, lc.abs(), 0.0)
        factor = g[i].abs() + gh[i].abs() * lca.sum(-1) / n.clamp_min(1)
        noise = (6 * EPS[dt] / torch.sqrt(3.0 * n.clamp_min(1)) + BIAS) * factor
        ent_term = gh[i].abs() * lca.sum(-1) / n.clamp_min(1)
        far = ((g_imp - g[i]).abs() > g_tight[i] + noise + 1e-30) & (n >= 64) & (g[i].abs() >= ent_term)
        assert not bool(far.any()), (f'{what}: the g implied by rows {run.tile_rows[i][far].tolist()[:8]} is '
                                     f'{g_imp[far].tolist()[:4]}, the port gives {g[i][far].tolist()[:4]}')


@pytest.mark.parametrize('case', CASES, ids=CASE_IDS)
def test_single_pass_against_float64(ops, case):
    run = Run(ops, case)
    run.launch(ops)
    c, o = case, case.opts
    what = case.id
    k = len(run.rows)
    # ---- outputs and guards ----
    written = torch.zeros(run.n_out, dtype=torch.bool, device=DEV)
    written[run.out[~run.ignored.to(DEV)]] = True
    run.lp.check(f'{what} log-probs', written)
    if run.ent is not None:
        run.ent.check(f'{what} entropy', written)
    run.scratch.check(f'{what} row scratch', guards_only=True)  # the per-segment words are written only when used
    # the work list (FusedRec, 48 bytes: g_row at bytes 8-15, y at bytes 36-39) against slot_order
    n = c.n_tile
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    want = torch.empty(n, dtype=torch.int64)
    want[torch.tensor(slot_order(c, min(sms, n)))] = torch.arange(n)
    rec = run.scratch.t[:12 * n]
    assert torch.equal(rec.view(torch.int64).view(n, 6)[:, 1].cpu(), want), f'{what}: work-list order'
    scored = torch.zeros(n, dtype=torch.bool)
    scored[run.tile_rows[~run.ignored.to(DEV)].cpu()] = True
    assert torch.equal((rec.view(n, 12)[:, 9] == -2).cpu(), ~scored[want]), f'{what}: zero-row records'
    if c.kind == 0:
        run.smax.check(f'{what} stat_max', torch.arange(run.smax.n, device=DEV) < k)
        run.slog.check(f'{what} stat_logsum', torch.arange(run.slog.n, device=DEV) < k)
    if c.kind == 1:
        run.coeff.check(f'{what} coeff')
    if c.kind >= 2:
        run.row_end.check(f'{what} row_end')
        run.total.check(f'{what} total')
        assert run.row_end.t.tolist() == c.row_end(), what
        assert float(run.total.t) == float(sum(c.row_end())), what
    assert bool(run.status & Lb.STATUS_LABEL_OOB) == bool(run.oob.any()), f'{what}: status {run.status:#x}'
    # ---- log-probs, statistics, entropy against float64 ----
    lp_k = run.lp.t[run.out]
    valid = ~run.ignored.to(DEV)
    lp64 = run.lp64
    if run.lp_dt == torch.float32:
        assert_close_f32(lp_k[valid], lp64[valid].float(), what=f'{what} log-probs')
    else:
        assert torch.equal(torch.isnan(lp_k), torch.isnan(lp64)), f'{what}: NaN pattern of the log-probs'
        fin = ~torch.isnan(lp64)
        err = (lp_k[fin].double() - lp64[fin]).abs()
        assert bool((err <= 2 * _half_ulp(lp64[fin], run.lp_dt)).all()), f'{what}: a log-prob beyond 1 ulp'
    if c.kind == 0:
        x = run.logits[run.tile_rows].float()
        assert torch.equal(run.smax.t[:k], x.amax(-1)), f'{what}: stat_max'
        st = (run.smax.t[:k] + run.slog.t[:k]).double()
        assert bool(((st - run.lse64).abs() <= 2e-5 * run.lse64.abs().clamp(min=1.0)).all()), f'{what}: stat_logsum'
    if run.ent is not None:
        h64 = torch.cat([entropy64(run.logits[run.tile_rows[s:s + 32]]) for s in range(0, k, 32)])
        assert float((run.ent.t[run.out].double() - h64).abs().max()) <= 1e-4, f'{what}: entropy'
    # ---- the tile ----
    g, gh = run.g_ref(lp_k)
    gmax = float(g.abs().max()) if k else 0.0
    if run.lp_dt != torch.float32 and run.faithful:
        g_err = EPS[run.lp_dt] * g.abs()
        g_tight = 0.5 * _half_ulp(g, run.lp_dt)  # a quarter ulp: the kernel's g and the port's are 16-bit numbers
    else:
        g_err = g_tight = G_REL_F32 * g.abs() + G_FLOOR_F32 * gmax
    on = g != 0
    # the clipped objective without a KL term: clipped tokens carry g == 0 (with the entropy bonus, g_H alone)
    if c.kind == 0 and 'lo' in o and 'kl' not in o and int(run.on.sum()) >= 12:
        assert bool(((g == 0) & run.on).any()), f'{what}: the case has no clipped token'
        if bool((gh != 0).any()):
            assert bool(((g == 0) & (gh != 0)).any()), f'{what}: no clipped token with an entropy gradient'
    _check_tile(run, g, gh, g_err, g_tight, what)
