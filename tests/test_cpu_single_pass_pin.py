"""The cases tests/test_gpu_single_pass_pin.py runs K1f (csrc/logprob_fused.cu) on, and the references it holds the
kernel to, checked without a GPU.

The case list lives here so that both files read the same one:
  * each case's geometry -- which tile rows are scored, each row's 16-byte phase in the logits and in the tile, its head
    peel, its body vectors and the stages of its last phase-A fold -- restated from the row plan in plain Python;
  * the work list the prep kernel builds (fused_actor_prep_kernel's `slot`) restated in Python and shown to be a
    permutation that keeps the scored rows in order;
  * every property a case claims (a stage edge, a phase mismatch, Z = 0, n_work around a multiple of the grid, a label
    in a peel, ...) shown to hold;
  * the instantiations `launch_fused_of` can select, each covered, the ones the trainers reach at a production V;
  * the per-segment coefficients of the prep kernel (actor_row_coeff, the token-mean coefficient, kl_term_coeff, the
    entropy gradient g_H and GRPO's aggregation coefficient) restated in float64 against autograd of the ports.
"""
from __future__ import annotations

import dataclasses
import itertools

import pytest
import torch

import kl_loss_port
import policy_loss_port
import ppo_objective_port

CONSUMERS, UNROLL = 992, 2       # logprob_fused.cu launch_fused_kernel
STAGE_VECS = CONSUMERS * UNROLL  # 16-byte vectors per ring stage; phase A folds two stages at a time
SMS = 132                        # H100 SXM: the persistent grid is min(SM count, n_work)
ESZ = {'bf16': 2, 'f16': 2, 'f32': 4}
PRODUCTION_V = (152064, 128256, 128257)
CROSSOVER_V = {'bf16': 98304, 'f32': 49152}  # ops._FUSED_MIN_ROW_BYTES

# entry variants: (C entry point, kind, flags (ENT, EGRAD, PM) the launch selects, options)
#   ent: entropy coefficient (None: no entropy buffer);  lo / hi / dual / agg: objective;  kl: (estimator, coeff)
#   pm: 'cispo' / 'sapo';  old_pol: GRPO's rollout-time log-probs given (False: NULL, the ratio is 1)
ENTRIES = {
    'actor': ('aa_logprob_actor_fused', 0, dict()),
    'actor_ent0': ('aa_logprob_actor_fused_entropy', 0, dict(ent=0.0)),
    'actor_ent': ('aa_logprob_actor_fused_entropy', 0, dict(ent=0.05)),
    'obj_hi': ('aa_logprob_actor_fused_obj', 0, dict(lo=0.2, hi=0.28)),
    'obj_dual_tm': ('aa_logprob_actor_fused_obj', 0, dict(lo=0.2, hi=0.2, dual=3.0, agg='token-mean')),
    'obj_dual_ent': ('aa_logprob_actor_fused_obj', 0, dict(lo=0.2, hi=0.28, dual=3.0, ent=0.05)),
    'obj_tm_ent': ('aa_logprob_actor_fused_obj', 0, dict(lo=0.2, hi=0.28, agg='token-mean', ent=0.05)),
    'kl_k1': ('aa_logprob_actor_fused_kl', 0, dict(lo=0.2, hi=0.28, kl=('k1', 0.1))),
    'kl_k2': ('aa_logprob_actor_fused_kl', 0, dict(lo=0.2, hi=0.2, agg='token-mean', kl=('k2', 0.25), ent=0.05)),
    'kl_k3': ('aa_logprob_actor_fused_kl', 0, dict(lo=0.2, hi=0.28, dual=3.0, kl=('k3', 0.1), ent=0.0)),
    'pm_cispo': ('aa_logprob_actor_fused_pm', 0, dict(pm='cispo', hi=0.28)),
    'pm_sapo': ('aa_logprob_actor_fused_pm', 0, dict(pm='sapo', agg='token-mean')),
    'pm_cispo_ek': ('aa_logprob_actor_fused_pm', 0, dict(pm='cispo', hi=0.28, agg='token-mean', ent=0.05,
                                                          kl=('k3', 0.1))),
    'pm_sapo_ek': ('aa_logprob_actor_fused_pm', 0, dict(pm='sapo', ent=0.05, kl=('k2', 0.1))),
    'ce': ('aa_logprob_ce_fused', 1, dict()),
    'grpo': ('aa_logprob_grpo_fused', 2, dict()),
    'grpo_ent': ('aa_logprob_grpo_fused_entropy', 2, dict(ent=0.0)),
    'grpo_egrad': ('aa_logprob_grpo_fused_entropy_grad', 2, dict(ent=0.1)),
    'gobj_nopol': ('aa_logprob_grpo_fused_obj', 3, dict(lo=0.2, hi=0.28, agg='token-mean')),
    'gobj_pol': ('aa_logprob_grpo_fused_obj', 3, dict(lo=0.2, hi=0.28, dual=3.0, agg='seq-mean-token-mean',
                                                      old_pol=True)),
    'gobj_norm_ent': ('aa_logprob_grpo_fused_obj', 3, dict(lo=0.2, hi=0.2, agg='seq-mean-token-sum-norm', old_pol=True,
                                                           ent=0.05)),
    'gobj_ent0': ('aa_logprob_grpo_fused_obj', 3, dict(lo=0.2, hi=0.28, old_pol=True, ent=0.0)),
    'gkl_k1': ('aa_logprob_grpo_fused_kl', 3, dict(lo=0.2, hi=0.28, kl=('k1', 0.04), old_pol=True)),
    'gkl_k2': ('aa_logprob_grpo_fused_kl', 3, dict(lo=0.2, hi=0.28, kl=('k2', 0.04), agg='seq-mean-token-mean')),
    'gkl_k3': ('aa_logprob_grpo_fused_kl', 3, dict(lo=0.2, hi=0.28, dual=3.0, kl=('k3', 0.04), old_pol=True,
                                                   ent=0.05)),
    'gpm_cispo': ('aa_logprob_grpo_fused_pm', 3, dict(pm='cispo', hi=0.28, old_pol=True, ent=0.05)),
    'gpm_sapo': ('aa_logprob_grpo_fused_pm', 3, dict(pm='sapo', old_pol=True, ent=0.05, kl=('k2', 0.04))),
    'gpm_cispo_ent0': ('aa_logprob_grpo_fused_pm', 3, dict(pm='cispo', hi=0.28, old_pol=True, ent=0.0)),
    'gpm_sapo_noent': ('aa_logprob_grpo_fused_pm', 3, dict(pm='sapo', agg='seq-mean-token-mean', old_pol=True)),
}


def entry_flags(entry):
    """(ENT, EGRAD, PM) of the kernel `launch_fused_of` selects for this entry variant."""
    name, kind, o = ENTRIES[entry]
    ent = o.get('ent')
    pm = 'pm' in o
    if kind == 1 or ent is None:
        return (False, False, pm)
    if kind == 0:  # logprob_actor_fused: an entropy buffer always runs the entropy-gradient kernel
        return (True, True, pm)
    if name == 'aa_logprob_grpo_fused_entropy':
        return (True, False, pm)
    if name == 'aa_logprob_grpo_fused_entropy_grad':
        return (True, True, pm)
    return (True, ent != 0.0, pm)


def instantiation(case):
    """(T, FAITHFUL, ENT, EGRAD, PM) of the kernel a case runs (cross-entropy always runs F32 mode; fp32 logits have
    no FAITHFUL instantiation of their own)."""
    kind = ENTRIES[case.entry][1]
    faithful = case.mode == 'faithful' and ESZ[case.dt] == 2 and kind != 1
    return (case.dt, faithful) + entry_flags(case.entry)


def all_instantiations():
    flags = {entry_flags(e) for e in ENTRIES}
    assert len(flags) == 6
    return {(dt, f) + fl for dt in ESZ for f in ((False, True) if ESZ[dt] == 2 else (False,)) for fl in flags}


@dataclasses.dataclass(frozen=True)
class Row:
    seg: int
    j: int          # index of the row among its segment's scored rows
    tile_row: int
    lab: int        # flat index into the labels tensor
    out: int        # flat index into the (n_seg, W) outputs


@dataclasses.dataclass(frozen=True)
class Case:
    """One K1f launch.  plan: 'dense' (the dense actor plan, rows [start, S - 1)), 'tail' (right-aligned tails of
    `lens` rows, first row S - len + shift), 'device' (DevicePlan from device lengths, < 0 clamps to 0), 'ce' (the
    dense single-segment RowPlan of causal_lm_loss), 'grpo' (the tail plan of the GRPO node: K rows per sample).
    layout: 'contig' | 'pitch' (logits and tile share a pitch > V) | 'odd' (logits base and tile one element off:
    same phases, non-empty head peels) | 'mismatch' (logits pitch V, tile pitch V + 1: the 16-byte phases of a
    row differ unless the row index is a multiple of 16 / element size, and the tile rows have head peels)."""
    entry: str
    dt: str
    mode: str
    V: int
    plan: str
    B: int
    S: int
    layout: str = 'contig'
    lens: tuple = ()
    start: int = 1
    K: int = 0
    eos: tuple = ()
    shift: int = -1
    oob: bool = False
    claims: tuple = ()
    adv: str = 'f32'  # kind 0: the advantages' dtype (FAITHFUL rounds the promoted products to it when it is 16-bit)

    @property
    def id(self):
        adv = '' if self.adv == 'f32' else f'-adv{self.adv}'
        return f'{self.entry}-{self.dt}-{self.mode}-V{self.V}-{self.plan}-{self.layout}-{self.B}x{self.S}{adv}'

    @property
    def kind(self):
        return ENTRIES[self.entry][1]

    @property
    def opts(self):
        return ENTRIES[self.entry][2]

    @property
    def esz(self):
        return ESZ[self.dt]

    @property
    def q(self):
        return 16 // self.esz

    def pitches(self):
        """-> (logits pitch, logits base offset, tile pitch, tile base offset), in elements."""
        V, q = self.V, self.q
        if self.layout == 'contig':
            return V, 0, V, 0
        if self.layout == 'pitch':
            P = (V + q - 1) // q * q + q
            return P, 0, P, 0
        if self.layout == 'odd':
            return V, 1, V, 1
        assert self.layout == 'mismatch'
        return V, 0, V + 1, 0

    @property
    def n_seg(self):
        return 1 if self.plan == 'ce' else self.B

    @property
    def n_tile(self):
        return self.B * self.S

    @property
    def W(self):
        """Width of the (n_seg, W) outputs (ce: (B, S))."""
        if self.plan == 'dense':
            return self.S - 1 - self.start
        if self.plan == 'tail':
            return max(max(self.lens), 1)
        if self.plan == 'device':
            return self.S - 1
        if self.plan == 'grpo':
            return self.K
        return self.S

    def label_shape(self):
        if self.plan in ('tail', 'grpo'):
            return (self.B, self.W)
        return (self.B, self.S)

    def seg_spans(self):
        """-> [(first tile row, scored rows)] per segment."""
        S, B = self.S, self.B
        if self.plan == 'dense':
            return [(b * S + self.start, self.W) for b in range(B)]
        if self.plan == 'tail':
            return [(b * S + S - r + self.shift, r) for b, r in enumerate(self.lens)]
        if self.plan == 'device':
            out = []
            for b, r in enumerate(self.lens):
                r = max(0, min(r, S - 1))
                out.append((b * S + S - r - 1, min(r, self.W)))
            return out
        if self.plan == 'grpo':
            return [(b * S + S - self.K - 1, self.K) for b in range(B)]
        return [(0, B * S)]

    def rows(self):
        out = []
        for seg, (first, n) in enumerate(self.seg_spans()):
            for j in range(n):
                if self.plan == 'device':
                    r = max(0, min(self.lens[seg], self.S - 1))
                    lab = seg * self.S + self.S - r + j
                elif self.plan == 'dense':
                    lab = seg * self.S + self.start + 1 + j
                elif self.plan == 'ce':
                    lab = j
                else:
                    lab = seg * self.W + j
                out.append(Row(seg, j, first + j, lab, j if self.plan == 'ce' else seg * self.W + j))
        return out

    # ---- the geometry each row has inside the kernel ----
    def row_geometry(self, tile_row):
        """-> (same_phase, head, nvec, tail0) of a scored row, as the kernel's consumers compute them."""
        lp, lo, gp, go = self.pitches()
        x, g = (lo + tile_row * lp) * self.esz, (go + tile_row * gp) * self.esz
        mis = (x % 16) // self.esz
        head = min(self.q - mis, self.V) if mis else 0
        nvec = (self.V - head) // self.q
        return (x - g) % 16 == 0, head, nvec, head + nvec * self.q

    def masked_off(self, seg, j):
        """kind 0: the mask bit of token (seg, j) is off.  Sample 1 (of three or more) has no masked-in token."""
        if self.kind != 0:
            return False
        return (self.B >= 3 and seg == 1) or (seg * 5 + j) % 7 == 3

    def row_end(self):
        """GRPO: counted tokens per sample (up to and including the first eos)."""
        return [self.K if e < 0 else e + 1 for e in self.eos]

    def on(self, r):
        if self.kind == 0:
            return not self.masked_off(r.seg, r.j)
        if self.kind >= 2:
            return r.j < self.row_end()[r.seg]
        return True

    def special_labels(self):
        """{row index: label column} of the rows whose labels sit at the edges (the rest are random)."""
        out = {}
        rows = self.rows()
        stage = STAGE_VECS * self.q
        for i, r in enumerate(rows):
            same, head, nvec, tail0 = self.row_geometry(r.tile_row)
            pick = {0: 0, 1: self.V - 1, 2: head - 1 if head > 0 else None, 3: tail0 if tail0 < self.V else None,
                    4: head + stage if head + stage < self.V else None,
                    5: head + stage - 1 if head + stage - 1 < tail0 else None,
                    6: head + 2 * stage if head + 2 * stage < tail0 else None}.get(i % 11)
            if pick is not None:
                out[i] = pick
        if self.oob:
            # one label above the vocabulary: on a masked-off / post-eos row (its log-prob is NaN, its gradient row 0)
            # or, for the cross-entropy, on a valid row (its row is -g * softmax)
            cand = [i for i, r in enumerate(rows) if not self.on(r)] if self.kind != 1 else [len(rows) // 2 + 1]
            out[cand[len(cand) // 2]] = self.V + 3
        return out

    def eos_id(self):
        return 2

    def ignored(self):
        """cross-entropy: flat label indices set to ignore_index."""
        if self.kind != 1:
            return set()
        sp = self.special_labels()
        return {r.lab for i, r in enumerate(self.rows()) if i % 7 == 5 and i not in sp}


IGNORE = -100


def C(entry, dt, mode, V, plan, B, S, **kw):
    return Case(entry, dt, mode, V, plan, B, S, **kw)


_TAIL = (5, 0, 9, 3, 11, 1)   # lengths of a tail plan: a length of 0, short and long tails
_DEV = (7, -2, 11, 0, 4, 11)  # device lengths: -2 clamps to 0
BF, H, F = 'bf16', 'f16', 'f32'
FA, F3 = 'faithful', 'f32'
# bf16 stage edges: one stage = 15872 elements; with head 0 the last fold's second stage is empty (one stage - 1
# vector, two stages + 1 vector), partial (one stage + 1 vector) or full (two stages)
CASES = [
    # ---- production vocabularies: every instantiation the trainers reach (bf16 / fp32, both modes, each flag set) --
    C('actor', BF, FA, 152064, 'dense', 3, 12, claims=('prod_v', 'empty_sample')),
    C('actor_ent', BF, FA, 152064, 'tail', 6, 13, lens=_TAIL, claims=('prod_v', 'len0', 'many_seg')),
    C('pm_sapo', BF, FA, 128256, 'dense', 3, 10, claims=('prod_v',)),
    C('pm_cispo_ek', BF, FA, 128257, 'device', 6, 12, lens=_DEV, claims=('prod_v', 'clamp', 'len0')),
    C('grpo_ent', BF, FA, 152064, 'grpo', 4, 10, K=6, eos=(3, -1, 0, 5), claims=('prod_v', 'eos_first')),
    C('gpm_cispo_ent0', BF, FA, 128256, 'grpo', 3, 9, K=6, eos=(-1, 2, 4), claims=('prod_v',)),
    C('obj_dual_tm', BF, F3, 128256, 'dense', 3, 12, claims=('prod_v',)),
    C('obj_dual_ent', BF, F3, 152064, 'dense', 3, 12, layout='odd', claims=('prod_v', 'head_peel')),
    C('pm_cispo', BF, F3, 152064, 'tail', 6, 13, lens=_TAIL, claims=('prod_v',)),
    C('gpm_sapo', BF, F3, 128257, 'grpo', 4, 9, K=6, eos=(-1, 0, 3, 5), claims=('prod_v',)),
    C('gobj_ent0', BF, F3, 152064, 'grpo', 3, 9, K=6, eos=(2, -1, 4), claims=('prod_v',)),
    C('gpm_sapo_noent', BF, F3, 128256, 'grpo', 3, 9, K=6, eos=(-1, 3, 1), claims=('prod_v',)),
    C('gpm_cispo_ent0', BF, F3, 128257, 'grpo', 3, 9, K=6, eos=(4, -1, 0), claims=('prod_v',)),
    C('kl_k1', F, F3, 152064, 'dense', 3, 10, claims=('prod_v',)),
    C('kl_k2', F, F3, 128257, 'tail', 6, 13, lens=_TAIL, layout='pitch', claims=('prod_v',)),
    C('pm_sapo_ek', F, F3, 128256, 'dense', 3, 10, claims=('prod_v',)),
    C('grpo_ent', F, FA, 128256, 'grpo', 3, 9, K=6, eos=(1, -1, 0), claims=('prod_v',)),
    C('gpm_cispo_ent0', F, F3, 152064, 'grpo', 3, 9, K=6, eos=(-1, 2, 4), claims=('prod_v',)),
    C('gpm_sapo_noent', F, FA, 128257, 'grpo', 3, 9, K=6, eos=(5, 0, -1), claims=('prod_v',)),
    C('ce', BF, F3, 128256, 'ce', 3, 14, claims=('prod_v', 'one_seg')),
    C('ce', F, F3, 128257, 'ce', 2, 13, layout='mismatch', oob=True, claims=('prod_v', 'one_seg', 'mismatch', 'oob')),
    C('grpo', BF, FA, 152064, 'grpo', 4, 10, K=6, eos=(3, -1, 0, 5), claims=('prod_v',)),
    C('grpo_egrad', BF, FA, 152064, 'grpo', 4, 10, K=6, eos=(3, -1, 0, 5), layout='pitch', claims=('prod_v',)),
    C('gobj_nopol', BF, F3, 128256, 'grpo', 4, 9, K=6, eos=(-1, -1, 0, 2), claims=('prod_v',)),
    C('gobj_pol', F, F3, 152064, 'grpo', 4, 9, K=6, eos=(-1, 4, 0, 2), claims=('prod_v',)),
    C('gobj_norm_ent', BF, FA, 128257, 'grpo', 4, 9, K=6, eos=(-1, 4, 0, 2), claims=('prod_v',)),
    C('gkl_k1', BF, FA, 152064, 'grpo', 3, 9, K=6, eos=(-1, 4, 0)),
    C('gkl_k2', BF, F3, 152064, 'grpo', 3, 9, K=6, eos=(-1, 4, 0)),
    C('gkl_k3', F, F3, 128256, 'grpo', 3, 9, K=6, eos=(-1, 4, 0)),
    C('gpm_cispo', BF, FA, 152064, 'grpo', 3, 9, K=6, eos=(-1, 4, 0)),
    C('gpm_sapo', F, F3, 152064, 'grpo', 3, 9, K=6, eos=(-1, 4, 0)),
    C('actor_ent0', BF, FA, 128257, 'dense', 3, 10),
    C('obj_hi', BF, FA, 152064, 'dense', 3, 10, layout='pitch'),
    C('obj_tm_ent', F, F3, 152064, 'dense', 3, 10),
    C('kl_k3', BF, FA, 152064, 'dense', 3, 10),
    # ---- FAITHFUL with 16-bit advantages, as the trainers run it (ops builds the advantages in the log-probs' dtype):
    # the row / token-mean coefficients, s1 / s2 and dual * adv round to the 16-bit dtype; SAPO's s stays fp32 --------
    C('actor', BF, FA, 128256, 'dense', 4, 12, adv='bf16', claims=('prod_v', 'adv16')),
    C('pm_sapo', BF, FA, 152064, 'dense', 3, 12, adv='bf16', claims=('prod_v', 'adv16')),
    C('pm_sapo_ek', BF, FA, 128257, 'tail', 6, 13, lens=_TAIL, adv='bf16', claims=('prod_v', 'adv16')),
    C('pm_cispo_ek', BF, FA, 152064, 'device', 6, 12, lens=_DEV, adv='bf16', claims=('prod_v', 'adv16')),
    C('obj_dual_tm', BF, FA, 128257, 'tail', 6, 13, lens=_TAIL, adv='bf16', claims=('prod_v', 'adv16')),
    C('kl_k3', BF, FA, 128256, 'dense', 3, 12, adv='bf16', claims=('prod_v', 'adv16')),
    C('obj_tm_ent', BF, FA, 152064, 'dense', 3, 12, adv='bf16', claims=('prod_v', 'adv16')),
    C('pm_sapo', H, FA, 521, 'dense', 2, 7, adv='f16', claims=('adv16',)),
    C('obj_dual_tm', H, FA, 521, 'dense', 2, 7, adv='f16', claims=('adv16',)),
    C('kl_k2', H, FA, 521, 'dense', 2, 7, adv='f16', claims=('adv16',)),
    # ---- crossover vocabularies, phase mismatch on on, masked and zero rows, out-of-range labels -------------------
    C('actor_ent', BF, FA, 98304, 'device', 6, 12, lens=_DEV, layout='mismatch', oob=True,
      claims=('crossover', 'mismatch', 'oob', 'clamp')),
    C('pm_sapo_ek', F, F3, 49152, 'dense', 3, 12, layout='mismatch', claims=('crossover', 'mismatch')),
    C('grpo_egrad', BF, F3, 98304, 'grpo', 4, 12, K=6, eos=(3, -1, 0, 5), layout='mismatch', oob=True,
      claims=('crossover', 'mismatch', 'oob')),
    C('obj_hi', F, F3, 49152, 'tail', 6, 13, lens=_TAIL, layout='odd', oob=True,
      claims=('crossover', 'head_peel', 'oob')),
    # ---- stage edges ---------------------------------------------------------------------------------------------
    C('actor', BF, FA, 15864, 'dense', 3, 10, claims=('stage-1vec', 'fold_empty')),
    C('kl_k2', BF, F3, 15880, 'dense', 3, 10, claims=('stage+1vec', 'fold_partial')),
    C('pm_cispo', BF, FA, 31744, 'dense', 3, 10, claims=('2stages', 'fold_full')),
    C('obj_tm_ent', BF, FA, 31752, 'tail', 6, 13, lens=_TAIL, claims=('2stages+1vec', 'fold_empty')),
    C('gobj_pol', BF, FA, 47624, 'grpo', 3, 9, K=6, eos=(-1, 2, 4), claims=('fold_partial',)),
    C('actor_ent', F, F3, 7932, 'dense', 3, 10, claims=('stage-1vec', 'fold_empty')),
    C('gkl_k1', F, F3, 7940, 'grpo', 3, 9, K=6, eos=(-1, 2, 4), claims=('stage+1vec', 'fold_partial')),
    C('ce', F, F3, 15872, 'ce', 3, 10, claims=('2stages', 'fold_full')),
    C('pm_sapo', F, FA, 15876, 'dense', 3, 10, layout='odd', claims=('2stages', 'fold_full', 'head_peel')),
    # ---- work list: n_work around multiples of the grid, several rounds, Z = 0, Z >> scored ------------------------
    C('actor', BF, F3, 4099, 'dense', 4, 25, claims=('nwork<G', 'many_seg')),
    C('pm_cispo_ek', BF, FA, 3001, 'tail', 1, 131, lens=(131,), shift=0, claims=('nwork=G-1', 'z0', 'one_seg')),
    C('obj_dual_ent', F, F3, 2053, 'tail', 4, 33, lens=(33,) * 4, shift=0, claims=('nwork=G', 'z0')),
    C('grpo_egrad', BF, FA, 2051, 'grpo', 7, 19, K=4, eos=(0, 0, 3, 0, -1, 0, 1), claims=('nwork=G+1',)),
    C('kl_k1', BF, FA, 5003, 'tail', 8, 33, lens=(3, 30, 0, 17, 32, 1, 9, 25), claims=('nwork=2G', 'many_seg', 'len0')),
    C('ce', BF, F3, 2999, 'ce', 5, 53, layout='mismatch', claims=('nwork=2G+1', 'mismatch', 'one_seg')),
    C('gpm_sapo', BF, FA, 4001, 'grpo', 12, 40, K=3, eos=(0,) * 10 + (-1, 1), claims=('rounds3', 'zmany', 'eos_first')),
    C('actor_ent', BF, FA, 15880, 'tail', 4, 104, lens=(104,) * 4, shift=0, claims=('rounds3', 'z0')),
    C('gobj_norm_ent', F, F3, 3000, 'grpo', 16, 30, K=5, eos=(0,) * 8 + (-1,) * 4 + (1, 2, 3, 4),
      layout='mismatch', claims=('rounds3', 'zmany', 'mismatch')),
    C('obj_dual_tm', BF, FA, 6007, 'device', 30, 14, lens=_DEV * 5, claims=('rounds3', 'clamp', 'many_seg')),
    # ---- fp16 through the C ABI (ops keeps fp16 off K1f; the instantiations ship) -------------------------------------
    C('actor', H, FA, 9001, 'dense', 3, 10),
    C('actor_ent', H, F3, 9001, 'dense', 3, 10, layout='odd'),
    C('pm_sapo', H, FA, 9001, 'dense', 3, 10),
    C('pm_cispo_ek', H, FA, 15880, 'tail', 6, 13, lens=_TAIL),
    C('grpo_ent', H, F3, 9001, 'grpo', 3, 9, K=6, eos=(-1, 2, 0)),
    C('gpm_cispo_ent0', H, FA, 9001, 'grpo', 3, 9, K=6, eos=(-1, 2, 0)),
    C('obj_dual_tm', H, F3, 9001, 'dense', 3, 10, layout='pitch'),
    C('grpo_egrad', H, FA, 9001, 'grpo', 3, 9, K=6, eos=(-1, 2, 0), layout='mismatch'),
    C('gpm_sapo_noent', H, F3, 9001, 'grpo', 3, 9, K=6, eos=(-1, 2, 0)),
    C('gpm_cispo_ent0', H, F3, 9001, 'grpo', 3, 9, K=6, eos=(0, 2, -1)),
    C('gobj_ent0', H, FA, 9001, 'grpo', 3, 9, K=6, eos=(-1, 2, 0)),
    C('gpm_sapo', H, F3, 9001, 'grpo', 3, 9, K=6, eos=(-1, 2, 0)),
    C('kl_k3', H, F3, 9001, 'dense', 3, 10),
    C('ce', H, F3, 9001, 'ce', 2, 9),
    # ---- tiny vocabularies through the ABI --------------------------------------------------------------------------
    C('actor_ent', BF, FA, 1, 'dense', 3, 8),
    C('gobj_pol', F, F3, 7, 'grpo', 3, 9, K=6, eos=(-1, 2, 0)),
    C('pm_cispo', BF, F3, 8, 'dense', 3, 8, layout='odd', claims=('head_peel',)),
    C('ce', BF, F3, 9, 'ce', 2, 9, oob=True, claims=('oob',)),
    C('kl_k2', H, FA, 9, 'tail', 6, 13, lens=_TAIL, layout='mismatch', claims=('mismatch',)),
]
CASE_IDS = [c.id for c in CASES]


# ---- the prep kernel's work list, restated ---------------------------------------------------------------------------
def slot_order(case, G):
    """-> list: record position of each work item (tile row), fused_actor_prep_kernel's `slot`: G scored rows, then G
    zero rows, round after round; whichever kind runs out first leaves the rest to the other."""
    spans = case.seg_spans()
    seq = case.n_tile // case.n_seg
    cum = [0]
    for _, n in spans:
        cum.append(cum[-1] + n)
    total = cum[-1]
    Z = case.n_seg * seq - total
    slots = []
    for seg, (first, n) in enumerate(spans):
        for k in range(seq):
            work = seg * seq + k
            j = work - first
            if 0 <= j < n:
                i = cum[seg] + j
                slots.append(i + min((i // G) * G, Z))
            else:
                z = work - (cum[seg] + min(max(j, 0), n))
                slots.append(min((z // G + 1) * G, total) + z)
    return slots


def grid_sizes(n_work):
    return sorted({min(SMS, n_work), min(114, n_work), min(7, n_work)})


@pytest.mark.parametrize('case', CASES, ids=CASE_IDS)
def test_work_list_is_a_permutation(case):
    """Every tile row gets exactly one record, the scored rows keep their flat order, and each round of G records is
    all scored or all zero rows until one kind runs out."""
    scored = {r.tile_row for r in case.rows()}
    for G in grid_sizes(case.n_tile):
        slots = slot_order(case, G)
        assert sorted(slots) == list(range(case.n_tile)), (case.id, G)
        kind = [None] * case.n_tile
        for work, s in enumerate(slots):
            kind[s] = work in scored
        flat = [s for work, s in enumerate(slots) if work in scored]
        assert flat == sorted(flat)
        n_sc, Z = len(scored), case.n_tile - len(scored)
        for i in range(min(n_sc, Z) // G):  # full rounds: G scored records, then G zero records
            assert all(kind[2 * i * G:(2 * i + 1) * G]) and not any(kind[(2 * i + 1) * G:(2 * i + 2) * G]), (case.id, G, i)


# ---- what each case claims ---------------------------------------------------------------------------------------------
def _last_fold(nvec):
    """(vectors of the first stage, vectors of the second stage) of the last phase-A fold of a body of nvec vectors."""
    if nvec == 0:
        return (0, 0)
    v0 = (nvec - 1) // (2 * STAGE_VECS) * 2 * STAGE_VECS
    return min(STAGE_VECS, nvec - v0), min(STAGE_VECS, max(nvec - v0 - STAGE_VECS, 0))


STAGE_EDGES = {'stage-1vec': STAGE_VECS - 1, 'stage+1vec': STAGE_VECS + 1, '2stages': 2 * STAGE_VECS,
               '2stages+1vec': 2 * STAGE_VECS + 1}


def _claim_holds(case, claim):
    rows = case.rows()
    geo = [case.row_geometry(r.tile_row) for r in rows]
    folds = [_last_fold(g[2]) for g in geo if g[0]]
    n_work, Z = case.n_tile, case.n_tile - len(rows)
    labels = case.special_labels()
    if claim == 'prod_v':
        return case.V in PRODUCTION_V
    if claim == 'crossover':
        return case.V == CROSSOVER_V[case.dt]
    if claim in STAGE_EDGES:  # body vectors of a same-phase scored row
        return any(g[0] and g[2] == STAGE_EDGES[claim] for g in geo)
    if claim == 'fold_empty':
        return any(f[1] == 0 for f in folds)
    if claim == 'fold_partial':
        return any(0 < f[1] < STAGE_VECS for f in folds)
    if claim == 'fold_full':
        return any(f[1] == STAGE_VECS for f in folds)
    if claim.startswith('nwork'):
        want = {'nwork<G': n_work < SMS, 'nwork=G-1': n_work == SMS - 1, 'nwork=G': n_work == SMS,
                'nwork=G+1': n_work == SMS + 1, 'nwork=2G': n_work == 2 * SMS, 'nwork=2G+1': n_work == 2 * SMS + 1}
        return want[claim]
    if claim == 'rounds3':
        return n_work > 3 * SMS
    if claim == 'z0':
        return Z == 0
    if claim == 'zmany':  # unscored tile rows and post-eos rows together: many times the counted rows
        counted = sum(case.on(r) for r in rows)
        return Z + len(rows) - counted > 4 * counted
    if claim == 'one_seg':
        return case.n_seg == 1
    if claim == 'many_seg':
        return case.n_seg >= 4
    if claim == 'len0':
        return any(n == 0 for _, n in case.seg_spans())
    if claim == 'clamp':
        return any(r < 0 for r in case.lens)
    if claim == 'mismatch':  # element loops on on rows and on masked / post-eos rows, and on zero rows of the tile
        lp, lo, gp, go = case.pitches()
        zero = [t for t in range(case.n_tile) if t not in {r.tile_row for r in rows}]
        zero_mis = any(((go + t * gp) * case.esz) % 16 != 0 for t in zero) or not zero
        on_mis = any(not g[0] and case.on(r) for g, r in zip(geo, rows))
        off_mis = case.kind == 1 or any(not g[0] and not case.on(r) for g, r in zip(geo, rows))
        same = any(g[0] for g in geo)
        return on_mis and off_mis and zero_mis and same
    if claim == 'head_peel':
        return any(g[0] and g[1] > 0 for g in geo)
    if claim == 'oob':
        return any(v >= case.V for v in labels.values())
    if claim == 'empty_sample':
        return any(all(case.masked_off(s, j) for j in range(n)) and n > 0 for s, (_, n) in enumerate(case.seg_spans()))
    if claim == 'adv16':
        return case.kind == 0 and case.mode == 'faithful' and case.adv == case.dt and ESZ[case.dt] == 2
    if claim == 'eos_first':
        return 0 in case.eos
    raise ValueError(claim)


@pytest.mark.parametrize('case', CASES, ids=CASE_IDS)
def test_case_has_the_properties_it_claims(case):
    for claim in case.claims:
        assert _claim_holds(case, claim), (case.id, claim)
    # every case: labels at column 0 and V - 1; where the row has them, in the head peel, the tail peel and on the first
    # and last column of a stage
    rows = case.rows()
    labels = case.special_labels()
    assert 0 in labels.values() and case.V - 1 in labels.values()
    if case.kind == 0:
        assert any(case.on(r) for r in rows) and any(not case.on(r) for r in rows)
    if case.kind >= 2:
        assert len(case.eos) == case.B and case.K <= case.S - 1
    if case.plan in ('tail',):
        assert all(0 <= n and first >= 0 for first, n in case.seg_spans())


def test_edge_labels_are_placed():
    """Across the case list, labels sit in a head peel, in a tail peel, on the first and the last column of a stage."""
    seen = set()
    for case in CASES:
        for i, y in case.special_labels().items():
            r = case.rows()[i]
            same, head, nvec, tail0 = case.row_geometry(r.tile_row)
            stage = STAGE_VECS * case.q
            if y < head:
                seen.add('head')
            if tail0 <= y < case.V:
                seen.add('tail')
            if y >= head and (y - head) % stage == 0 and y > head:
                seen.add('stage_first')
            if y < tail0 and (y - head) % stage == stage - 1:
                seen.add('stage_last')
    assert seen == {'head', 'tail', 'stage_first', 'stage_last'}, seen


def test_claims_cover_the_edges():
    claims = {c for case in CASES for c in case.claims}
    want = set(STAGE_EDGES) | {'prod_v', 'crossover', 'fold_empty', 'fold_partial', 'fold_full', 'nwork<G', 'nwork=G-1', 'nwork=G',
            'nwork=G+1', 'nwork=2G', 'nwork=2G+1', 'rounds3', 'z0', 'zmany', 'one_seg', 'many_seg', 'len0', 'clamp',
            'mismatch', 'head_peel', 'oob', 'empty_sample', 'eos_first', 'adv16'}
    assert want <= claims, want - claims
    assert {c.V for c in CASES} >= set(PRODUCTION_V) | {1, 7, 8, 9}
    assert {c.plan for c in CASES} == {'dense', 'tail', 'device', 'ce', 'grpo'}
    assert {c.layout for c in CASES} == {'contig', 'pitch', 'odd', 'mismatch'}
    assert set(ENTRIES) == {c.entry for c in CASES}


def test_every_instantiation_is_covered():
    """Each (T, FAITHFUL, ENT, EGRAD, PM) that launch_fused_of can select runs at least once; the ones the trainers
    reach (bf16 / fp32 logits, both modes, each flag set) at a production vocabulary."""
    seen = {instantiation(c) for c in CASES}
    assert all_instantiations() <= seen, all_instantiations() - seen
    prod = {instantiation(c) for c in CASES if c.V in PRODUCTION_V}
    trainers = {i for i in all_instantiations() if i[0] in ('bf16', 'f32')}
    assert trainers <= prod, trainers - prod


# ---- the per-segment coefficients, restated in float64 against autograd of the ports ---------------------------------
AGGS = ('seq-mean-token-mean', 'token-mean', 'seq-mean-token-sum-norm')


def token_coeff(agg, counts, B, W):
    """d loss / d (per-token term) of a masked-in token of row b, float64: actor_row_coeff (-(1/B) / count_b),
    actor_token_mean_coeff (-1 / total) and GRPO's 1 / (B * W) (the sign is the loss's: the actor's objective enters
    negated)."""
    total = float(sum(counts))
    if agg == 'seq-mean-token-mean':
        return [1.0 / (B * c) if c else float('inf') for c in counts]
    if agg == 'token-mean':
        return [1.0 / total] * B
    return [1.0 / (B * W)] * B


def entropy_grad_rows(kind, agg, mask, coeff):
    """g_H of every token, float64 (B, W): kind 0  -coeff / (B * count_b) (the seq-mean masked mean) or -coeff / total
    under token-mean;  GRPO  -coeff / total under every aggregation; 0 for tokens that do not count."""
    m = mask.double()
    B = m.size(0)
    if kind == 0 and agg != 'token-mean':
        return torch.where(mask, -coeff / (B * m.sum(-1, keepdim=True)), torch.zeros_like(m))
    return torch.where(mask, -coeff / m.sum(), torch.zeros_like(m))


def _mask(counts, W, seed):
    g = torch.Generator().manual_seed(seed)
    mask = torch.zeros(len(counts), W, dtype=torch.bool)
    for b, n in enumerate(counts):
        mask[b, torch.randperm(W, generator=g)[:n]] = True
    return mask


COUNTS = [(1,), (5, 0, 7), (300, 257, 1), (3, 3, 3, 3)]


@pytest.mark.parametrize('counts', COUNTS, ids=['1', '5-0-7', '300-257-1', '4x3'])
@pytest.mark.parametrize('agg', AGGS)
def test_segment_coefficients_match_autograd_of_the_ports(counts, agg):
    B, W = len(counts), max(counts) + 3
    mask = _mask(counts, W, sum(counts))
    lp = torch.randn(B, W, dtype=torch.float64, requires_grad=True)
    s = lp * 1.0
    loss = -policy_loss_port.aggregate(s, mask, agg)
    loss.backward()
    coeff = token_coeff(agg, counts, B, W)
    want = torch.tensor(coeff, dtype=torch.float64)[:, None].expand(B, W)
    on = mask & torch.tensor([c > 0 for c in counts])[:, None]
    assert torch.allclose(lp.grad[on], -want[on], rtol=1e-15, atol=0)
    # masked-off tokens: no gradient; a sample without a masked-in token is 0 / 0 under the per-sample mean
    filled = torch.tensor([c > 0 for c in counts])[:, None].expand(B, W)
    assert bool((lp.grad[~mask & filled] == 0).all())
    empty = lp.grad[~filled]
    if agg == 'seq-mean-token-mean':
        assert bool(torch.isnan(empty).all())
    else:
        assert bool((empty == 0).all())
    if agg == 'seq-mean-token-sum-norm':
        return
    # the actor's clipped objective and the KL term: d loss / d s and d total / d KL through the ports
    x = torch.randn(B, W, dtype=torch.float64, requires_grad=True)
    ppo_objective_port.actor_loss(x, x.detach(), torch.ones(B, W, dtype=torch.float64), mask, 0.2, 0.2,
                                  agg=agg).backward()
    assert torch.allclose(x.grad[on], -want[on], rtol=1e-14, atol=0)  # ratio 1, adv 1: d loss / d lp = the coefficient
    kl = torch.randn(B, W, dtype=torch.float64, requires_grad=True)
    c_kl = 0.25
    (c_kl * kl_loss_port.aggregate(kl, mask, agg)).backward()
    assert torch.allclose(kl.grad[on], c_kl * want[on], rtol=1e-15, atol=0)  # kl_term_coeff
    # the entropy bonus: -c * agg(H) gives g_H = -c * coefficient (ent_seg)
    h = torch.randn(B, W, dtype=torch.float64, requires_grad=True)
    c_h = 0.05
    (-c_h * policy_loss_port.aggregate(h, mask, agg)).backward()
    gh = entropy_grad_rows(0, agg, mask, c_h)
    assert torch.allclose(h.grad[on], gh[on], rtol=1e-15, atol=0)


@pytest.mark.parametrize('agg', AGGS)
def test_grpo_entropy_gradient_is_a_token_mean(agg):
    """GRPO's bonus is -c * (H * mask).sum() / mask.sum() under every aggregation of the loss."""
    mask = _mask((4, 6, 1), 8, 3)
    h = torch.randn(3, 8, dtype=torch.float64, requires_grad=True)
    (-0.1 * (h * mask).sum() / mask.sum()).backward()
    assert torch.allclose(h.grad, entropy_grad_rows(2, agg, mask, 0.1), rtol=1e-15, atol=0)


def test_restated_slot_order_matches_the_documented_interleave():
    """A hand-checked example: 5 scored rows, 4 zero rows, G = 2 -> s s z z s s z z s."""
    case = Case('actor', BF, FA, 16, 'tail', 3, 3, lens=(2, 1, 2), shift=0)
    slots = slot_order(case, 2)
    scored = {r.tile_row for r in case.rows()}
    order = [None] * case.n_tile
    for work, s in enumerate(slots):
        order[s] = 's' if work in scored else 'z'
    assert ''.join(order) == 'sszzsszzs'


def test_case_ids_are_unique():
    assert len(set(CASE_IDS)) == len(CASE_IDS)
    for a, b in itertools.combinations(CASES, 2):
        assert a != b
