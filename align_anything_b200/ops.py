"""Functional layer over libaa_b200.so: torch tensors in, torch tensors out, autograd wired.

Every function cites the reference function whose arithmetic it replaces (paths relative to
the reference's align_anything/).  PyTorch is used for device memory, streams and autograd
plumbing only; all arithmetic on the path runs in the hand-written sm_90a kernels.

`mode`:
  'faithful' (default for 16-bit tensors) -- fp32 arithmetic, rounded to the tensor dtype at the
             points where the reference's eager ops round (results carry the reference's dtypes);
  'f32'      -- fp32 outputs, no intermediate rounding.
"""
from __future__ import annotations

import ctypes
import dataclasses
import functools
import math
from typing import Sequence

import torch

from . import _lib as L

__all__ = [
    'gather_log_probabilities', 'masked_mean', 'sequence_log_probs', 'RowPlan', 'DeviceLens', 'DevicePlan', 'as_device_lens', 'rollout_layout', 'response_tail_log_probs', 'response_tail_log_probs_pair', 'dpo_loss_from_log_probs',
    'dpo_fused_loss', 'score_head', 'score_end', 'kl_rewards_and_gae', 'gae_from_rewards', 'estimator_returns', 'actor_loss', 'critic_loss',
    'move_padding_left', 'count_nonpad', 'strip_pad_tail', 'ppo_pack_metrics', 'check_status', 'raise_for_status', 'status_lane', 'causal_lm_loss', 'rm_pair_loss', 'cost_pair_loss','group_advantages', 'grpo_loss', 'tail_token_log_probs', 'pair_slices', 'slice_sums', 'tail_rows', 'linear_token_log_probs',
    'sequence_log_probs_from_hidden', 'fused_linear_token_log_probs', 'tail_log_probs_from_hidden', 'dense_log_probs_from_hidden', 'tail_actor_loss', 'tail_critic_loss', 'lm_head_weight',
    'causal_lm_loss_from_hidden', 'causal_lm_valid_rows', 'gather_log_probabilities_with_entropy',
    'response_tail_log_probs_pair_with_entropy', 'ActorObjective', 'token_mean', 'DpoObjective', 'whiten_advantages',
]

# Path knobs: plain module attributes, read at call time and never from the environment.  Every path is chosen from the
# input; these exist so that the tests, smoke() and bench.py can drive the other form of a node and compare the two.
_K6B = True  # False: lm_head path with gradient through chunked cuBLAS + K1 / K1b instead of the tensor-core kernels
_ZERO_SPANS = True  # False: K1b zero-fills every unscored tile row itself
_FUSED_ACTOR = True  # False: the PPO actor node runs K1 -> K5 -> K1b instead of the single-pass K1f
_FUSED_GRPO = True  # False: the GRPO loss runs K1 -> loss kernel -> K1b instead of the single-pass K1f
_FUSED_CE = True  # False: causal_lm_loss runs K1 -> mean NLL -> K1b instead of the single-pass K1f
# fp16 logits keep the two-pass path: under fp16 training the incoming scalar is the loss scale (2^16 ...), and the
# two-pass backward folds it into the per-row gradient BEFORE the tile is rounded to fp16; a tile born unscaled would lose its
# small entries to fp16 underflow -- exactly what loss scaling is there to prevent.  bf16 / fp32 have the exponent range.
_FUSED_F16 = False
# K1f keeps ONE row per SM in flight (that is what makes its second pass an L2 hit), so its per-row costs -- two block
# reductions, the boundary thread, ring fill / drain -- weigh more the shorter the row is, and a short-vocabulary row
# (32064 tokens) is faster on the two-pass path.  Rows below this many bytes keep K1 -> loss kernel -> K1b.
_FUSED_MIN_ROW_BYTES = 192 * 1024


def _mode_code(mode: str | None, dtype: torch.dtype) -> int:
    if mode is None:
        mode = 'faithful'
    if mode == 'faithful':
        return L.MODE_FAITHFUL
    if mode == 'f32':
        return L.MODE_F32
    raise ValueError(f"mode must be 'faithful' or 'f32', got {mode!r}")


# ---- per-device scratch (status word, last-block counters) ---------------------------------------
_scratch: dict = {}


def _device_scratch(device: torch.device):
    key = (device.type, device.index if device.index is not None else torch.cuda.current_device())
    s = _scratch.get(key)
    if s is None:
        s = {
            'status': torch.zeros(1, dtype=torch.int32, device=device),
            'counter': torch.zeros(8, dtype=torch.int32, device=device),
        }
        _scratch[key] = s
    return s


def raise_for_status(code, device=None, reset: bool = True) -> int:
    """`code` is the status word as it came back with a step's metrics (lane 7 of the DPO stats, lane 10 of the PPO
    stats; MAX-reduced across ranks, so every rank raises together).  Raises the error the reference would have raised
    eagerly; no host sync of its own.  trainers/*: called after the ONE `.tolist()` of the step."""
    v = int(code)
    if v and reset:
        device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        _device_scratch(device)['status'].zero_()
    return _raise_status_bits(v)


def status_lane(device) -> torch.Tensor:
    """The device status word as an fp32 (1,) tensor, to be concatenated to a step's metric vector (MAX lane) so that
    the step's ONE host read also reports what the reference would have raised on; see raise_for_status."""
    return _device_scratch(torch.device(device))['status'].float()


def check_status(device=None, reset: bool = True) -> int:
    """Read the device status word (ONE host sync).  Raises the error the reference would have
    raised eagerly: out-of-range labels (torch.gather), short sequences, empty mask rows."""
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    st = _device_scratch(device)['status']
    v = int(st.item())
    if reset and v:
        st.zero_()
    return _raise_status_bits(v)


def _raise_status_bits(v: int) -> int:
    if v & L.STATUS_LABEL_OOB:
        raise IndexError('align_anything_b200: a label is outside [0, vocab) (torch.gather would raise)')
    if v & L.STATUS_SHORT_SEQUENCE:
        raise ValueError('align_anything_b200: a sequence has fewer non-pad tokens than its response_len')
    if v & L.STATUS_EMPTY_MASK:
        raise IndexError('align_anything_b200: a mask row has no True element (m.nonzero()[-1] would raise)')
    if v & L.STATUS_DIVERGE_RANGE:
        raise AssertionError('diverge index is out of range!')  # trainers/text_to_text/simpo.py:72-73
    if v & L.STATUS_WHITEN_COUNT:
        raise ValueError('align_anything_b200: whitening the advantages needs at least 2 masked tokens over the rollout '
                         '(masked_var would raise)')
    return v


def _single_pass_ok(logits: torch.Tensor, enabled: bool = True, needs_grad: bool = True) -> bool:
    """Whether a single-pass node (K1f) takes this tile: the node's knob is on (`enabled`), a gradient tile is wanted
    (K1f's second pass writes it; without one K1 alone reads the rows once), the logits are not fp16 (the tile is
    written for an upstream gradient of 1 and scaled afterwards, see _FUSED_F16) and the rows are long enough for K1f
    to win (see _FUSED_MIN_ROW_BYTES).  The public wrappers decide with it and hand the answer to their node."""
    if not (enabled and needs_grad):
        return False
    if logits.dtype == torch.float16 and not _FUSED_F16:
        return False
    return logits.size(-1) * logits.element_size() >= _FUSED_MIN_ROW_BYTES


def _hand_over_once(ctx, g, *grads):
    """Backward of a node whose forward already wrote its gradients: multiply them in place by the incoming scalar `g`
    (aa_scale_tile, fp32 scalar; the kernel leaves at once when it is 1) and return them.  A second backward through
    the same graph would scale the handed-over tensors again, so it raises."""
    if getattr(ctx, 'consumed', False):
        raise RuntimeError('a single-pass loss node hands its gradient over once: compute the loss again to run backward '
                           'twice')
    ctx.consumed = True
    scale = g.detach().float().reshape(1).contiguous()
    for t in grads:
        if t is not None:
            L.check(L.lib().aa_scale_tile(t.data_ptr(), L.dtype_code(t.dtype), t.numel(), scale.data_ptr(), L.AA_F32,
                                          L.stream_ptr(t.device)))
    return grads


# ---- row plans -----------------------------------------------------------------------------------
class RowPlan:
    """Which logits rows are scored against which labels, and where the results go.

    Segment s = n[s] consecutive rows starting at element offset logit_off[s] (stride row_stride)
    of the logits tensor, labels starting at label_off[s], outputs at out_off[s] of the flat
    output buffer; tile_row[s] is the row index of the segment's first row in the gradient tile
    (the logits tensor viewed as (n_tile_rows, V))."""

    __slots__ = ('n_seg', 'n_rows', 'dev', 'out_shape', 'n_tile_rows', 'zero_spans', 'n_zero_spans', 'extra_zero_rows',
                 'n_extra')
    exact = True        # n_rows is the exact number of scored rows
    host_layout = True  # the complement of the segments is known on the host (memset spans / listed zero rows)

    # zero spans of at least this many rows go to the copy engine (cudaMemsetAsync, aa_zero_rows); shorter ones
    # are listed for the kernel (a memset launch costs ~2-3 us, a 256 KB row 40 ns of HBM time)
    MEMSET_MIN_ROWS = 16

    def __init__(self, logit_off, label_off, out_off, counts, tile_row, out_shape, n_tile_rows, device):
        n_seg = len(counts)
        cum = [0] * (n_seg + 1)
        for i, c in enumerate(counts):
            if c < 0:
                raise ValueError('negative row count in RowPlan')
            cum[i + 1] = cum[i] + c
        self.n_seg = n_seg
        self.n_rows = cum[-1]
        table = torch.tensor(
            [list(logit_off) + [0], list(label_off) + [0], list(out_off) + [0], cum, list(tile_row) + [0]],
            dtype=torch.int64,
        )
        self.dev = table.to(device, non_blocking=True)  # (5, n_seg+1)
        self.out_shape = tuple(out_shape)
        self.n_tile_rows = int(n_tile_rows)
        # complement of the segments inside the gradient tile, known on the host: (first_row, n_rows) spans
        self.zero_spans, self.n_zero_spans, self.extra_zero_rows, self.n_extra = None, 0, None, 0
        if self.n_tile_rows > 0:
            import ctypes

            big, small, at = [], [], 0
            for first, n in sorted((int(t), int(c)) for t, c in zip(tile_row, counts) if c > 0):
                if first < at:
                    raise ValueError('RowPlan segments overlap in the gradient tile')
                if first > at:
                    (big if first - at >= self.MEMSET_MIN_ROWS else small).append((at, first - at))
                at = first + n
            if at > self.n_tile_rows:
                raise ValueError('RowPlan segments exceed the gradient tile')
            if at < self.n_tile_rows:
                (big if self.n_tile_rows - at >= self.MEMSET_MIN_ROWS else small).append((at, self.n_tile_rows - at))
            flat = [v for span in big for v in span]
            self.zero_spans = (ctypes.c_int64 * max(len(flat), 1))(*flat)
            self.n_zero_spans = len(big)
            rows = [r for first, n in small for r in range(first, first + n)]
            self.n_extra = len(rows)
            if rows:
                self.extra_zero_rows = torch.tensor(rows, dtype=torch.int64).to(device, non_blocking=True)

    def ptrs(self):
        base = self.dev.data_ptr()
        step = self.dev.stride(0) * 8
        return base, base + step, base + 2 * step, base + 3 * step, base + 4 * step


class DeviceLens:
    """Per-sample response lengths that live on the DEVICE (int32 (B,)) plus a host-known upper bound -- what
    PPOTrainer.postprocess_generation returns instead of the reference's Python list
    (trainers/text_image_to_text/ppo.py:190-203).  Everything on the path takes the device tensor; the list protocol
    (`len`, iteration, indexing, `==`, `tolist`) is kept for reference code that reads `training_batch['response_lens']`
    and costs ONE host sync on first use."""

    __slots__ = ('dev', 'bound', '_host', '_plans')

    def __init__(self, dev: torch.Tensor, bound: int, host=None):
        self.dev = dev
        self.bound = int(bound)
        self._host = list(host) if host is not None else None
        self._plans = {}  # row plans built from these lengths (ops.device_tail_plan): one build per distinct tile layout

    def tolist(self):
        if self._host is None:
            self._host = self.dev.tolist()
        return self._host

    def __len__(self):
        return self.dev.numel()

    def __iter__(self):
        return iter(self.tolist())

    def __getitem__(self, i):
        return self.tolist()[i]

    def __eq__(self, other):
        return self.tolist() == list(other)

    def __repr__(self):
        return f'DeviceLens(B={len(self)}, bound={self.bound}, host={self._host})'


def device_tail_plan(lens: 'DeviceLens', *key) -> 'DevicePlan':
    """DevicePlan(lens, *key), built once per DeviceLens object and tile layout: the rollout (actor, reference) and the
    rl_step (actor) of one PPO step address tiles of the same shape, so one aa_tail_plan_build launch serves all three."""
    plan = lens._plans.get(key)
    if plan is None:
        plan = lens._plans[key] = DevicePlan(lens, *key)
    return plan


def as_device_lens(lens, device) -> DeviceLens:
    """A host list of lengths -> DeviceLens with the exact bound (one cached H2D copy, no sync)."""
    if isinstance(lens, DeviceLens):
        return lens
    host = tuple(int(r) for r in lens)
    return DeviceLens(_lens_tensor(host, str(device)), max(max(host), 1) if host else 1, host)


class DevicePlan:
    """RowPlan whose table is built ON THE DEVICE from DeviceLens (aa_tail_plan_build): n_rows is an upper bound (the
    kernels read the exact count from the table), the backward runs in tile mode (the prep kernel orders the work list:
    scored rows first, zero rows after), nothing about the row layout is known on the host."""

    __slots__ = ('n_seg', 'n_rows', 'dev', 'out_shape', 'n_tile_rows')
    exact = False        # out buffers must be zero-initialised: rows beyond a sample's length are padding
    host_layout = False  # no memset spans: K1b zero-fills every unscored tile row itself

    def __init__(self, lens: DeviceLens, seq: int, sample_stride: int, row_stride: int, label_row_stride: int,
                 label_tail_len: int, label_shift: int, row_shift: int, width: int, copies: int = 1,
                 copy_logit_delta: int = 0):
        B = len(lens)
        dev = lens.dev.device
        S = B * copies
        self.n_seg, self.n_rows, self.n_tile_rows = S, S * width, S * seq
        self.out_shape = (B, width) if copies == 1 else (copies, B, width)
        self.dev = torch.empty((5, S + 1), dtype=torch.int64, device=dev)
        L.check(L.lib().aa_tail_plan_build(lens.dev.data_ptr(), B, int(seq), int(sample_stride), int(row_stride),
                                           int(label_row_stride), int(label_tail_len), int(label_shift), int(row_shift),
                                           int(width), int(copies), int(copy_logit_delta), B * int(width),
                                           self.dev.data_ptr(), _device_scratch(dev)['status'].data_ptr(), L.stream_ptr(dev)))

    def ptrs(self):
        base = self.dev.data_ptr()
        step = self.dev.stride(0) * 8
        return base, base + step, base + 2 * step, base + 3 * step, base + 4 * step


@functools.lru_cache(maxsize=256)
def _dense_plan(B, rows, sb, sl, lab_sb, tile_row0, tile_sb, n_tile_rows, device_str):
    """Plan for a (B, rows, V) view: every row of every sample is scored."""
    device = torch.device(device_str)
    if B > 0 and sb == rows * sl and lab_sb == rows and tile_sb == rows:
        # rows are uniformly strided across samples: a single segment
        return RowPlan([0], [0], [0], [B * rows], [tile_row0], (B, rows), n_tile_rows, device)
    return RowPlan(
        [b * sb for b in range(B)], [b * lab_sb for b in range(B)], [b * rows for b in range(B)],
        [rows] * B, [tile_row0 + b * tile_sb for b in range(B)], (B, rows), n_tile_rows, device,
    )


@functools.lru_cache(maxsize=256)
def _tail_plan(lens: tuple, L_seq: int, sb: int, sl: int, lab_stride: int, lab_shift: int, row_shift: int,
               width: int | None, device_str: str):
    """Plan for per-sample response tails.  Sample i scores n_i = lens[i] - lab_shift rows starting at
    sequence position (L_seq - lens[i] + row_shift), against labels lab[i, lab_shift : lens[i]]."""
    device = torch.device(device_str)
    n = len(lens)
    counts = [max(r - lab_shift, 0) for r in lens]
    W = max(counts) if width is None else width
    first = [L_seq - r + row_shift for r in lens]
    return RowPlan(
        [i * sb + first[i] * sl for i in range(n)], [i * lab_stride + lab_shift for i in range(n)],
        [i * W for i in range(n)], counts, [i * L_seq + first[i] for i in range(n)], (n, W), n * L_seq, device,
    )


# ---- K1 / K1b autograd ---------------------------------------------------------------------------
def _launch_fwd(logits, labels, plan: RowPlan, out, stat_max, stat_logsum, ignore_index=None, entropy=None):
    """K1; with `entropy` (fp32, indexed like `out`, zero-initialised) the entropy variant, which writes the entropy of
    every scored row whose out position lies inside `entropy` and leaves every other output bit-identical."""
    dev = logits.device
    sc = _device_scratch(dev)
    p = plan.ptrs()
    args = (logits.data_ptr(), L.dtype_code(logits.dtype), logits.stride(-2), logits.size(-1), labels.data_ptr(),
            0 if ignore_index is None else int(ignore_index), 0 if ignore_index is None else 1,
            plan.n_seg, plan.n_rows, p[0], p[1], p[2], p[3], out.data_ptr(), L.dtype_code(out.dtype),
            L.ptr(stat_max), L.ptr(stat_logsum), sc['status'].data_ptr())
    if entropy is None:
        L.check(L.lib().aa_logprob_fwd(*args, L.stream_ptr(dev)))
    else:
        L.check(L.lib().aa_logprob_fwd_entropy(*args, entropy.data_ptr(), entropy.numel(), L.stream_ptr(dev)))


def _launch_bwd(logits, labels, plan: RowPlan, stat_max, stat_logsum, grad_rows, grad_seg, grad_scale,
                grad_logits, mode_code, scratch=None, ignore_index=None, grad_row_stride=None, entropy=None,
                grad_entropy=None):
    """K1b; with `entropy` (the forward's fp32 entropy) and `grad_entropy` (its upstream gradient, indexed like
    grad_rows) the entropy-gradient variant, which adds d H / d logits times g_H to every row with g_H != 0."""
    dev = logits.device
    p = plan.ptrs()
    V = logits.size(-1)
    grad_row_stride = V if grad_row_stride is None else int(grad_row_stride)
    n_tile_rows, extra, n_extra = plan.n_tile_rows, None, 0
    if n_tile_rows > 0 and _ZERO_SPANS and plan.host_layout:
        # the row layout is known on the host: long zero spans -> copy engine, isolated zero rows -> listed after the
        # scored rows (equal-cost rows first under the kernel's static stride), instead of "every tile row is work".
        # A pitched tile is cleared row by row (its pad columns are not the kernel's to touch)
        import ctypes

        if plan.n_zero_spans:
            L.check(L.lib().aa_zero_rows(grad_logits.data_ptr(), L.dtype_code(grad_logits.dtype), grad_row_stride, V,
                                         plan.n_tile_rows, ctypes.cast(plan.zero_spans, ctypes.c_void_p),
                                         plan.n_zero_spans, L.stream_ptr(dev)))
        n_tile_rows, extra, n_extra = 0, plan.extra_zero_rows, plan.n_extra
    if scratch is None:  # 32 (entropy variant: 48) bytes per work row: the row records of the TMA-staged K1b
        n_work = n_tile_rows if n_tile_rows > 0 else plan.n_rows + n_extra
        scratch = torch.empty(max(n_work, 1) * (4 if entropy is None else 6), dtype=torch.int64, device=dev)
    head = (logits.data_ptr(), L.dtype_code(logits.dtype), logits.stride(-2), logits.size(-1), labels.data_ptr(),
            0 if ignore_index is None else int(ignore_index), 0 if ignore_index is None else 1,
            plan.n_seg, plan.n_rows, p[0], p[1], p[2], p[3], p[4], stat_max.data_ptr(), stat_logsum.data_ptr(),
            L.ptr(grad_rows), L.dtype_code(grad_rows.dtype) if grad_rows is not None else L.AA_F32,
            L.ptr(grad_seg), L.ptr(grad_scale), L.dtype_code(grad_scale.dtype) if grad_scale is not None else L.AA_F32)
    tail = (grad_logits.data_ptr(), grad_row_stride, n_tile_rows, L.ptr(extra), n_extra, L.ptr(scratch), mode_code,
            L.stream_ptr(dev))
    if entropy is None:
        L.check(L.lib().aa_logprob_bwd(*head, *tail))
    else:
        L.check(L.lib().aa_logprob_bwd_entropy(*head, entropy.data_ptr(), grad_entropy.data_ptr(),
                                               L.dtype_code(grad_entropy.dtype), *tail))


def _rows_from(logits: torch.Tensor, first_row: int) -> torch.Tensor:
    return logits if first_row == 0 else logits.view(-1, logits.size(-1))[first_row:]


class _LogProbFn(torch.autograd.Function):
    """K1 forward / K1b backward.  `logits` is the tensor the gradient tile is shaped after; the plan
    addresses rows inside it, starting at row `first_row` of `logits` viewed as (rows, V) (nonzero only for
    the contiguous base of a rerouted view, see _try_reroute).  `entropy` (optional, fp32, plan.out_shape, zeros): the
    forward also writes each scored row's entropy there (a metric: no gradient flows through it).  `entropy_grad`: the
    node makes the entropy itself and returns (log-probs, entropy), both differentiable; the backward is K1b's entropy
    variant, or the plain K1b when the graph never used the entropy."""

    @staticmethod
    def forward(ctx, logits, labels, plan: RowPlan, mode_code: int, first_row: int = 0, entropy=None,
                entropy_grad: bool = False):
        ctx.entropy_grad = entropy_grad
        if entropy_grad:
            ctx.set_materialize_grads(False)
            entropy = torch.zeros(plan.out_shape, dtype=torch.float32, device=logits.device)
        out_dtype = logits.dtype if mode_code == L.MODE_FAITHFUL else torch.float32
        n_out = 1
        for d in plan.out_shape:
            n_out *= d
        fully_covered = plan.exact and (n_out == plan.n_rows)
        out = (torch.empty if fully_covered else torch.zeros)(plan.out_shape, dtype=out_dtype, device=logits.device)
        need_grad = ctx.needs_input_grad[0]  # grad mode is off inside forward(); this is the apply-time truth
        stat_max = stat_logsum = None
        if need_grad:
            stats = torch.empty((2, max(plan.n_rows, 1)), dtype=torch.float32, device=logits.device)
            stat_max, stat_logsum = stats[0], stats[1]
        _launch_fwd(_rows_from(logits, first_row), labels, plan, out, stat_max, stat_logsum, entropy=entropy)
        if need_grad:
            ctx.save_for_backward(logits, labels, stats, entropy if entropy_grad else None)
            ctx.plan, ctx.mode_code, ctx.first_row = plan, mode_code, first_row
        return (out, entropy) if entropy_grad else out

    @staticmethod
    def backward(ctx, grad_out, grad_entropy=None):
        logits, labels, stats, entropy = ctx.saved_tensors
        if grad_out is None:  # only the entropy reached the loss
            grad_out = torch.zeros(ctx.plan.out_shape, dtype=torch.float32, device=logits.device)
        grad_out = grad_out.contiguous()
        if grad_out.dtype not in (torch.float32, torch.bfloat16, torch.float16):
            grad_out = grad_out.float()
        if grad_entropy is not None:
            grad_entropy = grad_entropy.float().contiguous()
        else:
            entropy = None
        grad = torch.empty(logits.shape, dtype=logits.dtype, device=logits.device)
        _launch_bwd(_rows_from(logits, ctx.first_row), labels, ctx.plan, stats[0], stats[1], grad_out, None, None, grad,
                    ctx.mode_code, entropy=entropy, grad_entropy=grad_entropy)
        return grad, None, None, None, None, None, None


def _log_probs_and_entropy(logits, labels, plan, mode_code: int, first_row: int = 0, entropy_grad: bool = False):
    """_LogProbFn with the entropy variant of K1: -> (log-probs, fp32 entropy of the same shape, 0 where unscored).
    entropy_grad: the entropy is differentiable too (see _LogProbFn)."""
    if entropy_grad:
        return _LogProbFn.apply(logits, labels, plan, mode_code, first_row, None, True)
    entropy = torch.zeros(plan.out_shape, dtype=torch.float32, device=logits.device)
    out = _LogProbFn.apply(logits, labels, plan, mode_code, first_row, entropy)
    return out, entropy


def _contiguous_last(t: torch.Tensor) -> torch.Tensor:
    return t if t.stride(-1) == 1 else t.contiguous()


def _try_reroute(logits: torch.Tensor):
    """If `logits` is a row-aligned view of a contiguous base (e.g. `full[:, :-1]`,
    `full[idx][-R:]`), address the BASE instead so the backward writes the base's gradient tile
    directly (zero rows included) and autograd's slice-backward never materialises a padded copy."""
    if not logits._is_view():
        return None
    base = logits._base
    V = logits.size(-1)
    if base is None or base.dim() < 2 or base.size(-1) != V or not base.is_contiguous():
        return None
    if base.dtype != logits.dtype or logits.stride(-1) != 1 or logits.stride(-2) != V:
        return None
    off = logits.storage_offset() - base.storage_offset()
    if off < 0 or off % V or (logits.dim() == 3 and logits.stride(0) % V):
        return None
    return base, off // V


def gather_log_probabilities(logits: torch.Tensor, labels: torch.Tensor, mode: str | None = None) -> torch.Tensor:
    """Drop-in for utils/tools.py:402-413: log_softmax(logits, -1) gathered at `labels`, without ever
    writing the (B, L, V) log-prob tile.  logits (B, L, V) or (L, V), any batch/row strides (the
    callers pass `[:, :-1]` views); differentiable in `logits` (K1b)."""
    return _gather(logits, labels, mode, False)


def gather_log_probabilities_with_entropy(logits: torch.Tensor, labels: torch.Tensor, mode: str | None = None,
                                          entropy_grad: bool = False):
    """gather_log_probabilities plus the policy entropy of every row, -(softmax(x) * log_softmax(x)).sum(-1) of the fp32
    upcast logits, from the same K1 pass (one more FMA per logit; no extra read of the tile).  -> (log_probs, entropy):
    log_probs bit-identical to gather_log_probabilities (and as differentiable), entropy fp32 in both modes.  A -inf
    logit contributes 0 (the limit of p log p); a row of -inf only gets NaN.  By default the entropy never requires
    grad; entropy_grad=True makes it differentiable in `logits` (an entropy bonus): its gradient enters the same K1b
    launch as the log-probs' (-g_H p_k (l_k + H) per logit), and a graph that leaves the entropy unused runs the plain
    K1b."""
    return _gather(logits, labels, mode, True, entropy_grad)


def _gather(logits, labels, mode, with_entropy: bool, entropy_grad: bool = False):
    L.require_cuda(logits, labels)
    squeeze = logits.dim() == 2
    if squeeze:
        logits, labels = logits.unsqueeze(0), labels.unsqueeze(0)
    if logits.dim() != 3 or labels.shape != logits.shape[:2]:
        raise ValueError(f'expected logits (B, L, V) and labels (B, L); got {tuple(logits.shape)}, {tuple(labels.shape)}')
    logits = _contiguous_last(logits)
    if labels.dtype != torch.int64:
        labels = labels.to(torch.int64)
    labels = _contiguous_last(labels)
    B, rows, V = logits.shape
    mode_code = _mode_code(mode, logits.dtype)
    dev = str(logits.device)
    if B == 0 or rows == 0:
        out_dtype = logits.dtype if mode_code == L.MODE_FAITHFUL else torch.float32
        out = logits.new_zeros((B, rows), dtype=out_dtype)
        ent = logits.new_zeros((B, rows), dtype=torch.float32)
        if squeeze:
            out, ent = out.squeeze(0), ent.squeeze(0)
        return (out, ent) if with_entropy else out
    routed = _try_reroute(logits) if (logits.requires_grad and torch.is_grad_enabled()) else None
    lab_sb = labels.stride(0) if B > 1 else rows
    if routed is not None:
        base, row0 = routed
        n_tile = base.numel() // V
        sb_rows = logits.stride(0) // V if B > 1 else rows
        # logits offsets in the plan are relative to the view's first row (row0 of the base); tile rows are
        # rows of the base, whose shape the gradient takes
        plan = _dense_plan(B, rows, sb_rows * V, V, lab_sb, row0, sb_rows, n_tile, dev)
        tile, first_row = base, row0
    else:
        sb = logits.stride(0) if B > 1 else rows * logits.stride(1)
        plan = _dense_plan(B, rows, sb, logits.stride(1), lab_sb, 0, rows, B * rows, dev)
        tile, first_row = logits, 0
    if not with_entropy:
        out = _LogProbFn.apply(tile, labels, plan, mode_code, first_row)
        return out.squeeze(0) if squeeze else out
    out, ent = _log_probs_and_entropy(tile, labels, plan, mode_code, first_row,
                                      entropy_grad and logits.requires_grad and torch.is_grad_enabled())
    return (out.squeeze(0), ent.squeeze(0)) if squeeze else (out, ent)


# ---- lm_head x log-prob without the (rows, V) tile (SURVEY.md 8f rank 1, first step) ------------------------
def _mm_f32(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """a @ b with an fp32 result (cuBLAS accumulates in fp32 anyway; this keeps the accumulator's precision)."""
    if a.dtype == torch.float32:
        return torch.mm(a, b)
    try:
        return torch.mm(a, b, out_dtype=torch.float32)
    except (TypeError, NotImplementedError, RuntimeError):  # no mixed-dtype mm: one rounding per chunk
        return torch.mm(a, b).float()


def _pad_vocab(weight: torch.Tensor):
    """Weight with the vocabulary padded (zero rows) to a 16-byte multiple of logits per row.  V = 128257 is odd: a
    (rows, V) logits buffer then has 2-byte aligned rows, cuBLAS falls back to its unaligned kernels and K1 / K1b lose
    their 16-byte fast paths."""
    V, H = weight.shape
    q = 16 // weight.element_size()
    Vp = (V + q - 1) // q * q
    if Vp == V:
        return weight, V
    w = torch.zeros((Vp, H), dtype=weight.dtype, device=weight.device)
    w[:V].copy_(weight)
    return w, Vp


class _LinearLogProbFn(torch.autograd.Function):
    """log_softmax(hidden @ weight.T)[label] per row, `chunk` rows at a time: the GEMM (cuBLAS through
    torch.matmul -- a plain library GEMM, on a vocabulary-padded copy of the weight so that every leading dimension
    is 16-byte aligned) writes a (chunk, V_pad) buffer that K1 consumes immediately and the next chunk overwrites;
    the backward recomputes the chunk, K1b turns it into d(logits) in a second buffer (pad columns stay zero), and
    two more GEMMs accumulate d(hidden) and d(weight).  Only (max, log-sum) per row is saved.  HBM held: 2 chunk
    buffers, the padded weight and an fp32 d(weight) accumulator instead of two (rows, V) tiles."""

    @staticmethod
    def forward(ctx, hidden, weight, labels, chunk: int, mode_code: int, entropy=None, entropy_grad: bool = False):
        N, V = hidden.size(0), weight.size(0)
        dev = hidden.device
        ctx.set_materialize_grads(False)
        if entropy_grad:  # the node owns a differentiable entropy (see _LogProbFn)
            entropy = torch.zeros(N, dtype=torch.float32, device=dev)
        out_dtype = hidden.dtype if mode_code == L.MODE_FAITHFUL else torch.float32
        out = torch.empty(N, dtype=out_dtype, device=dev)
        need_grad = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        stats = torch.empty((2, max(N, 1)), dtype=torch.float32, device=dev) if need_grad else None
        w_pad, Vp = _pad_vocab(weight)
        buf = torch.empty((min(chunk, N), Vp), dtype=hidden.dtype, device=dev)
        for r0 in range(0, N, chunk):
            n = min(chunk, N - r0)
            torch.matmul(hidden[r0:r0 + n], w_pad.t(), out=buf[:n])  # the dtype rounding point of nn.Linear
            plan = _dense_plan(1, n, n * Vp, Vp, n, 0, n, 0, str(dev))
            _launch_fwd(buf[:n, :V], labels[r0:r0 + n], plan, out[r0:r0 + n],
                        stats[0, r0:r0 + n] if need_grad else None, stats[1, r0:r0 + n] if need_grad else None,
                        entropy=None if entropy is None else entropy[r0:r0 + n])
        if need_grad:
            ctx.save_for_backward(hidden, weight, labels, stats, entropy if entropy_grad else None)
            ctx.chunk, ctx.mode_code = chunk, mode_code
        return (out, entropy) if entropy_grad else out

    @staticmethod
    def backward(ctx, grad_out, grad_entropy=None):
        hidden, weight, labels, stats, entropy = ctx.saved_tensors
        N, V, chunk = hidden.size(0), weight.size(0), ctx.chunk
        dev = hidden.device
        grad_out, entropy, grad_entropy = _lm_head_grads(grad_out, entropy, grad_entropy, N, dev)
        need_h, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        w_pad, Vp = _pad_vocab(weight)
        d_hidden = torch.empty_like(hidden) if need_h else None
        d_weight = torch.zeros((Vp, weight.size(1)), dtype=torch.float32, device=dev) if need_w else None
        buf = torch.empty((min(chunk, N), Vp), dtype=hidden.dtype, device=dev)
        dbuf = torch.zeros_like(buf)  # K1b writes columns [0, V); the pad columns must stay 0 for the GEMMs below
        for r0 in range(0, N, chunk):
            n = min(chunk, N - r0)
            torch.matmul(hidden[r0:r0 + n], w_pad.t(), out=buf[:n])
            plan = _dense_plan(1, n, n * Vp, Vp, n, 0, n, 0, str(dev))
            _launch_bwd(buf[:n, :V], labels[r0:r0 + n], plan, stats[0, r0:r0 + n], stats[1, r0:r0 + n],
                        grad_out[r0:r0 + n], None, None, dbuf[:n, :V], ctx.mode_code, grad_row_stride=Vp,
                        entropy=None if entropy is None else entropy[r0:r0 + n],
                        grad_entropy=None if entropy is None else grad_entropy[r0:r0 + n])
            if need_h:
                torch.matmul(dbuf[:n], w_pad, out=d_hidden[r0:r0 + n])
            if need_w:  # fp32 accumulation across chunks, one rounding at the end (like a single GEMM)
                d_weight.add_(_mm_f32(dbuf[:n].t(), hidden[r0:r0 + n]))
        return d_hidden, (d_weight[:V].to(weight.dtype) if need_w else None), None, None, None, None, None


def _lm_head_grads(grad_out, entropy, grad_entropy, N, dev):
    """The upstream gradients of an lm_head node: the log-probs' (zeros when only the entropy reached the loss) and,
    when the entropy is differentiable and was used, the entropy with its fp32 gradient; otherwise (None, None)."""
    if grad_out is None:
        grad_out = torch.zeros(N, dtype=torch.float32, device=dev)
    grad_out = grad_out.contiguous()
    if grad_out.dtype not in (torch.float32, torch.bfloat16, torch.float16):
        grad_out = grad_out.float()
    if entropy is None or grad_entropy is None:
        return grad_out, None, None
    return grad_out, entropy, grad_entropy.float().contiguous()


class _LinearLogProbK6Fn(torch.autograd.Function):
    """The tensor-core path (bf16, H % 64 == 0; default).  Forward = K6 (no logits at all, saves (max, logsum) per row).
    Backward per row chunk = three tensor-core (wgmma) kernels on one (chunk, ld) bf16 d(logits) buffer: K6b recomputes the logits
    tile and turns it into d(logits) in its epilogue; aa_linear_dhidden = d(logits) @ W with W consumed MN-major in
    place; aa_linear_dweight accumulates d(logits)^T @ hidden in fp32 across chunks and rounds once at the end.  No
    library GEMM, no padded / transposed copy of the weight."""

    @staticmethod
    def forward(ctx, hidden, weight, labels, chunk: int, mode_code: int, entropy=None, entropy_grad: bool = False):
        ctx.set_materialize_grads(False)
        if entropy_grad:  # the node owns a differentiable entropy; its gradient enters K6b's epilogue
            entropy = torch.zeros(hidden.size(0), dtype=torch.float32, device=hidden.device)
        out, stats = _k6_forward(hidden, weight, labels, mode_code, True, entropy)
        ctx.save_for_backward(hidden, weight, labels, stats, entropy if entropy_grad else None)
        ctx.chunk, ctx.mode_code = chunk, mode_code
        return (out, entropy) if entropy_grad else out

    @staticmethod
    def backward(ctx, grad_out, grad_entropy=None):
        hidden, weight, labels, stats, entropy = ctx.saved_tensors
        N, (V, H), chunk = hidden.size(0), weight.shape, ctx.chunk
        dev = hidden.device
        grad_out, entropy, grad_entropy = _lm_head_grads(grad_out, entropy, grad_entropy, N, dev)
        ld = (V + 255) // 256 * 256
        need_h, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        d_hidden = torch.empty_like(hidden) if need_h else None
        d_weight = torch.empty_like(weight) if need_w else None
        n_chunks = (N + chunk - 1) // chunk
        # equal chunks of whole 256-row CTA-pair tiles: 16376 rows as 8192 + 8184 keep the last round of 256 x 256 tiles of
        # the d(hidden) GEMM full (512 tiles on 74 pairs = 6.9 rounds), 8320 + 8056 does not (528 tiles = 7.1 rounds run as 8)
        chunk = min(chunk, (-(-N // n_chunks) + 255) // 256 * 256)
        acc = torch.empty((V, H), dtype=torch.float32, device=dev) if (need_w and n_chunks > 1) else None
        dbuf = torch.empty((min(chunk, N), ld), dtype=torch.bfloat16, device=dev)
        lib, st = L.lib(), L.stream_ptr(dev)
        for i, r0 in enumerate(range(0, N, chunk)):
            n = min(chunk, N - r0)
            h = hidden[r0:r0 + n]
            head = (h.data_ptr(), n, H, h.stride(0), weight.data_ptr(), V, weight.stride(0), labels[r0:r0 + n].data_ptr(),
                    stats[0, r0:r0 + n].data_ptr(), stats[1, r0:r0 + n].data_ptr(), grad_out[r0:r0 + n].data_ptr(),
                    L.dtype_code(grad_out.dtype))
            if entropy is None:
                L.check(lib.aa_linear_dlogits(*head, dbuf.data_ptr(), ld, ctx.mode_code, st))
            else:
                L.check(lib.aa_linear_dlogits_entropy(*head, entropy[r0:r0 + n].data_ptr(),
                                                      grad_entropy[r0:r0 + n].data_ptr(), L.AA_F32, dbuf.data_ptr(),
                                                      ld, ctx.mode_code, st))
            if need_h:
                dh = d_hidden[r0:r0 + n]
                L.check(lib.aa_linear_dhidden(dbuf.data_ptr(), n, ld, weight.data_ptr(), V, H, weight.stride(0),
                                              dh.data_ptr(), dh.stride(0), st))
            if need_w:
                last = i == n_chunks - 1
                L.check(lib.aa_linear_dweight(dbuf.data_ptr(), n, ld, h.data_ptr(), H, h.stride(0), V, L.ptr(acc), H,
                                              1 if i > 0 else 0, d_weight.data_ptr() if last else None, d_weight.stride(0), st))
        return d_hidden, d_weight, None, None, None, None, None


def _wgmma_head(hidden: torch.Tensor, weight: torch.Tensor) -> bool:
    """Whether the tensor-core lm_head kernels (K6, K6b, aa_linear_dhidden / dweight) take these operands: bf16 hidden
    states and weight, a hidden size divisible by 64.  Other operands go through library GEMMs around K1 / K1b."""
    return hidden.dtype == weight.dtype == torch.bfloat16 and hidden.size(-1) % 64 == 0


def linear_token_log_probs(hidden: torch.Tensor, weight: torch.Tensor, labels: torch.Tensor,
                           chunk_rows: int | None = None, mode: str | None = None, return_entropy: bool = False,
                           entropy_grad: bool = False):
    """gather_log_probabilities(F.linear(hidden, weight), labels) for hidden (N, H), weight (V, H), labels (N,)
    without materialising the (N, V) logits / gradient tiles.  Differentiable in hidden and weight.  return_entropy:
    -> (log_probs, entropy), the fp32 entropy of every row from the forward pass that computes the log-probs (K6's
    entropy variant, or K1's on the library-GEMM path): no extra GEMM pass, and by default no gradient.  entropy_grad
    (with return_entropy): the entropy is differentiable in hidden and weight too; its gradient enters the d(logits)
    buffer in K6b's epilogue (K1b's entropy variant on the library-GEMM path), so the backward runs the same GEMMs."""
    L.require_cuda(hidden, weight, labels)
    if hidden.dim() != 2 or weight.dim() != 2 or hidden.size(1) != weight.size(1) or labels.shape != hidden.shape[:1]:
        raise ValueError('expected hidden (N, H), weight (V, H), labels (N,)')
    if hidden.dtype != weight.dtype:
        raise ValueError('hidden and weight must share a dtype')
    V = weight.size(0)
    if hidden.size(0) == 0:
        return (hidden.new_zeros((0,)), hidden.new_zeros((0,), dtype=torch.float32)) if return_entropy else hidden.new_zeros((0,))
    labels = labels.to(torch.int64).contiguous()
    entropy = torch.zeros(hidden.size(0), dtype=torch.float32, device=hidden.device) if return_entropy else None
    if _K6B and _wgmma_head(hidden, weight):
        if chunk_rows is None:  # ~2 GB of d(logits) per chunk: few read-modify-write passes over the fp32 d(weight)
            chunk_rows = max(128, (2 << 30) // ((V + 255) // 256 * 256 * 2) // 128 * 128)
        fn = _LinearLogProbK6Fn
    else:
        # f16 / f32 operands or H % 64 != 0: library GEMMs (cuBLAS) around K1 / K1b -- not the product's hot configuration
        if chunk_rows is None:  # ~256 MB of logits per chunk
            chunk_rows = max(128, (256 << 20) // (V * hidden.element_size()) // 128 * 128)
        fn = _LinearLogProbFn
    args = (hidden.contiguous(), weight.contiguous(), labels, int(chunk_rows), _mode_code(mode, hidden.dtype))
    if not return_entropy:
        return fn.apply(*args)
    if entropy_grad and torch.is_grad_enabled() and (hidden.requires_grad or weight.requires_grad):
        return fn.apply(*args, None, True)
    return fn.apply(*args, entropy), entropy


def fused_linear_token_log_probs(hidden: torch.Tensor, weight: torch.Tensor, labels: torch.Tensor,
                                 mode: str | None = None, return_stats: bool = False, return_entropy: bool = False):
    """K6 (wgmma): log_softmax(hidden @ weight.T)[label] per row in ONE kernel, no logits tile, for rows that
    carry NO gradient (reference model / rollout scoring).  hidden (N, H) bf16, weight (V, H) bf16, H % 64 == 0.
    return_stats adds the (2, N) (max, logsum); return_entropy adds the fp32 entropy per row (K6's entropy variant, the
    same log-probs and statistics bit for bit), in that order."""
    L.require_cuda(hidden, weight, labels)
    if hidden.dim() != 2 or weight.dim() != 2 or hidden.size(1) != weight.size(1) or labels.shape != hidden.shape[:1]:
        raise ValueError('expected hidden (N, H), weight (V, H), labels (N,)')
    if hidden.dtype != torch.bfloat16 or weight.dtype != torch.bfloat16:
        raise ValueError('K6 takes bf16 operands')
    hidden, weight = _contiguous_last(hidden.detach()), _contiguous_last(weight.detach())
    labels = labels.to(torch.int64).contiguous()
    entropy = torch.empty(hidden.size(0), dtype=torch.float32, device=hidden.device) if return_entropy else None
    out, stats = _k6_forward(hidden, weight, labels, _mode_code(mode, hidden.dtype), return_stats, entropy)
    return (out,) + ((stats,) if return_stats else ()) + ((entropy,) if return_entropy else ()) \
        if (return_stats or return_entropy) else out


def _k6_forward(hidden, weight, labels, mode_code: int, return_stats: bool, entropy=None):
    """One K6 launch (+ the split merge) on contiguous bf16 operands and int64 labels -> (out, stats or None); with
    `entropy` (fp32 (N,)) the entropy variant, which also fills it."""
    N, V = hidden.size(0), weight.size(0)
    out = torch.empty(N, dtype=torch.bfloat16 if mode_code == L.MODE_FAITHFUL else torch.float32, device=hidden.device)
    stats = torch.empty((2, max(N, 1)), dtype=torch.float32, device=hidden.device) if return_stats else None
    sc = _device_scratch(hidden.device)
    per_split = 3 if entropy is None else 4  # floats per (row, vocabulary split) of the merge scratch
    partial = torch.empty(per_split * max(132 * 128, 16 * N), dtype=torch.float32, device=hidden.device)
    args = (hidden.data_ptr(), N, hidden.size(1), hidden.stride(0), weight.data_ptr(), V, weight.stride(0), labels.data_ptr(),
            out.data_ptr(), L.dtype_code(out.dtype), L.ptr(stats[0]) if return_stats else None,
            L.ptr(stats[1]) if return_stats else None, partial.data_ptr(), partial.numel(), mode_code,
            sc['status'].data_ptr())
    if entropy is None:
        L.check(L.lib().aa_linear_logprob_fwd(*args, L.stream_ptr(hidden.device)))
    else:
        L.check(L.lib().aa_linear_logprob_fwd_entropy(*args, entropy.data_ptr(), L.stream_ptr(hidden.device)))
    return out, stats


def lm_head_weight(module) -> torch.Tensor:
    """The (V, H) weight of a causal LM's output head for the fused lm_head paths, or a clear error where those paths
    would be silently wrong: the weight is used OUTSIDE the module's forward, so it must be materialised here (under
    DeepSpeed ZeRO-3 it is a partitioned placeholder), and the head must be a plain bias-free projection of
    `hidden_states[-1]` without logit scaling / soft-capping (Gemma-2, Cohere)."""
    head = module.get_output_embeddings()
    weight = head.weight
    if hasattr(weight, 'ds_id') or weight.numel() == 0:
        raise RuntimeError('fused_lm_head is not supported under DeepSpeed ZeRO-3: the lm_head weight is partitioned outside '
                           'the module forward (use the default logits-tile path, or ZeRO <= 2)')
    if getattr(head, 'bias', None) is not None:
        raise RuntimeError('fused_lm_head needs a bias-free lm_head')
    cfg = getattr(module, 'config', None)
    for key in ('final_logit_softcapping', 'logit_scale'):
        if getattr(cfg, key, None) not in (None, 1.0):
            raise RuntimeError(f'fused_lm_head does not reproduce `{key}` = {getattr(cfg, key)}: use the default logits-tile path')
    if weight.dim() != 2:
        raise RuntimeError('fused_lm_head expects a (V, H) head weight')
    return weight


@functools.lru_cache(maxsize=64)
def _tail_indices(counts: tuple, first_pos: tuple, seq: int, W: int, device_str: str):
    """Host-built (cached, copied once) gather / scatter indices of the scored rows: flat position i * seq + first_i + k in
    the (n * seq, H) hidden matrix and i * W + k in the padded (n, W) output, k < counts_i.  The counts are host values
    (the callers hold the response lengths as Python ints), so no boolean indexing and no device->host sync is needed."""
    src, dst = [], []
    for i, (c, f) in enumerate(zip(counts, first_pos)):
        for k in range(max(int(c), 0)):
            src.append(i * seq + min(max(int(f) + k, 0), seq - 1))
            dst.append(i * W + k)
    dev = torch.device(device_str)
    return (torch.tensor(src, dtype=torch.int64).to(dev, non_blocking=True),
            torch.tensor(dst, dtype=torch.int64).to(dev, non_blocking=True))


def _tails_from_hidden(hidden, weight, labels_padded, lens, counts, first_pos, lab_shift, chunk_rows, mode,
                       return_entropy: bool = False, entropy_grad: bool = False):
    """Sample i scores counts[i] rows: hidden position first_pos[i] + k against labels_padded[i, lab_shift + k].
    The scored rows are gathered into a compact (rows, H) matrix: K6 when nothing needs a gradient, else K6 + K6b + the
    two backward GEMMs (linear_token_log_probs).  Returns (n, max(counts)) right-padded with 0; return_entropy: and the
    fp32 entropy of the same rows, laid out alike, from the same forward kernel."""
    n, seq, H = hidden.shape
    W = max(max(counts), 0)
    out_dtype = hidden.dtype if _mode_code(mode, hidden.dtype) == L.MODE_FAITHFUL else torch.float32
    if W == 0:
        out = hidden.new_zeros((n, 0), dtype=out_dtype)
        return (out, hidden.new_zeros((n, 0), dtype=torch.float32)) if return_entropy else out
    dev = hidden.device
    src, dst = _tail_indices(tuple(int(c) for c in counts), tuple(int(f) for f in first_pos), seq, W, str(dev))
    rows = hidden.reshape(n * seq, H).index_select(0, src)
    lab = labels_padded[:, lab_shift:lab_shift + W].reshape(-1).index_select(0, dst)
    needs_grad = torch.is_grad_enabled() and (hidden.requires_grad or weight.requires_grad)
    ent = None
    if not needs_grad and _wgmma_head(hidden, weight):  # K6: one tensor-core kernel, no logits at all
        lp = fused_linear_token_log_probs(rows, weight, lab, mode, return_entropy=return_entropy)
        if return_entropy:
            lp, ent = lp
    elif return_entropy:
        lp, ent = linear_token_log_probs(rows, weight, lab, chunk_rows, mode, return_entropy=True,
                                         entropy_grad=entropy_grad)
    else:
        lp = linear_token_log_probs(rows, weight, lab, chunk_rows, mode)
    out = torch.zeros(n * W, dtype=lp.dtype, device=dev).index_copy(0, dst, lp).view(n, W)
    if not return_entropy:
        return out
    return out, torch.zeros(n * W, dtype=torch.float32, device=dev).index_copy(0, dst, ent).view(n, W)


def sequence_log_probs_from_hidden(hidden: torch.Tensor, weight: torch.Tensor, input_ids: torch.Tensor,
                                   response_lens: Sequence[int], pad_id: int, strip: bool = True,
                                   chunk_rows: int | None = None, mode: str | None = None) -> torch.Tensor:
    """DPOTrainer.compute_log_probs (trainers/text_to_text/dpo.py:122-142) from the LAST HIDDEN STATES
    (2B, L, H) and the lm_head weight (V, H): the scored rows are gathered into a compact (rows, H) matrix and
    go through K6 / linear_token_log_probs, so no (2B, L, V) tile exists in either direction."""
    L.require_cuda(hidden, weight, input_ids)
    lens = tuple(int(r) for r in response_lens)
    seq = hidden.size(1)
    labels = strip_pad_tail(input_ids, lens, pad_id, strip)  # (n, max R); row i scores labels[i, 1:R_i]
    return _tails_from_hidden(hidden, weight, labels, lens, [max(r - 1, 0) for r in lens], [seq - r for r in lens], 1,
                              chunk_rows, mode)


def tail_log_probs_from_hidden(hidden: torch.Tensor, weight: torch.Tensor, input_ids: torch.Tensor,
                               response_lens: Sequence[int], chunk_rows: int | None = None,
                               mode: str | None = None, return_entropy: bool = False, entropy_grad: bool = False):
    """The multimodal PPO scoring rows (trainers/text_image_to_text/ppo.py:233-246, 296-309): sample b scores
    `logits[b, :-1][-R_b:]` against `input_ids[b, 1:][-R_b:]`, here from the last hidden states (B, L, H) and the
    lm_head weight -- hidden position L - 1 - R_b + k predicts token L - R_b + k.  return_entropy: -> (log_probs,
    entropy), the fp32 policy entropy of the same rows (0 in the padding) from the same forward kernel; entropy_grad:
    differentiable too (see linear_token_log_probs)."""
    L.require_cuda(hidden, weight, input_ids)
    lens = tuple(int(r) for r in response_lens)
    seq = hidden.size(1)
    labels = strip_pad_tail(input_ids, lens, 0, strip=False)  # (B, max R): input_ids[b, -R_b:]
    return _tails_from_hidden(hidden, weight, labels, lens, list(lens), [seq - 1 - r for r in lens], 0, chunk_rows, mode,
                              return_entropy, entropy_grad)


def dense_log_probs_from_hidden(hidden: torch.Tensor, weight: torch.Tensor, input_ids: torch.Tensor, start: int,
                                chunk_rows: int | None = None, mode: str | None = None, return_entropy: bool = False,
                                entropy_grad: bool = False):
    """`gather_log_probabilities(F.linear(hidden, weight)[:, :-1], input_ids[:, 1:])[:, start:]` from the last hidden
    states (B, L, H) and the lm_head weight (V, H), without the (B, L, V) logits tile: every sample scores the same rows,
    hidden positions [start, L - 1) against tokens [start + 1, L).  The text PPO rollout (start = 0), its rl_step
    (start = prompt_idx) and GRPO (start = L - 1 - logits_to_keep) all read this.  Without a gradient the rows go to K6;
    with one to linear_token_log_probs.  -> (B, L - 1 - start), the dtype gather_log_probabilities returns;
    return_entropy: (log_probs, fp32 entropy (B, L - 1 - start)) from the same forward kernel (no gradient unless
    entropy_grad, see linear_token_log_probs)."""
    L.require_cuda(hidden, weight, input_ids)
    if hidden.dim() != 3 or input_ids.shape != hidden.shape[:2]:
        raise ValueError('expected hidden (B, L, H) and input_ids (B, L)')
    B, seq = input_ids.shape
    start = int(start)
    if not 0 <= start <= seq - 1:
        raise ValueError(f'start = {start} lies outside [0, {seq - 1}] for sequences of {seq}')
    W = seq - 1 - start
    return _tails_from_hidden(hidden, weight, input_ids, (W,) * B, [W] * B, [start] * B, start + 1, chunk_rows, mode,
                              return_entropy, entropy_grad)


# ---- DPO -----------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=64)
def _lens_tensor(lens: tuple, device_str: str):
    return torch.tensor(lens, dtype=torch.int32).to(device_str, non_blocking=True)


def strip_pad_tail(input_ids: torch.Tensor, response_lens: Sequence[int], pad_id: int, strip: bool = True):
    """labels[i, :R_i] = strip_pad(input_ids[i])[-R_i:] (trainers/text_to_text/dpo.py:52-54,135-137),
    or the plain tail input_ids[i, -R_i:] when strip=False (text_audio_to_text/dpo.py:100).
    Returns an int64 (n, max R) buffer (entries beyond R_i undefined)."""
    L.require_cuda(input_ids)
    lens = tuple(int(r) for r in response_lens)
    n, seq = input_ids.shape
    if len(lens) != n:
        raise ValueError('response_lens must have one entry per row of input_ids')
    if min(lens) < 1 or max(lens) > seq:
        raise ValueError(f'response_lens must lie in [1, {seq}]; got {lens}')
    input_ids = _contiguous_last(input_ids)
    out = torch.empty((n, max(lens)), dtype=torch.int64, device=input_ids.device)
    sc = _device_scratch(input_ids.device)
    L.check(L.lib().aa_strip_pad_tail(
        input_ids.data_ptr(), n, seq, input_ids.stride(0), int(pad_id), 1 if strip else 0,
        _lens_tensor(lens, str(input_ids.device)).data_ptr(), out.data_ptr(), out.stride(0),
        sc['status'].data_ptr(), L.stream_ptr(input_ids.device)))
    return out


def _dpo_plan(logits: torch.Tensor, lens: tuple, label_stride: int):
    n, seq, V = logits.shape
    if logits.stride(-1) != 1:
        raise ValueError('logits must be contiguous in the vocab dimension')
    return _tail_plan(lens, seq, logits.stride(0), logits.stride(1), label_stride, 1, 0, None, str(logits.device))


def sequence_log_probs(logits: torch.Tensor, input_ids: torch.Tensor, response_lens: Sequence[int], pad_id: int,
                       strip: bool = True, mode: str | None = None) -> torch.Tensor:
    """The arithmetic of DPOTrainer.compute_log_probs after the model forward
    (trainers/text_to_text/dpo.py:129-142; text_image_to_text/dpo.py:92-105; strip=False:
    text_audio_to_text/dpo.py:93-105): for sample i the R_i - 1 log-probs of its response tail,
    right-padded with 0 to max(R) - 1.  ONE launch for all samples, no host sync."""
    L.require_cuda(logits, input_ids)
    lens = tuple(int(r) for r in response_lens)
    labels = strip_pad_tail(input_ids, lens, pad_id, strip)
    logits = _contiguous_last(logits)
    plan = _dpo_plan(logits, lens, labels.stride(0))
    return _LogProbFn.apply(logits, labels, plan, _mode_code(mode, logits.dtype))


DPO_LOSS_TYPES = {'sigmoid': 0, 'robust': 1, 'hinge': 2, 'ipo': 3, 'sppo_hard': 4, 'nca_pair': 5, 'apo_zero': 6,
                  'apo_down': 7, 'exo_pair': 8, 'discopop': 9, 'aot': 10, 'aot_pair': 11}  # include/aa_b200.h AA_DPO_*
DPO_F_DIVERGENCES = {'reverse_kl': 0, 'js_divergence': 1, 'alpha_divergence': 2}  # include/aa_b200.h AA_DPO_FDIV_*
DPO_AOT_MAX_PAIRS = 1024  # include/aa_b200.h AA_DPO_AOT_MAX_PAIRS: the pairs one rank's AOT sort takes
_DPO_EXT_TYPES = ('exo_pair', 'discopop', 'aot', 'aot_pair')  # aa_dpo_loss_ext's own types


@dataclasses.dataclass(frozen=True)
class DpoObjective:
    """The DPO objective options of TRL's DPOConfig (the reference's loss, trainers/text_to_text/dpo.py:166-203, when
    every field is at its default).  With a = pc - rc and b = pr - rr the policy-minus-reference log-prob sums of the
    chosen and rejected rows, h = a - b, z = beta * h and eps = label_smoothing, the per-pair loss is

        sigmoid    -(1 - eps) logsigmoid(z) - eps logsigmoid(-z)            (eps > 0: conservative DPO)
        robust     (-(1 - eps) logsigmoid(z) + eps logsigmoid(-z)) / (1 - 2 eps)
        hinge      relu(1 - z)
        ipo        (h - 1 / (2 beta))^2, each of pc, pr, rc, rr divided by its row's scored-token count first
        sppo_hard  (a - 1 / (2 beta))^2 + (b + 1 / (2 beta))^2
        nca_pair   -logsigmoid(beta a) - logsigmoid(-beta a) / 2 - logsigmoid(-beta b) / 2
        apo_zero   (1 - sigmoid(beta a)) + sigmoid(beta b)
        apo_down   sigmoid(beta a) + (1 - sigmoid(beta h))
        exo_pair   sigmoid(z) (logsigmoid(z) - log(1 - e')) + sigmoid(-z) (logsigmoid(-z) - log e'), e' = eps or 1e-3
        discopop   -logsigmoid(z) (1 - m) + exp(-z) m, m = sigmoid(z / discopop_tau)
        aot_pair   the kept pairs' a and, separately, their b sorted ascending (stable, NaN last); with
                   d_k = a_(k) - b_(k) the loss at position k is -(1 - eps) logsigmoid(beta d_k) - eps logsigmoid(-beta d_k)
        aot        the same with pc - pr and rc - rr sorted in place of a and b

    f_divergence_type replaces h before a loss type that reads z = beta * h (sigmoid, robust, hinge, exo_pair) does:
    'reverse_kl' keeps h = a - b, 'js_divergence' takes h - (softplus(a) - softplus(b)), 'alpha_divergence' takes
    (cap_exp(-alpha b) - cap_exp(-alpha a)) / alpha with alpha = f_alpha_divergence_coef and cap_exp(x) =
    exp(min(x, floor(log(finfo(dtype).max) * 1e4) / 1e4)) in the log-prob dtype (no gradient where the clamp holds).
    A field away from its default on a type that does not read it raises.

    The loss is the mean over the kept pairs; rpo_alpha > 0 adds rpo_alpha * NLL, NLL = -sum(pc) / sum(R_c - 1) over
    the kept pairs' chosen rows (RPO), reported as train/nll_loss.  reference_free: rc = rr = 0 and no reference model
    runs.  The metrics keep the reference's definitions for every loss type (from the unsorted ratios under AOT).
    Checked here, before anything runs."""

    loss_type: str = 'sigmoid'
    label_smoothing: float = 0.0
    rpo_alpha: float = 0.0
    reference_free: bool = False
    f_divergence_type: str = 'reverse_kl'
    f_alpha_divergence_coef: float = 1.0
    discopop_tau: float = 0.05

    def __post_init__(self):
        if self.loss_type not in DPO_LOSS_TYPES:
            raise ValueError(f'loss_type must be one of {sorted(DPO_LOSS_TYPES)}, got {self.loss_type!r}')
        eps, alpha = float(self.label_smoothing), float(self.rpo_alpha)
        if not 0.0 <= eps < 0.5:
            raise ValueError(f'label_smoothing must lie in [0, 0.5), got {self.label_smoothing!r}')
        if eps > 0.0 and self.loss_type not in ('sigmoid', 'robust', 'exo_pair', 'aot', 'aot_pair'):
            raise ValueError(f"label_smoothing applies to loss_type 'sigmoid', 'robust', 'exo_pair', 'aot' and 'aot_pair' "
                             f"only, not {self.loss_type!r}")
        if not (alpha >= 0.0 and math.isfinite(alpha)):
            raise ValueError(f'rpo_alpha must be a finite value >= 0, got {self.rpo_alpha!r}')
        if not isinstance(self.reference_free, bool):
            raise ValueError(f'reference_free must be a bool, got {self.reference_free!r}')
        if self.f_divergence_type not in DPO_F_DIVERGENCES:
            raise ValueError(f'f_divergence_type must be one of {sorted(DPO_F_DIVERGENCES)}, got {self.f_divergence_type!r}')
        if self.f_divergence_type != 'reverse_kl' and self.loss_type not in ('sigmoid', 'robust', 'hinge', 'exo_pair'):
            raise ValueError(f"f_divergence_type {self.f_divergence_type!r} applies to loss_type 'sigmoid', 'robust', "
                             f"'hinge' and 'exo_pair' only, not {self.loss_type!r}")
        coef, tau = float(self.f_alpha_divergence_coef), float(self.discopop_tau)
        if not (coef > 0.0 and math.isfinite(coef)):
            raise ValueError(f'f_alpha_divergence_coef must be a finite value > 0, got {self.f_alpha_divergence_coef!r}')
        if coef != 1.0 and self.f_divergence_type != 'alpha_divergence':
            raise ValueError("f_alpha_divergence_coef applies to f_divergence_type 'alpha_divergence' only")
        if not (tau > 0.0 and math.isfinite(tau)):
            raise ValueError(f'discopop_tau must be a finite value > 0, got {self.discopop_tau!r}')
        if tau != 0.05 and self.loss_type != 'discopop':
            raise ValueError(f"discopop_tau applies to loss_type 'discopop' only, not {self.loss_type!r}")

    @property
    def is_default(self) -> bool:
        """The reference's objective: K2 runs today's launch."""
        return (self.loss_type == 'sigmoid' and float(self.label_smoothing) == 0.0 and float(self.rpo_alpha) == 0.0
                and not self.reference_free and not self.needs_ext)

    @property
    def needs_ext(self) -> bool:
        """A loss type or f-divergence of K2's extended variant (aa_dpo_loss_ext)."""
        return self.loss_type in _DPO_EXT_TYPES or self.f_divergence_type != 'reverse_kl'

    @property
    def needs_counts(self) -> bool:
        return self.loss_type == 'ipo' or float(self.rpo_alpha) > 0.0


def _dpo_counts(obj: DpoObjective | None, response_lens, device):
    """int32 [2B] scored rows per sample (R_i - 1) when the objective divides by them, else None; a count it would
    divide by that is 0 raises here."""
    if obj is None or not obj.needs_counts:
        return None
    if response_lens is None:
        raise ValueError(f'loss_type={obj.loss_type!r} with rpo_alpha={obj.rpo_alpha} needs response_lens')
    counts = tuple(int(r) - 1 for r in response_lens)
    B = len(counts) // 2
    if obj.loss_type == 'ipo' and min(counts) < 1:
        raise ValueError(f'ipo divides each log-prob sum by its row count R_i - 1: a response of length 1 has none '
                         f'(response_lens {tuple(response_lens)})')
    if float(obj.rpo_alpha) > 0.0 and sum(counts[:B]) < 1:
        raise ValueError('rpo_alpha > 0 takes the token mean of the chosen responses: they score no token')
    return _lens_tensor(counts, str(device))


def _dpo_launch(policy_lp, ref_lp, scale_coeff, mode_code, input_ids, want_grad_seg, coll=None, obj=None, counts=None):
    """coll: an `_lib.AaColl` descriptor (utils.multi_process.FusedPackedAllReduce.next()) -> K2's last block
    also all-reduces the stats over NVLink; the reduced vector comes back as a 4th result.  obj: a non-default
    DpoObjective -> aa_dpo_loss_obj, or aa_dpo_loss_ext for its f-divergences and the types only that entry has (ref_lp
    None when reference-free; stats gets a 9th lane, the NLL, with rpo_alpha)."""
    import ctypes

    dev = policy_lp.device
    n2, W = policy_lp.shape
    B = n2 // 2
    per_pair = torch.empty((5, B), dtype=torch.float32, device=dev)
    stats = torch.empty(9 if obj is not None and float(obj.rpo_alpha) > 0.0 else 8, dtype=torch.float32, device=dev)
    grad_seg = torch.empty(n2, dtype=torch.float32, device=dev) if want_grad_seg or obj is not None else None
    sc = _device_scratch(dev)
    ids = None
    if input_ids is not None:
        ids = _contiguous_last(input_ids)
    ids_args = (L.ptr(ids), ids.size(1) if ids is not None else 0, ids.stride(0) if ids is not None else 0)
    if obj is not None:
        if coll is not None:
            raise ValueError('the DPO objective options have no in-kernel collective: all-reduce the stats instead')
        head = (policy_lp.data_ptr(), L.ptr(ref_lp), L.dtype_code(policy_lp.dtype), B, W, policy_lp.stride(0),
                float(scale_coeff), mode_code, DPO_LOSS_TYPES[obj.loss_type], float(obj.label_smoothing),
                float(obj.rpo_alpha))
        tail = (L.ptr(counts), *ids_args, per_pair.data_ptr(), grad_seg.data_ptr(), stats.data_ptr(),
                sc['counter'][0:1].data_ptr(), sc['status'].data_ptr(), L.stream_ptr(dev))
        if obj.needs_ext:
            if obj.loss_type in ('aot', 'aot_pair') and B > DPO_AOT_MAX_PAIRS:
                raise ValueError(f'{obj.loss_type} sorts at most {DPO_AOT_MAX_PAIRS} pairs per rank, got {B}')
            e = float(obj.label_smoothing) or 1e-3  # EXO's constants in double, as TRL forms them from the Python value
            L.check(L.lib().aa_dpo_loss_ext(*head, DPO_F_DIVERGENCES[obj.f_divergence_type],
                                            float(obj.f_alpha_divergence_coef), float(obj.discopop_tau),
                                            math.log(1 - e), math.log(e), *tail))
        else:
            L.check(L.lib().aa_dpo_loss_obj(*head, *tail))
        return per_pair, stats, grad_seg
    stats_global = torch.empty(8, dtype=torch.float32, device=dev) if coll is not None else None
    L.check(L.lib().aa_dpo_loss(
        policy_lp.data_ptr(), ref_lp.data_ptr(), L.dtype_code(policy_lp.dtype), B, W, policy_lp.stride(0),
        float(scale_coeff), mode_code, *ids_args, per_pair.data_ptr(), L.ptr(grad_seg), stats.data_ptr(),
        sc['counter'][0:1].data_ptr(), ctypes.byref(coll) if coll is not None else None, L.ptr(stats_global),
        sc['status'].data_ptr(), L.stream_ptr(dev)))
    if coll is not None:
        return per_pair, stats, grad_seg, stats_global
    return per_pair, stats, grad_seg


def _dpo_dict(per_pair, stats, out_dtype, skip_identical):
    loss_i, better, worse, _, valid = per_pair
    if skip_identical:  # the reference stacks only the kept pairs (data-dependent shape -> one sync)
        keep = valid.bool()
        better, worse = better[keep], worse[keep]
    better = better.to(out_dtype)
    worse = worse.to(out_dtype)
    return {
        'reward': better + worse,
        'better_sample_reward': better,
        'worse_sample_reward': worse,
        'reward_accuracy': stats[4],
        'reward_margin': better - worse,
    }


class _DpoFromLpFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, policy_lp, ref_lp, scale_coeff, mode_code, input_ids, obj=None, counts=None):
        per_pair, stats, grad_seg = _dpo_launch(policy_lp, ref_lp, scale_coeff, mode_code, input_ids, True, obj=obj,
                                                counts=counts)
        ctx.save_for_backward(grad_seg)
        ctx.lp_shape, ctx.lp_dtype = policy_lp.shape, policy_lp.dtype
        ctx.mark_non_differentiable(per_pair, stats)
        out_dtype = policy_lp.dtype if mode_code == L.MODE_FAITHFUL else torch.float32
        return stats[0].to(out_dtype), per_pair, stats

    @staticmethod
    def backward(ctx, g_loss, _g1, _g2):
        (grad_seg,) = ctx.saved_tensors
        g = (grad_seg * g_loss.float()).to(ctx.lp_dtype)
        return g.unsqueeze(1).expand(ctx.lp_shape), None, None, None, None, None, None


def _dpo_outputs(loss, per_pair, stats, out_dtype, skip_identical_pairs, obj):
    out = {'loss': loss}
    out.update(_dpo_dict(per_pair, stats, out_dtype, skip_identical_pairs))
    if obj is not None and float(obj.rpo_alpha) > 0.0:
        out['nll_loss'] = stats[8]
    out['_stats'] = stats
    return out


def dpo_loss_from_log_probs(policy_lp: torch.Tensor, ref_lp: torch.Tensor | None, scale_coeff: float,
                            input_ids: torch.Tensor | None = None, skip_identical_pairs: bool = False,
                            mode: str | None = None, objective: DpoObjective | None = None,
                            response_lens: Sequence[int] | None = None) -> dict[str, torch.Tensor]:
    """trainers/text_to_text/dpo.py:150-203 given the two (2B, W) log-prob tensors: ONE launch for
    the 4 sums per pair, the log-sigmoid loss and the five metrics (K2).  `skip_identical_pairs`:
    text_audio_to_text/dpo.py:134-139.  Extra key '_stats' = packed fp32[8] local means for
    the all-reduce (utils.multi_process.all_reduce_packed).  objective: a DpoObjective (ref_lp may be None when it is
    reference-free); response_lens (R_i per row) give the row counts that ipo and rpo_alpha divide by.  With rpo_alpha
    the dict also has 'nll_loss' and '_stats' a 9th lane."""
    obj = _objective(objective, DpoObjective)
    if obj is not None and obj.reference_free:
        ref_lp = None
    elif ref_lp is None:
        raise ValueError('ref_lp is None: only a reference_free objective runs without the reference log-probs')
    L.require_cuda(policy_lp, ref_lp)
    if policy_lp.dim() != 2 or policy_lp.size(0) % 2 or (ref_lp is not None and policy_lp.shape != ref_lp.shape):
        raise ValueError('policy / reference log-probs must both be (2B, W)')
    if response_lens is not None and len(response_lens) != policy_lp.size(0):
        raise ValueError('need one response_len per row of the log-probs')
    policy_lp = policy_lp if policy_lp.stride(1) == 1 or policy_lp.size(1) <= 1 else policy_lp.contiguous()
    if ref_lp is not None:
        ref_lp = ref_lp.to(policy_lp.dtype).contiguous()
        if policy_lp.stride(0) != ref_lp.stride(0):
            policy_lp = policy_lp.contiguous()
        ref_lp = ref_lp.detach()
    mode_code = _mode_code(mode, policy_lp.dtype)
    ids = input_ids if skip_identical_pairs else None
    counts = _dpo_counts(obj, response_lens, policy_lp.device)
    loss, per_pair, stats = _DpoFromLpFn.apply(policy_lp, ref_lp, scale_coeff, mode_code, ids, obj, counts)
    out_dtype = policy_lp.dtype if mode_code == L.MODE_FAITHFUL else torch.float32
    out = _dpo_outputs(loss, per_pair, stats, out_dtype, skip_identical_pairs, obj)
    out['_per_pair'] = per_pair
    return out


class _DpoFusedFn(torch.autograd.Function):
    """policy logits (grad) + reference logits (no grad) -> DPO loss.  Forward: K1 x2 (x1 reference-free), K2.
    Backward: ONE K1b launch taking the per-sample coefficient straight from K2 (no per-row gradient tensor)."""

    @staticmethod
    def forward(ctx, policy_logits, ref_logits, labels, plan, scale_coeff, mode_code, ids, coll=None, obj=None,
                counts=None):
        dev = policy_logits.device
        out_dtype = policy_logits.dtype if mode_code == L.MODE_FAITHFUL else torch.float32
        lp = torch.zeros((2,) + plan.out_shape, dtype=out_dtype, device=dev)
        need_grad = ctx.needs_input_grad[0]
        stats_rows = torch.empty((2, max(plan.n_rows, 1)), dtype=torch.float32, device=dev) if need_grad else None
        _launch_fwd(policy_logits, labels, plan, lp[0], stats_rows[0] if need_grad else None,
                    stats_rows[1] if need_grad else None)
        if ref_logits is not None:
            _launch_fwd(ref_logits, labels, plan, lp[1], None, None)
        res = _dpo_launch(lp[0], lp[1] if ref_logits is not None else None, scale_coeff, mode_code, ids, True, coll,
                          obj, counts)
        per_pair, stats, grad_seg = res[0], res[1], res[2]
        stats_global = res[3] if coll is not None else stats
        if need_grad:
            ctx.save_for_backward(policy_logits, labels, stats_rows, grad_seg)
            ctx.plan, ctx.mode_code = plan, mode_code
        ctx.mark_non_differentiable(per_pair, stats, lp, stats_global)
        return stats[0].to(out_dtype), per_pair, stats, lp, stats_global

    @staticmethod
    def backward(ctx, g_loss, *_):
        logits, labels, stats_rows, grad_seg = ctx.saved_tensors
        grad = torch.empty(logits.shape, dtype=logits.dtype, device=logits.device)
        scale = g_loss.detach().to(torch.float32).reshape(1).contiguous()
        _launch_bwd(logits, labels, ctx.plan, stats_rows[0], stats_rows[1], None, grad_seg, scale, grad,
                    ctx.mode_code)
        return grad, None, None, None, None, None, None, None, None, None


def dpo_fused_loss(policy_logits: torch.Tensor, ref_logits: torch.Tensor | None, input_ids: torch.Tensor,
                   response_lens: Sequence[int], pad_id: int, scale_coeff: float, strip: bool = True,
                   skip_identical_pairs: bool = False, mode: str | None = None, coll=None,
                   objective: DpoObjective | None = None) -> dict[str, torch.Tensor]:
    """The whole of DPOTrainer.loss after the two model forwards (trainers/text_to_text/dpo.py:144-203):
    5 launches forward (label extraction, K1 policy, K1 reference, K2), 1 launch backward (K1b).  objective: a
    DpoObjective; reference-free, ref_logits may be None and is not read (no reference K1)."""
    obj = _objective(objective, DpoObjective)
    if obj is not None and obj.reference_free:
        ref_logits = None
    elif ref_logits is None:
        raise ValueError('ref_logits is None: only a reference_free objective runs without the reference model')
    L.require_cuda(policy_logits, ref_logits, input_ids)
    if policy_logits.dim() != 3 or (ref_logits is not None and policy_logits.shape != ref_logits.shape):
        raise ValueError('policy / reference logits must both be (2B, L, V)')
    if policy_logits.size(0) % 2 or policy_logits.size(0) != len(response_lens):
        raise ValueError('need 2B rows (chosen first, rejected second) and one response_len per row')
    lens = tuple(int(r) for r in response_lens)
    labels = strip_pad_tail(input_ids, lens, pad_id, strip)
    policy_logits = _contiguous_last(policy_logits)
    if ref_logits is not None:
        ref_logits = ref_logits.detach()
        if ref_logits.stride() != policy_logits.stride() or ref_logits.dtype != policy_logits.dtype:
            ref_logits = ref_logits.to(policy_logits.dtype).contiguous()
            if ref_logits.stride() != policy_logits.stride():
                policy_logits = policy_logits.contiguous()
    plan = _dpo_plan(policy_logits, lens, labels.stride(0))
    mode_code = _mode_code(mode, policy_logits.dtype)
    ids = input_ids if skip_identical_pairs else None
    counts = _dpo_counts(obj, lens, policy_logits.device)
    loss, per_pair, stats, lp, stats_global = _DpoFusedFn.apply(policy_logits, ref_logits, labels, plan, scale_coeff,
                                                               mode_code, ids, coll, obj, counts)
    out_dtype = policy_logits.dtype if mode_code == L.MODE_FAITHFUL else torch.float32
    out = _dpo_outputs(loss, per_pair, stats, out_dtype, skip_identical_pairs, obj)
    if coll is not None:
        out['_stats_global'] = stats_global  # already averaged over the ranks by K2 itself (NVLink peer memory)
    out['_per_pair'] = per_pair
    out['_log_probs'] = lp
    return out


# ---- SimPO / ORPO / KTO pair bookkeeping ---------------------------------------------------------------
def pair_slices(input_ids: torch.Tensor, attention_mask: torch.Tensor) -> torch.Tensor:
    """trainers/text_to_text/simpo.py:61-77 for all pairs in one launch: int32 (4, B) = valid, diverge_index,
    end_better, end_worse (the reference: a Python loop with 4 host syncs per pair)."""
    L.require_cuda(input_ids, attention_mask)
    n, seq = input_ids.shape
    if n % 2 or attention_mask.shape != input_ids.shape:
        raise ValueError('input_ids / attention_mask must both be (2B, L)')
    ids = _contiguous_last(input_ids)
    mask = attention_mask
    kind = L.MASK_U8
    if mask.dtype == torch.int64:
        kind = L.MASK_I64
    elif mask.dtype != torch.bool:
        mask = mask != 0
    mask = _contiguous_last(mask)
    out = torch.empty((4, n // 2), dtype=torch.int32, device=ids.device)
    sc = _device_scratch(ids.device)
    L.check(L.lib().aa_pair_slices(ids.data_ptr(), ids.stride(0), mask.data_ptr(), kind, mask.stride(0), n // 2, seq,
                                   out.data_ptr(), sc['status'].data_ptr(), L.stream_ptr(ids.device)))
    return out


class _SliceSumFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, lp, slices, mode_code):
        n, W = lp.shape
        sums = torch.empty(n, dtype=torch.float32, device=lp.device)
        L.check(L.lib().aa_slice_sums(lp.data_ptr(), L.dtype_code(lp.dtype), lp.stride(0), n // 2, W, slices.data_ptr(),
                                      mode_code, sums.data_ptr(), L.stream_ptr(lp.device)))
        ctx.save_for_backward(slices)
        ctx.W, ctx.dtype = W, lp.dtype
        return sums.to(lp.dtype) if mode_code == L.MODE_FAITHFUL else sums

    @staticmethod
    def backward(ctx, g):
        (slices,) = ctx.saved_tensors
        B = slices.size(1)
        cols = torch.arange(ctx.W, device=g.device).unsqueeze(0)
        lo = slices[1].repeat(2).unsqueeze(1)
        hi = torch.cat([slices[2], slices[3]]).unsqueeze(1) + 1
        inside = (cols >= lo) & (cols < hi)
        return torch.where(inside, g.unsqueeze(1).to(ctx.dtype), torch.zeros((), dtype=ctx.dtype, device=g.device)), None, None


def slice_sums(sequence_log_probs: torch.Tensor, slices: torch.Tensor, mode: str | None = None) -> torch.Tensor:
    """sum(lp[r, diverge : end + 1]) for the 2B rows (simpo.py:78-79), one launch; differentiable in lp."""
    L.require_cuda(sequence_log_probs, slices)
    lp = _contiguous_last(sequence_log_probs)
    return _SliceSumFn.apply(lp, slices.contiguous(), _mode_code(mode, lp.dtype))


# ---- GRPO ---------------------------------------------------------------------------------------------
def group_advantages(rewards: torch.Tensor, num_generations: int, scale: bool = True) -> torch.Tensor:
    """trainers/text_to_text/grpo.py:268-274: rewards (B * G,) fp32 -> advantages (B * G, 1),
    (r - group mean) / (unbiased group std + 1e-4).  scale=False (Dr. GRPO): r - group mean."""
    L.require_cuda(rewards)
    r = rewards.detach().float().contiguous().view(-1)
    if r.numel() % num_generations:
        raise ValueError('rewards must hold B * num_generations values')
    adv = torch.empty_like(r)
    fn = L.lib().aa_group_advantages if scale else L.lib().aa_group_advantages_centered
    L.check(fn(r.data_ptr(), r.numel() // num_generations, int(num_generations), adv.data_ptr(), L.stream_ptr(r.device)))
    return adv.view(-1, 1)


class _GrpoLossFn(torch.autograd.Function):
    """GRPO's loss over per-token log-probs: the forward writes the loss and d loss / d lp in one launch
    (_grpo_loss_launch); obj / old / clip_frac select and feed the clipped objective."""

    @staticmethod
    def forward(ctx, lp, ref_lp, adv, tokens, eos_id, beta, mode_code, obj=None, old=None, clip_frac=None,
                sequence=False, topent=None, cov=None, pm=None):
        B, K = lp.shape
        dev = lp.device
        loss = torch.empty(1, dtype=torch.float32, device=dev)
        grad = torch.empty((B, K), dtype=lp.dtype, device=dev)
        row_end = torch.empty(B, dtype=torch.int32, device=dev)
        _grpo_loss_launch(lp, ref_lp, adv, tokens, eos_id, beta, mode_code, obj, old, loss, grad, clip_frac, row_end,
                          sequence=sequence, topent=topent, cov=cov, pm=pm)
        ctx.save_for_backward(grad)
        ctx.mark_non_differentiable(row_end)
        return loss[0], row_end

    @staticmethod
    def backward(ctx, g, _):
        (grad,) = ctx.saved_tensors
        return (grad.float() * g.float()).to(grad.dtype), None, None, None, None, None, None, None, None, None, None, None, \
            None, None


def _grpo_loss_launch(lp, ref_lp, adv, tokens, eos_id, beta, mode_code, obj, old, loss, grad, clip_frac, row_end,
                      scratch=None, sequence=False, topent=None, cov=None, pm=None):
    """GRPO's loss kernel, writing loss, row_end and (unless None) grad.  obj None: the reference loss (aa_grpo_loss);
    otherwise obj = _grpo_objective_args(...) for aa_grpo_loss_obj (aa_grpo_loss_kl unless the KL is k3), old = the old log-probs (None: the log-probs
    themselves, ratio 1) and clip_frac = an fp32[2] tensor for the clip fractions or None.  sequence (see
    _sequence_level; old is then given): GSPO's sequence-level ratio, aa_grpo_loss_seq.  topent: (entropy (B, K) fp32,
    thr fp32[1]) for the top-entropy mask, aa_grpo_loss_topent at either level (obj is then given).  scratch (fp32): the token
    count and the row sums, B + 1 values, and under the objective the rows' clip counts too, 1 + 4 B; None allocates it.
    cov (_CovTerm, obj given, token level): Clip-Cov / KL-Cov, the selection over GRPO's completion mask
    (grpo_row_end) then aa_grpo_loss_cov.  pm (_PmTerm, obj given, token level): CISPO / SAPO, aa_grpo_loss_pm."""
    B, K = lp.shape
    dev = lp.device
    if scratch is None:
        scratch = torch.empty(B + 1 if obj is None else 1 + 4 * B, dtype=torch.float32, device=dev)
    lib = L.lib()
    lps = (lp.data_ptr(), lp.stride(0), ref_lp.data_ptr(), ref_lp.stride(0))
    rows = (L.dtype_code(lp.dtype), adv.data_ptr(), tokens.data_ptr(), tokens.stride(0), int(eos_id), B, K, float(beta))
    out = (loss.data_ptr(), L.ptr(grad), grad.stride(0) if grad is not None else 0)
    tail = (row_end.data_ptr(), scratch.data_ptr(), _device_scratch(dev)['counter'][5:7].data_ptr(), L.stream_ptr(dev))
    if obj is None:
        L.check(lib.aa_grpo_loss(*lps, *rows, mode_code, *out, *tail))
    elif pm is not None:
        L.check(lib.aa_grpo_loss_pm(*lps, L.ptr(old), old.stride(0) if old is not None else 0, *rows, obj[1], obj[3],
                                    obj[4], pm.code, pm.tau_pos, pm.tau_neg, mode_code, *out, L.ptr(clip_frac), *tail))
    elif cov is not None:
        sel = _cov_select(lp, adv, old, None, grpo_row_end(tokens, eos_id), cov, obj[0], obj[1], mode_code)
        L.check(lib.aa_grpo_loss_cov(*lps, L.ptr(old), old.stride(0) if old is not None else 0, *rows, obj[0], obj[1],
                                     obj[3], obj[4], cov.code, cov.coef, sel.data_ptr(), sel.stride(0), mode_code, *out,
                                     L.ptr(clip_frac), *tail))
    elif topent is not None:
        ent, thr = topent
        L.check(lib.aa_grpo_loss_topent(*lps, L.ptr(old), old.stride(0) if old is not None else 0, *rows, *obj,
                                        int(bool(sequence)), mode_code, *out, L.ptr(clip_frac), ent.data_ptr(),
                                        ent.stride(0), thr.data_ptr(), *tail))
    elif sequence:
        L.check(lib.aa_grpo_loss_seq(*lps, old.data_ptr(), old.stride(0), *rows, *obj, mode_code, *out,
                                     L.ptr(clip_frac), *tail))
    elif obj[4] == KL_ESTIMATORS['k3']:
        L.check(lib.aa_grpo_loss_obj(*lps, L.ptr(old), old.stride(0) if old is not None else 0, *rows, *obj[:4],
                                     mode_code, *out, L.ptr(clip_frac), *tail))
    else:
        L.check(lib.aa_grpo_loss_kl(*lps, L.ptr(old), old.stride(0) if old is not None else 0, *rows, *obj, mode_code,
                                    *out, L.ptr(clip_frac), *tail))


def _grpo_objective_args(objective, old, return_clip_fraction: bool):
    """The one rule for GRPO's reference loss -- no objective or one with default fields, no old log-probs and no clip
    fractions: None, and the nodes run today's launches.  Otherwise GrpoObjective.args() and the KL estimator's code
    for the objective kernels (a default objective still gives its clip_range_ratio).  A sequence-level objective
    without old log-probs has w = 1: it is the token-level objective and takes its launches."""
    if old is None and getattr(objective, 'sequence_level', False):
        objective = dataclasses.replace(objective, importance_sampling_level='token')
    if _objective(objective, GrpoObjective) is None and old is None and not return_clip_fraction:
        return None
    objective = objective or GrpoObjective()
    return objective.args() + (KL_ESTIMATORS[objective.kl_estimator],)


def _sequence_level(objective, old) -> bool:
    """Whether GSPO's sequence-level ratio runs: a sequence-level objective with old log-probs (updates 2..mu).  Its
    tokens' gradients need the whole row's log-ratio first, so it runs on the composed path (aa_grpo_loss_seq), never
    on K1f's single pass."""
    return old is not None and getattr(objective, 'sequence_level', False)


def _top_entropy(objective) -> bool:
    """Whether the top-entropy mask runs (top_entropy_quantile < 1).  Every token's gradient needs the global entropy
    threshold first, so it runs on the composed path (selection -> aa_grpo_loss_topent), never on K1f's single pass."""
    return getattr(objective, 'top_entropy_quantile', 1.0) < 1.0


def grpo_row_end(completion_tokens: torch.Tensor, eos_token_id: int) -> torch.Tensor:
    """GRPO's completion mask as counted tokens per row: int32 (B,), row_end[b] = the tokens up to and including the
    first eos (K without one).  The GRPO loss kernels' own mask pass (aa_grpo_row_end), one launch."""
    L.require_cuda(completion_tokens)
    if completion_tokens.dim() != 2 or completion_tokens.numel() == 0:
        raise ValueError(f'completion tokens must be a non-empty (B, K) tensor, got {tuple(completion_tokens.shape)}')
    tok = _contiguous_last(completion_tokens.to(torch.int64))
    B, K = tok.shape
    dev = tok.device
    row_end = torch.empty(B, dtype=torch.int32, device=dev)
    total = torch.empty(1, dtype=torch.float32, device=dev)
    L.check(L.lib().aa_grpo_row_end(tok.data_ptr(), tok.stride(0), int(eos_token_id), B, K, row_end.data_ptr(),
                                    total.data_ptr(), _device_scratch(dev)['counter'][5:6].data_ptr(),
                                    L.stream_ptr(dev)))
    return row_end


_ENT_BINS = 1 << 16  # include/aa_b200.h aa_entropy_hist_hi / _lo: 16 bits a pass


def entropy_quantile_threshold(entropy: torch.Tensor, row_end_or_mask: torch.Tensor, q: float,
                               group=None) -> torch.Tensor:
    """torch.quantile(entropy[counted], q) (linear interpolation) over the counted tokens of every rank of `group`
    (torch.distributed; None: the default group) when torch.distributed is initialised with more than one rank, else
    over the local ones -> fp32 (1,) on the device.  entropy: fp32 (B, K); row_end_or_mask: int (B,) counted tokens per
    row (t < row_end[b], GRPO's completion mask: grpo_row_end) or a bool / integer (B, K) mask.  NaN when nothing is
    counted or a counted entropy is NaN (then `entropy >= thr` keeps nothing).
    Exact: a radix select on order-preserving keys, 16 bits a pass (aa_entropy_hist_hi, aa_entropy_select_hi,
    aa_entropy_hist_lo, aa_entropy_select_lo), the rank fp32 q * (N - 1) and ATen's lerp, so the value equals CUDA
    torch.quantile's wherever that accepts the input (up to 2^24 values) and keeps its formula beyond.  Across ranks
    the two histograms (integer counts) are all-reduced with SUM; no host sync.  Bad arguments raise ValueError here,
    before any launch."""
    if isinstance(q, bool) or not isinstance(q, (int, float)) or not 0.0 <= float(q) <= 1.0:
        raise ValueError(f'entropy_quantile_threshold: q must be a number in [0, 1], got {q!r}')
    if not isinstance(entropy, torch.Tensor) or entropy.dim() != 2 or entropy.numel() == 0 or \
            entropy.dtype != torch.float32:
        raise ValueError(f'entropy_quantile_threshold: entropy must be a non-empty fp32 (B, K) tensor, got '
                         f'{getattr(entropy, "dtype", None)} {tuple(getattr(entropy, "shape", ()))}')
    B, K = entropy.shape
    if B * K > 2 ** 31 - 1:
        raise ValueError(f'entropy_quantile_threshold: B * K = {B * K} exceeds 2^31 - 1')
    m = row_end_or_mask
    if not isinstance(m, torch.Tensor) or tuple(m.shape) not in ((B,), (B, K)) or \
            (m.dim() == 1 and (m.dtype.is_floating_point or m.dtype == torch.bool)):
        raise ValueError(f'entropy_quantile_threshold: row_end_or_mask must be integer (B,) = ({B},) row ends or a '
                         f'(B, K) = ({B}, {K}) mask, got {getattr(m, "dtype", None)} {tuple(getattr(m, "shape", ()))}')
    try:
        L.require_cuda(entropy, m)
    except RuntimeError as e:
        raise ValueError(f'entropy_quantile_threshold: {e}') from None
    dev = entropy.device
    ent = _contiguous_last(entropy.detach())
    if m.dim() == 1:
        row_end, mask, mask_stride = m.to(torch.int32).contiguous(), None, 0
    else:
        row_end, mask = None, _contiguous_last((m != 0).to(torch.uint8))
        mask_stride = mask.stride(0)
    hist_hi = torch.empty(_ENT_BINS + 1, dtype=torch.int32, device=dev)  # uint32 counts; + the NaN count
    hist_lo = torch.empty(2 * _ENT_BINS, dtype=torch.int32, device=dev)
    sel = torch.empty(8, dtype=torch.int32, device=dev)
    thr = torch.empty(1, dtype=torch.float32, device=dev)
    lib, stream = L.lib(), L.stream_ptr(dev)
    counted = (L.ptr(row_end), L.ptr(mask), mask_stride, B, K)
    dist = torch.distributed
    many = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
    L.check(lib.aa_entropy_hist_hi(ent.data_ptr(), ent.stride(0), *counted, hist_hi.data_ptr(), stream))
    if many:
        dist.all_reduce(hist_hi, op=dist.ReduceOp.SUM, group=group)
    L.check(lib.aa_entropy_select_hi(hist_hi.data_ptr(), float(q), sel.data_ptr(), stream))
    L.check(lib.aa_entropy_hist_lo(ent.data_ptr(), ent.stride(0), *counted, sel.data_ptr(), hist_lo.data_ptr(), stream))
    if many:
        dist.all_reduce(hist_lo, op=dist.ReduceOp.SUM, group=group)
    L.check(lib.aa_entropy_select_lo(hist_lo.data_ptr(), sel.data_ptr(), thr.data_ptr(), stream))
    return thr


def _top_entropy_args(objective, entropy, tok, eos_token_id, shape):
    """(entropy, thr) of the top-entropy mask for _grpo_loss_launch, or None when the objective keeps every token.
    thr: entropy_quantile_threshold at q = 1 - top_entropy_quantile over GRPO's completion mask."""
    if not _top_entropy(objective):
        return None
    if not isinstance(entropy, torch.Tensor) or tuple(entropy.shape) != tuple(shape):
        raise ValueError(f'top_entropy_quantile < 1 needs the policy entropy, a {tuple(shape)} tensor; got '
                         f'{tuple(getattr(entropy, "shape", ())) if entropy is not None else None}')
    ent = _contiguous_last(entropy.detach().float())
    thr = entropy_quantile_threshold(ent, grpo_row_end(tok, eos_token_id), 1.0 - objective.top_entropy_quantile)
    return ent, thr


def _old_log_probs(old, shape, dtype):
    """The rollout-time policy log-probs for the objective kernels: detached, contiguous, in the log-probs' dtype."""
    if old is None:
        return None
    if tuple(old.shape) != tuple(shape):
        raise ValueError(f'old_per_token_logps must be {tuple(shape)}, got {tuple(old.shape)}')
    return _contiguous_last(old.detach().to(dtype)).contiguous()


def grpo_loss(per_token_logps: torch.Tensor, ref_per_token_logps: torch.Tensor, advantages: torch.Tensor,
              completion_tokens: torch.Tensor, eos_token_id: int, beta: float, mode: str | None = None, *,
              objective: GrpoObjective | None = None, old_per_token_logps: torch.Tensor | None = None,
              return_clip_fraction: bool = False, entropy: torch.Tensor | None = None, cov_seed: int = 0):
    """The loss of GRPOTrainer.train_step (trainers/text_to_text/grpo.py:290-312): per-token k3 KL, per-token loss
    -(exp(lp - lp.detach()) * A - beta * KL), completion mask up to the first eos, token mean -> fp32 scalar,
    differentiable in per_token_logps.  Returns (loss, counted_tokens_per_row).
    objective (ops.GrpoObjective) / old_per_token_logps (the rollout-time policy log-probs, (B, K)): GRPO's clipped
    objective (aa_grpo_loss_obj) with ratio exp(lp - old); without old_per_token_logps the ratio is 1.  A sequence-level
    objective with old_per_token_logps: GSPO's one ratio per sequence (aa_grpo_loss_seq).  None / default fields and no
    old log-probs: today's launch.  return_clip_fraction appends the fp32[2] clip fractions.
    An objective with top_entropy_quantile = rho < 1 also needs `entropy`, the policy's fp32 entropy (B, K) of the same
    pass: only the counted tokens with entropy >= entropy_quantile_threshold(entropy, row_end, 1 - rho) (over every
    data-parallel rank) keep the policy term s; the others carry the KL term alone (aa_grpo_loss_topent).
    An objective with policy_loss_mode clip_cov / kl_cov: the selection of cov_token_selection over the completion mask
    (Clip-Cov hashes with cov_seed, see cov_hash_seed), then aa_grpo_loss_cov; its fp32 (1,) selected share follows
    row_end, before the clip fractions."""
    L.require_cuda(per_token_logps, ref_per_token_logps, advantages, completion_tokens)
    obj = _grpo_objective_args(objective, old_per_token_logps, return_clip_fraction)
    if per_token_logps.dim() != 2 or per_token_logps.shape != ref_per_token_logps.shape or \
            completion_tokens.shape != per_token_logps.shape:
        raise ValueError('per-token log-probs and completion tokens must all be (B, K)')
    lp = _contiguous_last(per_token_logps)
    rlp = _contiguous_last(ref_per_token_logps.detach().to(lp.dtype))
    adv = advantages.detach().float().contiguous().view(-1)
    if adv.numel() != lp.size(0):
        raise ValueError('one advantage per sequence expected')
    old = _old_log_probs(old_per_token_logps, lp.shape, lp.dtype)
    tok = _contiguous_last(completion_tokens.to(torch.int64))
    cf = torch.zeros(2, dtype=torch.float32, device=lp.device) if return_clip_fraction else None
    topent = _top_entropy_args(objective, entropy, tok, eos_token_id, lp.shape)
    cov = _cov_term(_objective(objective, GrpoObjective), cov_seed, lp.device)
    out = _GrpoLossFn.apply(lp, rlp, adv, tok, eos_token_id, beta, _mode_code(mode, lp.dtype), obj, old, cf,
                            _sequence_level(objective, old), topent, cov, _pm_term(_objective(objective, GrpoObjective)))
    if cov is not None:
        out += (cov.share,)
    return out + (cf,) if return_clip_fraction else out


def tail_token_log_probs(logits: torch.Tensor, input_ids: torch.Tensor, logits_to_keep: int, mode: str | None = None,
                         return_entropy: bool = False, entropy_grad: bool = False):
    """GRPOTrainer._get_per_token_logps after the model forward (trainers/text_to_text/grpo.py:205-210):
    log-probs of input_ids[:, -K:] under logits[:, :-1][:, -K:], one K1 launch, (B, K).  return_entropy: and the fp32
    entropy (B, K) of the same rows from that launch; entropy_grad: differentiable too (see _LogProbFn)."""
    L.require_cuda(logits, input_ids)
    B, seq, _ = logits.shape
    K = int(logits_to_keep)
    if not 0 < K < seq:
        raise ValueError('logits_to_keep must lie in (0, L)')
    logits = _contiguous_last(logits)
    lens = (K,) * B
    labels = strip_pad_tail(input_ids, lens, 0, strip=False)
    plan = _tail_plan(lens, seq, logits.stride(0), logits.stride(1), K, 0, -1, None, str(logits.device))
    if return_entropy:
        return _log_probs_and_entropy(logits, labels, plan, _mode_code(mode, logits.dtype), 0,
                                      entropy_grad and logits.requires_grad and torch.is_grad_enabled())
    return _LogProbFn.apply(logits, labels, plan, _mode_code(mode, logits.dtype))


class _GrpoFusedFn(torch.autograd.Function):
    """GRPO's policy log-probs, loss and d loss / d logits as ONE autograd node on K1f (aa_logprob_grpo_fused): the
    per-token loss needs the token's own log-prob, the reference log-prob and the sequence's advantage -- all there
    before the policy tile is read -- so the gradient tile is written in the same pass; aa_grpo_loss reduces the loss
    value from the log-probs that pass wrote."""

    @staticmethod
    def forward(ctx, logits, labels, plan, ref_lp, adv, tokens, eos_id, beta, mode_code, entropy=None,
                entropy_coeff=0.0, obj=None, old=None, clip_frac=None, pm=None):
        """obj: GrpoObjective.args() for aa_logprob_grpo_fused_obj + aa_grpo_loss_obj (old: the old log-probs or None,
        clip_frac: an fp32[2] tensor for the clip fractions or None); None: today's launches.  pm (_PmTerm, obj
        given): CISPO / SAPO, aa_logprob_grpo_fused_pm + aa_grpo_loss_pm."""
        dev = logits.device
        B, K = plan.out_shape
        lp_dtype = logits.dtype if mode_code == L.MODE_FAITHFUL else torch.float32
        lp = torch.zeros((B, K), dtype=lp_dtype, device=dev)
        grad = torch.empty(logits.shape, dtype=logits.dtype, device=dev)
        rows = torch.empty(plan.n_tile_rows * 6, dtype=torch.int64, device=dev)  # 48 bytes per tile row
        row_end = torch.empty(B, dtype=torch.int32, device=dev)
        scratch = torch.empty(B + 1, dtype=torch.float32, device=dev)  # K1f's token count; aa_grpo_loss's scratch too
        loss = torch.empty(1, dtype=torch.float32, device=dev)
        _k1f_grpo_launch(logits, labels, plan, lp, ref_lp, adv, tokens, eos_id, beta, mode_code, grad, rows, row_end,
                         scratch, entropy, entropy_coeff, obj, old, pm)
        _grpo_loss_launch(lp, ref_lp, adv, tokens, eos_id, beta, mode_code, obj, old, loss, None, clip_frac, row_end,
                          scratch if obj is None else None, pm=pm)
        ctx.save_for_backward(grad)
        if entropy_coeff == 0.0:
            ctx.mark_non_differentiable(lp, row_end)
            return loss[0], lp, row_end
        h_mean = _completion_mean(entropy, row_end)
        plain = loss[0].clone()
        ctx.mark_non_differentiable(lp, row_end, h_mean, plain)  # one call: a second one would replace the first
        return loss[0] - entropy_coeff * h_mean, lp, row_end, h_mean, plain

    @staticmethod
    def backward(ctx, g, *_unused):
        (grad,) = _hand_over_once(ctx, g, *ctx.saved_tensors)
        return grad, None, None, None, None, None, None, None, None, None, None, None, None, None, None


def _k1f_grpo_launch(logits, labels, plan, lp, ref_lp, adv, tokens, eos_id, beta, mode_code, grad, rows, row_end,
                     total, entropy, entropy_coeff, obj, old, pm=None):
    """K1f over GRPO's completion rows (`rows`: its int64 row records, 6 per tile row), writing lp, row_end, the token
    count `total[0]`, the gradient tile `grad` and (unless None) the fp32 entropy.  obj: GrpoObjective.args() for the objective entry point (aa_logprob_grpo_fused_obj, old: the old
    log-probs or None); None: the reference loss, plain, with the entropy, or with the entropy bonus's gradient.
    pm (_PmTerm, obj given): CISPO / SAPO's entry point (aa_logprob_grpo_fused_pm)."""
    dev = logits.device
    K = plan.out_shape[1]
    sc = _device_scratch(dev)
    p = plan.ptrs()
    lib = L.lib()
    head = (logits.data_ptr(), L.dtype_code(logits.dtype), logits.stride(-2), logits.size(-1), labels.data_ptr(),
            plan.n_seg, p[0], p[1], p[2], p[3], p[4], plan.n_tile_rows, lp.data_ptr(), L.dtype_code(lp.dtype),
            ref_lp.data_ptr(), ref_lp.stride(0))
    mid = (adv.data_ptr(), tokens.data_ptr(), tokens.stride(0), int(eos_id), K, float(beta))
    tail = (mode_code, grad.data_ptr(), logits.size(-1), rows.data_ptr(), row_end.data_ptr(), total.data_ptr(),
            sc['counter'][5:6].data_ptr(), sc['status'].data_ptr())
    if pm is not None:
        L.check(lib.aa_logprob_grpo_fused_pm(*head, L.ptr(old), *mid, obj[1], obj[3], obj[4], pm.code, pm.tau_pos,
                                             pm.tau_neg, *tail, L.ptr(entropy), float(entropy_coeff),
                                             L.stream_ptr(dev)))
    elif obj is not None and obj[4] == KL_ESTIMATORS['k3']:
        L.check(lib.aa_logprob_grpo_fused_obj(*head, L.ptr(old), *mid, *obj[:4], *tail, L.ptr(entropy),
                                              float(entropy_coeff), L.stream_ptr(dev)))
    elif obj is not None:  # another KL estimator: the same kernel with the estimator's code
        L.check(lib.aa_logprob_grpo_fused_kl(*head, L.ptr(old), *mid, *obj, *tail, L.ptr(entropy),
                                             float(entropy_coeff), L.stream_ptr(dev)))
    elif entropy is None:
        L.check(lib.aa_logprob_grpo_fused(*head, *mid, *tail, L.stream_ptr(dev)))
    elif entropy_coeff == 0.0:  # the same launch with the entropy of every completion row from its (max, sum-exp) pass
        L.check(lib.aa_logprob_grpo_fused_entropy(*head, *mid, *tail, entropy.data_ptr(), L.stream_ptr(dev)))
    else:  # ... and the entropy bonus's gradient in the tile
        L.check(lib.aa_logprob_grpo_fused_entropy_grad(*head, *mid, *tail, entropy.data_ptr(), float(entropy_coeff),
                                                       L.stream_ptr(dev)))


def _completion_mean(x: torch.Tensor, row_end: torch.Tensor) -> torch.Tensor:
    """GRPO's token mean of x (B, K) over the completion mask (tokens up to and including the first eos)."""
    mask = torch.arange(x.size(1), device=x.device) < row_end.unsqueeze(1)
    return (x * mask).sum() / mask.sum()


def grpo_loss_from_logits(logits: torch.Tensor, input_ids: torch.Tensor, logits_to_keep: int,
                          ref_per_token_logps: torch.Tensor, advantages: torch.Tensor, eos_token_id: int, beta: float,
                          mode: str | None = None, return_entropy: bool = False, entropy_coeff: float = 0.0, *,
                          objective: GrpoObjective | None = None, old_per_token_logps: torch.Tensor | None = None,
                          return_clip_fraction: bool = False, cov_seed: int = 0):
    """`_get_per_token_logps` of the policy + the loss of GRPOTrainer.train_step (trainers/text_to_text/grpo.py:205-210,
    290-312) from the policy's logits; the reference model's per-token log-probs must already be there.
    -> (loss fp32 scalar, policy per-token log-probs (B, K), counted tokens per row).  With a gradient: one pass over the
    completion rows (see _GrpoFusedFn); otherwise tail_token_log_probs + grpo_loss.  return_entropy appends the fp32
    policy entropy (B, K) of the completion rows, from the same pass (K1f's phase A, or K1's entropy variant); the
    other outputs are bit-identical.  entropy_coeff != 0 (entropy bonus): the loss is
    loss - entropy_coeff * (H * mask).sum() / mask.sum()  over the completion mask, and the detached entropy mean and
    the detached GRPO loss without the bonus follow row_end (before the entropy when return_entropy); the single pass is K1f's entropy-gradient variant, the
    composed path K1's entropy variant -> grpo_loss -> K1b's entropy variant.
    objective / old_per_token_logps: GRPO's clipped objective as in grpo_loss (K1f's objective entry point, or K1 ->
    aa_grpo_loss_obj -> K1b); the entropy bonus stays a token mean over the completion mask.  A sequence-level objective
    with old log-probs always takes the composed path (K1 -> aa_grpo_loss_seq -> K1b, see _sequence_level), and so does
    top_entropy_quantile < 1 (K1's entropy variant -> the entropy threshold -> aa_grpo_loss_topent -> K1b, see
    _top_entropy), and so does policy_loss_mode clip_cov / kl_cov (K1 -> selection -> aa_grpo_loss_cov -> K1b, seeded
    by cov_seed; the fp32 (1,) selected share is appended before the clip fractions).  return_clip_fraction appends
    the fp32[2] clip fractions last.  None / default fields and no old log-probs: today's launches."""
    L.require_cuda(logits, input_ids, ref_per_token_logps, advantages)
    obj = _grpo_objective_args(objective, old_per_token_logps, return_clip_fraction)
    K = int(logits_to_keep)
    tokens = input_ids[:, -K:]
    coeff = float(entropy_coeff)
    topent = _top_entropy(objective)
    cov = getattr(objective, 'policy_loss_mode', 'vanilla') in COV_MODES
    if _sequence_level(objective, old_per_token_logps) or topent or cov or \
            not _single_pass_ok(logits, _FUSED_GRPO, torch.is_grad_enabled() and logits.requires_grad):
        ent = None
        if return_entropy or coeff != 0.0 or topent:
            lp, ent = tail_token_log_probs(logits, input_ids, K, mode=mode, return_entropy=True,
                                           entropy_grad=coeff != 0.0)
        else:
            lp = tail_token_log_probs(logits, input_ids, K, mode=mode)
        scored = grpo_loss(lp, ref_per_token_logps, advantages, tokens, eos_token_id, beta, mode=mode,
                           objective=objective, old_per_token_logps=old_per_token_logps,
                           return_clip_fraction=return_clip_fraction, cov_seed=cov_seed,
                           **({'entropy': ent} if topent else {}))
        loss, row_end = scored[0], scored[1]
        out = (loss, lp.detach(), row_end)
        if coeff != 0.0:
            h_mean = _completion_mean(ent, row_end)
            out = (loss - coeff * h_mean, lp.detach(), row_end, h_mean.detach(), loss.detach())
        if return_entropy:
            out += (ent.detach(),)
        if cov:
            out += (scored[2],)
        return out + (scored[-1],) if return_clip_fraction else out
    B, seq, _ = logits.shape
    if not 0 < K < seq:
        raise ValueError('logits_to_keep must lie in (0, L)')
    if tuple(ref_per_token_logps.shape) != (B, K):
        raise ValueError('ref_per_token_logps must be (B, logits_to_keep)')
    logits = _contiguous_last(logits)
    mode_code = _mode_code(mode, logits.dtype)
    lp_dtype = logits.dtype if mode_code == L.MODE_FAITHFUL else torch.float32
    lens = (K,) * B
    labels = strip_pad_tail(input_ids, lens, 0, strip=False)
    plan = _tail_plan(lens, seq, logits.stride(0), logits.stride(1), K, 0, -1, None, str(logits.device))
    rlp = _contiguous_last(ref_per_token_logps.detach().to(lp_dtype))
    adv = advantages.detach().float().contiguous().view(-1)
    if adv.numel() != B:
        raise ValueError('one advantage per sequence expected')
    old = _old_log_probs(old_per_token_logps, (B, K), lp_dtype)
    tok = _contiguous_last(tokens.to(torch.int64))
    ent = torch.zeros((B, K), dtype=torch.float32, device=logits.device) if return_entropy or coeff != 0.0 else None
    cf = torch.zeros(2, dtype=torch.float32, device=logits.device) if return_clip_fraction else None
    out = _GrpoFusedFn.apply(logits, labels, plan, rlp, adv, tok, int(eos_token_id), float(beta), mode_code, ent, coeff,
                             obj, old, cf, _pm_term(_objective(objective, GrpoObjective)))
    if return_entropy:
        out += (ent,)
    return out + (cf,) if return_clip_fraction else out


# ---- reward-model pairwise loss -----------------------------------------------------------------------
class _RmPairLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, end_scores, regularization):
        n = end_scores.numel()
        dev = end_scores.device
        out = torch.empty(2, dtype=torch.float32, device=dev)
        grad = torch.empty(n, dtype=torch.float32, device=dev)
        L.check(L.lib().aa_rm_pair_loss(end_scores.data_ptr(), n // 2, float(regularization), out.data_ptr(),
                                        grad.data_ptr(), L.stream_ptr(dev)))
        ctx.save_for_backward(grad)
        ctx.shape = end_scores.shape
        ctx.mark_non_differentiable(out)
        return out[0].clone(), out

    @staticmethod
    def backward(ctx, g, _):
        (grad,) = ctx.saved_tensors
        return (grad * g).view(ctx.shape), None


def rm_pair_loss(end_scores: torch.Tensor, regularization: float = 0.0) -> dict[str, torch.Tensor]:
    """The loss tail of RMTrainer.loss (trainers/text_to_text/rm.py:111-124): end_scores (2B,) or (2B, 1)
    fp32, higher rows first -> {'loss', 'accuracy', 'higher_end_reward', 'lower_end_reward'}; one launch for
    forward + backward."""
    L.require_cuda(end_scores)
    flat = end_scores.reshape(-1)
    if flat.numel() % 2:
        raise ValueError('end_scores must hold 2B values (higher first, lower second)')
    flat = flat.float().contiguous()
    loss, out = _RmPairLossFn.apply(flat, regularization)
    higher, lower = flat.detach().chunk(2)
    return {'loss': loss, 'accuracy': out[1], 'higher_end_reward': higher, 'lower_end_reward': lower, '_stats': out}


# ---- cost-model pairwise loss -------------------------------------------------------------------------
class _CostPairLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, end_scores, better, worse, scale_coeff, regularization, mode_code, out_dtype):
        n = end_scores.numel()
        dev = end_scores.device
        loss = torch.empty((), dtype=out_dtype, device=dev)
        stats = torch.empty(2, dtype=torch.float32, device=dev)
        grad = torch.empty(n, dtype=end_scores.dtype, device=dev)
        L.check(L.lib().aa_cost_pair_loss(end_scores.data_ptr(), L.dtype_code(end_scores.dtype), better.data_ptr(),
                                          L.dtype_code(better.dtype), worse.data_ptr(), L.dtype_code(worse.dtype), n // 2,
                                          float(scale_coeff), float(regularization), mode_code, loss.data_ptr(),
                                          stats.data_ptr(), grad.data_ptr(), L.stream_ptr(dev)))
        ctx.save_for_backward(grad)
        ctx.mark_non_differentiable(stats)
        return loss, stats

    @staticmethod
    def backward(ctx, g, _):
        (grad,) = ctx.saved_tensors
        return grad * g, None, None, None, None, None, None


def cost_pair_loss(end_scores: torch.Tensor, better_signs, worse_signs, scale_coeff: float, regularization: float = 0.0,
                   mode: str | None = None) -> dict[str, torch.Tensor]:
    """The loss tail of CMTrainer.loss (trainers/text_to_text/cost_model.py:111-144): end_scores (2B,) or (2B, 1) in
    bf16 / f16 / fp32, higher-cost rows first; better_signs / worse_signs are meta_info's is_better_safe /
    is_worse_safe lists -> {'loss', 'accuracy', 'higher_end_reward', 'lower_end_reward', '_stats'}; one launch for
    forward + backward.

    Each sign list becomes a tensor through `torch.tensor(list)` as in the reference, so its dtype (int64, fp32 or
    bool) decides the arithmetic: h * sb is in torch.result_type(h, sb), and the loss is fp32 as soon as one product
    is.  The loss has the reference's dtype in both modes.  A sign list whose length is not B raises RuntimeError
    (the reference's broadcast would accept a one-element list; the collator never produces one).  Every error is
    raised on the host, before the launch."""
    flat = end_scores.reshape(-1)
    if flat.numel() % 2:
        raise ValueError('end_scores must hold 2B values (higher-cost rows first, lower-cost second)')
    B = flat.numel() // 2
    flat = flat.contiguous()
    sb, sw = torch.tensor(better_signs), torch.tensor(worse_signs)
    for name, s in (('is_better_safe', sb), ('is_worse_safe', sw)):
        if s.dim() != 1 or s.numel() != B:
            raise RuntimeError(f'{name} holds {s.numel()} values for {B} pairs: the sizes of the end scores '
                               f'and the signs must match')
    L.require_cuda(end_scores)
    sb, sw = sb.to(torch.result_type(flat, sb)), sw.to(torch.result_type(flat, sw))
    # both sign vectors go to the device in ONE copy (the second starts 4-byte aligned)
    off = (sb.numel() * sb.element_size() + 3) // 4 * 4
    host = torch.zeros(off + sw.numel() * sw.element_size(), dtype=torch.uint8)
    host[:sb.numel() * sb.element_size()] = sb.view(torch.uint8)
    host[off:] = sw.view(torch.uint8)
    signs = host.to(flat.device)
    d_sb, d_sw = signs[:sb.numel() * sb.element_size()].view(sb.dtype), signs[off:].view(sw.dtype)
    out_dtype = torch.promote_types(sb.dtype, sw.dtype)
    loss, stats = _CostPairLossFn.apply(flat, d_sb, d_sw, scale_coeff, regularization,
                                        _mode_code(mode, flat.dtype), out_dtype)
    higher, lower = flat.detach().chunk(2)
    return {'loss': loss, 'accuracy': stats[1], 'higher_end_reward': higher, 'lower_end_reward': lower,
            '_stats': stats}


# ---- causal-LM cross-entropy (SFT loss, PPO ptx term) -------------------------------------------------
class _CausalLMLossFn(torch.autograd.Function):
    """Mean NLL over labels != ignore_index, times `loss_scale`.
    With a gradient (default, K1f): ONE pass over the valid rows produces the fp32 log-probs AND the gradient tile
    (every valid row's upstream gradient is the same -loss_scale / n_valid, counted on the device before the pass;
    each row is streamed twice by one CTA, the second time out of L2); backward hands the tile over, multiplied in
    place only if the incoming scalar is not 1.  `single_pass` False (see _single_pass_ok) / no gradient: K1 in fp32
    mode over every position (ignored labels cost no traffic), mean-NLL epilogue; backward: one K1b launch with the
    scalar -loss_scale / n_valid as upstream gradient.  -> (loss_scale * loss, loss)."""

    @staticmethod
    def forward(ctx, logits, shift_labels, ignore_index, loss_scale, single_pass):
        B, seq, V = logits.shape
        dev = logits.device
        plan = _dense_plan(B, seq, logits.stride(0) if B > 1 else seq * logits.stride(1), logits.stride(1), seq, 0, seq,
                           B * seq, str(dev))
        need_grad = ctx.needs_input_grad[0]
        ctx.fused = bool(single_pass)
        sc = _device_scratch(dev)
        out = torch.empty(3, dtype=torch.float32, device=dev)  # [loss, -1 / n_valid, -loss_scale / n_valid]
        if ctx.fused:
            logp = torch.zeros((B, seq), dtype=torch.float32, device=dev)
            grad = torch.empty(logits.shape, dtype=logits.dtype, device=dev)
            scratch = torch.empty(B * seq * 6, dtype=torch.int64, device=dev)  # 48 bytes per tile row
            p = plan.ptrs()
            L.check(L.lib().aa_logprob_ce_fused(
                logits.data_ptr(), L.dtype_code(logits.dtype), logits.stride(-2), V, shift_labels.data_ptr(), B * seq,
                int(ignore_index), plan.n_seg, p[0], p[1], p[2], p[3], p[4], B * seq, logp.data_ptr(), float(loss_scale),
                grad.data_ptr(), V, scratch.data_ptr(), out[2:3].data_ptr(), sc['status'].data_ptr(), L.stream_ptr(dev)))
        else:
            logp = torch.empty((B, seq), dtype=torch.float32, device=dev)
            stats = torch.empty((2, B * seq), dtype=torch.float32, device=dev) if need_grad else None
            _launch_fwd(logits, shift_labels, plan, logp, stats[0] if need_grad else None, stats[1] if need_grad else None,
                        ignore_index=ignore_index)
        partial = torch.empty(512, dtype=torch.float32, device=dev)
        L.check(L.lib().aa_nll_mean(logp.data_ptr(), L.AA_F32, shift_labels.data_ptr(), B * seq, int(ignore_index),
                                    out[0:1].data_ptr(), out[1:2].data_ptr(), partial.data_ptr(),
                                    sc['counter'][4:5].data_ptr(), L.stream_ptr(dev)))
        if ctx.fused:
            ctx.save_for_backward(grad)
        elif need_grad:
            ctx.save_for_backward(logits, shift_labels, stats, out)
            ctx.plan, ctx.ignore_index = plan, int(ignore_index)
        ctx.loss_scale = float(loss_scale)
        loss = out[0]
        scaled = loss if loss_scale == 1.0 else loss * float(loss_scale)
        ctx.mark_non_differentiable(loss)
        return scaled.clone() if scaled is loss else scaled, loss

    @staticmethod
    def backward(ctx, g, _unused):
        if ctx.fused:
            (grad,) = _hand_over_once(ctx, g, *ctx.saved_tensors)
            return grad, None, None, None, None
        logits, shift_labels, stats, out = ctx.saved_tensors
        grad = torch.empty(logits.shape, dtype=logits.dtype, device=logits.device)
        scale = (out[1] * (g.float() * ctx.loss_scale)).reshape(1).contiguous()
        _launch_bwd(logits, shift_labels, ctx.plan, stats[0], stats[1], None, None, scale, grad, L.MODE_F32,
                    ignore_index=ctx.ignore_index)
        return grad, None, None, None, None


def _shifted_labels(logits: torch.Tensor, labels: torch.Tensor, ignore_index: int):
    L.require_cuda(logits, labels)
    if logits.dim() != 3 or labels.shape != logits.shape[:2]:
        raise ValueError('expected logits (B, L, V) and labels (B, L)')
    logits = _contiguous_last(logits)
    if logits.size(0) > 1 and logits.stride(0) != logits.size(1) * logits.stride(1):
        logits = logits.contiguous()
    shift = torch.full(labels.shape, int(ignore_index), dtype=torch.int64, device=labels.device)
    shift[:, :-1] = labels[:, 1:]
    return logits, shift


def causal_lm_loss(logits: torch.Tensor, labels: torch.Tensor, ignore_index: int = -100) -> torch.Tensor:
    """The `outputs.loss` of an HF causal LM (transformers ForCausalLMLoss: logits upcast to fp32, labels
    shifted by one, mean cross-entropy over labels != ignore_index) without the fp32 copy of the logits
    tile or the (rows, V) log-softmax tile: the loss of SupervisedTrainer.loss
    (trainers/text_to_text/sft.py:95-98) and of PPOTrainer.ptx_step (trainers/text_to_text/ppo.py:400-408).
    logits (B, L, V) in the model dtype, labels (B, L) -> fp32 scalar, differentiable in logits."""
    logits, shift = _shifted_labels(logits, labels, ignore_index)
    single_pass = _single_pass_ok(logits, _FUSED_CE, torch.is_grad_enabled() and logits.requires_grad)
    return _CausalLMLossFn.apply(logits, shift, int(ignore_index), 1.0, single_pass)[0]


def causal_lm_loss_scaled(logits: torch.Tensor, labels: torch.Tensor, loss_scale: float, ignore_index: int = -100):
    """-> (loss_scale * loss, loss.detach()).  Backpropagate the FIRST: the gradient tile is born multiplied by
    `loss_scale` (ptx_step's `ptx_coeff * ptx_loss`, trainers/text_to_text/ppo.py:405), so no pass over the tile is spent
    on the multiplication; log the second."""
    logits, shift = _shifted_labels(logits, labels, ignore_index)
    single_pass = _single_pass_ok(logits, _FUSED_CE, torch.is_grad_enabled() and logits.requires_grad)
    return _CausalLMLossFn.apply(logits, shift, int(ignore_index), float(loss_scale), single_pass)


# ---- causal-LM cross-entropy from the last hidden states (fused lm_head SFT) ---------------------------------------
def causal_lm_valid_rows(labels: torch.Tensor, ignore_index: int = -100):
    """The rows a causal-LM cross-entropy scores: flat position b * L + t, t < L - 1, with labels[b, t + 1] !=
    ignore_index (prompt and padding rows never meet the head).  ONE `nonzero`, so ONE host read: SupervisedTrainer
    takes it before the model forward, when the queue is already drained by the previous step's read.
    -> (index (N,) int64 on the labels' device, N)."""
    B, seq = labels.shape
    valid = torch.zeros((B, seq), dtype=torch.bool, device=labels.device)
    valid[:, :-1] = labels[:, 1:] != int(ignore_index)
    idx = valid.view(-1).nonzero().view(-1)
    return idx, int(idx.numel())


def _ce_chunks(N: int, V: int, chunk_rows: int | None):
    """Row chunks (r0, n) of the fused lm_head cross-entropy.  Default: two (chunk, ld) bf16 buffers (the logits and
    d(logits) of one chunk) of about 1 GB each, together what the single d(logits) buffer of the K6b backward holds;
    then equal chunks of whole 256-row tiles, as in _LinearLogProbK6Fn.backward."""
    ld = (V + 255) // 256 * 256
    if chunk_rows is None:
        chunk_rows = max(128, (1 << 30) // (ld * 2) // 128 * 128)
    chunk = int(chunk_rows)
    if chunk < 1:
        raise ValueError(f'chunk_rows must be positive, got {chunk_rows}')
    if N == 0:
        return []
    n_chunks = (N + chunk - 1) // chunk
    chunk = min(chunk, (-(-N // n_chunks) + 255) // 256 * 256)
    return [(r0, min(chunk, N - r0)) for r0 in range(0, N, chunk)]


def _ce_loss_launch(logp, labels, n, ignore_index, out, dev):
    partial = torch.empty(512, dtype=torch.float32, device=dev)
    L.check(L.lib().aa_nll_mean(logp.data_ptr(), L.AA_F32, labels.data_ptr(), n, int(ignore_index), out[0:1].data_ptr(),
                                out[1:2].data_ptr(), partial.data_ptr(), _device_scratch(dev)['counter'][4:5].data_ptr(),
                                L.stream_ptr(dev)))


class _LinearCrossEntropyFn(torch.autograd.Function):
    """Mean NLL of log_softmax(rows @ weight.T) at `lab` over the N valid rows, times `loss_scale`, where the gradient is
    formed in the FORWARD: every row's upstream gradient is the host constant -loss_scale / N, so per row chunk
      K6s   the GEMM once: the bf16 logits into `lbuf`, (max, logsum, fp32 log-prob) from the same rounded values;
      K1b   f32 mode, `lbuf` -> `dbuf`: ATen's fp32 softmax gradient of the upcast logits, cast to bf16 (ForCausalLMLoss);
      aa_linear_dhidden / aa_linear_dweight on `dbuf` (d(weight) accumulated in fp32 across chunks, rounded once)
    -- three GEMM passes over 2 * N * H * V instead of K6 + K6b + the two backward GEMMs.  K1b runs out of place: its
    kernels read `logits` and write `grad` through __restrict__ / non-coherent loads.  The backward only scales the two
    gradients by the incoming scalar (aa_scale_tile; nothing to do when it is 1) and hands them over, once.
    Without a gradient (neither input needs one; causal_lm_loss_from_hidden detaches both under torch.no_grad, since
    needs_input_grad follows requires_grad and not the grad mode): K6s and the loss only.  K6s still stores each logits
    chunk, into a `lbuf` that nothing reads then (about 1 GB at the default chunk): the price of statistics over the
    bf16-rounded logits, which K6 only offers with a bf16-rounded log-prob.  N == 0: the loss aa_nll_mean gives over all-ignored labels (what
    causal_lm_loss returns then), zero gradients.  -> (loss_scale * loss, loss)."""

    @staticmethod
    def forward(ctx, rows, weight, lab, shift_flat, ignore_index, loss_scale, chunk_rows):
        N, (V, H) = rows.size(0), weight.shape
        dev = rows.device
        need_h, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        out = torch.empty(2, dtype=torch.float32, device=dev)  # [loss, -1 / n_valid]
        d_rows = d_weight = None
        if N == 0:
            _ce_loss_launch(torch.zeros(shift_flat.numel(), dtype=torch.float32, device=dev), shift_flat,
                            shift_flat.numel(), ignore_index, out, dev)
            d_rows = torch.zeros_like(rows) if need_h else None
            d_weight = torch.zeros_like(weight) if need_w else None
        else:
            chunks = _ce_chunks(N, V, chunk_rows)
            ld, cmax = (V + 255) // 256 * 256, max(n for _, n in chunks)
            lib, st, sc = L.lib(), L.stream_ptr(dev), _device_scratch(dev)
            logp = torch.empty(N, dtype=torch.float32, device=dev)
            stats = torch.empty((2, N), dtype=torch.float32, device=dev)
            partial = torch.empty(3 * max(132 * 128, 16 * cmax), dtype=torch.float32, device=dev)  # split-vocabulary statistics
            lbuf = torch.empty((cmax, ld), dtype=torch.bfloat16, device=dev)
            if need_h or need_w:
                dbuf = torch.empty((cmax, ld), dtype=torch.bfloat16, device=dev)
                dbuf[:, V:].zero_()  # K1b writes columns [0, V); the GEMMs read all ld
                seed = torch.full((1,), -float(loss_scale) / N, dtype=torch.float32, device=dev)
                d_rows = torch.empty_like(rows) if need_h else None
                d_weight = torch.empty_like(weight) if need_w else None
                acc = torch.empty((V, H), dtype=torch.float32, device=dev) if (need_w and len(chunks) > 1) else None
            for i, (r0, n) in enumerate(chunks):
                h, y = rows[r0:r0 + n], lab[r0:r0 + n]
                L.check(lib.aa_linear_logits(
                    h.data_ptr(), n, H, h.stride(0), weight.data_ptr(), V, weight.stride(0), y.data_ptr(),
                    logp[r0:r0 + n].data_ptr(), L.AA_F32, stats[0, r0:r0 + n].data_ptr(), stats[1, r0:r0 + n].data_ptr(),
                    partial.data_ptr(), partial.numel(), L.MODE_F32, sc['status'].data_ptr(), lbuf.data_ptr(), ld, st))
                if not (need_h or need_w):
                    continue
                plan = _dense_plan(1, n, n * ld, ld, n, 0, n, 0, str(dev))
                _launch_bwd(lbuf[:n, :V], y, plan, stats[0, r0:r0 + n], stats[1, r0:r0 + n], None, None, seed,
                            dbuf[:n, :V], L.MODE_F32, grad_row_stride=ld)
                if need_h:
                    dh = d_rows[r0:r0 + n]
                    L.check(lib.aa_linear_dhidden(dbuf.data_ptr(), n, ld, weight.data_ptr(), V, H, weight.stride(0),
                                                  dh.data_ptr(), dh.stride(0), st))
                if need_w:
                    last = i == len(chunks) - 1
                    L.check(lib.aa_linear_dweight(dbuf.data_ptr(), n, ld, h.data_ptr(), H, h.stride(0), V, L.ptr(acc), H,
                                                  1 if i > 0 else 0, d_weight.data_ptr() if last else None,
                                                  d_weight.stride(0), st))
            _ce_loss_launch(logp, lab, N, ignore_index, out, dev)
        ctx.save_for_backward(d_rows, d_weight)
        loss = out[0]
        scaled = loss if loss_scale == 1.0 else loss * float(loss_scale)
        ctx.mark_non_differentiable(loss)
        return scaled.clone() if scaled is loss else scaled, loss

    @staticmethod
    def backward(ctx, g, _unused):
        d_rows, d_weight = _hand_over_once(ctx, g, *ctx.saved_tensors)
        return d_rows, d_weight, None, None, None, None, None


def causal_lm_loss_from_hidden(hidden: torch.Tensor, weight: torch.Tensor, labels: torch.Tensor, ignore_index: int = -100,
                               loss_scale: float = 1.0, chunk_rows: int | None = None, valid_rows=None):
    """causal_lm_loss_scaled(F.linear(hidden, weight), labels, loss_scale, ignore_index) from the last hidden states
    (B, L, H) bf16 and the lm_head weight (V, H) bf16, H % 64 == 0, without the (B, L, V) logits and gradient tiles:
    the valid rows (causal_lm_valid_rows; pass its result as `valid_rows` to take the host read earlier) are gathered
    into a compact (N, H) matrix and go through _LinearCrossEntropyFn in chunks of `chunk_rows`.  Differentiable in
    hidden and weight; the graph can be backpropagated ONCE.  -> (loss_scale * loss, loss)."""
    L.require_cuda(hidden, weight, labels)
    if hidden.dim() != 3 or weight.dim() != 2 or labels.shape != hidden.shape[:2] or weight.size(1) != hidden.size(2):
        raise ValueError('expected hidden (B, L, H), weight (V, H) and labels (B, L)')
    if hidden.dtype != torch.bfloat16 or weight.dtype != torch.bfloat16:
        raise ValueError(f'causal_lm_loss_from_hidden takes bf16 hidden states and head weight, got {hidden.dtype} and '
                         f'{weight.dtype}: use causal_lm_loss on the logits')
    B, seq, H = hidden.shape
    if H % 64:
        raise ValueError(f'causal_lm_loss_from_hidden needs a hidden size divisible by 64, got {H}: use causal_lm_loss '
                         'on the logits')
    if not torch.is_grad_enabled():  # eval under no_grad: a Parameter head would still report needs_input_grad
        hidden, weight = hidden.detach(), weight.detach()
    labels = labels.to(torch.int64)
    idx, _ = causal_lm_valid_rows(labels, ignore_index) if valid_rows is None else valid_rows
    shift = torch.full((B, seq), int(ignore_index), dtype=torch.int64, device=labels.device)
    shift[:, :-1] = labels[:, 1:]
    shift = shift.view(-1)
    rows = hidden.reshape(B * seq, H).index_select(0, idx)
    return _LinearCrossEntropyFn.apply(rows, _contiguous_last(weight), shift.index_select(0, idx), shift, int(ignore_index),
                                       float(loss_scale), chunk_rows)


# ---- masked mean ---------------------------------------------------------------------------------
class _MaskedMeanFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, m):
        B, W = x.shape
        dev = x.device
        out = torch.empty(1, dtype=torch.float32, device=dev)
        rows = torch.empty(B, dtype=torch.float32, device=dev)
        sc = _device_scratch(dev)
        L.check(L.lib().aa_masked_mean(x.data_ptr(), L.dtype_code(x.dtype), x.stride(0), L.ptr(m),
                                       m.stride(0) if m is not None else 0, B, W, out.data_ptr(), rows.data_ptr(),
                                       sc['counter'][1:2].data_ptr(), L.stream_ptr(dev)))
        ctx.save_for_backward(m)
        ctx.shape, ctx.dtype = x.shape, x.dtype
        return out[0]

    @staticmethod
    def backward(ctx, g):
        (m,) = ctx.saved_tensors
        B, W = ctx.shape
        if m is None:
            return (g / (B * W)).to(ctx.dtype).expand(B, W), None
        coef = g / (B * m.sum(dim=-1, keepdim=True).float())
        return (m * coef).to(ctx.dtype), None


def masked_mean(x: torch.Tensor, mask: torch.Tensor | None = None) -> torch.Tensor:
    """utils/tools.py:460-467: mean over rows of masked row means -> fp32 scalar (NaN when a row is
    fully masked, like the reference).  Differentiable in x."""
    L.require_cuda(x, mask)
    if x.dim() != 2:
        raise ValueError('masked_mean expects (B, L)')
    x = _contiguous_last(x)
    if x.dtype not in (torch.float32, torch.bfloat16, torch.float16):
        x = x.float()
    m = None
    if mask is not None:
        m = _contiguous_last(mask.to(torch.bool))
    return _MaskedMeanFn.apply(x, m)


# ---- K3 score head -------------------------------------------------------------------------------
class _ScoreHeadFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, hidden, weight, out_dtype, mode_code):
        Bsz, seq, H = hidden.shape
        dev = hidden.device
        scores = torch.empty((Bsz, seq), dtype=out_dtype, device=dev)
        L.check(L.lib().aa_score_head_fwd(hidden.data_ptr(), L.dtype_code(hidden.dtype), Bsz * seq, H,
                                          hidden.stride(1), weight.data_ptr(), scores.data_ptr(),
                                          L.dtype_code(out_dtype), mode_code, L.stream_ptr(dev)))
        ctx.save_for_backward(hidden, weight)
        ctx.mode_code = mode_code
        return scores

    @staticmethod
    def backward(ctx, g):
        hidden, weight = ctx.saved_tensors
        Bsz, seq, H = hidden.shape
        dev = hidden.device
        g = g.contiguous()
        if g.dtype not in (torch.float32, torch.bfloat16, torch.float16):
            g = g.float()
        if ctx.mode_code == L.MODE_FAITHFUL and g.dtype != hidden.dtype:
            # `.float()` after nn.Linear: autograd casts the incoming gradient back to the hidden dtype first
            g = g.to(hidden.dtype)
        need_h, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        grad_hidden = torch.empty_like(hidden, memory_format=torch.contiguous_format) if need_h else None
        grad_w32 = torch.empty(H, dtype=torch.float32, device=dev)
        import ctypes

        n_part = ctypes.c_int32(0)
        lib = L.lib()
        common = (hidden.data_ptr(), L.dtype_code(hidden.dtype), Bsz * seq, H, hidden.stride(1), weight.data_ptr(),
                  g.data_ptr(), L.dtype_code(g.dtype), L.ptr(grad_hidden), H, grad_w32.data_ptr())
        L.check(lib.aa_score_head_bwd(*common, None, ctypes.byref(n_part), ctx.mode_code, L.stream_ptr(dev)))
        partial = torch.empty((n_part.value, H), dtype=torch.float32, device=dev)
        L.check(lib.aa_score_head_bwd(*common, partial.data_ptr(), ctypes.byref(n_part), ctx.mode_code,
                                      L.stream_ptr(dev)))
        grad_w = grad_w32.to(weight.dtype).view_as(weight) if need_w else None
        return grad_hidden, grad_w, None, None


def score_head(last_hidden: torch.Tensor, weight: torch.Tensor, upcast: bool = True, mode: str | None = None):
    """scores = score_head(last_hidden_state)[.float()]  (models/llama.py:62-63; qwen2_vl.py:59-60 keeps
    the hidden dtype: upcast=False).  last_hidden (B, L, H), weight (1, H) or (H,) -> (B, L)."""
    L.require_cuda(last_hidden, weight)
    if last_hidden.dim() != 3:
        raise ValueError('last_hidden must be (B, L, H)')
    H = last_hidden.size(-1)
    if weight.numel() != H:
        raise ValueError('score_head weight must have H elements (nn.Linear(H, 1, bias=False))')
    hidden = last_hidden
    if hidden.stride(-1) != 1 or hidden.stride(0) != hidden.size(1) * hidden.stride(1) or \
            (hidden.stride(1) * hidden.element_size()) % 16 or hidden.data_ptr() % 16:
        hidden = hidden.contiguous()
    w = weight.to(hidden.dtype).contiguous()
    mode_code = _mode_code(mode, hidden.dtype)
    out_dtype = torch.float32 if (upcast or mode_code == L.MODE_F32) else hidden.dtype
    return _ScoreHeadFn.apply(hidden, w, out_dtype, mode_code)


def score_end(scores: torch.Tensor, attention_mask: torch.Tensor | None, last_hidden: torch.Tensor | None = None):
    """end_index / end_scores / end_last_hidden_state (models/llama.py:71-93): last attended position
    per row (attention_mask given) or position L-1 (attention_mask None: llava.py:64-66,
    qwen2_vl.py:62-64).  No host sync (the reference loops `m.nonzero()[-1]` per sample)."""
    L.require_cuda(scores, attention_mask, last_hidden)
    B, seq = scores.shape
    dev = scores.device
    scores = _contiguous_last(scores.detach())
    mask = None
    kind = L.MASK_U8
    if attention_mask is not None:
        mask = attention_mask
        if mask.dtype == torch.bool:
            mask = _contiguous_last(mask)
        elif mask.dtype == torch.int64:
            kind = L.MASK_I64
            mask = _contiguous_last(mask)
        else:
            mask = _contiguous_last(mask != 0)
    end_index = torch.empty(B, dtype=torch.int64, device=dev)
    end_scores = torch.empty(B, dtype=torch.float32, device=dev)
    end_hidden = None
    hid = None
    if last_hidden is not None:
        hid = _contiguous_last(last_hidden.detach())
        end_hidden = torch.empty((B, hid.size(-1)), dtype=hid.dtype, device=dev)
    sc = _device_scratch(dev)
    L.check(L.lib().aa_score_end(
        scores.data_ptr(), L.dtype_code(scores.dtype), scores.stride(0), L.ptr(mask), kind,
        mask.stride(0) if mask is not None else 0, B, seq, end_index.data_ptr(), end_scores.data_ptr(),
        L.ptr(hid), L.dtype_code(hid.dtype) if hid is not None else L.AA_F32,
        hid.stride(0) if hid is not None else 0, hid.stride(1) if hid is not None else 0,
        hid.size(-1) if hid is not None else 0, L.ptr(end_hidden), sc['status'].data_ptr(), L.stream_ptr(dev)))
    return end_index, end_scores, end_hidden


# ---- K4 / K5 PPO ---------------------------------------------------------------------------------
def _promote(a: torch.dtype, b: torch.dtype) -> torch.dtype:
    return a if a == b else torch.float32


# the per-token KL estimators of the PPO reward penalty and of GRPO's loss (include/aa_b200.h AA_KL_*), d = lp - ref:
#   k1  lp - ref ;  k2  0.5 * (lp - ref) ** 2 ;  k3  exp(ref - lp) - (ref - lp) - 1  (eager ops in this order)
KL_ESTIMATORS = {'k1': 0, 'k2': 1, 'k3': 2}


def kl_estimator_code(name: str) -> int:
    """The AA_KL_* code of an estimator name; anything else is refused here, before a launch."""
    if name not in KL_ESTIMATORS:
        raise ValueError(f'kl_estimator must be one of {sorted(KL_ESTIMATORS)}, got {name!r}')
    return KL_ESTIMATORS[name]


def kl_rewards_and_gae(reward, log_probs, ref_log_probs, values, sequence_mask, start: int, kl_coeff: float,
                       clip_range_score: float, gamma: float, gae_lambda: float, mode: str | None = None,
                       kl_estimator: str = 'k1'):
    """add_kl_divergence_regularization (trainers/text_to_text/ppo.py:528-547) +
    get_advantages_and_returns (:487-508) in ONE launch (K4).  Returns
    (old_rewards (B, W), advantages (B, W-start), returns (B, W-start), row_stats (B, 8) fp32).
    kl_estimator ('k1', the reference's, or 'k2' / 'k3', see KL_ESTIMATORS): the estimate the penalty
    -kl_coeff * KL is formed from (aa_ppo_prep_kl); row_stats[:, 0] stays the k1 row sum behind train/kl_divergence."""
    est = kl_estimator_code(kl_estimator)
    if est != KL_ESTIMATORS['k1'] and not math.isfinite(float(kl_coeff)):
        raise ValueError(f'kl_coeff must be finite, got {kl_coeff!r}')
    L.require_cuda(reward, log_probs, ref_log_probs, values, sequence_mask)
    if log_probs.dim() != 2:
        raise ValueError('log_probs must be (B, W)')
    B, W = log_probs.shape
    # the kernel indexes every (B, W) operand with W taken from log_probs: a narrower mask / values tensor would be
    # read past its end (the reference's elementwise ops raise a broadcast error instead)
    if not (tuple(ref_log_probs.shape) == tuple(values.shape) == tuple(sequence_mask.shape) == (B, W)):
        raise ValueError(f'ref_log_probs {tuple(ref_log_probs.shape)}, values {tuple(values.shape)} and sequence_mask '
                         f'{tuple(sequence_mask.shape)} must all match log_probs {(B, W)}')
    if reward.numel() != B:
        raise ValueError(f'reward must hold one value per sample ({B}); got {tuple(reward.shape)}')
    dev = log_probs.device
    lp = _contiguous_last(log_probs.detach())
    rlp = ref_log_probs.detach().to(lp.dtype)
    rlp = rlp if rlp.stride() == lp.stride() else rlp.contiguous()
    if rlp.stride() != lp.stride():
        lp = lp.contiguous()
    vals = _contiguous_last(values.detach())
    mask = _contiguous_last(sequence_mask.to(torch.bool))
    rew = reward.detach().to(torch.float32).contiguous()
    mode_code = _mode_code(mode, lp.dtype)
    faithful = mode_code == L.MODE_FAITHFUL
    rew_dtype = lp.dtype if faithful else torch.float32
    adv_dtype = _promote(vals.dtype, lp.dtype) if faithful else torch.float32
    old_rewards = torch.empty((B, W), dtype=rew_dtype, device=dev)
    adv = torch.empty((B, W - start), dtype=adv_dtype, device=dev)
    ret = torch.empty((B, W - start), dtype=adv_dtype, device=dev)
    row_stats = torch.empty((B, 8), dtype=torch.float32, device=dev)
    sc = _device_scratch(dev)
    head = (lp.data_ptr(), rlp.data_ptr(), L.dtype_code(lp.dtype), lp.stride(0), rew.data_ptr(), vals.data_ptr(),
            L.dtype_code(vals.dtype), vals.stride(0), mask.data_ptr(), mask.stride(0), B, W, int(start), float(kl_coeff))
    tail = (float(clip_range_score), float(gamma), float(gae_lambda), mode_code, old_rewards.data_ptr(),
            L.dtype_code(rew_dtype), adv.data_ptr(), ret.data_ptr(), L.dtype_code(adv_dtype), row_stats.data_ptr(),
            sc['status'].data_ptr(), L.stream_ptr(dev))
    if est == KL_ESTIMATORS['k1']:
        L.check(L.lib().aa_ppo_prep(*head, *tail))
    else:
        L.check(L.lib().aa_ppo_prep_kl(*head, est, *tail))
    return old_rewards, adv, ret, row_stats


def gae_from_rewards(values, rewards, sequence_mask, start: int, gamma: float, gae_lambda: float,
                     mode: str | None = None):
    """PPOTrainer.get_advantages_and_returns on its own (trainers/text_to_text/ppo.py:487-508): the
    GAE half of K4 on precomputed per-token rewards.  Returns (advantages, returns, row_stats)."""
    L.require_cuda(values, rewards, sequence_mask)
    if rewards.dim() != 2 or not (tuple(values.shape) == tuple(sequence_mask.shape) == tuple(rewards.shape)):
        raise ValueError(f'values {tuple(values.shape)}, rewards {tuple(rewards.shape)} and sequence_mask '
                         f'{tuple(sequence_mask.shape)} must share one (B, W) shape')
    B, W = rewards.shape
    dev = rewards.device
    rew = rewards.detach().contiguous()
    if rew.dtype not in (torch.float32, torch.bfloat16, torch.float16):
        rew = rew.float()
    vals = _contiguous_last(values.detach())
    mask = _contiguous_last(sequence_mask.to(torch.bool))
    mode_code = _mode_code(mode, rew.dtype)
    faithful = mode_code == L.MODE_FAITHFUL
    adv_dtype = _promote(vals.dtype, rew.dtype) if faithful else torch.float32
    adv = torch.empty((B, W - start), dtype=adv_dtype, device=dev)
    ret = torch.empty((B, W - start), dtype=adv_dtype, device=dev)
    row_stats = torch.empty((B, 8), dtype=torch.float32, device=dev)
    sc = _device_scratch(dev)
    L.check(L.lib().aa_ppo_prep(
        None, None, L.dtype_code(rew.dtype), 0, None, vals.data_ptr(), L.dtype_code(vals.dtype), vals.stride(0),
        mask.data_ptr(), mask.stride(0), B, W, int(start), 0.0, 0.0, float(gamma), float(gae_lambda), mode_code,
        rew.data_ptr(), L.dtype_code(rew.dtype), adv.data_ptr(), ret.data_ptr(), L.dtype_code(adv_dtype),
        row_stats.data_ptr(), sc['status'].data_ptr(), L.stream_ptr(dev)))
    return adv, ret, row_stats


ESTIMATORS = {'reinforce': 0, 'rloo': 1, 'reinforce_baseline': 2, 'group_norm': 3}  # include/aa_b200.h AA_EST_*


def estimator_returns(rewards, sequence_mask, start: int, estimator: str, n_samples_per_prompt: int, gamma: float,
                      mode: str | None = None, row_stats=None, mask_outputs: bool = True):
    """Multi-PPO's get_advantages_and_returns for the non-GAE estimators (trainers/text_to_text/multi_ppo.py:510-591:
    the group statistic, then cumulative_returns) in ONE launch (K4r).  `rewards` is the (B, W) output of
    add_kl_divergence_regularization.  Returns (advantages, returns), both (B, W - start) in the rewards dtype ('f32'
    mode: fp32).  With `row_stats` (K4's (B, 8) fp32 output) lanes 3 and 4 are overwritten with the masked row means
    of the new advantages and returns, so ppo_pack_metrics reports them.  mask_outputs=False with 'reinforce' is
    `cumulative_returns` on its own: the returns are not multiplied by the mask afterwards.

    The grouping is the reference's: `rewards.reshape(-1, n)` of the (B, W) token rewards, i.e. n consecutive flat
    elements (SURVEY.md H9).  Errors are raised here, before the launch, like the reference raises them."""
    if estimator == 'gae':
        raise ValueError("estimator_returns: 'gae' is K4's scan (kl_rewards_and_gae / gae_from_rewards)")
    if estimator not in ESTIMATORS:
        raise ValueError(f'Unknown estimator: {estimator}')
    n = int(n_samples_per_prompt)
    group = estimator != 'reinforce'
    if group and n < 2:
        raise ValueError(f'{estimator} requires n_samples_per_prompt > 1')
    if n < 1:
        raise ValueError(f'n_samples_per_prompt must be >= 1, got {n}')
    if rewards.dim() != 2 or tuple(sequence_mask.shape) != tuple(rewards.shape):
        raise ValueError(f'rewards {tuple(rewards.shape)} and sequence_mask {tuple(sequence_mask.shape)} must share one '
                         f'(B, W) shape')
    B, W = rewards.shape
    if group and (B * W) % n != 0:  # what `rewards.reshape(-1, n)` raises
        raise RuntimeError(f"shape '[-1, {n}]' is invalid for input of size {B * W}")
    if not 0 <= int(start) < W:
        raise ValueError(f'start={start} must lie in [0, {W})')
    L.require_cuda(rewards, sequence_mask, row_stats)
    dev = rewards.device
    rew = rewards.detach()
    if rew.dtype not in (torch.float32, torch.bfloat16, torch.float16):
        rew = rew.float()
    rew = rew.contiguous()
    mask = _contiguous_last(sequence_mask.to(torch.bool))
    mode_code = _mode_code(mode, rew.dtype)
    out_dtype = rew.dtype if mode_code == L.MODE_FAITHFUL else torch.float32
    adv = torch.empty((B, W - int(start)), dtype=out_dtype, device=dev)
    ret = torch.empty((B, W - int(start)), dtype=out_dtype, device=dev)
    if row_stats is not None and (row_stats.dtype != torch.float32 or tuple(row_stats.shape) != (B, 8)
                                  or not row_stats.is_contiguous()):
        raise ValueError(f'row_stats must be a contiguous fp32 (B, 8) tensor, got {row_stats.dtype} {tuple(row_stats.shape)}')
    L.check(L.lib().aa_ppo_returns(
        rew.data_ptr(), L.dtype_code(rew.dtype), rew.stride(0), mask.data_ptr(), mask.stride(0), B, W, int(start),
        ESTIMATORS[estimator], n, float(gamma), mode_code, int(bool(mask_outputs)), adv.data_ptr(), ret.data_ptr(), L.dtype_code(out_dtype),
        L.ptr(row_stats), L.stream_ptr(dev)))
    return adv, ret


def whiten_advantages(advantages: list[torch.Tensor], masks: list[torch.Tensor], group=None) -> list[torch.Tensor]:
    """TRL's / verl's masked_whiten(A, m, shift_mean=True) over ALL the micro-batches of one rollout, and over every rank
    of `group` (torch.distributed; None: the default group) when torch.distributed is initialised with more than one:
        n = sum m,  mean = sum m A / n,  var = sum m (A - mean) ** 2 / (n - 1),
        A' = (A - mean) * rsqrt(var + 1e-8) where m, 0 where not m.
    `advantages[k]` is micro-batch k's (B_k, W_k) advantages (bf16 / fp16 / fp32; the widths may differ) and `masks[k]`
    its mask of the same shape.  The statistics are fp64 and every sum has a fixed order, so the result is
    deterministic; mean and rstd are rounded once to fp32 and A' once to the advantages' dtype.  The tensors are
    rewritten in place (a copy first when the last dimension is strided) and returned.
    Launches: aa_whiten_moments per micro-batch, aa_whiten_reduce, all_reduce(SUM) of the (3,) fp64 triple across
    ranks, aa_whiten_apply per micro-batch; no host sync.  Fewer than 2 masked tokens in all sets a status bit, raised
    as ValueError at the next status read (check_status, or a PPO step's metrics), and leaves the advantages unchanged.
    Bad arguments raise ValueError here, before any launch."""
    advantages, masks = list(advantages), list(masks)
    if not advantages or len(advantages) != len(masks):
        raise ValueError(f'whiten_advantages needs one mask per advantages tensor and at least one of each, got '
                         f'{len(advantages)} and {len(masks)}')
    for a, m in zip(advantages, masks):
        if not (isinstance(a, torch.Tensor) and isinstance(m, torch.Tensor)) or a.dim() != 2 or \
                tuple(m.shape) != tuple(a.shape) or a.numel() == 0:
            raise ValueError(f'whiten_advantages: advantages and masks must be matching non-empty (B, W) tensors, got '
                             f'{tuple(getattr(a, "shape", ()))} and {tuple(getattr(m, "shape", ()))}')
        if a.dtype not in (torch.bfloat16, torch.float16, torch.float32):
            raise ValueError(f'whiten_advantages: advantages must be bf16 / fp16 / fp32, got {a.dtype}')
    try:
        L.require_cuda(*advantages, *masks)
    except RuntimeError as e:
        raise ValueError(f'whiten_advantages: {e}') from None
    dev = advantages[0].device
    outs = [a if a.stride(-1) == 1 else a.contiguous() for a in advantages]
    masks = [_contiguous_last(m.to(torch.bool)) for m in masks]
    K = len(outs)
    moments = torch.empty((K, 3), dtype=torch.float64, device=dev)
    total = torch.empty(3, dtype=torch.float64, device=dev)
    lib, stream = L.lib(), L.stream_ptr(dev)
    for k, (a, m) in enumerate(zip(outs, masks)):
        L.check(lib.aa_whiten_moments(a.data_ptr(), L.dtype_code(a.dtype), a.stride(0), m.data_ptr(), m.stride(0),
                                      a.size(0), a.size(1), moments.data_ptr(), k, K, stream))
    L.check(lib.aa_whiten_reduce(moments.data_ptr(), K, total.data_ptr(), stream))
    dist = torch.distributed
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(total, op=dist.ReduceOp.SUM, group=group)
    status = _device_scratch(dev)['status']
    for a, m in zip(outs, masks):
        L.check(lib.aa_whiten_apply(a.data_ptr(), L.dtype_code(a.dtype), a.stride(0), m.data_ptr(), m.stride(0),
                                    a.size(0), a.size(1), total.data_ptr(), status.data_ptr(), stream))
    return outs


LOSS_AGG_MODES = {'seq-mean-token-mean': 0, 'token-mean': 1}  # include/aa_b200.h AA_AGG_*
# include/aa_b200.h AA_COV_* (clip_cov, kl_cov) and AA_PM_* (cispo, sapo)
POLICY_LOSS_MODES = {'vanilla': 0, 'clip_cov': 1, 'kl_cov': 2, 'cispo': 3, 'sapo': 4}
COV_MODES = ('clip_cov', 'kl_cov')  # the modes that select tokens by covariance (_cov_term)
PM_MODES = ('cispo', 'sapo')  # the per-token policy losses of the AA_PM_* entry points (_pm_term)
# verl's defaults of the Clip-Cov / KL-Cov keys (ActorObjective: None takes these)
COV_DEFAULTS = {'clip_cov_ratio': 2e-4, 'clip_cov_lb': 1.0, 'clip_cov_ub': 5.0, 'kl_cov_ratio': 2e-4, 'ppo_kl_coef': 1.0}
# TRL's defaults of SAPO's temperatures (ActorObjective: None takes these)
SAPO_DEFAULTS = {'sapo_temperature_pos': 1.0, 'sapo_temperature_neg': 1.05}


@dataclasses.dataclass(frozen=True)
class ActorObjective:
    """The PPO actor's clipped-ratio objective (the reference's actor_loss_fn, trainers/text_to_text/ppo.py:291-307,
    when every field is at its default):

        ratio = exp(lp - old_lp) ;  s = min(A * ratio, A * clamp(ratio, 1 - clip_range_ratio_low, 1 + clip_range_ratio_high))
        dual-clip:  s = where(A < 0, max(s, dual_clip_ratio * A), s)
        loss = -masked_mean(s, mask)                (loss_agg_mode 'seq-mean-token-mean': mean of per-sample means)
             = -(s * mask).sum() / mask.sum()       ('token-mean': mean over the micro-batch's response tokens)

    clip_range_ratio_low / _high: None takes the trainer's clip_range_ratio (clip-higher: high > low); dual_clip_ratio:
    None = off, otherwise c > 1.
    policy_loss_mode (Cui et al. 2025; verl's policy_loss.loss_mode): 'vanilla' (the above), 'clip_cov' or 'kl_cov'.
    Over the counted tokens of one loss call, cov_t = (A_t - mean A) * (lp_t - mean lp) (fp64 means rounded to fp32,
    the product fp32; cov_token_selection).  'clip_cov': among the counted, unclipped tokens with
    clip_cov_lb < cov_t < clip_cov_ub, max(int(clip_cov_ratio * N), 1) (N = counted tokens) chosen by a hash of the
    flat index and the seed lose their objective term and its gradient.  'kl_cov': the objective is unclipped, s = A *
    ratio, and the max(1, int(kl_cov_ratio * N)) tokens with the largest cov_t take s - ppo_kl_coef * |lp - old|.  The
    five keys are None for their defaults (2e-4, 1.0, 5.0, 2e-4, 1.0) and refused under any other mode; neither mode
    takes dual_clip_ratio, and 'kl_cov' refuses an explicit clip range, which it would ignore.
    policy_loss_mode 'cispo' (MiniMax-M1, 2025) and 'sapo' (Qwen's Soft Adaptive Policy Optimization, 2025; TRL's
    GRPO loss_type 'cispo' / 'sapo') replace the clipped ratio per token, with s the negated loss term aggregated as
    above (tests/policy_loss_port.py is the specification):
        'cispo'  w = clamp(ratio, max = 1 + clip_range_ratio_high).detach() ;  s = w * A * lp     (every token keeps
                 the gradient w * A; train/actor_clip_fraction counts ratio > 1 + clip_range_ratio_high)
        'sapo'   tau = sapo_temperature_pos where A > 0, else sapo_temperature_neg ;
                 s = sigmoid(tau * (ratio - 1)) * 4 / tau * A                                     (fp32; nothing clipped)
    Neither takes dual_clip_ratio; 'cispo' refuses clip_range_ratio_low and 'sapo' any clip range, which they would
    ignore.  sapo_temperature_pos / _neg: None for 1.0 / 1.05, finite and > 0 as fp32 (the kernels' type), refused
    under any mode but 'sapo'.
    Both stay on K1f's single pass: each token's loss and gradient need that token alone.  The fields are checked
    here, on the host, before anything is launched."""

    clip_range_ratio_low: float | None = None
    clip_range_ratio_high: float | None = None
    dual_clip_ratio: float | None = None
    loss_agg_mode: str = 'seq-mean-token-mean'
    policy_loss_mode: str = 'vanilla'
    clip_cov_ratio: float | None = None
    clip_cov_lb: float | None = None
    clip_cov_ub: float | None = None
    kl_cov_ratio: float | None = None
    ppo_kl_coef: float | None = None
    sapo_temperature_pos: float | None = None
    sapo_temperature_neg: float | None = None
    _MODES = LOSS_AGG_MODES  # the aggregations this objective takes (a class attribute, not a field)

    def __post_init__(self):
        lo, hi, c = self.clip_range_ratio_low, self.clip_range_ratio_high, self.dual_clip_ratio
        if lo is not None and not (0.0 <= float(lo) < 1.0):
            raise ValueError(f'clip_range_ratio_low must be in [0, 1), got {lo!r}')
        if hi is not None and not (float(hi) >= 0.0):
            raise ValueError(f'clip_range_ratio_high must be >= 0, got {hi!r}')
        if c is not None and not (float(c) > 1.0 and math.isfinite(float(c))):
            raise ValueError(f'dual_clip_ratio must be None (off) or a finite value > 1, got {c!r}')
        if self.loss_agg_mode not in self._MODES:
            raise ValueError(f'loss_agg_mode must be one of {sorted(self._MODES)}, got {self.loss_agg_mode!r}')
        self._check_cov()

    def _check_cov(self):
        mode = self.policy_loss_mode
        if mode not in POLICY_LOSS_MODES:
            raise ValueError(f'policy_loss_mode must be one of {tuple(POLICY_LOSS_MODES)}, got {mode!r}')
        temps = {k: getattr(self, k) for k in SAPO_DEFAULTS}
        given = [k for k, v in temps.items() if v is not None]
        if given and mode != 'sapo':
            raise ValueError(f'{", ".join(given)} need policy_loss_mode sapo (it is {mode})')
        for k, v in temps.items():
            # the kernels take the temperature as an fp32: it must stay finite and > 0 there too (1e39 is inf and
            # 1e-50 is 0 in fp32, which the C argument checks refuse)
            if v is not None and (isinstance(v, bool) or not isinstance(v, (int, float)) or
                                  not (math.isfinite(ctypes.c_float(float(v)).value) and
                                       ctypes.c_float(float(v)).value > 0.0)):
                raise ValueError(f'{k} must be a finite number > 0 in fp32, got {v!r}')
        keys = {k: getattr(self, k) for k in COV_DEFAULTS}
        if mode not in COV_MODES:
            given = [k for k, v in keys.items() if v is not None]
            if given:
                raise ValueError(f'{", ".join(given)} need policy_loss_mode clip_cov or kl_cov (it is {mode})')
        if mode == 'vanilla':
            return
        if self.dual_clip_ratio is not None:
            raise ValueError(f'policy_loss_mode {mode!r} has no dual-clip: dual_clip_ratio must be unset')
        if mode in ('kl_cov', 'sapo') and (self.clip_range_ratio_low is not None or
                                           self.clip_range_ratio_high is not None):
            raise ValueError(f'policy_loss_mode {mode} is unclipped: clip_range_ratio_low / _high would be ignored')
        if mode == 'cispo' and self.clip_range_ratio_low is not None:
            raise ValueError('policy_loss_mode cispo truncates the ratio from above only: clip_range_ratio_low would be '
                             'ignored')
        if mode in PM_MODES:
            return
        for k, v in keys.items():
            if v is not None and (isinstance(v, bool) or not isinstance(v, (int, float))):
                raise ValueError(f'{k} must be a number, got {v!r}')
        for k in ('clip_cov_ratio', 'kl_cov_ratio'):
            if not 0.0 < self.cov_value(k) <= 1.0:
                raise ValueError(f'{k} must lie in (0, 1], got {keys[k]!r}')
        lb, ub = self.cov_value('clip_cov_lb'), self.cov_value('clip_cov_ub')
        if not (math.isfinite(lb) and math.isfinite(ub) and lb < ub):
            raise ValueError(f'clip_cov_lb < clip_cov_ub must be finite, got {lb!r}, {ub!r}')
        c = self.cov_value('ppo_kl_coef')
        if not (math.isfinite(c) and c >= 0.0):
            raise ValueError(f'ppo_kl_coef must be finite and >= 0, got {c!r}')

    def sapo_value(self, key: str) -> float:
        """One of SAPO's temperatures in effect: the field, or its default (SAPO_DEFAULTS) when None."""
        v = getattr(self, key)
        return float(SAPO_DEFAULTS[key] if v is None else v)

    def cov_value(self, key: str) -> float:
        """One of the Clip-Cov / KL-Cov keys in effect: the field, or its default (COV_DEFAULTS) when None."""
        v = getattr(self, key)
        return float(COV_DEFAULTS[key] if v is None else v)

    @property
    def is_default(self) -> bool:
        """The reference's objective: the kernels run today's launches."""
        return (self.clip_range_ratio_low is None and self.clip_range_ratio_high is None and self.dual_clip_ratio is None
                and self.loss_agg_mode == 'seq-mean-token-mean' and self.policy_loss_mode == 'vanilla')

    @property
    def token_mean(self) -> bool:
        return self.loss_agg_mode == 'token-mean'

    def args(self, clip_range_ratio: float) -> tuple[float, float, float, int]:
        """-> (clip_low, clip_high, dual_clip (0 = off), loss_agg code) of the C entry points."""
        lo = float(clip_range_ratio if self.clip_range_ratio_low is None else self.clip_range_ratio_low)
        hi = float(clip_range_ratio if self.clip_range_ratio_high is None else self.clip_range_ratio_high)
        if not (0.0 <= lo < 1.0 and hi >= 0.0):
            raise ValueError(f'clip range [1 - {lo}, 1 + {hi}]: need 0 <= low < 1 and high >= 0')
        return lo, hi, float(self.dual_clip_ratio or 0.0), self._MODES[self.loss_agg_mode]


# include/aa_b200.h AA_AGG_*: GRPO also takes Dr. GRPO's constant normaliser
GRPO_LOSS_AGG_MODES = {**LOSS_AGG_MODES, 'seq-mean-token-sum-norm': 2}
# GRPO's importance ratio: per token (aa_grpo_loss_obj / _kl) or per sequence (GSPO, aa_grpo_loss_seq)
IMPORTANCE_SAMPLING_LEVELS = ('token', 'sequence')


@dataclasses.dataclass(frozen=True)
class GrpoObjective(ActorObjective):
    """GRPO's clipped objective (DeepSeekMath's GRPO over several updates per rollout, with DAPO's clip-higher and
    Dr. GRPO's aggregation), the fields and checks of ActorObjective with GRPO's defaults:

        ratio = exp(lp - old_lp) ;  s = min(A * ratio, A * clamp(ratio, 1 - low, 1 + high))
        dual-clip:  s = where(A < 0, max(s, dual_clip_ratio * A), s) ;  per-token loss = -(s - beta * KL)
        loss = (ptl * mask).sum() / mask.sum()                      ('token-mean', the default: the reference's loss)
             = ((ptl * mask).sum(-1) / mask.sum(-1)).mean()         ('seq-mean-token-mean')
             = (ptl * mask).sum() / (B * K)                         ('seq-mean-token-sum-norm', K = logits_to_keep)

    clip_range_ratio: the ε of both bounds when clip_range_ratio_low / _high are None.  With old_lp = lp (the first
    update of a rollout) the ratio is 1 and nothing is clipped.  kl_estimator: the per-token KL ('k3', the reference's,
    or 'k1' / 'k2': KL_ESTIMATORS).  importance_sampling_level: 'token' (the ratio above) or 'sequence' (GSPO, Zheng et
    al. 2025; TRL's importance_sampling_level): one fp32 ratio per sequence, w = exp(sum((lp - old) * mask) / n) with
    n = the sequence's counted tokens, clipped in place of each token's ratio (aa_grpo_loss_seq).  Without old
    log-probs w is 1 and the token-level launches run.  top_entropy_quantile rho in [0, 1] (Wang et al. 2025; TRL's
    top_entropy_quantile): only the counted tokens whose policy entropy H is >= torch.quantile(H[counted], 1 - rho)
    over every rank keep s, per-token loss = -(s * keep - beta * KL); the denominators, the KL term, the entropy bonus,
    GSPO's ratio and the clip fractions stay over the whole completion mask.  1 (the default) masks nothing.
    policy_loss_mode 'clip_cov' / 'kl_cov' (ActorObjective) over the completion mask with the row's advantage, per-token
    loss -(s - beta * KL); token level only.  On the first update (ratio 1) KL-Cov selects tokens but changes nothing:
    |lp - old| = 0 and its gradient sign(0) = 0.  Checked on the host when constructed."""

    loss_agg_mode: str = 'token-mean'
    clip_range_ratio: float = 0.2
    kl_estimator: str = 'k3'
    importance_sampling_level: str = 'token'
    top_entropy_quantile: float = 1.0
    _MODES = GRPO_LOSS_AGG_MODES

    def __post_init__(self):
        super().__post_init__()
        self.args()  # the clip range with clip_range_ratio filled in
        kl_estimator_code(self.kl_estimator)
        if self.importance_sampling_level not in IMPORTANCE_SAMPLING_LEVELS:
            raise ValueError(f'importance_sampling_level must be one of {IMPORTANCE_SAMPLING_LEVELS}, got '
                             f'{self.importance_sampling_level!r}')
        rho = self.top_entropy_quantile
        if isinstance(rho, bool) or not isinstance(rho, (int, float)) or not 0.0 <= float(rho) <= 1.0:
            raise ValueError(f'top_entropy_quantile must be a number in [0, 1], got {rho!r}')
        if self.policy_loss_mode != 'vanilla' and (self.sequence_level or rho < 1.0):
            raise ValueError(f'policy_loss_mode {self.policy_loss_mode!r} is token-level and takes every token: it '
                             f'refuses importance_sampling_level="sequence" and top_entropy_quantile < 1')

    @property
    def is_default(self) -> bool:
        """The reference's loss when the ratio is 1: the kernels run today's launches."""
        return (self.clip_range_ratio_low is None and self.clip_range_ratio_high is None and self.dual_clip_ratio is None
                and self.loss_agg_mode == 'token-mean' and self.kl_estimator == 'k3'
                and self.importance_sampling_level == 'token' and self.top_entropy_quantile == 1.0
                and self.policy_loss_mode == 'vanilla')

    @property
    def sequence_level(self) -> bool:
        return self.importance_sampling_level == 'sequence'

    def args(self, clip_range_ratio: float | None = None) -> tuple[float, float, float, int]:
        return super().args(self.clip_range_ratio if clip_range_ratio is None else clip_range_ratio)


def _objective(objective: ActorObjective | None, cls: type = ActorObjective) -> ActorObjective | None:
    """None for the reference's objective (None, or every field at its default: today's launches), else the objective,
    which must be a `cls`."""
    if objective is None:
        return None
    if not isinstance(objective, cls):
        raise TypeError(f'objective must be an ops.{cls.__name__}, got {type(objective).__name__}')
    return None if objective.is_default else objective


_U32 = 0xffffffff


def _fmix32(h: int) -> int:
    """MurmurHash3's 32-bit finaliser (the device's fmix32)."""
    h &= _U32
    h ^= h >> 16
    h = (h * 0x85ebca6b) & _U32
    h ^= h >> 13
    h = (h * 0xc2b2ae35) & _U32
    return h ^ (h >> 16)


def cov_hash_seed(seed: int, rank: int, call: int) -> int:
    """Clip-Cov's 32-bit hash seed s = fmix32(fmix32(fmix32(seed) ^ rank) ^ call): `seed` the run's seed, `rank` the
    data-parallel rank, `call` the count of the trainer's earlier Clip-Cov loss calls.  Token t of the call is chosen
    by its key fmix32(t ^ s), so the choice is reproducible without RNG state (and differs from verl's
    torch.randperm stream)."""
    return _fmix32(_fmix32(_fmix32(int(seed)) ^ (int(rank) & _U32)) ^ (int(call) & _U32))


class _CovTerm:
    """Clip-Cov / KL-Cov of one loss call: the mode's AA_COV_* code, the selection ratio, Clip-Cov's bounds and
    KL-Cov's coefficient (an ActorObjective's values in effect), the hash seed, and `share`, the fp32[1] the selection
    writes the selected share of the counted tokens into."""

    def __init__(self, objective: ActorObjective, seed: int, device):
        self.code = POLICY_LOSS_MODES[objective.policy_loss_mode]
        clip = self.code == POLICY_LOSS_MODES['clip_cov']
        self.ratio = objective.cov_value('clip_cov_ratio' if clip else 'kl_cov_ratio')
        self.lb, self.ub = objective.cov_value('clip_cov_lb'), objective.cov_value('clip_cov_ub')
        self.coef = 0.0 if clip else objective.cov_value('ppo_kl_coef')
        self.seed = int(seed) & _U32
        self.share = torch.empty(1, dtype=torch.float32, device=device)


def _cov_term(objective, seed: int, device) -> _CovTerm | None:
    """None unless the objective's policy_loss_mode is clip_cov or kl_cov."""
    if objective is None or objective.policy_loss_mode not in COV_MODES:
        return None
    return _CovTerm(objective, seed, device)


class _PmTerm:
    """CISPO / SAPO of one loss call: the mode's AA_PM_* code and SAPO's temperatures in effect (CISPO ignores them).
    `sapo`: s, and so the loss, is fp32 whatever the dtypes (the temperature tensor is fp32)."""

    def __init__(self, objective: ActorObjective):
        self.code = POLICY_LOSS_MODES[objective.policy_loss_mode]
        self.sapo = objective.policy_loss_mode == 'sapo'
        self.tau_pos = objective.sapo_value('sapo_temperature_pos')
        self.tau_neg = objective.sapo_value('sapo_temperature_neg')


def _pm_term(objective) -> _PmTerm | None:
    """None unless the objective's policy_loss_mode is cispo or sapo."""
    if objective is None or objective.policy_loss_mode not in PM_MODES:
        return None
    return _PmTerm(objective)


def _cov_select(x, aux, old, mask, row_end, cov: _CovTerm, clip_lo: float, clip_hi: float, mode_code: int):
    """The selection of one loss call -> uint8 (B, W), and cov.share: aa_cov_moments -> aa_cov_keys ->
    aa_cov_select_hi -> aa_cov_hist_lo -> aa_cov_select_lo -> aa_cov_mark, no host sync.  x: the log-probs the loss
    kernel reads; with `mask` (PPO) aux holds (B, W) advantages, with `row_end` (GRPO) fp32 (B,) ones."""
    B, W = x.shape
    dev = x.device
    state = torch.empty(16, dtype=torch.int32, device=dev)  # uint32 words
    keys = torch.empty(B * W, dtype=torch.int32, device=dev)
    elig = torch.empty(B * W, dtype=torch.uint8, device=dev)
    hist = torch.empty(_ENT_BINS, dtype=torch.int32, device=dev)
    ties = torch.empty(B, dtype=torch.int32, device=dev)
    sel = torch.empty((B, W), dtype=torch.uint8, device=dev)
    lib, stream = L.lib(), L.stream_ptr(dev)
    rows = (x.data_ptr(), x.stride(0), L.dtype_code(x.dtype), aux.data_ptr(), aux.stride(0) if mask is not None else 0,
            L.dtype_code(aux.dtype), L.ptr(mask), mask.stride(0) if mask is not None else 0, L.ptr(row_end), B, W)
    L.check(lib.aa_cov_moments(*rows, state.data_ptr(), stream))
    L.check(lib.aa_cov_keys(cov.code, *rows[:2], L.ptr(old), old.stride(0) if old is not None else 0, *rows[2:],
                            float(clip_lo), float(clip_hi), cov.lb, cov.ub, cov.seed, mode_code, state.data_ptr(),
                            keys.data_ptr(), elig.data_ptr(), hist.data_ptr(), stream))
    L.check(lib.aa_cov_select_hi(hist.data_ptr(), ctypes.byref(ctypes.c_double(cov.ratio)), state.data_ptr(), stream))
    L.check(lib.aa_cov_hist_lo(keys.data_ptr(), elig.data_ptr(), B * W, state.data_ptr(), hist.data_ptr(), stream))
    L.check(lib.aa_cov_select_lo(hist.data_ptr(), state.data_ptr(), cov.share.data_ptr(), stream))
    L.check(lib.aa_cov_mark(keys.data_ptr(), elig.data_ptr(), B, W, state.data_ptr(), ties.data_ptr(), sel.data_ptr(),
                            sel.stride(0), stream))
    return sel


def cov_token_selection(log_probs: torch.Tensor, advantages: torch.Tensor, mask_or_row_end: torch.Tensor,
                        policy_loss_mode: str, *, old_log_probs: torch.Tensor | None = None,
                        clip_range_ratio_low: float = 0.2, clip_range_ratio_high: float = 0.2,
                        clip_cov_ratio: float | None = None, clip_cov_lb: float | None = None,
                        clip_cov_ub: float | None = None, kl_cov_ratio: float | None = None, seed: int = 0,
                        mode: str | None = None, return_share: bool = False):
    """The tokens Clip-Cov or KL-Cov selects in one loss call (see ActorObjective) -> uint8 (B, W), 1 = selected;
    return_share: and the fp32 (1,) selected share of the counted tokens (0 when none is counted).
    log_probs (B, W) fp32 / bf16 / fp16, the current log-probs as the loss kernel reads them; mask_or_row_end: a
    (B, W) mask with (B, W) advantages (PPO), or int (B,) counted tokens per row (t < row_end[b], GRPO's completion
    mask: grpo_row_end) with one advantage per row.  Clip-Cov: old_log_probs (None: ratio 1) and the clip range give
    the clipped tokens, `seed` the 32-bit hash seed (cov_hash_seed), `mode` the ratio's rounding.  The selection is
    local to this call (no collective) and exact: a radix select on 32-bit keys with ties to the smaller flat index.
    Bad arguments raise ValueError here, before any launch."""
    keys = {'clip_cov_ratio': clip_cov_ratio, 'clip_cov_lb': clip_cov_lb, 'clip_cov_ub': clip_cov_ub,
            'kl_cov_ratio': kl_cov_ratio}
    if policy_loss_mode not in ('clip_cov', 'kl_cov'):
        raise ValueError(f'cov_token_selection: policy_loss_mode must be clip_cov or kl_cov, got {policy_loss_mode!r}')
    objective = ActorObjective(policy_loss_mode=policy_loss_mode, **keys)
    for name, t in (('log_probs', log_probs), ('advantages', advantages), ('mask_or_row_end', mask_or_row_end)):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f'cov_token_selection: {name} must be a tensor')
    if log_probs.dim() != 2 or log_probs.numel() == 0 or log_probs.dtype not in (torch.float32, torch.bfloat16,
                                                                                 torch.float16):
        raise ValueError(f'cov_token_selection: log_probs must be a non-empty fp32 / bf16 / fp16 (B, W) tensor, got '
                         f'{log_probs.dtype} {tuple(log_probs.shape)}')
    B, W = log_probs.shape
    if B * W > 2 ** 31 - 1:
        raise ValueError(f'cov_token_selection: B * W = {B * W} exceeds 2^31 - 1')
    m = mask_or_row_end
    if tuple(m.shape) == (B, W):
        if tuple(advantages.shape) != (B, W):
            raise ValueError(f'cov_token_selection: with a mask the advantages must be (B, W) = ({B}, {W})')
        mask, row_end = _contiguous_last((m != 0).to(torch.uint8)), None
        aux = _contiguous_last(advantages.detach())
        if aux.dtype not in (torch.float32, torch.bfloat16, torch.float16):
            aux = aux.float()
    elif tuple(m.shape) == (B,) and not m.dtype.is_floating_point and m.dtype != torch.bool:
        if advantages.numel() != B:
            raise ValueError(f'cov_token_selection: with row ends one advantage per row ({B}) is expected')
        mask, row_end = None, m.to(torch.int32).contiguous()
        aux = advantages.detach().float().contiguous().view(-1)
    else:
        raise ValueError(f'cov_token_selection: mask_or_row_end must be a (B, W) = ({B}, {W}) mask or integer (B,) row '
                         f'ends, got {m.dtype} {tuple(m.shape)}')
    if old_log_probs is not None and tuple(old_log_probs.shape) != (B, W):
        raise ValueError(f'cov_token_selection: old_log_probs must be (B, W) = ({B}, {W})')
    lo, hi = float(clip_range_ratio_low), float(clip_range_ratio_high)
    if not (0.0 <= lo < 1.0 and hi >= 0.0):
        raise ValueError(f'cov_token_selection: clip range [1 - {lo}, 1 + {hi}]: need 0 <= low < 1 and high >= 0')
    try:
        L.require_cuda(log_probs, advantages, m, *((old_log_probs,) if old_log_probs is not None else ()))
    except RuntimeError as e:
        raise ValueError(f'cov_token_selection: {e}') from None
    x = _contiguous_last(log_probs.detach())
    old = _contiguous_last(old_log_probs.detach().to(x.dtype)) if old_log_probs is not None else None
    cov = _CovTerm(objective, seed, x.device)
    sel = _cov_select(x, aux, old, mask, row_end, cov, lo, hi, _mode_code(mode, x.dtype))
    return (sel, cov.share) if return_share else sel


def token_mean(x: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """(x * mask).sum() / mask.sum() over the whole (B, W) tensor -> fp32 scalar (NaN without a masked-in token): the
    masked_mean kernel on the tensor as one row, differentiable in x."""
    return masked_mean(x.reshape(1, -1), mask.reshape(1, -1))


def _ppo_loss_launch(x, old, aux, mask, clip, mode_code, actor: bool, x_tail=None, obj=None, clip_frac=None, kl=None,
                     cov=None, pm=None):
    """K5: -> (loss fp32[2], loss as a 0-dim tensor of the promoted dtype (a view, no launch), grad (B, Wm), row_mean).
    x_tail = (DeviceLens, src_width): `x` is the raw (B, src_width) tensor and the kernel reads the per-sample tails.
    Actor only: obj = ActorObjective.args(...) (None: the reference's objective), clip_frac = an fp32[2] tensor the
    kernel fills with the clip fractions (aa_ppo_actor_loss_obj); kl = _KlLossTerm: the KL loss term
    (aa_ppo_actor_loss_kl: grad is d (loss + coeff * agg(KL)) / d x, kl.out receives agg(KL), `loss` stays the
    clipped objective).  cov = _CovTerm (obj given): Clip-Cov / KL-Cov, the selection (_cov_select) then
    aa_ppo_actor_loss_cov, with the KL loss term when kl is given.  pm = _PmTerm (obj given): CISPO / SAPO,
    aa_ppo_actor_loss_pm, with the KL loss term when kl is given (SAPO's loss is fp32)."""
    B, Wm = old.shape
    dev = x.device
    loss = torch.empty(2, dtype=torch.float32, device=dev)
    grad = torch.empty((B, Wm), dtype=x.dtype, device=dev)
    rows = torch.empty(B, dtype=torch.float32, device=dev)
    row_mean = torch.empty(B, dtype=torch.float32, device=dev)
    sc = _device_scratch(dev)
    lib = L.lib()
    if actor and pm is not None:
        _, hi, _, agg = obj
        rows = torch.empty(5 * B, dtype=torch.float32, device=dev)
        L.check(lib.aa_ppo_actor_loss_pm(
            x.data_ptr(), x.stride(0), old.data_ptr(), old.stride(0), L.dtype_code(x.dtype), aux.data_ptr(),
            aux.stride(0), L.dtype_code(aux.dtype), mask.data_ptr(), mask.stride(0), B, Wm, float(hi), int(agg),
            pm.code, pm.tau_pos, pm.tau_neg, mode_code, kl.ref.data_ptr() if kl is not None else None,
            kl.ref.stride(0) if kl is not None else 0, kl.coeff if kl is not None else 0.0,
            kl.estimator if kl is not None else 0, loss.data_ptr(), kl.out.data_ptr() if kl is not None else None,
            grad.data_ptr(), grad.stride(0), L.ptr(clip_frac), rows.data_ptr(), sc['counter'][2:3].data_ptr(),
            L.stream_ptr(dev)))
    elif actor and cov is not None:
        lo, hi, _, agg = obj
        sel = _cov_select(x, aux, old, mask, None, cov, lo, hi, mode_code)
        rows = torch.empty(5 * B, dtype=torch.float32, device=dev)
        L.check(lib.aa_ppo_actor_loss_cov(
            x.data_ptr(), x.stride(0), old.data_ptr(), old.stride(0), L.dtype_code(x.dtype), aux.data_ptr(),
            aux.stride(0), L.dtype_code(aux.dtype), mask.data_ptr(), mask.stride(0), B, Wm, float(lo), float(hi),
            int(agg), cov.code, cov.coef, sel.data_ptr(), sel.stride(0), mode_code,
            kl.ref.data_ptr() if kl is not None else None, kl.ref.stride(0) if kl is not None else 0,
            kl.coeff if kl is not None else 0.0, kl.estimator if kl is not None else 0, loss.data_ptr(),
            kl.out.data_ptr() if kl is not None else None, grad.data_ptr(), grad.stride(0), L.ptr(clip_frac),
            rows.data_ptr(), sc['counter'][2:3].data_ptr(), L.stream_ptr(dev)))
    elif actor and kl is not None:
        lo, hi, dual, agg = obj if obj is not None else (clip, clip, 0.0, 0)
        rows = torch.empty(5 * B, dtype=torch.float32, device=dev)
        L.check(lib.aa_ppo_actor_loss_kl(
            x.data_ptr(), x.stride(0), old.data_ptr(), old.stride(0), L.dtype_code(x.dtype), aux.data_ptr(),
            aux.stride(0), L.dtype_code(aux.dtype), mask.data_ptr(), mask.stride(0), B, Wm, float(lo), float(hi),
            float(dual), int(agg), mode_code, kl.ref.data_ptr(), kl.ref.stride(0), kl.coeff, kl.estimator,
            loss.data_ptr(), kl.out.data_ptr(), grad.data_ptr(), grad.stride(0), L.ptr(clip_frac), rows.data_ptr(),
            sc['counter'][2:3].data_ptr(), L.stream_ptr(dev)))
    elif actor and (obj is not None or clip_frac is not None):
        lo, hi, dual, agg = obj if obj is not None else (clip, clip, 0.0, 0)
        rows = torch.empty(4 * B, dtype=torch.float32, device=dev)
        L.check(lib.aa_ppo_actor_loss_obj(
            x.data_ptr(), x.stride(0), old.data_ptr(), old.stride(0), L.dtype_code(x.dtype), aux.data_ptr(),
            aux.stride(0), L.dtype_code(aux.dtype), mask.data_ptr(), mask.stride(0), B, Wm, float(lo), float(hi),
            float(dual), int(agg), mode_code, loss.data_ptr(), grad.data_ptr(), grad.stride(0), L.ptr(clip_frac),
            rows.data_ptr(), sc['counter'][2:3].data_ptr(), L.stream_ptr(dev)))
    elif actor:
        L.check(lib.aa_ppo_actor_loss(
            x.data_ptr(), x.stride(0), old.data_ptr(), old.stride(0), L.dtype_code(x.dtype), aux.data_ptr(),
            aux.stride(0), L.dtype_code(aux.dtype), mask.data_ptr(), mask.stride(0), B, Wm, float(clip),
            mode_code, loss.data_ptr(), grad.data_ptr(), grad.stride(0), rows.data_ptr(),
            sc['counter'][2:3].data_ptr(), L.stream_ptr(dev)))
    else:
        L.check(lib.aa_ppo_critic_loss(
            x.data_ptr(), x.stride(0), old.data_ptr(), old.stride(0), L.dtype_code(x.dtype), aux.data_ptr(),
            aux.stride(0), L.dtype_code(aux.dtype), mask.data_ptr(), mask.stride(0), B, Wm, float(clip),
            mode_code, loss.data_ptr(), grad.data_ptr(), grad.stride(0), row_mean.data_ptr(), rows.data_ptr(),
            sc['counter'][3:4].data_ptr(), x_tail[0].dev.data_ptr() if x_tail else None, int(x_tail[1]) if x_tail else 0,
            L.stream_ptr(dev)))
    faithful = mode_code == L.MODE_FAITHFUL and not (pm is not None and pm.sapo)
    out_dtype = _promote(x.dtype, aux.dtype) if faithful else torch.float32
    cast = loss[0] if out_dtype == torch.float32 else loss[1:2].view(out_dtype)[0]
    return loss, cast, grad, row_mean


class _PpoLossFn(torch.autograd.Function):
    """K5: forward computes the loss AND d loss / d x in the same launch; backward scales it.  With the KL loss term
    (kl, actor only) the first output is  loss + kl.coeff * agg(KL)  (fp32) and its gradient is K5's."""

    @staticmethod
    def forward(ctx, x, old, aux, mask, clip, mode_code, actor: bool, obj=None, clip_frac=None, kl=None, cov=None,
                pm=None):
        loss, cast, grad, row_mean = _ppo_loss_launch(x, old, aux, mask, clip, mode_code, actor, obj=obj,
                                                      clip_frac=clip_frac, kl=kl, cov=cov, pm=pm)
        ctx.save_for_backward(grad)
        ctx.mark_non_differentiable(row_mean, loss)
        return (cast if kl is None else kl.regularised(loss[0])), row_mean, loss

    @staticmethod
    def backward(ctx, g_loss, _g, _l):
        (grad,) = ctx.saved_tensors
        return (grad.float() * g_loss.float()).to(grad.dtype), None, None, None, None, None, None, None, None, None, \
            None, None


def _k1f_actor_launch(logits, ids, plan, lp, old, aux, mask, clip, mode_code, grad, obj, coeff, ent, kl=None, pm=None):
    """K1f over the actor's scored rows, writing lp and the gradient tile `grad`.  obj: ActorObjective.args(...) for
    the objective entry point (aa_logprob_actor_fused_obj), None for the reference's objective -- with an entropy
    bonus (`ent`, the fp32 entropy out) the entropy-gradient entry point, otherwise the plain one.  kl (_KlLossTerm):
    the KL loss term's entry point (aa_logprob_actor_fused_kl), whatever the objective.  pm (_PmTerm, obj given):
    CISPO / SAPO's entry point (aa_logprob_actor_fused_pm), with the KL loss term and the entropy as given."""
    dev = logits.device
    # 48 bytes per tile row (the row records); the entropy-gradient and objective forms add 4 per segment (the rows'
    # g_H coefficients), the KL form 8 (and the rows' KL coefficients)
    extra = plan.n_seg if kl is not None or pm is not None else \
        (plan.n_seg + 1) // 2 if obj is not None or ent is not None else 0
    scratch = torch.empty(plan.n_tile_rows * 6 + extra, dtype=torch.int64, device=dev)
    p = plan.ptrs()
    lib = L.lib()
    head = (logits.data_ptr(), L.dtype_code(logits.dtype), logits.stride(-2), logits.size(-1), ids.data_ptr(),
            plan.n_seg, p[0], p[1], p[2], p[3], p[4], plan.n_tile_rows, lp.data_ptr(), L.dtype_code(lp.dtype), None,
            None, old.data_ptr(), old.stride(0), aux.data_ptr(), aux.stride(0), L.dtype_code(aux.dtype),
            mask.data_ptr(), mask.stride(0), lp.size(1))
    tail = (mode_code, grad.data_ptr(), logits.size(-1), scratch.data_ptr(), _device_scratch(dev)['status'].data_ptr())
    if pm is not None:
        L.check(lib.aa_logprob_actor_fused_pm(*head, float(obj[1]), int(obj[3]), pm.code, pm.tau_pos, pm.tau_neg,
                                              *tail, coeff, L.ptr(ent), L.ptr(kl.ref if kl is not None else None),
                                              kl.coeff if kl is not None else 0.0, kl.estimator if kl is not None else 0,
                                              L.stream_ptr(dev)))
    elif kl is not None:
        L.check(lib.aa_logprob_actor_fused_kl(*head, *(obj if obj is not None else (clip, clip, 0.0, 0)), *tail, coeff,
                                              L.ptr(ent), kl.ref.data_ptr(), kl.coeff, kl.estimator, L.stream_ptr(dev)))
    elif obj is not None:
        L.check(lib.aa_logprob_actor_fused_obj(*head, *obj, *tail, coeff, L.ptr(ent), L.stream_ptr(dev)))
    elif ent is not None:
        L.check(lib.aa_logprob_actor_fused_entropy(*head, float(clip), *tail, coeff, ent.data_ptr(), L.stream_ptr(dev)))
    else:
        L.check(lib.aa_logprob_actor_fused(*head, float(clip), *tail, L.stream_ptr(dev)))


class _TailActorLossFn(torch.autograd.Function):
    """The actor half of the multimodal rl_step as ONE autograd node (trainers/text_image_to_text/ppo.py:298-316).

    Default (K1f, aa_logprob_actor_fused): the forward makes ONE pass over the scored rows and already writes the
    gradient tile -- the objective is a masked mean of per-token terms, so d loss / d log-prob needs nothing but the
    token's own log-prob; each row is streamed twice by the same CTA and the second pass comes out of L2.  K5 then reduces
    the loss value from the log-probs; backward hands the tile over (aa_scale_tile multiplies it by the incoming scalar
    on the device iff that is not 1).
    `single_pass` False (see _single_pass_ok), or a plan K1f does not take: forward = K1 over the response tails + K5;
    backward = K1b taking K5's d loss / d log-probs as its per-row upstream gradient and the incoming scalar as a device
    scale.
    entropy_coeff != 0 (entropy bonus): the node's loss is  actor_loss - entropy_coeff * masked_mean(H, mask)  and a
    fourth output, the detached masked-mean entropy, follows; the third stays the actor loss without the bonus.  K1f's
    entropy-gradient variant (aa_logprob_actor_fused_entropy), or K1's entropy variant + K5 + masked_mean and, in the
    backward, K1b's entropy variant with g_H = -entropy_coeff * mask / (B * mask count of the row).
    objective (a non-default ActorObjective): K1f's objective entry point (aa_logprob_actor_fused_obj) and K5's
    (aa_ppo_actor_loss_obj); under token-mean the entropy term is a token mean too.  clip_frac: an fp32[2] tensor K5
    fills with the clip fractions.  kl (_KlLossTerm): the node's loss gains  + kl.coeff * agg(KL)  (fp32; the third
    output stays the actor loss without it), K1f's KL entry point (aa_logprob_actor_fused_kl) writes its gradient into
    the tile, K5's (aa_ppo_actor_loss_kl) the loss value, agg(KL) into kl.out and, for K1b, d total / d log-probs.
    cov (_CovTerm, with single_pass False): Clip-Cov / KL-Cov -- the selection needs every log-prob of the call first,
    so K1 -> selection -> aa_ppo_actor_loss_cov -> K1b.  pm (_PmTerm): CISPO / SAPO, K1f's and K5's PM entry points
    (aa_logprob_actor_fused_pm, aa_ppo_actor_loss_pm), or K1 -> aa_ppo_actor_loss_pm -> K1b."""

    @staticmethod
    def forward(ctx, logits, ids, plan, old, aux, mask, clip, mode_code, single_pass, entropy_coeff=0.0, objective=None,
                clip_frac=None, kl=None, cov=None, pm=None):
        out_dtype = logits.dtype if mode_code == L.MODE_FAITHFUL else torch.float32
        dev = logits.device
        coeff = float(entropy_coeff)
        obj = objective.args(clip) if objective is not None else None
        lp = torch.zeros(plan.out_shape, dtype=out_dtype, device=dev)
        ctx.fused = bool(single_pass and plan.n_tile_rows > 0 and plan.n_seg > 0 and plan.n_tile_rows % plan.n_seg == 0
                         and len(plan.out_shape) == 2)
        ctx.bonus = coeff != 0.0
        ent = torch.zeros(plan.out_shape, dtype=torch.float32, device=dev) if ctx.bonus else None
        if ctx.fused:
            grad = torch.empty(logits.shape, dtype=logits.dtype, device=dev)
            _k1f_actor_launch(logits, ids, plan, lp, old, aux, mask, clip, mode_code, grad, obj, coeff, ent, kl, pm)
            ctx.save_for_backward(grad)
        else:
            stats = torch.empty((2, max(plan.n_rows, 1)), dtype=torch.float32, device=dev)
            _launch_fwd(logits, ids, plan, lp, stats[0], stats[1], entropy=ent)
        loss, cast, grad_lp, _ = _ppo_loss_launch(lp, old, aux, mask, clip, mode_code, True, obj=obj, clip_frac=clip_frac,
                                                  kl=kl, cov=cov, pm=pm)
        tm = objective is not None and objective.token_mean
        if not ctx.fused:
            if ctx.bonus:
                # d (-coeff * mean(H)) / d H on masked-in tokens (0, not 0 * -inf, elsewhere: K1f forms g_H for
                # masked-in tokens only): the masked mean's coefficient as _MaskedMeanFn's backward forms it, or
                # -coeff / (masked-in tokens of the micro-batch) under token-mean
                den = mask.sum().float() if tm else mask.size(0) * mask.sum(dim=-1, keepdim=True).float()
                g_h = torch.where(mask, -coeff / den, 0.0)
                ctx.save_for_backward(logits, ids, stats, grad_lp, ent, g_h)
            else:
                ctx.save_for_backward(logits, ids, stats, grad_lp)
            ctx.plan, ctx.mode_code = plan, mode_code
        if not ctx.bonus:
            ctx.mark_non_differentiable(lp, loss)
            return (cast if kl is None else kl.regularised(loss[0])), lp, loss
        h_mean = token_mean(ent, mask) if tm else masked_mean(ent, mask)
        reg = (loss[0] if kl is None else kl.regularised(loss[0])) - coeff * h_mean
        ctx.mark_non_differentiable(lp, loss, h_mean)
        return reg, lp, loss, h_mean

    @staticmethod
    def backward(ctx, g_loss, *_unused):
        if ctx.fused:
            (grad,) = _hand_over_once(ctx, g_loss, *ctx.saved_tensors)
            return grad, None, None, None, None, None, None, None, None, None, None, None, None, None, None
        scale = g_loss.detach().reshape(1)
        if scale.dtype not in (torch.float32, torch.bfloat16, torch.float16):
            scale = scale.float()
        scale = scale.contiguous()
        if ctx.bonus:
            logits, ids, stats, grad_lp, ent, g_h = ctx.saved_tensors
        else:
            (logits, ids, stats, grad_lp), ent, g_h = ctx.saved_tensors, None, None
        grad = torch.empty(logits.shape, dtype=logits.dtype, device=logits.device)
        _launch_bwd(logits, ids, ctx.plan, stats[0], stats[1], grad_lp, None, scale, grad, ctx.mode_code, entropy=ent,
                    grad_entropy=g_h)
        return grad, None, None, None, None, None, None, None, None, None, None, None, None, None, None


class _TailCriticLossFn(torch.autograd.Function):
    """The critic half (text_image_to_text/ppo.py:318-337): forward = K5 reading `scores.squeeze(-1)[:, :-1]` through
    the per-sample tail indexing; backward = ONE launch that scatters K5's gradient back into the raw (B, L[, 1]) scores
    layout, zeros and the upstream scalar included."""

    @staticmethod
    def forward(ctx, scores, lens_dev, bound, old, aux, mask, clip, mode_code):
        raw = scores.squeeze(-1) if scores.dim() == 3 else scores  # (B, L)
        raw = _contiguous_last(raw)
        src_width = raw.size(1) - 1  # `[:, :-1]`
        lens = DeviceLens(lens_dev, bound)
        loss, cast, grad, row_mean = _ppo_loss_launch(raw, old, aux, mask, clip, mode_code, False, x_tail=(lens, src_width))
        ctx.save_for_backward(grad, lens_dev)
        ctx.shape, ctx.src_width = scores.shape, src_width
        ctx.mark_non_differentiable(row_mean, loss)
        return cast, row_mean, loss

    @staticmethod
    def backward(ctx, g_loss, _r, _l):
        grad, lens_dev = ctx.saved_tensors
        B, W = grad.shape
        Lq = ctx.src_width + 1
        out = torch.empty((B, Lq), dtype=grad.dtype, device=grad.device)
        scale = g_loss.detach().reshape(1)
        if scale.dtype not in (torch.float32, torch.bfloat16, torch.float16):
            scale = scale.float()
        L.check(L.lib().aa_tail_scatter_scaled(grad.data_ptr(), L.dtype_code(grad.dtype), grad.stride(0), lens_dev.data_ptr(), B, W,
                                               ctx.src_width, scale.data_ptr(), L.dtype_code(scale.dtype), out.data_ptr(),
                                               out.stride(0), Lq, L.stream_ptr(grad.device)))
        return out.view(ctx.shape), None, None, None, None, None, None, None


def _k5_operands(old, aux, mask, dtype):
    """K5's detached operands beside the differentiated input: old in that input's dtype `dtype`, aux (advantages or
    returns) in a dtype the kernel reads, mask as bool; each contiguous along the last dimension."""
    old = _contiguous_last(old.detach().to(dtype))
    aux = _contiguous_last(aux.detach())
    if aux.dtype not in (torch.float32, torch.bfloat16, torch.float16):
        aux = aux.float()
    return old, aux, _contiguous_last(mask.to(torch.bool))


class _KlLossTerm:
    """The KL loss term  coeff * agg(KL(lp, ref), mask)  of an actor node: `ref` the reference log-probs, detached, in
    the dtype the kernels read the log-probs in and contiguous (K1f reads it at each log-prob's own index), `estimator`
    its AA_KL_* code, `out` the fp32[1] K5 writes agg(KL) into."""

    def __init__(self, ref, coeff: float, estimator: int, out):
        self.ref, self.coeff, self.estimator, self.out = ref, coeff, estimator, out

    def regularised(self, loss):
        """loss + coeff * agg(KL), fp32 (one launch)."""
        return torch.add(loss, self.out[0], alpha=self.coeff)


def _kl_loss_args(ref_log_probs, old_log_probs, kl_loss_coeff, kl_loss_estimator) -> tuple[float, int] | None:
    """None when kl_loss_coeff is 0 (no term: today's calls), otherwise (coefficient, estimator code).  The
    coefficient must be finite and > 0, the estimator one of KL_ESTIMATORS and ref_log_probs shaped like
    old_log_probs; anything else raises ValueError."""
    coeff = float(kl_loss_coeff)
    if coeff == 0.0:
        return None
    if not (math.isfinite(coeff) and coeff > 0.0):
        raise ValueError(f'kl_loss_coeff must be finite and > 0, got {kl_loss_coeff!r}')
    est = kl_estimator_code(kl_loss_estimator)
    if ref_log_probs is None or tuple(ref_log_probs.shape) != tuple(old_log_probs.shape):
        raise ValueError('a KL loss term (kl_loss_coeff != 0) needs ref_log_probs with the shape of old_log_probs')
    return coeff, est


def _kl_loss_term(ref_log_probs, old_log_probs, kl_loss_coeff, kl_loss_estimator, dtype) -> _KlLossTerm | None:
    """_kl_loss_args as the term the kernels take: ref_log_probs detached, cast to `dtype` (as _k5_operands casts
    old_log_probs) and contiguous."""
    args = _kl_loss_args(ref_log_probs, old_log_probs, kl_loss_coeff, kl_loss_estimator)
    if args is None:
        return None
    coeff, est = args
    L.require_cuda(ref_log_probs)
    ref = ref_log_probs.detach().to(dtype).contiguous()
    return _KlLossTerm(ref, coeff, est, torch.empty(1, dtype=torch.float32, device=ref.device))


def _loss_inputs(x, old, aux, mask):
    L.require_cuda(x, old, aux, mask)
    if not (x.shape == old.shape == aux.shape == mask.shape) or x.dim() != 2:
        raise ValueError('loss inputs must all be (B, W)')
    x = _contiguous_last(x)
    return (x, *_k5_operands(old, aux, mask, x.dtype))


def actor_loss(log_probs, old_log_probs, advantages, mask, clip_range_ratio: float, mode: str | None = None,
               objective: ActorObjective | None = None, return_clip_fraction: bool = False, ref_log_probs=None,
               kl_loss_coeff: float = 0.0, kl_loss_estimator: str = 'k3', cov_seed: int = 0):
    """PPOTrainer.actor_loss_fn (trainers/text_to_text/ppo.py:291-307), differentiable in log_probs.
    objective: an ActorObjective (None: the reference's).  return_clip_fraction: -> (loss, fp32[2] device tensor: the
    clipped fraction and the dual-clip fraction, aggregated like the loss; see aa_ppo_actor_loss_obj).
    kl_loss_coeff != 0 (a KL loss term, see _actor_loss): the loss is  actor_loss + kl_loss_coeff * agg(KL)  (fp32)
    and the detached agg(KL) follows it, before the clip fractions.  An objective with policy_loss_mode clip_cov /
    kl_cov: the selection of cov_token_selection (Clip-Cov hashes with cov_seed, see cov_hash_seed) and K5's Cov entry
    point; its fp32 (1,) selected share follows agg(KL), before the clip fractions."""
    loss, _, kl, cf, share = _actor_loss(log_probs, old_log_probs, advantages, mask, clip_range_ratio, mode, objective,
                                         return_clip_fraction, ref_log_probs, kl_loss_coeff, kl_loss_estimator, cov_seed)
    out = (loss,) + ((kl,) if kl is not None else ()) + ((share,) if share is not None else ()) + \
        ((cf,) if return_clip_fraction else ())
    return out if len(out) > 1 else loss


def _actor_loss(log_probs, old_log_probs, advantages, mask, clip_range_ratio, mode, objective, return_clip_fraction,
                ref_log_probs, kl_loss_coeff, kl_loss_estimator, cov_seed: int = 0):
    """actor_loss -> (loss, the actor loss without the KL term for ppo_pack_metrics (the loss itself without the term,
    K5's fp32[2] with it), the detached agg(KL) or None, clip fractions or None, the Clip-Cov / KL-Cov selected share
    or None).  The KL loss term: KL(lp, ref) by `kl_loss_estimator` (KL_ESTIMATORS), aggregated over the same mask as
    the objective (its loss_agg_mode), its gradient added to K5's (aa_ppo_actor_loss_kl, or aa_ppo_actor_loss_cov
    under Clip-Cov / KL-Cov)."""
    objective = _objective(objective)
    x, old, aux, m = _loss_inputs(log_probs, old_log_probs, advantages, mask)
    kl = _kl_loss_term(ref_log_probs, old_log_probs, kl_loss_coeff, kl_loss_estimator, x.dtype)
    obj = objective.args(clip_range_ratio) if objective is not None else None
    cov = _cov_term(objective, cov_seed, x.device)
    cf = torch.zeros(2, dtype=torch.float32, device=x.device) if return_clip_fraction else None
    loss, _, loss32 = _PpoLossFn.apply(x, old, aux, m, clip_range_ratio, _mode_code(mode, x.dtype), True, obj, cf, kl,
                                       cov, _pm_term(objective))
    share = cov.share if cov is not None else None
    if kl is None:
        return loss, loss, None, cf, share
    return loss, loss32, kl.out[0], cf, share


def critic_loss(values, old_values, returns, mask, clip_range_value: float, mode: str | None = None,
                return_row_mean: bool = False):
    """PPOTrainer.critic_loss_fn (trainers/text_to_text/ppo.py:510-526), differentiable in values."""
    x, old, aux, m = _loss_inputs(values, old_values, returns, mask)
    loss, row_mean, _ = _PpoLossFn.apply(x, old, aux, m, clip_range_value, _mode_code(mode, x.dtype), False)
    return (loss, row_mean) if return_row_mean else loss


def tail_actor_loss(logits: torch.Tensor, input_ids: torch.Tensor, lens, old_log_probs, advantages, mask,
                    clip_range_ratio: float, mode: str | None = None, entropy_coeff: float = 0.0,
                    objective: ActorObjective | None = None, return_clip_fraction: bool = False, ref_log_probs=None,
                    kl_loss_coeff: float = 0.0, kl_loss_estimator: str = 'k3', cov_seed: int = 0):
    """response_tail_log_probs + actor_loss as one autograd node (see _TailActorLossFn).
    -> (actor loss, new log-probs (B, W), the loss as fp32[2] for ppo_pack_metrics).  entropy_coeff != 0: the first
    output is  actor_loss - entropy_coeff * masked_mean(H, mask)  (fp32), the third stays the actor loss without the
    bonus, and the detached masked-mean entropy follows as a fourth.  objective: an ActorObjective (None: the
    reference's; under token-mean the entropy term is a token mean too).  kl_loss_coeff != 0 (a KL loss term, as
    actor_loss; ref_log_probs (B, W) aligned with old_log_probs): the first output gains  + kl_loss_coeff * agg(KL),
    the third stays without it and the detached agg(KL) follows the entropy mean (if any).  An objective with
    policy_loss_mode clip_cov / kl_cov (seeded by cov_seed, as actor_loss) runs the composed path, K1 -> selection ->
    aa_ppo_actor_loss_cov -> K1b, and its fp32 (1,) selected share follows agg(KL).  return_clip_fraction: the fp32[2]
    clip fractions (see actor_loss) follow as the last output."""
    objective = _objective(objective)
    L.require_cuda(logits, input_ids, old_log_probs, advantages, mask)
    lens = as_device_lens(lens, logits.device)
    B, K, _ = logits.shape
    if lens.bound > K - 1:
        raise ValueError(f'the logits tile holds {K} positions: too few for responses of up to {lens.bound} tokens')
    if not (tuple(old_log_probs.shape) == tuple(advantages.shape) == tuple(mask.shape) == (B, lens.bound)):
        raise ValueError('old_log_probs, advantages and mask must all be (B, W), W = the bound of the response lengths')
    logits, ids = _contiguous_last(logits), input_ids.contiguous()
    mode_code = _mode_code(mode, logits.dtype)
    lp_dtype = logits.dtype if mode_code == L.MODE_FAITHFUL else torch.float32
    old, aux, m = _k5_operands(old_log_probs, advantages, mask, lp_dtype)
    kl = _kl_loss_term(ref_log_probs, old_log_probs, kl_loss_coeff, kl_loss_estimator, lp_dtype)
    plan = device_tail_plan(lens, K, logits.stride(0), logits.stride(1), ids.stride(0), ids.size(1), 0, -1, lens.bound)
    cov = _cov_term(objective, cov_seed, logits.device)
    single_pass = cov is None and _single_pass_ok(logits, _FUSED_ACTOR, torch.is_grad_enabled() and logits.requires_grad)
    if objective is not None:
        objective.args(clip_range_ratio)  # a bad clip range fails here, before the node launches anything
    cf = torch.zeros(2, dtype=torch.float32, device=logits.device) if return_clip_fraction else None
    out = _TailActorLossFn.apply(logits, ids, plan, old, aux, m, clip_range_ratio, mode_code, single_pass,
                                 float(entropy_coeff), objective, cf, kl, cov, _pm_term(objective))
    return (*out, *((kl.out[0],) if kl is not None else ()), *((cov.share,) if cov is not None else ()),
            *((cf,) if return_clip_fraction else ()))


@functools.lru_cache(maxsize=64)
def _dense_actor_plan(B: int, L: int, start: int, sb: int, sl: int, lab_sb: int, device_str: str) -> RowPlan:
    """One segment per sample: rows [start, L - 1) of the (B, L, V) tile against labels ids[b, start + 1 :]."""
    W = L - 1 - start
    return RowPlan([b * sb + start * sl for b in range(B)], [b * lab_sb + start + 1 for b in range(B)],
                   [b * W for b in range(B)], [W] * B, [b * L + start for b in range(B)], (B, W), B * L,
                   torch.device(device_str))


def dense_actor_loss(logits: torch.Tensor, input_ids: torch.Tensor, start: int, old_log_probs, advantages, mask,
                     clip_range_ratio: float, mode: str | None = None, entropy_coeff: float = 0.0,
                     objective: ActorObjective | None = None, return_clip_fraction: bool = False, ref_log_probs=None,
                     kl_loss_coeff: float = 0.0, kl_loss_estimator: str = 'k3', cov_seed: int = 0):
    """The actor half of the text rl_step (trainers/text_to_text/ppo.py:336-349) as one autograd node:
    `gather_log_probabilities(logits[:, :-1], ids[:, 1:])[:, start:]` -> `actor_loss_fn` -> backward up to d logits.
    Only the rows `[start, L - 1)` are read (the reference scores every position and slices afterwards); with a
    gradient and rows long enough (see _single_pass_ok) the node is the single-pass K1f (see _TailActorLossFn), otherwise the
    composed ops gather_log_probabilities -> actor_loss.  old_log_probs / advantages / mask: (B, L - 1 - start).
    -> (actor loss, new log-probs (B, L - 1 - start), the loss for ppo_pack_metrics: fp32[2] buffer or the 0-dim loss).
    entropy_coeff != 0 (entropy bonus): the first output is  actor_loss - entropy_coeff * masked_mean(H, mask)  (fp32),
    the third stays the actor loss without the bonus and the detached masked-mean entropy follows as a fourth; the
    single pass is K1f's entropy-gradient variant, the composed path K1's entropy variant -> K5 + masked_mean -> K1b's
    entropy variant.  objective / return_clip_fraction / the KL loss term (ref_log_probs (B, L - 1 - start),
    kl_loss_coeff, kl_loss_estimator): as tail_actor_loss (agg(KL) after the entropy mean, the clip fractions last);
    the composed path runs K5's KL entry point, whose gradient K1b carries to the tile.  An objective with
    policy_loss_mode clip_cov / kl_cov always takes the composed path (K1 -> selection -> aa_ppo_actor_loss_cov ->
    K1b; the selection needs every log-prob of the call first) and its selected share follows agg(KL), as
    tail_actor_loss."""
    objective = _objective(objective)
    L.require_cuda(logits, input_ids, old_log_probs, advantages, mask)
    if logits.dim() != 3 or input_ids.shape != logits.shape[:2]:
        raise ValueError('expected logits (B, L, V) and input_ids (B, L)')
    B, Lq, _ = logits.shape
    start = int(start)
    W = Lq - 1 - start
    if start < 0 or W <= 0:
        raise ValueError(f'start = {start} leaves no scored position in a sequence of {Lq}')
    if not (tuple(old_log_probs.shape) == tuple(advantages.shape) == tuple(mask.shape) == (B, W)):
        raise ValueError('old_log_probs, advantages and mask must all be (B, L - 1 - start)')
    if objective is not None:
        objective.args(clip_range_ratio)  # a bad clip range fails here, before any launch
    cov_mode = objective is not None and objective.policy_loss_mode in COV_MODES
    if cov_mode or not _single_pass_ok(logits, _FUSED_ACTOR, torch.is_grad_enabled() and logits.requires_grad):
        # short rows, fp16, no gradient: the composed ops (K1 over the response rows -> K5, which takes the objective;
        # backward K1b)
        rows, labels = logits[:, start:-1], input_ids[:, start + 1:]
        _kl_loss_args(ref_log_probs, old_log_probs, kl_loss_coeff, kl_loss_estimator)  # a bad term fails before K1
        if entropy_coeff != 0.0:
            lp, ent = gather_log_probabilities_with_entropy(rows, labels, mode=mode, entropy_grad=True)
        else:
            lp = gather_log_probabilities(rows, labels, mode=mode)
        loss, loss32, kl, cf, share = _actor_loss(lp, old_log_probs, advantages, mask, clip_range_ratio, mode, objective,
                                                  return_clip_fraction, ref_log_probs, kl_loss_coeff, kl_loss_estimator,
                                                  cov_seed)
        tail = ((kl,) if kl is not None else ()) + ((share,) if share is not None else ()) + \
            ((cf,) if return_clip_fraction else ())
        if entropy_coeff == 0.0:
            return (loss, lp.detach(), loss32, *tail)
        m = mask.to(torch.bool)
        h_mean = token_mean(ent, m) if objective is not None and objective.token_mean else masked_mean(ent, m)
        return (loss - float(entropy_coeff) * h_mean, lp.detach(), loss32, h_mean.detach(), *tail)
    logits, ids = _contiguous_last(logits), input_ids.contiguous()
    if B > 1 and (logits.stride(0) != Lq * logits.stride(1)):
        logits = logits.contiguous()  # the gradient tile is shaped after the logits: rows must be uniformly strided
    mode_code = _mode_code(mode, logits.dtype)
    lp_dtype = logits.dtype if mode_code == L.MODE_FAITHFUL else torch.float32
    old, aux, m = _k5_operands(old_log_probs, advantages, mask, lp_dtype)
    kl = _kl_loss_term(ref_log_probs, old_log_probs, kl_loss_coeff, kl_loss_estimator, lp_dtype)
    plan = _dense_actor_plan(B, Lq, start, logits.stride(0), logits.stride(1), ids.stride(0), str(logits.device))
    cf = torch.zeros(2, dtype=torch.float32, device=logits.device) if return_clip_fraction else None
    out = _TailActorLossFn.apply(logits, ids, plan, old, aux, m, clip_range_ratio, mode_code, True,
                                 float(entropy_coeff), objective, cf, kl, None, _pm_term(objective))
    return (*out, *((kl.out[0],) if kl is not None else ()), *((cf,) if return_clip_fraction else ()))


def tail_critic_loss(scores: torch.Tensor, lens, old_values, returns, mask, clip_range_value: float,
                     mode: str | None = None):
    """critic_loss on `pad_sequence([scores.squeeze(-1)[b, :-1][-R_b:]])` without materialising that tensor (see
    _TailCriticLossFn).  scores (B, L, 1) or (B, L).  -> (critic loss, masked row means of the new values, loss fp32[2])."""
    L.require_cuda(scores, old_values, returns, mask)
    lens = as_device_lens(lens, scores.device)
    B = scores.size(0)
    if not (tuple(old_values.shape) == tuple(returns.shape) == tuple(mask.shape) == (B, lens.bound)):
        raise ValueError('old_values, returns and mask must all be (B, W), W = the bound of the response lengths')
    if lens.bound > scores.size(1) - 1:
        raise ValueError('the scores tensor is too short for the response lengths')
    x = scores if scores.dtype in (torch.float32, torch.bfloat16, torch.float16) else scores.float()
    old, aux, m = _k5_operands(old_values, returns, mask, x.dtype)
    return _TailCriticLossFn.apply(x, lens.dev, lens.bound, old, aux, m, clip_range_value, _mode_code(mode, x.dtype))


def ppo_pack_metrics(row_stats, reward, value_row_mean, actor_loss_t, critic_loss_t, coll=None) -> torch.Tensor:
    """The ten local metric scalars of trainers/text_to_text/ppo.py:360-381 as ONE fp32[12] vector
    (entries 0..8 AVG-reduced, entry 9 MAX-reduced).  With `coll` (FusedPackedAllReduce.next((9,))) the same
    kernel also performs that reduction over NVLink peer memory."""
    import ctypes

    dev = row_stats.device
    B = row_stats.size(0)
    stats = torch.empty(12, dtype=torch.float32, device=dev)
    a, c = actor_loss_t.detach(), critic_loss_t.detach()  # 0-dim losses or the fp32[2] buffers of the fused loss nodes
    a = a if (a.dtype == torch.float32 and a.dim() == 1) else a.float().reshape(1).contiguous()
    c = c if (c.dtype == torch.float32 and c.dim() == 1) else c.float().reshape(1).contiguous()
    L.check(L.lib().aa_ppo_pack_metrics(row_stats.data_ptr(), reward.detach().float().contiguous().data_ptr(),
                                        L.ptr(value_row_mean), a.data_ptr(), c.data_ptr(), B, stats.data_ptr(),
                                        ctypes.byref(coll) if coll is not None else None,
                                        _device_scratch(dev)['status'].data_ptr(), L.stream_ptr(dev)))
    return stats


# ---- integer layout ------------------------------------------------------------------------------
def move_padding_left(input_tensor: torch.Tensor, padding_value: int = 0) -> torch.Tensor:
    """trainers/text_image_to_text/ppo.py:56-87 / utils/tools.py:615-639, bit-exact, one launch."""
    L.require_cuda(input_tensor)
    if input_tensor.dim() != 2 or input_tensor.dtype != torch.int64:
        raise ValueError('move_padding_left expects an int64 (B, L) tensor')
    x = _contiguous_last(input_tensor)
    out = torch.empty(x.shape, dtype=torch.int64, device=x.device)
    L.check(L.lib().aa_move_padding_left(x.data_ptr(), x.size(0), x.size(1), x.stride(0), int(padding_value),
                                         out.data_ptr(), L.stream_ptr(x.device)))
    return out


class _TailRowsFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, lens_dev, rmax):
        B, W = x.shape
        out = torch.empty((B, rmax), dtype=x.dtype, device=x.device)
        L.check(L.lib().aa_tail_rows(x.data_ptr(), L.dtype_code(x.dtype), x.stride(0), lens_dev.data_ptr(), B, W, rmax,
                                     out.data_ptr(), out.stride(0), 0, L.stream_ptr(x.device)))
        ctx.save_for_backward(lens_dev)
        ctx.W = W
        return out

    @staticmethod
    def backward(ctx, g):
        (lens_dev,) = ctx.saved_tensors
        g = _contiguous_last(g)
        B, rmax = g.shape
        out = torch.empty((B, ctx.W), dtype=g.dtype, device=g.device)
        L.check(L.lib().aa_tail_rows(g.data_ptr(), L.dtype_code(g.dtype), g.stride(0), lens_dev.data_ptr(), B, ctx.W, rmax,
                                     out.data_ptr(), out.stride(0), 1, L.stream_ptr(g.device)))
        return out, None, None


def tail_rows(x: torch.Tensor, lens: Sequence[int]) -> torch.Tensor:
    """pad_sequence([x[b][-R_b:] for b], batch_first=True) for a (B, W) tensor
    (trainers/text_image_to_text/ppo.py:233-249, 318-330) in one launch, differentiable in x."""
    L.require_cuda(x)
    if isinstance(lens, DeviceLens):  # lengths on the device: the width is the host-known bound
        if x.dim() != 2 or len(lens) != x.size(0) or not 0 < lens.bound <= x.size(1):
            raise ValueError('tail_rows: x must be (B, W) with 0 <= R_b <= bound <= W')
        return _TailRowsFn.apply(_contiguous_last(x), lens.dev, lens.bound)
    lens = tuple(int(r) for r in lens)
    if x.dim() != 2 or len(lens) != x.size(0) or not 0 < max(lens) <= x.size(1) or min(lens) < 0:
        raise ValueError('tail_rows: x must be (B, W) with 0 <= R_b <= W')
    return _TailRowsFn.apply(_contiguous_last(x), _lens_tensor(lens, str(x.device)), max(lens))


def rollout_layout(prompt_ids: torch.Tensor, sequences: torch.Tensor, pad_id: int):
    """Everything trainers/text_image_to_text/ppo.py:185-203 does after `generate`, ONE launch, no host sync:
    -> (move_padding_left(sequences), its attention mask, DeviceLens of the response lengths).  The bound of the
    lengths is the number of generated positions (a response cannot be longer)."""
    L.require_cuda(prompt_ids, sequences)
    if prompt_ids.dim() != 2 or sequences.dim() != 2 or prompt_ids.size(0) != sequences.size(0) or \
            prompt_ids.dtype != torch.int64 or sequences.dtype != torch.int64:
        raise ValueError('rollout_layout expects int64 prompt_ids (B, P) and sequences (B, L)')
    p, x = _contiguous_last(prompt_ids), _contiguous_last(sequences)
    B, Lq = x.shape
    moved = torch.empty((B, Lq), dtype=torch.int64, device=x.device)
    mask = torch.empty((B, Lq), dtype=torch.bool, device=x.device)
    lens = torch.empty(B, dtype=torch.int32, device=x.device)
    L.check(L.lib().aa_ppo_rollout_layout(p.data_ptr(), p.size(1), p.stride(0), x.data_ptr(), Lq, x.stride(0), B, int(pad_id),
                                          moved.data_ptr(), mask.data_ptr(), lens.data_ptr(), L.stream_ptr(x.device)))
    return moved, mask, DeviceLens(lens, max(Lq - p.size(1), 1))


def response_tail_log_probs(logits: torch.Tensor, input_ids: torch.Tensor, lens, mode: str | None = None) -> torch.Tensor:
    """The multimodal PPO scoring rows (trainers/text_image_to_text/ppo.py:229-246, 296-309): sample b scores
    `logits[b, :-1][-R_b:]` against `input_ids[b, 1:][-R_b:]`, right-padded with 0 to (B, W), W = the lengths' bound.
    `logits` is (B, K, V) with K <= L: the LAST K positions of the sequences (K = L: the whole tile; K = W + 1: the
    `logits_to_keep` tail tile).  The labels are read in place from input_ids, the row plan is built on the device."""
    L.require_cuda(logits, input_ids)
    lens = as_device_lens(lens, logits.device)
    B, K, _ = logits.shape
    if input_ids.shape[0] != B or len(lens) != B or K > input_ids.size(1):
        raise ValueError('response_tail_log_probs: logits (B, K, V), input_ids (B, L >= K), one length per sample')
    if lens.bound > K - 1:
        raise ValueError(f'the logits tile holds {K} positions: too few for responses of up to {lens.bound} tokens')
    logits, ids = _contiguous_last(logits), input_ids.contiguous()
    plan = device_tail_plan(lens, K, logits.stride(0), logits.stride(1), ids.stride(0), ids.size(1), 0, -1, lens.bound)
    return _LogProbFn.apply(logits, ids, plan, _mode_code(mode, logits.dtype))


def response_tail_log_probs_pair(logits_a: torch.Tensor, logits_b: torch.Tensor, input_ids: torch.Tensor, lens,
                                 mode: str | None = None):
    """response_tail_log_probs of TWO logits tensors of identical shape / dtype / strides against the same labels (the
    rollout's actor and reference model, text_image_to_text/ppo.py:229-246) in ONE K1 launch: the second tensor is
    addressed relative to the first one's base pointer.  No gradient.  -> (log_probs_a, log_probs_b), each (B, W)."""
    return _tail_pair(logits_a, logits_b, input_ids, lens, mode, False)


def response_tail_log_probs_pair_with_entropy(logits_a: torch.Tensor, logits_b: torch.Tensor, input_ids: torch.Tensor,
                                              lens, mode: str | None = None):
    """response_tail_log_probs_pair plus the fp32 policy entropy of the FIRST tensor's scored rows (the actor's), from
    the same single launch (K1's entropy variant; the second copy's rows skip the store).  -> (log_probs_a, log_probs_b,
    entropy_a), each (B, W); the log-probs are bit-identical to response_tail_log_probs_pair's."""
    return _tail_pair(logits_a, logits_b, input_ids, lens, mode, True)


def _tail_pair(logits_a, logits_b, input_ids, lens, mode, with_entropy: bool):
    L.require_cuda(logits_a, logits_b, input_ids)
    lens = as_device_lens(lens, logits_a.device)
    a, b = _contiguous_last(logits_a.detach()), _contiguous_last(logits_b.detach())
    if a.shape != b.shape or a.dtype != b.dtype or a.stride() != b.stride():
        raise ValueError('both logits tensors must share shape, dtype and strides')
    B, K, _ = a.shape
    if lens.bound > K - 1:
        raise ValueError(f'the logits tile holds {K} positions: too few for responses of up to {lens.bound} tokens')
    delta = b.data_ptr() - a.data_ptr()
    if delta % a.element_size():
        raise ValueError('logits tensors are not element-aligned relative to each other')
    ids = input_ids.contiguous()
    plan = device_tail_plan(lens, K, a.stride(0), a.stride(1), ids.stride(0), ids.size(1), 0, -1, lens.bound, 2,
                            delta // a.element_size())
    mode_code = _mode_code(mode, a.dtype)
    out = torch.zeros(plan.out_shape, dtype=a.dtype if mode_code == L.MODE_FAITHFUL else torch.float32, device=a.device)
    if not with_entropy:
        _launch_fwd(a, ids, plan, out, None, None)
        return out[0], out[1]
    entropy = torch.zeros(plan.out_shape[1:], dtype=torch.float32, device=a.device)  # room for the first copy only
    _launch_fwd(a, ids, plan, out, None, None, entropy=entropy)
    return out[0], out[1], entropy


def count_nonpad(ids: torch.Tensor, pad_id: int) -> torch.Tensor:
    """Per-row number of tokens != pad (int32, on device): the bookkeeping behind
    trainers/text_image_to_text/ppo.py:190-203 without the per-sample `.tolist()`."""
    L.require_cuda(ids)
    x = _contiguous_last(ids)
    out = torch.empty(x.size(0), dtype=torch.int32, device=x.device)
    L.check(L.lib().aa_count_nonpad(x.data_ptr(), x.size(0), x.size(1), x.stride(0), int(pad_id), out.data_ptr(),
                                    L.stream_ptr(x.device)))
    return out
