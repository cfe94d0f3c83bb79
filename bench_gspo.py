"""bench_gspo.py -- what GSPO's sequence-level ratio costs GRPO's policy node on one H100.

    python bench_gspo.py [--rounds R] [--iters N]

Forward + backward of the GRPO node at an update 2..mu (rollout-time old log-probs), with the same objective fields
(ops.GrpoObjective(0.2, 0.28, None, 'seq-mean-token-mean')) at importance_sampling_level 'token' and 'sequence', the
two arms alternating within one process on one card (CUDA events around N back-to-back steps per round; the median of
R rounds per arm):
  single pass vs composed at C4: K1f's GRPO node (token level) against the composed sequence-level node,
     K1 -> aa_grpo_loss_seq -> K1b, at bench.py's C4 shape, 32 completions of 512 tokens over V = 152064 bf16 logits;
  composed at C4: both levels forced through the composed path, which isolates the loss kernel's sequence pass;
  lm_head: the fused lm_head GRPO node at the C2 lm_head shape (8 x 2047 = 16 376 rows, H = 4096, V = 128257, bf16):
     K6 -> GRPO loss forward, K6b + d(hidden) + d(weight) backward, at each level.
Prints one JSON line with the card's name and power limit next to the times.
"""
from __future__ import annotations

import argparse
import json

import torch

from align_anything_b200 import ops
from bench_entropy import _alternate, _card

FIELDS = (0.2, 0.28, None, 'seq-mean-token-mean')
OBJECTIVES = {level: ops.GrpoObjective(*FIELDS, importance_sampling_level=level) for level in ('token', 'sequence')}


def _arms(loss_fn, lp_old: torch.Tensor) -> dict:
    """{'token': the token-level ratio, 'sequence': GSPO's}, both with old log-probs."""
    return {level: (lambda obj=obj: loss_fn({'objective': obj, 'old_per_token_logps': lp_old}))
            for level, obj in OBJECTIVES.items()}


def _tile_arms(B: int, K: int, V: int, single_pass: bool) -> dict:
    gen = torch.Generator(device='cuda').manual_seed(V)
    L = K + 1
    logits = (torch.randn(B, L, V, device='cuda', generator=gen) * 2.0).to(torch.bfloat16).requires_grad_(True)
    ids = torch.randint(2, V, (B, L), device='cuda', generator=gen)
    with torch.no_grad():
        lp = ops.tail_token_log_probs(logits, ids, K)
    ref = (lp.float() + torch.randn(B, K, device='cuda', generator=gen) * 0.1).to(lp.dtype)
    old = (lp.float() + torch.randn(B, K, device='cuda', generator=gen) * 0.3).to(lp.dtype)  # some ratios clip
    adv = torch.randn(B, 1, device='cuda', generator=gen)

    def run(kw):
        logits.grad = None
        saved = ops._FUSED_GRPO
        ops._FUSED_GRPO = single_pass  # the sequence level takes the composed path either way
        try:
            out = ops.grpo_loss_from_logits(logits, ids, K, ref, adv, 1, 0.04, **kw)
        finally:
            ops._FUSED_GRPO = saved
        out[0].backward()

    return _arms(run, old)


def _lm_head_arms() -> dict:
    gen = torch.Generator(device='cuda').manual_seed(2)
    B, L, H, V = 8, 2048, 4096, 128257
    K = L - 1
    hidden = torch.randn(B, L, H, device='cuda', generator=gen).bfloat16().requires_grad_(True)
    weight = (torch.randn(V, H, device='cuda', generator=gen) * 0.02).bfloat16().requires_grad_(True)
    ids = torch.randint(2, V, (B, L), device='cuda', generator=gen)
    with torch.no_grad():
        lp = ops.dense_log_probs_from_hidden(hidden, weight, ids, 0)
    ref = (lp.float() + torch.randn(B, K, device='cuda', generator=gen) * 0.1).to(lp.dtype)
    old = (lp.float() + torch.randn(B, K, device='cuda', generator=gen) * 0.3).to(lp.dtype)
    adv = torch.randn(B, 1, device='cuda', generator=gen)

    def run(kw):
        hidden.grad = weight.grad = None
        x = ops.dense_log_probs_from_hidden(hidden, weight, ids, 0)
        ops.grpo_loss(x, ref, adv, ids[:, -K:], 1, 0.04, **kw)[0].backward()

    return _arms(run, old)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--iters', type=int, default=5)
    a = ap.parse_args()
    res = {'card': _card()}
    res['single_pass_token_vs_composed_sequence_c4'] = _alternate(_tile_arms(32, 512, 152064, True), a.rounds, a.iters)
    torch.cuda.empty_cache()
    res['composed_c4'] = _alternate(_tile_arms(32, 512, 152064, False), a.rounds, a.iters)
    torch.cuda.empty_cache()
    res['lm_head_c2'] = _alternate(_lm_head_arms(), a.rounds, 2)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
