"""bench_top_entropy.py -- what high-entropy token masking (top_entropy_quantile = rho) costs GRPO's policy node on one
H100.

    python bench_top_entropy.py [--rounds R] [--iters N]

Forward + backward of the GRPO node at rho = 1 (no mask) and rho = 0.2, the arms alternating within one process on one
card (CUDA events around N back-to-back steps per round; the median of R rounds per arm):
  single pass vs composed at C4: K1f's GRPO node (rho = 1) against the masked node, K1's entropy variant -> the entropy
     quantile -> aa_grpo_loss_topent -> K1b, at bench.py's C4 shape, 32 completions of 512 tokens over V = 152064 bf16
     logits;
  composed at C4: both arms forced through the composed path, which isolates the selection and the mask;
  selection at C4: aa_grpo_row_end and the four selection launches alone, over 32 x 512 tokens;
  lm_head: the fused lm_head GRPO node at the C2 lm_head shape (8 x 2047 = 16 376 rows, H = 4096, V = 128257, bf16):
     K6 with the entropy -> GRPO loss forward, K6b + d(hidden) + d(weight) backward, at each rho.
Prints one JSON line with the card's name and power limit next to the times.
"""
from __future__ import annotations

import argparse
import json

import torch

from align_anything_b200 import ops
from bench_entropy import _alternate, _card

OBJECTIVES = {'rho=1': ops.GrpoObjective(), 'rho=0.2': ops.GrpoObjective(top_entropy_quantile=0.2)}


def _tile_arms(B: int, K: int, V: int, single_pass: bool) -> dict:
    gen = torch.Generator(device='cuda').manual_seed(V)
    L = K + 1
    logits = (torch.randn(B, L, V, device='cuda', generator=gen) * 2.0).to(torch.bfloat16).requires_grad_(True)
    ids = torch.randint(2, V, (B, L), device='cuda', generator=gen)
    with torch.no_grad():
        lp = ops.tail_token_log_probs(logits, ids, K)
    ref = (lp.float() + torch.randn(B, K, device='cuda', generator=gen) * 0.1).to(lp.dtype)
    adv = torch.randn(B, 1, device='cuda', generator=gen)

    def run(obj):
        logits.grad = None
        saved = ops._FUSED_GRPO
        ops._FUSED_GRPO = single_pass  # rho < 1 takes the composed path either way
        try:
            out = ops.grpo_loss_from_logits(logits, ids, K, ref, adv, 1, 0.04, objective=obj)
        finally:
            ops._FUSED_GRPO = saved
        out[0].backward()

    return {k: (lambda obj=obj: run(obj)) for k, obj in OBJECTIVES.items()}


def _selection_arms(B: int, K: int) -> dict:
    gen = torch.Generator(device='cuda').manual_seed(K)
    ent = torch.rand(B, K, device='cuda', generator=gen) * 4
    tokens = torch.randint(2, 1000, (B, K), device='cuda', generator=gen)
    tokens[::3, K // 2] = 1

    def run():
        ops.entropy_quantile_threshold(ent, ops.grpo_row_end(tokens, 1), 0.8)

    return {'row_end+selection': run}


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
    adv = torch.randn(B, 1, device='cuda', generator=gen)

    def run(obj):
        hidden.grad = weight.grad = None
        if ops._top_entropy(obj):  # the trainer asks K6 for the entropy only when the mask needs it
            x, ent = ops.dense_log_probs_from_hidden(hidden, weight, ids, 0, return_entropy=True)
            kw = {'entropy': ent}
        else:
            x, kw = ops.dense_log_probs_from_hidden(hidden, weight, ids, 0), {}
        ops.grpo_loss(x, ref, adv, ids[:, -K:], 1, 0.04, objective=obj, **kw)[0].backward()

    return {k: (lambda obj=obj: run(obj)) for k, obj in OBJECTIVES.items()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--iters', type=int, default=5)
    a = ap.parse_args()
    res = {'card': _card()}
    res['single_pass_vs_masked_c4'] = _alternate(_tile_arms(32, 512, 152064, True), a.rounds, a.iters)
    torch.cuda.empty_cache()
    res['composed_c4'] = _alternate(_tile_arms(32, 512, 152064, False), a.rounds, a.iters)
    torch.cuda.empty_cache()
    res['selection_c4'] = _alternate(_selection_arms(32, 512), a.rounds, 20)
    res['lm_head_c2'] = _alternate(_lm_head_arms(), a.rounds, 2)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
