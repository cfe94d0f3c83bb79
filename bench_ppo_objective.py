"""bench_ppo_objective.py -- what the PPO actor objective options cost the actor node on one H100.

    python bench_ppo_objective.py [--rounds R] [--iters N]

Forward + backward of the actor node with the reference's objective against clip-higher + dual-clip + token-mean
(ops.ActorObjective(0.2, 0.28, 3.0, 'token-mean')), the two arms alternating within one process on one card (CUDA events
around N back-to-back steps per round; the median of R rounds per arm):
  single pass: the K1f actor node (ops.dense_actor_loss) at bench.py's C4 shape, 32 responses of 512 tokens over
     V = 152064 bf16 logits (16 384 scored rows);
  composed at C4: the same shape forced through the composed path, K1 -> K5 -> K1b;
  lm_head: the fused lm_head actor node at the C2 lm_head shape (8 x 2047 = 16 376 rows, H = 4096, V = 128257, bf16):
     K6 -> K5 forward, K6b + d(hidden) + d(weight) backward.
Prints one JSON line with the card's name and power limit next to the times.
"""
from __future__ import annotations

import argparse
import json

import torch

from align_anything_b200 import ops
from bench_entropy import _alternate, _card

OBJECTIVES = {'reference': None, 'clip_higher_dual_token_mean': ops.ActorObjective(0.2, 0.28, 3.0, 'token-mean')}


def _actor_arms(B: int, R: int, V: int, single_pass: bool) -> dict:
    gen = torch.Generator(device='cuda').manual_seed(V)
    L, start = R + 1, 0
    logits = (torch.randn(B, L, V, device='cuda', generator=gen) * 2.0).to(torch.bfloat16).requires_grad_(True)
    ids = torch.randint(0, V, (B, L), device='cuda', generator=gen)
    with torch.no_grad():
        old = ops.gather_log_probabilities(logits[:, :-1], ids[:, 1:]).float()
    old = old + torch.randn(B, R, device='cuda', generator=gen) * 0.3  # ratios inside and outside the clip range
    adv = torch.randn(B, R, device='cuda', generator=gen)
    mask = torch.ones(B, R, dtype=torch.bool, device='cuda')

    def step(objective):
        def run():
            logits.grad = None
            saved = ops._FUSED_ACTOR
            ops._FUSED_ACTOR = single_pass
            try:
                out = ops.dense_actor_loss(logits, ids, start, old, adv, mask, 0.2, objective=objective)
            finally:
                ops._FUSED_ACTOR = saved
            out[0].backward()
        return run

    return {name: step(obj) for name, obj in OBJECTIVES.items()}


def _lm_head_arms() -> dict:
    gen = torch.Generator(device='cuda').manual_seed(2)
    B, L, H, V = 8, 2048, 4096, 128257
    hidden = torch.randn(B, L, H, device='cuda', generator=gen).bfloat16().requires_grad_(True)
    weight = (torch.randn(V, H, device='cuda', generator=gen) * 0.02).bfloat16().requires_grad_(True)
    ids = torch.randint(0, V, (B, L), device='cuda', generator=gen)
    with torch.no_grad():
        old = ops.dense_log_probs_from_hidden(hidden, weight, ids, 0).float()
    adv = torch.randn(B, L - 1, device='cuda', generator=gen)
    mask = torch.ones(B, L - 1, dtype=torch.bool, device='cuda')

    def step(objective):
        def run():
            hidden.grad = weight.grad = None
            lp = ops.dense_log_probs_from_hidden(hidden, weight, ids, 0)
            ops.actor_loss(lp, old, adv, mask, 0.2, objective=objective).backward()
        return run

    return {name: step(obj) for name, obj in OBJECTIVES.items()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--iters', type=int, default=5)
    a = ap.parse_args()
    res = {'card': _card()}
    res['single_pass_c4'] = _alternate(_actor_arms(32, 512, 152064, True), a.rounds, a.iters)
    torch.cuda.empty_cache()
    res['composed_c4'] = _alternate(_actor_arms(32, 512, 152064, False), a.rounds, a.iters)
    torch.cuda.empty_cache()
    res['lm_head_c2'] = _alternate(_lm_head_arms(), a.rounds, 2)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
