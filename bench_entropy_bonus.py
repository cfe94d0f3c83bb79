"""bench_entropy_bonus.py -- what the entropy bonus costs the PPO actor node on one H100.

    python bench_entropy_bonus.py [--rounds R] [--iters N]

Forward + backward of ops.dense_actor_loss with entropy_coeff = 0 against entropy_coeff = 0.01, the two arms alternating
within one process on one card (CUDA events around N back-to-back steps per round; the median of R rounds per arm):
  single pass: the K1f actor node at bench.py's C4 shape, 32 responses of 512 tokens over V = 152064 bf16 logits
     (16 384 scored rows), the bonus from K1f's entropy-gradient variant;
  composed: a C3 vocabulary, V = 32064 (below K1f's row threshold), 16 384 scored rows: K1 -> K5 -> K1b, the bonus
     from K1's and K1b's entropy variants;
  composed at C4: the C4 shape forced through the composed path, the yardstick the single pass with the bonus must beat;
  lm_head: the fused lm_head actor node at the C2 lm_head shape (8 x 2047 = 16 376 rows, H = 4096, V = 128257, bf16):
     K6 -> K5 (+ masked_mean) forward, K6b + d(hidden) + d(weight) backward; the bonus from K6's entropy variant and
     K6b's entropy epilogue.
Prints one JSON line with the card's name and power limit next to the times.
"""
from __future__ import annotations

import argparse
import json

import torch

from align_anything_b200 import ops
from bench_entropy import _alternate, _card


def _actor_arms(B: int, R: int, V: int, single_pass: bool) -> dict:
    gen = torch.Generator(device='cuda').manual_seed(V)
    L, start = R + 1, 0
    logits = (torch.randn(B, L, V, device='cuda', generator=gen) * 2.0).to(torch.bfloat16).requires_grad_(True)
    ids = torch.randint(0, V, (B, L), device='cuda', generator=gen)
    with torch.no_grad():
        old = ops.gather_log_probabilities(logits[:, :-1], ids[:, 1:]).float()
    adv = torch.randn(B, R, device='cuda', generator=gen)
    mask = torch.ones(B, R, dtype=torch.bool, device='cuda')

    def step(coeff):
        def run():
            logits.grad = None
            saved = ops._FUSED_ACTOR
            ops._FUSED_ACTOR = single_pass
            try:
                out = ops.dense_actor_loss(logits, ids, start, old, adv, mask, 0.2, entropy_coeff=coeff)
            finally:
                ops._FUSED_ACTOR = saved
            out[0].backward()
        return run

    return {'coeff_0': step(0.0), 'coeff_0.01': step(0.01)}


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

    def step(coeff):
        def run():
            hidden.grad = weight.grad = None
            if coeff == 0.0:
                lp = ops.dense_log_probs_from_hidden(hidden, weight, ids, 0)
                loss = ops.actor_loss(lp, old, adv, mask, 0.2)
            else:
                lp, ent = ops.dense_log_probs_from_hidden(hidden, weight, ids, 0, return_entropy=True, entropy_grad=True)
                loss = ops.actor_loss(lp, old, adv, mask, 0.2) - coeff * ops.masked_mean(ent, mask)
            loss.backward()
        return run

    return {'coeff_0': step(0.0), 'coeff_0.01': step(0.01)}


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
    res['composed_c3_vocab'] = _alternate(_actor_arms(32, 512, 32064, True), a.rounds, a.iters)
    torch.cuda.empty_cache()
    res['lm_head_c2'] = _alternate(_lm_head_arms(), a.rounds, 2)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
