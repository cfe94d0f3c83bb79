"""bench_dpo_objective.py -- what the DPO objective options cost the DPO node on one H100.

    python bench_dpo_objective.py [--rounds R] [--iters N]

Forward + backward of the DPO node with three objectives, the arms alternating within one process on one card (CUDA
events around N back-to-back steps per round; the median of R rounds per arm):
  reference:       the reference's loss (aa_dpo_loss);
  ipo_rpo:         ops.DpoObjective(loss_type='ipo', rpo_alpha=1.0) (aa_dpo_loss_obj with the row counts);
  reference_free:  ops.DpoObjective(reference_free=True): no reference K1 pass.
Two nodes:
  tile_c2: ops.dpo_fused_loss at bench.py's C2 shape, 16 pairs of 2048 tokens over V = 128257 bf16 logits (K1 x2, K2,
     K1b; the reference logits are given to every arm, as a trainer's reference forward would have made them);
  lm_head_c2: the fused lm_head DPO node at bench.py's lm_head leg shape (4 pairs x 2048, H = 4096, V = 128257, bf16):
     ops.sequence_log_probs_from_hidden for the policy (and the reference) + ops.dpo_loss_from_log_probs, backward down
     to the hidden states and the lm_head weight.
Prints one JSON line with the card's name and power limit next to the times.
"""
from __future__ import annotations

import argparse
import json

import torch

from align_anything_b200 import ops
from bench_entropy import _alternate, _card

OBJECTIVES = {'reference': None, 'ipo_rpo': ops.DpoObjective(loss_type='ipo', rpo_alpha=1.0),
              'reference_free': ops.DpoObjective(reference_free=True)}
BETA = 0.1


def _ids(n: int, L: int, V: int, gen):
    ids = torch.randint(0, V - 1, (n, L), device='cuda', generator=gen)  # V - 1 is the pad id: no pad in the rows
    return ids, [L - 16 - 8 * (i % 4) for i in range(n)], V - 1


def _tile_arms(pairs: int = 16, L: int = 2048, V: int = 128257) -> dict:
    gen = torch.Generator(device='cuda').manual_seed(V)
    n = 2 * pairs
    logits = torch.randn((n, L, V), device='cuda', generator=gen, dtype=torch.bfloat16).requires_grad_(True)
    ref = torch.randn((n, L, V), device='cuda', generator=gen, dtype=torch.bfloat16)
    ids, lens, pad = _ids(n, L, V, gen)

    def step(objective):
        def run():
            logits.grad = None
            ops.dpo_fused_loss(logits, ref, ids, lens, pad, BETA, objective=objective)['loss'].backward()
        return run

    return {name: step(obj) for name, obj in OBJECTIVES.items()}


def _lm_head_arms(pairs: int = 4, L: int = 2048, H: int = 4096, V: int = 128257) -> dict:
    gen = torch.Generator(device='cuda').manual_seed(2)
    n = 2 * pairs
    hidden = torch.randn((n, L, H), device='cuda', generator=gen).bfloat16().requires_grad_(True)
    ref_hidden = torch.randn((n, L, H), device='cuda', generator=gen).bfloat16()
    weight = (torch.randn((V, H), device='cuda', generator=gen) * 0.02).bfloat16().requires_grad_(True)
    ids, lens, pad = _ids(n, L, V, gen)

    def step(objective):
        def run():
            hidden.grad = weight.grad = None
            lp = ops.sequence_log_probs_from_hidden(hidden, weight, ids, lens, pad)
            ref_lp = None
            if objective is None or not objective.reference_free:
                with torch.no_grad():
                    ref_lp = ops.sequence_log_probs_from_hidden(ref_hidden, weight, ids, lens, pad)
            ops.dpo_loss_from_log_probs(lp, ref_lp, BETA, objective=objective, response_lens=lens)['loss'].backward()
        return run

    return {name: step(obj) for name, obj in OBJECTIVES.items()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--iters', type=int, default=3)
    a = ap.parse_args()
    res = {'card': _card()}
    res['tile_c2'] = _alternate(_tile_arms(), a.rounds, a.iters)
    torch.cuda.empty_cache()
    res['lm_head_c2'] = _alternate(_lm_head_arms(), a.rounds, a.iters)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
