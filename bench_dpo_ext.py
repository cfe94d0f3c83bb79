"""bench_dpo_ext.py -- what the further DPO objectives cost the DPO node on one H100.

    python bench_dpo_ext.py [--rounds R] [--iters N]

Forward + backward of the DPO node with three objectives, the arms alternating within one process on one card (CUDA
events around N back-to-back steps per round; the median of R rounds per arm):
  reference:   the reference's loss (aa_dpo_loss);
  js_exo:      ops.DpoObjective(loss_type='exo_pair', f_divergence_type='js_divergence') (aa_dpo_loss_ext);
  aot:         ops.DpoObjective(loss_type='aot') (aa_dpo_loss_ext, with the in-kernel sort).
Two nodes:
  tile_c2: ops.dpo_fused_loss at bench.py's C2 shape, 16 pairs of 2048 tokens over V = 128257 bf16 logits (K1 x2, K2,
     K1b);
  lm_head_c2: the fused lm_head DPO node at bench.py's lm_head leg shape (4 pairs x 2048, H = 4096, V = 128257, bf16):
     ops.sequence_log_probs_from_hidden for the policy and the reference + ops.dpo_loss_from_log_probs, backward down
     to the hidden states and the lm_head weight.
The reference model's inputs are the policy's plus a little noise, so the log-ratios are of the size training sees.
With independent random logits they run to hundreds, a saturating objective's seeds round to exactly 0, and K1b skips
the rows of a zero seed: such an arm would time less work, not the objective.  `zero_seeds` reports, per arm, how many
of the B chosen-row seeds are exactly 0 (the times compare only when the arms do the same work).
Prints one JSON line with the card's name, power limit and max SM clock next to the times.
"""
from __future__ import annotations

import argparse
import json

import torch

from align_anything_b200 import ops
from bench_dpo_objective import _ids
from bench_entropy import _alternate, _card

OBJECTIVES = {'reference': None, 'js_exo': ops.DpoObjective(loss_type='exo_pair', f_divergence_type='js_divergence'),
              'aot': ops.DpoObjective(loss_type='aot')}
BETA = 0.1


def _zero_seeds(out) -> int:
    return int((out['_per_pair'][3] == 0).sum())  # per_pair[3]: d loss / d chosen sum, one per pair


def _tile_arms(pairs: int = 16, L: int = 2048, V: int = 128257):
    gen = torch.Generator(device='cuda').manual_seed(V)
    n = 2 * pairs
    logits = torch.randn((n, L, V), device='cuda', generator=gen, dtype=torch.bfloat16).requires_grad_(True)
    ref = torch.randn((n, L, V), device='cuda', generator=gen, dtype=torch.bfloat16).mul_(0.05).add_(logits.detach())
    ids, lens, pad = _ids(n, L, V, gen)
    zeros = {}

    def step(name, objective):
        def run():
            logits.grad = None
            out = ops.dpo_fused_loss(logits, ref, ids, lens, pad, BETA, objective=objective)
            out['loss'].backward()
            return out
        zeros[name] = _zero_seeds(run())
        return run

    return {name: step(name, obj) for name, obj in OBJECTIVES.items()}, zeros


def _lm_head_arms(pairs: int = 4, L: int = 2048, H: int = 4096, V: int = 128257):
    gen = torch.Generator(device='cuda').manual_seed(2)
    n = 2 * pairs
    hidden = torch.randn((n, L, H), device='cuda', generator=gen).bfloat16().requires_grad_(True)
    ref_hidden = (hidden.detach().float() + 0.05 * torch.randn((n, L, H), device='cuda', generator=gen)).bfloat16()
    weight = (torch.randn((V, H), device='cuda', generator=gen) * 0.02).bfloat16().requires_grad_(True)
    ids, lens, pad = _ids(n, L, V, gen)
    zeros = {}

    def step(name, objective):
        def run():
            hidden.grad = weight.grad = None
            lp = ops.sequence_log_probs_from_hidden(hidden, weight, ids, lens, pad)
            with torch.no_grad():
                ref_lp = ops.sequence_log_probs_from_hidden(ref_hidden, weight, ids, lens, pad)
            out = ops.dpo_loss_from_log_probs(lp, ref_lp, BETA, objective=objective, response_lens=lens)
            out['loss'].backward()
            return out
        zeros[name] = _zero_seeds(run())
        return run

    return {name: step(name, obj) for name, obj in OBJECTIVES.items()}, zeros


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--iters', type=int, default=3)
    a = ap.parse_args()
    res = {'card': _card()}
    for node, make in (('tile_c2', _tile_arms), ('lm_head_c2', _lm_head_arms)):
        arms, zeros = make()
        res[node] = _alternate(arms, a.rounds, a.iters)
        res[node]['zero_seeds'] = zeros
        del arms
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
