"""bench_policy_loss.py -- what CISPO and SAPO (policy_loss_mode 'cispo' / 'sapo') cost the PPO actor node and GRPO's
policy node on one H100.

    python bench_policy_loss.py [--rounds R] [--iters N]

Forward + backward of each node, the arms alternating within one process on one card (CUDA events around N
back-to-back steps per round; the median, min and max of R rounds per arm):
  ppo_actor_c4: the PPO actor node (ops.dense_actor_loss) over 32 responses of 512 tokens, V = 152064 bf16 logits:
     K1f's single pass under vanilla, cispo and sapo, and the composed path K1 -> K5 -> K1b under vanilla;
  grpo_c4: GRPO's node (ops.grpo_loss_from_logits) at bench.py's C4 shape, update 2 (with old log-probs), the same
     four arms;
  lm_head_c2: the fused lm_head GRPO node at the C2 lm_head shape (8 x 2047 = 16 376 rows, H = 4096, V = 128257,
     bf16): K6 -> GRPO loss forward, K6b + d(hidden) + d(weight) backward, per mode.
Prints one JSON line with the card's name and power limit next to the times.
"""
from __future__ import annotations

import argparse
import json

import torch

from align_anything_b200 import ops
from bench_cov import _forced
from bench_entropy import _alternate, _card

ACTOR = {'vanilla': None, 'cispo': ops.ActorObjective(policy_loss_mode='cispo'),
         'sapo': ops.ActorObjective(policy_loss_mode='sapo')}
GRPO = {'vanilla': ops.GrpoObjective(), 'cispo': ops.GrpoObjective(policy_loss_mode='cispo'),
        'sapo': ops.GrpoObjective(policy_loss_mode='sapo')}
ARMS = (('k1f_vanilla', 'vanilla', True), ('k1f_cispo', 'cispo', True), ('k1f_sapo', 'sapo', True),
        ('composed_vanilla', 'vanilla', False))


def _ppo_arms(B: int, W: int, V: int) -> dict:
    gen = torch.Generator(device='cuda').manual_seed(V)
    logits = (torch.randn(B, W + 1, V, device='cuda', generator=gen) * 2.0).to(torch.bfloat16).requires_grad_(True)
    ids = torch.randint(2, V, (B, W + 1), device='cuda', generator=gen)
    with torch.no_grad():
        lp = ops.gather_log_probabilities(logits[:, :-1], ids[:, 1:])
    old = (lp.float() + torch.randn(B, W, device='cuda', generator=gen) * 0.1).to(lp.dtype)
    adv = torch.randn(B, W, device='cuda', generator=gen)
    mask = torch.rand(B, W, device='cuda', generator=gen) < 0.9

    def run(obj, single_pass):
        logits.grad = None
        out = _forced('_FUSED_ACTOR', single_pass,
                      lambda: ops.dense_actor_loss(logits, ids, 0, old, adv, mask, 0.2, objective=obj))
        out[0].backward()

    return {name: (lambda m=m, s=s: run(ACTOR[m], s)) for name, m, s in ARMS}


def _grpo_arms(B: int, K: int, V: int) -> dict:
    gen = torch.Generator(device='cuda').manual_seed(V + 1)
    logits = (torch.randn(B, K + 1, V, device='cuda', generator=gen) * 2.0).to(torch.bfloat16).requires_grad_(True)
    ids = torch.randint(2, V, (B, K + 1), device='cuda', generator=gen)
    with torch.no_grad():
        lp = ops.tail_token_log_probs(logits, ids, K)
    ref = (lp.float() + torch.randn(B, K, device='cuda', generator=gen) * 0.1).to(lp.dtype)
    old = (lp.float() + torch.randn(B, K, device='cuda', generator=gen) * 0.1).to(lp.dtype)
    adv = torch.randn(B, 1, device='cuda', generator=gen)

    def run(obj, single_pass):
        logits.grad = None
        out = _forced('_FUSED_GRPO', single_pass,
                      lambda: ops.grpo_loss_from_logits(logits, ids, K, ref, adv, 1, 0.04, objective=obj,
                                                        old_per_token_logps=old))
        out[0].backward()

    return {name: (lambda m=m, s=s: run(GRPO[m], s)) for name, m, s in ARMS}


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
    old = (lp.float() + torch.randn(B, K, device='cuda', generator=gen) * 0.1).to(lp.dtype)
    adv = torch.randn(B, 1, device='cuda', generator=gen)

    def run(obj):
        hidden.grad = weight.grad = None
        x = ops.dense_log_probs_from_hidden(hidden, weight, ids, 0)
        ops.grpo_loss(x, ref, adv, ids[:, -K:], 1, 0.04, objective=obj, old_per_token_logps=old)[0].backward()

    return {k: (lambda obj=obj: run(obj)) for k, obj in GRPO.items()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--iters', type=int, default=5)
    a = ap.parse_args()
    res = {'card': _card()}
    res['ppo_actor_c4'] = _alternate(_ppo_arms(32, 512, 152064), a.rounds, a.iters)
    torch.cuda.empty_cache()
    res['grpo_c4'] = _alternate(_grpo_arms(32, 512, 152064), a.rounds, a.iters)
    torch.cuda.empty_cache()
    res['lm_head_c2'] = _alternate(_lm_head_arms(), a.rounds, 2)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
