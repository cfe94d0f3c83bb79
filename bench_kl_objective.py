"""bench_kl_objective.py -- what the KL estimator options cost on one H100.

    python bench_kl_objective.py [--rounds R] [--iters N]

Each pair of arms alternates within one process on one card (CUDA events around N back-to-back steps per round; the
median of R rounds per arm):
  k4_c4: K4 (ops.kl_rewards_and_gae) at bench.py's C4 rollout shape, 32 responses of 512 tokens after 512 prompt
     tokens, bf16 log-probs: the reference's k1 penalty (aa_ppo_prep) against k3 (aa_ppo_prep_kl), 100 x N launches
     per round;
  grpo_single_pass_c4: forward + backward of K1f's GRPO node (ops.grpo_loss_from_logits) over 32 completions of 512
     tokens, V = 152064 bf16 logits: the reference's loss (k3, today's launch) against k2 on the objective kernel;
  grpo_composed_c4: the same shape forced through the composed path, K1 -> aa_grpo_loss{,_kl} -> K1b.
Prints one JSON line with the card's name, power limit and max SM clock next to the times.
"""
from __future__ import annotations

import argparse
import json

import torch

from align_anything_b200 import ops
from bench_entropy import _alternate, _card


def _k4_arms(B: int, P: int, R: int) -> dict:
    gen = torch.Generator(device='cuda').manual_seed(4)
    W = P + R
    lp = (-torch.rand(B, W, device='cuda', generator=gen) * 4).bfloat16()
    ref = (lp.float() + torch.randn(B, W, device='cuda', generator=gen) * 0.3).bfloat16()
    values = torch.randn(B, W, device='cuda', generator=gen).bfloat16()
    mask = torch.ones(B, W, dtype=torch.bool, device='cuda')
    reward = torch.randn(B, device='cuda', generator=gen)

    def step(est):
        return lambda: ops.kl_rewards_and_gae(reward, lp, ref, values, mask, P, 0.02, 50.0, 1.0, 0.95, kl_estimator=est)

    return {'k1': step('k1'), 'k3': step('k3')}


def _grpo_arms(B: int, K: int, V: int, single_pass: bool) -> dict:
    gen = torch.Generator(device='cuda').manual_seed(V)
    L = K + 1
    logits = (torch.randn(B, L, V, device='cuda', generator=gen) * 2.0).to(torch.bfloat16).requires_grad_(True)
    ids = torch.randint(2, V, (B, L), device='cuda', generator=gen)
    with torch.no_grad():
        ref = ops.tail_token_log_probs(logits, ids, K).float()
    ref = ref + torch.randn(B, K, device='cuda', generator=gen) * 0.3
    adv = torch.randn(B, 1, device='cuda', generator=gen)

    def step(objective):
        def run():
            logits.grad = None
            saved = ops._FUSED_GRPO
            ops._FUSED_GRPO = single_pass
            try:
                out = ops.grpo_loss_from_logits(logits, ids, K, ref, adv, 1, 0.04, objective=objective)
            finally:
                ops._FUSED_GRPO = saved
            out[0].backward()
        return run

    return {'reference_k3': step(None), 'k2': step(ops.GrpoObjective(kl_estimator='k2'))}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--iters', type=int, default=5)
    a = ap.parse_args()
    res = {'card': _card()}
    # K4 is a ~50 us launch: 100 x iters back-to-back launches per round, so a round is ~25 ms and launch jitter
    # averages out of the round time
    res['k4_c4'] = _alternate(_k4_arms(32, 512, 512), a.rounds, 100 * a.iters)
    res['grpo_single_pass_c4'] = _alternate(_grpo_arms(32, 512, 152064, True), a.rounds, a.iters)
    torch.cuda.empty_cache()
    res['grpo_composed_c4'] = _alternate(_grpo_arms(32, 512, 152064, False), a.rounds, a.iters)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
