"""bench_kl_loss.py -- what the KL term in the PPO actor loss costs on one H100.

    python bench_kl_loss.py [--rounds R] [--iters N]

Forward + backward of the actor node without and with a k3 KL loss term (kl_loss_coeff 0.1), the two arms alternating
within one process on one card (CUDA events around N back-to-back steps per round; the median of R rounds per arm):
  single pass: the K1f actor node (ops.dense_actor_loss) at bench.py's C4 shape, 32 responses of 512 tokens over
     V = 152064 bf16 logits (16 384 scored rows): aa_logprob_actor_fused -> K5 against their _kl entry points;
  composed at C4: the same shape forced through the composed path, K1 -> K5 -> K1b;
  lm_head: the fused lm_head actor node at the C2 lm_head shape (8 x 2047 = 16 376 rows, H = 4096, V = 128257, bf16):
     K6 -> K5 forward, K6b + d(hidden) + d(weight) backward;
  k5: K5 alone on the C4 log-probs (32 x 512), 200 back-to-back launches per round: aa_ppo_actor_loss_obj against
     aa_ppo_actor_loss_kl, where the per-token KL is the whole difference.
Prints one JSON line with the card's name, power limit and max SM clock next to the times.
"""
from __future__ import annotations

import argparse
import json

import torch

from align_anything_b200 import ops
from bench_entropy import _alternate, _card

KL = {'plain': {}, 'kl_k3': {'kl_loss_coeff': 0.1, 'kl_loss_estimator': 'k3'}}


def _actor_arms(B: int, R: int, V: int, single_pass: bool) -> dict:
    gen = torch.Generator(device='cuda').manual_seed(V)
    L, start = R + 1, 0
    logits = (torch.randn(B, L, V, device='cuda', generator=gen) * 2.0).to(torch.bfloat16).requires_grad_(True)
    ids = torch.randint(0, V, (B, L), device='cuda', generator=gen)
    with torch.no_grad():
        old = ops.gather_log_probabilities(logits[:, :-1], ids[:, 1:]).float()
    ref = old + torch.randn(B, R, device='cuda', generator=gen) * 0.3
    old = old + torch.randn(B, R, device='cuda', generator=gen) * 0.3  # ratios inside and outside the clip range
    adv = torch.randn(B, R, device='cuda', generator=gen)
    mask = torch.ones(B, R, dtype=torch.bool, device='cuda')

    def step(kw):
        def run():
            logits.grad = None
            saved = ops._FUSED_ACTOR
            ops._FUSED_ACTOR = single_pass
            try:
                out = ops.dense_actor_loss(logits, ids, start, old, adv, mask, 0.2, ref_log_probs=ref, **kw)
            finally:
                ops._FUSED_ACTOR = saved
            out[0].backward()
        return run

    return {name: step(kw) for name, kw in KL.items()}


def _lm_head_arms() -> dict:
    gen = torch.Generator(device='cuda').manual_seed(2)
    B, L, H, V = 8, 2048, 4096, 128257
    hidden = torch.randn(B, L, H, device='cuda', generator=gen).bfloat16().requires_grad_(True)
    weight = (torch.randn(V, H, device='cuda', generator=gen) * 0.02).bfloat16().requires_grad_(True)
    ids = torch.randint(0, V, (B, L), device='cuda', generator=gen)
    with torch.no_grad():
        old = ops.dense_log_probs_from_hidden(hidden, weight, ids, 0).float()
    ref = old + torch.randn(B, L - 1, device='cuda', generator=gen) * 0.3
    adv = torch.randn(B, L - 1, device='cuda', generator=gen)
    mask = torch.ones(B, L - 1, dtype=torch.bool, device='cuda')

    def step(kw):
        def run():
            hidden.grad = weight.grad = None
            lp = ops.dense_log_probs_from_hidden(hidden, weight, ids, 0)
            out = ops.actor_loss(lp, old, adv, mask, 0.2, ref_log_probs=ref, **kw)
            (out[0] if kw else out).backward()
        return run

    return {name: step(kw) for name, kw in KL.items()}


def _k5_arms(B: int = 32, R: int = 512) -> dict:
    from align_anything_b200 import _lib as L

    gen = torch.Generator(device='cuda').manual_seed(5)
    lp = (-torch.rand(B, R, device='cuda', generator=gen) * 4).bfloat16()
    old = (lp.float() + torch.randn(B, R, device='cuda', generator=gen) * 0.3).bfloat16()
    ref = (lp.float() + torch.randn(B, R, device='cuda', generator=gen) * 0.3).bfloat16()
    adv = torch.randn(B, R, device='cuda', generator=gen)
    mask = torch.ones(B, R, dtype=torch.uint8, device='cuda')
    loss, kl = torch.empty(2, device='cuda'), torch.empty(1, device='cuda')
    grad = torch.empty_like(lp)
    rows = torch.empty(5 * B, device='cuda')
    counter = torch.zeros(1, dtype=torch.int32, device='cuda')
    lib, st = L.lib(), L.stream_ptr()
    head = (lp.data_ptr(), R, old.data_ptr(), R, L.AA_BF16, adv.data_ptr(), R, L.AA_F32, mask.data_ptr(), R, B, R,
            0.2, 0.2, 0.0, 0, L.MODE_FAITHFUL)
    tail = (grad.data_ptr(), R, None, rows.data_ptr(), counter.data_ptr(), st)

    def plain():
        for _ in range(200):
            L.check(lib.aa_ppo_actor_loss_obj(*head, loss.data_ptr(), *tail))

    def with_kl():
        for _ in range(200):
            L.check(lib.aa_ppo_actor_loss_kl(*head, ref.data_ptr(), R, 0.1, 2, loss.data_ptr(), kl.data_ptr(), *tail))

    return {'plain': plain, 'kl_k3': with_kl}


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
    torch.cuda.empty_cache()
    k5 = _alternate(_k5_arms(), a.rounds, 1)
    res['k5_c4_per_launch'] = {k: {m: t / 200 for m, t in v.items()} for k, v in k5.items()}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
