"""bench_entropy.py -- what the policy entropy costs the log-prob kernels on one H100.

    python bench_entropy.py [--rounds R] [--iters N]

Two kernels, each timed with and without its entropy accumulator, the two arms alternating within one process on one
card (CUDA events around N back-to-back launches per round; the median of R rounds is reported per arm):
  K1 (aa_logprob_fwd vs aa_logprob_fwd_entropy): the PPO rollout scoring shape of bench.py's C4 config, 32 responses of
     512 tokens over V = 152064 bf16 logits (16 384 rows, 5.0 GB read per launch);
  K6 (aa_linear_logprob_fwd vs aa_linear_logprob_fwd_entropy): the C2 lm_head shape, 16 376 rows, H = 4096,
     V = 128257, bf16.
Prints one JSON line with the card's name and power limit next to the times.  Inputs are seeded; before timing, the
outputs of the two arms are checked bit for bit.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess

import torch

from align_anything_b200 import _lib as L
from align_anything_b200 import ops


def _card() -> dict:
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (f.strip() for f in q.split(','))
        return {'name': name, 'power_limit': power, 'max_sm_clock': clock}
    except Exception as e:  # the times stand without it; say so
        return {'name': torch.cuda.get_device_name(), 'power_limit': f'unknown ({e})'}


def _time(fn, iters: int) -> float:
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def _alternate(arms: dict, rounds: int, iters: int) -> dict:
    for fn in arms.values():  # warm-up: module load, occupancy queries, attribute setting
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for r in range(rounds):
        order = list(arms) if r % 2 == 0 else list(reversed(arms))
        for k in order:
            times[k].append(_time(arms[k], iters))
    return {k: {'median_ms': statistics.median(v), 'min_ms': min(v), 'max_ms': max(v)} for k, v in times.items()}


def bench_k1(rounds: int, iters: int) -> dict:
    B, R, V = 32, 512, 152064
    dev = torch.device('cuda')
    gen = torch.Generator(device=dev).manual_seed(0)
    logits = (torch.randn((B * R, V), generator=gen, device=dev) * 3).to(torch.bfloat16)
    labels = torch.randint(0, V, (B * R,), generator=gen, device=dev)
    plan = ops._dense_plan(B, R, R * V, V, R, 0, R, B * R, str(dev))
    p = plan.ptrs()
    out = {k: torch.zeros(B * R, dtype=torch.bfloat16, device=dev) for k in ('off', 'on')}
    ent = torch.zeros(B * R, dtype=torch.float32, device=dev)
    st = L.stream_ptr(dev)

    def args(o):
        return (logits.data_ptr(), L.AA_BF16, V, V, labels.data_ptr(), 0, 0, plan.n_seg, plan.n_rows, p[0], p[1], p[2],
                p[3], o.data_ptr(), L.AA_BF16, None, None, None)

    arms = {'off': lambda: L.check(L.lib().aa_logprob_fwd(*args(out['off']), st)),
            'on': lambda: L.check(L.lib().aa_logprob_fwd_entropy(*args(out['on']), ent.data_ptr(), ent.numel(), st))}
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    assert torch.equal(out['off'].view(torch.int16), out['on'].view(torch.int16)), 'K1 log-probs differ'
    res = _alternate(arms, rounds, iters)
    gb = B * R * V * 2 / 1e9
    for v in res.values():
        v['read_TB_per_s'] = gb / v['median_ms']
    return {'shape': f'{B * R} rows x V={V} bf16 (C4 rollout scoring)', 'GB_read_per_launch': gb, **res,
            'overhead': res['on']['median_ms'] / res['off']['median_ms'] - 1}


def bench_k6(rounds: int, iters: int) -> dict:
    N, H, V = 16376, 4096, 128257
    dev = torch.device('cuda')
    gen = torch.Generator(device=dev).manual_seed(1)
    hidden = torch.randn((N, H), generator=gen, device=dev).to(torch.bfloat16)
    weight = (torch.randn((V, H), generator=gen, device=dev) * 0.02).to(torch.bfloat16)
    labels = torch.randint(0, V, (N,), generator=gen, device=dev)
    out = {k: torch.empty(N, dtype=torch.bfloat16, device=dev) for k in ('off', 'on')}
    ent = torch.empty(N, dtype=torch.float32, device=dev)
    part = torch.empty(4 * max(132 * 128, 16 * N), dtype=torch.float32, device=dev)
    st = L.stream_ptr(dev)

    def args(o, per_split):
        return (hidden.data_ptr(), N, H, H, weight.data_ptr(), V, H, labels.data_ptr(), o.data_ptr(), L.AA_BF16, None,
                None, part.data_ptr(), per_split * max(132 * 128, 16 * N), L.MODE_FAITHFUL, None)

    arms = {'off': lambda: L.check(L.lib().aa_linear_logprob_fwd(*args(out['off'], 3), st)),
            'on': lambda: L.check(L.lib().aa_linear_logprob_fwd_entropy(*args(out['on'], 4), ent.data_ptr(), st))}
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    assert torch.equal(out['off'].view(torch.int16), out['on'].view(torch.int16)), 'K6 log-probs differ'
    res = _alternate(arms, rounds, iters)
    for v in res.values():
        v['TFLOP_per_s'] = 2 * N * H * V / 1e12 / (v['median_ms'] / 1e3)
    return {'shape': f'{N} rows, H={H}, V={V} bf16 (C2 lm_head)', **res,
            'overhead': res['on']['median_ms'] / res['off']['median_ms'] - 1}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=11)
    ap.add_argument('--iters', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_entropy.py measures on the GPU; no CUDA device is visible')
    k1 = bench_k1(args.rounds, args.iters)
    k6 = bench_k6(args.rounds, max(2, args.iters // 4))
    print(json.dumps({'bench': 'entropy', 'card': _card(), 'rounds': args.rounds, 'K1': k1, 'K6': k6}))


if __name__ == '__main__':
    main()
