"""The fused lm_head cross-entropy of SFT on one GPU; prints ONE JSON line.

    python bench_fused_sft.py [--steps K] [--warmup W] [--rounds R]

Llama-3-8B lm_head shapes (H = 4096, V = 128257, bf16); the model is a stub that hands out fixed last hidden states, so
what is measured is the loss forward + backward from the last hidden states to d(hidden) and d(weight):
  * `S1`: B = 8, L = 2048, a 512-token masked prompt and seeded right padding;
  * `S2`: B = 1, L = 32768, a 4096-token masked prompt.
Three arms:
  * `tile`: today's SupervisedTrainer.loss on `F.linear(hidden, weight)` logits (K1f on the (B, L, V) tile, ATen's
    linear backward) -- 3 GEMM passes over every position;
  * `composed`: ops.linear_token_log_probs over the valid rows (f32 log-probs) and their mean -- K6, then K6b, d(hidden)
    and d(weight) in the backward: 4 GEMM passes over the valid rows and no new kernel;
  * `fused`: SupervisedTrainer.loss with `fused_lm_head = True` (ops.causal_lm_loss_from_hidden: K6s, K1b, d(hidden),
    d(weight) in the forward) -- 3 GEMM passes over the valid rows.
Per arm: the median CUDA-event milliseconds of loss + backward after warm-up (the valid-row index and its host read are
inside the window where the arm needs them), the peak of torch.cuda.max_memory_allocated (reset before the arm; the
resident hidden states and weight are counted in every arm), TFLOP/s over the GEMM passes the arm performs, and the
largest relative difference of the loss, d(hidden) and d(weight) from `tile` (max |a - b| / max |b|).  `composed` and
`fused` are timed alternately for `--rounds` rounds in the same process: `spread_ms` is the range of their per-round
medians.  The card's name, power limit and maximum SM clock are read (read-only) with `nvidia-smi --query-gpu` in the
same run.  Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_fused_rl import LM, card, timed  # noqa: E402

H, V = 4096, 128257
DEV = 'cuda'
IGN = -100


def shape(name):
    gen = torch.Generator(device=DEV).manual_seed(3)
    if name == 'S1':
        B, L, P = 8, 2048, 512
        pads = torch.randint(0, 512, (B,), generator=gen, device=DEV).tolist()
    else:
        B, L, P = 1, 32768, 4096
        pads = [0]
    labels = torch.randint(0, V, (B, L), generator=gen, device=DEV)
    labels[:, :P] = IGN
    for b, p in enumerate(pads):
        if p:
            labels[b, L - p:] = IGN
    hidden = torch.randn(B, L, H, generator=gen, device=DEV).bfloat16().requires_grad_(True)
    weight = (torch.randn(V, H, generator=gen, device=DEV) * (2.5 / H ** 0.5)).bfloat16().requires_grad_(True)
    return {'B': B, 'L': L, 'prompt': P, 'pads': pads}, hidden, weight, labels


def make_steps(hidden, weight, labels):
    from align_anything_b200 import ops
    from align_anything_b200.trainers.text_to_text.sft import SupervisedTrainer

    lm = LM(hidden, weight)
    batch = {'input_ids': labels.clamp(min=0), 'labels': labels}
    trainers = {}
    for fused in (False, True):
        tr = SupervisedTrainer(None, lm)
        tr.fused_lm_head = fused
        trainers[fused] = tr

    def clear():
        hidden.grad = weight.grad = None

    def tile():
        clear()
        loss = trainers[False].loss(batch)['loss']
        loss.backward()
        return loss

    def composed():
        clear()
        idx, n = ops.causal_lm_valid_rows(labels, IGN)
        shift = torch.full_like(labels, IGN)
        shift[:, :-1] = labels[:, 1:]
        rows = hidden.reshape(-1, H).index_select(0, idx)
        lp = ops.linear_token_log_probs(rows, weight, shift.view(-1).index_select(0, idx), mode='f32')
        loss = -lp.sum() / n
        loss.backward()
        return loss

    def fused():
        clear()
        loss = trainers[True].loss(batch)['loss']
        loss.backward()
        return loss

    return {'tile': tile, 'composed': composed, 'fused': fused}


def rel(a, b):
    return float((a.float() - b.float()).abs().max() / b.float().abs().max().clamp(min=1e-30))


def bench(name, steps, warmup, rounds):
    info, hidden, weight, labels = shape(name)
    from align_anything_b200 import ops

    _, N = ops.causal_lm_valid_rows(labels, IGN)
    B, L = info['B'], info['L']
    gemm = 2.0 * H * V  # flops of one GEMM pass per row
    passes = {'tile': 3 * B * L * gemm, 'composed': 4 * N * gemm, 'fused': 3 * N * gemm}
    fns = make_steps(hidden, weight, labels)
    out = {'shape': {**info, 'valid_rows': N, 'H': H, 'V': V, 'dtype': 'bf16'}, 'tile_gb': round(B * L * V * 2 / 1e9, 3)}
    ref = None
    for arm in ('tile', 'composed', 'fused'):  # outputs against `tile`, then the peak memory of one warm step per arm
        loss = fns[arm]()
        torch.cuda.synchronize()
        got = (loss.detach().float(), hidden.grad.clone(), weight.grad.clone())
        if ref is None:
            ref = got
        out[arm] = {'loss_rel': rel(got[0], ref[0]), 'dhidden_rel': rel(got[1], ref[1]), 'dweight_rel': rel(got[2], ref[2])}
        del got, loss
        hidden.grad = weight.grad = None
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        fns[arm]()
        torch.cuda.synchronize()
        hidden.grad = weight.grad = None
        out[arm]['peak_gb'] = round(torch.cuda.max_memory_allocated() / 1e9, 3)
    del ref
    ops.check_status()
    times = {arm: [] for arm in fns}
    times['tile'].append(timed(fns['tile'], steps, warmup))
    for _ in range(rounds):  # composed and fused alternately
        for arm in ('composed', 'fused'):
            times[arm].append(timed(fns[arm], steps, warmup))
    for arm, ts in times.items():
        ms = statistics.median(ts)
        out[arm].update({'ms': round(ms, 2), 'tflops': round(passes[arm] / ms / 1e9, 1)})
        if arm != 'tile':
            out[arm]['spread_ms'] = [round(min(ts), 2), round(max(ts), 2)]
    out['fused_vs_composed'] = round(out['composed']['ms'] / out['fused']['ms'], 3)
    out['tiles_saved'] = round((out['tile']['peak_gb'] - out['fused']['peak_gb']) / out['tile_gb'], 2)
    hidden.grad = weight.grad = None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--rounds', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_fused_sft.py needs a CUDA device')
    torch.cuda.set_device(0)
    res = {'bench': 'fused_sft', 'card': card()}
    for name in ('S1', 'S2'):
        res[name] = bench(name, a.steps, a.warmup, a.rounds)
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
