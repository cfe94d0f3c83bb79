"""Cost-model (Safe RLHF) training-step tail on one GPU; prints ONE JSON line.

    python bench_cost_model.py [--steps K] [--warmup W]

  * the card: name, power limit and maximum SM clock, read (read-only) with `nvidia-smi --query-gpu` in the same run;
  * `step_tail`: what CMTrainer.train_step runs after the backbone, with LLaVA-1.5-7B shapes (H = 4096, the 'last'
    end position, fp32 scores), 4 pairs per device (the per_device_train_batch_size of
    configs/train/text_image_to_text/cost_model.yaml), L = 2048, bf16 hidden states that require a gradient:
      - `grafted`: K3 score head forward, the cost loss (one launch), K3 backward to the hidden states and the
        weight, the packed metrics with the status lane, ONE host read;
      - `eager`: the reference's ops on ATen CUDA for the same tail (score head, CMTrainer.loss's arithmetic,
        autograd, `loss.item()` and `accuracy.item()`; the two all-reduces are no-ops on one process);
  * `loss_node`: the loss with its backward alone, on (2B, 1) fp32 end scores -- aa_cost_pair_loss against the
    reference's ops.
CUDA events, warm-up, median of the timed repeats.  There is no CPU path: without a GPU the script fails.  Nothing is
written to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from bench_multi_ppo import card, timed  # noqa: E402

PAIRS, L, H = 4, 2048, 4096
SCALE, REG = 1, 0.001


def _signs(gen):
    """Harmless rates times -1, as the SafeRLHF_V_Cost template stores them (ints)."""
    return ([int(v) for v in torch.randint(-3, 4, (PAIRS,), generator=gen)],
            [int(v) for v in torch.randint(-3, 4, (PAIRS,), generator=gen)])


class _Engine:
    optimizer = SimpleNamespace(param_groups=[{'lr': 3e-5}])

    def __init__(self, fn):
        self.fn = fn

    def __call__(self, **kw):
        return self.fn()

    def backward(self, loss):
        loss.backward()

    def step(self):
        pass


def bench_step_tail(steps, warmup):
    import cost_model_port as P

    from align_anything_b200.models.reward_model import score_model_outputs
    from align_anything_b200.trainers.text_to_text.cost_model import CMTrainer
    from oracle import ref_port as O

    gen = torch.Generator().manual_seed(0)
    dev = 'cuda'
    hidden = torch.randn(2 * PAIRS, L, H, generator=gen).bfloat16().to(dev).requires_grad_(True)
    weight = (0.02 * torch.randn(1, H, generator=gen)).bfloat16().to(dev).requires_grad_(True)
    better, worse = _signs(gen)
    batch = {'input_ids': torch.zeros(2 * PAIRS, L, dtype=torch.int64, device=dev),
             'attention_mask': torch.ones(2 * PAIRS, L, dtype=torch.bool, device=dev),
             'meta_info': {'is_better_safe': better, 'is_worse_safe': worse}}
    tr = CMTrainer(SimpleNamespace(train_cfgs=SimpleNamespace(scale_coeff=SCALE, regularization=REG)),
                   _Engine(lambda: score_model_outputs(hidden, weight, None, 'last', True)))

    def grafted():
        hidden.grad = weight.grad = None
        tr.train_step(batch)

    def eager():
        hidden.grad = weight.grad = None
        so = O.score_head(hidden, weight, None, 'last', True)
        res = P.cm_loss(so['end_scores'], better, worse, SCALE, REG)
        res['loss'].backward()
        res['loss'].item()
        res['accuracy'].item()

    t_g = timed(grafted, steps, warmup)
    t_e = timed(eager, steps, warmup)
    return {'shape': {'pairs': PAIRS, 'L': L, 'H': H, 'hidden': 'bf16', 'end_mode': 'last'},
            'grafted_us': round(t_g * 1e3, 1), 'eager_us': round(t_e * 1e3, 1), 'speedup': round(t_e / t_g, 2)}


def bench_loss_node(steps, warmup):
    import cost_model_port as P

    from align_anything_b200 import ops

    gen = torch.Generator().manual_seed(1)
    end = torch.randn(2 * PAIRS, 1, generator=gen).to('cuda').requires_grad_(True)
    better, worse = _signs(gen)

    def ours():
        end.grad = None
        ops.cost_pair_loss(end, better, worse, SCALE, REG)['loss'].backward()

    def eager():
        end.grad = None
        P.cm_loss(end, better, worse, SCALE, REG)['loss'].backward()

    t_o = timed(ours, max(steps, 50), warmup)
    t_e = timed(eager, max(steps, 50), warmup)
    return {'ours_us': round(t_o * 1e3, 1), 'eager_us': round(t_e * 1e3, 1), 'speedup': round(t_e / t_o, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_cost_model.py measures on a CUDA device and found none')
    torch.cuda.set_device(0)
    res = {'bench': 'cost_model', 'card': card(), 'step_tail': bench_step_tail(a.steps, a.warmup),
           'loss_node': bench_loss_node(a.steps, a.warmup)}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
