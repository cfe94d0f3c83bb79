"""The fused lm_head switch of the text RL trainers on one GPU; prints ONE JSON line.

    python bench_fused_rl.py [--steps K] [--warmup W] [--lm-head-chunk-rows N]

Llama-3-8B lm_head shapes (H = 4096, V = 128257, bf16); the models are stubs that hand out fixed last hidden states, so
what is measured is everything from the last hidden states on:
  * `ppo`: text PPOTrainer.score_rollout (reward / critic stubs, actor and reference log-probs of every position) plus
    rl_step (K4, the actor node and its backward down to d(hidden) and d(weight), the critic loss, the packed metrics and
    the step's one host read), B = 8, L = 2048, a 512-token prompt;
  * `grpo`: GRPOTrainer.step_from_rollout, 2 prompts x 8 generations, L = 2048, 1536 completion tokens.
Two arms each: `materialised` -- the stub returns `F.linear(hidden, weight)` logits and the trainer runs today's default
path (K1 / K1f / the GRPO kernels on the (B, L, V) tile); `fused` -- `fused_lm_head = True`, no logits tile.  Per arm:
median CUDA-event milliseconds of a whole step after warm-up, and the peak of torch.cuda.max_memory_allocated over the
arm's steps (reset before the arm; the resident inputs -- hidden states, weights, ids -- are counted in both arms).
`tiles_saved` = (materialised peak - fused peak) / the bytes of one (B, L, V) bf16 tile.  `--lm-head-chunk-rows` sets
the trainers' `lm_head_chunk_rows` in the fused arm (default None: about 2 GB of d(logits) per backward chunk).  The
card's name, power limit and maximum SM clock are read (read-only) with `nvidia-smi --query-gpu` in the same run.
Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
from types import SimpleNamespace

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

H, V = 4096, 128257
DEV = 'cuda'


def card() -> dict:
    q = 'name,power.limit,clocks.max.sm'
    try:
        r = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader,nounits', '-i', '0'],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(',')]
        return {'name': name, 'power_limit_w': float(power), 'max_sm_clock_mhz': float(clock)}
    except Exception as e:  # the measurement still stands; say why the card is unknown
        return {'name': torch.cuda.get_device_name(0), 'error': str(e)}


def timed(fn, steps: int, warmup: int) -> float:
    """Median milliseconds of `fn` over `steps` runs after `warmup` runs (CUDA events around each run)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


class LM:
    """A causal LM reduced to its last hidden states and lm_head: logits = F.linear(hidden, weight) on the default path,
    the hidden states when the fused path asks for them."""

    def __init__(self, hidden, weight):
        self.hidden, self.weight = hidden, weight
        self.optimizer = SimpleNamespace(param_groups=[{'lr': 1e-6}])

    def __call__(self, output_hidden_states=False, logits_to_keep=0, **kw):
        if output_hidden_states:
            return SimpleNamespace(hidden_states=(self.hidden,), logits=None)
        return SimpleNamespace(logits=F.linear(self.hidden, self.weight))

    def get_output_embeddings(self):
        return SimpleNamespace(weight=self.weight)

    def backward(self, loss):
        loss.backward()

    def step(self):
        self.hidden.grad = None
        self.weight.grad = None

    def zero_grad(self):
        pass


class Stub:
    def __init__(self, fn):
        self.fn = fn
        self.optimizer = SimpleNamespace(param_groups=[{'lr': 1e-6}])

    def __call__(self, **kw):
        return self.fn()

    def backward(self, loss):
        loss.backward()

    def step(self):
        pass


class Phased:
    """The actor engine: the rollout model while scoring, the trained model (hidden states and weight with a gradient)
    in rl_step."""

    def __init__(self, roll, train):
        self.roll, self.train_lm, self.phase = roll, train, 'rollout'
        self.optimizer = SimpleNamespace(param_groups=[{'lr': 1e-6}])

    def _cur(self):
        return self.roll if self.phase == 'rollout' else self.train_lm

    def __call__(self, **kw):
        return self._cur()(**kw)

    def get_output_embeddings(self):
        return self._cur().get_output_embeddings()

    def backward(self, loss):
        loss.backward()

    def step(self):
        self.train_lm.step()


def measure(step, steps, warmup):
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    resident = torch.cuda.memory_allocated()
    ms = timed(step, steps, warmup)
    torch.cuda.synchronize()
    return {'ms': round(ms, 2), 'peak_gb': round(torch.cuda.max_memory_allocated() / 1e9, 3),
            'resident_gb': round(resident / 1e9, 3)}


def bench_ppo(steps, warmup, chunk_rows):
    from align_anything_b200.models.reward_model import ScoreModelOutput
    from align_anything_b200.trainers.text_to_text.ppo import PPOTrainer

    gen = torch.Generator(device=DEV).manual_seed(0)
    B, L, P = 8, 2048, 512
    ids = torch.randint(2, V, (B, L), generator=gen, device=DEV)
    for b in range(B):  # left-padded prompts, right-padded responses
        ids[b, :16 * b] = 0
        ids[b, L - 97 * b:] = 0
    batch = {'input_ids': ids, 'attention_mask': ids != 0}
    w = (torch.randn(V, H, generator=gen, device=DEV) * (2.5 / H ** 0.5)).bfloat16()
    w_ref = (w.float() + 0.01 * torch.randn(V, H, generator=gen, device=DEV)).bfloat16()
    hid_roll, hid_ref, hid_new = (torch.randn(B, L, H, generator=gen, device=DEV).bfloat16() for _ in range(3))
    h_new, w_new = hid_new.requires_grad_(True), w.clone().requires_grad_(True)
    reward = torch.randn(B, 1, device=DEV)
    critic = torch.randn(B, L, 1, device=DEV).requires_grad_(True)
    actor = Phased(LM(hid_roll, w), LM(h_new, w_new))
    out = {'shape': {'B': B, 'L': L, 'prompt': P, 'H': H, 'V': V, 'dtype': 'bf16'},
           'tile_gb': round(B * L * V * 2 / 1e9, 3)}
    for fused in (False, True):
        tr = PPOTrainer(None, actor, LM(hid_ref, w_ref), Stub(lambda: ScoreModelOutput(end_scores=reward)),
                        Stub(lambda: ScoreModelOutput(scores=critic)), SimpleNamespace(pad_token_id=0))
        tr.fused_lm_head, tr.lm_head_chunk_rows = fused, chunk_rows

        def step():
            actor.phase = 'rollout'
            inference, training = tr.score_rollout(batch, P)
            actor.phase = 'train'
            critic.grad = None
            tr.rl_step(inference, training)

        out['fused' if fused else 'materialised'] = measure(step, steps, warmup)
    return out


def bench_grpo(steps, warmup, chunk_rows):
    from align_anything_b200.trainers.text_to_text.grpo import GRPOTrainer

    gen = torch.Generator(device=DEV).manual_seed(1)
    prompts, G, L, K = 2, 8, 2048, 1536
    B = prompts * G
    seq = torch.randint(2, V, (B, L), generator=gen, device=DEV)
    for b in range(0, B, 3):  # every third completion ends at an eos and is padded after it
        seq[b, L - K + 100 * b + 7] = 1
        seq[b, L - K + 100 * b + 8:] = 0
    w = (torch.randn(V, H, generator=gen, device=DEV) * (2.5 / H ** 0.5)).bfloat16()
    w_ref = (w.float() + 0.01 * torch.randn(V, H, generator=gen, device=DEV)).bfloat16()
    hid, hid_ref = (torch.randn(B, L, H, generator=gen, device=DEV).bfloat16() for _ in range(2))
    h, wt = hid.requires_grad_(True), w.clone().requires_grad_(True)
    rewards = torch.randn(B, generator=gen, device=DEV)
    out = {'shape': {'prompts': prompts, 'generations': G, 'L': L, 'completion': K, 'H': H, 'V': V, 'dtype': 'bf16'},
           'tile_gb': round(B * L * V * 2 / 1e9, 3)}
    for fused in (False, True):
        tr = GRPOTrainer(None, LM(h, wt), LM(hid_ref, w_ref), SimpleNamespace(pad_token_id=0, eos_token_id=1),
                         beta=0.04, num_generations=G)
        tr.fused_lm_head, tr.lm_head_chunk_rows = fused, chunk_rows
        out['fused' if fused else 'materialised'] = measure(lambda: tr.step_from_rollout(seq, L - K, rewards), steps,
                                                            warmup)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--lm-head-chunk-rows', type=int, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_fused_rl.py needs a CUDA device')
    torch.cuda.set_device(0)
    res = {'bench': 'fused_rl', 'card': card(), 'lm_head_chunk_rows': a.lm_head_chunk_rows}
    for name, fn in (('ppo', bench_ppo), ('grpo', bench_grpo)):
        r = fn(a.steps, a.warmup, a.lm_head_chunk_rows)
        r['tiles_saved'] = round((r['materialised']['peak_gb'] - r['fused']['peak_gb']) / r['tile_gb'], 2)
        r['speedup'] = round(r['materialised']['ms'] / r['fused']['ms'], 2)
        res[name] = r
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
