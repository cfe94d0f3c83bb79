"""Multi-PPO measurements on one GPU; prints ONE JSON line.

    python bench_multi_ppo.py [--steps K] [--warmup W]

  * the card: name, power limit and maximum SM clock, read (read-only) with `nvidia-smi --query-gpu` in the same run;
  * `prep`: advantage / return preparation per estimator -- ours (K4 + K4r; 'gae' is K4 alone) against the
    reference's arithmetic on ATen CUDA (the KL-shaped rewards + get_advantages_and_returns / cumulative_returns
    loop) -- for B = 32 (8 prompts x 4 samples), L = 2048, a 512-token prompt, bf16 log-probs, fp32 values.
    CUDA events, warm-up, median of the timed repeats, in microseconds;
  * `rl_step`: the whole grafted Multi-PPO rl_step (K4 [+ K4r], the single-pass actor node over resident bf16 logits,
    the critic loss, the packed metrics) with Llama-3-8B shapes (V = 128257), B = 8 (2 prompts x 4), L = 2048, engines
    stubbed: tokens (B * L) per second, 'reinforce' against 'gae'.
Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

ESTIMATORS = ('gae', 'reinforce', 'rloo', 'reinforce_baseline', 'group_norm')


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


def rollout_mask(B, W, start, gen):
    mask = torch.zeros(B, W, dtype=torch.bool)
    for b in range(B):
        left = int(torch.randint(0, 64, (1,), generator=gen))
        resp = int(torch.randint(W // 4, W - start + 1, (1,), generator=gen))
        mask[b, left:start + resp] = True
    return mask


def bench_prep(steps, warmup):
    import multi_ppo_port as P

    from align_anything_b200 import ops
    from oracle import ref_port as O

    gen = torch.Generator().manual_seed(0)
    B, L, prompt = 32, 2048, 512
    W, start, n = L - 1, prompt - 1, 4
    dev = 'cuda'
    lp = (-3 * torch.rand(B, W, generator=gen)).bfloat16().to(dev)
    rlp = (lp.float().cpu() + 0.2 * torch.randn(B, W, generator=gen)).bfloat16().to(dev)
    reward = torch.randn(B, generator=gen).to(dev)
    values = torch.randn(B, W, generator=gen).to(dev)
    mask = rollout_mask(B, W, start, gen).to(dev)
    hp = O.PPO_DEFAULTS
    out = {}
    for est in ESTIMATORS:
        def ours():
            rew, adv, ret, rs = ops.kl_rewards_and_gae(reward, lp, rlp, values, mask, start, hp['kl_coeff'],
                                                       hp['clip_range_score'], 1.0, hp['gae_lambda'])
            if est != 'gae':
                ops.estimator_returns(rew, mask, start, est, n, 1.0, row_stats=rs)

        def eager():
            with torch.no_grad():
                rew = O.kl_shaped_rewards(reward, lp, rlp, mask, hp['kl_coeff'], hp['clip_range_score'])
                P.advantages_and_returns(values, rew, mask, start, est, n, 1.0, hp['gae_lambda'])

        t_ours = timed(ours, max(steps, 20), warmup)
        t_eager = timed(eager, steps, min(warmup, 2))
        out[est] = {'ours_us': round(t_ours * 1e3, 1), 'eager_us': round(t_eager * 1e3, 1),
                    'speedup': round(t_eager / t_ours, 1)}
    return {'shape': {'B': B, 'L': L, 'prompt': prompt, 'n_samples_per_prompt': n}, **out}


class _Engine:
    def __init__(self, fn):
        self.fn = fn
        self.optimizer = SimpleNamespace(param_groups=[{'lr': 1e-6}])

    def __call__(self, **kw):
        return self.fn()

    def backward(self, loss):
        loss.backward()

    def step(self):
        pass


def bench_rl_step(steps, warmup):
    from align_anything_b200.models.reward_model import ScoreModelOutput
    from align_anything_b200.trainers.text_to_text.multi_ppo import PPOTrainer

    gen = torch.Generator().manual_seed(1)
    B, L, V, prompt, n = 8, 2048, 128257, 512, 4
    dev = 'cuda'
    ids = torch.randint(2, V - 1, (B, L), generator=gen).to(dev)
    attn = torch.ones(B, L, dtype=torch.bool, device=dev)
    for b in range(B):
        attn[b, L - 1 - 97 * b:] = False
    logits = torch.empty(B, L, V, dtype=torch.bfloat16, device=dev).normal_(0.0, 2.5).requires_grad_(True)
    scores = torch.randn(B, L, 1, device=dev).requires_grad_(True)
    start = prompt - 1
    W = L - 1
    training = {'prompt_idx': start,
                'log_probs': (-3 * torch.rand(B, W, device=dev)).bfloat16(),
                'ref_log_probs': (-3 * torch.rand(B, W, device=dev)).bfloat16(),
                'reward': torch.randn(B, device=dev), 'reward_values': torch.randn(B, W, device=dev),
                'action_mask': attn[:, 1:]}
    inference = {'input_ids': ids, 'attention_mask': attn}
    actor = _Engine(lambda: SimpleNamespace(logits=logits))
    critic = _Engine(lambda: ScoreModelOutput(scores=scores))
    out = {'shape': {'B': B, 'L': L, 'V': V, 'prompt': prompt, 'dtype': 'bf16'}}
    for est in ('reinforce', 'gae'):
        tr = PPOTrainer(None, actor, None, None, critic, SimpleNamespace(pad_token_id=0), advantage_estimator=est,
                        n_samples_per_prompt=n)

        def step():
            logits.grad = None
            scores.grad = None
            tr.rl_step(inference, training)

        ms = timed(step, steps, warmup)
        out[est] = {'ms': round(ms, 3), 'tokens_per_s': round(B * L / (ms * 1e-3))}
    del logits
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = {'bench': 'multi_ppo', 'card': card(), 'prep': bench_prep(a.steps, a.warmup),
           'rl_step': bench_rl_step(a.steps, a.warmup)}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
