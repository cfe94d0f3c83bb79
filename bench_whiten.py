"""bench_whiten.py -- what whitening a rollout's advantages costs next to one PPO rl_step on one H100.

    python bench_whiten.py [--rounds R] [--iters N]

At bench.py's C4 shape (Qwen2-VL-7B, V = 152064, H = 3584, 32 prompts of 512 tokens with responses of 64..512 tokens,
the text+image PPO trainer on the tail layout):
  rl_step: one rl_step of the multimodal trainer with whiten_advantages off (K4, the K1f actor node, the critic node,
     the packed metrics), after one score_rollout; CUDA events around N steps;
  whiten K = 1: ops.whiten_advantages on the rollout's one (32, 512) micro-batch, as the image / video trainers make it
     (aa_whiten_moments, aa_whiten_reduce, aa_whiten_apply); CUDA events around N back-to-back calls;
  whiten K = 32: the same 32 x 512 advantages as 32 micro-batches of one row, as the text and audio trainers make them
     with per_device_train_batch_size 1 (65 launches).
The advantages are K4's on the scored rollout, in the dtype K4 gives them.  The median of R rounds per arm.  Prints one
JSON line with the card's name and power limit next to the times.
"""
from __future__ import annotations

import argparse
import json
from types import SimpleNamespace

import torch

from align_anything_b200 import ops
from bench import CONFIGS, Engine, synth_logits
from bench_entropy import _alternate, _card


def _c4_trainer():
    """The C4 trainer and one scored rollout (bench.ppo_bench's inputs, one rank)."""
    from align_anything_b200.models.reward_model import score_model_outputs
    from align_anything_b200.trainers.text_image_to_text.ppo import PPOTrainer

    c = CONFIGS['C4']
    V, H, Bp, pad = c['V'], c['H'], c['prompts_per_rank'], c['pad']
    L = c['prompt_len'] + c['max_response']
    dev = torch.device('cuda')
    gen = torch.Generator().manual_seed(777)
    resp = torch.randint(64, c['max_response'] + 1, (Bp,), generator=gen).tolist()
    prompt = torch.randint(2, pad, (Bp, c['prompt_len']), generator=gen)
    seq = torch.full((Bp, L), pad, dtype=torch.int64)
    seq[:, : c['prompt_len']] = prompt
    for b, r in enumerate(resp):
        seq[b, c['prompt_len']: c['prompt_len'] + r] = torch.randint(2, pad, (r,), generator=gen)
    tr = PPOTrainer(None, tokenizer=SimpleNamespace(pad_token_id=pad))
    K = c['max_response'] + 1
    actor = synth_logits(Bp, K, V, dev, 31).requires_grad_(True)
    refl = synth_logits(Bp, K, V, dev, 57, like=actor)
    g2 = torch.Generator(device=dev).manual_seed(5)
    critic_h = torch.randn((Bp, L, H), generator=g2, device=dev).bfloat16().requires_grad_(True)
    rm_h = torch.randn((Bp, L, H), generator=g2, device=dev).bfloat16()
    w_c = (0.02 * torch.randn((1, H), generator=g2, device=dev)).bfloat16().requires_grad_(True)
    w_r = (0.02 * torch.randn((1, H), generator=g2, device=dev)).bfloat16()
    tr.actor_model = Engine(lambda: SimpleNamespace(logits=actor), (actor,))
    tr.actor_reference_model = Engine(lambda: SimpleNamespace(logits=refl))
    tr.reward_model = Engine(lambda: score_model_outputs(rm_h, w_r, None, 'last', False))
    tr.reward_critic_model = Engine(lambda: score_model_outputs(critic_h, w_c, None, 'last', False), (critic_h, w_c))
    moved, attn, lens = tr.postprocess_generation(prompt.to(dev), seq.to(dev))
    inference, training = tr.score_rollout({'input_ids': moved, 'attention_mask': attn}, lens)
    return tr, inference, training


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--iters', type=int, default=200)
    a = ap.parse_args()
    res = {'card': _card()}
    tr, inference, training = _c4_trainer()
    _, adv, _, _ = ops.kl_rewards_and_gae(training['reward'], training['log_probs'], training['ref_log_probs'],
                                          training['reward_values'], training['response_mask'], 0, tr.kl_coeff,
                                          tr.clip_range_score, tr.gamma, tr.gae_lambda)
    mask = training['response_mask']
    rows = [adv[b:b + 1].clone() for b in range(adv.size(0))]
    row_masks = [mask[b:b + 1] for b in range(mask.size(0))]
    res['shape'] = {'advantages': list(adv.shape), 'dtype': str(adv.dtype), 'masked_tokens': int(mask.sum())}
    res['rl_step'] = _alternate({'rl_step': lambda: tr.rl_step(inference, training)}, a.rounds, 3)
    res['whiten'] = _alternate({'K1': lambda: ops.whiten_advantages([adv], [mask]),
                                'K32': lambda: ops.whiten_advantages(rows, row_masks)}, a.rounds, a.iters)
    ops.check_status()
    step = res['rl_step']['rl_step']['median_ms']
    res['share_of_rl_step'] = {k: v['median_ms'] / step for k, v in res['whiten'].items()}
    print(json.dumps(res))


if __name__ == '__main__':
    main()
