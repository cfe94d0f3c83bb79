"""Generate tests/golden/multi_ppo*.pt by running the UNMODIFIED reference's Multi-PPO trainer
(trainers/text_to_text/multi_ppo.py, imported through oracle/ref_shim.py) on small seeded inputs:

    AA_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_multi_ppo.py

It has its own seeded generator and writes only multi_ppo*.pt, so the fixtures of make_golden.py are untouched.

  * 'estimators': add_kl_divergence_regularization + get_advantages_and_returns for all five estimators, bf16 and
    fp32 log-probs, n in {2, 3, 4} with W % n != 0, gamma 1.0 and 0.99, left and right pads and an interior hole,
    and (group_norm) a group of equal non-zero rewards.
  * 'rl_step': rollout scoring + one rl_step per estimator with the engines stubbed (fixed logits / scores), with the
    gradients of the actor logits and of the critic scores.
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from make_golden import save  # noqa: E402

from oracle import ref_shim  # noqa: E402

ESTIMATORS = ('gae', 'reinforce', 'rloo', 'reinforce_baseline', 'group_norm')
HP = dict(kl_coeff=0.02, clip_range_ratio=0.2, clip_range_score=50.0, clip_range_value=5.0, gae_lambda=0.95)


def make_trainer(estimator, n, gamma):
    """object.__new__ the reference's Multi-PPO trainer with only the attributes the loss path reads."""
    ref_shim.install()
    from align_anything.trainers.text_to_text.multi_ppo import PPOTrainer

    p = object.__new__(PPOTrainer)
    for k, v in HP.items():
        setattr(p, k, v)
    p.gamma = gamma
    p.advantage_estimator = estimator
    p.n_samples_per_prompt = n
    return p


def golden_estimators(gen):
    out = {}
    B, W = 12, 23  # B * W divisible by 2, 3 and 4; W is not
    start = 7
    mask = torch.zeros(B, W, dtype=torch.bool)
    for b in range(B):
        left = int(torch.randint(0, 3, (1,), generator=gen))
        resp = int(torch.randint(3, W - start + 1, (1,), generator=gen))
        mask[b, left:start + resp] = True  # left pads in the prompt, right pads after the response
    mask[0] = False
    mask[0, 1:W - 1] = True  # row 0: one left and one right pad, room for the constant group below
    mask[3, start + 2] = False  # an interior hole
    for dname, dtype in (('bf16', torch.bfloat16), ('f32', torch.float32)):
        lp = (-3 * torch.rand(B, W, generator=gen)).to(dtype)
        rlp = (lp.float() + 0.2 * torch.randn(B, W, generator=gen)).to(dtype)
        reward = torch.randn(B, generator=gen)
        vals = torch.randn(B, W, generator=gen)
        cases = {}
        out[dname] = dict(start=start, mask=mask, log_probs=lp, ref_log_probs=rlp, reward=reward, values=vals,
                          cases=cases)
        for n in (2, 3, 4):
            for gamma in (1.0, 0.99):
                for est in ESTIMATORS:
                    p = make_trainer(est, n, gamma)
                    rew = p.add_kl_divergence_regularization(reward, lp, rlp, mask)
                    if est == 'group_norm':  # a constant non-zero group inside the attended span of row 0
                        g0 = (start + 1 + n - 1) // n * n
                        rew = rew.clone()
                        rew.view(-1)[g0:g0 + n] = 0.5
                    adv, ret = p.get_advantages_and_returns(vals, rew, mask, start)
                    cases[f'{est}_n{n}_g{gamma}'] = dict(estimator=est, n=n, gamma=gamma, rewards=rew,
                                                         advantages=adv.detach(), returns=ret.detach())
    return out


def golden_rl_step(gen):
    t = ref_shim.tools()
    out = {}
    n, prompts = 3, 2
    B, L, V = n * prompts, 18, 131
    pad = V - 1
    prompt_len = 7
    ids = torch.randint(2, V - 1, (B, L), generator=gen)
    ids[0, :2] = pad
    ids[3, :1] = pad
    ids[0, 15:] = pad  # right pads after eos
    ids[4, 12:] = pad
    attn = ids != pad
    start = prompt_len - 1
    for dname, dtype in (('bf16', torch.bfloat16), ('f32', torch.float32)):
        actor = (torch.randn(B, L, V, generator=gen) * 2.5).to(dtype)
        refl = (actor.float() + 0.3 * torch.randn(B, L, V, generator=gen)).to(dtype)
        new_actor = (actor.float() + 0.2 * torch.randn(B, L, V, generator=gen)).to(dtype)
        end_scores = torch.randn(B, 1, generator=gen)
        critic = torch.randn(B, L, 1, generator=gen)
        new_critic = critic + 0.4 * torch.randn(B, L, 1, generator=gen)
        case = dict(input_ids=ids, attention_mask=attn, start=start, n=n, actor_logits=actor, ref_logits=refl,
                    new_actor_logits=new_actor, end_scores=end_scores, critic_scores=critic,
                    new_critic_scores=new_critic)
        lp = t.gather_log_probabilities(actor[:, :-1], ids[:, 1:])
        rlp = t.gather_log_probabilities(refl[:, :-1], ids[:, 1:])
        reward = end_scores.squeeze(-1)
        old_vals = critic.squeeze(-1)[:, :-1]
        seq_mask = attn[:, 1:]
        case.update(log_probs=lp, ref_log_probs=rlp)
        for est in ESTIMATORS:
            # multi_ppo.py:330-391 with the engines stubbed
            p = make_trainer(est, n, 1.0)
            rew = p.add_kl_divergence_regularization(reward, lp, rlp, seq_mask)
            adv, ret = p.get_advantages_and_returns(old_vals, rew, seq_mask, start)
            leaf = new_actor.clone().requires_grad_(True)
            nlp = t.gather_log_probabilities(leaf[:, :-1], ids[:, 1:])
            al = p.actor_loss_fn(nlp[:, start:], lp[:, start:], adv, seq_mask[:, start:])
            al.backward()
            cleaf = new_critic.clone().requires_grad_(True)
            nv = cleaf.squeeze(-1)[:, :-1]
            cl = p.critic_loss_fn(nv[:, start:], old_vals[:, start:], ret, seq_mask[:, start:])
            cl.backward()
            m = seq_mask[:, start:]
            metrics = {
                'actor_loss': al.detach(), 'reward_critic_loss': cl.detach(), 'reward': reward.mean(),
                'reward_with_kl_penalty': (rew[:, start:] * m).sum(-1).mean(),
                'reward_advantage': t.masked_mean(adv, m), 'reward_return': t.masked_mean(ret, m),
                'reward_value': t.masked_mean(nv[:, start:], m).detach(),
                'kl_divergence': ((lp - rlp)[:, start:] * m).sum(-1).mean(),
                'mean_generated_length': m.sum(-1).float().mean(), 'max_generated_length': m.sum(-1).float().max(),
            }
            case[est] = dict(old_rewards=rew, advantages=adv.detach(), returns=ret.detach(), metrics=metrics,
                             grad_actor_logits=leaf.grad, grad_critic_scores=cleaf.grad)
        out[dname] = case
    return out


def main():
    gen = torch.Generator().manual_seed(20261015)
    data = {'estimators': golden_estimators(gen), 'rl_step': golden_rl_step(gen)}
    paths = save('multi_ppo', data)
    print('multi_ppo', sum(os.path.getsize(p) for p in paths) // 1024, 'KiB in', len(paths), 'file(s)')


if __name__ == '__main__':
    main()
