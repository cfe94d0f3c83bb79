"""The oracle port against the unmodified reference's own outputs on seeded inputs.  The inputs are rebuilt here from
their seeds; what the reference returned for them is stored in tests/golden/reference_ports*.pt (written by
tests/golden/make_golden.py, which runs the reference).  Every comparison is exact."""

import pytest
import torch

from oracle import ref_port as O

MODALITIES = ('text', 'image', 'audio')
PPO_DTYPES = ((torch.bfloat16, torch.float32), (torch.bfloat16, torch.bfloat16), (torch.float32, torch.float32))
DTYPE_NAMES = {torch.bfloat16: 'bf16', torch.float32: 'f32'}


def _same(a, b):
    assert a.dtype == b.dtype and a.shape == b.shape
    assert torch.equal(torch.nan_to_num(a.float()), torch.nan_to_num(b.float()))


def dpo_case(seed, dtype):
    """(policy logits, reference logits, ids, response lengths, pad) of one DPO case."""
    gen = torch.Generator().manual_seed(seed)
    V, L, B, pad = 211 + seed, 14 + seed, 2 + seed % 2, 0
    lens = torch.randint(2, L // 2, (2 * B,), generator=gen).tolist()
    ids = torch.randint(1, V, (2 * B, L), generator=gen)
    for i, r in enumerate(lens):
        ids[i, : L - r - 2] = pad
    if seed % 2:
        ids[0, L - 2] = pad  # interior pad
    pol = (torch.randn(2 * B, L, V, generator=gen) * 2.5).to(dtype)
    ref = (pol.float() + 0.3 * torch.randn(2 * B, L, V, generator=gen)).to(dtype)
    return pol, ref, ids, lens, pad


def ppo_cases(seed):
    """Yields (dtype, vdtype, modality, inputs) of the PPO cases of one seed; `inputs` holds what both sides consume."""
    gen = torch.Generator().manual_seed(100 + seed)
    B, W, start = 3, 17 + seed, 4
    for dtype, vdtype in PPO_DTYPES:
        for modality in MODALITIES:
            lp = (-3 * torch.rand(B, W, generator=gen)).to(dtype)
            rlp = (lp.float() + 0.2 * torch.randn(B, W, generator=gen)).to(dtype)
            mask = torch.zeros(B, W, dtype=torch.bool)
            for b in range(B):
                mask[b, 1 : start + 3 + 2 * b] = True
            reward = torch.randn(B, generator=gen)
            vals = torch.randn(B, W, generator=gen).to(vdtype)
            nlp = (lp.float() + 0.3 * torch.randn(B, W, generator=gen)).to(dtype)
            nv = (vals.float() + 0.5 * torch.randn(B, W, generator=gen)).to(vdtype)
            yield dtype, vdtype, modality, dict(lp=lp, rlp=rlp, mask=mask, reward=reward, vals=vals, nlp=nlp, nv=nv, start=start)


def layout_case():
    gen = torch.Generator().manual_seed(3)
    ids = torch.randint(0, 3, (32, 41), generator=gen)
    ids[:, :4] = 0
    return ids


@pytest.mark.parametrize('seed', range(4))
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32])
def test_dpo_port_vs_live_reference(seed, dtype, golden):
    want_all = golden('reference_ports')['dpo'][f'{DTYPE_NAMES[dtype]}_{seed}']
    pol, ref, ids, lens, pad = dpo_case(seed, dtype)
    for modality in MODALITIES:
        want = want_all[modality]
        got, grad = O.dpo_forward_backward(pol, ref, ids, lens, pad, 0.1, strip=(modality != 'audio'),
                                           skip_identical_pairs=(modality == 'audio'))
        assert set(got) >= set(want['loss'])
        for k, v in want['loss'].items():
            _same(got[k].detach(), v)
        _same(grad, want['grad'])


@pytest.mark.parametrize('seed', range(3))
def test_ppo_port_vs_live_reference(seed, golden):
    want_all = golden('reference_ports')['ppo'][seed]
    hp = O.PPO_DEFAULTS
    n = 0
    for dtype, vdtype, modality, x in ppo_cases(seed):
        want = want_all[f'{DTYPE_NAMES[dtype]}_{DTYPE_NAMES[vdtype]}_{modality}']
        s, mask = x['start'], x['mask']
        _same(O.kl_shaped_rewards(x['reward'], x['lp'], x['rlp'], mask, hp['kl_coeff'], hp['clip_range_score']), want['rewards'])
        a2, t2 = O.gae_advantages_and_returns(x['vals'], want['rewards'], mask, s, hp['gamma'], hp['gae_lambda'])
        _same(a2, want['advantages'])
        _same(t2, want['returns'])
        _same(O.actor_loss(x['nlp'][:, s:], x['lp'][:, s:], want['advantages'], mask[:, s:], hp['clip_range_ratio']),
              want['actor_loss'])
        _same(O.critic_loss(x['nv'][:, s:], x['vals'][:, s:], want['returns'], mask[:, s:], hp['clip_range_value']),
              want['critic_loss'])
        n += 1
    assert n == len(want_all) == len(PPO_DTYPES) * len(MODALITIES)


def test_layout_port_vs_live_reference(golden):
    _same(O.move_padding_left(layout_case(), 0), golden('reference_ports')['layout'])
