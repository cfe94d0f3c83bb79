"""Generate tests/golden/cost_model.pt by running the UNMODIFIED reference's cost-model trainer
(trainers/text_to_text/cost_model.py, imported through oracle/ref_shim.py) on small seeded inputs:

    AA_REFERENCE_ROOT=<checkout> python tests/golden/make_golden_cost_model.py

It has its own seeded generator and writes only cost_model.pt, so the fixtures of make_golden.py are untouched.

  * 'cases': CMTrainer.loss + backward with the engine stubbed (fixed `scores` / `end_scores` leaves) over
    B in {1, 4, 7}, fp32 and bf16 end scores, five kinds of sign lists (int harmless rates in -3..3 with 0, floats,
    bools, a mixed int / float list, and better / worse lists of different dtypes), scale_coeff in {1, 0.5} and
    regularization in {0, 0.001}.  With B >= 4 row 0 is a tie (h == l) and rows 1-2 saturate logsigmoid (|z| >= 30).
    Recorded: the loss (value and dtype), the accuracy and d loss / d end_scores.
  * 'audio_rm': the audio RMTrainer.loss (trainers/text_audio_to_text/rm.py) on the same end scores.
  * 'missing_safety_fields': the KeyError of CMTrainer.loss on a batch whose meta_info has no safety signs.
"""
from __future__ import annotations

import os
import sys
from types import SimpleNamespace

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from make_golden import save  # noqa: E402

from oracle import ref_shim  # noqa: E402

SIGN_KINDS = ('int', 'float', 'bool', 'mixed', 'int_float')
DTYPES = (('f32', torch.float32), ('bf16', torch.bfloat16))


def signs(kind, B, gen):
    """(is_better_safe, is_worse_safe) as the collator hands them over: Python lists."""
    ints = lambda: [int(v) for v in torch.randint(-3, 4, (B,), generator=gen)]
    floats = lambda: [round(float(v), 3) for v in (torch.rand(B, generator=gen) * 6 - 3)]
    bools = lambda: [bool(v) for v in torch.randint(0, 2, (B,), generator=gen)]
    if kind == 'int':
        b, w = ints(), ints()
        b[0] = 0  # a harmless rate of 0
    elif kind == 'float':
        b, w = floats(), floats()
    elif kind == 'bool':
        b, w = bools(), bools()
    elif kind == 'mixed':  # ints and floats in one list -> float32
        b, w = ints(), floats()
        b[-1] = 1.5
        w[0] = -2
    else:  # better int64, worse float32
        b, w = ints(), floats()
    return b, w


def end_scores(B, dtype, gen):
    h = torch.randn(B, generator=gen) * 3
    lo = torch.randn(B, generator=gen) * 3
    if B >= 4:
        lo[0] = h[0]  # tie
        h[1], lo[1] = 35.0, -2.0  # z = h - l saturates
        h[2], lo[2] = -4.0, 31.5
    return torch.cat([h, lo]).unsqueeze(-1).to(dtype)


class _Engine:
    """Stands in for the DeepSpeed engine: returns the fixed leaves."""

    def __init__(self, scores, end):
        self.scores, self.end = scores, end

    def __call__(self, **kw):
        return SimpleNamespace(scores=self.scores, end_scores=self.end)


def make_trainer(cls_path, scale_coeff, reg):
    ref_shim.install()
    from align_anything.utils.tools import dict_to_namedtuple

    mod, name = cls_path.rsplit('.', 1)
    cls = getattr(__import__(mod, fromlist=[name]), name)
    t = object.__new__(cls)
    t.cfgs = dict_to_namedtuple({'train_cfgs': {'regularization': reg, 'scale_coeff': scale_coeff}})
    t.scale_coeff = scale_coeff
    t.infer_batch = lambda b: {k: v for k, v in b.items() if k != 'meta_info'}
    return t


def run(cls_path, end, scale_coeff, reg, meta_info, L=3):
    n = end.size(0)
    scores = end.float().expand(n, L).unsqueeze(-1).to(end.dtype).clone().requires_grad_(True)
    leaf = end.clone().requires_grad_(True)
    t = make_trainer(cls_path, scale_coeff, reg)
    t.model = _Engine(scores, leaf)
    batch = {'input_ids': torch.zeros(n, L, dtype=torch.int64), 'attention_mask': torch.ones(n, L, dtype=torch.bool),
             'meta_info': meta_info}
    out = t.loss(batch)
    out['loss'].backward()
    return dict(loss=out['loss'].detach(), loss_dtype=out['loss'].dtype, accuracy=out['accuracy'].detach(),
                grad=leaf.grad)


CM = 'align_anything.trainers.text_to_text.cost_model.CMTrainer'
AUDIO_RM = 'align_anything.trainers.text_audio_to_text.rm.RMTrainer'


def main():
    gen = torch.Generator().manual_seed(20261016)
    cases, audio = {}, {}
    for B in (1, 4, 7):
        for dname, dtype in DTYPES:
            end = end_scores(B, dtype, gen)
            for kind in SIGN_KINDS:
                b, w = signs(kind, B, gen)
                for scale in (1, 0.5):
                    for reg in (0.0, 0.001):
                        r = run(CM, end, scale, reg, {'is_better_safe': b, 'is_worse_safe': w})
                        cases[f'B{B}_{dname}_{kind}_s{scale}_r{reg}'] = dict(
                            B=B, end_scores=end, better=b, worse=w, scale_coeff=scale, regularization=reg, **r)
            for reg in (0.0, 0.001):
                audio[f'B{B}_{dname}_r{reg}'] = dict(end_scores=end, regularization=reg,
                                                     **run(AUDIO_RM, end, 1, reg, {}))
    try:
        run(CM, end_scores(2, torch.float32, gen), 1, 0.001, {'better_response': ['a', 'b']})
        raise AssertionError('the reference accepted a batch without safety signs')
    except KeyError as e:
        missing = e.args[0]
    data = {'cases': cases, 'audio_rm': audio, 'missing_safety_fields': missing}
    paths = save('cost_model', data)
    print('cost_model', len(cases), 'cases,', sum(os.path.getsize(p) for p in paths) // 1024, 'KiB in', len(paths),
          'file(s)')


if __name__ == '__main__':
    main()
