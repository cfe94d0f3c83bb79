"""align_anything_b200 -- the RLHF loss hot path of PKU-Alignment/align-anything (per-token
log-prob extraction, DPO pairwise loss, PPO rollout scoring) as hand-written sm_90a CUDA behind a
C ABI (include/aa_b200.h), with a Python host layer that mirrors the reference's own names:

    align_anything_b200.utils.tools            <-> align_anything/utils/tools.py
    align_anything_b200.utils.multi_process    <-> align_anything/utils/multi_process.py
    align_anything_b200.models.reward_model    <-> align_anything/models/reward_model.py (+ score heads)
    align_anything_b200.trainers.<modality>.{dpo,ppo}  <-> align_anything/trainers/<modality>/{dpo,ppo}.py
    align_anything_b200.patch.install()        swaps the bodies inside an importable `align_anything`

There is no CPU fallback: the compute functions raise on non-CUDA tensors and on a missing library.
"""
__version__ = '0.1.0'

from . import _lib  # noqa: F401  (does not load the .so until first use)
