"""Same names and signatures as the hot-path helpers of align_anything/utils/tools.py; bodies run on
the sm_90a kernels (align_anything_b200.ops)."""
from __future__ import annotations

import torch

from .. import ops

__all__ = ['gather_log_probabilities', 'masked_mean', 'move_padding_left', 'strip_pad']


def gather_log_probabilities(logits: torch.Tensor, labels: torch.LongTensor) -> torch.Tensor:
    """utils/tools.py:402-413.  (B, L, V), (B, L) -> (B, L) in the logits dtype; differentiable."""
    return ops.gather_log_probabilities(logits, labels)


def masked_mean(x: torch.Tensor, mask: torch.BoolTensor | None = None) -> torch.Tensor:
    """utils/tools.py:460-467."""
    return ops.masked_mean(x, mask).to(x.dtype if x.is_floating_point() else torch.float32)


def move_padding_left(input_tensor: torch.Tensor, padding_value: int = 0) -> torch.Tensor:
    """utils/tools.py:615-639 (dup trainers/text_image_to_text/ppo.py:56-87)."""
    return ops.move_padding_left(input_tensor, padding_value)


def strip_pad(seq: torch.Tensor, pad_token_id: int) -> torch.Tensor:
    """utils/tools.py:642 / trainers/text_to_text/dpo.py:52-54.  Data-dependent output shape, so this
    stays a (syncing) torch boolean index; the trainers here never call it -- they use
    ops.strip_pad_tail, which produces the labels the reference derives from it without a sync."""
    return seq[seq != pad_token_id]
