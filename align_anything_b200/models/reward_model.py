"""The scalar-head tail of the reference's reward / critic models on the sm_90a kernels (K3).

`ScoreModelOutput` has the fields of align_anything/models/reward_model.py:22-32.  The backbones
(HF transformers) are untouched; only what follows `outputs.hidden_states[-1]` is replaced:

    models/llama.py:62-101, opt.py, qwen2_audio.py:75-110 -> score_model_outputs(..., end_mode='mask')
    models/llava.py:62-76                                 -> end_mode='last'
    models/qwen2_vl.py:58-74                              -> end_mode='last', upcast_scores=False
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

from .. import ops

__all__ = ['ScoreModelOutput', 'score_model_outputs', 'B200ScoreHeadMixin']


@dataclass
class ScoreModelOutput:
    """Field-compatible with align_anything/models/reward_model.py:22-32."""

    scores: torch.Tensor | None = None  # (B, L, 1)
    clipped_scores: torch.Tensor | None = None
    end_scores: torch.Tensor | None = None  # (B, 1)
    last_hidden_state: torch.Tensor | None = None  # (B, L, H)
    clipped_states: torch.Tensor | None = None
    end_last_hidden_state: torch.Tensor | None = None  # (B, H)
    end_index: torch.Tensor | None = None  # (B,)


def score_model_outputs(last_hidden_state: torch.Tensor, score_head_weight: torch.Tensor,
                        attention_mask: torch.Tensor | None, end_mode: str = 'mask', upcast_scores: bool = True,
                        mode: str | None = None) -> ScoreModelOutput:
    """scores = score_head(last_hidden)[.float()], end_index = last attended position (or the -1
    placeholder), end_scores, end_last_hidden_state -- two launches, no host sync."""
    B, seq, _ = last_hidden_state.shape
    scores = ops.score_head(last_hidden_state, score_head_weight, upcast=upcast_scores, mode=mode)  # (B, L)
    if end_mode == 'mask':
        if attention_mask is None:
            if B > 1:
                raise ValueError("'attention_mask' is required when batch size > 1.")  # models/llama.py:66-68
            attention_mask = torch.ones((B, seq), dtype=torch.bool, device=last_hidden_state.device)
        end_index, end_scores, end_hidden = ops.score_end(scores, attention_mask, last_hidden_state)
        if scores.requires_grad:  # reward-model training: keep end_scores (and the end hidden state) in the graph
            end_scores = scores.gather(1, end_index.unsqueeze(1)).squeeze(1).float()
            pick = end_index.view(B, 1, 1).expand(-1, -1, last_hidden_state.size(-1))
            end_hidden = last_hidden_state.gather(1, pick).squeeze(1)
    elif end_mode == 'last':
        if scores.requires_grad:
            end_scores = scores[:, -1].float()
        else:
            _, end_scores, _ = ops.score_end(scores, None, None)
        end_hidden = last_hidden_state[:, -1, :]  # a view, like models/llava.py:65
        end_index = -torch.ones((B,))  # models/llava.py:64 (a CPU float placeholder in the reference too)
    else:
        raise ValueError(f"end_mode must be 'mask' or 'last', got {end_mode!r}")
    return ScoreModelOutput(
        scores=scores.unsqueeze(-1), end_scores=end_scores.unsqueeze(-1), last_hidden_state=last_hidden_state,
        end_last_hidden_state=end_hidden, end_index=end_index,
    )


class B200ScoreHeadMixin:
    """Mix into (or monkey-patch onto) an Accustomed*RewardModel: keeps the backbone call of the
    reference's forward and swaps the head tail.  Class attributes select the variant."""

    end_mode = 'mask'  # 'last' for LLaVA / Qwen2-VL
    upcast_scores = True  # False for Qwen2-VL (models/qwen2_vl.py:60)
    mask_from_outputs = False  # True for Qwen2-Audio (models/qwen2_audio.py:75)
    # How the reference's forward reaches the backbone:
    #   'prefix' -- `self.model(input_ids, attention_mask=..., output_hidden_states=True, **kwargs)` on the module named
    #               by base_model_prefix (models/llama.py:55-60, opt.py, llava.py:53-58, qwen2_audio.py:69-74);
    #   'super'  -- `super().forward(**kwargs, output_hidden_states=True)` (models/qwen2_vl.py:58): the reward model IS a
    #               Qwen2VLForConditionalGeneration, whose forward embeds pixel_values / image_grid_thw and builds the
    #               M-RoPE position ids.  On transformers 4.50-4.51 `self.model` is the text-only decoder, so going
    #               through the prefix there would drop (or choke on) the image path.
    backbone_call = 'prefix'
    _b200_super_forward = None  # set by patch.install(): the parent class's forward (plain function)
    _b200_super_kwargs: dict = {}  # {'logits_to_keep': 1} when that forward takes it: the lm_head the reference runs
    #                                and discards (SURVEY.md 8f rank 1) then touches one position instead of all

    def forward(self, input_ids=None, attention_mask=None, **kwargs):
        if self.backbone_call == 'super':
            parent = self._b200_super_forward
            if parent is None:  # mixed in by inheritance rather than patched: the next forward in the MRO
                parent = super(B200ScoreHeadMixin, self).forward
            extra = {k: v for k, v in self._b200_super_kwargs.items() if k not in kwargs}
            outputs = parent(input_ids=input_ids, attention_mask=attention_mask, output_hidden_states=True, **extra, **kwargs)
        else:
            backbone = getattr(self, self.base_model_prefix)
            outputs = backbone(input_ids, attention_mask=attention_mask, output_hidden_states=True, **kwargs)
        last_hidden_state = outputs.hidden_states[-1]
        if self.mask_from_outputs:
            attention_mask = outputs.attention_mask
        return score_model_outputs(last_hidden_state, self.score_head.weight, attention_mask, self.end_mode,
                                   self.upcast_scores)
