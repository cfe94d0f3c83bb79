"""TEST INFRASTRUCTURE ONLY -- bootstrap that imports the *unmodified* reference
(a checkout of PKU-Alignment/align-anything named by AA_REFERENCE_ROOT) so that
golden vectors of the reference's own functions can be generated
(tests/golden/make_golden.py).

Nothing in tests/, `__graft_entry__.smoke()` or `bench.py` imports this module:
they read the stored golden vectors instead.  It touches no
reference file; it only arranges `sys.modules` so that the reference's heavy
optional dependencies (deepspeed, accelerate, peft, diffusers, librosa, ray,
bitsandbytes) resolve to permissive stubs -- none of them is on the arithmetic
path (SURVEY.md section 8c, Appendix B).
"""
from __future__ import annotations

import importlib.machinery
import os
import sys
import types
from types import SimpleNamespace
from unittest.mock import MagicMock

REF = os.environ.get('AA_REFERENCE_ROOT', '')

_installed = False


def available() -> bool:
    return bool(REF) and os.path.isdir(os.path.join(REF, 'align_anything'))


class _Stub(types.ModuleType):
    def __init__(self, name):
        super().__init__(name)
        self.__path__ = []
        self.__spec__ = importlib.machinery.ModuleSpec(name, None, is_package=True)

    def __getattr__(self, k):
        if k.startswith('__'):
            raise AttributeError(k)
        return MagicMock(name=f'{self.__name__}.{k}')


class _Finder:
    ROOTS = ('librosa', 'deepspeed', 'accelerate', 'peft', 'diffusers', 'bitsandbytes', 'ray')

    def find_spec(self, name, path=None, target=None):
        if name.split('.')[0] in self.ROOTS:
            return importlib.machinery.ModuleSpec(name, self, is_package=True)
        return None

    def create_module(self, spec):
        return _Stub(spec.name)

    def exec_module(self, m):
        pass


def _bare_pkg(name, path):
    m = types.ModuleType(name)
    m.__path__ = [path]
    m.__package__ = name
    m.__spec__ = importlib.machinery.ModuleSpec(name, None, is_package=True)
    m.__spec__.submodule_search_locations = [path]
    sys.modules[name] = m


def install() -> None:
    """Make `import align_anything.<...>` resolve to the reference sources."""
    global _installed
    if _installed:
        return
    if not available():
        raise RuntimeError(f'reference not present at {REF}')
    # 1) the real stack first, so transformers caches "accelerate/peft/deepspeed absent"
    import torch  # noqa: F401
    import transformers  # noqa: F401
    from transformers import (  # noqa: F401
        AutoModelForCausalLM,
        AutoProcessor,
        AutoTokenizer,
        GenerationConfig,
        PreTrainedModel,
        get_scheduler,
    )
    import transformers.integrations.deepspeed  # noqa: F401

    # 2) permissive stubs for absent deps that are not on the arithmetic path
    sys.meta_path.insert(0, _Finder())
    # 3) bare packages so the reference's package __init__ (-> librosa, read_video) never runs
    _bare_pkg('align_anything', REF + '/align_anything')
    _bare_pkg('align_anything.configs', REF + '/align_anything/configs')
    # 4) transformers 5.x moved these names
    import transformers.tokenization_utils as _tu
    import transformers.tokenization_utils_base as _tub

    for n in ('BatchEncoding', 'PaddingStrategy', 'TruncationStrategy'):
        if not hasattr(_tu, n):
            setattr(_tu, n, getattr(_tub, n))
    _installed = True


def tools():
    install()
    import align_anything.utils.tools as t

    return t


class _FakeLM:
    """Stands in for `engine.module`: returns a fixed logits tile."""

    def __init__(self, logits):
        self._logits = logits

    def __call__(self, **kw):
        return SimpleNamespace(logits=self._logits)


def make_dpo_trainer(policy_logits, ref_logits, pad_token_id, scale_coeff=0.1, modality='text'):
    """object.__new__ a reference DPOTrainer with only the attributes loss() reads."""
    install()
    if modality == 'text':
        from align_anything.trainers.text_to_text.dpo import DPOTrainer
    elif modality == 'image':
        from align_anything.trainers.text_image_to_text.dpo import DPOTrainer
    elif modality == 'audio':
        from align_anything.trainers.text_audio_to_text.dpo import DPOTrainer
    elif modality == 'simpo':
        from align_anything.trainers.text_to_text.simpo import SimPOTrainer as DPOTrainer
    elif modality == 'orpo':
        from align_anything.trainers.text_to_text.orpo import ORPOTrainer as DPOTrainer
    elif modality == 'kto':
        from align_anything.trainers.text_to_text.kto import KTOTrainer as DPOTrainer
    else:
        raise ValueError(modality)
    from align_anything.utils.tools import dict_to_namedtuple

    t = object.__new__(DPOTrainer)
    t.cfgs = dict_to_namedtuple({'train_cfgs': {'scale_coeff': scale_coeff, 'gamma': 0.5, 'scale_better': 1.0,
                                                'scale_worse': 1.33}})
    t.kl = 0.07
    t.tokenizer = SimpleNamespace(pad_token_id=pad_token_id)
    t.infer_batch = lambda b: {k: v for k, v in b.items() if k != 'meta_info'}
    t.model = SimpleNamespace(module=_FakeLM(policy_logits))
    t.reference_model = SimpleNamespace(module=_FakeLM(ref_logits))
    return t


def make_ppo_trainer(
    kl_coeff=0.02,
    clip_range_ratio=0.2,
    clip_range_score=50.0,
    clip_range_value=5.0,
    gamma=1.0,
    gae_lambda=0.95,
    modality='text',
):
    install()
    if modality == 'text':
        from align_anything.trainers.text_to_text.ppo import PPOTrainer
    elif modality == 'image':
        from align_anything.trainers.text_image_to_text.ppo import PPOTrainer
    elif modality == 'audio':
        from align_anything.trainers.text_audio_to_text.ppo import PPOTrainer
    elif modality == 'saferlhf':
        from align_anything.trainers.text_image_to_text.saferlhf import SafeRLHFVTrainer as PPOTrainer
    else:
        raise ValueError(modality)
    p = object.__new__(PPOTrainer)
    p.kl_coeff = kl_coeff
    p.clip_range_ratio = clip_range_ratio
    p.clip_range_score = clip_range_score
    p.clip_range_value = clip_range_value
    p.gamma = gamma
    p.gae_lambda = gae_lambda
    return p
