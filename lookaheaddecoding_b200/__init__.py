"""lookaheaddecoding_b200 -- H100-native (sm_90a) lookahead/verification decoding step.

Drop-in for the hot path of hao-ai-lab/LookaheadDecoding behind the reference's plugin surface
(lade/__init__.py:1-5):  ``augment_all()``, ``config_lade(...)``, then plain ``model.generate(...)``.
"""
from .utils import augment_llama
from .utils import augment_generate
from .utils import augment_all
from .utils import config_lade, save_log, log_history, restore_generate
from .lade_distributed import get_device, distributed
from .engine import LookaheadEngine
from ._cabi import LadeError

__all__ = [
    "augment_llama", "augment_generate", "augment_all", "config_lade", "save_log", "log_history",
    "restore_generate", "get_device", "distributed", "LookaheadEngine", "LadeError",
]
