"""ring_flash_attn_b200 - Hopper-native context-parallel flash attention.

Public surface mirrors zhuzilin/ring-flash-attention (/root/reference/ring_flash_attn/__init__.py:1-35).
The Hugging Face adapter is imported lazily so that ``import ring_flash_attn_b200`` never requires
``transformers`` (the reference imports it eagerly and breaks on transformers 5.x).
"""
from .parallel.api import *  # noqa: F401,F403
from .parallel.api import __all__ as _api_all

__version__ = "0.2.0"

_LAZY = {
    "substitute_hf_flash_attn": ("ring_flash_attn_b200.models.hf_adapter", "substitute_hf_flash_attn"),
    "update_ring_flash_attn_params": ("ring_flash_attn_b200.models.hf_adapter", "update_ring_flash_attn_params"),
    "use_ring_attn": ("ring_flash_attn_b200.models.hf_adapter", "use_ring_attn"),
}


def __getattr__(name):
    if name in _LAZY:
        import importlib

        mod, attr = _LAZY[name]
        return getattr(importlib.import_module(mod), attr)
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")


__all__ = list(_api_all) + list(_LAZY)
