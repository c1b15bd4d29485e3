"""Loader for the in-tree sm_90a extension (``ring_flash_attn_b200/_C*.so``).

The extension is built ahead of time by ``__graft_entry__.build()`` / ``python setup.py build_ext
--inplace`` (nvcc cross-compiles without a GPU) so that it travels with the source tree.  On a
Hopper GPU a missing extension is a hard error - the CUDA path must never silently fall back.
"""
from __future__ import annotations

import functools
import importlib
import os

import torch


@functools.lru_cache(maxsize=None)
def _device_is_sm90(index: int) -> bool:
    major, _minor = torch.cuda.get_device_capability(index)
    return major == 9


@functools.lru_cache(maxsize=None)
def load():
    try:
        return importlib.import_module("ring_flash_attn_b200._C")
    except ImportError as e:  # pragma: no cover - exercised only on broken installs
        raise RuntimeError(
            "ring_flash_attn_b200._C (the sm_90a extension) is not built; run "
            "`python -c 'import __graft_entry__ as g; g.build()'` or `python setup.py build_ext --inplace`"
        ) from e


def available_for(t: torch.Tensor) -> bool:
    """True when ``t`` lives on a Hopper GPU (then the extension is mandatory)."""
    if not t.is_cuda or os.environ.get("RFA_B200_FORCE_TORCH", "0") == "1":
        return False
    if not _device_is_sm90(t.device.index if t.device.index is not None else torch.cuda.current_device()):
        return False
    load()
    return True


class _LaunchCounter:
    """Counts launches of this library's own kernels (bench.py reports it as ``gpu_launches``)."""

    def __init__(self):
        self.value = 0

    def reset(self):
        self.value = 0


_COUNTER = _LaunchCounter()


def launch_counter() -> _LaunchCounter:
    return _COUNTER


def note_launch(n: int = 1) -> None:
    _COUNTER.value += n
