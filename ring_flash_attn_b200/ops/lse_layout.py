"""Varlen LSE layout converters.

Parity with the reference's ``flatten_varlen_lse`` / ``unflatten_varlen_lse`` (TorchScript:
/root/reference/ring_flash_attn/utils.py:76-95; Triton kernels: triton_utils.py:6-137): convert
between the padded ``(batch, H, max_seqlen)`` layout of old flash-attn and the packed ``(H, total)``
layout.  On CUDA the work is done by the small sm_90a copy kernels in ``csrc/lse_layout.cu``; on CPU
(and as the oracle for the kernels) by the torch implementation below.
"""
from __future__ import annotations

import torch


def _flatten_torch(lse: torch.Tensor, cu_seqlens: torch.Tensor) -> torch.Tensor:
    cu = [int(c) for c in cu_seqlens.tolist()]
    return torch.cat([lse[i, :, : b - a] for i, (a, b) in enumerate(zip(cu[:-1], cu[1:]))], dim=-1)


def _unflatten_torch(lse: torch.Tensor, cu_seqlens: torch.Tensor, max_seqlen: int) -> torch.Tensor:
    cu = [int(c) for c in cu_seqlens.tolist()]
    n = len(cu) - 1
    heads = lse.shape[1]
    out = torch.empty((n, max_seqlen, heads, 1), dtype=torch.float32, device=lse.device)
    for i, (a, b) in enumerate(zip(cu[:-1], cu[1:])):
        out[i, : b - a] = lse[a:b]
    return out.squeeze(-1).transpose(1, 2).contiguous()


def flatten_varlen_lse(lse: torch.Tensor, cu_seqlens: torch.Tensor) -> torch.Tensor:
    """``(batch, H, max_seqlen)`` -> ``(H, total_tokens)``."""
    if lse.is_cuda:
        from . import cuda_ext

        if cuda_ext.available_for(lse):
            return cuda_ext.load().lse_flatten(lse.contiguous(), cu_seqlens.to(torch.int32))
    return _flatten_torch(lse, cu_seqlens)


def unflatten_varlen_lse(lse: torch.Tensor, cu_seqlens: torch.Tensor, max_seqlen: int) -> torch.Tensor:
    """``(total_tokens, H, 1)`` -> ``(batch, H, max_seqlen)``; padding is left uninitialised."""
    if lse.is_cuda:
        from . import cuda_ext

        if cuda_ext.available_for(lse):
            return cuda_ext.load().lse_unflatten(lse.contiguous(), cu_seqlens.to(torch.int32), int(max_seqlen))
    return _unflatten_torch(lse, cu_seqlens, max_seqlen)
