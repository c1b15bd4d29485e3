"""Block-scaled fp8 inputs (extension; the reference has no fp8 path).

BASELINE.json config 5 asks for stripe attention on block-scaled fp8 Q/K/V.  fp8 (e4m3 / e5m2) tensors travel with a
``descale`` tensor.  e4m3 q / k / v of head size 128 whose descales are per tensor, per head or per token block x head
(k / v: blocks that are whole 128-key tiles) go straight into the fp8 forward kernel (``kind::f8f6f4``, one byte per
element on the NVLink wire, scales applied to the fp32 scores / folded into P; ``parallel/api.py:_fp8_kernel_scales``,
``csrc/attn_fwd_sm90.cu``); everything else (e5m2, scales that vary inside a row such as MX per-32 along head_dim,
sliding windows, other head sizes) is expanded to bf16 right before the attention call.  The scale layout is
deliberately general: ``descale.shape[d]`` must divide ``x.shape[d]`` in every dimension, the quotient is the block
size along that dimension (``float8_e8m0fnu`` scales are accepted as well).  Forward only: fp8 tensors carry no
gradient.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import torch

FP8_DTYPES = tuple(getattr(torch, n) for n in ("float8_e4m3fn", "float8_e5m2") if hasattr(torch, n))


def is_fp8(t: torch.Tensor) -> bool:
    return t.dtype in FP8_DTYPES


def _expand_scale(scale: torch.Tensor, shape: Sequence[int]) -> torch.Tensor:
    scale = scale.float()
    while scale.dim() < len(shape):
        scale = scale.unsqueeze(-1)
    if scale.dim() != len(shape):
        raise ValueError(f"descale has more dimensions ({scale.dim()}) than the data ({len(shape)})")
    for d, (n, s) in enumerate(zip(shape, scale.shape)):
        if n % s:
            raise ValueError(f"descale dim {d} ({s}) must divide the data dim ({n})")
        if s not in (1, n):
            scale = scale.repeat_interleave(n // s, dim=d)
    return scale


def dequantize(x: torch.Tensor, descale: Optional[torch.Tensor], out_dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """``x_fp8 * descale`` (block-broadcast) in ``out_dtype``."""
    if not is_fp8(x):
        return x
    if descale is None:
        raise ValueError("fp8 inputs need their descale tensor (q_descale / k_descale / v_descale or descale=...)")
    return (x.float() * _expand_scale(descale, x.shape)).to(out_dtype)


def quantize_blockwise(x: torch.Tensor, block: Sequence[int], dtype: torch.dtype = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Quantise to fp8 with one fp32 descale per ``block`` (block[d] elements along dim d; 0 or -1 = whole dim).

    Returns ``(x_fp8, descale)`` with ``descale.shape[d] == x.shape[d] // block[d]``."""
    dtype = dtype or torch.float8_e4m3fn
    fmax = torch.finfo(dtype).max
    block = [x.shape[d] if b in (0, -1) else b for d, b in enumerate(block)]
    view, red = [], []
    for d, (n, b) in enumerate(zip(x.shape, block)):
        if n % b:
            raise ValueError(f"block {b} does not divide dim {d} ({n})")
        view += [n // b, b]
        red.append(2 * d + 1)
    amax = x.float().reshape(view).abs().amax(dim=red).clamp_min(1e-12)
    descale = amax / fmax
    q = (x.float() / _expand_scale(descale, x.shape)).clamp(-fmax, fmax).to(dtype)
    return q, descale


def quantize_per_head(x: torch.Tensor, keep_dims: Sequence[int] = (), dtype: torch.dtype = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """One descale per head (heads at dim -2), plus one per index of every dim listed in ``keep_dims`` (e.g. the
    pack dim of a kv / qkv tensor).  The coarsest granularity the fp8 forward kernel consumes natively; token-block x
    head scales (``quantize_blockwise(x, [1, 128, 1, 0])``) are native as well, scales along head_dim are not.

        q8, dq = quantize_per_head(q)                       # q (B, S, H, D)       -> dq (1, 1, H, 1)
        kv8, dkv = quantize_per_head(kv, keep_dims=(2,))    # kv (B, S, 2, Hkv, D) -> dkv (1, 1, 2, Hkv, 1)
    """
    nd = x.dim()
    keep = {d % nd for d in keep_dims} | {nd - 2}
    return quantize_blockwise(x, [1 if d in keep else 0 for d in range(nd)], dtype)

