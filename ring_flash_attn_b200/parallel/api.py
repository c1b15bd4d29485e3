"""Public attention entry points - the 18 functions of the reference plus ``prepare``.

Signatures, defaults and return values follow the reference exactly
(/root/reference/ring_flash_attn/__init__.py:1-35; batch: ring_flash_attn.py:223-301,
zigzag_ring_flash_attn.py:268-346, stripe_flash_attn.py:300-378; varlen:
ring_flash_attn_varlen.py:268-358, zigzag_ring_flash_attn_varlen.py:415-505,
llama3_flash_attn_varlen.py:390-504) so a user can switch by changing the import.

Unlike the reference there is a single autograd bridge: each scheme only contributes a *plan*
(``ops/plan.py``); the engine (``parallel/engine.py``) runs it on the fused sm_90a path or on the
torch.distributed fallback.
"""
from __future__ import annotations

import functools
import os
from typing import Optional, Tuple

import torch

from . import ops as O
from .comm import group_info
from .ops import cu_seqlens_to_host  # noqa: F401  (re-exported: models/hf_adapter.py, tests)

__all__ = [
    "ring_flash_attn_func", "ring_flash_attn_kvpacked_func", "ring_flash_attn_qkvpacked_func",
    "zigzag_ring_flash_attn_func", "zigzag_ring_flash_attn_kvpacked_func", "zigzag_ring_flash_attn_qkvpacked_func",
    "stripe_flash_attn_func", "stripe_flash_attn_kvpacked_func", "stripe_flash_attn_qkvpacked_func",
    "ring_flash_attn_varlen_func", "ring_flash_attn_varlen_kvpacked_func", "ring_flash_attn_varlen_qkvpacked_func",
    "zigzag_ring_flash_attn_varlen_func", "zigzag_ring_flash_attn_varlen_kvpacked_func",
    "zigzag_ring_flash_attn_varlen_qkvpacked_func",
    "llama3_flash_attn_varlen_func", "llama3_flash_attn_varlen_kvpacked_func",
    "llama3_flash_attn_varlen_qkvpacked_func", "llama3_flash_attn_prepare_cu_seqlens",
    # beyond the reference (its README lists "zigzag llama3" as a TODO)
    "zigzag_llama3_flash_attn_varlen_func", "zigzag_llama3_flash_attn_varlen_kvpacked_func",
    "zigzag_llama3_flash_attn_varlen_qkvpacked_func",
]


# ----------------------------------------------------------------------------------------------
# the op: one torch.library custom op for every scheme (parallel/ops.py)
# ----------------------------------------------------------------------------------------------

KERNEL_HEAD_DIMS = (64, 128)  # the sm_90a kernels are instantiated for these head sizes
KERNEL_HEAD_DIM = KERNEL_HEAD_DIMS[-1]


def _pad_head_dim(q) -> int:
    """Columns of zero padding that bring the head size to the next one the kernels are instantiated for (64, 128).

    Zero columns change neither Q.K^T nor the first ``d`` columns of P.V, and their gradients are exactly zero,
    so e.g. head size 80 or 96 runs on the wgmma kernels as 128 (at the cost of the padded FLOPs) and 32 as 64,
    instead of dropping to the dense torch blocks.  ``RFA_B200_PAD_HEAD_DIM=0`` disables it, ``=force`` applies it
    on any device (used by the CPU tests)."""
    mode = os.environ.get("RFA_B200_PAD_HEAD_DIM", "1")
    d = q.shape[-1]
    if mode == "0" or d >= KERNEL_HEAD_DIM or d in KERNEL_HEAD_DIMS:
        return 0
    target = min(x for x in KERNEL_HEAD_DIMS if x > d)
    if mode == "force":
        return target - d
    if q.dtype in (torch.bfloat16, torch.float16):
        from ..ops import cuda_ext

        if cuda_ext.available_for(q):
            return target - d
    return 0


class _Unpack(torch.autograd.Function):
    """``packed.unbind(dim)`` whose backward is ONE concatenation.

    Autograd's own formula for ``qkv[:, :, i]`` allocates a zero tensor of the packed shape per slice, copies the slice
    gradient into it and then sums the three tensors: about 11x the bytes of the packed gradient per step (0.8 GB at
    the 1-GPU benchmark shape, i.e. ~9 GB of HBM traffic next to a 36 ms step).  Here dq / dk / dv are written into the
    packed gradient once.  The reference slices the same way (/root/reference/ring_flash_attn/ring_flash_attn.py:276-301)
    and pays the generic formula."""

    @staticmethod
    def forward(ctx, packed, dim):
        ctx.dim = dim
        return packed.unbind(dim)

    @staticmethod
    def backward(ctx, *grads):
        return torch.stack(grads, dim=ctx.dim), None


def _unpack(packed: torch.Tensor, dim: int):
    """Slices of a packed qkv / kv tensor along ``dim`` (views, no copy).  Under ``torch.compile`` the plain slices are
    traced: the compiler fuses their backward itself."""
    if packed.requires_grad and torch.is_grad_enabled() and not torch.compiler.is_compiling():
        return _Unpack.apply(packed, dim)
    return packed.unbind(dim)


def _cp_apply(q, k, v, scheme, spec, cu_a, cu_b, scale, group, deterministic, fp8=None):
    """Token-major q (T,Hq,D), k / v (T,Hkv,D) -> (out, lse) through ``torch.ops.rfa_b200.cp_attn_fwd``.

    Everything here is traceable by dynamo (shapes, strings, ints); plans, cu_seqlens reads, peer memory and the
    launches live inside the op, so ``torch.compile(fullgraph=True)`` works on the public functions."""
    gname = O.group_name(group)
    if fp8 is not None:
        # fp8 forward kernel: e4m3 q / k / v straight into the kernels (and over the wire), bf16 out.
        # Forward only - fp8 tensors carry no gradient.
        with torch.no_grad():
            return O.cp_attn_fwd(q, k, v, cu_a, cu_b, fp8[0], fp8[1], fp8[2], scheme, gname, spec, scale, deterministic)
    pad = _pad_head_dim(q)
    if pad:
        d = q.shape[-1]
        q, k, v = (torch.nn.functional.pad(t, (0, pad)) for t in (q, k, v))
        out, lse = O.cp_attn_fwd(q, k, v, cu_a, cu_b, None, None, None, scheme, gname, spec, scale, deterministic)
        return out[..., :d].contiguous(), lse
    return O.cp_attn_fwd(q, k, v, cu_a, cu_b, None, None, None, scheme, gname, spec, scale, deterministic)


def _as_cu_tensor(cu) -> torch.Tensor:
    return cu if isinstance(cu, torch.Tensor) else torch.tensor([int(x) for x in cu], dtype=torch.int32)


def _scale_table(descale, x) -> Optional[torch.Tensor]:
    """Canonical form of a descale the fp8 forward kernel can apply: an fp32 table ``(n_blocks, H)`` with one entry
    per block of consecutive token-major rows and head (``x``: ``(B, S, H, D)`` or ``(T, H, D)``), or None when the
    descale varies inside a row (MX-style per-32-element scales along head_dim) or does not tile the tokens evenly.

    Accepted: None / python scalars / one-element tensors (per tensor), ``(1, 1, H, 1)`` (per head), ``(B, S/blk, H, 1)``
    or ``(1, S/blk, H, 1)`` (per token block x head), ``(T/blk, H, 1)`` for packed layouts; H may be 1."""
    heads = x.shape[-2]
    if descale is None:
        return torch.ones((1, heads), dtype=torch.float32, device=x.device)
    if not isinstance(descale, torch.Tensor):
        return torch.full((1, heads), float(descale), dtype=torch.float32, device=x.device)
    d = descale.to(device=x.device, dtype=torch.float32)
    if d.numel() == 1:
        return d.reshape(1, 1).expand(1, heads).contiguous()
    if d.dim() != x.dim() or d.shape[-1] != 1 or d.shape[-2] not in (1, heads):
        return None
    tokens, blocks = tuple(x.shape[:-2]), tuple(d.shape[:-2])
    if any(n % s for n, s in zip(tokens, blocks)):
        return None
    if len(tokens) == 2:
        if blocks[0] not in (1, tokens[0]):
            return None
        t = d.reshape(blocks[0], blocks[1], d.shape[-2]).expand(tokens[0], blocks[1], heads)
        if blocks == (1, 1):
            t = t[:1]
        return t.reshape(-1, heads).contiguous()
    return d.reshape(blocks[0], d.shape[-2]).expand(blocks[0], heads).contiguous()


def _fp8_kernel_scales(q, k, v, dq, dk, dv, window_size):
    """Descale tables ``(q, k, v)`` for the fp8 forward kernel, or None when the call does not qualify: e4m3 q/k/v
    with head_dim 128 on a Hopper GPU, descales per tensor / head / token block x head (``_scale_table``), no
    sliding window, ``RFA_B200_FP8_KERNEL`` != 0.  Whether the K / V blocks line up with the 128-key tiles of the plan
    is decided inside the op (parallel/ops.py); anything else takes the dequantise-to-bf16 path."""
    if os.environ.get("RFA_B200_FP8_KERNEL", "2") == "0":
        return None
    if not (q.dtype == k.dtype == v.dtype == torch.float8_e4m3fn) or q.shape[-1] != 128:
        return None
    if tuple(window_size) != (-1, -1):
        return None
    from ..ops import cuda_ext

    if not cuda_ext.available_for(q):
        return None
    tq, tk, tv = _scale_table(dq, q), _scale_table(dk, k), _scale_table(dv, v)
    if tq is None or tk is None or tv is None or tk.shape[0] != tv.shape[0]:
        return None
    return tq, tk, tv


def _maybe_dequant(q, k, v, descale, window_size=(-1, -1)):
    """fp8 extension (utils/fp8.py): ``descale`` is a tensor for a packed input or a (q, k, v) tuple.

    Returns (q, k, v, fp8_scales): either dequantised tensors and None, or - for calls that qualify for the fp8
    forward kernel - the untouched e4m3 tensors and their descale tables."""
    from ..utils import fp8

    if not (fp8.is_fp8(q) or fp8.is_fp8(k) or fp8.is_fp8(v)):
        return q, k, v, None
    if descale is None:
        raise ValueError("fp8 q/k/v need descale=(q_descale, k_descale, v_descale)")
    dq, dk, dv = descale if isinstance(descale, (tuple, list)) else (descale, descale, descale)
    scales = _fp8_kernel_scales(q, k, v, dq, dk, dv, window_size)
    if scales is not None:
        return q, k, v, scales
    return fp8.dequantize(q, dq), fp8.dequantize(k, dk), fp8.dequantize(v, dv), None


def _split_descale(descale, pack_dim: int, n: int):
    """descale of a packed (kv / qkv) tensor -> per-tensor descales.  A tensor that carries the pack dimension
    (size n) is sliced like the data, anything else (None, a scalar tensor, per-head scales, ...) is shared."""
    if descale is None or isinstance(descale, (tuple, list)):
        return descale
    if isinstance(descale, torch.Tensor) and descale.dim() > pack_dim and descale.shape[pack_dim] == n:
        return tuple(descale.select(pack_dim, i) for i in range(n))
    return tuple(descale for _ in range(n))


def _check_common(q, dropout_p, window_size, alibi_slopes):
    if alibi_slopes is not None:
        raise NotImplementedError("alibi_slopes is not supported (same as the reference)")
    if dropout_p != 0.0:
        raise NotImplementedError("dropout_p > 0 is not supported by context-parallel attention")
    if len(tuple(window_size)) != 2:
        raise ValueError("window_size must be (left, right)")


def _scale(q, softmax_scale):
    return q.shape[-1] ** (-0.5) if softmax_scale is None else float(softmax_scale)


def _window(window_size) -> Tuple[int, int]:
    left, right = (int(x) for x in window_size)
    return (-1 if left < 0 else left, -1 if right < 0 else right)


def _run_batch(scheme, q, k, v, dropout_p, softmax_scale, causal, window_size, alibi_slopes,
               deterministic, return_attn_probs, group, descale=None):
    _check_common(q, dropout_p, window_size, alibi_slopes)
    q, k, v, fp8 = _maybe_dequant(q, k, v, descale, window_size)
    if scheme in ("zigzag", "stripe") and not causal:
        raise AssertionError(f"{scheme} attention only supports causal=True (as in the reference)")
    b, s, hq, d = q.shape
    wl, wr = _window(window_size)
    out, lse = _cp_apply(q.reshape(b * s, hq, d), k.reshape(b * s, k.shape[2], d), v.reshape(b * s, v.shape[2], d),
                         scheme, [b, s, int(bool(causal)), wl, wr], None, None, _scale(q, softmax_scale), group,
                         bool(deterministic), fp8)
    out = out.view(b, s, hq, d)
    if not return_attn_probs:
        return out
    return out, lse.view(hq, b, s).permute(1, 0, 2).contiguous(), None


def _run_varlen(scheme, q, k, v, cu_seqlens, max_seqlen, dropout_p, softmax_scale, causal, window_size,
                alibi_slopes, deterministic, return_attn_probs, group, descale=None):
    _check_common(q, dropout_p, window_size, alibi_slopes)
    q, k, v, fp8 = _maybe_dequant(q, k, v, descale, window_size)
    if scheme == "zigzag" and not causal:
        raise AssertionError("zigzag attention only supports causal=True (as in the reference)")
    wl, wr = _window(window_size)
    out, lse = _cp_apply(q, k, v, scheme + "_varlen", [int(bool(causal)), wl, wr], _as_cu_tensor(cu_seqlens), None,
                         _scale(q, softmax_scale), group, bool(deterministic), fp8)
    return (out, lse, None) if return_attn_probs else out


# ----------------------------------------------------------------------------------------------
# batch layout: ring / zigzag / stripe
# ----------------------------------------------------------------------------------------------

def _define_batch(scheme, prefix):
    def func(q, k, v, dropout_p=0.0, softmax_scale=None, causal=False, window_size=(-1, -1),
             alibi_slopes=None, deterministic=False, return_attn_probs=False, group=None, *, descale=None):
        return _run_batch(scheme, q, k, v, dropout_p, softmax_scale, causal, window_size, alibi_slopes,
                          deterministic, return_attn_probs, group, descale)

    def kvpacked_func(q, kv, dropout_p=0.0, softmax_scale=None, causal=False, window_size=(-1, -1),
                      alibi_slopes=None, deterministic=False, return_attn_probs=False, group=None, *,
                      descale=None):
        if descale is not None:  # (q_descale, kv_descale)
            dq, dkv = descale
            dk, dv = _split_descale(dkv, 2, 2)
            descale = (dq, dk, dv)
        return _run_batch(scheme, q, *_unpack(kv, 2), dropout_p, softmax_scale, causal,
                          window_size, alibi_slopes, deterministic, return_attn_probs, group, descale)

    def qkvpacked_func(qkv, dropout_p=0.0, softmax_scale=None, causal=False, window_size=(-1, -1),
                       alibi_slopes=None, deterministic=False, return_attn_probs=False, group=None, *,
                       descale=None):
        return _run_batch(scheme, *_unpack(qkv, 2), dropout_p, softmax_scale,
                          causal, window_size, alibi_slopes, deterministic, return_attn_probs, group,
                          _split_descale(descale, 2, 3))

    doc = ("{name}: q (B, S_local, Hq, D), k/v (B, S_local, Hkv, D) [kv (B,S_local,2,Hkv,D); "
           "qkv (B,S_local,3,H,D)] sharded with the '" + scheme + "' layout over `group`.  Returns out "
           "(and (out, softmax_lse (B,Hq,S_local), None) when return_attn_probs).")
    for f, suffix in ((func, "func"), (kvpacked_func, "kvpacked_func"), (qkvpacked_func, "qkvpacked_func")):
        f.__name__ = f.__qualname__ = f"{prefix}_flash_attn_{suffix}"
        f.__doc__ = doc.format(name=f.__name__)
    return func, kvpacked_func, qkvpacked_func


ring_flash_attn_func, ring_flash_attn_kvpacked_func, ring_flash_attn_qkvpacked_func = _define_batch("ring", "ring")
(zigzag_ring_flash_attn_func, zigzag_ring_flash_attn_kvpacked_func,
 zigzag_ring_flash_attn_qkvpacked_func) = _define_batch("zigzag", "zigzag_ring")
stripe_flash_attn_func, stripe_flash_attn_kvpacked_func, stripe_flash_attn_qkvpacked_func = _define_batch(
    "stripe", "stripe")


# ----------------------------------------------------------------------------------------------
# varlen layout: ring / zigzag
# ----------------------------------------------------------------------------------------------

def _define_varlen(scheme, prefix):
    def func(q, k, v, cu_seqlens, max_seqlen, dropout_p=0.0, softmax_scale=None, causal=False,
             window_size=(-1, -1), alibi_slopes=None, deterministic=False, return_attn_probs=False,
             group=None, *, descale=None):
        return _run_varlen(scheme, q, k, v, cu_seqlens, max_seqlen, dropout_p, softmax_scale, causal,
                           window_size, alibi_slopes, deterministic, return_attn_probs, group, descale)

    def kvpacked_func(q, kv, cu_seqlens, max_seqlen, dropout_p=0.0, softmax_scale=None, causal=False,
                      window_size=(-1, -1), alibi_slopes=None, deterministic=False,
                      return_attn_probs=False, group=None, *, descale=None):
        if descale is not None:
            dq, dkv = descale
            dk, dv = _split_descale(dkv, 1, 2)
            descale = (dq, dk, dv)
        return _run_varlen(scheme, q, *_unpack(kv, 1), cu_seqlens, max_seqlen, dropout_p, softmax_scale,
                           causal, window_size, alibi_slopes, deterministic, return_attn_probs, group, descale)

    def qkvpacked_func(qkv, cu_seqlens, max_seqlen, dropout_p=0.0, softmax_scale=None, causal=False,
                       window_size=(-1, -1), alibi_slopes=None, deterministic=False,
                       return_attn_probs=False, group=None, *, descale=None):
        return _run_varlen(scheme, *_unpack(qkv, 1), cu_seqlens, max_seqlen, dropout_p,
                           softmax_scale, causal, window_size, alibi_slopes, deterministic,
                           return_attn_probs, group, _split_descale(descale, 1, 3))

    doc = ("{name}: packed q (T_local, Hq, D), k/v (T_local, Hkv, D) with ONE local cu_seqlens "
           "(global cu_seqlens // world_size); every document is sharded with the '" + scheme +
           "' layout.  Returns out (and (out, softmax_lse (Hq,T_local), None) when return_attn_probs).")
    for f, suffix in ((func, "func"), (kvpacked_func, "kvpacked_func"), (qkvpacked_func, "qkvpacked_func")):
        f.__name__ = f.__qualname__ = f"{prefix}_flash_attn_varlen_{suffix}"
        f.__doc__ = doc.format(name=f.__name__)
    return func, kvpacked_func, qkvpacked_func


(ring_flash_attn_varlen_func, ring_flash_attn_varlen_kvpacked_func,
 ring_flash_attn_varlen_qkvpacked_func) = _define_varlen("ring", "ring")
(zigzag_ring_flash_attn_varlen_func, zigzag_ring_flash_attn_varlen_kvpacked_func,
 zigzag_ring_flash_attn_varlen_qkvpacked_func) = _define_varlen("zigzag", "zigzag_ring")


# ----------------------------------------------------------------------------------------------
# llama3 (all-gather style context parallelism, varlen only)
# ----------------------------------------------------------------------------------------------

def llama3_flash_attn_prepare_cu_seqlens(cu_seqlens: torch.Tensor, causal: bool, rank: int, world_size: int):
    """Per-rank cu_seqlens for the llama3 layout (flat token stream split contiguously).

    Same outputs as the reference (/root/reference/ring_flash_attn/llama3_flash_attn_varlen.py:10-60):
    ``(cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, local_k_slice)``.  The arithmetic is
    done once on the host (one device read instead of the reference's seven ``.item()`` syncs)."""
    cu = list(cu_seqlens_to_host(cu_seqlens))
    total = cu[-1]
    if total % world_size:
        raise AssertionError("total length must be divisible by world_size")
    L = total // world_size
    lo, hi = rank * L, (rank + 1) * L
    # documents overlapping [lo, hi): first doc whose end is > lo ... last doc whose start is < hi
    left = max(i for i in range(len(cu) - 1) if cu[i] <= lo)
    right = min(i for i in range(1, len(cu)) if cu[i] >= hi)
    window = cu[left:right + 1]
    cu_q = [min(max(x - lo, 0), L) for x in window]
    cu_q[0], cu_q[-1] = 0, L
    slice_left = cu[left]
    slice_right = hi if causal else cu[right]
    cu_k = list(window)
    cu_k[-1] = slice_right
    cu_k = [x - slice_left for x in cu_k]
    dev = cu_seqlens.device if isinstance(cu_seqlens, torch.Tensor) else None
    dt = cu_seqlens.dtype if isinstance(cu_seqlens, torch.Tensor) else torch.int32
    cu_q_t = torch.tensor(cu_q, dtype=dt, device=dev)
    cu_k_t = torch.tensor(cu_k, dtype=dt, device=dev)
    cu_q_t._rfa_host = (cu_q_t._version, tuple(cu_q))  # saves the entry point one device read (optional)
    cu_k_t._rfa_host = (cu_k_t._version, tuple(cu_k))
    max_q = max(b - a for a, b in zip(cu_q[:-1], cu_q[1:]))
    max_k = max(b - a for a, b in zip(cu_k[:-1], cu_k[1:]))
    return cu_q_t, cu_k_t, max_q, max_k, slice(slice_left, slice_right)


def llama3_flash_attn_varlen_func(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k,
                                  heads_k_stride, local_k_slice, dropout_p=0.0, softmax_scale=None,
                                  causal=False, window_size=(-1, -1), alibi_slopes=None,
                                  deterministic=False, return_attn_probs=False, group=None, *, descale=None):
    """llama3-style CP: q/k/v (T_local, H*, D) are a contiguous slice of the flat token stream; the
    cu_seqlens / local_k_slice come from :func:`llama3_flash_attn_prepare_cu_seqlens`."""
    _check_common(q, dropout_p, window_size, alibi_slopes)
    q, k, v, fp8 = _maybe_dequant(q, k, v, descale, window_size)
    k_start = int(local_k_slice.start or 0)
    wl, wr = _window(window_size)
    # any valid (cu_seqlens_q, cu_seqlens_k, local_k_slice) stays on the fused path: what each peer needs of this
    # rank's K/V is learnt from the peers at run time (parallel/symm.py), not from attributes of these tensors
    out, lse = _cp_apply(q, k, v, "llama3", [k_start, int(bool(causal)), wl, wr, int(heads_k_stride)],
                         _as_cu_tensor(cu_seqlens_q), _as_cu_tensor(cu_seqlens_k), _scale(q, softmax_scale), group,
                         bool(deterministic), fp8)
    return (out, lse, None) if return_attn_probs else out


def llama3_flash_attn_varlen_kvpacked_func(q, kv, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k,
                                           heads_k_stride, local_k_slice, dropout_p=0.0, softmax_scale=None,
                                           causal=False, window_size=(-1, -1), alibi_slopes=None,
                                           deterministic=False, return_attn_probs=False, group=None, *,
                                           descale=None):
    """kv (T_local, 2, Hkv, D) variant of :func:`llama3_flash_attn_varlen_func`."""
    if descale is not None:
        dq, dkv = descale
        dk, dv = _split_descale(dkv, 1, 2)
        descale = (dq, dk, dv)
    return llama3_flash_attn_varlen_func(q, *_unpack(kv, 1), cu_seqlens_q, cu_seqlens_k, max_seqlen_q,
                                         max_seqlen_k, heads_k_stride, local_k_slice, dropout_p, softmax_scale,
                                         causal, window_size, alibi_slopes, deterministic, return_attn_probs,
                                         group, descale=descale)


def llama3_flash_attn_varlen_qkvpacked_func(qkv, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k,
                                            heads_k_stride, local_k_slice, dropout_p=0.0, softmax_scale=None,
                                            causal=False, window_size=(-1, -1), alibi_slopes=None,
                                            deterministic=False, return_attn_probs=False, group=None, *,
                                            descale=None):
    """qkv (T_local, 3, H, D) variant of :func:`llama3_flash_attn_varlen_func`."""
    return llama3_flash_attn_varlen_func(*_unpack(qkv, 1), cu_seqlens_q, cu_seqlens_k,
                                         max_seqlen_q, max_seqlen_k, heads_k_stride, local_k_slice, dropout_p,
                                         softmax_scale, causal, window_size, alibi_slopes, deterministic,
                                         return_attn_probs, group, descale=_split_descale(descale, 1, 3))


# ----------------------------------------------------------------------------------------------
# zigzag llama3: flat packed stream, rank r holds chunks r and 2W-1-r of 2W (beyond the reference)
# ----------------------------------------------------------------------------------------------

def zigzag_llama3_flash_attn_varlen_func(q, k, v, cu_seqlens, dropout_p=0.0, softmax_scale=None, causal=True,
                                         window_size=(-1, -1), alibi_slopes=None, deterministic=False,
                                         return_attn_probs=False, group=None, *, descale=None):
    """Load-balanced context parallelism for packed documents of ARBITRARY lengths.

    The flat token stream (all documents back to back, ``cu_seqlens`` = the GLOBAL cumulative lengths, the same on
    every rank) is cut into ``2 * world_size`` equal chunks and rank r holds chunks ``r`` and ``2W-1-r``
    (``parallel.layouts.shard_zigzag_llama3``).  Unlike the llama3 layout every rank does the same amount of causal
    work, and unlike the zigzag varlen layout no document length has to be divisible by ``2 * world_size``.
    q (T_local, Hq, D), k / v (T_local, Hkv, D); returns out (and (out, lse (Hq, T_local), None))."""
    _check_common(q, dropout_p, window_size, alibi_slopes)
    q, k, v, fp8 = _maybe_dequant(q, k, v, descale, window_size)
    wl, wr = _window(window_size)
    out, lse = _cp_apply(q, k, v, "zigzag_llama3", [int(bool(causal)), wl, wr], _as_cu_tensor(cu_seqlens), None,
                         _scale(q, softmax_scale), group, bool(deterministic), fp8)
    return (out, lse, None) if return_attn_probs else out


def zigzag_llama3_flash_attn_varlen_kvpacked_func(q, kv, cu_seqlens, dropout_p=0.0, softmax_scale=None, causal=True,
                                                  window_size=(-1, -1), alibi_slopes=None, deterministic=False,
                                                  return_attn_probs=False, group=None, *, descale=None):
    """kv (T_local, 2, Hkv, D) variant of :func:`zigzag_llama3_flash_attn_varlen_func`."""
    if descale is not None:
        dq, dkv = descale
        dk, dv = _split_descale(dkv, 1, 2)
        descale = (dq, dk, dv)
    return zigzag_llama3_flash_attn_varlen_func(q, *_unpack(kv, 1), cu_seqlens, dropout_p, softmax_scale, causal,
                                                window_size, alibi_slopes, deterministic, return_attn_probs, group,
                                                descale=descale)


def zigzag_llama3_flash_attn_varlen_qkvpacked_func(qkv, cu_seqlens, dropout_p=0.0, softmax_scale=None, causal=True,
                                                   window_size=(-1, -1), alibi_slopes=None, deterministic=False,
                                                   return_attn_probs=False, group=None, *, descale=None):
    """qkv (T_local, 3, H, D) variant of :func:`zigzag_llama3_flash_attn_varlen_func`."""
    return zigzag_llama3_flash_attn_varlen_func(*_unpack(qkv, 1), cu_seqlens, dropout_p, softmax_scale,
                                                causal, window_size, alibi_slopes, deterministic, return_attn_probs,
                                                group, descale=_split_descale(descale, 1, 3))

