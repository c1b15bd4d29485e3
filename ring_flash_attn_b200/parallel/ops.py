"""``torch.library`` registration of the context-parallel attention op.

Two custom ops, ``rfa_b200::cp_attn_fwd`` and ``rfa_b200::cp_attn_bwd``, with fake (meta) implementations and an
autograd formula, so that ``torch.compile(fullgraph=True)`` traces THROUGH the public functions without a graph
break: dynamo only sees tensors, ints, floats and strings crossing the op boundary; everything that is host code
by nature - reading ``cu_seqlens``, building / caching the plan, peer-memory contexts, kernel launches - happens
inside the opaque op.  The reference runs every test a second time under ``torch.compile``
(/root/reference/test/test.sh:23-25, test/test_ring_flash_attn_func.py:97-100).

What crosses the boundary instead of Python objects:

* the scheme as a string plus a short list of ints (``spec``) - enough to rebuild the (cached) plan,
* ``cu_seqlens`` tensors as tensors (read on the host inside the op; pass CPU tensors to avoid a device sync),
* the process group as its ``group_name`` (resolved back with c10d's registry; "" = default group).
"""
from __future__ import annotations

import functools
from typing import List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist
from torch import Tensor

from ..ops import plan as P
from ..utils import trace
from . import engine
from .comm import group_info

BATCH_SCHEMES = ("ring", "zigzag", "stripe")
VARLEN_SCHEMES = ("ring_varlen", "zigzag_varlen")


# ----------------------------------------------------------------------------------------------
# process groups <-> names
# ----------------------------------------------------------------------------------------------

def group_name(group) -> str:
    if group is None or not (dist.is_available() and dist.is_initialized()):
        return ""
    return str(group.group_name)


def resolve_group(name: str):
    if not name or not (dist.is_available() and dist.is_initialized()):
        return None
    from torch.distributed.distributed_c10d import _resolve_process_group

    return _resolve_process_group(name)


# ----------------------------------------------------------------------------------------------
# cu_seqlens on the host
# ----------------------------------------------------------------------------------------------

def cu_seqlens_to_host(cu) -> Tuple[int, ...]:
    """Host copy of a cu_seqlens tensor.  A device tensor is read back once; the result is remembered ON the
    tensor object together with its version counter (never keyed by address: the caching allocator hands the
    same address to the next batch's cu_seqlens)."""
    if not isinstance(cu, torch.Tensor):
        return tuple(int(x) for x in cu)
    if cu.device.type == "cpu":
        return tuple(int(x) for x in cu.tolist())
    cached = getattr(cu, "_rfa_host", None)
    if cached is not None and cached[0] == cu._version:
        return cached[1]
    vals = tuple(int(x) for x in cu.tolist())
    try:
        cu._rfa_host = (cu._version, vals)
    except AttributeError:  # pragma: no cover - exotic tensor subclasses
        pass
    return vals


# ----------------------------------------------------------------------------------------------
# plans (cached per (scheme, rank, shapes, ...)); each plan can produce its peers' plans
# ----------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=512)
def batch_plan(scheme, rank, world, batch, seqlen, causal, window=(-1, -1)):
    if scheme == "ring":
        plan = P.plan_ring(rank, world, batch, seqlen, causal, window)
    elif scheme == "zigzag":
        plan = P.plan_zigzag(rank, world, batch, seqlen, window)
    elif scheme == "stripe":
        plan = P.plan_stripe(rank, world, batch, seqlen, window)
    else:
        raise ValueError(scheme)
    plan.peer = lambda r: batch_plan(scheme, r, world, batch, seqlen, causal, window)
    return plan


@functools.lru_cache(maxsize=512)
def varlen_plan(scheme, rank, world, cu, causal, window=(-1, -1)):
    if scheme == "ring":
        plan = P.plan_ring_varlen(rank, world, cu, causal, window)
    elif scheme == "zigzag":
        plan = P.plan_zigzag_varlen(rank, world, cu, window)
    else:
        raise ValueError(scheme)
    plan.peer = lambda r: varlen_plan(scheme, r, world, cu, causal, window)
    return plan


@functools.lru_cache(maxsize=512)
def zigzag_llama3_plan(rank, world, global_cu, causal, window=(-1, -1)):
    plan = P.plan_zigzag_llama3(rank, world, global_cu, causal, window)
    plan.peer = lambda r: zigzag_llama3_plan(r, world, global_cu, causal, window)
    return plan


@functools.lru_cache(maxsize=512)
def llama3_plan(rank, world, tokens, cu_q, cu_k, k_start, causal, window=(-1, -1)):
    """The llama3 entry point only receives THIS rank's slice description, so the plan cannot derive its peers'
    plans (``plan.peer`` is absent): the fused path learns what every peer needs from the peers themselves, inside
    the launch (``parallel/symm.py``: needs exchange over the signal pads)."""
    return P.plan_llama3(rank, world, tokens, cu_q, cu_k, k_start, causal, window)


def resolve_plan(scheme: str, spec: Sequence[int], cu_a: Optional[Tensor], cu_b: Optional[Tensor], q_rows: int,
                 group):
    """(plan, transport, heads_k_stride) for one call."""
    rank, world = group_info(group)
    spec = [int(x) for x in spec]
    if scheme in BATCH_SCHEMES:
        b, s, causal, wl, wr = spec
        return batch_plan(scheme, rank, world, b, s, bool(causal), (wl, wr)), "ring", 1
    if scheme in VARLEN_SCHEMES:
        causal, wl, wr = spec
        cu = cu_seqlens_to_host(cu_a)
        plan = varlen_plan(scheme[:-len("_varlen")], rank, world, cu, bool(causal), (wl, wr))
        if plan.q_rows != q_rows:
            raise ValueError(f"cu_seqlens[-1]={plan.q_rows} does not match the {q_rows} local tokens")
        return plan, "ring", 1
    if scheme == "llama3":
        k_start, causal, wl, wr, stride = spec
        plan = llama3_plan(rank, world, q_rows, cu_seqlens_to_host(cu_a), cu_seqlens_to_host(cu_b), k_start,
                           bool(causal), (wl, wr))
        return plan, "allgather", stride
    if scheme == "zigzag_llama3":
        causal, wl, wr = spec
        cu = cu_seqlens_to_host(cu_a)
        if cu[-1] != q_rows * world:
            raise ValueError(f"cu_seqlens[-1]={cu[-1]} must equal local tokens ({q_rows}) x world size ({world}): "
                             "this entry point takes the GLOBAL cu_seqlens")
        return zigzag_llama3_plan(rank, world, cu, bool(causal), (wl, wr)), "ring", 1
    raise ValueError(f"unknown scheme {scheme!r}")


# ----------------------------------------------------------------------------------------------
# the ops
# ----------------------------------------------------------------------------------------------

def _out_dtype(q: Tensor) -> torch.dtype:
    return torch.bfloat16 if q.element_size() == 1 else q.dtype  # fp8 inputs produce bf16 outputs


def _fp8_kernel_takes(plan, q: Tensor, k: Tensor, kv_block: int) -> bool:
    """The fp8 forward kernel (e4m3, head_dim 128, Hopper GPU) reads one K and one V descale per 128-key tile:
    descale blocks must be whole tiles (multiples of 128 rows, with every key segment starting on a tile boundary)
    or cover the whole local shard; windows are not instantiated for fp8.  ``RFA_B200_FP8_KERNEL=0`` disables it."""
    import os

    from ..ops import attn_cuda, cuda_ext

    if os.environ.get("RFA_B200_FP8_KERNEL", "2") == "0" or not attn_cuda.is_fp8_kernel_input(q, k):
        return False
    if not cuda_ext.available_for(q) or engine.plan_has_window(plan):
        return False
    return kv_block == k.shape[0] or (kv_block % 128 == 0 and all(s.kv_row0 % 128 == 0 for s in plan.segments))


@torch.library.custom_op("rfa_b200::cp_attn_fwd", mutates_args=())
def cp_attn_fwd(q: Tensor, k: Tensor, v: Tensor, cu_a: Optional[Tensor], cu_b: Optional[Tensor],
                scale_q: Optional[Tensor], scale_k: Optional[Tensor], scale_v: Optional[Tensor], scheme: str,
                group: str, spec: List[int], softmax_scale: float, deterministic: bool) -> Tuple[Tensor, Tensor]:
    """q (T, Hq, D), k / v (T, Hkv, D) token-major -> (out (T, Hq, D), lse (Hq, T) fp32).

    ``scale_q`` (nq, Hq) / ``scale_k``, ``scale_v`` (nk, Hkv): block descale tables of fp8 q / k / v (None for
    bf16 / fp16): one fp32 per block of T / nq (T / nk) consecutive token-major rows and head."""
    pg = resolve_group(group)
    plan, transport, stride = resolve_plan(scheme, spec, cu_a, cu_b, q.shape[0], pg)
    with trace.nvtx(f"rfa.{scheme}.fwd", q):
        return _cp_attn_fwd_impl(plan, transport, stride, pg, q, k, v, scale_q, scale_k, scale_v, softmax_scale)


def _cp_attn_fwd_impl(plan, transport, stride, pg, q, k, v, scale_q, scale_k, scale_v, softmax_scale):
    if scale_q is not None:
        from ..ops import attn_cuda

        q_block, kv_block = -(-q.shape[0] // scale_q.shape[0]), -(-k.shape[0] // scale_k.shape[0])
        if _fp8_kernel_takes(plan, q, k, kv_block):
            sc = attn_cuda.Fp8Scales(scale_q.float().contiguous(), q_block, scale_k.float().contiguous(),
                                     scale_v.float().contiguous(), kv_block)
            with attn_cuda.fp8_scales(sc):
                return engine.cp_forward(plan, q, k, v, softmax_scale, pg, transport, stride)
        # key tiles would straddle descale blocks (or no kernel for this input): expand to bf16 in front of the op
        def deq(x, table, block):
            return (x.float() * table.float().repeat_interleave(block, dim=0)[:x.shape[0]].unsqueeze(-1)).to(torch.bfloat16)

        q, k, v = deq(q, scale_q, q_block), deq(k, scale_k, kv_block), deq(v, scale_v, kv_block)
    return engine.cp_forward(plan, q, k, v, softmax_scale, pg, transport, stride)


@cp_attn_fwd.register_fake
def _(q, k, v, cu_a, cu_b, scale_q, scale_k, scale_v, scheme, group, spec, softmax_scale, deterministic):
    return (q.new_empty(q.shape, dtype=_out_dtype(q)), q.new_empty((q.shape[1], q.shape[0]), dtype=torch.float32))


@torch.library.custom_op("rfa_b200::cp_attn_bwd", mutates_args=())
def cp_attn_bwd(dout: Tensor, q: Tensor, k: Tensor, v: Tensor, out: Tensor, lse: Tensor, cu_a: Optional[Tensor],
                cu_b: Optional[Tensor], scheme: str, group: str, spec: List[int], softmax_scale: float,
                deterministic: bool) -> Tuple[Tensor, Tensor, Tensor]:
    pg = resolve_group(group)
    plan, transport, stride = resolve_plan(scheme, spec, cu_a, cu_b, q.shape[0], pg)
    with trace.nvtx(f"rfa.{scheme}.bwd", q):
        return engine.cp_backward(plan, dout, q, k, v, out, lse, softmax_scale, pg, transport, stride, deterministic)


@cp_attn_bwd.register_fake
def _(dout, q, k, v, out, lse, cu_a, cu_b, scheme, group, spec, softmax_scale, deterministic):
    return torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)


def _setup_context(ctx, inputs, output):
    q, k, v, cu_a, cu_b, _sq, _sk, _sv, scheme, group, spec, softmax_scale, deterministic = inputs
    out, lse = output
    ctx.save_for_backward(q, k, v, out, lse, cu_a, cu_b)
    ctx.meta = (scheme, group, list(spec), softmax_scale, deterministic)
    ctx.set_materialize_grads(False)


def _backward(ctx, dout, _dlse):
    q, k, v, out, lse, cu_a, cu_b = ctx.saved_tensors
    scheme, group, spec, softmax_scale, deterministic = ctx.meta
    if dout is None:
        dout = torch.zeros_like(out)
    dq, dk, dv = cp_attn_bwd(dout, q, k, v, out, lse, cu_a, cu_b, scheme, group, spec, softmax_scale, deterministic)
    return dq, dk, dv, None, None, None, None, None, None, None, None, None, None


torch.library.register_autograd("rfa_b200::cp_attn_fwd", _backward, setup_context=_setup_context)
