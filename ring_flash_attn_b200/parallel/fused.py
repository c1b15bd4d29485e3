"""Fused sm_90a execution of a context-parallel plan.

``world == 1``: one forward launch and one backward launch over the whole plan.
``world > 1`` : the same kernels, with every remote K/V shard arriving through peer-mapped staging
buffers that the *attention kernel's own communication CTAs* fill over NVLink while the math on the
local shard runs (``parallel/symm.py`` + ``csrc/comm_sm90.cu``).  No NCCL call is on this path.

Replaces the per-step Python loops of the reference (flash-attn call + fp32 merge + batch_isend_irecv per ring
step: /root/reference/ring_flash_attn/ring_flash_attn.py:7-154, zigzag_ring_flash_attn.py:7-199,
stripe_flash_attn.py:7-231, and the all-gather / reduce-scatter loop of llama3_flash_attn_varlen.py:63-299).
"""
from __future__ import annotations

import os

import torch

from ..ops import attn_cuda
from ..ops.plan import CPPlan
from .comm import group_info


def available(q: torch.Tensor, group) -> bool:
    _rank, world = group_info(group)
    if world == 1:
        return True
    if os.environ.get("RFA_B200_DISABLE_P2P", "0") == "1":
        return False
    from . import symm

    return symm.peer_context(group, q.device) is not None


# ----------------------------------------------------------------------------------------------
# single GPU
# ----------------------------------------------------------------------------------------------

def _forward_local(plan: CPPlan, q, k, v, scale):
    if attn_cuda.has_window(plan.segments):  # kWindow kernel variant with per-item trimmed tables
        return attn_cuda.segments_forward(plan, plan.segments, q, k, v, scale)
    items, segs, covered = attn_cuda.fwd_tables(plan, plan.segments, {plan.rank: 0}, q.device, ("local",))
    return attn_cuda.forward_launch(q, k, v, items, segs, covered, scale)


def _backward_local(plan: CPPlan, dout, q, k, v, out, lse, scale, deterministic=False):
    delta = attn_cuda.compute_delta(out, dout)
    dq = attn_cuda.dq_workspace.acquire(q)  # zeroed fp32 accumulator, re-zeroed by dq_finalize
    if attn_cuda.has_window(plan.segments):
        # windowed tables may leave key tiles without any query: start from zeros (model dtype)
        dk, dv = torch.zeros_like(k), torch.zeros_like(v)
        attn_cuda.segments_backward(plan, plan.segments, dout, q, k, v, lse, delta, scale, dq, dk, dv, deterministic)
    else:
        items, qsegs, *bounds = attn_cuda.bwd_tables(plan, plan.segments, {plan.rank: 0}, q.device, ("local",),
                                                     ordered=deterministic)
        # every key tile has exactly one writer and the epilogue stores the model dtype: no memset, no cast
        alloc = torch.empty_like if attn_cuda.bwd_tables_cover(plan, q.device, ("local",)) else torch.zeros_like
        dk, dv = alloc(k), alloc(v)
        attn_cuda.backward_launch(q, dout, k, v, lse, delta, items, qsegs, scale, dq, dk, dv,
                                  bounds[0] if bounds else None)
    return attn_cuda.dq_workspace.finalize(dq, q), dk, dv


def forward(plan: CPPlan, q, k, v, scale, group):
    if plan.world == 1:
        return _forward_local(plan, q, k, v, scale)
    from . import symm

    return symm.fused_forward(plan, q, k, v, scale, group)


def backward(plan: CPPlan, dout, q, k, v, out, lse, scale, group, deterministic=False):
    if plan.world == 1:
        return _backward_local(plan, dout, q, k, v, out, lse, scale, deterministic)
    from . import symm

    return symm.fused_backward(plan, dout, q, k, v, out, lse, scale, group, deterministic)
