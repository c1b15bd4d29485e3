"""Plan executors: run a :class:`~ring_flash_attn_b200.ops.plan.CPPlan` forward and backward.

Two transports, selected per call:

* ``fused``   - sm_90a kernels; the attention kernel's own communication CTAs push the K/V rows each
                peer needs into that peer's memory over NVLink, and the backward stores dK/dV partials
                straight into the owner's inbox (``parallel/fused.py`` / ``parallel/symm.py``).  Used
                whenever the tensors live on Hopper GPUs of one node with peer access.
* ``ring`` / ``allgather`` - torch.distributed fallback (gloo on CPU, NCCL on GPUs without peer
                access): the reference's own communication pattern
                (/root/reference/ring_flash_attn/ring_flash_attn.py:26-63,97-152 and
                llama3_flash_attn_varlen.py:89-158,218-297) around ``ops.dense`` blocks (CPU) or the
                single-GPU sm_90a kernel (CUDA).

All tensors here are token-major: q ``(Tq,Hq,D)``, k/v ``(Tk,Hkv,D)``, lse ``(Hq,Tq)`` fp32.
"""
from __future__ import annotations

import os
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist

from ..ops import dense
from ..ops.merge import merge_partial
from ..ops.plan import CPPlan, Segment
from .comm import AllGatherComm, RingComm


# ----------------------------------------------------------------------------------------------
# per-source block execution (one ring step / one gathered slab)
# ----------------------------------------------------------------------------------------------

def _use_cuda_kernels(q: torch.Tensor, k: Optional[torch.Tensor] = None) -> bool:
    """True when the sm_90a kernels handle this call (Hopper GPU, bf16/fp16, head_dim 128).

    Other CUDA inputs (e.g. head_dim 64) run the dense torch blocks on the GPU - slow but correct."""
    from ..ops import attn_cuda, cuda_ext

    if not cuda_ext.available_for(q):  # False for anything that is not a Hopper GPU tensor
        return False
    if attn_cuda.is_fp8_kernel_input(q, q if k is None else k):
        return attn_cuda.current_fp8_scales() is not None  # experimental fp8 forward (parallel/api.py)
    return attn_cuda.supported(q, q if k is None else k)


def plan_has_window(plan: CPPlan) -> bool:
    """Sliding-window plans carry a lower bound per segment."""
    cached = getattr(plan, "_has_window", None)
    if cached is None:
        cached = any(s.lo is not None for s in plan.segments)
        plan._has_window = cached
    return cached


def _kernels_take(plan: CPPlan) -> bool:
    """Windowed plans run on the kWindow kernel variants unless RFA_B200_WINDOW_KERNEL=0 (see
    ``ops/attn_cuda.py:window_kernels_enabled``); then on the dense torch blocks, on any device."""
    if not plan_has_window(plan):
        return True
    from ..ops import attn_cuda

    if attn_cuda.window_kernels_enabled():
        return True
    _warn_once("RFA_B200_WINDOW_KERNEL=0: sliding-window plans run on the dense torch blocks (slow)")
    return False


def _dense_tiles(row0: int, n_rows: int, s: Segment):
    """Cut one (chunk x segment) block of the dense torch path into sub-blocks whose fp32 score matrix stays
    small (``RFA_B200_DENSE_TILE`` query rows x 4x as many keys, default 1024 x 4096), so that the fallback for
    shapes the kernels do not cover is slow but never allocates an S x S matrix.  Yields
    (query rows, key rows, diag, lo) with the band offsets re-based to the sub-block; sub-blocks that lie
    entirely outside the band are skipped."""
    tq = max(1, int(os.environ.get("RFA_B200_DENSE_TILE", "1024")))
    tk = 4 * tq
    for oq in range(0, n_rows, tq):
        nq = min(tq, n_rows - oq)
        for ok in range(0, s.kv_len, tk):
            nk = min(tk, s.kv_len - ok)
            diag = None if s.diag is None else s.diag + oq - ok
            lo = None if s.lo is None else s.lo + oq - ok
            if diag is not None and diag + nq - 1 < 0:
                continue  # even the last query row ends in front of this key block
            if lo is not None and lo > nk - 1:
                continue  # even the first query row starts behind it
            yield (slice(row0 + oq, row0 + oq + nq), slice(s.kv_row0 + ok, s.kv_row0 + ok + nk), diag, lo)


def step_forward(plan: CPPlan, segs: List[Segment], q, k_src, v_src, scale, out, lse):
    """Fold the contribution of one source shard into the running (out, lse)."""
    if not segs:
        return out, lse
    if _use_cuda_kernels(q, k_src) and _kernels_take(plan):
        from ..ops import attn_cuda

        sc = attn_cuda.current_fp8_scales()
        if sc is not None and sc.world_rows:  # fp8: this launch reads source `src`'s rows as a local tensor
            with attn_cuda.fp8_scales(sc.for_source(segs[0].src)):
                p_out, p_lse = attn_cuda.segments_forward(plan, segs, q, k_src, v_src, scale)
        else:
            p_out, p_lse = attn_cuda.segments_forward(plan, segs, q, k_src, v_src, scale)
        return merge_partial(out, lse, p_out, p_lse)
    if out is None:
        out = torch.zeros(q.shape, dtype=torch.float32, device=q.device)
        lse = torch.full((q.shape[1], q.shape[0]), float("-inf"), dtype=torch.float32, device=q.device)
    for s in segs:
        ch = plan.q_chunks[s.chunk]
        for rows, kv, diag, lo in _dense_tiles(ch.row0, ch.rows, s):
            b_out, b_lse = dense.block_fwd(q[rows], k_src[kv], v_src[kv], scale, diag, lo)
            merge_partial(out, lse, b_out, b_lse, rows)
    return out, lse


def step_backward(plan: CPPlan, segs: List[Segment], dout, q, k_src, v_src, lse, delta, scale,
                  dq, deterministic: bool = False):
    """dq += (local); returns fp32 (dk, dv) of this source shard's rows (zeros where unseen)."""
    dk = torch.zeros(k_src.shape, dtype=torch.float32, device=q.device)
    dv = torch.zeros(v_src.shape, dtype=torch.float32, device=q.device)
    if not segs:
        return dk, dv
    if _use_cuda_kernels(q, k_src) and _kernels_take(plan):
        from ..ops import attn_cuda

        attn_cuda.segments_backward(plan, segs, dout, q, k_src, v_src, lse, delta, scale, dq, dk, dv,
                                    deterministic)
        return dk, dv
    for s in segs:
        ch = plan.q_chunks[s.chunk]
        for rows, kv, diag, lo in _dense_tiles(ch.row0, ch.rows, s):
            b_dq, b_dk, b_dv = dense.block_bwd(dout[rows], q[rows], k_src[kv], v_src[kv], lse[:, rows],
                                               delta[:, rows], scale, diag, lo)
            dq[rows] += b_dq
            dk[kv] += b_dk
            dv[kv] += b_dv
    return dk, dv


def _out_dtype(q: torch.Tensor) -> torch.dtype:
    return torch.bfloat16 if q.element_size() == 1 else q.dtype  # fp8 inputs produce bf16 outputs


def _finish_forward(q, out, lse):
    if out is None:  # nothing visible at all (cannot happen for valid plans, but stay total)
        out = torch.zeros(q.shape, dtype=torch.float32, device=q.device)
        lse = torch.full((q.shape[1], q.shape[0]), float("-inf"), dtype=torch.float32, device=q.device)
    return out.to(_out_dtype(q)), lse


def compute_delta(out: torch.Tensor, dout: torch.Tensor) -> torch.Tensor:
    """delta[h, t] = sum_d out[t,h,d] * dout[t,h,d]  (fp32, (H,T))."""
    return (out.float() * dout.float()).sum(-1).transpose(0, 1).contiguous()


# ----------------------------------------------------------------------------------------------
# ring transport (reference pattern: K/V hop to the next rank every step; dK/dV travel with them)
# ----------------------------------------------------------------------------------------------

def ring_forward(plan: CPPlan, q, k, v, scale, group) -> Tuple[torch.Tensor, torch.Tensor]:
    comm = RingComm(group)
    by_src = plan.by_src()
    out = lse = None
    cur_k, cur_v = k.contiguous(), v.contiguous()
    for step in range(plan.world):
        src = (plan.rank - step) % plan.world
        last = step + 1 == plan.world
        if not last:
            nxt_k, nxt_v = comm.send_recv_kv(cur_k, cur_v)
        out, lse = step_forward(plan, by_src.get(src, []), q, cur_k, cur_v, scale, out, lse)
        if not last:
            comm.wait()
            cur_k, cur_v = nxt_k, nxt_v
    return _finish_forward(q, out, lse)


def ring_backward(plan: CPPlan, dout, q, k, v, out, lse, scale, group, deterministic=False):
    kv_comm, dkv_comm = RingComm(group), RingComm(group)
    by_src = plan.by_src()
    delta = compute_delta(out, dout)
    dq = torch.zeros(q.shape, dtype=torch.float32, device=q.device)
    cur_k, cur_v = k.contiguous(), v.contiguous()
    dk = dv = nxt_dk = nxt_dv = None
    for step in range(plan.world):
        src = (plan.rank - step) % plan.world
        last = step + 1 == plan.world
        if not last:
            nxt_k, nxt_v = kv_comm.send_recv_kv(cur_k, cur_v)
        b_dk, b_dv = step_backward(plan, by_src.get(src, []), dout, q, cur_k, cur_v, lse, delta, scale,
                                   dq, deterministic)
        if step == 0:
            dk, dv = b_dk, b_dv
        else:
            dkv_comm.wait()  # accumulator of shard `src` arriving from the previous rank
            dk, dv = nxt_dk + b_dk, nxt_dv + b_dv
        if not last:
            kv_comm.wait()
            cur_k, cur_v = nxt_k, nxt_v
        nxt_dk, nxt_dv = dkv_comm.send_recv_kv(dk, dv)
    dkv_comm.wait()  # one extra hop brings every accumulator home
    return dq.to(q.dtype), nxt_dk.to(k.dtype), nxt_dv.to(v.dtype)


# ----------------------------------------------------------------------------------------------
# all-gather transport (llama3 pattern: gather a group of kv heads, attend, reduce-scatter grads)
# ----------------------------------------------------------------------------------------------

def _head_group_scales(q_heads: slice, kv_heads: slice):
    """fp8 forward: a launch over a group of heads indexes its descales by LOCAL head."""
    from ..ops import attn_cuda

    scales = attn_cuda.current_fp8_scales()
    if scales is None:
        import contextlib

        return contextlib.nullcontext()
    return attn_cuda.fp8_scales(scales.heads(q_heads, kv_heads))


def _head_groups(hkv: int, stride: int):
    if hkv % stride:
        raise ValueError(f"heads_k_stride={stride} must divide the number of kv heads ({hkv})")
    return range(0, hkv, stride)


def _gather_heads(comm: AllGatherComm, k, v, h0, stride, buf):
    comm.all_gather(buf[0], k[:, h0:h0 + stride].contiguous())
    comm.all_gather(buf[1], v[:, h0:h0 + stride].contiguous())


def allgather_forward(plan: CPPlan, q, k, v, scale, group, heads_k_stride: int):
    W, L = plan.world, plan.kv_rows
    hq, hkv, d = q.shape[1], k.shape[1], k.shape[2]
    rep = hq // hkv
    comm = AllGatherComm(group)
    by_src = plan.by_src()
    bufs = [torch.empty((2, W * L, heads_k_stride, d), dtype=k.dtype, device=k.device) for _ in range(2)]
    out = torch.empty(q.shape, dtype=_out_dtype(q), device=q.device)
    lse = torch.empty((hq, q.shape[0]), dtype=torch.float32, device=q.device)
    groups = list(_head_groups(hkv, heads_k_stride))
    _gather_heads(comm, k, v, groups[0], heads_k_stride, bufs[0])
    for gi, h0 in enumerate(groups):
        comm.wait()
        cur = bufs[gi % 2]
        if gi + 1 < len(groups):  # double buffering: next group's gather overlaps this group's math
            _gather_heads(comm, k, v, groups[gi + 1], heads_k_stride, bufs[(gi + 1) % 2])
        qs = slice(h0 * rep, (h0 + heads_k_stride) * rep)
        q_g = q[:, qs]
        o_g = l_g = None
        with _head_group_scales(qs, slice(h0, h0 + heads_k_stride)):
            for src in range(W):
                o_g, l_g = step_forward(plan, by_src.get(src, []), q_g, cur[0, src * L:(src + 1) * L],
                                        cur[1, src * L:(src + 1) * L], scale, o_g, l_g)
        o_g, l_g = _finish_forward(q_g, o_g, l_g)
        out[:, qs] = o_g
        lse[qs] = l_g
    return out, lse


def allgather_backward(plan: CPPlan, dout, q, k, v, out, lse, scale, group, heads_k_stride: int,
                       deterministic=False):
    W, L = plan.world, plan.kv_rows
    hq, hkv, d = q.shape[1], k.shape[1], k.shape[2]
    rep = hq // hkv
    comm = AllGatherComm(group)
    by_src = plan.by_src()
    delta = compute_delta(out, dout)
    bufs = [torch.empty((2, W * L, heads_k_stride, d), dtype=k.dtype, device=k.device) for _ in range(2)]
    dq = torch.zeros(q.shape, dtype=torch.float32, device=q.device)
    dk = torch.empty(k.shape, dtype=k.dtype, device=k.device)
    dv = torch.empty(v.shape, dtype=v.dtype, device=v.device)
    groups = list(_head_groups(hkv, heads_k_stride))
    _gather_heads(comm, k, v, groups[0], heads_k_stride, bufs[0])
    for gi, h0 in enumerate(groups):
        comm.wait()
        cur = bufs[gi % 2]
        if gi + 1 < len(groups):
            _gather_heads(comm, k, v, groups[gi + 1], heads_k_stride, bufs[(gi + 1) % 2])
        qs = slice(h0 * rep, (h0 + heads_k_stride) * rep)
        dq_g = torch.zeros(q[:, qs].shape, dtype=torch.float32, device=q.device)
        dkv_full = torch.zeros((2, W * L, heads_k_stride, d), dtype=torch.float32, device=q.device)
        for src in range(W):
            sl = slice(src * L, (src + 1) * L)
            b_dk, b_dv = step_backward(plan, by_src.get(src, []), dout[:, qs], q[:, qs], cur[0, sl],
                                       cur[1, sl], lse[qs], delta[qs], scale, dq_g, deterministic)
            dkv_full[0, sl] = b_dk
            dkv_full[1, sl] = b_dv
        dq[:, qs] = dq_g
        if W > 1:
            red = torch.empty((2, L, heads_k_stride, d), dtype=torch.float32, device=q.device)
            dist.reduce_scatter_tensor(red[0], dkv_full[0], group=group)
            dist.reduce_scatter_tensor(red[1], dkv_full[1], group=group)
        else:
            red = dkv_full
        dk[:, h0:h0 + heads_k_stride] = red[0].to(k.dtype)
        dv[:, h0:h0 + heads_k_stride] = red[1].to(v.dtype)
    return dq.to(q.dtype), dk, dv


# ----------------------------------------------------------------------------------------------
# entry points used by the autograd bridge
# ----------------------------------------------------------------------------------------------

def _fused_ok(q: torch.Tensor, k: torch.Tensor, group, plan=None) -> bool:
    if not _use_cuda_kernels(q, k):
        return False
    if q.element_size() == 1 and os.environ.get("RFA_B200_FP8_KERNEL", "2") == "1":
        return False  # =1: fp8 kernel on the per-source transports only (e4m3 over NCCL), not inside the fused launch
    if plan is not None and not _kernels_take(plan):
        return False
    from . import fused

    if not fused.available(q, group):
        return False
    if plan is not None and plan.world > 1:
        from . import symm

        if symm.is_dynamic(plan) and not symm.dynamic_ok(plan):
            _warn_once("plan reads more than %d separate row ranges of one source shard: using the "
                       "torch.distributed transport instead of the fused NVLink path" % symm.NEED_RANGES)
            return False
    return True


_WARNED = set()


def _warn_once(msg: str) -> None:
    """Falling off the fused path is a performance cliff: say so, once per distinct reason."""
    if msg not in _WARNED:
        _WARNED.add(msg)
        import warnings

        warnings.warn("ring_flash_attn_b200: " + msg, RuntimeWarning, stacklevel=3)


def fused_heads_per_pass(plan: CPPlan, k: torch.Tensor, heads_k_stride: int, strict_env: bool = True) -> int:
    """How many kv heads one fused launch covers.

    The reference gathers ``heads_k_stride`` kv heads at a time so that the gathered K/V buffer stays bounded
    (/root/reference/ring_flash_attn/llama3_flash_attn_varlen.py:89-115), and its ring schemes hold one K/V shard in
    flight (utils.py:117).  On the fused path the quantity that grows with the number of heads is the peer-mapped
    staging buffer (every source's rows x heads, two call parities), so ``heads_k_stride`` is the granularity and
    ``RFA_B200_STAGE_BUDGET_MB`` (default 8192) the cap: as many multiples of ``heads_k_stride`` heads per launch as
    fit the budget - all of them when memory allows, because one launch over all heads is the fastest schedule.
    ``RFA_B200_LLAMA3_HEAD_GROUPS=strict`` (llama3 only, ``strict_env``) uses exactly ``heads_k_stride`` heads per
    launch (the reference's memory behaviour)."""
    hkv = k.shape[1]
    stride = max(1, min(int(heads_k_stride), hkv))
    if hkv % stride:
        raise ValueError(f"heads_k_stride={stride} must divide the number of kv heads ({hkv})")
    if strict_env and os.environ.get("RFA_B200_LLAMA3_HEAD_GROUPS", "auto") == "strict":
        return stride
    budget = int(os.environ.get("RFA_B200_STAGE_BUDGET_MB", "8192")) << 20
    per_head = 2 * 2 * plan.world * plan.kv_rows * k.shape[2] * k.element_size()  # parities x (K, V) x sources x rows
    g = hkv
    while g > stride and g * per_head > budget:
        g -= stride
        while g > stride and hkv % g:
            g -= stride
    return g


def _fused_by_head_groups(plan, k, heads_k_stride, transport):
    """(heads per pass) when the fused path must run in several passes over kv-head groups, else None.

    llama3 (``allgather`` transport): granularity ``heads_k_stride``.  Ring / zigzag / stripe schemes: granularity
    one kv head, only when the staging of all heads would exceed ``RFA_B200_STAGE_BUDGET_MB`` - per-GPU staging is
    then O(S * g / Hkv) for g heads per pass instead of O(S)."""
    if plan.world == 1:
        return None
    if transport == "allgather":
        g = fused_heads_per_pass(plan, k, heads_k_stride)
    else:
        g = fused_heads_per_pass(plan, k, 1, strict_env=False)
    return g if g < k.shape[1] else None


def cp_forward(plan: CPPlan, q, k, v, scale, group, transport="ring", heads_k_stride: int = 1):
    if plan.world > 1 and _use_cuda_kernels(q, k):
        from ..ops import attn_cuda

        sc = attn_cuda.current_fp8_scales()
        if sc is not None and not sc.world_rows:
            # fp8: every transport reads remote K/V rows, so it needs their descales too (tables of all shards)
            with attn_cuda.fp8_scales(sc.gathered(group, plan.rank, plan.world, plan.kv_rows)):
                return cp_forward(plan, q, k, v, scale, group, transport, heads_k_stride)
    if _fused_ok(q, k, group, plan):
        from . import fused

        g = _fused_by_head_groups(plan, k, heads_k_stride, transport)
        if g is None:
            return fused.forward(plan, q, k, v, scale, group)
        rep = q.shape[1] // k.shape[1]
        outs, lses = [], []
        for h0 in range(0, k.shape[1], g):  # one fused launch per group of kv heads: staging holds g heads only
            qs = slice(h0 * rep, (h0 + g) * rep)
            with _head_group_scales(qs, slice(h0, h0 + g)):
                o, l = fused.forward(plan, q[:, qs], k[:, h0:h0 + g], v[:, h0:h0 + g], scale, group)
            outs.append(o)
            lses.append(l)
        return torch.cat(outs, dim=1), torch.cat(lses, dim=0)
    if transport == "allgather":
        return allgather_forward(plan, q, k, v, scale, group, heads_k_stride)
    return ring_forward(plan, q, k, v, scale, group)


def deterministic_mode() -> str:
    """``RFA_B200_DETERMINISTIC``: ``strict`` (default) - ``deterministic=True`` makes out / lse / dQ / dK / dV bitwise
    reproducible; ``fast`` - keep the fastest schedule (dK / dV reproducible, dQ summed in no fixed order)."""
    return os.environ.get("RFA_B200_DETERMINISTIC", "strict")


def cp_backward(plan: CPPlan, dout, q, k, v, out, lse, scale, group, transport="ring",
                heads_k_stride: int = 1, deterministic: bool = False):
    # The reference forwards the flag to flash-attn's backward (ring_flash_attn.py:119).  On the sm_90a path out / lse
    # never depend on timing, dK / dV have one writer per tile and a fixed-order owner-side sum; dQ tiles are added
    # with unordered fp32 L2 reductions.  ``ordered``: launch the key tiles in groups with disjoint query rows
    # (ops/attn_cuda.py:ordered_dq_groups) and, across GPUs, move K/V and dK/dV with the fixed-order ring /
    # all-gather transports instead of the fused launch (whose key tiles of all sources share one launch).
    kernels = _use_cuda_kernels(q, k) and _kernels_take(plan)
    ordered = bool(deterministic) and kernels and deterministic_mode() != "fast"
    if ordered:
        _warn_once("deterministic=True: the backward runs one launch per group of key tiles with disjoint query rows"
                   + (" and uses the torch.distributed transport instead of the fused NVLink path"
                      if plan.world > 1 else "") +
                   " (bitwise reproducible dQ / dK / dV, several times slower; RFA_B200_DETERMINISTIC=fast keeps "
                   "the fast schedule with reproducible dK / dV and an unordered fp32 sum for dQ)")
    elif deterministic and kernels:
        _warn_once("deterministic=True with RFA_B200_DETERMINISTIC=fast: dK / dV are bitwise reproducible, dQ is "
                   "accumulated with fp32 reductions whose order is not fixed (run-to-run differences of ~1 ulp of fp32)")
    if _fused_ok(q, k, group, plan) and not (ordered and plan.world > 1):
        from . import fused

        g = _fused_by_head_groups(plan, k, heads_k_stride, transport)
        if g is None:
            return fused.backward(plan, dout, q, k, v, out, lse, scale, group, ordered)
        rep = q.shape[1] // k.shape[1]
        dqs, dks, dvs = [], [], []
        for h0 in range(0, k.shape[1], g):
            qs = slice(h0 * rep, (h0 + g) * rep)
            dq_g, dk_g, dv_g = fused.backward(plan, dout[:, qs], q[:, qs], k[:, h0:h0 + g], v[:, h0:h0 + g],
                                              out[:, qs], lse[qs], scale, group, ordered)
            dqs.append(dq_g)
            dks.append(dk_g)
            dvs.append(dv_g)
        return torch.cat(dqs, dim=1), torch.cat(dks, dim=1), torch.cat(dvs, dim=1)
    if transport == "allgather":
        return allgather_backward(plan, dout, q, k, v, out, lse, scale, group, heads_k_stride, ordered)
    return ring_backward(plan, dout, q, k, v, out, lse, scale, group, ordered)
