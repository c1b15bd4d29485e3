"""Python side of the sm_90a attention kernels: plan -> device work tables -> launches.

The kernels (``csrc/attn_fwd_sm90.cu`` / ``attn_bwd_sm90.cu``) consume a :class:`CPPlan` as two small
int32 tables.  Tables are cached on the plan object (plans themselves are lru-cached per shape), so the
steady state of a training loop performs no host work beyond the launches.

The launches stand where the reference calls flash-attn's private ops
(``_flash_attn_forward`` / ``_flash_attn_backward`` and their varlen forms,
/root/reference/ring_flash_attn/ring_flash_attn.py:53,131, ring_flash_attn_varlen.py:77,169,
llama3_flash_attn_varlen.py:147,282); what the reference expresses as per-step slicing of q / k / v / lse
(zigzag_ring_flash_attn.py:60-84, zigzag_ring_flash_attn_varlen.py:24-71) is a row of the work table here.
"""
from __future__ import annotations

import contextlib
import threading
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import cuda_ext
from .plan import CPPlan, Segment

DIAG_FULL = 1 << 29
Q_ITEM_ROWS = 128  # rows per forward CTA (two 64-row wgmma tiles)
K_TILE_ROWS = 128  # keys per backward CTA


KERNEL_HEAD_DIMS = (64, 128)  # instantiations of both kernels (template parameter kD)


def supported(q: torch.Tensor, k: torch.Tensor) -> bool:
    return q.shape[-1] in KERNEL_HEAD_DIMS and q.dtype in (torch.bfloat16, torch.float16) and k.dtype == q.dtype


def _diag(d: Optional[int]) -> int:
    return DIAG_FULL if d is None else int(d)


# ---- fp8 forward (e4m3 q / k / v with block descales; RFA_B200_FP8_KERNEL=0 disables) -------------------
# The descales of the running call; set by parallel/ops.py around the engine call so that the executors (which
# only know q / k / v) can hand them to the launch.
_FP8_STATE = threading.local()


class Fp8Scales:
    """Block descales in the form the forward kernel reads (csrc/attn_common.h: FwdParams::q_scale ...).

    ``q``: (ceil(Tq / q_block), Hq) fp32, one per ``q_block`` consecutive token-major query rows and head.
    ``k`` / ``v``: (n, Hkv) fp32, one per ``kv_block`` consecutive key rows and kv head, covering either this rank's
    shard (``world_rows == 0``) or every rank's shard back to back (``world_rows`` = rows per shard; produced by
    :meth:`gathered`), exactly like the staging buffer.  ``v_ref``: (Hkv,) the largest V descale of each head."""

    def __init__(self, q, q_block, k, v, kv_block, v_ref=None, world_rows=0, kv_row0=0):
        self.q, self.q_block, self.k, self.v, self.kv_block = q, int(q_block), k, v, int(kv_block)
        self.v_ref = v.amax(dim=0).contiguous() if v_ref is None else v_ref
        self.world_rows, self.kv_row0 = int(world_rows), int(kv_row0)

    def gathered(self, group, rank: int, world: int, rows: int) -> "Fp8Scales":
        """Tables of every rank's shard (two tiny all-gathers + one all-reduce on the current stream)."""
        import torch.distributed as dist

        if world == 1 or self.world_rows:
            return self
        if rows % self.kv_block and self.k.shape[0] != 1:
            raise ValueError("k / v descale blocks must tile the local shard")
        nb = self.k.shape[0]
        k_all = torch.empty((world * nb, self.k.shape[1]), dtype=torch.float32, device=self.k.device)
        v_all = torch.empty_like(k_all)
        dist.all_gather_into_tensor(k_all, self.k.contiguous(), group=group)
        dist.all_gather_into_tensor(v_all, self.v.contiguous(), group=group)
        v_ref = self.v_ref.clone()
        dist.all_reduce(v_ref, op=dist.ReduceOp.MAX, group=group)
        kv_block = rows if nb == 1 else self.kv_block
        return Fp8Scales(self.q, self.q_block, k_all, v_all, kv_block, v_ref, world_rows=rows, kv_row0=rank * rows)

    def for_source(self, src: int) -> "Fp8Scales":
        """Per-source launches of the torch.distributed transports read source ``src``'s K/V as a local tensor."""
        if not self.world_rows:
            return self
        return Fp8Scales(self.q, self.q_block, self.k, self.v, self.kv_block, self.v_ref, self.world_rows,
                         kv_row0=src * self.world_rows)

    def heads(self, q_heads: slice, kv_heads: slice) -> "Fp8Scales":
        return Fp8Scales(self.q[:, q_heads].contiguous(), self.q_block, self.k[:, kv_heads].contiguous(),
                         self.v[:, kv_heads].contiguous(), self.kv_block, self.v_ref[kv_heads].contiguous(),
                         self.world_rows, self.kv_row0)

    def args(self):
        return (self.q, self.q_block, self.k, self.v, self.kv_block, self.v_ref, self.kv_row0)


@contextlib.contextmanager
def fp8_scales(scales: "Fp8Scales"):
    prev = getattr(_FP8_STATE, "scales", None)
    _FP8_STATE.scales = scales
    try:
        yield
    finally:
        _FP8_STATE.scales = prev


def current_fp8_scales() -> Optional["Fp8Scales"]:
    return getattr(_FP8_STATE, "scales", None)


def is_fp8_kernel_input(q: torch.Tensor, k: torch.Tensor) -> bool:
    return q.dtype == torch.float8_e4m3fn and k.dtype == torch.float8_e4m3fn and q.shape[-1] == 128


def out_dtype(q: torch.Tensor) -> torch.dtype:
    """fp8 inputs produce bf16 outputs."""
    return torch.bfloat16 if q.element_size() == 1 else q.dtype


LO_NONE = -(1 << 29)  # "no lower bound" in the sliding-window tables


def has_window(segs: Sequence[Segment]) -> bool:
    return any(s.lo is not None for s in segs)


def window_kernels_enabled() -> bool:
    """Sliding-window plans run on the kWindow kernel variants.  ``RFA_B200_WINDOW_KERNEL=0`` forces the dense torch
    blocks (``parallel/engine.py``) for debugging."""
    import os

    return os.environ.get("RFA_B200_WINDOW_KERNEL", "1") != "0"


# ----------------------------------------------------------------------------------------------
# forward tables
# ----------------------------------------------------------------------------------------------

def fwd_tables_host(plan: CPPlan, segs: Sequence[Segment], row_offset: Dict[int, int],
                    flag_of_src: Optional[Dict[int, int]] = None) -> Tuple[List[List[int]], List[List[int]], bool]:
    """(items, segments, all_chunks_covered).  ``row_offset[src]`` is where source ``src``'s shard
    starts inside the K/V tensor handed to the launch; ``flag_of_src`` (fused mode) maps a source to
    the ready flag the loader must wait on."""
    by_chunk: Dict[int, List[Segment]] = {}
    for s in segs:
        by_chunk.setdefault(s.chunk, []).append(s)
    items, seg_rows = [], []
    for ci, ch in enumerate(plan.q_chunks):
        cs = by_chunk.get(ci)
        if not cs or ch.rows == 0:
            continue
        begin = len(seg_rows)
        for s in cs:
            flag = -1 if flag_of_src is None else flag_of_src.get(s.src, -1)
            seg_rows.append([row_offset[s.src] + s.kv_row0, s.kv_len, _diag(s.diag), flag])
        for off in range(0, ch.rows, Q_ITEM_ROWS):
            rows = min(Q_ITEM_ROWS, ch.rows - off)
            work = 0
            for s in cs:
                d = _diag(s.diag)
                work += max(0, min(s.kv_len, off + rows + d))
            items.append((work, [ch.row0 + off, rows, off, begin, len(cs), 0, 0, 0]))
    items.sort(key=lambda t: -t[0])  # heaviest first
    covered = all((ci in by_chunk) or ch.rows == 0 for ci, ch in enumerate(plan.q_chunks))
    return [it for _, it in items], seg_rows, covered


def fwd_tables_window_host(plan: CPPlan, segs: Sequence[Segment], row_offset: Dict[int, int],
                           flag_of_src: Optional[Dict[int, int]] = None):
    """Forward tables for sliding-window plans: (items, segments, seg_lo, all_rows_covered).

    Key j of a segment is visible to chunk row i iff ``i + lo <= j <= i + diag``.  Every work item (128 query
    rows starting at chunk row ``off``) gets its OWN copy of each segment, trimmed at the front to the first key
    its first row can see (``off + lo``): the kernel's key loop then still starts at tile 0 and only has to mask
    the slanted lower edge, for which ``seg_lo`` carries the re-based offset."""
    by_chunk: Dict[int, List[Segment]] = {}
    for s in segs:
        by_chunk.setdefault(s.chunk, []).append(s)
    items, seg_rows, seg_lo = [], [], []
    covered = True
    for ci, ch in enumerate(plan.q_chunks):
        if ch.rows == 0:
            continue
        cs = by_chunk.get(ci)
        if not cs:
            covered = False
            continue
        for off in range(0, ch.rows, Q_ITEM_ROWS):
            rows = min(Q_ITEM_ROWS, ch.rows - off)
            begin = len(seg_rows)
            work = 0
            for s in cs:
                j_min = 0 if s.lo is None else max(0, off + s.lo)
                if j_min >= s.kv_len:
                    continue  # even the first row's window starts behind the last key
                if s.diag is not None and off + rows - 1 + s.diag < j_min:
                    continue  # even the last row ends in front of the first key
                d = DIAG_FULL if s.diag is None else s.diag - j_min
                flag = -1 if flag_of_src is None else flag_of_src.get(s.src, -1)
                seg_rows.append([row_offset[s.src] + s.kv_row0 + j_min, s.kv_len - j_min, d, flag])
                seg_lo.append(LO_NONE if s.lo is None else s.lo - j_min)
                work += max(0, min(s.kv_len - j_min, off + rows + d))
            if len(seg_rows) == begin:
                covered = False  # nothing visible: out / lse of these rows keep their initial 0 / -inf
                continue
            items.append((work, [ch.row0 + off, rows, off, begin, len(seg_rows) - begin, 0, 0, 0]))
    items.sort(key=lambda t: -t[0])
    return [it for _, it in items], seg_rows, seg_lo, covered


def bwd_tables_window_host(plan: CPPlan, segs: Sequence[Segment], row_offset: Dict[int, int],
                           flag_of_src: Optional[Dict[int, int]] = None, fused: bool = False):
    """Backward tables for sliding-window plans.  Same exclusive key tiles as :func:`bwd_tables_host`; a query
    segment additionally carries ``lo`` (re-based to the tile's first key) and its length is cut behind the last
    chunk row that can still see the tile's last key.

    ``fused=True`` follows :func:`bwd_tables_fused`: items carry owner / row-in-owner-shard, are emitted in ring
    order, tiles without any query segment are kept (they store zeros into the owner's inbox), and the third
    return value counts the tiles per owner."""
    by_src: Dict[int, List[Segment]] = {}
    for s in segs:
        by_src.setdefault(s.src, []).append(s)
    items, qsegs = [], []
    per_owner = [0] * plan.world
    for src, ss in by_src.items():
        cuts = sorted({s.kv_row0 for s in ss} | {s.kv_row0 + s.kv_len for s in ss})
        for lo_cut, hi_cut in zip(cuts[:-1], cuts[1:]):
            cover = [s for s in ss if s.kv_row0 <= lo_cut and s.kv_row0 + s.kv_len >= hi_cut]
            for t0 in range(lo_cut, hi_cut, K_TILE_ROWS) if cover else ():
                rows = min(K_TILE_ROWS, hi_cut - t0)
                begin = len(qsegs)
                work = 0
                for s in cover:
                    ch = plan.q_chunks[s.chunk]
                    shift = t0 - s.kv_row0
                    d = DIAG_FULL if s.diag is None else s.diag - shift
                    q_len = ch.rows
                    lo = LO_NONE
                    if s.lo is not None:
                        lo = s.lo - shift
                        q_len = min(q_len, rows - lo)  # chunk row i sees tile key j iff i <= j - lo <= rows - 1 - lo
                    first = max(0, -d)  # first chunk row that sees tile key 0
                    if q_len <= 0 or first >= q_len:
                        continue
                    qsegs.append([ch.row0, q_len, d, lo])
                    work += q_len - first
                flag = -1 if flag_of_src is None else flag_of_src.get(src, -1)
                if fused:
                    step = (plan.rank - src) % plan.world
                    items.append(((step, -work), [row_offset[src] + t0, rows, begin, len(qsegs) - begin, flag, src, t0, 0]))
                    per_owner[src] += 1
                elif len(qsegs) > begin:
                    items.append(((0, -work), [row_offset[src] + t0, rows, begin, len(qsegs) - begin, flag, 0, 0, 0]))
    items.sort(key=lambda t: t[0])
    if fused:
        return [it for _, it in items], qsegs, per_owner
    return [it for _, it in items], qsegs


def bwd_tables_host(plan: CPPlan, segs: Sequence[Segment], row_offset: Dict[int, int],
                    flag_of_src: Optional[Dict[int, int]] = None):
    """Backward tables: key tiles that exclusively own their dK/dV rows + the query chunks that see them."""
    by_src: Dict[int, List[Segment]] = {}
    for s in segs:
        by_src.setdefault(s.src, []).append(s)
    items, qsegs = [], []
    for src, ss in by_src.items():
        cuts = sorted({s.kv_row0 for s in ss} | {s.kv_row0 + s.kv_len for s in ss})
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            cover = [s for s in ss if s.kv_row0 <= lo and s.kv_row0 + s.kv_len >= hi]
            if not cover:
                continue
            for t0 in range(lo, hi, K_TILE_ROWS):
                rows = min(K_TILE_ROWS, hi - t0)
                begin = len(qsegs)
                work = 0
                for s in cover:
                    ch = plan.q_chunks[s.chunk]
                    d = DIAG_FULL if s.diag is None else s.diag - (t0 - s.kv_row0)
                    if ch.rows - 1 + d < 0:
                        continue  # no query of this chunk reaches the tile
                    qsegs.append([ch.row0, ch.rows, d, 0])
                    work += ch.rows - max(0, -d)
                if len(qsegs) == begin:
                    continue
                flag = -1 if flag_of_src is None else flag_of_src.get(src, -1)
                items.append((work, [row_offset[src] + t0, rows, begin, len(qsegs) - begin, flag, 0, 0, 0]))
    items.sort(key=lambda t: -t[0])
    return [it for _, it in items], qsegs


def bwd_covers_all_rows(items: List[List[int]], kv_rows: int) -> bool:
    """True when the (exclusive) key tiles of a backward table write every one of ``kv_rows`` dK/dV rows."""
    return sum(it[1] for it in items) == kv_rows


def ordered_dq_groups(items: List[List[int]], qsegs: List[List[int]]) -> Tuple[List[List[int]], List[int]]:
    """Reorder a backward item table into LAUNCH GROUPS for a bitwise reproducible dQ.

    A key-tile CTA adds its dQ^T partial tiles into the fp32 accumulator with unordered L2 reductions, so two key
    tiles that reach the same query rows inside one launch make the rounding of dQ depend on timing.  Items of one
    group reach pairwise disjoint query rows (all heads of an item run in the same launch: heads never share dQ
    elements); the groups are launched one after the other on the stream, which fixes the order of the fp32 additions
    of every dQ element to the group order.  Greedy first-fit in table order (heaviest tiles first).  Returns
    (items in group order, group boundaries ``[0, n_0, n_0 + n_1, ...]``).

    One causal sequence of T keys needs T / 128 groups (every key tile reaches the last query row), packed documents
    run side by side.  This is the cost of ``deterministic=True`` (the reference forwards the flag to flash-attn's
    backward, /root/reference/ring_flash_attn/ring_flash_attn.py:119, which serialises its dQ accumulation too)."""
    groups: List[Tuple[List[int], List[Tuple[int, int]]]] = []  # (item indices, query-row intervals they reach)
    for idx, it in enumerate(items):
        spans = []
        for q_row0, q_len, d, _lo in qsegs[it[2]:it[2] + it[3]]:
            first = max(0, -d)  # first chunk row that sees key 0 of the tile
            if first < q_len:
                spans.append((q_row0 + first, q_row0 + q_len))
        for members, taken in groups:
            if all(a1 <= b0 or b1 <= a0 for a0, a1 in spans for b0, b1 in taken):
                members.append(idx)
                taken.extend(spans)
                break
        else:
            groups.append(([idx], list(spans)))
    order, bounds = [], [0]
    for members, _ in groups:
        order.extend(members)
        bounds.append(len(order))
    return [items[i] for i in order], bounds


def bwd_tables_fused(plan: CPPlan, row_offset: Dict[int, int], device, flag_of_src: Dict[int, int]):
    """Backward tables for the fused multi-GPU launch: every key tile carries its owner rank and its row
    inside the owner's shard; tiles that no local query reaches are still emitted (they store zeros into
    the owner's inbox so that the owner-side reduction never reads stale memory).  Cached on the plan."""
    c = _cache(plan)
    key = ("bwd_fused", device.index)
    if key in c:
        return c[key]
    by_src: Dict[int, List[Segment]] = {}
    for s in plan.segments:
        by_src.setdefault(s.src, []).append(s)
    items, qsegs = [], []
    per_owner = [0] * plan.world
    for src, ss in by_src.items():
        cuts = sorted({s.kv_row0 for s in ss} | {s.kv_row0 + s.kv_len for s in ss})
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            cover = [s for s in ss if s.kv_row0 <= lo and s.kv_row0 + s.kv_len >= hi]
            if not cover:
                continue
            for t0 in range(lo, hi, K_TILE_ROWS):
                rows = min(K_TILE_ROWS, hi - t0)
                begin = len(qsegs)
                work = 0
                for s in cover:
                    ch = plan.q_chunks[s.chunk]
                    d = DIAG_FULL if s.diag is None else s.diag - (t0 - s.kv_row0)
                    if ch.rows - 1 + d < 0:
                        continue
                    qsegs.append([ch.row0, ch.rows, d, 0])
                    work += ch.rows - max(0, -d)
                flag = flag_of_src.get(src, -1)
                # launch order: local keys first, then sources in ring order (the order their K/V arrives),
                # heaviest tiles first inside a source
                step = (plan.rank - src) % plan.world
                items.append(((step, -work), [row_offset[src] + t0, rows, begin, len(qsegs) - begin, flag, src, t0, 0]))
                per_owner[src] += 1
    items.sort(key=lambda t: t[0])
    c[key] = (_to_dev([it for _, it in items], 8, device), _to_dev(qsegs if qsegs else [[0, 0, 0, 0]], 4, device),
              per_owner)
    return c[key]


class _DqWorkspace:
    """fp32 dQ accumulators, one per (device, stream, element count), kept ZEROED between calls: the backward
    kernel adds its partial tiles into it and ``dq_finalize`` (csrc/comm_sm90.cu) writes the model-dtype result and
    zeroes the accumulator again in the same pass.  Replaces a ``torch.zeros`` before and a ``.to(dtype)`` after
    every backward (the reference's fp32 dq bookkeeping: /root/reference/ring_flash_attn/ring_flash_attn.py:134-154)."""

    def __init__(self):
        self._bufs: Dict[tuple, list] = {}

    @staticmethod
    def _key(q: torch.Tensor) -> tuple:
        stream = torch.cuda.current_stream(q.device).cuda_stream if q.is_cuda else 0
        return (str(q.device), stream, q.numel())

    MAX_BYTES = 2 << 30  # total fp32 workspace kept alive across calls (beyond it the oldest shapes are dropped)

    def acquire(self, q: torch.Tensor) -> torch.Tensor:
        key = self._key(q)
        ent = self._bufs.get(key)
        if ent is None:
            need = 4 * q.numel()
            while self._bufs and (len(self._bufs) >= 8 or
                                  need + sum(4 * e[0].numel() for e in self._bufs.values()) > self.MAX_BYTES):
                self._bufs.pop(next(iter(self._bufs)))  # a handful of live shapes; drop the oldest
            ent = [torch.zeros(q.numel(), dtype=torch.float32, device=q.device), False]
            self._bufs[key] = ent
        elif ent[1]:  # a previous backward died between launch and finalize: do not trust the contents
            ent[0].zero_()
        ent[1] = True
        return ent[0].view(q.shape)

    def finalize(self, acc: torch.Tensor, q: torch.Tensor) -> torch.Tensor:
        out = torch.empty(q.shape, dtype=q.dtype, device=q.device)
        cuda_ext.load().dq_finalize(acc.view(-1), out.view(-1))
        cuda_ext.note_launch()
        ent = self._bufs.get(self._key(q))
        if ent is not None and ent[0].data_ptr() == acc.data_ptr():
            ent[1] = False
        return out


dq_workspace = _DqWorkspace()


def _to_dev(rows: List[List[int]], width: int, device) -> torch.Tensor:
    if not rows:
        return torch.zeros((0, width), dtype=torch.int32, device=device)
    return torch.tensor(rows, dtype=torch.int32).to(device, non_blocking=True)


def _cache(plan: CPPlan) -> dict:
    c = getattr(plan, "_cuda_tables", None)
    if c is None:
        c = {}
        plan._cuda_tables = c
    return c


def fwd_tables(plan, segs, row_offset, device, key, flag_of_src=None):
    c = _cache(plan)
    k = ("fwd", key, device.index)
    if k not in c:
        items, seg_rows, covered = fwd_tables_host(plan, segs, row_offset, flag_of_src)
        c[k] = (_to_dev(items, 8, device), _to_dev(seg_rows, 4, device), covered)
    return c[k]


def bwd_tables(plan, segs, row_offset, device, key, flag_of_src=None, ordered=False):
    """(items, qsegs) device tables; ``ordered=True`` (deterministic dQ) returns (items, qsegs, group bounds) with the
    items arranged in the launch groups of :func:`ordered_dq_groups`."""
    c = _cache(plan)
    k = ("bwd_ordered" if ordered else "bwd", key, device.index)
    if k not in c:
        items, qsegs = bwd_tables_host(plan, segs, row_offset, flag_of_src)
        c[("bwd", key, device.index, "covered")] = bwd_covers_all_rows(items, plan.kv_rows)
        if ordered:
            items, bounds = ordered_dq_groups(items, qsegs)
            c[k] = (_to_dev(items, 8, device), _to_dev(qsegs, 4, device), bounds)
        else:
            c[k] = (_to_dev(items, 8, device), _to_dev(qsegs, 4, device))
    return c[k]


def bwd_tables_cover(plan, device, key) -> bool:
    """Whether the cached backward table ``key`` writes every local dK/dV row (else the outputs start as zeros)."""
    return bool(_cache(plan).get(("bwd", key, device.index, "covered"), False))


# ----------------------------------------------------------------------------------------------
# launches
# ----------------------------------------------------------------------------------------------

def _rows3(t: torch.Tensor) -> torch.Tensor:
    """The kernels take (rows, heads, 128) views with a unit inner stride and 16-byte aligned strides."""
    if t.stride(-1) != 1 or (t.stride(0) * t.element_size()) % 16 or (t.stride(1) * t.element_size()) % 16 \
            or t.data_ptr() % 16:
        return t.contiguous()
    return t


def forward_launch(q, k, v, items, segs, covered, scale, out=None, lse=None):
    """Run the forward kernel over prepared tables.  Returns (out (Tq,Hq,128) in q.dtype, lse (Hq,Tq) fp32)."""
    C = cuda_ext.load()
    tq, hq, d = q.shape
    if out is None:
        out = (torch.empty if covered else torch.zeros)((tq, hq, d), dtype=out_dtype(q), device=q.device)
    if lse is None:
        lse = torch.empty((hq, tq), dtype=torch.float32, device=q.device)
        if not covered:
            lse.fill_(float("-inf"))
    if items.shape[0]:
        if is_fp8_kernel_input(q, k):
            scales = current_fp8_scales()
            if scales is None:
                raise RuntimeError("fp8 tensors reached the kernel launch without descales (attn_cuda.fp8_scales)")
            C.attn_fwd_fp8(_rows3(q), _rows3(k), _rows3(v), items, segs, *scales.args(), out, lse, tq, float(scale))
        else:
            C.attn_fwd(_rows3(q), _rows3(k), _rows3(v), items, segs, out, lse, tq, float(scale))
        cuda_ext.note_launch()
    return out, lse


def _segments_forward_window(plan: CPPlan, segs: Sequence[Segment], q, k_src, v_src, scale):
    C = cuda_ext.load()
    src = segs[0].src
    c = _cache(plan)
    key = ("fwd_window", src, q.device.index)
    if key not in c:
        items, seg_rows, seg_lo, covered = fwd_tables_window_host(plan, segs, {src: 0})
        c[key] = (_to_dev(items, 8, q.device), _to_dev(seg_rows if seg_rows else [[0, 0, 0, -1]], 4, q.device),
                  torch.tensor(seg_lo if seg_lo else [LO_NONE], dtype=torch.int32).to(q.device), covered)
    items, seg_t, lo_t, covered = c[key]
    tq, hq, d = q.shape
    out = (torch.empty if covered else torch.zeros)((tq, hq, d), dtype=q.dtype, device=q.device)
    lse = torch.empty((hq, tq), dtype=torch.float32, device=q.device)
    if not covered:
        lse.fill_(float("-inf"))
    if items.shape[0]:
        C.attn_fwd_window(_rows3(q), _rows3(k_src), _rows3(v_src), items, seg_t, lo_t, out, lse, tq, float(scale))
        cuda_ext.note_launch()
    return out, lse


def segments_forward(plan: CPPlan, segs: Sequence[Segment], q, k_src, v_src, scale):
    """Partial attention of the local queries against ONE source shard (torch.distributed fallback path)."""
    if has_window(segs):
        return _segments_forward_window(plan, segs, q, k_src, v_src, scale)
    src = segs[0].src
    items, seg_t, covered = fwd_tables(plan, segs, {src: 0}, q.device, ("step", src))
    return forward_launch(q, k_src, v_src, items, seg_t, covered, scale)


def compute_delta(out, dout, hq_rows=None) -> torch.Tensor:
    C = cuda_ext.load()
    tq, hq, _ = out.shape
    delta = torch.empty((hq, tq), dtype=torch.float32, device=out.device)
    C.attn_bwd_delta(_rows3(out), _rows3(dout), delta, tq)
    cuda_ext.note_launch()
    return delta


def backward_launch(q, dout, k, v, lse, delta, items, qsegs, scale, dq_accum, dk, dv, bounds=None, window=False):
    """One backward launch over the item table, or one per launch group (``bounds`` from :func:`ordered_dq_groups`)."""
    C = cuda_ext.load()
    launch = C.attn_bwd_window if window else C.attn_bwd
    if not items.shape[0]:
        return
    args = (_rows3(q), _rows3(dout), _rows3(k), _rows3(v), dq_accum)
    for a, b in ((0, items.shape[0]),) if bounds is None else zip(bounds[:-1], bounds[1:]):
        launch(*args, items[a:b], qsegs, lse, delta, dk, dv, q.shape[0], float(scale))
        cuda_ext.note_launch()


def segments_backward(plan: CPPlan, segs: Sequence[Segment], dout, q, k_src, v_src, lse, delta, scale, dq, dk, dv,
                      deterministic=False):
    """Gradient contribution of ONE source shard: dq (fp32) accumulates, dk/dv (fp32 or model dtype, zeroed) are
    filled.  ``deterministic``: one launch per group of key tiles with disjoint query rows (ordered dQ additions)."""
    src = segs[0].src
    lse, delta = lse.contiguous(), delta.contiguous()
    if has_window(segs):
        c = _cache(plan)
        key = ("bwd_window_ordered" if deterministic else "bwd_window", src, q.device.index)
        if key not in c:
            items, qsegs = bwd_tables_window_host(plan, segs, {src: 0})
            bounds = None
            if deterministic:
                items, bounds = ordered_dq_groups(items, qsegs)
            c[key] = (_to_dev(items, 8, q.device), _to_dev(qsegs if qsegs else [[0, 0, 0, 0]], 4, q.device), bounds)
        items, qsegs, bounds = c[key]
        backward_launch(q, dout, k_src, v_src, lse, delta, items, qsegs, scale, dq, dk, dv, bounds, window=True)
        return
    items, qsegs, *rest = bwd_tables(plan, segs, {src: 0}, q.device, ("step", src), ordered=deterministic)
    backward_launch(q, dout, k_src, v_src, lse, delta, items, qsegs, scale, dq, dk, dv, rest[0] if rest else None)
