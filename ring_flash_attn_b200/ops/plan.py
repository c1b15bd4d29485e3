"""Context-parallel attention plans.

Every sharding scheme of the reference is a statement about *global token positions*:

* ring      - rank r holds positions ``[r*L, (r+1)*L)``            (ring_flash_attn.py:26-63)
* zigzag    - rank r holds chunks ``r`` and ``2W-1-r`` of ``2W``    (zigzag_ring_flash_attn.py:60-84)
* stripe    - rank r holds positions ``r, r+W, r+2W, ...``          (stripe_flash_attn.py:29-97)
* varlen    - the same, independently per packed document           (ring_flash_attn_varlen.py:56-59,
                                                                    zigzag_ring_flash_attn_varlen.py:99-108)
* llama3    - contiguous split of the flat token stream             (llama3_flash_attn_varlen.py:10-60)

Instead of hand-writing a per-scheme step loop, this module turns (scheme, rank, world, shapes,
cu_seqlens) into a *plan*: local query chunks plus, for every source rank, the key segments each
chunk may see and the diagonal offset of the causal boundary (key ``j`` visible to query ``i`` iff
``j <= i + diag``).  The torch fallback executes a plan with ``ops.dense.block_fwd``; the sm_90a
kernels consume the very same plan as a device table and compute the masks in-kernel.

Rows are token-major: a batch tensor ``(B, S_l, H, D)`` is the row range ``[b*S_l, (b+1)*S_l)``.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple


@dataclass(frozen=True)
class QChunk:
    row0: int  # first local query row
    rows: int  # number of rows (contiguous, contiguous positions)


@dataclass(frozen=True)
class Segment:
    chunk: int  # index into CPPlan.q_chunks
    src: int  # source rank (within the CP group) that owns the keys
    kv_row0: int  # first row inside the source rank's local K/V
    kv_len: int
    diag: Optional[int]  # None = no upper bound; else key j visible to query i only if j <= i + diag
    lo: Optional[int] = None  # sliding window: key j visible only if j >= i + lo (None = no lower bound)


@dataclass
class CPPlan:
    world: int
    rank: int
    q_rows: int  # local query rows
    kv_rows: int  # local key rows on every rank (shards are equal sized)
    q_chunks: List[QChunk] = field(default_factory=list)
    segments: List[Segment] = field(default_factory=list)

    def by_src(self) -> Dict[int, List[Segment]]:
        out: Dict[int, List[Segment]] = {}
        for s in self.segments:
            out.setdefault(s.src, []).append(s)
        return out

    def needed_kv_rows(self, src: int) -> Optional[Tuple[int, int]]:
        """[lo, hi) row range of ``src``'s shard that this rank reads, or None if nothing."""
        segs = [s for s in self.segments if s.src == src]
        if not segs:
            return None
        return min(s.kv_row0 for s in segs), max(s.kv_row0 + s.kv_len for s in segs)

    def flops(self, heads_q: int, head_dim: int) -> int:
        """Forward matmul FLOPs of this rank's share (2 GEMMs, masked area excluded)."""
        total = 0
        for s in self.segments:
            n = self.q_chunks[s.chunk].rows
            total += visible_area(n, s.kv_len, s.diag, s.lo)
        return 4 * total * heads_q * head_dim


def visible_area(q_len: int, kv_len: int, diag: Optional[int], lo: Optional[int] = None) -> int:
    """Number of (query, key) pairs with ``i + lo <= j <= i + diag`` in a q_len x kv_len block."""
    if lo is not None:
        # pairs below the lower bound are those with j <= i + lo - 1
        below = visible_area(q_len, kv_len, lo - 1)
        return visible_area(q_len, kv_len, diag) - (below if diag is None else min(below, visible_area(q_len, kv_len, diag)))
    if diag is None:
        return q_len * kv_len
    lo = max(0, -diag)  # first row that sees at least one key
    full_from = max(lo, kv_len - 1 - diag)  # first row that sees every key
    ramp_hi = min(q_len, full_from)
    area = 0
    if ramp_hi > lo:
        area += ((lo + diag + 1) + (ramp_hi - 1 + diag + 1)) * (ramp_hi - lo) // 2
    if q_len > full_from:
        area += (q_len - full_from) * kv_len
    return area


def _ceil_div(a: int, b: int) -> int:
    return -((-a) // b)


def _classify(q_pos0: int, q_len: int, k_pos0: int, k_len: int, causal: bool, stride: int = 1,
              q_phase: int = 0, k_phase: int = 0, window: Tuple[int, int] = (-1, -1)):
    """Visibility of a key run against a query run: "skip", or (lo, hi) index offsets with None = unbounded
    (key j visible to query i iff i + lo <= j <= i + hi).

    Positions are ``pos0 + idx * stride + phase``; stride > 1 is the striped layout.  ``window`` follows
    flash-attn: key position p_k is visible to query position p_q iff p_q - left <= p_k <= p_q + right,
    -1 meaning unbounded; ``causal`` forces right = 0."""
    left, right = window
    if causal:
        right = 0
    # upper bound: p_k <= p_q + right   <=>   j <= i + floor((dq + right) / stride)
    d = (q_pos0 - k_pos0) * stride + (q_phase - k_phase)  # p_q - p_k at i == j
    hi = None if right < 0 else (d + right) // stride
    # lower bound: p_k >= p_q - left    <=>   j >= i + ceil((d - left) / stride)
    lo = None if left < 0 else _ceil_div(d - left, stride)
    if hi is not None and hi + (q_len - 1) < 0:
        return "skip"
    if lo is not None and lo > k_len - 1:
        return "skip"
    if hi is not None and lo is not None and lo > hi:
        return "skip"
    if hi is not None and hi >= k_len - 1:
        hi = None
    if lo is not None and lo + (q_len - 1) <= 0:
        lo = None
    return (lo, hi)


def _add(plan: CPPlan, chunk: int, src: int, kv_row0: int, kv_len: int, vis) -> None:
    if vis == "skip" or kv_len <= 0:
        return
    lo, hi = vis
    # coalesce with the previous segment when it continues the same key run on the same diagonals
    if plan.segments:
        p = plan.segments[-1]
        if p.chunk == chunk and p.src == src and p.kv_row0 + p.kv_len == kv_row0 and p.lo is None and lo is None:
            if p.diag is None and hi is None:
                plan.segments[-1] = Segment(chunk, src, p.kv_row0, p.kv_len + kv_len, None)
                return
            if p.diag is not None and hi is not None and hi == p.diag - p.kv_len:
                plan.segments[-1] = Segment(chunk, src, p.kv_row0, p.kv_len + kv_len, p.diag)
                return
    plan.segments.append(Segment(chunk, src, kv_row0, kv_len, hi, lo))


def _src_order(rank: int, world: int) -> List[int]:
    # ring schedule: own shard first, then the shard that started 1, 2, ... hops upstream
    return [(rank - s) % world for s in range(world)]


# ----------------------------------------------------------------------------------------------
# batch layouts
# ----------------------------------------------------------------------------------------------

def plan_ring(rank: int, world: int, batch: int, seqlen_local: int, causal: bool,
              window: Tuple[int, int] = (-1, -1)) -> CPPlan:
    L = seqlen_local
    plan = CPPlan(world, rank, batch * L, batch * L)
    for b in range(batch):
        plan.q_chunks.append(QChunk(b * L, L))
    for src in _src_order(rank, world):
        for b in range(batch):
            _add(plan, b, src, b * L, L, _classify(rank * L, L, src * L, L, causal, window=window))
    return plan


def plan_zigzag(rank: int, world: int, batch: int, seqlen_local: int, window: Tuple[int, int] = (-1, -1)) -> CPPlan:
    L = seqlen_local
    if L % 2:
        raise ValueError("zigzag needs an even local sequence length")
    c = L // 2
    plan = CPPlan(world, rank, batch * L, batch * L)
    for b in range(batch):
        plan.q_chunks.append(QChunk(b * L, c))
        plan.q_chunks.append(QChunk(b * L + c, c))
    qpos = (rank * c, (2 * world - 1 - rank) * c)
    for src in _src_order(rank, world):
        kpos = (src * c, (2 * world - 1 - src) * c)
        for b in range(batch):
            for qi in range(2):
                for ki in range(2):
                    _add(plan, 2 * b + qi, src, b * L + ki * c, c,
                         _classify(qpos[qi], c, kpos[ki], c, True, window=window))
    return plan


def plan_stripe(rank: int, world: int, batch: int, seqlen_local: int, window: Tuple[int, int] = (-1, -1)) -> CPPlan:
    L = seqlen_local
    plan = CPPlan(world, rank, batch * L, batch * L)
    for b in range(batch):
        plan.q_chunks.append(QChunk(b * L, L))
    for src in _src_order(rank, world):
        for b in range(batch):
            _add(plan, b, src, b * L, L,
                 _classify(0, L, 0, L, True, stride=world, q_phase=rank, k_phase=src, window=window))
    return plan


# ----------------------------------------------------------------------------------------------
# varlen layouts (one shared local cu_seqlens; every document is split evenly over the ranks)
# ----------------------------------------------------------------------------------------------

def plan_ring_varlen(rank: int, world: int, cu_seqlens: Sequence[int], causal: bool,
                     window: Tuple[int, int] = (-1, -1)) -> CPPlan:
    cu = [int(x) for x in cu_seqlens]
    total = cu[-1]
    plan = CPPlan(world, rank, total, total)
    for a, b in zip(cu[:-1], cu[1:]):
        plan.q_chunks.append(QChunk(a, b - a))
    for src in _src_order(rank, world):
        for d, (a, b) in enumerate(zip(cu[:-1], cu[1:])):
            n = b - a
            _add(plan, d, src, a, n, _classify(rank * n, n, src * n, n, causal, window=window))
    return plan


def plan_zigzag_varlen(rank: int, world: int, cu_seqlens: Sequence[int], window: Tuple[int, int] = (-1, -1)) -> CPPlan:
    cu = [int(x) for x in cu_seqlens]
    total = cu[-1]
    plan = CPPlan(world, rank, total, total)
    for a, b in zip(cu[:-1], cu[1:]):
        if (b - a) % 2:
            raise ValueError("zigzag varlen needs every local document length to be even")
        c = (b - a) // 2
        plan.q_chunks.append(QChunk(a, c))
        plan.q_chunks.append(QChunk(a + c, c))
    for src in _src_order(rank, world):
        for d, (a, b) in enumerate(zip(cu[:-1], cu[1:])):
            c = (b - a) // 2
            qpos = (rank * c, (2 * world - 1 - rank) * c)
            kpos = (src * c, (2 * world - 1 - src) * c)
            for qi in range(2):
                for ki in range(2):
                    _add(plan, 2 * d + qi, src, a + ki * c, c,
                         _classify(qpos[qi], c, kpos[ki], c, True, window=window))
    return plan


# ----------------------------------------------------------------------------------------------
# llama3 layout (contiguous split of the flat stream; documents may straddle ranks)
# ----------------------------------------------------------------------------------------------

def plan_llama3(rank: int, world: int, tokens_local: int, cu_seqlens_q: Sequence[int],
                cu_seqlens_k: Sequence[int], k_slice_start: int, causal: bool,
                window: Tuple[int, int] = (-1, -1)) -> CPPlan:
    """Plan from the outputs of ``llama3_flash_attn_prepare_cu_seqlens``.

    ``cu_seqlens_k`` is relative to ``k_slice_start`` in the *global* (gathered) key stream; the
    causal mask is bottom-right aligned per document (llama3_flash_attn_varlen.py:44-48)."""
    cuq = [int(x) for x in cu_seqlens_q]
    cuk = [int(x) for x in cu_seqlens_k]
    L = tokens_local
    plan = CPPlan(world, rank, L, L)
    for a, b in zip(cuq[:-1], cuq[1:]):
        plan.q_chunks.append(QChunk(a, b - a))
    pieces = []  # (src, doc, kv_row0, len, vis)
    for d in range(len(cuq) - 1):
        qn = cuq[d + 1] - cuq[d]
        k0 = k_slice_start + cuk[d]
        k1 = k_slice_start + cuk[d + 1]
        kn = k1 - k0
        # position of the chunk's first query inside its document (document key 0 sits at k0).  Causal:
        # bottom-right alignment as flash-attn defines it (prepare() trims the keys at the last local query,
        # so both expressions agree); non-causal windows need the true position because the keys run on to
        # the end of the document
        base_diag = kn - qn if causal else rank * L + cuq[d] - k0
        for src in range(world):
            lo, hi = max(k0, src * L), min(k1, (src + 1) * L)
            if hi <= lo:
                continue
            # key j' (within this piece) is doc key j' + (lo - k0)
            if causal or window != (-1, -1):
                # query i of the chunk sits at document key position i + base_diag
                vis = _classify(base_diag, qn, lo - k0, hi - lo, causal, window=window)
            else:
                vis = (None, None)
            pieces.append((src, d, lo - src * L, hi - lo, vis))
    for src in _src_order(rank, world):
        for (s, d, r0, n, vis) in pieces:
            if s == src:
                _add(plan, d, src, r0, n, vis)
    return plan


# ----------------------------------------------------------------------------------------------
# flat layouts: every rank owns a list of ranges of the packed token stream
# ----------------------------------------------------------------------------------------------

def zigzag_flat_ranges(rank: int, world: int, total: int) -> List[Tuple[int, int]]:
    """Chunks ``rank`` and ``2W-1-rank`` of the flat stream cut into ``2W`` equal chunks."""
    if total % (2 * world):
        raise ValueError(f"total tokens ({total}) must be divisible by 2 * world_size ({2 * world})")
    c = total // (2 * world)
    return [(rank * c, (rank + 1) * c), ((2 * world - 1 - rank) * c, (2 * world - rank) * c)]


def plan_flat(rank: int, world: int, global_cu: Sequence[int], ranges_of, causal: bool,
              window: Tuple[int, int] = (-1, -1)) -> CPPlan:
    """Packed documents (``global_cu``) over a flat token stream where rank r owns ``ranges_of(r)`` - a list of
    ``[g0, g1)`` global ranges stored back to back in its local tensors.  Documents may be cut anywhere.

    With ``zigzag_flat_ranges`` this is the load-balanced llama3 variant the reference lists as a TODO
    (/root/reference/README.md:130): the causal work of every rank is equal for any packing, and no document length
    has to be divisible by the world size."""
    cu = [int(x) for x in global_cu]
    owned = [ranges_of(r) for r in range(world)]
    L = sum(b - a for a, b in owned[rank])
    if any(sum(b - a for a, b in o) != L for o in owned):
        raise ValueError("every rank must own the same number of tokens")
    plan = CPPlan(world, rank, L, L)
    # local query chunks: (owned range x document) pieces
    q_pieces = []  # (chunk index, global start, rows)
    base = 0
    for a, b in owned[rank]:
        for d0, d1 in zip(cu[:-1], cu[1:]):
            lo, hi = max(a, d0), min(b, d1)
            if hi > lo:
                q_pieces.append((len(plan.q_chunks), lo, hi - lo, d0, d1))
                plan.q_chunks.append(QChunk(base + lo - a, hi - lo))
        base += b - a
    for src in _src_order(rank, world):
        kbase = 0
        for ka, kb in owned[src]:
            for ci, q0, qn, d0, d1 in q_pieces:
                lo, hi = max(ka, d0), min(kb, d1)
                if hi > lo:
                    vis = _classify(q0 - d0, qn, lo - d0, hi - lo, causal, window=window) \
                        if (causal or window != (-1, -1)) else (None, None)
                    _add(plan, ci, src, kbase + lo - ka, hi - lo, vis)
            kbase += kb - ka
    return plan


def plan_zigzag_llama3(rank: int, world: int, global_cu: Sequence[int], causal: bool = True,
                       window: Tuple[int, int] = (-1, -1)) -> CPPlan:
    total = int(global_cu[-1])
    return plan_flat(rank, world, global_cu, lambda r: zigzag_flat_ranges(r, world, total), causal, window)

