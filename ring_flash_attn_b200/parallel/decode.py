"""Context-parallel decoding over a sharded KV cache: ``cp_flash_attn_with_kvcache``.

After a prefill with any scheme, rank ``r`` holds its shard of K and V.  Without windows or positional biases,
decode attention does not depend on where a cached key sits, so every rank attends the new query tokens to its own
shard, and the per-rank partial ``(out, lse)`` results are merged with the online-softmax identity
``lse = logsumexp_r(lse_r)``, ``out = sum_r exp(lse_r - lse) out_r``.  The only traffic between ranks is one
all-gather of those partials (a few KB per layer).

On Hopper the local step is the split-KV kernel of ``csrc/decode_sm90.cu``: the query heads of a GQA group and the
new tokens share the wgmma M dimension, one sequence's keys are spread over many CTAs, and one combine kernel merges
the per-split partials and then, with the same code, the gathered per-rank partials.  Every rank combines the same
gathered partials in rank order, so ``out`` and ``lse`` are bitwise identical on every rank.

The dense path (CPU / gloo, other GPUs, ``RFA_B200_FORCE_TORCH=1``, and shapes the kernel is not instantiated for)
computes the local partial with ``ops.dense.block_fwd`` and merges the gathered partials with
``ops.merge.merge_partial`` in the same rank order.
"""
from __future__ import annotations

import functools
import warnings
from typing import Optional, Tuple

import torch
import torch.distributed as dist
from torch import Tensor

from ..ops import cuda_ext
from ..ops.dense import block_fwd
from ..ops.merge import merge_partial
from .comm import _wire, group_info
from .ops import group_name, resolve_group

KERNEL_HEAD_DIMS = (64, 128)  # the decode kernel is instantiated for these head sizes
KEY_TILE = 128  # keys per K / V tile of the kernel
ROWS_PER_CTA = 64  # packed (token, head-in-group) query rows per CTA


@functools.lru_cache(maxsize=None)
def _sm_count(index: int) -> int:
    return torch.cuda.get_device_properties(index).multi_processor_count


def num_splits(batch: int, sq: int, hq: int, hkv: int, s_cap: int, sm_count: int) -> int:
    """Key-range splits per (sequence, kv head, row tile).  The kernel keeps one CTA per SM (its K/V ring fills the
    shared memory), so the grid is sized to one full wave: more CTAs would leave a ragged second wave.  Derived from
    shapes only, never from ``cache_seqlens``: splits past a sequence's valid keys exit at once, and nothing is read
    back to the host (a decode step can be captured in a CUDA graph)."""
    row_tiles = -(-sq * (hq // hkv) // ROWS_PER_CTA)
    tiles = max(1, -(-s_cap // KEY_TILE))
    return max(1, min(tiles, sm_count // (batch * hkv * row_tiles)))


def tile_slots(batch: int, total_q: int, max_seqlen_q: int, hq: int, hkv: int) -> int:
    """Row-tile slots of a varlen call's grid (per split and kv head): ``min(B * ceil(max_seqlen_q * G / 64),
    (total_q * G + 63 * B) // 64)``, an upper bound from shapes on ``sum_b ceil(n_b * G / 64)`` for any counts
    ``n_b <= max_seqlen_q`` summing to ``total_q``.  Each CTA maps its slot to a (sequence, row tile) on the device;
    slots past the last real tile exit at once."""
    g = hq // hkv
    per_seq = -(-max_seqlen_q * g // ROWS_PER_CTA)
    return min(batch * per_seq, (total_q * g + (ROWS_PER_CTA - 1) * batch) // ROWS_PER_CTA)


def num_splits_varlen(batch: int, total_q: int, max_seqlen_q: int, hq: int, hkv: int, s_cap: int,
                      sm_count: int) -> int:
    """:func:`num_splits` for a varlen call: :func:`tile_slots` takes the place of ``B * row_tiles``.  With equal
    counts (``total_q = B * max_seqlen_q``) it is exactly :func:`num_splits` of the uniform call."""
    tiles = max(1, -(-s_cap // KEY_TILE))
    slots = max(1, tile_slots(batch, total_q, max_seqlen_q, hq, hkv))
    return max(1, min(tiles, sm_count // (slots * hkv)))


def prefix_tile_slots(n: int, sq: int, hq: int, hkv: int, total_q: Optional[int] = None) -> int:
    """Row-tile slots of the shared-prefix pass per (prefix, kv head): ``ceil(rows * G / 64)`` for the ``rows`` of
    one group of ``n`` sequences, ``n * sq``, or ``min(n * max_seqlen_q, total_q)`` for a varlen call.  From shapes
    only; slots past a group's last real tile exit at once."""
    rows = n * sq if total_q is None else min(n * sq, total_q)
    return -(-rows * (hq // hkv) // ROWS_PER_CTA)


def num_splits_prefix(n_prefix: int, slots: int, hkv: int, p_cap: int, sm_count: int) -> int:
    """Key-range splits of the shared-prefix pass: :func:`num_splits` with ``P`` prefixes of ``slots`` row tiles
    (:func:`prefix_tile_slots`) for the ``B`` sequences, and ``P_cap`` for ``S_cap``.  One full wave, from shapes
    only, never from ``prefix_seqlens``."""
    tiles = max(1, -(-p_cap // KEY_TILE))
    return max(1, min(tiles, sm_count // (n_prefix * hkv * max(1, slots))))


_warned = set()


def _kernel_takes(q: Tensor) -> bool:
    if not cuda_ext.available_for(q):
        return False
    if q.dtype in (torch.bfloat16, torch.float16, torch.float8_e4m3fn) and q.shape[-1] in KERNEL_HEAD_DIMS:
        return True
    key = (q.dtype, q.shape[-1])
    if key not in _warned:
        _warned.add(key)
        warnings.warn(f"cp_flash_attn_with_kvcache: no sm_90a decode kernel for {q.dtype} with head_dim {q.shape[-1]} "
                      f"(instantiated: bf16 / fp16, and e4m3 over e4m3 caches, head_dim {KERNEL_HEAD_DIMS}); running "
                      "the dense torch path", RuntimeWarning, stacklevel=3)
    return False


def _gather(local: Tensor, pg, world: int) -> Tensor:
    """(world, n) stack of every rank's flat fp32 partial, rank order, on the caller's stream."""
    buf = local.new_empty(world * local.numel())  # flat: gloo takes only the concatenated form
    dist.all_gather_into_tensor(_wire(buf), _wire(local), group=pg)
    return buf.view(world, local.numel())


# ----------------------------------------------------------------------------------------------
# sm_90a path
# ----------------------------------------------------------------------------------------------

def _capacity(k_cache: Tensor, block_table: Optional[Tensor]) -> int:
    """Cache rows per sequence: ``S_cap``, or ``max_blocks * page_size`` for a paged cache."""
    return k_cache.shape[1] if block_table is None else block_table.shape[1] * k_cache.shape[1]


def _out_dtype(q: Tensor) -> torch.dtype:
    """``out``'s dtype: q's, or bf16 for an e4m3 ``q`` (flash-attn 3's rule)."""
    return torch.bfloat16 if q.dtype == torch.float8_e4m3fn else q.dtype


def kernel_decode(q: Tensor, k_cache: Tensor, v_cache: Tensor, cache_seqlens: Tensor, k: Optional[Tensor],
                  v: Optional[Tensor], causal: bool, softmax_scale: float, pg=None, world: int = 1,
                  splits: Optional[int] = None, block_table: Optional[Tensor] = None,
                  k_descale: Optional[Tensor] = None, v_descale: Optional[Tensor] = None,
                  cu_seqlens_q: Optional[Tensor] = None, max_seqlen_q: Optional[int] = None,
                  rotary_cos: Optional[Tensor] = None, rotary_sin: Optional[Tensor] = None,
                  rotary_seqlens: Optional[Tensor] = None, rotary_interleaved: bool = True,
                  q_descale: Optional[Tensor] = None, cache_batch_idx: Optional[Tensor] = None,
                  cache_leftpad: Optional[Tensor] = None, prefix_k_cache: Optional[Tensor] = None,
                  prefix_v_cache: Optional[Tensor] = None, prefix_seqlens: Optional[Tensor] = None,
                  prefix_k_descale: Optional[Tensor] = None, prefix_v_descale: Optional[Tensor] = None,
                  prefix_splits: Optional[int] = None, tree_mask: Optional[Tensor] = None,
                  prefix_block_table: Optional[Tensor] = None) -> Tuple[Tensor, Tensor]:
    """Local split-KV kernel (appending ``k`` / ``v`` first when given), then the combine over the splits and, for
    ``world > 1``, over the gathered per-rank partials.  ``splits`` overrides :func:`num_splits`.  With
    ``block_table`` the caches are page pools (see :func:`cp_flash_attn_with_kvcache`).  e4m3 caches take contiguous
    fp32 ``(B, Hkv)`` ``k_descale`` / ``v_descale``.  With ``cu_seqlens_q`` (and ``max_seqlen_q``) ``q`` / ``k`` /
    ``v`` are varlen ``(total_q, H, D)`` and the result is ``out (total_q, Hq, D)``, ``lse (Hq, total_q)``.  With
    ``rotary_cos`` / ``rotary_sin`` (and ``rotary_seqlens``, required here) the kernel rotates ``q`` as it loads it
    and ``k`` before it stores it, as :func:`apply_rotary` does, at positions clamped to the tables.  An e4m3 ``q``
    (over e4m3 caches) takes a contiguous fp32 ``(B, Hkv)`` ``q_descale`` and gives a bf16 ``out``; e4m3 ``k`` / ``v``
    over e4m3 caches are stored as they are.  ``cache_batch_idx`` / ``cache_leftpad`` (contiguous ``(B,)`` int32,
    contiguous caches only) select each sequence's cache slot and first key row, read on the device only.  With
    ``prefix_k_cache`` / ``prefix_v_cache`` ``(P, P_cap, Hkv, D)`` (contiguous), ``prefix_seqlens`` ``(P,)`` int32 and,
    for e4m3 caches, contiguous fp32 ``(P, Hkv)`` ``prefix_k_descale`` / ``prefix_v_descale``, a second kernel adds
    the attention of sequence ``b`` to prefix ``b // (B // P)``, in ``prefix_splits`` (default
    :func:`num_splits_prefix`) more partial slabs that the same combine merges; with ``prefix_block_table``
    ``(P, max_prefix_blocks)`` int32 the prefix caches are page pools, as ``block_table`` makes the caches, and may be
    the very tensors ``k_cache`` / ``v_cache``.  ``tree_mask`` (contiguous bool
    ``(B, Sq, Sq)``, or ``(total_q, max_seqlen_q)`` when varlen; needs ``causal``) says which appended keys each new
    token sees and sets the rotary positions of ``q`` and ``k`` (see :func:`cp_flash_attn_with_kvcache`); it is passed
    on every rank."""
    C = cuda_ext.load()
    varlen = cu_seqlens_q is not None
    if varlen:  # the partials are the uniform layout at batch 1, Sq = total_q
        b = cache_seqlens.shape[0]
        total_q, hq, d = q.shape
        rows_b, rows_sq = 1, total_q
    else:
        b, sq, hq, d = q.shape
        rows_b, rows_sq = b, sq
    q = q.contiguous()
    if k is not None:
        k, v = k.contiguous(), v.contiguous()
    if splits is None:
        dev = q.device.index if q.device.index is not None else torch.cuda.current_device()
        s_cap, hkv = _capacity(k_cache, block_table), k_cache.shape[2]
        if varlen:
            splits = num_splits_varlen(b, total_q, max_seqlen_q, hq, hkv, s_cap, _sm_count(dev))
        else:
            splits = num_splits(b, sq, hq, hkv, s_cap, _sm_count(dev))
    prefix = prefix_k_cache is not None
    if prefix and prefix_splits is None:
        dev = q.device.index if q.device.index is not None else torch.cuda.current_device()
        n_prefix = prefix_k_cache.shape[0] if prefix_block_table is None else prefix_block_table.shape[0]
        hkv = prefix_k_cache.shape[2]
        slots = prefix_tile_slots(b // n_prefix, max_seqlen_q if varlen else sq, hq, hkv,
                                  total_q if varlen else None)
        prefix_splits = num_splits_prefix(n_prefix, slots, hkv, _capacity(prefix_k_cache, prefix_block_table),
                                          _sm_count(dev))
    n_slabs = splits + (prefix_splits if prefix else 0)
    n_out = rows_b * rows_sq * hq * d
    size = n_out + rows_b * hq * rows_sq
    # every split's partial starts 8-byte aligned (the kernel stores out as float2): rows * Hq * (D + 1) is odd when
    # rows and Hq are
    parts = torch.empty((n_slabs, size + size % 2), dtype=torch.float32, device=q.device)[:, :size]
    extra = () if q_descale is None else (q_descale,)  # decode_fwd takes q_descale only for an e4m3 q
    if cache_batch_idx is not None or cache_leftpad is not None:
        extra = (q_descale, cache_batch_idx, cache_leftpad)
    if tree_mask is not None:  # (rows, Sq): row = packed query row
        tree_mask = tree_mask.view(-1, tree_mask.shape[-1])
        extra = (q_descale, cache_batch_idx, cache_leftpad, tree_mask)
    C.decode_fwd(q, k_cache, v_cache, cache_seqlens, k, v, causal, softmax_scale, parts[:splits], block_table,
                 k_descale, v_descale, cu_seqlens_q, int(max_seqlen_q) if varlen else 0, rotary_cos, rotary_sin,
                 rotary_seqlens, bool(rotary_interleaved), *extra)
    cuda_ext.note_launch(2 if k is not None else 1)
    if prefix:  # the prefix partials go to the slabs after the suffix pass's
        pextra = () if tree_mask is None else (tree_mask,)
        if prefix_block_table is not None:
            pextra = (tree_mask, prefix_block_table)
        C.decode_prefix_fwd(q, prefix_k_cache, prefix_v_cache, prefix_seqlens, causal, softmax_scale, parts[splits:],
                            prefix_k_descale, prefix_v_descale, cu_seqlens_q, int(max_seqlen_q) if varlen else 0,
                            rotary_cos, rotary_sin, rotary_seqlens, bool(rotary_interleaved), *pextra)
        cuda_ext.note_launch()
    if world > 1:
        mine = torch.empty(size, dtype=torch.float32, device=q.device)
        C.decode_combine(parts, mine[:n_out].view(rows_b, rows_sq, hq, d), mine[n_out:].view(rows_b, hq, rows_sq))
        cuda_ext.note_launch()
        parts = _gather(mine, pg, world)
    out = torch.empty(q.shape, dtype=_out_dtype(q), device=q.device)
    lse = torch.empty((rows_b, hq, rows_sq), dtype=torch.float32, device=q.device)
    C.decode_combine(parts, out.view(rows_b, rows_sq, hq, d), lse)
    cuda_ext.note_launch()
    return out, (lse.view(hq, rows_sq) if varlen else lse)


# ----------------------------------------------------------------------------------------------
# dense path
# ----------------------------------------------------------------------------------------------

def quantize_e4m3(x: Tensor, descale: Tensor) -> Tensor:
    """``x`` (..., Hkv, D) as stored in an e4m3 cache with per-kv-head ``descale`` (Hkv,): IEEE division, saturation
    to +-448, then round-to-nearest-even (NaN stays NaN)."""
    return (x.float() / descale[:, None]).clamp(-448, 448).to(torch.float8_e4m3fn)


def apply_rotary(x: Tensor, cos: Tensor, sin: Tensor, positions: Tensor, interleaved: bool = True) -> Tensor:
    """``x`` ``(..., H, D)`` with rotary embeddings at table rows ``positions`` (shape ``x.shape[:-2]``), from the
    ``(seqlen_ro, rotary_dim / 2)`` tables ``cos`` / ``sin``.  Columns below ``rotary_dim`` are rotated in pairs
    ``(i, i + rotary_dim / 2)`` (GPT-NeoX / Llama), or ``(2i, 2i + 1)`` when ``interleaved`` (GPT-J); the rest are left
    as they are.  For a pair ``(a, b)`` and ``c = cos[pos, i]``, ``s = sin[pos, i]``: ``a' = a c - b s``,
    ``b' = b c + a s``, with every operand widened to fp32, each product and the sum or difference rounded to fp32
    (no FMA), and the result rounded to nearest even into x's dtype.  The sm_90a decode kernel computes exactly this,
    so a fused call is bitwise a plain call on rotated inputs."""
    h = cos.shape[1]
    c = cos[positions].float().unsqueeze(-2)  # (..., 1, h)
    s = sin[positions].float().unsqueeze(-2)
    xr = x[..., :2 * h].float()
    a, b = (xr[..., 0::2], xr[..., 1::2]) if interleaved else (xr[..., :h], xr[..., h:])
    a2 = a * c - b * s  # separate torch ops: each rounded to fp32
    b2 = b * c + a * s
    y = torch.stack([a2, b2], dim=-1).flatten(-2) if interleaved else torch.cat([a2, b2], dim=-1)
    return torch.cat([y.to(x.dtype), x[..., 2 * h:]], dim=-1)


def tree_depths(tree_mask: Tensor, spans) -> list:
    """Per packed new token, its depth: the True entries among the first ``n_b`` of its ``(rows, Sq)`` tree-mask row,
    minus one (0 for an empty row).  The rotary offset of a new token with a tree mask."""
    depths = []
    for lo, n in spans:
        depths += (tree_mask[lo:lo + n, :n].sum(1) - 1).clamp(min=0).tolist()
    return depths


def _rotary_positions(rotary_seqlens: Tensor, spans, seqlen_ro: int, causal: bool, device, depths=None):
    """Table rows of the packed new tokens, (keys, queries): key t of sequence b at ``rotary_seqlens[b] + t``, query
    token t there too when causal, at ``rotary_seqlens[b]`` otherwise; with a tree mask both at
    ``rotary_seqlens[b] + depths[row]``.  ``ValueError`` for a position outside the tables (the kernel clamps
    instead)."""
    keys, queries = [], []
    for i, (start, (lo, n)) in enumerate(zip(rotary_seqlens.tolist(), spans)):
        if depths is not None:
            pos = [start + x for x in depths[lo:lo + n]]
            if pos and not (0 <= min(pos) and max(pos) < seqlen_ro):
                raise ValueError(f"rotary positions [{min(pos)}, {max(pos)}] of sequence {i} are outside the "
                                 f"{seqlen_ro}-row rotary tables")
            keys += pos
            queries += pos
            continue
        if n and not 0 <= start <= seqlen_ro - n:
            raise ValueError(f"rotary positions [{start}, {start + n}) of sequence {i} are outside the "
                             f"{seqlen_ro}-row rotary tables")
        keys += range(start, start + n)
        queries += range(start, start + n) if causal else [start] * n
    return (torch.tensor(keys, dtype=torch.long, device=device), torch.tensor(queries, dtype=torch.long,
                                                                              device=device))


def _varlen_spans(cu_seqlens_q: Tensor, total_q: int, max_seqlen_q: int):
    """(first row, count) of every sequence of a varlen call; ``ValueError`` for a malformed ``cu_seqlens_q``."""
    cu = cu_seqlens_q.tolist()
    if cu[0] != 0 or cu[-1] != total_q:
        raise ValueError(f"cu_seqlens_q must start at 0 and end at total_q = {total_q}, not {cu[0]} ... {cu[-1]}")
    spans = [(lo, hi - lo) for lo, hi in zip(cu[:-1], cu[1:])]
    if any(n < 0 for _, n in spans):
        raise ValueError("cu_seqlens_q must not decrease")
    if any(n > max_seqlen_q for _, n in spans):
        raise ValueError(f"cu_seqlens_q has a count above max_seqlen_q = {max_seqlen_q}")
    return spans


def _dense_decode(q, k_cache, v_cache, cache_seqlens, k, v, causal, softmax_scale, pg, world, block_table=None,
                  k_descale=None, v_descale=None, cu_seqlens_q=None, max_seqlen_q=0, rotary=None, q_descale=None,
                  cache_batch_idx=None, cache_leftpad=None, prefix=None, tree_mask=None):
    # every sequence is a (first row, count) span of the packed rows: (b * Sq, Sq) for a uniform q
    out_dtype = _out_dtype(q)
    b = cache_seqlens.shape[0]
    hq, d = q.shape[-2:]
    if cu_seqlens_q is not None:
        spans = _varlen_spans(cu_seqlens_q, q.shape[0], max_seqlen_q)
    else:
        sq = q.shape[1]
        spans = [(i * sq, sq) for i in range(b)]
        q = q.reshape(b * sq, hq, d)
        if k is not None:
            k, v = k.reshape(b * sq, *k.shape[2:]), v.reshape(b * sq, *v.shape[2:])
    if rotary is not None:  # (cos, sin, rotary_seqlens, interleaved): q on every rank, k where it is appended
        cos, sin, rotary_seqlens, interleaved = rotary
        depths = None if tree_mask is None else tree_depths(tree_mask, spans)
        key_pos, q_pos = _rotary_positions(rotary_seqlens, spans, cos.shape[0], causal, q.device, depths)
        q = apply_rotary(q, cos, sin, q_pos, interleaved)
        if k is not None:
            k = apply_rotary(k, cos, sin, key_pos, interleaved)
    if q_descale is not None:  # e4m3 q: the query it stands for, q.float() * q_descale[b, h // G]
        g = hq // q_descale.shape[1]
        q = torch.cat([q[lo:lo + n].float() * q_descale[i].repeat_interleave(g)[:, None]
                       for i, (lo, n) in enumerate(spans)])
    rows = q.shape[0]
    s_cap = _capacity(k_cache, block_table)
    lens = [max(0, min(int(x), s_cap)) for x in cache_seqlens.tolist()]
    ps, n_pages = k_cache.shape[1], k_cache.shape[0]
    table = block_table.tolist() if block_table is not None else None
    fp8 = k_descale is not None
    # sequence i's cache slot and first key row (the kernel path reads both on the device only and does not check them)
    slots = list(range(b)) if cache_batch_idx is None else cache_batch_idx.tolist()
    pads = [0] * b if cache_leftpad is None else cache_leftpad.tolist()
    for i, (slot, lp) in enumerate(zip(slots, pads)):
        if cache_batch_idx is not None and not 0 <= slot < n_pages:
            raise ValueError(f"cache_batch_idx[{i}] = {slot} is outside the {n_pages}-slot cache")
        if not 0 <= lp <= lens[i]:
            raise ValueError(f"cache_leftpad[{i}] = {lp} is outside [0, cache_seqlens[{i}]] = [0, {lens[i]}]")
    # shared prefixes (prefix_k, prefix_v, prefix_seqlens, prefix_k_descale, prefix_v_descale, prefix_block_table):
    # sequence i reads rows [0, plens[i // n]) of prefix i // n ahead of its own keys
    plens = []
    if prefix is not None:
        pk, pv, pseq, pkd, pvd, ptable = prefix
        n_per = b // pseq.shape[0]
        p_cap = _capacity(pk, ptable)
        plens = pseq.tolist()
        for j, x in enumerate(plens):
            if not 0 <= x <= p_cap:
                raise ValueError(f"prefix_seqlens[{j}] = {x} is outside [0, P_cap] = [0, {p_cap}]")
        if ptable is not None:  # the pages holding the visible rows, in table order, checked before any append
            pps = pk.shape[1]
            ppages = [row[:-(-n // pps)] for row, n in zip(ptable.tolist(), plens)]
            for j, pages in enumerate(ppages):
                if not all(0 <= x < pk.shape[0] for x in pages):
                    raise ValueError(f"prefix_block_table[{j}] points outside the {pk.shape[0]}-page pool for a "
                                     "page it reads")
    if k is not None:  # rows past the capacity (or whose page is outside the pool) are dropped, as in the kernel path
        if fp8 and k.dtype != torch.float8_e4m3fn:  # pre-quantised e4m3 k / v are stored as they are
            k = torch.cat([quantize_e4m3(k[lo:lo + n], k_descale[i]) for i, (lo, n) in enumerate(spans)])
            v = torch.cat([quantize_e4m3(v[lo:lo + n], v_descale[i]) for i, (lo, n) in enumerate(spans)])
        for i, n in enumerate(lens):
            lo, cnt = spans[i]
            m = min(cnt, s_cap - n)
            if table is None:
                k_cache[slots[i], n:n + m] = k[lo:lo + m]
                v_cache[slots[i], n:n + m] = v[lo:lo + m]
                continue
            for t in range(m):
                page = table[i][(n + t) // ps]
                if 0 <= page < n_pages:
                    k_cache[page, (n + t) % ps] = k[lo + t]
                    v_cache[page, (n + t) % ps] = v[lo + t]
    out = torch.zeros((rows, hq, d), dtype=torch.float32, device=q.device)
    lse = torch.full((hq, rows), float("-inf"), dtype=torch.float32, device=q.device)
    for i, n in enumerate(lens):
        lo, cnt = spans[i]
        n_new = cnt if k is not None else 0
        n_keys = min(n + n_new, s_cap)
        lp = pads[i]  # rows [lp, n_keys) of the slot
        n_pre = plens[i // n_per] if prefix is not None else 0
        if n_keys - lp + n_pre == 0 or cnt == 0:
            continue
        if table is None:
            kk, vv = k_cache[slots[i], lp:n_keys], v_cache[slots[i], lp:n_keys]
        else:  # the pages holding the visible rows, in table order
            pages = table[i][:-(-n_keys // ps)]
            if not all(0 <= x < n_pages for x in pages):
                raise ValueError(f"block_table[{i}] points outside the {n_pages}-page pool for a page it reads")
            kk, vv = k_cache[pages].flatten(0, 1)[:n_keys], v_cache[pages].flatten(0, 1)[:n_keys]
        if fp8:  # the dequantised rows
            kk, vv = kk.float() * k_descale[i][:, None], vv.float() * v_descale[i][:, None]
        if n_pre:  # the prefix rows come first, and every query token sees them
            p = i // n_per
            if ptable is None:
                pkk, pvv = pk[p, :n_pre], pv[p, :n_pre]
            else:
                pkk, pvv = pk[ppages[p]].flatten(0, 1)[:n_pre], pv[ppages[p]].flatten(0, 1)[:n_pre]
            if fp8:
                pkk, pvv = pkk.float() * pkd[p][:, None], pvv.float() * pvd[p][:, None]
            kk, vv = torch.cat([pkk.to(kk.dtype), kk]), torch.cat([pvv.to(vv.dtype), vv])
        # appended key u (row n + u) is visible to token t iff u <= t, i.e. row j <= t + n (j counted from lp, after
        # the prefix rows); with a tree mask iff tree_mask[lo + t, u], every earlier row staying visible
        diag = n_pre + n - lp if (n_new and causal and tree_mask is None) else None
        mask = None
        if n_new and tree_mask is not None:
            mask = torch.cat([torch.ones(cnt, n_pre + n - lp, dtype=torch.bool, device=q.device),
                              tree_mask[lo:lo + cnt, :n_keys - n]], dim=1)
        out[lo:lo + cnt], lse[:, lo:lo + cnt] = block_fwd(q[lo:lo + cnt], kk, vv, softmax_scale, diag, mask=mask)
    if world > 1:
        parts = _gather(torch.cat([out.reshape(-1), lse.reshape(-1)]), pg, world)
        n_out = out.numel()
        acc_o = acc_l = None
        for r in range(world):  # rank order: the same on every rank
            acc_o, acc_l = merge_partial(acc_o, acc_l, parts[r, :n_out].view(rows, hq, d),
                                         parts[r, n_out:].view(hq, rows))
        out, lse = acc_o, acc_l
    if cu_seqlens_q is None:  # back to (B, Sq, Hq, D) and (B, Hq, Sq)
        out = out.reshape(b, sq, hq, d)
        lse = lse.reshape(hq, b, sq).permute(1, 0, 2).contiguous()
    return out.to(out_dtype), lse


# ----------------------------------------------------------------------------------------------
# the op and the public function
# ----------------------------------------------------------------------------------------------

@torch.library.custom_op("rfa_b200::cp_decode", mutates_args=("k_cache", "v_cache"))
def cp_decode(q: Tensor, k_cache: Tensor, v_cache: Tensor, cache_seqlens: Tensor, k: Optional[Tensor],
              v: Optional[Tensor], append_rank: int, softmax_scale: float, causal: bool, group: str,
              block_table: Optional[Tensor], k_descale: Optional[Tensor], v_descale: Optional[Tensor],
              cu_seqlens_q: Optional[Tensor], max_seqlen_q: int, rotary_cos: Optional[Tensor] = None,
              rotary_sin: Optional[Tensor] = None, rotary_seqlens: Optional[Tensor] = None,
              rotary_interleaved: bool = True, q_descale: Optional[Tensor] = None,
              cache_batch_idx: Optional[Tensor] = None, cache_leftpad: Optional[Tensor] = None,
              prefix_k_cache: Optional[Tensor] = None, prefix_v_cache: Optional[Tensor] = None,
              prefix_seqlens: Optional[Tensor] = None, prefix_k_descale: Optional[Tensor] = None,
              prefix_v_descale: Optional[Tensor] = None, tree_mask: Optional[Tensor] = None,
              prefix_block_table: Optional[Tensor] = None) -> Tuple[Tensor, Tensor]:
    """q (B, Sq, Hq, D) -> (out (B, Sq, Hq, D) in q.dtype (bf16 for an e4m3 q), lse (B, Hq, Sq) fp32).  ``k`` /
    ``v`` are appended to the caches of rank ``append_rank`` only (-1: no append); ``group`` is the process group's
    name ("" = world); with ``block_table`` the caches are this rank's page pools; e4m3 caches come with contiguous
    fp32 (B, Hkv) ``k_descale`` / ``v_descale``.  With ``cu_seqlens_q`` q / k / v are varlen (total_q, H, D), out is
    (total_q, Hq, D) and lse (Hq, total_q); ``max_seqlen_q`` bounds the counts (0 when uniform).  With
    ``rotary_cos`` / ``rotary_sin`` / ``rotary_seqlens``, every rank rotates q and the append rank rotates k before
    it stores it.  An e4m3 q comes with a contiguous fp32 (B, Hkv) ``q_descale``.  ``cache_batch_idx`` /
    ``cache_leftpad`` (B,) int32 pick each sequence's cache slot and first key row.  ``prefix_k_cache`` /
    ``prefix_v_cache`` (P, P_cap, Hkv, D) with ``prefix_seqlens`` (P,) int32 (and fp32 (P, Hkv) descales for e4m3)
    are this rank's shards of the prefixes shared by consecutive groups of B / P sequences (read-only).  ``tree_mask``
    (B, Sq, Sq) bool, or (total_q, max_seqlen_q) when varlen, says which appended keys each new token sees; it is
    passed on every rank, since it also sets the rotary positions of q.  With ``prefix_block_table``
    (P, max_prefix_blocks) int32 the prefix caches are a page pool, possibly ``k_cache`` / ``v_cache`` themselves: they
    stay out of ``mutates_args`` because the op never writes them (appends land in the suffix's pages only)."""
    pg = resolve_group(group)
    rank, world = group_info(pg)
    if k is not None and not 0 <= append_rank < world:
        raise ValueError(f"append_rank={append_rank} is not a rank of the {world}-rank group")
    if rank != append_rank:
        k = v = None
    if _kernel_takes(q):
        return kernel_decode(q, k_cache, v_cache, cache_seqlens, k, v, causal, softmax_scale, pg, world,
                             block_table=block_table, k_descale=k_descale, v_descale=v_descale,
                             cu_seqlens_q=cu_seqlens_q, max_seqlen_q=max_seqlen_q, rotary_cos=rotary_cos,
                             rotary_sin=rotary_sin, rotary_seqlens=rotary_seqlens,
                             rotary_interleaved=rotary_interleaved, q_descale=q_descale,
                             cache_batch_idx=cache_batch_idx, cache_leftpad=cache_leftpad,
                             prefix_k_cache=prefix_k_cache, prefix_v_cache=prefix_v_cache,
                             prefix_seqlens=prefix_seqlens, prefix_k_descale=prefix_k_descale,
                             prefix_v_descale=prefix_v_descale, tree_mask=tree_mask,
                             prefix_block_table=prefix_block_table)
    rotary = None if rotary_cos is None else (rotary_cos, rotary_sin, rotary_seqlens, rotary_interleaved)
    prefix = None if prefix_k_cache is None else (prefix_k_cache, prefix_v_cache, prefix_seqlens, prefix_k_descale,
                                                  prefix_v_descale, prefix_block_table)
    return _dense_decode(q, k_cache, v_cache, cache_seqlens, k, v, causal, softmax_scale, pg, world, block_table,
                         k_descale, v_descale, cu_seqlens_q, max_seqlen_q, rotary, q_descale, cache_batch_idx,
                         cache_leftpad, prefix, None if tree_mask is None else tree_mask.view(-1, tree_mask.shape[-1]))


@cp_decode.register_fake
def _(q, k_cache, v_cache, cache_seqlens, k, v, append_rank, softmax_scale, causal, group, block_table, k_descale,
      v_descale, cu_seqlens_q, max_seqlen_q, rotary_cos=None, rotary_sin=None, rotary_seqlens=None,
      rotary_interleaved=True, q_descale=None, cache_batch_idx=None, cache_leftpad=None, prefix_k_cache=None,
      prefix_v_cache=None, prefix_seqlens=None, prefix_k_descale=None, prefix_v_descale=None, tree_mask=None,
      prefix_block_table=None):
    out = q.new_empty(q.shape, dtype=_out_dtype(q))
    if cu_seqlens_q is not None:
        total_q, hq, _ = q.shape
        return out, q.new_empty((hq, total_q), dtype=torch.float32)
    b, sq, hq, _ = q.shape
    return out, q.new_empty((b, hq, sq), dtype=torch.float32)


def _valid_page_size(ps: int) -> bool:
    return ps in (16, 32, 64) or (ps > 0 and ps % KEY_TILE == 0)


def _check_block_table(q, k_cache, v_cache, block_table, b, name="block_table", rows="B", blocks="max_blocks"):
    if (block_table.dtype != torch.int32 or block_table.dim() != 2 or block_table.shape[0] != b
            or block_table.shape[1] < 1 or block_table.stride(1) != 1):
        raise ValueError(f"{name} must be a ({rows}, {blocks}) int32 tensor with stride(1) == 1")
    if block_table.device != q.device:
        raise ValueError(f"{name} must be on q's device")
    n_blocks, ps = k_cache.shape[:2]
    if not _valid_page_size(ps):
        raise ValueError(f"page_size {ps} is not supported: use 16, 32, 64 or a positive multiple of 128")
    for c in (k_cache, v_cache):
        if c.stride(0) != ps * c.stride(1) or c.stride(3) != 1:
            raise ValueError("the page pools must be mergeable: stride(0) == page_size * stride(1), stride(3) == 1")
    if n_blocks * ps >= 2 ** 31 or block_table.shape[1] * ps >= 2 ** 31:
        raise ValueError(f"num_blocks * page_size and {blocks} * page_size must be below 2^31")


def _check_descale(name, x, q, b, hkv):
    """An fp8 cache's descale as the contiguous (B, Hkv) fp32 tensor the kernels read."""
    if x is None:
        raise ValueError(f"fp8 caches need {name} (fp32, shape (), (Hkv,) or (B, Hkv))")
    if not isinstance(x, Tensor) or x.dtype != torch.float32:
        raise ValueError(f"fp8 {name} must be a float32 tensor")
    if x.device != q.device:
        raise ValueError(f"fp8 {name} must be on q's device")
    if tuple(x.shape) not in ((), (hkv,), (b, hkv)):
        raise ValueError(f"fp8 {name} must have shape (), (Hkv,) or (B, Hkv) = {(b, hkv)}, not {tuple(x.shape)}")
    return x.expand(b, hkv).contiguous()


def _check_cache_index(name, x, q, b):
    if (not isinstance(x, Tensor) or x.dtype != torch.int32 or tuple(x.shape) != (b,) or not x.is_contiguous()):
        raise ValueError(f"{name} must be a contiguous (B,) = ({b},) int32 tensor")
    if x.device != q.device:
        raise ValueError(f"{name} must be on q's device")


def _check_prefix(q, k_cache, pk, pv, pseq, pkd, pvd, b, hkv, d, pbt=None):
    """Checks the shared prefixes (a page pool with ``pbt``, the prefix block table) and returns their descales as
    the contiguous (P, Hkv) fp32 tensors the kernels read (None for bf16 / fp16 caches)."""
    if pk is None or pv is None or pseq is None:
        raise ValueError("pass prefix_k_cache, prefix_v_cache and prefix_seqlens together"
                         + (" (prefix_block_table names pages of the prefix caches)" if pbt is not None else ""))
    if q.dtype == torch.float8_e4m3fn:
        raise ValueError("a shared prefix needs a bf16 / fp16 q: q_descale varies per sequence inside a packed prefix "
                         "tile, which fp8 (e4m3) queries with a prefix do not support")
    paged = pbt is not None
    for name, x, c in (("prefix_k_cache", pk, k_cache), ("prefix_v_cache", pv, k_cache)):
        if not isinstance(x, Tensor) or x.dim() != 4 or not (paged or x.is_contiguous()):
            raise ValueError(f"{name} must be a (num_blocks, page_size, Hkv, D) page pool with prefix_block_table"
                             if paged else f"{name} must be a contiguous (P, P_cap, Hkv, D) tensor")
        if x.dtype != c.dtype:
            raise ValueError(f"{name} must have the cache's dtype ({c.dtype}), not {x.dtype}")
    if pk.shape != pv.shape or tuple(pk.shape[2:]) != (hkv, d):
        raise ValueError(f"prefix_k_cache {tuple(pk.shape)} and prefix_v_cache {tuple(pv.shape)} must both be "
                         f"{'(num_blocks, page_size' if paged else '(P, P_cap'}, Hkv, D) with (Hkv, D) = {(hkv, d)}")
    if paged:
        if not isinstance(pbt, Tensor) or pbt.dim() != 2 or pbt.shape[0] < 1:
            raise ValueError("prefix_block_table must be a (P, max_prefix_blocks) int32 tensor with stride(1) == 1")
        _check_block_table(q, pk, pv, pbt, pbt.shape[0], "prefix_block_table", "P", "max_prefix_blocks")
        if pk.stride() != pv.stride():
            raise ValueError("the prefix page pools must have the same strides")
        n_prefix, p_cap = pbt.shape[0], _capacity(pk, pbt)
    else:
        n_prefix, p_cap = pk.shape[:2]
        if n_prefix < 1 or p_cap < 1 or n_prefix * p_cap >= 2 ** 31:
            raise ValueError(f"prefix caches: P = {n_prefix} and P_cap = {p_cap} must be >= 1 with P * P_cap < 2^31")
    if pk.device != q.device or pv.device != q.device:
        raise ValueError("prefix_k_cache / prefix_v_cache must be on q's device")
    if b % n_prefix != 0:
        raise ValueError(f"the batch (B = {b}) must be a multiple of the prefix count (P = {n_prefix}): sequence b "
                         "uses prefix b // (B // P)")
    if (not isinstance(pseq, Tensor) or pseq.dtype != torch.int32 or tuple(pseq.shape) != (n_prefix,)
            or not pseq.is_contiguous()):
        raise ValueError(f"prefix_seqlens must be a contiguous (P,) = ({n_prefix},) int32 tensor")
    if pseq.device != q.device:
        raise ValueError("prefix_seqlens must be on q's device")
    if k_cache.dtype != torch.float8_e4m3fn:
        if pkd is not None or pvd is not None:
            raise ValueError("prefix_k_descale / prefix_v_descale are only taken with fp8 (float8_e4m3fn) caches")
        return None, None
    out = []
    for name, x in (("prefix_k_descale", pkd), ("prefix_v_descale", pvd)):
        if x is None:
            raise ValueError(f"fp8 prefix caches need {name} (fp32, shape (), (Hkv,) or (P, Hkv))")
        if not isinstance(x, Tensor) or x.dtype != torch.float32 or x.device != q.device:
            raise ValueError(f"fp8 {name} must be a float32 tensor on q's device")
        if tuple(x.shape) not in ((), (hkv,), (n_prefix, hkv)):
            raise ValueError(f"fp8 {name} must have shape (), (Hkv,) or (P, Hkv) = {(n_prefix, hkv)}, not "
                             f"{tuple(x.shape)}")
        out.append(x.expand(n_prefix, hkv).contiguous())
    return tuple(out)


def _check_rotary(cos, sin, rotary_seqlens, q, b, d, cache_seqlens, group):
    """Checks the rotary tables and returns the (B,) positions the kernels read: ``rotary_seqlens``, or
    ``cache_seqlens`` in a one-rank group."""
    if cos is None or sin is None:
        raise ValueError("pass both rotary_cos and rotary_sin, or neither")
    for name, x in (("rotary_cos", cos), ("rotary_sin", sin)):
        if not isinstance(x, Tensor) or x.dim() != 2 or not x.is_contiguous():
            raise ValueError(f"{name} must be a contiguous (seqlen_ro, rotary_dim / 2) tensor")
        if x.dtype != q.dtype:
            raise ValueError(f"{name} must have q's dtype ({q.dtype}), not {x.dtype}")
        if x.device != q.device:
            raise ValueError(f"{name} must be on q's device")
    if cos.shape != sin.shape:
        raise ValueError(f"rotary_cos {tuple(cos.shape)} and rotary_sin {tuple(sin.shape)} must have the same shape")
    rotary_dim = 2 * cos.shape[1]
    if rotary_dim == 0 or rotary_dim % 16 != 0 or rotary_dim > d:
        raise ValueError(f"rotary_dim = 2 * rotary_cos.shape[1] = {rotary_dim} must be a positive multiple of 16 "
                         f"and at most head_dim = {d}")
    if not 1 <= cos.shape[0] < 2 ** 31:
        raise ValueError(f"rotary_cos must have between 1 and 2^31 - 1 rows, not {cos.shape[0]}")
    if rotary_seqlens is None:
        if group_info(resolve_group(group_name(group)))[1] > 1:
            raise ValueError("rotary_seqlens is required in a group of more than one rank: cache_seqlens are the "
                             "lengths of this rank's shard, not the positions of the new tokens")
        return cache_seqlens
    if (not isinstance(rotary_seqlens, Tensor) or rotary_seqlens.dtype != torch.int32
            or tuple(rotary_seqlens.shape) != (b,) or not rotary_seqlens.is_contiguous()):
        raise ValueError(f"rotary_seqlens must be a contiguous (B,) = ({b},) int32 tensor")
    if rotary_seqlens.device != q.device:
        raise ValueError("rotary_seqlens must be on q's device")
    return rotary_seqlens


MAX_TREE_TOKENS = 128  # new tokens per sequence with a tree mask: they span at most two key tiles


def _check_tree_mask(tree_mask, q, k, causal, shape):
    if k is None:
        raise ValueError("tree_mask needs k / v: it says which of the keys this call appends each new token sees")
    if not causal:
        raise ValueError("tree_mask replaces the causal rule among the appended keys: it needs causal=True")
    if not isinstance(tree_mask, Tensor) or tree_mask.dtype != torch.bool:
        raise ValueError("tree_mask must be a torch.bool tensor")
    if tuple(tree_mask.shape) != tuple(shape) or not tree_mask.is_contiguous():
        raise ValueError(f"tree_mask must be contiguous with shape {tuple(shape)} ((B, Sq, Sq), or (total_q, "
                         f"max_seqlen_q) with cu_seqlens_q), not {tuple(tree_mask.shape)}")
    if tree_mask.device != q.device:
        raise ValueError("tree_mask must be on q's device")
    if shape[-1] > MAX_TREE_TOKENS:
        raise ValueError(f"tree_mask takes at most {MAX_TREE_TOKENS} new tokens per sequence, not {shape[-1]}")


def cp_flash_attn_with_kvcache(q, k_cache, v_cache, cache_seqlens, k=None, v=None, append_rank=None,
                               softmax_scale=None, causal=True, return_softmax_lse=False, group=None, *,
                               block_table=None, k_descale=None, v_descale=None, cu_seqlens_q=None,
                               max_seqlen_q=None, rotary_cos=None, rotary_sin=None, rotary_interleaved=True,
                               rotary_seqlens=None, window_size=(-1, -1), alibi_slopes=None, q_descale=None,
                               cache_batch_idx=None, cache_leftpad=None, prefix_k_cache=None, prefix_v_cache=None,
                               prefix_seqlens=None, prefix_k_descale=None, prefix_v_descale=None, tree_mask=None,
                               prefix_block_table=None):
    """Decode attention of new query tokens against a KV cache sharded over ``group`` (modelled on flash-attn's
    ``flash_attn_with_kvcache``).  Inference only: no gradient.

    * ``q`` ``(B, Sq, Hq, D)``, the same on every rank; ``Sq >= 1`` (one token, or a few speculative ones).
    * ``k_cache`` / ``v_cache`` ``(B, S_cap, Hkv, D)``: this rank's shard, in any row order (the local K / V of a
      ring / zigzag / stripe / llama3 / zigzag-llama3 prefill can be used as is).  Batch and sequence dimensions must
      be mergeable (``stride(0) == S_cap * stride(1)``).
    * ``block_table`` ``(B, max_blocks)`` int32 on q's device (``stride(1) == 1``), optional: the cache is paged.
      ``k_cache`` / ``v_cache`` are then this rank's page pool ``(num_blocks, page_size, Hkv, D)``, with
      ``stride(0) == page_size * stride(1)``, and row ``j`` of sequence ``b`` lives at row ``j % page_size`` of page
      ``block_table[b, j // page_size]``.  Each rank has its own pool and table.  ``S_cap`` is
      ``max_blocks * page_size``; ``page_size`` is 16, 32, 64 or a positive multiple of 128, and
      ``num_blocks * page_size < 2**31``.  Entries of pages that hold no visible row are never read (-1 is fine).
      On the append rank the caller allocates the pages of rows ``[0, cache_seqlens[b] + Sq)`` before the call.
      An entry outside the pool for a page that is read is a caller error: the kernel's result is then undefined,
      but it never accesses memory outside the pool (the dense path raises ``ValueError``).
    * fp8 caches: ``k_cache`` / ``v_cache`` may both be ``torch.float8_e4m3fn`` (contiguous or paged), with a bf16 /
      fp16 ``q``.  ``k_descale`` / ``v_descale`` are then required: fp32 tensors on q's device of shape ``()``,
      ``(Hkv,)`` or ``(B, Hkv)``, and the cache stands for ``k_cache.float() * k_descale[b, h]`` (the same for V).
      Each rank passes the descales of its own shard; ranks may differ.  They are read on the device only (a CUDA
      graph replay uses their current contents) and are not validated: non-finite or non-positive descales give an
      undefined result.  The appended ``k`` / ``v`` stay in q's dtype and are stored as
      ``(x.float() / descale).clamp(-448, 448).to(torch.float8_e4m3fn)``.  An e4m3 cache holds twice the tokens of
      a bf16 one and a decode step reads half the bytes.  Descales given with a bf16 / fp16 cache, ``float8_e5m2``
      caches, mixed cache dtypes and fp8 caches with an fp32 ``q`` raise ``ValueError``.
    * fp8 queries (flash-attn 3's ``q_descale``): over e4m3 caches, ``q`` may be ``torch.float8_e4m3fn``, with
      ``q_descale`` required: an fp32 tensor on q's device of shape ``()``, ``(Hkv,)`` or ``(B, Hkv)``, the same on
      every rank.  The query stands for ``q.float() * q_descale[b, h // G]``, and ``out`` is bf16.  The kernel runs
      ``Q K^T`` as an e4m3 tensor-core product straight on the cache's fp8 K tiles and widens only V.  ``q_descale``
      is read on the device only (a CUDA graph replay uses its current contents) and is not validated.  With an e4m3
      ``q``, ``k`` / ``v`` may be ``torch.float8_e4m3fn`` (both): their bytes are stored as they are, and they stand
      for ``k.float() * k_descale`` like the cache; bf16 / fp16 ``k`` / ``v`` are quantised as above.  ``q_descale``
      with a bf16 / fp16 ``q``, an e4m3 ``q`` without it or over a bf16 / fp16 cache, a ``float8_e5m2`` ``q`` and
      rotary with an e4m3 ``q`` (rotate before quantising) raise ``ValueError``.
    * ``cache_seqlens`` ``(B,)`` int32 on q's device: valid rows of this rank's shard (0 = empty shard).
    * ``cache_batch_idx`` ``(B,)`` int32 on q's device, contiguous, optional (flash-attn's argument): sequence ``b``
      reads and appends slot ``cache_batch_idx[b]`` of ``(B_cache, S_cap, Hkv, D)`` caches, for any
      ``B_cache >= 1`` with ``B_cache * S_cap < 2**31`` (a pool of slots decoded a changing subset at a time, or
      several sequences reading one shared prompt).  ``cache_seqlens``, ``cache_leftpad``, the descales and
      ``rotary_seqlens`` stay indexed by ``b``, not by the slot.  Slots not named are never read or written.
      Duplicate indices are allowed; with ``k`` / ``v``, which duplicate's rows land in the shared slot is
      unspecified.  Each rank passes its own.  Not with ``block_table`` (the table already gives every sequence
      its own pages).
    * ``cache_leftpad`` ``(B,)`` int32 on q's device, contiguous, optional (flash-attn's argument): the keys of
      sequence ``b`` are rows ``[cache_leftpad[b], cache_seqlens[b])`` of its slot plus the appended rows, which
      still start at ``cache_seqlens[b]``; rows below the pad may hold anything, NaN included, and are never loaded.
      A left-padded batch prefilled with the ring, zigzag or stripe layout keeps its pad tokens in a leading row
      range of every shard, so each rank passes the count of its own pad rows.  Rotary positions do not change.
      Not with ``block_table``.  The kernel path reads both tensors on the device only (a CUDA graph replay uses
      their current contents) and does not validate them: an index outside ``[0, B_cache)`` or a pad outside
      ``[0, cache_seqlens[b]]`` gives an undefined result but no access outside the caches (the sequence sees no key
      on this rank and its append is dropped; the pad is clamped).  The dense path raises ``ValueError`` for both.
    * Shared prefixes (one long prompt, many continuations: best-of-n, parallel sampling, RL rollouts, one system
      prompt under many requests): ``prefix_k_cache`` / ``prefix_v_cache`` ``(P, P_cap, Hkv, D)``, contiguous, in the
      dtype of ``k_cache`` / ``v_cache``, are this rank's shard of ``P >= 1`` prompts, with ``B % P == 0`` and
      ``P * P_cap < 2**31``.  Sequence ``b`` uses prefix ``b // (B // P)``: the ``B / P`` samples of a prompt are
      consecutive (``repeat_interleave`` order).  ``prefix_seqlens`` ``(P,)`` int32 on q's device, contiguous, gives
      the valid rows of each prefix shard on this rank (0 is allowed); each rank passes its own.  With e4m3 caches
      ``prefix_k_descale`` / ``prefix_v_descale`` (fp32, ``()``, ``(Hkv,)`` or ``(P, Hkv)``) are required, as
      ``k_descale`` is.  On this rank sequence ``b`` sees rows ``[0, prefix_seqlens[p])`` of its prefix, visible to
      every query token with or without ``causal``, followed by everything it sees without a prefix: its own cache
      (slots, left pad, pages, e4m3), and the appended tokens under the causal rule.  ``k`` / ``v`` go to the
      sequence's own cache; the prefix is never written.  ``cache_seqlens`` still counts the sequence's own rows
      (0 is allowed).  The result is that of a plain call on a cache holding the prefix rows followed by the
      sequence's rows, up to fp32 summation order; rotary positions are those of that plain call, so in a one-rank
      group ``rotary_seqlens`` defaults to ``prefix_seqlens[p] + cache_seqlens[b]``.  The kernel runs a second pass in
      which the query rows of a prompt's samples share one 64-row tile and each prefix K / V tile is read once for all
      of them; its partials merge with the suffix pass's in the one combine.  ``prefix_seqlens`` is read on the device
      only and clamped to ``[0, P_cap]`` (a CUDA graph replay uses its current contents); the dense path raises
      ``ValueError`` for a value outside that range.  Missing pieces, shape / dtype / device / contiguity mismatches,
      ``B % P != 0`` and an e4m3 ``q`` with a prefix (``q_descale`` would vary inside a packed prefix tile) raise
      ``ValueError``.  Prefixes shared by non-consecutive sequences and nested prefixes are not supported.
    * Paged prefixes: ``prefix_block_table`` ``(P, max_prefix_blocks)`` int32 on q's device (``stride(1) == 1``),
      optional, follows the rules of ``block_table``.  ``prefix_k_cache`` / ``prefix_v_cache`` are then this rank's
      page pool ``(num_blocks, page_size, Hkv, D)``, with ``stride(0) == page_size * stride(1)``, in the dtype of
      ``k_cache``; ``page_size`` is 16, 32, 64 or a positive multiple of 128, and ``num_blocks * page_size < 2**31``.
      Row ``j`` of prefix ``p`` lives at row ``j % page_size`` of page ``prefix_block_table[p, j // page_size]``.
      ``P`` is ``prefix_block_table.shape[0]`` and ``P_cap`` is ``max_prefix_blocks * page_size``; ``prefix_seqlens``
      and the prefix descales keep their shapes.  The pool may be the very tensors ``k_cache`` / ``v_cache`` of a
      paged call (one pool per rank, the prompt's pages named in ``prefix_block_table`` and each sample's own pages
      in ``block_table``, as paged serving engines keep them), or a pool of its own beside a contiguous suffix cache,
      with or without ``cache_batch_idx`` / ``cache_leftpad``.  Appends go to the suffix only, before either pass
      reads; a sample whose appended rows land in a page of its prompt is a caller error (the prompt's rows are then
      overwritten).  Entries of pages that hold no visible prefix row are never read (-1 is fine).  An entry outside
      the pool for a page that is read gives an undefined result on the kernel path, but no access outside the pool;
      the dense path raises ``ValueError``.  The kernel path reads the table on the device only (a CUDA graph replay
      uses its current contents).  The result is bitwise that of the contiguous prefix call on the same rows at equal
      ``P_cap`` and split counts.
    * ``k`` / ``v`` ``(B, Sq, Hkv, D)``, optional, the same on every rank: written in place into the caches of rank
      ``append_rank`` only, at rows ``[cache_seqlens[b], cache_seqlens[b] + Sq)``, before attention (rows past
      ``S_cap`` are dropped).  The caller advances ``cache_seqlens``.  ``append_rank`` is required with ``k`` / ``v``
      and must be ``None`` without them; it must be the same int on every rank (e.g. ``step % world``).
    * Query token ``t`` sees every valid cached key of every rank and, with ``causal=True``, the appended keys
      ``0..t`` of its own call (flash-attn's bottom-right alignment); with ``causal=False`` all ``Sq`` of them.
    * Varlen queries (flash-attn's ``cu_seqlens_q`` / ``max_seqlen_q``): every sequence may bring a different
      number of new tokens.  ``q`` is then ``(total_q, Hq, D)``, and sequence ``b`` owns rows
      ``cu_seqlens_q[b]:cu_seqlens_q[b + 1]`` (0 rows is allowed); ``B`` is ``cache_seqlens.shape[0]`` and
      ``cu_seqlens_q`` a contiguous ``(B + 1,)`` int32 tensor on q's device, the same on every rank.  ``max_seqlen_q``
      (a host int >= 1, required with ``cu_seqlens_q`` and rejected without it) bounds every count.  ``k`` / ``v``
      are ``(total_q, Hkv, D)`` with the same row ranges; sequence ``b``'s ``n_b`` rows go to cache rows
      ``[cache_seqlens[b], cache_seqlens[b] + n_b)``.  ``out`` is ``(total_q, Hq, D)`` and ``softmax_lse``
      ``(Hq, total_q)`` (flash-attn's varlen layout).  Masking is per sequence, as above, with ``n_b`` for ``Sq``.
      Composes with ``block_table`` and e4m3 caches.  The kernel path reads ``cu_seqlens_q`` on the device only (a
      step with fixed ``total_q`` / ``max_seqlen_q`` can be captured in a CUDA graph, and a replay uses the current
      contents) and does not validate it: malformed values give an undefined result for the affected rows, but no
      access outside ``q``, ``k``, ``v`` or the caches.  The dense path raises ``ValueError`` for them
      (``cu_seqlens_q[0] != 0``, a decreasing entry, ``cu_seqlens_q[B] != total_q``, a count above
      ``max_seqlen_q``).  Long chunks are correct but not efficient: every 64-row tile reads the whole shard.
    * Tree attention (speculative decoding: EAGLE, Medusa and other draft trees verified in one call):
      ``tree_mask``, a contiguous ``torch.bool`` tensor on q's device, the same on every rank, of shape
      ``(B, Sq, Sq)``, or ``(total_q, max_seqlen_q)`` with ``cu_seqlens_q``.  Its rows are the packed query rows and
      column ``u`` is new key ``u`` of the row's own sequence (in a varlen call columns at or past ``n_b`` are
      ignored): new token ``t`` of sequence ``b`` sees appended key ``u`` iff ``tree_mask[row(b, t), u]``.  This
      replaces the causal rule among the appended keys only; every valid cached key (own cache, prefix, pages, slots,
      left pad) stays visible to every new token.  Any boolean matrix is accepted; a tree's ancestor mask (ancestors
      plus the node itself) is the intended use, and a lower-triangular mask gives exactly the causal call.  It needs
      ``k`` / ``v``, ``causal=True`` and at most 128 new tokens per sequence.  With rotary, new token ``t`` (query and
      key) sits at ``rotary_seqlens[b] + max(n_t - 1, 0)``, ``n_t`` being the True entries of its row: a node's depth
      in a tree, and ``t`` for a lower-triangular mask.  Node ``u`` is still appended at row
      ``cache_seqlens[b] + u`` of the append rank; keeping the accepted nodes (moving their rows to
      ``cache_seqlens[b] + [0, n_accepted)``) and advancing ``cache_seqlens`` is the caller's job.  The kernel path
      reads the mask on the device only and never validates it, so a CUDA graph replay uses its current contents.
      Masks over cached keys, a mask without ``causal`` and bit-packed masks are not supported; a wrong dtype,
      shape, device or contiguity raises ``ValueError``.
    * Returns ``out`` ``(B, Sq, Hq, D)`` in q.dtype (bf16 for an e4m3 ``q``), and ``softmax_lse`` ``(B, Hq, Sq)``
      fp32 when ``return_softmax_lse``.  Both are bitwise identical on every rank.
    * ``window_size``, ``alibi_slopes``, ``D > 128`` and ``Hq % Hkv != 0`` raise ``ValueError``.  The sm_90a kernel
      covers a bf16 / fp16 ``q`` with ``D`` in {64, 128}, over caches in q's dtype or e4m3, and an e4m3 ``q`` over
      e4m3 caches; other head sizes run the dense torch path with a one-time warning (an e4m3 ``q`` dequantised with
      ``q_descale``).
    * Rotary embeddings (flash-attn's ``rotary_cos`` / ``rotary_sin`` / ``rotary_interleaved``, and flash-attn 3's
      ``rotary_seqlens``): ``rotary_cos`` / ``rotary_sin`` are contiguous ``(seqlen_ro, rotary_dim / 2)`` tensors in
      q's dtype on q's device, the same on every rank; ``rotary_dim`` is a multiple of 16 and at most ``D``, and
      columns at or past it are left as they are.  ``rotary_interleaved=True`` pairs columns ``(2i, 2i + 1)``
      (GPT-J), ``False`` pairs ``i`` and ``i + rotary_dim / 2`` (GPT-NeoX / Llama).  ``rotary_seqlens`` ``(B,)``
      int32 on q's device, the same on every rank, is the global position of each sequence's first new token: new key
      ``t`` of sequence ``b`` is rotated at ``rotary_seqlens[b] + t``, and query token ``t`` there too when
      ``causal``, at ``rotary_seqlens[b]`` otherwise (``t`` counts from ``cu_seqlens_q[b]`` in a varlen call).
      ``cache_seqlens`` are shard lengths, not positions, so ``rotary_seqlens`` is required in a group of more than
      one rank; in a one-rank group it defaults to ``cache_seqlens`` (flash-attn's rule).  Rotary needs ``k`` /
      ``v``.  The appended ``k`` is stored rotated (for an e4m3 cache, rotated, rounded to q's dtype, then
      quantised).  The rotation is :func:`apply_rotary`'s exactly, so a call is bitwise a call without rotary on
      rotated ``q`` / ``k``.  The kernel path reads ``rotary_seqlens`` on the device only (a CUDA graph replay uses
      its current contents) and clamps every position to ``[0, seqlen_ro - 1]``; the dense path raises
      ``ValueError`` for a position outside the tables.  Malformed tables or ``rotary_seqlens`` (one of cos / sin,
      shapes, dtype, device, ``rotary_dim``) raise ``ValueError``.
    * Nothing is read back to the host on the kernel path, so a decode step can be captured in a CUDA graph."""
    if tuple(window_size) != (-1, -1):
        raise ValueError("cp_flash_attn_with_kvcache: sliding windows are not supported in decode")
    if alibi_slopes is not None:
        raise ValueError("cp_flash_attn_with_kvcache: alibi_slopes are not supported in decode")
    varlen = cu_seqlens_q is not None
    if varlen:
        if q.dim() != 3:
            raise ValueError(f"with cu_seqlens_q, q must be (total_q, Hq, D), not {tuple(q.shape)}")
        if max_seqlen_q is None:
            raise ValueError("max_seqlen_q is required with cu_seqlens_q")
        if isinstance(max_seqlen_q, bool) or not isinstance(max_seqlen_q, int) or max_seqlen_q < 1:
            raise ValueError(f"max_seqlen_q must be a host int >= 1, not {max_seqlen_q!r}")
        if not isinstance(cache_seqlens, Tensor) or cache_seqlens.dim() != 1:
            raise ValueError("cache_seqlens must be a (B,) int32 tensor on q's device")
    else:
        if max_seqlen_q is not None:
            raise ValueError("max_seqlen_q is only taken with cu_seqlens_q")
        if q.dim() == 3:
            raise ValueError("a 3-D (total_q, Hq, D) q needs cu_seqlens_q")
    if q.dim() != (3 if varlen else 4) or k_cache.dim() != 4 or tuple(k_cache.shape) != tuple(v_cache.shape):
        raise ValueError("q must be (B, Sq, Hq, D) and k_cache / v_cache the same (B, S_cap, Hkv, D) shape")
    if varlen:
        b, sq = cache_seqlens.shape[0], max_seqlen_q
        total_q, hq, d = q.shape
    else:
        b, sq, hq, d = q.shape
    hkv = k_cache.shape[2]
    if block_table is not None and cache_batch_idx is not None:
        raise ValueError("cache_batch_idx takes a contiguous cache: a paged cache does not support cache_batch_idx "
                         "(the block table already gives every sequence its own pages)")
    if block_table is not None and cache_leftpad is not None:
        raise ValueError("cache_leftpad takes a contiguous cache: a paged cache does not support cache_leftpad")
    if cache_batch_idx is not None:
        _check_cache_index("cache_batch_idx", cache_batch_idx, q, b)
        if k_cache.shape[0] < 1 or k_cache.shape[0] * k_cache.shape[1] >= 2 ** 31:
            raise ValueError(f"with cache_batch_idx, B_cache * S_cap = {k_cache.shape[0]} * {k_cache.shape[1]} must "
                             "be between 1 and 2^31 - 1")
    if cache_leftpad is not None:
        _check_cache_index("cache_leftpad", cache_leftpad, q, b)
    if ((block_table is None and cache_batch_idx is None and k_cache.shape[0] != b) or k_cache.shape[3] != d
            or sq < 1):
        raise ValueError(f"q {tuple(q.shape)} does not match the cache {tuple(k_cache.shape)}")
    if varlen and (not isinstance(cu_seqlens_q, Tensor) or cu_seqlens_q.dtype != torch.int32
                   or tuple(cu_seqlens_q.shape) != (b + 1,) or not cu_seqlens_q.is_contiguous()):
        raise ValueError(f"cu_seqlens_q must be a contiguous (B + 1,) = ({b + 1},) int32 tensor")
    if varlen and cu_seqlens_q.device != q.device:
        raise ValueError("cu_seqlens_q must be on q's device")
    q8 = q.dtype == torch.float8_e4m3fn
    if q.element_size() == 1 and not q8:
        raise ValueError(f"cp_flash_attn_with_kvcache: fp8 queries must be torch.float8_e4m3fn, not {q.dtype}")
    if q8 and not (k_cache.dtype == v_cache.dtype == torch.float8_e4m3fn):
        raise ValueError("cp_flash_attn_with_kvcache: fp8 (e4m3) queries need e4m3 caches, not "
                         f"{k_cache.dtype} / {v_cache.dtype}")
    if q8:
        if q_descale is None:
            raise ValueError("cp_flash_attn_with_kvcache: fp8 queries (e4m3) need q_descale (fp32, shape (), (Hkv,) "
                             "or (B, Hkv))")
        q_descale = _check_descale("q_descale", q_descale, q, b, hkv)
    elif q_descale is not None:
        raise ValueError("q_descale is only taken with an fp8 (float8_e4m3fn) q")
    if k_cache.element_size() == 1 or v_cache.element_size() == 1:
        if k_cache.dtype != v_cache.dtype:
            raise ValueError(f"fp8 caches: k_cache ({k_cache.dtype}) and v_cache ({v_cache.dtype}) must both be "
                             "torch.float8_e4m3fn")
        if k_cache.dtype != torch.float8_e4m3fn:
            raise ValueError(f"fp8 caches must be torch.float8_e4m3fn, not {k_cache.dtype}")
        if q.dtype not in (torch.bfloat16, torch.float16, torch.float8_e4m3fn):
            raise ValueError(f"fp8 caches need a bf16 / fp16 q, or an e4m3 q with q_descale, not {q.dtype}")
        k_descale = _check_descale("k_descale", k_descale, q, b, hkv)
        v_descale = _check_descale("v_descale", v_descale, q, b, hkv)
    else:
        if k_cache.dtype != q.dtype or v_cache.dtype != q.dtype:
            raise ValueError("k_cache / v_cache must have q's dtype")
        if k_descale is not None or v_descale is not None:
            raise ValueError("k_descale / v_descale are only taken with fp8 (float8_e4m3fn) caches")
    if d > 128:
        raise ValueError(f"cp_flash_attn_with_kvcache: head_dim {d} > 128 is not supported")
    if hq % hkv != 0:
        raise ValueError(f"query heads ({hq}) must be a multiple of kv heads ({hkv})")
    if (cache_seqlens.dtype != torch.int32 or tuple(cache_seqlens.shape) != (b,)
            or cache_seqlens.device != q.device):
        raise ValueError("cache_seqlens must be a (B,) int32 tensor on q's device")
    if block_table is not None:
        _check_block_table(q, k_cache, v_cache, block_table, b)
    if (k is None) != (v is None):
        raise ValueError("pass both k and v, or neither")
    if k is not None:
        if append_rank is None:
            raise ValueError("append_rank is required when k / v are given")
        if q8:  # pre-quantised e4m3 k / v (stored as they are), or bf16 / fp16 ones (quantised as they are stored)
            if k.dtype != v.dtype or k.dtype not in (torch.float8_e4m3fn, torch.bfloat16, torch.float16):
                raise ValueError(f"with an e4m3 q, k / v must both be float8_e4m3fn, bf16 or fp16, not {k.dtype} / "
                                 f"{v.dtype}")
        for t in (k, v):
            dtype_ok = t.dtype == k.dtype if q8 else t.dtype == q.dtype
            if varlen and (tuple(t.shape) != (total_q, hkv, d) or not dtype_ok):
                raise ValueError(f"with cu_seqlens_q, k / v must be (total_q, Hkv, D) = {(total_q, hkv, d)} in "
                                 "q's dtype")
            if not varlen and (tuple(t.shape) != (b, sq, hkv, d) or not dtype_ok):
                raise ValueError(f"k / v must be (B, Sq, Hkv, D) = {(b, sq, hkv, d)} in q's dtype")
    elif append_rank is not None:
        raise ValueError("append_rank must be None when no k / v are given")
    has_prefix = (prefix_k_cache is not None or prefix_v_cache is not None or prefix_seqlens is not None
                  or prefix_block_table is not None)
    if has_prefix:
        prefix_k_descale, prefix_v_descale = _check_prefix(q, k_cache, prefix_k_cache, prefix_v_cache, prefix_seqlens,
                                                           prefix_k_descale, prefix_v_descale, b, hkv, d,
                                                           prefix_block_table)
    elif prefix_k_descale is not None or prefix_v_descale is not None:
        raise ValueError("prefix_k_descale / prefix_v_descale are only taken with prefix_k_cache / prefix_v_cache")
    if rotary_cos is not None or rotary_sin is not None:
        if q8:
            raise ValueError("rotary_cos / rotary_sin need a bf16 / fp16 q: the rotation belongs before quantisation, "
                             "so rotate q and k, then quantise them")
        default_pos = rotary_seqlens is None
        rotary_seqlens = _check_rotary(rotary_cos, rotary_sin, rotary_seqlens, q, b, d, cache_seqlens, group)
        if default_pos and has_prefix:  # the keys before the new tokens: the prefix rows, then the sequence's own
            rotary_seqlens = (cache_seqlens + prefix_seqlens.repeat_interleave(b // prefix_seqlens.shape[0])).to(
                torch.int32)
        if k is None:
            raise ValueError("rotary_cos / rotary_sin need k / v: the rotation applies to the new tokens")
    elif rotary_seqlens is not None:
        raise ValueError("rotary_seqlens is only taken with rotary_cos / rotary_sin")
    if tree_mask is not None:
        _check_tree_mask(tree_mask, q, k, causal, (total_q, sq) if varlen else (b, sq, sq))
    scale = float(softmax_scale) if softmax_scale is not None else d ** -0.5
    out, lse = cp_decode(q, k_cache, v_cache, cache_seqlens, k, v, -1 if append_rank is None else int(append_rank),
                         scale, bool(causal), group_name(group), block_table, k_descale, v_descale, cu_seqlens_q,
                         max_seqlen_q if varlen else 0, rotary_cos, rotary_sin, rotary_seqlens,
                         bool(rotary_interleaved), q_descale, cache_batch_idx, cache_leftpad, prefix_k_cache,
                         prefix_v_cache, prefix_seqlens, prefix_k_descale, prefix_v_descale, tree_mask,
                         prefix_block_table)
    return (out, lse) if return_softmax_lse else out
