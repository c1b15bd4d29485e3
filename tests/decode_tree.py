"""Inputs and an fp64 oracle for decode calls with a tree mask (``tree_mask=``).

* :func:`random_parents`: a seeded random tree as a parent array (node 0 is the root, ``parents[i] < i``).
* :func:`ancestor_mask`: its ``(n, n)`` mask, True on a node's ancestors and on itself.
* :func:`depths`: every node's depth (the root's is 0), the rotary offset a tree call gives it.
* :func:`build`: one call's inputs over a chosen cache layout, with the logical (contiguous, dequantised) view the
  oracle reads.
* :func:`oracle`: the call's result straight from the definition, in fp64: new token ``t`` of sequence ``b`` sees the
  prefix rows, the cached rows ``[lp, seqlen)`` and the appended rows ``u`` with ``tree_mask[row(b, t), u]``.
"""
from __future__ import annotations

import itertools
from dataclasses import dataclass, field
from typing import List, Optional

import torch

from ring_flash_attn_b200.parallel import decode as dec

E4M3 = torch.float8_e4m3fn
LAYOUTS = ("contiguous", "paged16", "e4m3", "q8", "slots", "prefix")


def random_parents(n: int, gen: torch.Generator) -> List[int]:
    """A random tree of ``n`` nodes: node i > 0 hangs under a node drawn from [max(0, i - 6), i)."""
    return [-1] + [int(torch.randint(max(0, i - 6), i, (1,), generator=gen)) for i in range(1, n)]


def full_tree(widths) -> List[int]:
    """Parent array of the full tree in which every node at depth i has widths[i] children (breadth-first order)."""
    parents, level = [-1], [0]
    for w in widths:
        nxt = []
        for p in level:
            for _ in range(w):
                parents.append(p)
                nxt.append(len(parents) - 1)
        level = nxt
    return parents


def ancestor_mask(parents: List[int]) -> torch.Tensor:
    n = len(parents)
    m = torch.zeros(n, n, dtype=torch.bool)
    for i in range(n):
        j = i
        while j >= 0:
            m[i, j] = True
            j = parents[j]
    return m


def depths(parents: List[int]) -> List[int]:
    out = []
    for p in parents:
        out.append(0 if p < 0 else out[p] + 1)
    return out


def packed_mask(masks: List[torch.Tensor], sq: int, gen: torch.Generator, varlen: bool) -> torch.Tensor:
    """The call's tree_mask from per-sequence (n_b, n_b) masks: (total_q, sq), or (B, sq, sq) when uniform.  Columns
    at or past n_b hold random bits, which the call must ignore."""
    rows = []
    for m in masks:
        n = m.shape[0]
        r = torch.rand(n, sq, generator=gen) < 0.5
        r[:, :n] = m
        rows.append(r)
    out = torch.cat(rows) if rows else torch.zeros(0, sq, dtype=torch.bool)
    return out if varlen else out.view(len(masks), sq, sq)


def tree_masks(counts, gen: torch.Generator) -> List[torch.Tensor]:
    return [ancestor_mask(random_parents(n, gen)) if n else torch.zeros(0, 0, dtype=torch.bool) for n in counts]


def tril_masks(counts) -> List[torch.Tensor]:
    return [torch.ones(n, n, dtype=torch.bool).tril() for n in counts]


@dataclass
class Call:
    """One call's arguments (``q`` / ``k`` / ``v`` uniform or packed) and the logical view the oracle reads."""
    counts: tuple
    varlen: bool
    q: torch.Tensor
    k: torch.Tensor
    v: torch.Tensor
    k_cache: torch.Tensor
    v_cache: torch.Tensor
    seqlens: torch.Tensor
    kwargs: dict
    # logical view: contiguous fp64 caches before the append, pads, prefix rows, the new rows in q's dtype
    lk: torch.Tensor
    lv: torch.Tensor
    lens: List[int]
    pads: List[int]
    prefix_k: List[torch.Tensor] = field(default_factory=list)  # per sequence, fp64 (rows, Hkv, D)
    prefix_v: List[torch.Tensor] = field(default_factory=list)
    k_descale: Optional[torch.Tensor] = None  # (B, Hkv), e4m3 caches
    v_descale: Optional[torch.Tensor] = None
    q_descale: Optional[torch.Tensor] = None
    q_rows: Optional[torch.Tensor] = None  # (total_q, Hq, D) in bf16 / fp16 (before any quantisation)
    k_rows: Optional[torch.Tensor] = None
    v_rows: Optional[torch.Tensor] = None

    @property
    def spans(self):
        cu = [0] + list(itertools.accumulate(self.counts))
        return [(lo, n) for lo, n in zip(cu[:-1], self.counts)]

    def fresh(self):
        """(q, k_cache, v_cache, seqlens, k, v, kwargs) with fresh copies of the caches."""
        return (self.q, self.k_cache.clone(), self.v_cache.clone(), self.seqlens, self.k, self.v, dict(self.kwargs))


def _rows_to_call(x: torch.Tensor, counts, varlen: bool) -> torch.Tensor:
    return x if varlen else x.view(len(counts), counts[0], *x.shape[1:])


def build(layout: str, dtype, d: int, counts, seqlens, s_cap: int, device, seed: int = 0, hq: int = 8, hkv: int = 2,
          varlen: bool = True) -> Call:
    """Seeded inputs (drawn on the CPU) for one call over ``layout``: cached rows are finite, rows past them (and pad
    rows, and unused slots or pages) NaN.  ``varlen=False`` needs equal counts.  ``prefix`` needs an even B."""
    assert layout in LAYOUTS
    g = torch.Generator().manual_seed(seed)
    b, total = len(counts), sum(counts)
    assert varlen or len(set(counts)) == 1
    fp8 = layout in ("e4m3", "q8")
    kc, vc = (torch.randn(b, s_cap, hkv, d, generator=g) for _ in range(2))
    pads = [0] * b
    if layout == "slots":
        pads = [int(torch.randint(0, n + 1, (1,), generator=g)) for n in seqlens]
    for i, n in enumerate(seqlens):
        kc[i, n:] = vc[i, n:] = float("nan")
        kc[i, :pads[i]] = vc[i, :pads[i]] = float("nan")
    q_rows = torch.randn(total, hq, d, generator=g).to(dtype)
    k_rows, v_rows = (torch.randn(total, hkv, d, generator=g).to(dtype) for _ in range(2))
    kd = vd = qd = None
    kw = {}
    if fp8:
        kd = 0.3 * (1 + 0.1 * torch.arange(b * hkv, dtype=torch.float32)).view(b, hkv)
        vd = 0.45 * (1 + 0.05 * torch.arange(b * hkv, dtype=torch.float32)).view(b, hkv)
        kc8 = torch.stack([dec.quantize_e4m3(kc[i], kd[i]) for i in range(b)])
        vc8 = torch.stack([dec.quantize_e4m3(vc[i], vd[i]) for i in range(b)])
        lk = kc8.double() * kd.double()[:, None, :, None]
        lv = vc8.double() * vd.double()[:, None, :, None]
        kc, vc = kc8, vc8
        kw.update(k_descale=kd.to(device), v_descale=vd.to(device))
    else:
        kc, vc = kc.to(dtype), vc.to(dtype)
        lk, lv = kc.double(), vc.double()
    q = q_rows
    if layout == "q8":
        qd = 0.05 * (1 + 0.1 * torch.arange(b * hkv, dtype=torch.float32)).view(b, hkv)
        q = torch.cat([dec.quantize_e4m3(q_rows[lo:lo + n], qd[i].repeat_interleave(hq // hkv))
                       for i, (lo, n) in enumerate(_spans(counts))])
        kw.update(q_descale=qd.to(device))
    sl = torch.tensor(seqlens, dtype=torch.int32)
    k_cache, v_cache = kc, vc
    if layout == "paged16":
        from test_decode_paged import to_pool
        alloc = torch.tensor([min(n + c, s_cap) for n, c in zip(seqlens, counts)])
        k_cache, v_cache, table = to_pool(kc, vc, sl, 16, alloc=alloc, seed=seed)
        kw.update(block_table=table.to(device))
    elif layout == "slots":
        n_slots = b + 3
        idx = torch.randperm(n_slots, generator=g)[:b]
        shape = (n_slots,) + tuple(kc.shape[1:])
        k_cache = torch.full(shape, float("nan"), dtype=torch.float32).to(kc.dtype)
        v_cache = k_cache.clone()
        k_cache[idx], v_cache[idx] = kc, vc
        kw.update(cache_batch_idx=idx.to(torch.int32).to(device),
                  cache_leftpad=torch.tensor(pads, dtype=torch.int32, device=device))
    call = Call(tuple(counts), varlen, _rows_to_call(q, counts, varlen).to(device),
                _rows_to_call(k_rows, counts, varlen).to(device), _rows_to_call(v_rows, counts, varlen).to(device),
                k_cache.to(device), v_cache.to(device), sl.to(device), kw, lk, lv, list(seqlens), pads, k_descale=kd,
                v_descale=vd, q_descale=qd, q_rows=q_rows, k_rows=k_rows, v_rows=v_rows)
    if layout == "prefix":
        assert b % 2 == 0
        p_cap, plens = 200, [150, 0]
        pk, pv = (torch.randn(2, p_cap, hkv, d, generator=g) for _ in range(2))
        for i, n in enumerate(plens):
            pk[i, n:] = pv[i, n:] = float("nan")
        pk, pv = pk.to(dtype), pv.to(dtype)
        per = b // 2
        call.prefix_k = [pk[i // per, :plens[i // per]].double() for i in range(b)]
        call.prefix_v = [pv[i // per, :plens[i // per]].double() for i in range(b)]
        kw.update(prefix_k_cache=pk.to(device), prefix_v_cache=pv.to(device),
                  prefix_seqlens=torch.tensor(plens, dtype=torch.int32, device=device))
    if varlen:
        cu = [0] + list(itertools.accumulate(counts))
        kw.update(cu_seqlens_q=torch.tensor(cu, dtype=torch.int32, device=device), max_seqlen_q=max(max(counts), 1))
    return call


def _spans(counts):
    cu = [0] + list(itertools.accumulate(counts))
    return [(lo, n) for lo, n in zip(cu[:-1], counts)]


def oracle(call: Call, tree_mask: torch.Tensor, scale: float, rotary=None, s_cap: Optional[int] = None):
    """fp64 (out (total_q, Hq, D), lse (Hq, total_q)) of a tree call, from the definition.  ``tree_mask`` is the call's
    (uniform (B, Sq, Sq) or packed); ``rotary`` = (cos, sin, rotary_seqlens, interleaved) rotates q and k (in q's
    dtype, as :func:`dec.apply_rotary` does) at ``rotary_seqlens[b] + depth``.  Appended rows past ``s_cap`` are
    dropped, as the call drops them."""
    tm = tree_mask.reshape(-1, tree_mask.shape[-1]).cpu()
    spans = call.spans
    q, k = call.q_rows, call.k_rows
    v = call.v_rows
    if rotary is not None:
        cos, sin, rs, inter = rotary
        pos = []
        for (lo, n), start in zip(spans, rs.tolist()):
            pos += [start + x for x in dec.tree_depths(tm, [(lo, n)])]
        pos = torch.tensor(pos, dtype=torch.long)
        q = dec.apply_rotary(q, cos.cpu(), sin.cpu(), pos, inter)
        k = dec.apply_rotary(k, cos.cpu(), sin.cpu(), pos, inter)
    hq, d = q.shape[1:]
    hkv = k.shape[1]
    if call.q_descale is not None:  # the e4m3 q the call takes, dequantised
        q = torch.cat([dec.quantize_e4m3(q[lo:lo + n], call.q_descale[i].repeat_interleave(hq // hkv)).double()
                       * call.q_descale[i].double().repeat_interleave(hq // hkv)[:, None]
                       for i, (lo, n) in enumerate(spans)])
    q = q.double()
    if call.k_descale is not None:  # appended rows as the e4m3 cache stores them
        k = torch.cat([dec.quantize_e4m3(k[lo:lo + n], call.k_descale[i]).double() * call.k_descale[i].double()[:, None]
                       for i, (lo, n) in enumerate(spans)])
        v = torch.cat([dec.quantize_e4m3(v[lo:lo + n], call.v_descale[i]).double() * call.v_descale[i].double()[:, None]
                       for i, (lo, n) in enumerate(spans)])
    k, v = k.double(), v.double()
    cap = s_cap if s_cap is not None else call.lk.shape[1]
    out = torch.zeros(q.shape[0], hq, d, dtype=torch.float64)
    lse = torch.full((hq, q.shape[0]), float("-inf"), dtype=torch.float64)
    g = hq // hkv
    for i, (lo, n) in enumerate(spans):
        if n == 0:
            continue
        seqlen, lp = call.lens[i], call.pads[i]
        m_new = max(0, min(n, cap - seqlen))
        pre_k = call.prefix_k[i] if call.prefix_k else call.lk.new_zeros(0, hkv, d)
        pre_v = call.prefix_v[i] if call.prefix_v else call.lv.new_zeros(0, hkv, d)
        keys = torch.cat([pre_k, call.lk[i, lp:seqlen], k[lo:lo + m_new]])
        vals = torch.cat([pre_v, call.lv[i, lp:seqlen], v[lo:lo + m_new]])
        n_old = keys.shape[0] - m_new
        vis = torch.cat([torch.ones(n, n_old, dtype=torch.bool), tm[lo:lo + n, :m_new]], dim=1)  # (n, keys)
        kk = keys.repeat_interleave(g, dim=1).transpose(0, 1)  # (Hq, keys, D)
        vv = vals.repeat_interleave(g, dim=1).transpose(0, 1)
        s = torch.matmul(q[lo:lo + n].transpose(0, 1), kk.transpose(1, 2)) * scale  # (Hq, n, keys)
        s = s.masked_fill(~vis, float("-inf"))
        l = torch.logsumexp(s, dim=-1)
        p = torch.exp(s - torch.where(torch.isinf(l), torch.zeros_like(l), l)[..., None]).masked_fill(~vis, 0.0)
        out[lo:lo + n] = torch.matmul(p, vv).transpose(0, 1)
        lse[:, lo:lo + n] = l
    return out, lse


def packed(call: Call, out: torch.Tensor, lse: torch.Tensor):
    """A call's (out, lse) as (total_q, Hq, D) and (Hq, total_q) on the CPU, whether uniform or varlen."""
    out, lse = out.cpu(), lse.cpu()
    if call.varlen:
        return out, lse
    b, sq, hq, d = out.shape
    return out.reshape(b * sq, hq, d), lse.permute(1, 0, 2).reshape(hq, b * sq)


def raw(x: torch.Tensor) -> torch.Tensor:
    """x's bytes, for bitwise comparisons that hold for NaN too."""
    return x.contiguous().view(torch.uint8)
