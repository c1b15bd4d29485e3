"""Plain-PyTorch fp32 blockwise attention: the numerical oracle and the CPU/gloo compute path.

These functions play the role that flash_attn's private ``_flash_attn_{,varlen_}{forward,backward}``
ops play for the reference (/root/reference/ring_flash_attn/ring_flash_attn.py:3,53,131) but are
expressed against the *diagonal-offset* mask used everywhere in this library:

    key ``j`` of a segment is visible to query ``i`` of a chunk  iff  ``j <= i + diag``

(``diag=None`` means "everything visible").  Every sharding scheme (ring / zigzag / stripe / llama3,
batch or varlen) reduces to a list of (query-chunk, key-segment, diag) triples - see ``ops/plan.py``.

All math is fp32; callers cast.  Layouts are token-major: q ``(Tq, Hq, D)``, k/v ``(Tk, Hkv, D)``,
lse ``(Hq, Tq)``.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

NEG_INF = float("-inf")


def _expand_kv(x: torch.Tensor, n_rep: int) -> torch.Tensor:
    # (Tk, Hkv, D) -> (Tk, Hkv * n_rep, D); q head h uses kv head h // n_rep (FA's GQA convention).
    return x if n_rep == 1 else x.repeat_interleave(n_rep, dim=1)


def diag_mask(tq: int, tk: int, diag: Optional[int], device, lo: Optional[int] = None) -> Optional[torch.Tensor]:
    """Boolean (tq, tk) mask, True = visible (``i + lo <= j <= i + diag``); None when everything is visible."""
    hi_free = diag is None or diag >= tk - 1
    lo_free = lo is None or lo + (tq - 1) <= 0
    if hi_free and lo_free:
        return None
    i = torch.arange(tq, device=device).unsqueeze(1)
    j = torch.arange(tk, device=device).unsqueeze(0)
    m = torch.ones(tq, tk, dtype=torch.bool, device=device)
    if not hi_free:
        m &= j <= i + diag
    if not lo_free:
        m &= j >= i + lo
    return m


def block_fwd(
    q: torch.Tensor,
    k: torch.Tensor,
    v: torch.Tensor,
    scale: float,
    diag: Optional[int] = None,
    lo: Optional[int] = None,
    mask: Optional[torch.Tensor] = None,
) -> Tuple[torch.Tensor, torch.Tensor]:
    """One (query chunk x key segment) block.  Returns (out fp32 (Tq,Hq,D), lse fp32 (Hq,Tq)).

    ``mask``, optional, is an explicit boolean (Tq, Tk) mask (True = visible), applied together with
    the ``diag`` / ``lo`` rule.  Rows that see no key get ``out = 0`` and ``lse = -inf`` so that they
    are the identity of the online-softmax merge (``ops/merge.py``).
    """
    tq, hq, _ = q.shape
    tk, hkv, _ = k.shape
    n_rep = hq // hkv
    qf = q.float().transpose(0, 1)  # (Hq, Tq, D)
    kf = _expand_kv(k.float(), n_rep).transpose(0, 1)
    vf = _expand_kv(v.float(), n_rep).transpose(0, 1)
    s = torch.matmul(qf, kf.transpose(1, 2)) * scale  # (Hq, Tq, Tk)
    m = diag_mask(tq, tk, diag, q.device, lo)
    if mask is not None:
        m = mask if m is None else m & mask
    if m is not None:
        s = s.masked_fill(~m, NEG_INF)
    lse = torch.logsumexp(s, dim=-1)  # (Hq, Tq); -inf for empty rows
    p = torch.exp(s - torch.where(torch.isinf(lse), torch.zeros_like(lse), lse).unsqueeze(-1))
    if m is not None:
        p = p.masked_fill(~m, 0.0)
    out = torch.matmul(p, vf).transpose(0, 1).contiguous()  # (Tq, Hq, D)
    return out, lse


def block_bwd(
    dout: torch.Tensor,
    q: torch.Tensor,
    k: torch.Tensor,
    v: torch.Tensor,
    lse: torch.Tensor,
    delta: torch.Tensor,
    scale: float,
    diag: Optional[int] = None,
    lo: Optional[int] = None,
) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Gradient contribution of one block given the *global* lse and delta = rowsum(dout * out).

    Same contract as FA's backward used blockwise by the reference
    (/root/reference/ring_flash_attn/ring_flash_attn.py:104-131): P is re-materialised from the
    final lse, so block gradients simply add up.  Returns fp32 (dq, dk, dv); dk/dv are reduced over
    the query heads that share a kv head.
    """
    tq, hq, d = q.shape
    tk, hkv, _ = k.shape
    n_rep = hq // hkv
    qf = q.float().transpose(0, 1)
    kf = _expand_kv(k.float(), n_rep).transpose(0, 1)
    vf = _expand_kv(v.float(), n_rep).transpose(0, 1)
    dof = dout.float().transpose(0, 1)  # (Hq, Tq, D)
    s = torch.matmul(qf, kf.transpose(1, 2)) * scale
    lse_safe = torch.where(torch.isinf(lse), torch.zeros_like(lse), lse)
    p = torch.exp(s - lse_safe.unsqueeze(-1))
    m = diag_mask(tq, tk, diag, q.device, lo)
    if m is not None:
        p = p.masked_fill(~m, 0.0)
    dv = torch.matmul(p.transpose(1, 2), dof)  # (Hq, Tk, D)
    dp = torch.matmul(dof, vf.transpose(1, 2))  # (Hq, Tq, Tk)
    ds = p * (dp - delta.unsqueeze(-1)) * scale
    dq = torch.matmul(ds, kf).transpose(0, 1).contiguous()  # (Tq, Hq, D)
    dk = torch.matmul(ds.transpose(1, 2), qf)  # (Hq, Tk, D)
    if n_rep > 1:
        dk = dk.view(hkv, n_rep, tk, d).sum(1)
        dv = dv.view(hkv, n_rep, tk, d).sum(1)
    return dq, dk.transpose(0, 1).contiguous(), dv.transpose(0, 1).contiguous()


# ----------------------------------------------------------------------------------------------
# Whole-problem oracles (what the reference's tests use flash_attn_*_func for,
# /root/reference/test/test_ring_flash_attn_func.py:46-54).
# ----------------------------------------------------------------------------------------------

def attention_oracle(
    q: torch.Tensor,
    k: torch.Tensor,
    v: torch.Tensor,
    causal: bool,
    softmax_scale: Optional[float] = None,
    window_size: Tuple[int, int] = (-1, -1),
) -> Tuple[torch.Tensor, torch.Tensor]:
    """Dense fp32 attention for batch layout.  q (B,S,Hq,D), k/v (B,S,Hkv,D).

    Returns (out (B,S,Hq,D) fp32, lse (B,Hq,S) fp32).  Differentiable (plain autograd)."""
    b, s, hq, d = q.shape
    hkv = k.shape[2]
    scale = softmax_scale if softmax_scale is not None else d ** -0.5
    n_rep = hq // hkv
    qf = q.float().permute(0, 2, 1, 3)
    kf = k.float().repeat_interleave(n_rep, dim=2).permute(0, 2, 1, 3)
    vf = v.float().repeat_interleave(n_rep, dim=2).permute(0, 2, 1, 3)
    sc = torch.matmul(qf, kf.transpose(-1, -2)) * scale
    left, right = window_size
    if causal:
        right = 0
    if right >= 0 or left >= 0:
        sk = k.shape[1]
        i = torch.arange(s, device=q.device).unsqueeze(1) + (sk - s)  # bottom-right aligned positions
        j = torch.arange(sk, device=q.device).unsqueeze(0)
        vis = torch.ones(s, sk, dtype=torch.bool, device=q.device)
        if right >= 0:
            vis &= j <= i + right
        if left >= 0:
            vis &= j >= i - left
        sc = sc.masked_fill(~vis, NEG_INF)
    lse = torch.logsumexp(sc, dim=-1)
    p = torch.softmax(sc, dim=-1)
    out = torch.matmul(p, vf).permute(0, 2, 1, 3).contiguous()
    return out, lse


def varlen_attention_oracle(
    q: torch.Tensor,
    k: torch.Tensor,
    v: torch.Tensor,
    cu_seqlens: torch.Tensor,
    causal: bool,
    softmax_scale: Optional[float] = None,
    window_size: Tuple[int, int] = (-1, -1),
) -> Tuple[torch.Tensor, torch.Tensor]:
    """Dense fp32 attention over packed documents.  q (T,Hq,D), k/v (T,Hkv,D), one shared cu_seqlens.

    Returns (out (T,Hq,D), lse (Hq,T)).  Differentiable."""
    outs, lses = [], []
    cu = [int(x) for x in cu_seqlens.tolist()]
    for a, b in zip(cu[:-1], cu[1:]):
        o, l = attention_oracle(q[None, a:b], k[None, a:b], v[None, a:b], causal, softmax_scale, window_size)
        outs.append(o[0])
        lses.append(l[0])
    return torch.cat(outs, dim=0), torch.cat(lses, dim=-1)


def default_scale(head_dim: int) -> float:
    return 1.0 / math.sqrt(head_dim)
