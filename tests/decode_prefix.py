"""Inputs and references for decode calls with shared prefixes (``prefix_k_cache`` / ``prefix_v_cache`` /
``prefix_seqlens``), built on ``tests/decode_oracle.py``.

A prefix call attends every sequence to its prefix's rows and then to its own keys.  Both key sets enter one softmax,
so the oracle of a prefix call is the merge of two plain oracles, exactly as the kernel's combine merges its two
passes:

* the suffix pass: ``decode_oracle.references`` of the plain inputs (the sequence's own cache and append);
* the prefix pass: the same for a plain call without an append whose cache holds, for sequence ``b``, the rows of
  prefix ``b // (B // P)`` (:func:`prefix_view`): every row visible to every query token, q rotated as in the call.

:func:`concatenated` builds the equivalent plain call's cache: the prefix rows followed by the sequence's own rows.
"""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass
from typing import List, Optional

import torch

import decode_oracle as DO
from ring_flash_attn_b200.parallel import decode as dec

E4M3 = torch.float8_e4m3fn


@dataclass
class Prefix:
    k: torch.Tensor  # (P, P_cap, Hkv, D) in the cache dtype, NaN past each prefix's valid rows
    v: torch.Tensor
    lens: List[int]
    seqlens: torch.Tensor  # (P,) int32
    k_descale: Optional[torch.Tensor] = None  # (P, Hkv) fp32 with e4m3 caches
    v_descale: Optional[torch.Tensor] = None

    @property
    def n(self) -> int:
        return self.k.shape[0]

    def kwargs(self) -> dict:
        kw = dict(prefix_k_cache=self.k, prefix_v_cache=self.v, prefix_seqlens=self.seqlens)
        if self.k_descale is not None:
            kw.update(prefix_k_descale=self.k_descale, prefix_v_descale=self.v_descale)
        return kw


def make_prefix(case: DO.Case, dtype, d: int, device, lens: List[int], p_cap: int, seed: int = 7,
                draw="cpu") -> Prefix:
    """Seeded prefix shards (drawn on ``draw``, the CPU by default): ``len(lens)`` prefixes of ``p_cap`` rows, NaN
    past ``lens``; with an e4m3 case, quantised with their own descales."""
    g = torch.Generator(device=draw).manual_seed(seed)
    n_prefix, hkv = len(lens), case.hkv
    k, v = (torch.randn(n_prefix, p_cap, hkv, d, generator=g, device=draw) for _ in range(2))
    for i, n in enumerate(lens):
        k[i, n:] = float("nan")
        v[i, n:] = float("nan")
    kd = vd = None
    if case.fp8:
        kd, vd = 1.3 * DO.descales(n_prefix, hkv, "k", draw), 0.8 * DO.descales(n_prefix, hkv, "v", draw)
        k = torch.stack([dec.quantize_e4m3(k[i], kd[i]) for i in range(n_prefix)])
        v = torch.stack([dec.quantize_e4m3(v[i], vd[i]) for i in range(n_prefix)])
        kd, vd = kd.to(device), vd.to(device)
    else:
        k, v = k.to(dtype), v.to(dtype)
    return Prefix(k.to(device), v.to(device), list(lens), torch.tensor(lens, dtype=torch.int32, device=device), kd, vd)


def prefix_view(inp: DO.Inputs, pre: Prefix) -> DO.Inputs:
    """The prefix pass as plain inputs: sequence b's cache is its prefix, no append (``references`` must then be
    called with ``appended_here=False``), the same q and rotary positions."""
    case = inp.case
    n = case.b // pre.n
    idx = [b // n for b in range(case.b)]
    g = torch.tensor(idx, device=pre.k.device)
    lens = [pre.lens[i] for i in idx]
    pcase = dataclasses.replace(case, seqlens=tuple(lens), s_cap=pre.k.shape[1], append=False, layout="contiguous",
                                page_size=0, splits=None, rotary=None)
    return dataclasses.replace(inp, case=pcase, lens=lens, kc0=pre.k[g], vc0=pre.v[g],
                               k_descale=None if pre.k_descale is None else pre.k_descale[g],
                               v_descale=None if pre.v_descale is None else pre.v_descale[g])


def references(inp: DO.Inputs, pre: Prefix, n_splits: int, prefix_splits: int,
               appended_here: Optional[bool] = None):
    """(out64, lse64, out32, lse32) of the prefix call: the suffix and prefix oracles merged (fp64, and in fp32 as the
    combine merges partials)."""
    suf = DO.references(inp, n_splits, appended_here=appended_here)
    pre_ref = DO.references(prefix_view(inp, pre), prefix_splits, appended_here=False)
    return parts_merged([suf, pre_ref])


def parts_merged(refs):
    """Merge several ``references`` results (per pass, per rank) in order."""
    o64, l64 = DO.combine_ranks64([(r[0], r[1]) for r in refs])
    o32, l32 = DO.combine_ranks32([(r[2], r[3]) for r in refs])
    return o64, l64, o32, l32


def concatenated(inp: DO.Inputs, pre: Prefix):
    """(k_cache, v_cache, cache_seqlens) of the equivalent plain call: row block ``[0, prefix len)`` of sequence b is
    its prefix, followed by the sequence's own ``S_cap`` rows (a contiguous case with no overflowing append)."""
    case = inp.case
    n = case.b // pre.n
    p_cap = pre.k.shape[1]
    shape = (case.b, p_cap + case.s_cap) + tuple(inp.kc0.shape[2:])
    kc = torch.zeros(shape, dtype=inp.kc0.dtype, device=inp.kc0.device)
    vc = torch.zeros_like(kc)
    lens = []
    for b in range(case.b):
        pl = pre.lens[b // n]
        raw(kc)[b, :pl] = raw(pre.k)[b // n, :pl]
        raw(vc)[b, :pl] = raw(pre.v)[b // n, :pl]
        raw(kc)[b, pl:pl + case.s_cap] = raw(inp.k_cache)[b]
        raw(vc)[b, pl:pl + case.s_cap] = raw(inp.v_cache)[b]
        lens.append(pl + int(inp.seqlens[b]))
    return kc, vc, torch.tensor(lens, dtype=torch.int32, device=inp.seqlens.device)


def raw(x: torch.Tensor) -> torch.Tensor:
    return x.view(torch.uint8) if x.element_size() == 1 else x.view(torch.int16)
