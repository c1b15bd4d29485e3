"""Paged shared prefixes (``prefix_block_table=``) for the decode tests, built on ``tests/decode_prefix.py``.

A paged prefix holds exactly the rows of a contiguous :class:`decode_prefix.Prefix` in the pages of a pool, drawn in
a seeded random order, with the table padded with -1 past the pages that hold visible rows.  Every result of a paged
prefix call must then be bitwise that of the contiguous prefix call on the same rows (at equal ``P_cap`` and split
counts on the kernel path), so the contiguous call, itself held to the fp64 oracle, is the reference.

:func:`share_pool` merges a paged suffix's pool and a paged prefix's pool into one, as a paged serving engine keeps
them: the prompt's pages are named by ``prefix_block_table`` and each sample's own pages by ``block_table``.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

import decode_prefix as DP
from test_decode_paged import to_pool


@dataclass
class PagedPrefix:
    pre: DP.Prefix  # the same rows as a contiguous (P, P_cap, Hkv, D) prefix
    k: torch.Tensor  # (num_blocks, page_size, Hkv, D) pool in the cache dtype, NaN in unused rows and spare pages
    v: torch.Tensor
    table: torch.Tensor  # (P, P_cap / page_size) int32, -1 past the pages of each prefix's visible rows

    def kwargs(self) -> dict:
        kw = self.pre.kwargs()
        kw.update(prefix_k_cache=self.k, prefix_v_cache=self.v, prefix_block_table=self.table)
        return kw


def page(pre: DP.Prefix, page_size: int, seed: int = 0, spare: int = 3) -> PagedPrefix:
    """``pre``'s rows in pages of ``page_size`` (which must divide P_cap), in a seeded random order."""
    k, v, table = to_pool(pre.k, pre.v, pre.lens, page_size, spare=spare, seed=seed)
    return PagedPrefix(pre, k, v, table)


def raw(x: torch.Tensor) -> torch.Tensor:
    return x.view(torch.uint8) if x.element_size() == 1 else x.view(torch.int16)


def share_pool(k_suffix: torch.Tensor, v_suffix: torch.Tensor, suffix_table: torch.Tensor, pp: PagedPrefix,
               seed: int = 0):
    """(k_pool, v_pool, block_table, prefix_block_table): the pages of a paged suffix and of ``pp`` in one pool of
    the same page size, interleaved in a seeded random order, and both tables renamed to match (-1 stays -1)."""
    assert k_suffix.shape[1:] == pp.k.shape[1:] and k_suffix.dtype == pp.k.dtype
    n_s = k_suffix.shape[0]
    total = n_s + pp.k.shape[0]
    dev = k_suffix.device
    perm = torch.randperm(total, generator=torch.Generator().manual_seed(seed)).to(dev)  # old page i -> perm[i]
    pools = []
    for a, b in ((k_suffix, pp.k), (v_suffix, pp.v)):
        old = torch.cat([raw(a), raw(b)])
        new = torch.empty_like(old)
        new[perm] = old
        pools.append(new.view(a.dtype))

    def rename(t, offset):
        return torch.where(t >= 0, perm[(t.long() + offset).clamp(min=0)].to(torch.int32), t)

    return pools[0], pools[1], rename(suffix_table, 0), rename(pp.table, n_s)


def prompt_pages(table: torch.Tensor) -> torch.Tensor:
    """The distinct pages a prefix table names (its entries >= 0)."""
    return table[table >= 0].unique().long()
