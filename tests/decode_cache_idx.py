"""Inputs and references for decode calls with cache slots (``cache_batch_idx``) and left padding (``cache_leftpad``),
built on ``tests/decode_oracle.py``.

Both arguments only move where a sequence's keys start, so every reference here is a plain call's:

* a slot call over a pool equals the plain call on the gathered cache ``pool[cache_batch_idx]``;
* a left-padded call over a slot whose keys start at row ``lp`` equals the plain call on the slot shifted down by
  ``lp`` rows, with the same ``S_cap``, as long as no appended row overflows the capacity.

:func:`build` makes the plain case's inputs with :func:`decode_oracle.build_inputs` (the *logical* cache, NaN past the
valid rows) and then the caches the call gets: each sequence's rows moved up by its pad (NaN below), placed in a
seeded slot of a larger pool whose other slots hold NaN.  ``decode_oracle.references`` of the plain inputs is then
the oracle of the padded / slotted call.
"""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass
from typing import List, Optional

import torch

import decode_oracle as DO
import decode_q8 as Q8

E4M3 = torch.float8_e4m3fn


def nan_like(x: torch.Tensor) -> torch.Tensor:
    """A tensor of x's shape and dtype full of NaN (0x7F bytes for e4m3)."""
    if x.dtype == E4M3:
        return torch.full(x.shape, 0x7F, dtype=torch.uint8, device=x.device).view(E4M3)
    return torch.full_like(x, float("nan"))


def raw(x: torch.Tensor) -> torch.Tensor:
    return x.view(torch.uint8) if x.element_size() == 1 else x.view(torch.int16)


def slot_indices(b: int, n_slots: int, seed: int, duplicates: bool = False) -> List[int]:
    """B seeded slots of an ``n_slots`` pool: distinct, or with every other sequence sharing its neighbour's slot."""
    perm = torch.randperm(n_slots, generator=torch.Generator().manual_seed(seed)).tolist()
    if not duplicates:
        return perm[:b]
    return [perm[i // 2] for i in range(b)]


def leftpads(case: DO.Case, seed: int) -> List[int]:
    """Seeded pads that leave every appended row inside the capacity: ``lens[b] + pad + count <= S_cap``."""
    g = torch.Generator().manual_seed(seed)
    pads = []
    for n, c in zip(case.seqlens, case.counts):
        room = case.s_cap - min(max(n, 0), case.s_cap) - (c if case.append else 0)
        pads.append(int(torch.randint(0, max(room, 0) + 1, (1,), generator=g)) if room > 0 else 0)
    return pads


@dataclass
class SlotInputs:
    plain: DO.Inputs  # the plain call's inputs: inp.kc0 / vc0 is the logical (gathered, shifted) cache
    k_pool: torch.Tensor  # (n_slots, S_cap, Hkv, D): what the call gets
    v_pool: torch.Tensor
    idx: Optional[List[int]]  # cache_batch_idx, None: slot b
    pads: Optional[List[int]]  # cache_leftpad, None: no pad
    seqlens: torch.Tensor  # cache_seqlens of the call: the plain ones plus the pads
    q8: Optional[torch.Tensor] = None  # e4m3 q and its descale, and the query they stand for (fp64 reference input)
    q_descale: Optional[torch.Tensor] = None
    q64: Optional[torch.Tensor] = None

    def kwargs(self) -> dict:
        """The new arguments as tensors on the caches' device."""
        dev = self.k_pool.device
        kw = {}
        if self.idx is not None:
            kw["cache_batch_idx"] = torch.tensor(self.idx, dtype=torch.int32, device=dev)
        if self.pads is not None:
            kw["cache_leftpad"] = torch.tensor(self.pads, dtype=torch.int32, device=dev)
        return kw


def build(case: DO.Case, dtype, d: int, device, idx: Optional[List[int]] = None, n_slots: Optional[int] = None,
          pads: Optional[List[int]] = None, q8: bool = False, regime: str = "randn", seed: int = 0,
          cache_seed: Optional[int] = None) -> SlotInputs:
    """The inputs of a slot / left-padded call and of its plain equivalent.  With duplicate slots, the sequence with
    the most valid rows fills the shared slot and its sharers read its rows (the plain cache is then ``pool[idx]``).
    ``q8``: an e4m3 q (with an e4m3 cache)."""
    assert case.layout == "contiguous"
    inp = DO.build_inputs(case, dtype, d, regime, device, seed, cache_seed=cache_seed)
    b, s_cap = case.b, case.s_cap
    kc, vc = inp.kc0, inp.vc0
    if pads is not None:  # rows [lp, lp + S_cap - lp) of the padded slot are rows [0, S_cap - lp) of the plain one
        pk, pv = nan_like(kc), nan_like(vc)
        for i, lp in enumerate(pads):
            raw(pk)[i, lp:] = raw(kc)[i, :s_cap - lp]
            raw(pv)[i, lp:] = raw(vc)[i, :s_cap - lp]
        kc, vc = pk, pv
    k_pool, v_pool = kc, vc
    if idx is not None:
        n_slots = max(idx) + 1 if n_slots is None else n_slots
        k_pool = nan_like(kc.new_empty((n_slots,) + tuple(kc.shape[1:])))
        v_pool = nan_like(k_pool)
        order = sorted(range(b), key=lambda i: inp.lens[i])  # the longest sharer writes last
        for i in order:
            raw(k_pool)[idx[i]] = raw(kc)[i]
            raw(v_pool)[idx[i]] = raw(vc)[i]
        if len(set(idx)) < b:  # sharers read the writer's rows: the plain cache is the gathered pool, unshifted
            assert pads is None, "duplicate slots are built without pads"
            g = torch.tensor(idx, device=k_pool.device)
            kc0, vc0 = k_pool[g].clone(), v_pool[g].clone()
            inp = dataclasses.replace(inp, kc0=kc0, vc0=vc0, k_cache=kc0.clone(), v_cache=vc0.clone())
    seqlens = inp.seqlens + (torch.tensor(pads, dtype=torch.int32, device=inp.seqlens.device) if pads else 0)
    out = SlotInputs(inp, k_pool.clone(), v_pool.clone(), idx, pads, seqlens.to(torch.int32))
    if q8:
        out.q8, out.q_descale, out.q64 = Q8.quantise_q(inp)
    return out


def expected_pool(si: SlotInputs, with_append: bool):
    """The pool after the call: the plain call's appended rows, moved up by the pads, in each sequence's slot."""
    inp, case = si.plain, si.plain.case
    want_k, want_v = si.k_pool.clone(), si.v_pool.clone()
    if not with_append:
        return want_k, want_v
    for b, (lo, n) in enumerate(DO.spans(case)):
        slot = b if si.idx is None else si.idx[b]
        lp = 0 if si.pads is None else si.pads[b]
        for t in range(n):
            row = inp.lens[b] + lp + t
            if row < case.s_cap:
                raw(want_k)[slot, row] = raw(inp.stored_k)[lo + t]
                raw(want_v)[slot, row] = raw(inp.stored_v)[lo + t]
    return want_k, want_v


def call_args(si: SlotInputs, with_append: bool, bf16_append_for_q8: bool = True):
    """(q, k, v, extra kwargs) of the slot / left-padded call, in ``kernel_decode`` / public-call form."""
    inp = si.plain
    src = inp if si.q8 is None else dataclasses.replace(inp, q=si.q8)
    q, k, v = DO.call_views(src, with_append)
    kw = dict(DO.call_kwargs(inp), **si.kwargs())
    if si.q8 is not None:
        kw["q_descale"] = si.q_descale
    return q, k, v, kw


def plain_inputs_for_reference(si: SlotInputs) -> DO.Inputs:
    """What ``decode_oracle.references`` takes: the plain inputs, with an e4m3 q's fp64 value as q."""
    return si.plain if si.q64 is None else dataclasses.replace(si.plain, q=si.q64)
