"""fp64 and precision-matched references for the multi-GPU context-parallel paths, built from the plans the API builds.

Every rank's plan (``parallel/ops.py``: ``batch_plan``, ``varlen_plan``, ``llama3_plan``, ``zigzag_llama3_plan``) is
run through ``kernel_oracle.plan_forward`` / ``plan_backward`` over ONE key space: the source shards back to back,
each segment's ``kv_row0`` rebased by ``src * kv_rows``.  The precision-matched side rounds where each transport
rounds:

* ``fused`` (``parallel/symm.py``: one launch over every source): ``out`` is rounded once; dq is accumulated in fp32
  and rounded once; every rank stores its dK / dV partial for each source's rows into the owner's inbox in the model
  dtype, and ``reduce_dkv`` sums the slots in fp32 and rounds again.
* ``ring`` / ``allgather`` (the torch.distributed fallback, ``parallel/engine.py``): ``segments_forward`` returns each
  source's partial in the model dtype, ``merge_partial`` merges them in fp32 in the transport's source order and
  the result is rounded once; dK / dV stay fp32 until the owner rounds once.

The backward's matched side takes lse and delta from the matched forward (delta from the rounded out), as
``kernel_oracle.api_reference`` does; the fp64 side uses the fp64 lse and delta.  Bounds: ``kernel_oracle``'s
:func:`~kernel_oracle.assert_accurate` / :func:`~kernel_oracle.assert_lse`.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, replace
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch

import kernel_oracle as KO
from ring_flash_attn_b200.ops import plan as P

BATCH = ("ring", "zigzag", "stripe")
# Regimes whose backward is held to the bound.  With nearly one-hot rows (``peaked``) the gradient of a row's maximum
# key is dominated by delta = rowsum(out * dout), i.e. by the rounding of the implementation's OWN out, which the
# precision-matched reference cannot mirror (it rounds its own out); a key that is the maximum of many rows sums that
# error over them, so the ratio of two such independent errors has a heavy tail (2.07x measured on a CPU replay).
BACKWARD_REGIMES = ("randn",)
FALLBACK_ORDER = {"ring": "ring", "zigzag": "ring", "stripe": "ring", "ring_varlen": "ring", "zigzag_varlen": "ring",
                  "zigzag_llama3": "ring", "llama3": "allgather"}


@dataclass(frozen=True)
class Case:
    """One context-parallel call: ``rows`` local tokens per rank (batch schemes: ``batch`` sequences of
    ``rows // batch``), ``window`` as flash-attn's ``window_size``."""
    scheme: str
    world: int
    rows: int
    hq: int
    hkv: int
    d: int
    dtype: torch.dtype
    causal: bool = True
    window: Tuple[int, int] = (-1, -1)
    regime: str = "randn"
    batch: int = 1
    stride: int = 1  # llama3 heads_k_stride

    @property
    def total(self) -> int:
        return self.world * self.rows

    @property
    def scale(self) -> float:
        return self.d ** -0.5

    def with_(self, **kw) -> "Case":
        return replace(self, **kw)

    def name(self) -> str:
        dt = str(self.dtype).replace("torch.", "")
        win = "plain" if self.window == (-1, -1) else f"window{self.window}"
        mode = "" if self.causal else " non-causal"
        return (f"{self.scheme}{mode} W{self.world} rows {self.rows} h{self.hq}/{self.hkv} D{self.d} {dt} {win} "
                f"{self.regime}")


def window_for(causal: bool, total: int) -> Tuple[int, int]:
    """A sliding window reaching a few shards back (about a sixth of the sequence, through several 128-key tiles);
    non-causal: a right edge as well."""
    left = max(37, total // 6 + 5)
    return (left, 0) if causal else (left, total // 10 + 3)


def global_cu(case: Case) -> Tuple[int, ...]:
    """Global cu_seqlens of the packed schemes.  ring / zigzag varlen: documents in units of 2W tokens; llama3 layouts:
    cuts anywhere, with a one-token document and documents that straddle ranks."""
    T = case.total
    if case.scheme in ("ring_varlen", "zigzag_varlen"):
        unit = 2 * case.world
        n = T // unit
        return (0, unit * max(1, n * 3 // 10), unit * max(2, n * 7 // 10), T)
    a = T * 3 // 10 + 1
    return (0, a, a + 1, T * 7 // 10 + 5, T)


def local_cu(case: Case) -> Tuple[int, ...]:
    return tuple(c // case.world for c in global_cu(case))


def build_plans(case: Case) -> List[P.CPPlan]:
    """Every rank's plan, from the same cached builders the API resolves (``parallel/ops.py``)."""
    from ring_flash_attn_b200.parallel import api, ops

    W = case.world
    if case.scheme in BATCH:
        return [ops.batch_plan(case.scheme, r, W, case.batch, case.rows // case.batch, case.causal, case.window)
                for r in range(W)]
    if case.scheme in ("ring_varlen", "zigzag_varlen"):
        return [ops.varlen_plan(case.scheme[:-len("_varlen")], r, W, local_cu(case), case.causal, case.window)
                for r in range(W)]
    if case.scheme == "zigzag_llama3":
        return [ops.zigzag_llama3_plan(r, W, global_cu(case), case.causal, case.window) for r in range(W)]
    if case.scheme == "llama3":
        cu = torch.tensor(global_cu(case), dtype=torch.int32)
        plans = []
        for r in range(W):
            cq, ck, _mq, _mk, ks = api.llama3_flash_attn_prepare_cu_seqlens(cu, case.causal, r, W)
            plans.append(ops.llama3_plan(r, W, case.rows, tuple(cq.tolist()), tuple(ck.tolist()), int(ks.start),
                                         case.causal, case.window))
        return plans
    raise ValueError(case.scheme)


def source_order(transport: str, rank: int, world: int) -> List[int]:
    """The order in which a transport folds the sources into the running result (``engine.ring_forward``:
    own shard, then 1, 2, ... hops upstream; ``engine.allgather_forward``: rank order)."""
    if transport == "allgather":
        return list(range(world))
    return [(rank - s) % world for s in range(world)]


def make_inputs(case: Case, seed: int, device="cpu"):
    """Per-rank local q, k, v, dout (token-major, ``case.dtype``) from one seed: every process of a group draws the
    same tensors.  ``peaked``: logits span about +-30 and rise with the key's index in the source-major key space, so
    a row's maximum is its last visible key of the highest source it sees - a remote source's last tile for most
    rows - and the online softmax's running maximum changes at every source.  Only the forward is held to the bound
    in this regime (:data:`BACKWARD_REGIMES`)."""
    g = torch.Generator().manual_seed(seed)
    W, L, d = case.world, case.rows, case.d

    def rn(h):
        return torch.randn((W * L, h, d), generator=g, dtype=torch.float32)

    q, k, v, do = rn(case.hq), rn(case.hkv), rn(case.hkv), rn(case.hq)
    if case.regime == "peaked":
        ramp = torch.linspace(-1.0, 1.0, W * L)
        q = 1.0 + 0.1 * q
        k = (30.0 / math.sqrt(d)) * ramp.view(-1, 1, 1) + 0.1 * k
    elif case.regime != "randn":
        raise ValueError(case.regime)
    return tuple([t[r * L:(r + 1) * L].to(case.dtype).to(device) for r in range(W)] for t in (q, k, v, do))


# ----------------------------------------------------------------------------------------------
# references
# ----------------------------------------------------------------------------------------------

def global_segments(plan: P.CPPlan) -> List[P.Segment]:
    """The plan's segments over the source shards concatenated in rank order."""
    L = plan.kv_rows
    return [P.Segment(s.chunk, 0, s.src * L + s.kv_row0, s.kv_len, s.diag, s.lo) for s in plan.segments]


def merge_fp32(out, lse, p_out, p_lse):
    """fp32 online-softmax merge of one source's partial into the running (out (T, H, D), lse (H, T)); -inf lse is
    the identity."""
    p_out, p_lse = p_out.float(), p_lse.float()
    if out is None:
        return p_out.clone(), p_lse.clone()
    new = torch.logaddexp(lse, p_lse)
    safe = torch.where(torch.isinf(new), torch.zeros_like(new), new)
    w_old = torch.exp(lse - safe).transpose(0, 1).unsqueeze(-1)
    w_new = torch.exp(p_lse - safe).transpose(0, 1).unsqueeze(-1)
    return out * w_old + p_out * w_new, new


def rank_forward(plan: P.CPPlan, q, ks: Sequence, vs: Sequence, scale: float, dtype, transport: str,
                 skip_source: Optional[int] = None):
    """(fp64 (out, lse), matched (out, lse)) of one rank.  ``transport``: ``fused``, ``ring`` or ``allgather``.
    ``skip_source`` leaves one source out of the matched merge (a planted error for the CPU self-test)."""
    K, V = torch.cat(list(ks)), torch.cat(list(vs))
    gsegs = global_segments(plan)
    o64, l64 = KO.plan_forward(plan, gsegs, q, K, V, scale)
    if transport == "fused":
        olp, llp = KO.plan_forward(plan, gsegs, q, K, V, scale, p_dtype=dtype)
        return (o64, l64), (olp, llp)
    out = lse = None
    by_src = plan.by_src()
    for src in source_order(transport, plan.rank, plan.world):
        segs = by_src.get(src, [])
        if not segs or src == skip_source:
            continue
        p_out, p_lse = KO.plan_forward(plan, segs, q, ks[src], vs[src], scale, p_dtype=dtype)  # out in the model dtype
        out, lse = merge_fp32(out, lse, p_out, p_lse)
    if out is None:
        out = torch.zeros(q.shape, dtype=torch.float32, device=q.device)
        lse = torch.full((q.shape[1], q.shape[0]), float("-inf"), device=q.device)
    return (o64, l64), (out.to(dtype), lse)


def rank_backward(plan: P.CPPlan, q, ks: Sequence, vs: Sequence, dout, fwd64, fwdlp, scale: float, dtype,
                  transport: str):
    """(fp64 (dq, dk, dv), matched (dq, dk, dv)) of one rank; dk / dv over the whole source-major key space: this
    rank's partial for every source's rows, fp64 / fp32 (rounded to ``dtype`` first on the fused path)."""
    K, V = torch.cat(list(ks)), torch.cat(list(vs))
    gsegs = global_segments(plan)
    (o64, l64), (olp, llp) = fwd64, fwdlp
    delta64 = (o64 * dout.double()).sum(-1).transpose(0, 1)
    deltalp = (olp.float() * dout.float()).sum(-1).transpose(0, 1)
    g64 = KO.plan_backward(plan, gsegs, q, K, V, dout, l64, delta64, scale)
    dkv_dtype = dtype if transport == "fused" else torch.float32
    dq, dk, dv = KO.plan_backward(plan, gsegs, q, K, V, dout, llp, deltalp, scale, mm_dtype=dtype,
                                  dkv_dtype=dkv_dtype, dq_dtype=dtype)
    return g64, (dq, dk.float(), dv.float())


def references(case: Case, plans, q, k, v, dout, transport: str, ranks: Optional[Sequence[int]] = None,
               all_reduce: Optional[Callable] = None, backward: bool = True,
               bwd_transport: Optional[str] = None) -> Dict[int, Tuple[dict, dict]]:
    """{rank: (fp64, matched)} dicts of out / lse (and dq / dk / dv) for ``ranks`` (default: all).

    dK / dV of a shard are the sum of every rank's partial: with ``all_reduce`` (an in-place sum over the process
    group) each process computes its own ranks' partials only; without it ``ranks`` must be every rank.
    ``bwd_transport``: the backward's transport when it differs from the forward's (``deterministic=True`` across
    GPUs runs the fused forward and the fallback's ordered backward)."""
    W, L = case.world, case.rows
    ranks = list(range(W)) if ranks is None else list(ranks)
    bwd_transport = bwd_transport or transport
    res = {}
    parts64 = partslp = None
    for r in ranks:
        f64, flp = rank_forward(plans[r], q[r], k, v, case.scale, case.dtype, transport)
        res[r] = (dict(out=f64[0], lse=f64[1]), dict(out=flp[0], lse=flp[1]))
        if not backward:
            continue
        g64, glp = rank_backward(plans[r], q[r], k, v, dout[r], f64, flp, case.scale, case.dtype, bwd_transport)
        res[r][0]["dq"], res[r][1]["dq"] = g64[0], glp[0]
        s64, slp = torch.stack(g64[1:]), torch.stack(glp[1:])
        parts64 = s64 if parts64 is None else parts64 + s64
        partslp = slp if partslp is None else partslp + slp
    if not backward:
        return res
    if all_reduce is not None:
        all_reduce(parts64)
        all_reduce(partslp)
    else:
        assert len(ranks) == W, "without all_reduce every rank's partial is needed"
    for r in ranks:
        rows = slice(r * L, (r + 1) * L)
        res[r][0]["dk"], res[r][0]["dv"] = parts64[0, rows], parts64[1, rows]
        res[r][1]["dk"], res[r][1]["dv"] = partslp[0, rows].to(case.dtype), partslp[1, rows].to(case.dtype)
    return res


def check(name: str, got: dict, ref64: dict, reflp: dict, report: str, factor: Optional[float] = None,
          lse_rel: Optional[float] = None, per_block: bool = False) -> None:
    """Every output in ``got`` (token-major out / dq / dk / dv, lse (Hq, T)) within the precision-matched bound
    (``per_block``: within every ``kernel_oracle.work_units`` block too)."""
    for key, val in got.items():
        if key == "lse":
            KO.assert_lse(f"{name}: lse", val, ref64["lse"], reflp["lse"], report="lse " + report, rel_limit=lse_rel)
        else:
            assert val.dtype == reflp[key].dtype, (name, key, val.dtype, reflp[key].dtype)
            KO.assert_accurate(f"{name}: {key}", val, ref64[key], reflp[key], factor=factor, report=report,
                               **(KO.work_units(key) if per_block else {}))


def report_key(transport: str, world: int) -> str:
    return f"cp {transport} W{world}"


# ----------------------------------------------------------------------------------------------
# every rank's plan replayed in one process, source by source
# ----------------------------------------------------------------------------------------------

def replay(case: Case, plans, q, k, v, dout, deterministic: bool = False, backward: bool = True,
           step_forward: Optional[Callable] = None) -> Dict[int, dict]:
    """What the torch.distributed fallback computes, without a process group: every rank's plan through
    ``engine.step_forward`` / ``step_backward`` (the per-source kernel launches), the partials merged in the
    transport's source order, dq accumulated in fp32, each shard's dK / dV summed over the ranks in fp32 and rounded
    once.  ``step_forward`` replaces the engine's (planted errors in the CPU self-test)."""
    from ring_flash_attn_b200.parallel import engine

    step_forward = step_forward or engine.step_forward
    transport = FALLBACK_ORDER[case.scheme]
    W = case.world
    got = {}
    dkv = [None] * W
    for r, plan in enumerate(plans):
        by_src = plan.by_src()
        order = source_order(transport, r, W)
        out = lse = None
        for src in order:
            out, lse = step_forward(plan, by_src.get(src, []), q[r], k[src], v[src], case.scale, out, lse)
        out = out.to(case.dtype)
        got[r] = dict(out=out, lse=lse)
        if not backward:
            continue
        delta = engine.compute_delta(out, dout[r])
        dq = torch.zeros(q[r].shape, dtype=torch.float32, device=q[r].device)
        for src in order:
            b_dk, b_dv = engine.step_backward(plan, by_src.get(src, []), dout[r], q[r], k[src], v[src], lse, delta,
                                              case.scale, dq, deterministic)
            part = torch.stack([b_dk, b_dv])
            dkv[src] = part if dkv[src] is None else dkv[src] + part
        got[r]["dq"] = dq.to(case.dtype)
    if backward:
        for r in range(W):
            got[r]["dk"], got[r]["dv"] = dkv[r][0].to(case.dtype), dkv[r][1].to(case.dtype)
    return got


# ----------------------------------------------------------------------------------------------
# the public API on one rank's shard
# ----------------------------------------------------------------------------------------------

def api_call(case: Case, rank: int, q, k, v, deterministic: bool = False, group=None):
    """Run the public entry point of ``case.scheme`` on this rank's token-major shard: (out (T, Hq, D),
    lse (Hq, T))."""
    import ring_flash_attn_b200 as rfa

    kw = dict(causal=case.causal, window_size=case.window, deterministic=deterministic, return_attn_probs=True,
              group=group)
    dev = q.device
    if case.scheme in BATCH:
        B, s = case.batch, case.rows // case.batch
        fn = getattr(rfa, {"ring": "ring", "zigzag": "zigzag_ring", "stripe": "stripe"}[case.scheme] +
                     "_flash_attn_func")
        out, lse, _ = fn(*(t.view(B, s, *t.shape[1:]) for t in (q, k, v)), **kw)
        return out.reshape(case.rows, case.hq, case.d), lse.permute(1, 0, 2).reshape(case.hq, case.rows)
    if case.scheme in ("ring_varlen", "zigzag_varlen"):
        cu = torch.tensor(local_cu(case), dtype=torch.int32, device=dev)
        fn = rfa.ring_flash_attn_varlen_func if case.scheme == "ring_varlen" else rfa.zigzag_ring_flash_attn_varlen_func
        out, lse, _ = fn(q, k, v, cu, int((cu[1:] - cu[:-1]).max()), **kw)
        return out, lse
    if case.scheme == "llama3":
        cu = torch.tensor(global_cu(case), dtype=torch.int32, device=dev)
        cq, ck, mq, mk, ks = rfa.llama3_flash_attn_prepare_cu_seqlens(cu, case.causal, rank, case.world)
        out, lse, _ = rfa.llama3_flash_attn_varlen_func(q, k, v, cq, ck, mq, mk, heads_k_stride=case.stride,
                                                        local_k_slice=ks, **kw)
        return out, lse
    if case.scheme == "zigzag_llama3":
        cu = torch.tensor(global_cu(case), dtype=torch.int32, device=dev)
        out, lse, _ = rfa.zigzag_llama3_flash_attn_varlen_func(q, k, v, cu, **kw)
        return out, lse
    raise ValueError(case.scheme)


def api_train(case: Case, rank: int, q, k, v, dout, deterministic: bool = False, group=None,
              backward: bool = True) -> dict:
    """Forward (+ backward with ``dout``) through the public API: dict of out, lse and dq / dk / dv."""
    xs = [t.detach().clone().requires_grad_(backward) for t in (q, k, v)]
    out, lse = api_call(case, rank, *xs, deterministic=deterministic, group=group)
    got = dict(out=out.detach(), lse=lse.detach())
    if backward:
        out.backward(dout)
        got.update(dq=xs[0].grad, dk=xs[1].grad, dv=xs[2].grad)
    return got
