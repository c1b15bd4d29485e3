"""fp64 and precision-matched references for the sm_90a attention kernels, and the block-level sweep built on them.

The kernels are judged by flash-attn's convention: an output may be at most twice as far from the fp64 result as a
reference that computes the same math in fp32 and rounds where the kernels round (:func:`assert_accurate`).  Both
references work on a :class:`CPPlan` and a list of its segments, exactly what ``attn_cuda.segments_forward`` /
``segments_backward`` launch: a chunk attends to the concatenation of its segments, each with its own ``diag`` / ``lo``.

The sweep (:func:`run_forward`, :func:`run_backward`, :func:`run_invisibility`) runs on whatever
``cuda_ext.load()`` returns: the sm_90a extension in ``tests/test_gpu_kernel_accuracy.py``, ``tests/fake_ext.py`` and
mutated copies of it in ``tests/test_kernel_oracle_cpu.py``.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence, Tuple

import torch

from ring_flash_attn_b200.ops import attn_cuda, cuda_ext
from ring_flash_attn_b200.ops import plan as P
from ring_flash_attn_b200.ops.dense import diag_mask

LOG2E = 1.4426950408889634
MAX_RATIO = 2.0  # kernel error / precision-matched error
# |q|, |k| ~ 30: a score is an fp32 sum of terms ~1e3, and its rounding, which depends on the summation order and no
# reference can mirror, dominates P wherever a row is not exactly one-hot (the backward amplifies it by |k| ~ 30).
# Two fp32 implementations then differ by a random factor: fp32 torch (tests/fake_ext.py) against the reference
# measured 3.4x (dq, fp16, D 128); the sm_90a kernels measured at most 1.9x on an H100.
LARGE_RATIO = 4.0
LSE_REL = 1e-4  # lse: fp32 max + ex2.approx + __log2f, bounded by LSE_REL * (1 + |lse|)
# e4m3 wgmma does not accumulate Q K^T in full fp32 (Hopper keeps about 14 mantissa bits), which no fp32 reference can
# mirror.  Measured on an H100: out 2.15x the precision-matched error, lse 6.1e-4 (1 + |lse|).
FP8_RATIO = 4.0
FP8_LSE_REL = 2e-3

# The per-block bound (``assert_accurate(blocks=...)``).  A block's baseline is the max of few roundings - the elements
# in the top binade of a 64 x D block are a handful - so two implementations that differ by less than an output ulp
# can be further apart than 2x there.  Measured on an H100 (700 W) at the long-context shapes
# (tests/test_gpu_long_context.py): up to 2.46x for bf16 out / dq over 16K blocks per tensor.  On the CPU a correct
# fp32 implementation that rounds P where the kernels do reaches 2.4x at 8K tokens while passing the tensor-wide bound
# (test_kernel_oracle_cpu.py::test_legitimate_per_block_ratio_exceeds_2x).  The planted errors the bound exists for
# measured 15x (dK / dV rounded after every query tile) to 290x (tests/test_kernel_oracle_cpu.py).
BLOCK_RATIO = 4.0
# The backward keeps a key tile's dK / dV in one wgmma fp32 accumulator while its CTA sweeps every query tile of every
# query head of the GQA group, 4 wgmma (k = 16) per 64-row tile.  Each wgmma adds into the accumulator with truncation
# (round toward zero), so the result drifts toward zero by up to one fp32 ulp of the accumulator per addition: 2e-3
# relative for MQA at 32K (32 heads x 512 tiles x 4), measured on an H100 and replayed in
# tests/test_gpu_long_context.py.  An fp32 reference cannot round like that without replaying the sweep, so the dK / dV
# bound gains ACCUM_ULP * additions * max|ref64| (:func:`wgmma_additions`).
WGMMA_PER_TILE = 4
ACCUM_ULP = 2.0 ** -23

# worst observed ratio per report key (filled by assert_accurate / assert_lse; handy for a summary after a run)
WORST: Dict[str, float] = {}


def _by_chunk(segs: Sequence[P.Segment]) -> Dict[int, list]:
    out: Dict[int, list] = {}
    for s in segs:
        out.setdefault(s.chunk, []).append(s)
    return out


# The references work in blocks of at most ROW_BLOCK query rows of one chunk x a group of query heads, over the keys
# each block can see, so that no (Hq, rows, keys) score tensor of a whole chunk is ever formed: at 139K tokens x 32
# heads that would be terabytes.  A group's heads are sized to keep heads x rows x keys near BLOCK_ELEMS.
ROW_BLOCK = 1024
BLOCK_ELEMS = 1 << 27


def _key_range(s: P.Segment, r0: int, r1: int) -> Tuple[int, int]:
    """The keys [a, b) of segment ``s`` that rows r0 .. r1 - 1 of its chunk may see; every other key is masked for
    all of them (``diag`` / ``lo``), so leaving it out drops exact zeros."""
    a = 0 if s.lo is None else min(max(r0 + s.lo, 0), s.kv_len)
    b = s.kv_len if s.diag is None else min(max(r1 + s.diag, 0), s.kv_len)
    return a, max(a, b)


def _head_groups(hq: int, rep: int, per_head: int):
    """(h0, h1) query-head ranges of about ``BLOCK_ELEMS / per_head`` heads: whole GQA groups, or a part of one
    group when a single group is too large, so that a range reads one kv head or whole kv heads."""
    n = max(1, BLOCK_ELEMS // max(per_head, 1))
    if n >= rep:
        step = (min(n, hq) // rep) * rep
    else:
        step = max(d for d in range(1, rep + 1) if rep % d == 0 and d <= n)
    return [(h0, min(h0 + step, hq)) for h0 in range(0, hq, step)]


def _row_blocks(ch: P.QChunk, cs: Sequence[P.Segment]):
    """(r0, r1, [(segment, a, b)]) per block of ROW_BLOCK rows of a chunk (rows relative to the chunk)."""
    for r0 in range(0, ch.rows, ROW_BLOCK):
        r1 = min(r0 + ROW_BLOCK, ch.rows)
        yield r0, r1, [(s, *_key_range(s, r0, r1)) for s in cs]


def _kv(x, s: P.Segment, a: int, b: int, h0: int, h1: int, rep: int, cd):
    """Keys a .. b - 1 of segment ``s`` for query heads h0 .. h1 - 1 (head h reads kv head h // rep): (b - a, h1 - h0,
    D) in ``cd``."""
    x = x[s.kv_row0 + a:s.kv_row0 + b, h0 // rep:(h1 - 1) // rep + 1].to(cd)
    return x.repeat_interleave(rep, dim=1)[:, h0 % rep:h0 % rep + h1 - h0] if rep > 1 else x


def _scores(qb, kk, s: P.Segment, r0: int, a: int):
    """Raw scores q . k (no softmax scale) of rows r0 .. of a chunk against keys a .. of one segment, -inf where
    invisible: (heads, n, keys)."""
    sc = torch.einsum("nhd,khd->hnk", qb, kk)
    diag = None if s.diag is None else s.diag + r0 - a
    lo = None if s.lo is None else s.lo + r0 - a
    m = diag_mask(qb.shape[0], kk.shape[0], diag, qb.device, lo)
    return sc if m is None else sc.masked_fill(~m, float("-inf"))


def _exp2_fma(x, t2: float, sub):
    """``exp2(fmaf(x, t2, -sub))`` of fp32 ``x`` / ``sub``: the product is exact, one rounding after the subtraction
    (how both kernels form P; a plain fp32 ``x * t2 - sub`` would make the row maximum exactly 1)."""
    return torch.exp2((x.double() * t2 - sub.double()).float())


def plan_forward(plan: P.CPPlan, segs: Sequence[P.Segment], q, k, v, scale: float,
                 p_dtype: Optional[torch.dtype] = None, out_dtype: Optional[torch.dtype] = None):
    """Forward over ``plan``'s chunks: (out (Tq, Hq, D), lse (Hq, Tq)).  Rows outside every chunk, and rows that see no
    key, get out = 0 and lse = -inf.

    ``p_dtype=None``: fp64 throughout.  Otherwise the precision-matched reference: fp32 scores, P = exp2 relative to
    the row maximum in log2 units (``attn_fwd_sm90.cu``), rounded to ``p_dtype`` before P V, the row sum of the
    unrounded P, and ``out`` rounded to ``out_dtype``."""
    lowp = p_dtype is not None
    cd = torch.float32 if lowp else torch.float64
    tq, hq, d = q.shape
    rep = hq // k.shape[1]
    out = torch.zeros((tq, hq, d), dtype=cd, device=q.device)
    lse = torch.full((hq, tq), float("-inf"), dtype=cd, device=q.device)
    t2 = float(torch.tensor(scale * LOG2E, dtype=torch.float32))
    for ci, cs in _by_chunk(segs).items():
        ch = plan.q_chunks[ci]
        for r0, r1, ranges in _row_blocks(ch, cs):
            n_keys = sum(b - a for _, a, b in ranges)
            if n_keys == 0:
                continue
            rows = slice(ch.row0 + r0, ch.row0 + r1)
            for h0, h1 in _head_groups(hq, rep, (r1 - r0) * n_keys):
                qb = q[rows, h0:h1].to(cd)
                sc = torch.cat([_scores(qb, _kv(k, s, a, b, h0, h1, rep, cd), s, r0, a) for s, a, b in ranges],
                               dim=-1)  # (heads, n, keys)
                vv = torch.cat([_kv(v, s, a, b, h0, h1, rep, cd) for s, a, b in ranges], dim=0)
                mx = sc.amax(dim=-1, keepdim=True)
                empty = torch.isinf(mx)
                if lowp:
                    m2 = torch.where(empty, torch.zeros_like(mx), mx * t2)
                    p = _exp2_fma(sc, t2, m2)
                    l = p.sum(dim=-1, keepdim=True)
                    row_lse = (m2 + torch.log2(l)) * math.log(2.0)
                    p = p.to(p_dtype).to(cd)
                else:
                    m = torch.where(empty, torch.zeros_like(mx), mx)
                    p = torch.exp((sc - m) * scale)
                    l = p.sum(dim=-1, keepdim=True)
                    row_lse = m * scale + torch.log(l)
                del sc
                o = torch.einsum("hnk,khd->nhd", p, vv) / torch.where(empty, torch.ones_like(l), l).permute(1, 0, 2)
                out[rows, h0:h1] = torch.where(empty.permute(1, 0, 2), torch.zeros_like(o), o)
                lse[h0:h1, rows] = torch.where(empty, torch.full_like(row_lse, float("-inf")), row_lse).squeeze(-1)
    if lowp:
        out = out.to(out_dtype or p_dtype)
    return out, lse


def _group_sum(x, h0: int, h1: int, rep: int):
    """(keys, h1 - h0, D) per query head -> per kv head h0 // rep ..: summed over each GQA group's heads."""
    if h1 - h0 < rep:
        return x.sum(1, keepdim=True)
    return x.reshape(x.shape[0], (h1 - h0) // rep, rep, x.shape[2]).sum(2)


def plan_backward(plan: P.CPPlan, segs: Sequence[P.Segment], q, k, v, dout, lse, delta, scale: float,
                  mm_dtype: Optional[torch.dtype] = None, dkv_dtype: Optional[torch.dtype] = None,
                  dq_dtype: Optional[torch.dtype] = None):
    """(dq (Tq, Hq, D), dk, dv (Tk, Hkv, D)) over ``plan``'s chunks given the final ``lse`` and ``delta`` (Hq, Tq).

    ``mm_dtype=None``: fp64 throughout.  Otherwise the precision-matched reference: fp32, P^T and dS^T rounded to
    ``mm_dtype`` before their GEMMs (``attn_bwd_sm90.cu``), dQ accumulated in fp32 and rounded once to ``dq_dtype``,
    dK / dV reduced over the GQA group in fp32 and rounded once to ``dkv_dtype`` (default fp32)."""
    lowp = mm_dtype is not None
    cd = torch.float32 if lowp else torch.float64
    tq, hq, d = q.shape
    tk, hkv, _ = k.shape
    rep = hq // hkv
    dq = torch.zeros((tq, hq, d), dtype=cd, device=q.device)
    dk = torch.zeros((tk, hkv, d), dtype=cd, device=q.device)
    dv = torch.zeros_like(dk)
    lse, delta = lse.to(cd), delta.to(cd)
    t2 = float(torch.tensor(scale * LOG2E, dtype=torch.float32))
    rnd = (lambda x: x.to(mm_dtype).to(cd)) if lowp else (lambda x: x)
    for ci, cs in _by_chunk(segs).items():
        ch = plan.q_chunks[ci]
        for r0, r1, ranges in _row_blocks(ch, cs):
            rows = slice(ch.row0 + r0, ch.row0 + r1)
            for s, a, b in ranges:
                if a == b:
                    continue
                keys = slice(s.kv_row0 + a, s.kv_row0 + b)
                for h0, h1 in _head_groups(hq, rep, (r1 - r0) * (b - a)):
                    kvh = slice(h0 // rep, (h1 - 1) // rep + 1)
                    qb, dob = q[rows, h0:h1].to(cd), dout[rows, h0:h1].to(cd)
                    lr = lse[h0:h1, rows].unsqueeze(-1)
                    lr = torch.where(torch.isinf(lr), torch.full_like(lr, float("inf")), lr)  # no key seen: P = 0
                    kk, vv = _kv(k, s, a, b, h0, h1, rep, cd), _kv(v, s, a, b, h0, h1, rep, cd)
                    sc = _scores(qb, kk, s, r0, a)
                    if lowp:
                        p = _exp2_fma(sc, t2, (lr * LOG2E).float())
                    else:
                        p = torch.exp(sc * scale - lr)
                    del sc
                    dp = torch.einsum("nhd,khd->hnk", dob, vv)
                    ds = p * (dp - delta[h0:h1, rows].unsqueeze(-1)) * scale
                    del dp
                    p, ds = rnd(p), rnd(ds)
                    dq[rows, h0:h1] += torch.einsum("hnk,khd->nhd", ds, kk)
                    dk[keys, kvh] += _group_sum(torch.einsum("hnk,nhd->khd", ds, qb), h0, h1, rep)
                    dv[keys, kvh] += _group_sum(torch.einsum("hnk,nhd->khd", p, dob), h0, h1, rep)
    if lowp:
        dq = dq.to(dq_dtype or torch.float32)
        dk, dv = dk.to(dkv_dtype or torch.float32), dv.to(dkv_dtype or torch.float32)
    return dq, dk, dv


# ----------------------------------------------------------------------------------------------
# error bounds
# ----------------------------------------------------------------------------------------------

def _where(idx: int, shape, dims, row_ids=None) -> str:
    coords = []
    for n in reversed(shape):
        coords.append(idx % n)
        idx //= n
    coords = coords[::-1]
    if row_ids is not None and "row" in dims:
        r = dims.index("row")
        coords[r] = int(row_ids[coords[r]])
    return ", ".join(f"{name} {c}" for name, c in zip(dims, coords))


def _record(key: Optional[str], ratio: float):
    if key is not None:
        WORST[key] = max(WORST.get(key, 0.0), ratio)


def _block_max(x: torch.Tensor, blocks) -> torch.Tensor:
    """Max of a non-negative ``x`` over blocks of ``blocks[i]`` consecutive indices along dim ``i`` (None: the whole
    dim); a ragged last block is padded with zeros."""
    pad, shape = [], []
    for n, b in zip(x.shape, blocks):
        b = n if b is None else b
        nb = -(-n // b)
        pad = [0, nb * b - n] + pad
        shape += [nb, b]
    x = torch.nn.functional.pad(x, pad).view(shape)
    return x.amax(dim=tuple(range(1, len(shape), 2)))


def _block_where(idx: int, nblocks, blocks, shape, dims, row_ids=None) -> str:
    coords = []
    for n, b, full in zip(reversed(nblocks), reversed(blocks), reversed(shape)):
        coords.append((idx % n, full if b is None else b, full))
        idx //= n
    parts = []
    for name, (c, b, full) in zip(dims, reversed(coords)):
        if b >= full and b > 1:
            continue
        lo, hi = c * b, min(c * b + b, full) - 1
        if row_ids is not None and name == "row":
            lo, hi = int(row_ids[lo]), int(row_ids[hi])
        parts.append(f"{name} {lo}" if lo == hi else f"{name}s {lo}..{hi}")
    return ", ".join(parts) or "the whole tensor"


def assert_accurate(name: str, got, ref64, ref_lowp, dims=("row", "head", "col"), row_ids=None,
                    factor: Optional[float] = None, report: Optional[str] = None, blocks=None,
                    additions: int = 0) -> float:
    """``max|got - ref64| <= factor * max|ref_lowp - ref64| + 1e-6 max|ref64|``, and the same bound on the mean
    absolute error (which catches small errors spread over many elements).  Returns the max-error ratio.

    ``blocks`` (a block size per dim, None for the whole dim) also holds the max bound within every block, with
    factor ``max(factor, BLOCK_RATIO)`` and the floor from the block's own ``max|ref64|``: at long rows the
    tensor-wide baseline is set by the short rows, whose outputs are far larger, and a lost or mis-scaled work unit
    would hide under it.  The worst block ratio is recorded under ``report + " per-block"``.

    ``additions``: truncating fp32 additions into the kernel's accumulator per element (dK / dV, see
    :data:`ACCUM_ULP`); the floor gains ``ACCUM_ULP * additions * max|ref64|`` (the block's, within a block)."""
    factor = MAX_RATIO if factor is None else factor
    got, ref64, low = got.detach().double(), ref64.detach().double(), ref_lowp.detach().double()
    assert got.shape == ref64.shape == low.shape, (name, got.shape, ref64.shape, low.shape)
    if got.numel() == 0:
        return 0.0
    bad = ~torch.isfinite(got)
    if bad.any():
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{name}: non-finite value at {_where(i, got.shape, dims, row_ids)}")
    err, base = (got - ref64).abs(), (low - ref64).abs()
    if blocks is not None:
        assert len(blocks) == got.dim(), (name, blocks, got.shape)
        eb, bb = _block_max(err, blocks), _block_max(base, blocks)
        rmax = _block_max(ref64.abs(), blocks)
        fb = 1e-6 * rmax.clamp_min(1.0) + ACCUM_ULP * additions * rmax
        rb = eb / torch.maximum(bb, fb)
        limit = max(factor, BLOCK_RATIO)
        over = eb > limit * bb + fb
        if over.any():
            i = int(torch.where(over, rb, torch.zeros_like(rb)).flatten().argmax())
            raise AssertionError(
                f"{name}: block {_block_where(i, rb.shape, blocks, got.shape, dims, row_ids)}: max |err| "
                f"{eb.flatten()[i].item():.3e} is {rb.flatten()[i].item():.2f}x the block's precision-matched "
                f"{bb.flatten()[i].item():.3e} (limit {limit}x + {fb.flatten()[i].item():.1e})")
        del eb, bb, fb, rmax
        if report is not None:
            _record(report + " per-block", rb.max().item())
    # (at least 1e-6 absolute: where every row sees a single key, dS and with it dq / dk are exactly 0, and what is left
    # is the fp32 rounding of dP - delta, with which the precision-matched reference may happen to agree exactly)
    rmax = ref64.abs().max().item()
    floor = 1e-6 * max(rmax, 1.0) + ACCUM_ULP * additions * rmax
    ratios = []
    for what, e, b in (("max", err.max().item(), base.max().item()), ("mean", err.mean().item(), base.mean().item())):
        ratio = e / max(b, floor, 1e-300)
        ratios.append(ratio)
        if e > factor * b + floor:
            i = int(err.flatten().argmax())
            raise AssertionError(
                f"{name}: {what} |err| {e:.3e} is {ratio:.2f}x the precision-matched {b:.3e} (limit {factor}x "
                f"+ {floor:.1e}); worst at {_where(i, got.shape, dims, row_ids)}: got {got.flatten()[i].item():.6g}, "
                f"fp64 {ref64.flatten()[i].item():.6g}, matched {low.flatten()[i].item():.6g}")
    _record(report, ratios[0])
    return ratios[0]


def assert_lse(name: str, got, ref64, ref_lowp=None, dims=("head", "row"), row_ids=None,
               report: Optional[str] = None, rel_limit: Optional[float] = None) -> float:
    """-inf exactly where the fp64 lse is -inf (rows that see no key), elsewhere ``|err| <= 1e-4 (1 + |lse|)``.

    lse is not rounded to a dtype, but its scores are fp32 dot products: with |q|, |k| ~ 30 a score near 0 is the
    difference of terms of ~1e3, and its fp32 rounding alone exceeds 1e-4 (it fails fp32 torch as well).  Where the
    precision-matched lse ``ref_lowp`` (fp32 scores) is that far off, an element may be twice as far off as it.
    Returns the largest ``|err| / (1 + |lse|)``."""
    rel_limit = LSE_REL if rel_limit is None else rel_limit
    got, ref64 = got.detach().double(), ref64.detach().double()
    assert got.shape == ref64.shape, (name, got.shape, ref64.shape)
    empty = torch.isneginf(ref64)
    mism = empty != torch.isneginf(got)
    if mism.any():
        i = int(mism.flatten().nonzero()[0])
        raise AssertionError(f"{name}: -inf mismatch at {_where(i, got.shape, dims, row_ids)}: got "
                             f"{got.flatten()[i].item()}, fp64 {ref64.flatten()[i].item()}")
    if empty.all():
        return 0.0
    tol = 1 + ref64.abs()
    if ref_lowp is not None:
        base = (ref_lowp.detach().double() - ref64).abs()
        tol = torch.maximum(tol, torch.where(empty, torch.zeros_like(base), base) * (MAX_RATIO / rel_limit))
    rel = torch.where(empty, torch.zeros_like(got), (got - ref64).abs() / tol)
    rel = torch.where(torch.isnan(rel), torch.full_like(rel, float("inf")), rel)
    worst = rel.max().item()
    if worst > rel_limit:
        i = int(rel.flatten().argmax())
        raise AssertionError(f"{name}: |err| / (1 + |lse|) = {worst:.3e} > {rel_limit} at "
                             f"{_where(i, got.shape, dims, row_ids)}: got {got.flatten()[i].item():.8g}, "
                             f"fp64 {ref64.flatten()[i].item():.8g}")
    _record(report, worst)
    return worst


# ----------------------------------------------------------------------------------------------
# the sweep: geometries x value regimes
# ----------------------------------------------------------------------------------------------

def _g(name, tq, tk, hq, hkv, chunks, segs):
    """segs: (chunk, kv_row0, kv_len, diag, lo).  ``lo`` is used by the sliding-window runs only."""
    return dict(name=name, tq=tq, tk=tk, hq=hq, hkv=hkv, chunks=chunks, segs=segs)


def _one(name, sq, sk, hq, hkv, diag, lo=None):
    return _g(name, sq, sk, hq, hkv, [(0, sq)], [(0, 0, sk, diag, lo)])


GEOMETRIES = [
    # one chunk x one segment: query rows and key lengths at item / warpgroup / tile edges
    _one("q1_k1", 1, 1, 1, 1, None),
    _one("q63_k64_causal", 63, 64, 2, 1, 0),
    _one("q64_k65_gqa2", 64, 65, 4, 2, 1),
    _one("q65_k127_gqa8", 65, 127, 8, 1, None),
    _one("q127_k128_diag-1", 127, 128, 2, 2, -1),
    _one("q128_k128", 128, 128, 1, 1, None),
    _one("q128_k128_causal", 128, 128, 1, 1, 0),
    _one("q129_k129_gqa8", 129, 129, 16, 2, 0),
    _one("q193_k1024_causal", 193, 1024, 4, 1, 900),
    _one("q256_k256_gqa2", 256, 256, 2, 1, 0),
    _one("q384_k512_gqa2", 384, 512, 4, 2, 128),
    _one("q200_k333", 200, 333, 2, 2, 40),
    _one("q77_k50", 77, 50, 1, 1, None),
    _one("q300_k300_diag-1", 300, 300, 2, 2, -1),
    _one("q512_k1024", 512, 1024, 2, 1, None),
    _one("q100_k65_diag_past_end", 100, 65, 4, 4, 500),
    # whole 64-row backward query tiles see nothing (t_begin > 0); a second chunk sees no key at all
    _g("diag-200_and_blind_chunk", 364, 333, 2, 2, [(0, 300), (300, 64)],
       [(0, 0, 333, -200, None), (1, 0, 333, -64, None)]),
    # several chunks with row0 != 0, kv_row0 off the 128 grid, a gap of rows outside every chunk
    _g("chunks_row0_kvrow0", 520, 1100, 4, 2, [(3, 383), (390, 129), (519, 1)],
       [(0, 5, 333, 200, -100), (1, 77, 129, 0, -64), (2, 0, 1024, None, -1000)]),
    # zigzag-like: adjacent segments, each with its own diag
    _g("zigzag_adjacent", 256, 512, 4, 2, [(0, 128), (128, 128)],
       [(0, 0, 256, None, None), (0, 256, 128, 0, None), (1, 0, 128, None, None), (1, 384, 128, 0, -40)]),
    # llama3-like: overlapping segments of one chunk
    _g("overlapping_segments", 200, 400, 2, 1, [(0, 200)],
       [(0, 0, 300, 100, None), (0, 150, 200, -50, -120)]),
    # sliding windows: a lower bound through a tile, one that leaves a warpgroup's tile invisible, lo > 0, rows whose
    # window starts behind the last key
    _one("window_lo-10", 256, 256, 4, 2, 0, -10),
    _one("window_lo100_diag400", 300, 700, 2, 2, 400, 100),
    _g("window_two_segs", 333, 433, 8, 2, [(0, 333)], [(0, 0, 333, None, -5), (0, 333, 100, 50, -200)]),
    _one("window_rows_past_keys", 200, 150, 2, 1, None, 0),
]

GEOMETRY_NAMES = [g["name"] for g in GEOMETRIES]
WINDOW_AUTO = 70  # window runs of geometries without a lower bound use lo = diag - WINDOW_AUTO

REGIMES = ("randn", "peaked", "peaked_reverse", "large")
REGIME_GEOMETRIES = ("q64_k65_gqa2", "q65_k127_gqa8", "q384_k512_gqa2", "chunks_row0_kvrow0", "zigzag_adjacent",
                     "window_two_segs")

# invisibility: rows 70..135 and 186..199 of Q are in no chunk; keys 0..4, 105..199 and 277..399 in no segment
INVISIBLE_GEOMETRY = _g("invisible_rows", 200, 400, 4, 2, [(0, 70), (136, 50)],
                        [(0, 5, 100, None, None), (1, 200, 77, 30, None), (1, 5, 100, 0, None)])


def single_segment(sq: int, sk: int, hq: int, hkv: int, diag: Optional[int]) -> dict:
    """One chunk of ``sq`` rows x one segment of ``sk`` keys."""
    return _one(f"q{sq}_k{sk}_h{hq}_{hkv}_diag{diag}", sq, sk, hq, hkv, diag)


def geometry(name: str) -> dict:
    return next(g for g in GEOMETRIES + [INVISIBLE_GEOMETRY] if g["name"] == name)


def sweep_cases(geometries=GEOMETRY_NAMES, regime_geometries=REGIME_GEOMETRIES):
    """(geometry name, regime) pairs: every geometry with randn inputs, a subset with the other regimes."""
    cases = [(g, "randn") for g in geometries]
    cases += [(g, r) for r in REGIMES[1:] for g in regime_geometries if g in geometries]
    return cases


def build_plan(geom: dict, window: bool) -> P.CPPlan:
    """A fresh plan per run: device tables are cached on the plan object."""
    auto = window and all(s[4] is None for s in geom["segs"])
    segs = []
    for ch, r0, n, diag, lo in geom["segs"]:
        if not window:
            lo = None
        elif auto:
            lo = (0 if diag is None else diag) - WINDOW_AUTO
        segs.append(P.Segment(ch, 0, r0, n, diag, lo))
    return P.CPPlan(1, 0, geom["tq"], geom["tk"], [P.QChunk(r0, n) for r0, n in geom["chunks"]], segs)


def chunk_rows(plan: P.CPPlan, device) -> torch.Tensor:
    rows = sorted({r for ch in plan.q_chunks for r in range(ch.row0, ch.row0 + ch.rows)})
    return torch.tensor(rows, dtype=torch.long, device=device)


def segment_keys(plan: P.CPPlan, device) -> torch.Tensor:
    keys = sorted({j for s in plan.segments for j in range(s.kv_row0, s.kv_row0 + s.kv_len)})
    return torch.tensor(keys, dtype=torch.long, device=device)


def make_inputs(geom: dict, d: int, dtype, regime: str, device, seed: int = 0):
    """q, k, v, dout in ``dtype``.  ``peaked``: logits span about +-30 and rise with the key index, so a row's maximum
    is its last visible key and every key tile raises the running max (``peaked_reverse``: the maximum is in the first
    tile).  ``large``: |q|, |k| about 30, P nearly one-hot."""
    g = torch.Generator(device=device).manual_seed(seed)
    tq, tk, hq, hkv = geom["tq"], geom["tk"], geom["hq"], geom["hkv"]

    def rn(*shape):
        return torch.randn(shape, generator=g, device=device, dtype=torch.float32)

    q, k, v, do = rn(tq, hq, d), rn(tk, hkv, d), rn(tk, hkv, d), rn(tq, hq, d)
    if regime in ("peaked", "peaked_reverse"):
        ramp = torch.linspace(-1.0, 1.0, tk, device=device)
        if regime == "peaked_reverse":
            ramp = ramp.flip(0)
        q = 1.0 + 0.1 * q  # q . k / sqrt(d) ~ 30 * ramp
        k = (30.0 / math.sqrt(d)) * ramp.view(-1, 1, 1) + 0.1 * k
    elif regime == "large":
        q, k = 30.0 * q.sign() + q, 30.0 * k.sign() + k
    elif regime != "randn":
        raise ValueError(regime)
    return q.to(dtype), k.to(dtype), v.to(dtype), do.to(dtype)


def _tag(kind, geom, d, dtype, window, regime):
    return f"{kind} {geom['name']} D{d} {str(dtype).replace('torch.', '')} {'window' if window else 'plain'} {regime}"


def report_key(kind: str, d: int, dtype, window: bool, regime: str = "randn") -> str:
    key = f"{kind} {str(dtype).replace('torch.', '')} D{d} {'window' if window else 'plain'}"
    return key + " (large)" if regime == "large" else key


def _factor(regime: str) -> float:
    return LARGE_RATIO if regime == "large" else MAX_RATIO


def run_forward(geom: dict, d: int, dtype, window: bool, regime: str, device, seed: int = 0):
    plan = build_plan(geom, window)
    q, k, v, _ = make_inputs(geom, d, dtype, regime, device, seed)
    scale = d ** -0.5
    out, lse = attn_cuda.segments_forward(plan, plan.segments, q, k, v, scale)
    o64, l64 = plan_forward(plan, plan.segments, q, k, v, scale)
    olp, llp = plan_forward(plan, plan.segments, q, k, v, scale, p_dtype=dtype)
    rows = chunk_rows(plan, device)
    tag, key = _tag("fwd", geom, d, dtype, window, regime), report_key("fwd", d, dtype, window, regime)
    assert out.dtype == dtype
    assert_accurate(f"{tag}: out", out[rows], o64[rows], olp[rows], row_ids=rows, factor=_factor(regime), report=key)
    assert_lse(f"{tag}: lse", lse[:, rows], l64[:, rows], llp[:, rows], row_ids=rows, report="lse")


def run_backward(geom: dict, d: int, dtype, window: bool, regime: str, device, dkv_dtype=torch.float32, seed: int = 0,
                 deterministic: bool = False):
    """lse and delta come from the fp64 oracle, so the backward is tested apart from the forward.  ``dkv_dtype``:
    fp32 (the per-source transports) or the model dtype (world size 1 / the fused path).  ``deterministic``: the
    ordered launch groups of ``deterministic=True``.  Returns the kernels' (dq, dk, dv)."""
    plan = build_plan(geom, window)
    q, k, v, do = make_inputs(geom, d, dtype, regime, device, seed)
    scale = d ** -0.5
    o64, l64 = plan_forward(plan, plan.segments, q, k, v, scale)
    delta64 = (o64 * do.double()).sum(-1).transpose(0, 1).contiguous()
    lse32, delta32 = l64.float().contiguous(), delta64.float().contiguous()
    dq = torch.zeros(q.shape, dtype=torch.float32, device=device)
    dk = torch.zeros(k.shape, dtype=dkv_dtype, device=device)
    dv = torch.zeros(v.shape, dtype=dkv_dtype, device=device)
    attn_cuda.segments_backward(plan, plan.segments, do, q, k, v, lse32, delta32, scale, dq, dk, dv, deterministic)
    g64 = plan_backward(plan, plan.segments, q, k, v, do, l64, delta64, scale)
    glp = plan_backward(plan, plan.segments, q, k, v, do, lse32, delta32, scale, mm_dtype=dtype, dkv_dtype=dkv_dtype)
    rows = chunk_rows(plan, device)
    tag, key = _tag("bwd", geom, d, dtype, window, regime), report_key("bwd", d, dtype, window, regime)
    outside = torch.ones(q.shape[0], dtype=torch.bool, device=device)
    outside[rows] = False
    assert not dq[outside].any(), f"{tag}: dq of rows outside every chunk changed"
    f = _factor(regime)
    assert_accurate(f"{tag}: dq", dq[rows], g64[0][rows], glp[0][rows], row_ids=rows, factor=f, report=key)
    assert_accurate(f"{tag}: dk", dk, g64[1], glp[1], factor=f, report=key)
    assert_accurate(f"{tag}: dv", dv, g64[2], glp[2], factor=f, report=key)
    return dq, dk, dv


def _poison(x: torch.Tensor, idx: torch.Tensor):
    """Rows ``idx`` of ``x`` (dim 0) set to +-1e4 (a fixed sign pattern)."""
    sign = torch.ones(x[idx].shape, device=x.device)
    sign.view(sign.shape[0], -1)[:, 1::2] = -1.0
    sign[1::2] *= -1.0
    x = x.clone()
    x[idx] = (1e4 * sign).to(x.dtype)
    return x


def run_invisibility(d: int, dtype, window: bool, backward: bool, device):
    """Rows the plan leaves invisible do not change one bit of the result: K / V rows outside every segment (inside
    the key tiles the kernels load) and Q / dO rows outside every chunk (inside the 64- and 128-row query tiles)."""
    geom = INVISIBLE_GEOMETRY
    q, k, v, do = make_inputs(geom, d, dtype, "randn", device)
    scale = d ** -0.5
    plan = build_plan(geom, window)
    rows, keys = chunk_rows(plan, device), segment_keys(plan, device)
    free_q = torch.tensor([r for r in range(geom["tq"]) if r not in set(rows.tolist())], device=device)
    free_k = torch.tensor([j for j in range(geom["tk"]) if j not in set(keys.tolist())], device=device)
    assert free_q.numel() and free_k.numel()
    o64, l64 = plan_forward(plan, plan.segments, q, k, v, scale)
    delta = (o64 * do.double()).sum(-1).transpose(0, 1).float().contiguous()
    lse = l64.float().contiguous()

    def zero(x, idx):
        x = x.clone()
        x[idx] = 0
        return x

    results = []
    for fill in (zero, _poison):
        qq, dd = fill(q, free_q), fill(do, free_q)
        kk, vv = fill(k, free_k), fill(v, free_k)
        p = build_plan(geom, window)
        if not backward:
            out, l = attn_cuda.segments_forward(p, p.segments, qq, kk, vv, scale)
            results.append((out[rows], l[:, rows]))
        else:
            ll = fill(lse.transpose(0, 1), free_q).transpose(0, 1).contiguous()
            de = fill(delta.transpose(0, 1), free_q).transpose(0, 1).contiguous()
            dq = torch.zeros(q.shape, dtype=torch.float32, device=device)
            dk = torch.zeros(k.shape, dtype=torch.float32, device=device)
            dv = torch.zeros_like(dk)
            attn_cuda.segments_backward(p, p.segments, dd, qq, kk, vv, ll, de, scale, dq, dk, dv)
            results.append((dq, dk, dv))
    for name, a, b in zip(("out", "lse") if not backward else ("dq", "dk", "dv"), *results):
        assert torch.isfinite(a).all() or name == "lse", name
        diff = (a != b) & ~(torch.isnan(a) & torch.isnan(b))
        assert torch.equal(a, b), f"{name} changed at {diff.nonzero()[:4].tolist()} when invisible rows were filled"


def run_delta_and_dq_finalize(dtype, d: int, device):
    """``bwd_delta_kernel`` against the fp64 row sums (also through a head-strided view); ``dq_finalize`` rounds the
    fp32 accumulator once and leaves it zeroed."""
    g = torch.Generator(device=device).manual_seed(5)
    o = torch.randn((333, 3, d), generator=g, device=device).to(dtype)
    do = torch.randn((333, 3, d), generator=g, device=device).to(dtype)
    got = attn_cuda.compute_delta(o, do)
    want64 = (o.double() * do.double()).sum(-1).transpose(0, 1)
    want32 = (o.float() * do.float()).sum(-1).transpose(0, 1)
    assert_accurate(f"delta {dtype} D{d}", got, want64, want32, dims=("head", "row"), report="delta")
    assert torch.equal(attn_cuda.compute_delta(o[:, ::2], do[:, ::2]), got[::2])

    acc = torch.randn((333, 3, d), generator=g, device=device) * 100
    want = acc.to(dtype)
    out = torch.empty_like(want)
    cuda_ext.load().dq_finalize(acc.view(-1), out.view(-1))
    assert torch.equal(out, want)
    assert not acc.any(), "dq_finalize must leave the accumulator zeroed"


def quantize_e4m3(x: torch.Tensor, block: int):
    """(x8, descale (ceil(T / block), H), dequantised fp32) with one descale per ``block`` rows x head of (T, H, D)."""
    t, h, d = x.shape
    nb = -(-t // block)
    xp = torch.cat([x, x.new_zeros(nb * block - t, h, d)]) if nb * block > t else x
    scale = (xp.view(nb, block, h, d).abs().amax(dim=(1, 3)) / 448.0).clamp_min(1e-8)
    per_row = scale.repeat_interleave(block, dim=0)[:t].unsqueeze(-1)
    x8 = (x / per_row).to(torch.float8_e4m3fn)
    return x8, scale.contiguous(), x8.float() * per_row


def run_fp8_forward(geom: dict, blocks: str, device, seed: int = 0):
    """The e4m3 forward (head_dim 128, bf16 out): the oracles see the dequantised inputs, the precision-matched one
    rounds P to bf16.  ``blocks``: one descale per head, or per 64 query rows / 128 keys x head (row-dependent
    magnitudes, so that the block descales differ).  Key blocks must start on the 128-key grid: the kernel takes one
    K / V descale per key tile."""
    d, scale = 128, 128 ** -0.5
    assert all(s[1] % 128 == 0 for s in geom["segs"]) or blocks == "per_head"
    q, k, v, _ = make_inputs(geom, d, torch.float32, "randn", device, seed)
    g = torch.Generator(device=device).manual_seed(seed + 1)
    q = q * (1 + 3 * torch.rand(q.shape[0], 1, 1, generator=g, device=device))
    amp = 1 + 3 * torch.rand(k.shape[0], 1, 1, generator=g, device=device)
    k, v = k * amp, v * amp
    qb, kb = (64, 128) if blocks == "block_scaled" else (geom["tq"], geom["tk"])
    q8, qs, qd = quantize_e4m3(q, qb)
    k8, ks, kd = quantize_e4m3(k, kb)
    v8, vs, vd = quantize_e4m3(v, kb)
    plan = build_plan(geom, False)
    with attn_cuda.fp8_scales(attn_cuda.Fp8Scales(qs, qb, ks, vs, kb)):
        out, lse = attn_cuda.segments_forward(plan, plan.segments, q8, k8, v8, scale)
    o64, l64 = plan_forward(plan, plan.segments, qd, kd, vd, scale)
    olp, llp = plan_forward(plan, plan.segments, qd, kd, vd, scale, p_dtype=torch.bfloat16)
    rows = chunk_rows(plan, device)
    tag = f"fwd fp8 {geom['name']} {blocks}"
    assert out.dtype == torch.bfloat16
    assert_accurate(f"{tag}: out", out[rows], o64[rows], olp[rows], row_ids=rows, factor=FP8_RATIO,
                    report="fwd e4m3 D128 plain")
    assert_lse(f"{tag}: lse", lse[:, rows], l64[:, rows], llp[:, rows], row_ids=rows, report="lse e4m3",
               rel_limit=FP8_LSE_REL)


# ----------------------------------------------------------------------------------------------
# whole-problem references for the public API at world size 1
# ----------------------------------------------------------------------------------------------

def api_reference(q, k, v, dout, cu_seqlens, causal: bool, window=(-1, -1), scale: Optional[float] = None,
                  dtype: Optional[torch.dtype] = None):
    """Packed documents q (T, Hq, D), k / v (T, Hkv, D) (``attention_oracle``'s masks, one chunk and one segment per
    document).  Returns (fp64, precision-matched) dicts of out, lse (Hq, T), and - with ``dout`` - dq, dk, dv.

    The precision-matched side follows the training path in ``dtype`` (default q's; bf16 for dequantised fp8 inputs):
    P and out rounded, delta = rowsum(rounded out * dout) in fp32, P^T / dS^T rounded, dq / dk / dv rounded once."""
    cu = [int(x) for x in cu_seqlens]
    left, right = window
    if causal:
        right = 0
    diag = right if right >= 0 else None
    lo = -left if left >= 0 else None
    chunks = [P.QChunk(a, b - a) for a, b in zip(cu[:-1], cu[1:])]
    segs = [P.Segment(i, 0, ch.row0, ch.rows, diag, lo) for i, ch in enumerate(chunks)]
    plan = P.CPPlan(1, 0, q.shape[0], k.shape[0], chunks, segs)
    scale = q.shape[-1] ** -0.5 if scale is None else scale
    dtype = dtype or q.dtype
    o64, l64 = plan_forward(plan, segs, q, k, v, scale)
    olp, llp = plan_forward(plan, segs, q, k, v, scale, p_dtype=dtype)
    ref64, reflp = dict(out=o64, lse=l64), dict(out=olp, lse=llp)
    if dout is not None:
        delta64 = (o64 * dout.double()).sum(-1).transpose(0, 1)
        deltalp = (olp.float() * dout.float()).sum(-1).transpose(0, 1)
        ref64.update(zip(("dq", "dk", "dv"), plan_backward(plan, segs, q, k, v, dout, l64, delta64, scale)))
        reflp.update(zip(("dq", "dk", "dv"), plan_backward(plan, segs, q, k, v, dout, llp, deltalp, scale,
                                                           mm_dtype=dtype, dkv_dtype=dtype, dq_dtype=dtype)))
    return ref64, reflp


def work_units(key: str) -> dict:
    """``assert_accurate`` blocks (and dim names) of a token-major output: the kernels' units of work, per (query
    head, 64-row block) for out / dq, per (kv head, 128-key tile) for dk / dv."""
    if key in ("dk", "dv"):
        return dict(blocks=(128, 1, None), dims=("key", "kv head", "col"))
    return dict(blocks=(64, 1, None), dims=("row", "head", "col"))


def wgmma_additions(tq: int, hq: int, hkv: int) -> int:
    """An upper bound on the additions into one key tile's dK / dV accumulator at world size 1: every 64-row query
    tile of every query head of the GQA group, :data:`WGMMA_PER_TILE` each."""
    return WGMMA_PER_TILE * (hq // hkv) * -(-tq // 64)


def assert_api(name: str, got: dict, ref64: dict, reflp: dict, fp8: bool = False, per_block: bool = False,
               report: Optional[str] = None):
    """Every output in ``got`` (out / dq / dk / dv token-major, lse (Hq, T)) against :func:`api_reference`
    (``fp8``: the e4m3 forward's bounds; ``per_block``: the bound within every :func:`work_units` block too).  dK /
    dV allow for the backward's accumulator (:func:`wgmma_additions`)."""
    for key, val in got.items():
        if key == "lse":
            assert_lse(f"{name}: lse", val, ref64["lse"], reflp["lse"], report="lse e4m3" if fp8 else "lse",
                       rel_limit=FP8_LSE_REL if fp8 else None)
        else:
            assert val.dtype == reflp[key].dtype, (name, key, val.dtype)
            assert_accurate(f"{name}: {key}", val, ref64[key], reflp[key], factor=FP8_RATIO if fp8 else None,
                            report=report or f"api {'e4m3' if fp8 else val.dtype}",
                            additions=_additions(key, ref64), **(work_units(key) if per_block else {}))


def run_api(fn_name: str, b: int, s: int, hq: int, hkv: int, d: int, dtype, causal: bool = True, window=(-1, -1),
            regime: str = "randn", backward: bool = True, kv_heads=None, device="cuda", seed: int = 0,
            report: Optional[str] = None):
    """One batched call of a public world-1 entry point (``*_qkvpacked_func`` or ``*_kvpacked_func``; inputs drawn on
    ``device``), forward and optionally backward, against :func:`api_reference` with the bound held within every
    :func:`work_units` block as well.  ``kv_heads``: check only these kv heads and their query heads (every head
    runs).  Returns the outputs (token-major, lse (Hq, T)) and the inputs (q, k, v, dout)."""
    import ring_flash_attn_b200 as rfa

    t = b * s
    q, k, v, dout = make_inputs(dict(tq=t, tk=t, hq=hq, hkv=hkv), d, dtype, regime, device, seed)
    fn = getattr(rfa, fn_name)
    kw = dict(causal=causal, window_size=window, return_attn_probs=True)
    if "qkvpacked" in fn_name:
        x = torch.stack([q, k, v], dim=1).view(b, s, 3, hq, d).requires_grad_(backward)
        out, lse, _ = fn(x, **kw)
    else:
        xq = q.view(b, s, hq, d).clone().requires_grad_(backward)
        x = torch.stack([k, v], dim=1).view(b, s, 2, hkv, d).requires_grad_(backward)
        out, lse, _ = fn(xq, x, **kw)
    got = dict(out=out.detach().reshape(t, hq, d), lse=lse.detach().permute(1, 0, 2).reshape(hq, t))
    if backward:
        out.backward(dout.view(out.shape))
        if "qkvpacked" in fn_name:
            g = x.grad.view(t, 3, hq, d)
            got.update(dq=g[:, 0], dk=g[:, 1], dv=g[:, 2])
        else:
            g = x.grad.view(t, 2, hkv, d)
            got.update(dq=xq.grad.view(t, hq, d), dk=g[:, 0], dv=g[:, 1])
    del out, lse, x
    check_api_heads(f"{fn_name} B{b} S{s} h{hq}/{hkv} D{d} {regime}", got, q, k, v, dout if backward else None,
                    list(range(0, t + 1, s)), causal, window, kv_heads, report)
    return got, (q, k, v, dout)


def _additions(key: str, ref64: dict) -> int:
    if key not in ("dk", "dv") or "dq" not in ref64:
        return 0
    tq, hq, _ = ref64["dq"].shape
    return wgmma_additions(tq, hq, ref64["dk"].shape[1])


def check_api_heads(name: str, got: dict, q, k, v, dout, cu, causal: bool, window, kv_heads=None,
                    report: Optional[str] = None):
    """:func:`assert_api` with ``per_block``, on every head or on ``kv_heads`` and their GQA groups only: the
    reference then computes those heads alone."""
    hq, hkv = q.shape[1], k.shape[1]
    qh = kh = slice(None)
    if kv_heads is not None:
        rep = hq // hkv
        qh, kh = [h * rep + i for h in kv_heads for i in range(rep)], list(kv_heads)
    got = {key: (val[qh] if key == "lse" else val[:, kh if key in ("dk", "dv") else qh]) for key, val in got.items()}
    ref64, reflp = api_reference(q[:, qh], k[:, kh], v[:, kh], None if dout is None else dout[:, qh], cu, causal,
                                 window)
    assert_api(name, got, ref64, reflp, per_block=True, report=report)
