"""fp64 and precision-matched references for the sm_90a split-KV decode kernel (``csrc/decode_sm90.cu``), and the
sweep built on them.

A case (:class:`Case`) is one ``kernel_decode`` call: the sequences' cache lengths and new-token counts, the heads,
the capacity, the split count, causal or not, whether ``k`` / ``v`` are appended, the cache layout (contiguous, paged,
or K / V as views of one packed tensor), the cache dtype (native or e4m3) and rotary embeddings.  :func:`run_decode`
builds seeded inputs for it, calls ``parallel.decode.kernel_decode`` through whatever ``cuda_ext.load()`` returns (the
sm_90a extension in ``tests/test_gpu_decode_accuracy.py``, ``tests/fake_ext.FakeDecodeExt`` and mutated copies of it in
``tests/test_decode_oracle_cpu.py``), and holds the result to ``kernel_oracle``'s bound: at most twice as far from the
fp64 result as a reference that rounds where the kernel rounds.  After the call it checks the cache bytes.

The fp64 reference (:func:`references`) works from first principles: the dequantised cache, q (and a bf16 / fp16
cache's appended k) rotated in fp64 from the unrotated inputs, the visibility rule of the ``decode_sm90.cu`` file
comment, one softmax over every visible key.  An e4m3 cache's appended rows enter as the bytes the append must store
(checked bitwise on their own), so that e4m3 quantisation stays out of the bound.  The precision-matched reference
rotates with ``apply_rotary`` (bitwise the kernel's rotation), splits the keys into the kernel's ranges of
``tiles_per_split`` 128-key tiles, forms P with ``exp2(fmaf(s, t2, -m))`` against each split's row maximum, rounds P to
q's dtype before P V, and merges the split partials in fp32 before one rounding to q's dtype.
"""
from __future__ import annotations

import dataclasses
import math
from dataclasses import dataclass
from typing import Optional, Tuple

import torch

import kernel_oracle as KO
from ring_flash_attn_b200.parallel import decode as dec
from test_decode_paged import to_pool
from test_decode_rotary import rope_tables
from test_decode_varlen import appended, cu_of, pack
from test_gpu_decode_fp8 import bytes_of

LN2 = math.log(2.0)
TILE = dec.KEY_TILE
SM_COUNT_CPU = 132  # the split count a CPU run assumes for ``splits=None`` (an H100 SXM has 132 SMs)


@dataclass(frozen=True)
class Case:
    """One decode call.  ``counts``: new tokens per sequence (all equal unless ``varlen``); ``seqlens``: the
    ``cache_seqlens`` (may exceed ``s_cap``); ``splits=None``: the ``num_splits`` default.  ``layout``: "contiguous",
    "paged" (``page_size``, shuffled table, -1 past the allocated pages), "packed_kv" (views ``kv[:, :, 0]`` /
    ``kv[:, :, 1]`` of one ``(B, S_cap, 2, Hkv, D)`` tensor) or "head_strided" (views of ``(B, S_cap, Hkv, 2, D)``).
    ``rotary``: ``(rotary_dim, interleaved)`` with rotary_dim 16, "half" or "full".  ``saturate``: with an e4m3 cache,
    some appended values are far past +-448 times their descale."""
    name: str
    counts: Tuple[int, ...]
    seqlens: Tuple[int, ...]
    s_cap: int
    hq: int = 8
    hkv: int = 2
    varlen: bool = False
    splits: Optional[int] = None
    causal: bool = True
    append: bool = True
    layout: str = "contiguous"
    page_size: int = 0
    fp8: bool = False
    saturate: bool = False
    rotary: Optional[Tuple[object, bool]] = None

    def __post_init__(self):
        assert len(self.counts) == len(self.seqlens) and self.hq % self.hkv == 0
        assert self.varlen or len(set(self.counts)) == 1
        assert (self.layout == "paged") == (self.page_size > 0)
        assert self.page_size == 0 or self.s_cap % self.page_size == 0
        assert self.rotary is None or self.append

    @property
    def b(self) -> int:
        return len(self.seqlens)

    @property
    def group(self) -> int:
        return self.hq // self.hkv

    def rotary_dim(self, d: int) -> int:
        r = self.rotary[0]
        return d // 2 if r == "half" else (d if r == "full" else int(r))


def _u(name, b, sq, s_cap, seqlens, **kw):
    return Case(name, (sq,) * b, tuple(seqlens), s_cap, **kw)


def _v(name, counts, s_cap, seqlens, **kw):
    return Case(name, tuple(counts), tuple(seqlens), s_cap, varlen=True, **kw)


# 44 sequences (two 32-sequence steps of the varlen prefix sum): zero counts, single tokens, one 20-token chunk (80
# packed rows at G = 4: two row tiles) past index 32, and zero counts at the end, so that tile slots sit idle
VARLEN_COUNTS = tuple(20 if i == 35 else (0, 1, 2, 1, 3, 0, 1, 1)[i % 8] for i in range(42)) + (0, 0)
VARLEN_SEQLENS = tuple((37 * i + 5) % 600 for i in range(44))

GEOMETRIES = [
    # packed rows Sq * G at the 64-row tile edges, G = 1, 2, 3, 4, 8, 16
    _u("rows1_g1", 2, 1, 700, (650, 3), hq=2, hkv=2),
    # (rows63_g1: Hq = 1 and 63 rows make the partial of a split an odd number of floats, so split 1 starts 4 bytes
    # off the 8-byte alignment of the kernel's float2 stores, unless kernel_decode pads the partial stride)
    _u("rows63_g1", 1, 63, 600, (500,), hq=1, hkv=1, splits=2),
    _u("rows64_g16", 2, 4, 900, (800, 37), hq=16, hkv=1),
    _u("rows64_g2", 2, 32, 512, (400, 100), hq=4, hkv=2, causal=False),
    _u("rows65_g1_one_live_row", 1, 65, 700, (300,), hq=2, hkv=2, causal=False),
    _u("rows128_g8", 1, 16, 1000, (900,), hq=16, hkv=2),
    _u("rows129_g3", 1, 43, 800, (700,), hq=6, hkv=2, splits=3),
    # visible keys at the 128-key tile edges: 0, 1, 127, 128, 129 without an append (n_vis = 0 though causal), and
    # the same counts reached through a causal append; more splits than the visible keys need
    _u("keys_0_1_127_128_129", 5, 2, 300, (0, 1, 127, 128, 129), append=False, splits=3),
    _u("keys_1_127_128_129_by_append", 4, 1, 300, (0, 126, 127, 128), splits=3, hq=4, hkv=1),
    # one key below, at and above the split boundary tiles_per_split * 128 = 512 (2048 keys, 4 splits)
    _u("split_edge", 3, 2, 2048, (511, 512, 513), append=False, splits=4, causal=False),
    _u("split_edge_by_append", 3, 4, 2048, (508, 510, 512), splits=4),
    # split counts: 1, the default, 3 of 10 tiles (tiles_per_split 4: the last split has 2), 8 of 3 tiles
    _u("splits1", 2, 2, 1500, (1400, 1000), splits=1, causal=False),
    _u("splits_default", 2, 3, 3000, (2900, 1700)),
    _u("splits3_of_10_tiles", 2, 2, 1280, (1250, 1270), splits=3),
    _u("splits8_of_3_tiles", 2, 1, 300, (1, 200), splits=8, hq=4, hkv=1),
    # S_cap edges: not a multiple of 128 and filled by the append; an append that overflows (some rows and all rows
    # dropped); cache_seqlens > S_cap; empty shards with and without an append
    _u("scap300_filled", 2, 4, 300, (296, 300), splits=2),
    _u("append_overflow", 3, 4, 520, (518, 520, 600), causal=False),
    _u("empty_shard_append", 2, 3, 400, (0, 0)),
    _u("empty_shard_no_append", 2, 3, 400, (0, 250), append=False),
    _u("no_append_noncausal", 2, 2, 900, (899, 300), append=False, causal=False),
    # paged caches: every page size, shuffled tables; one split over 80+ pages (the table window refills twice);
    # page 256 with tiles_per_split 1, so that odd splits start mid-page
    _u("paged16", 3, 4, 1024, (1000, 15, 500), layout="paged", page_size=16),
    _u("paged32", 2, 2, 800, (790, 31), layout="paged", page_size=32, causal=False),
    _u("paged64", 2, 3, 768, (700, 63), layout="paged", page_size=64, splits=4),
    _u("paged128", 2, 4, 1024, (1000, 127), layout="paged", page_size=128, splits=3),
    _u("paged256_mid_page_split", 2, 2, 1024, (1000, 255), layout="paged", page_size=256, splits=8),
    _u("paged16_refill", 1, 2, 1600, (1400,), layout="paged", page_size=16, splits=1),
    # caches whose row and head strides are not the defaults
    _u("packed_kv", 2, 3, 700, (650, 100), layout="packed_kv"),
    _u("head_strided", 2, 2, 600, (590, 40), layout="head_strided", causal=False),
    # e4m3 only: appended values that saturate at +-448
    _u("saturating_append", 2, 3, 400, (300, 50), saturate=True),
    # varlen: contiguous and paged
    _v("varlen44", VARLEN_COUNTS, 640, VARLEN_SEQLENS),
    _v("varlen44_paged32", VARLEN_COUNTS, 640, VARLEN_SEQLENS, layout="paged", page_size=32, causal=False),
    # rotary: interleaved and not, rotary_dim 16 / D/2 / D, causal and not, with varlen and a paged cache
    _u("rotary16_interleaved", 2, 4, 600, (500, 30), rotary=(16, True)),
    _u("rotary_half_neox_noncausal", 2, 3, 600, (550, 7), rotary=("half", False), causal=False),
    _u("rotary_full_neox_paged64", 2, 2, 512, (300, 17), layout="paged", page_size=64, rotary=("full", False)),
    _v("rotary_full_interleaved_varlen_noncausal", (3, 0, 1, 5), 400, (350, 9, 0, 200), rotary=("full", True),
       causal=False),
    _v("rotary_half_neox_varlen", (2, 6, 1), 400, (100, 390, 3), rotary=("half", False)),
    # one long shard with the default split count
    _u("long20k", 1, 2, 20000, (19990,), hq=8, hkv=1),
]

GEOMETRY_NAMES = [g.name for g in GEOMETRIES]
REGIMES = ("randn", "peaked", "peaked_reverse", "large", "v_offset")
# peaked: the dominant key is each row's last visible one, in the last tile of the last non-empty split
# (splits3_of_10_tiles, split_edge_by_append); peaked_reverse: it is key 0, in the first split
REGIME_GEOMETRIES = ("rows129_g3", "split_edge_by_append", "splits3_of_10_tiles", "paged256_mid_page_split",
                     "varlen44")


def geometry(name: str, **overrides) -> Case:
    g = next(g for g in GEOMETRIES if g.name == name)
    return dataclasses.replace(g, **overrides) if overrides else g


def sweep_cases(geometries=GEOMETRY_NAMES, regime_geometries=REGIME_GEOMETRIES):
    """(geometry name, regime) pairs: every geometry with randn inputs, a subset with the other regimes."""
    cases = [(g, "randn") for g in geometries]
    cases += [(g, r) for r in REGIMES[1:] for g in regime_geometries if g in geometries]
    return cases


def spans(case: Case):
    """(first packed row, count) of every sequence."""
    cu = cu_of(case.counts).tolist()
    return [(cu[i], n) for i, n in enumerate(case.counts)]


def descales(b: int, hkv: int, which: str, device) -> torch.Tensor:
    """Per-(sequence, kv head) descales, not powers of two, different for K and V."""
    base, step = (0.37, 0.1) if which == "k" else (0.55, 0.07)
    return (base * (1 + step * torch.arange(b * hkv, dtype=torch.float32))).view(b, hkv).to(device)


def default_splits(case: Case, device) -> int:
    dev = torch.device(device)
    sm = dec._sm_count(dev.index if dev.index is not None else torch.cuda.current_device()) \
        if dev.type == "cuda" else SM_COUNT_CPU
    s_cap, sq = case.s_cap, max(max(case.counts), 1)
    if case.varlen:
        return dec.num_splits_varlen(case.b, sum(case.counts), sq, case.hq, case.hkv, s_cap, sm)
    return dec.num_splits(case.b, sq, case.hq, case.hkv, s_cap, sm)


# ----------------------------------------------------------------------------------------------
# inputs
# ----------------------------------------------------------------------------------------------

@dataclass
class Inputs:
    case: Case
    dtype: torch.dtype
    d: int
    q: torch.Tensor  # (rows, Hq, D) packed, unrotated
    k_new: torch.Tensor  # (rows, Hkv, D) packed, unrotated
    v_new: torch.Tensor
    lens: list  # cache_seqlens clamped to [0, S_cap]
    seqlens: torch.Tensor  # (B,) int32, as passed
    kc0: torch.Tensor  # (B, S_cap, Hkv, D) the logical cache before the call, in the cache dtype (NaN past lens)
    vc0: torch.Tensor
    k_cache: torch.Tensor  # what the kernel gets (and appends to), in the case's layout
    v_cache: torch.Tensor
    table: Optional[torch.Tensor]
    k_descale: Optional[torch.Tensor]  # (B, Hkv) fp32
    v_descale: Optional[torch.Tensor]
    rotary: Optional[tuple]  # (cos, sin, rotary_seqlens list, interleaved)
    stored_k: torch.Tensor  # (rows, Hkv, D) in the cache dtype: what the append must store
    stored_v: torch.Tensor


def _ramp(n_keys: int, positions: torch.Tensor, reverse: bool) -> torch.Tensor:
    r = (-1.0 + 2.0 * positions.float() / max(n_keys - 1, 1)).clamp(-1.0, 1.0)
    return -r if reverse else r


def _layout(case: Case, kc: torch.Tensor, vc: torch.Tensor, lens, seed: int):
    """(k_cache, v_cache, block_table) holding the logical cache ``kc`` / ``vc`` in the case's layout."""
    b, s_cap, hkv, d = kc.shape
    if case.layout == "contiguous":
        return kc.clone(), vc.clone(), None
    if case.layout == "packed_kv":
        kv = torch.empty((b, s_cap, 2, hkv, d), dtype=kc.dtype, device=kc.device)
        kv[:, :, 0], kv[:, :, 1] = kc, vc
        return kv[:, :, 0], kv[:, :, 1], None
    if case.layout == "head_strided":
        kv = torch.empty((b, s_cap, hkv, 2, d), dtype=kc.dtype, device=kc.device)
        kv[:, :, :, 0], kv[:, :, :, 1] = kc, vc
        return kv[:, :, :, 0], kv[:, :, :, 1], None
    assert case.layout == "paged"
    alloc = [min(n + (c if case.append else 0), s_cap) for n, c in zip(lens, case.counts)]
    return to_pool(kc, vc, lens, case.page_size, alloc=alloc, seed=seed)


def build_inputs(case: Case, dtype, d: int, regime: str, device, seed: int = 0,
                 cache_seed: Optional[int] = None, draw="cpu") -> Inputs:
    """Seeded inputs, drawn on ``draw``: the CPU by default, so the same on every device; ``draw=device`` for caches
    of gigabytes.  q / k / v come from ``seed``, the cache from ``cache_seed`` (default ``seed + 1``), so ranks can
    share the new tokens and hold different shards.  Regimes:
    ``randn``; ``peaked`` (logits span about +-30 and rise with the key position, so a row's maximum is its last
    visible key) and ``peaked_reverse`` (key 0); ``large`` (|q|, |k| about 30); ``v_offset`` (V = 50 + randn)."""
    b, hq, hkv, s_cap = case.b, case.hq, case.hkv, case.s_cap
    smax = max(max(case.counts), 1)
    gq = torch.Generator(device=draw).manual_seed(seed)
    gc = torch.Generator(device=draw).manual_seed(seed + 1 if cache_seed is None else cache_seed)

    def rn(*shape, g):
        return torch.randn(shape, generator=g, device=draw)

    q4 = rn(b, smax, hq, d, g=gq)
    kn4, vn4 = rn(b, smax, hkv, d, g=gq), rn(b, smax, hkv, d, g=gq)
    kc, vc = rn(b, s_cap, hkv, d, g=gc), rn(b, s_cap, hkv, d, g=gc)
    lens = [min(max(int(s), 0), s_cap) for s in case.seqlens]
    if regime in ("peaked", "peaked_reverse"):
        rev = regime == "peaked_reverse"
        amp = 30.0 / math.sqrt(d)  # q . k / sqrt(d) ~ 30 * ramp
        q4 = 1.0 + 0.1 * q4
        for i, (n, c) in enumerate(zip(lens, case.counts)):
            vis = min(n + (c if case.append else 0), s_cap)
            kc[i] = amp * _ramp(vis, torch.arange(s_cap, device=draw), rev).view(-1, 1, 1) + 0.1 * kc[i]
            kn4[i] = amp * _ramp(vis, n + torch.arange(smax, device=draw), rev).view(-1, 1, 1) + 0.1 * kn4[i]
    elif regime == "large":
        q4, kn4, kc = (30.0 * x.sign() + x for x in (q4, kn4, kc))
    elif regime == "v_offset":
        vn4, vc = vn4 + 50.0, vc + 50.0
    elif regime != "randn":
        raise ValueError(regime)
    fp8 = case.fp8
    if fp8 and case.saturate:  # +-1000: past 448 * descale for every descale here
        sign = torch.ones(smax, hkv, device=draw)
        sign[1::2] = -1.0
        kn4[..., 3] = 1000.0 * sign
        vn4[..., 5] = -1000.0 * sign
    for i, n in enumerate(lens):  # rows past the valid ones must never reach a result
        kc[i, n:] = float("nan")
        vc[i, n:] = float("nan")
    q4, kn4, vn4 = q4.to(dtype), kn4.to(dtype), vn4.to(dtype)
    q, k_new, v_new = (pack(x, case.counts).to(device) for x in (q4, kn4, vn4))
    kd = vd = None
    if fp8:
        kd, vd = descales(b, hkv, "k", draw), descales(b, hkv, "v", draw)
        kc = torch.stack([dec.quantize_e4m3(kc[i], kd[i]) for i in range(b)])
        vc = torch.stack([dec.quantize_e4m3(vc[i], vd[i]) for i in range(b)])
        kd, vd = kd.to(device), vd.to(device)
    else:
        kc, vc = kc.to(dtype), vc.to(dtype)
    kc0, vc0 = kc.to(device), vc.to(device)
    k_cache, v_cache, table = _layout(case, kc0, vc0, lens, seed)
    rotary = None
    k_rot = k_new
    sp = spans(case)
    if case.rotary is not None:
        rs = [2 * n + 5 for n in lens]  # positions of the first new tokens: not the cache lengths
        cos, sin = rope_tables(max(r + c for r, c in zip(rs, case.counts)) + 3, case.rotary_dim(d), dtype, device)
        rotary = (cos, sin, rs, case.rotary[1])
        key_pos = torch.tensor([r + t for r, (_, c) in zip(rs, sp) for t in range(c)], dtype=torch.long,
                               device=device)
        k_rot = dec.apply_rotary(k_new, cos, sin, key_pos, case.rotary[1])
    if fp8:
        stored_k = torch.cat([dec.quantize_e4m3(k_rot[lo:lo + n], kd[i]) for i, (lo, n) in enumerate(sp)])
        stored_v = torch.cat([dec.quantize_e4m3(v_new[lo:lo + n], vd[i]) for i, (lo, n) in enumerate(sp)])
    else:
        stored_k, stored_v = k_rot, v_new
    seqlens = torch.tensor(case.seqlens, dtype=torch.int32, device=device)
    return Inputs(case, dtype, d, q, k_new, v_new, lens, seqlens, kc0, vc0, k_cache, v_cache,
                  table.to(device) if table is not None else None, kd, vd, rotary, stored_k, stored_v)


# ----------------------------------------------------------------------------------------------
# references
# ----------------------------------------------------------------------------------------------

def _rotate64(x: torch.Tensor, cos, sin, pos: torch.Tensor, interleaved: bool) -> torch.Tensor:
    """x (n, H, D) rotated in fp64 at table rows ``pos`` (n,): column pairs (2i, 2i + 1) when interleaved, else
    (i, i + rotary_dim / 2), ``a' = a cos - b sin``, ``b' = b cos + a sin``; columns past rotary_dim unchanged."""
    h = cos.shape[1]
    c, s = cos[pos].double().unsqueeze(1), sin[pos].double().unsqueeze(1)
    x = x.double()
    y = x.clone()
    ia, ib = (slice(0, 2 * h, 2), slice(1, 2 * h, 2)) if interleaved else (slice(0, h), slice(h, 2 * h))
    a, b = x[..., ia], x[..., ib]
    y[..., ia] = a * c - b * s
    y[..., ib] = b * c + a * s
    return y


def _grouped_scores(q, k, hkv):
    """q (t, Hq, D), k (j, Hkv, D) -> (Hq, t, j); query head h reads kv head h // G."""
    t, hq, d = q.shape
    return torch.einsum("tkgd,jkd->kgtj", q.view(t, hkv, hq // hkv, d), k).reshape(hq, t, k.shape[0])


def references(inp: Inputs, n_splits: int, appended_here: Optional[bool] = None, scale: Optional[float] = None):
    """(out64 (rows, Hq, D), lse64 (Hq, rows)) in fp64 and the precision-matched (out32, lse32) in fp32, before the
    final rounding of out to q's dtype.  ``appended_here``: whether this shard takes the append (default: the
    case's)."""
    case, dtype, d = inp.case, inp.dtype, inp.d
    hq, hkv, s_cap, g = case.hq, case.hkv, case.s_cap, case.group
    appended_here = case.append if appended_here is None else appended_here
    scale = d ** -0.5 if scale is None else scale
    dev = inp.q.device
    rows = inp.q.shape[0]
    out64 = torch.zeros((rows, hq, d), dtype=torch.float64, device=dev)
    lse64 = torch.full((hq, rows), float("-inf"), dtype=torch.float64, device=dev)
    out32 = torch.zeros((rows, hq, d), dtype=torch.float32, device=dev)
    lse32 = torch.full((hq, rows), float("-inf"), dtype=torch.float32, device=dev)
    tiles = max(1, -(-s_cap // TILE))
    span = -(-tiles // n_splits) * TILE  # keys per split
    t2 = torch.tensor(scale * KO.LOG2E, dtype=torch.float32, device=dev)
    fp8 = case.fp8
    for b, (lo, cnt) in enumerate(spans(case)):
        if cnt == 0:
            continue
        n = inp.lens[b]
        m = min(cnt, s_cap - n) if appended_here else 0  # appended rows that fit
        t = torch.arange(cnt, device=dev)
        n_vis = (t + 1 if case.causal else torch.full_like(t, cnt)) if appended_here else torch.zeros_like(t)
        lim = (n + n_vis).clamp(max=s_cap)
        keys = n + m
        vis = torch.arange(keys, device=dev).unsqueeze(0) < lim.unsqueeze(1)  # (cnt, keys)
        new = slice(lo, lo + m)
        qrows = inp.q[lo:lo + cnt]
        # ---- fp64: dequantised cache, fp64 rotation from the unrotated inputs
        if fp8:
            kd, vd = inp.k_descale[b].double()[:, None], inp.v_descale[b].double()[:, None]
            k64 = torch.cat([inp.kc0[b, :n].double(), inp.stored_k[new].double()]) * kd
            v64 = torch.cat([inp.vc0[b, :n].double(), inp.stored_v[new].double()]) * vd
        else:
            kn = inp.k_new[new].double()
            if inp.rotary is not None:
                cos, sin, rs, inter = inp.rotary
                kn = _rotate64(inp.k_new[new], cos, sin, rs[b] + torch.arange(m, device=dev), inter)
            k64 = torch.cat([inp.kc0[b, :n].double(), kn])
            v64 = torch.cat([inp.vc0[b, :n].double(), inp.v_new[new].double()])
        q64, qlp = qrows.double(), qrows
        if inp.rotary is not None:
            cos, sin, rs, inter = inp.rotary
            qpos = rs[b] + (t if case.causal else torch.zeros_like(t))
            q64 = _rotate64(qrows, cos, sin, qpos, inter)
            qlp = dec.apply_rotary(qrows, cos, sin, qpos, inter)
        s = (_grouped_scores(q64, k64, hkv) * scale).masked_fill(~vis, float("-inf"))  # (Hq, cnt, keys)
        l64 = torch.logsumexp(s, dim=-1)
        p = torch.exp(s - torch.where(torch.isinf(l64), torch.zeros_like(l64), l64).unsqueeze(-1))
        o = torch.einsum("kgtj,jkd->tkgd", p.view(hkv, g, cnt, keys), v64).reshape(cnt, hq, d)
        out64[lo:lo + cnt] = o
        lse64[:, lo:lo + cnt] = l64
        # ---- precision-matched: the kernel's split ranges, fp32 scores, P rounded to q's dtype, fp32 combine
        klp = torch.cat([inp.kc0[b, :n], inp.stored_k[new]]).to(dtype).float()  # e4m3 widens exactly
        vlp = torch.cat([inp.vc0[b, :n], inp.stored_v[new]]).to(dtype).float()
        pad = n_splits * span - keys
        s32 = _grouped_scores(qlp.float(), klp, hkv).masked_fill(~vis, float("-inf"))
        s32 = torch.nn.functional.pad(s32, (0, pad), value=float("-inf")).view(hq, cnt, n_splits, span)
        tt = t2 * inp.k_descale[b].repeat_interleave(g).view(hq, 1, 1, 1) if fp8 else t2
        mx = s32.amax(dim=-1, keepdim=True)
        empty = torch.isinf(mx)
        m2 = torch.where(empty, torch.zeros_like(mx), mx * tt)
        p = KO._exp2_fma(s32, tt, m2)
        l = p.sum(dim=-1, keepdim=True)
        vp = torch.nn.functional.pad(vlp, (0, 0, 0, 0, 0, pad)).view(n_splits, span, hkv, d)
        o = torch.einsum("kgtsj,sjkd->kgtsd", p.to(dtype).float().view(hkv, g, cnt, n_splits, span), vp)
        inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
        if fp8:
            inv = inv * inp.v_descale[b].repeat_interleave(g).view(hq, 1, 1, 1)
        o = o.reshape(hq, cnt, n_splits, d) * inv
        lse_s = torch.where(empty, torch.full_like(l, float("-inf")), (m2 + torch.log2(l)) * LN2)
        oc, lc = _combine32(o, lse_s, dim=2)
        out32[lo:lo + cnt] = oc.permute(1, 0, 2)
        lse32[:, lo:lo + cnt] = lc
    return out64, lse64, out32, lse32


def _combine32(o: torch.Tensor, lse: torch.Tensor, dim: int):
    """``decode_combine_kernel`` in fp32 over ``dim`` of partial ``o`` (..., P, D) and ``lse`` (..., P, 1): partials
    with lse = -inf skipped, lse = max + log(sum exp(lse_p - max)), out = sum exp(lse_p - lse) out_p."""
    skip = torch.isneginf(lse)
    mx = lse.amax(dim=dim, keepdim=True)
    ok = ~torch.isneginf(mx)
    mx0 = torch.where(ok, mx, torch.zeros_like(mx))
    tot = torch.where(skip, torch.zeros_like(lse), torch.exp(lse - mx0)).sum(dim=dim, keepdim=True)
    lc = torch.where(ok, mx + torch.log(tot), torch.full_like(mx, float("-inf")))
    w = torch.where(skip | ~ok, torch.zeros_like(lse), torch.exp(lse - torch.where(ok, lc, torch.zeros_like(lc))))
    return (w * o).sum(dim=dim), lc.squeeze(dim).squeeze(-1)


def combine_ranks64(parts):
    """fp64 merge of per-rank (out (rows, Hq, D), lse (Hq, rows)) results."""
    lse = torch.logsumexp(torch.stack([l for _, l in parts]), dim=0)
    safe = torch.where(torch.isinf(lse), torch.zeros_like(lse), lse)
    out = sum(o * torch.exp(l - safe).transpose(0, 1).unsqueeze(-1) for o, l in parts)
    return out, lse


def combine_ranks32(parts):
    """The rank combine as the kernel runs it: fp32 partials in rank order."""
    o = torch.stack([x for x, _ in parts], dim=2)  # (rows, Hq, P, D)
    l = torch.stack([y.transpose(0, 1) for _, y in parts], dim=2).unsqueeze(-1)  # (rows, Hq, P, 1)
    oc, lc = _combine32(o, l, dim=2)
    return oc, lc.transpose(0, 1)


# ----------------------------------------------------------------------------------------------
# the driver
# ----------------------------------------------------------------------------------------------

def report_key(dtype, d: int, fp8: bool, regime: str = "randn") -> str:
    key = f"decode {str(dtype).replace('torch.', '')} D{d} {'e4m3' if fp8 else 'native'}"
    return key + " (large)" if regime == "large" else key


def packed(case: Case, out: torch.Tensor, lse: torch.Tensor):
    """A uniform call's (B, Sq, Hq, D) / (B, Hq, Sq) results as (rows, Hq, D) / (Hq, rows)."""
    if case.varlen:
        return out, lse
    b, sq, hq, d = out.shape
    return out.reshape(b * sq, hq, d), lse.permute(1, 0, 2).reshape(hq, b * sq)


def call_kwargs(inp: Inputs) -> dict:
    case = inp.case
    kw = dict(block_table=inp.table, k_descale=inp.k_descale, v_descale=inp.v_descale)
    if case.varlen:
        kw.update(cu_seqlens_q=cu_of(case.counts, inp.q.device), max_seqlen_q=max(max(case.counts), 1))
    if inp.rotary is not None:
        cos, sin, rs, inter = inp.rotary
        kw.update(rotary_cos=cos, rotary_sin=sin, rotary_interleaved=inter,
                  rotary_seqlens=torch.tensor(rs, dtype=torch.int32, device=inp.q.device))
    return kw


def call_views(inp: Inputs, with_append: bool):
    """q, k, v as ``kernel_decode`` takes them: (B, Sq, H, D) for a uniform case, packed for varlen."""
    case = inp.case
    if case.varlen:
        q, k, v = inp.q, inp.k_new, inp.v_new
    else:
        q, k, v = (x.view(case.b, case.counts[0], *x.shape[1:]) for x in (inp.q, inp.k_new, inp.v_new))
    return (q, k, v) if with_append else (q, None, None)


def expected_caches(inp: Inputs, k0: torch.Tensor, v0: torch.Tensor, with_append: bool):
    if not with_append:
        return k0, v0
    case = inp.case
    return (appended(k0, inp.table, case.seqlens, inp.stored_k, case.counts),
            appended(v0, inp.table, case.seqlens, inp.stored_v, case.counts))


def sequence_blocks(case: Case):
    """``assert_accurate`` blocks of a uniform call's packed (rows, Hq, D) out: one per (sequence, kv head)."""
    assert not case.varlen
    return (case.counts[0], case.group, None)


def run_decode(case: Case, dtype, d: int, regime: str, device, seed: int = 0, draw="cpu", per_block: bool = False):
    """One case through ``kernel_decode`` against both references, then the cache bytes.  ``per_block`` (a uniform
    case): the bound also holds within every (sequence, kv head), the kernel's unit of work."""
    inp = build_inputs(case, dtype, d, regime, device, seed, draw=draw)
    n_splits = case.splits if case.splits is not None else default_splits(case, device)
    k0, v0 = inp.k_cache.clone(), inp.v_cache.clone()
    q, k, v = call_views(inp, case.append)
    # splits=None takes kernel_decode's own default on a GPU; a CPU run has no SM count to take it from
    splits = case.splits if torch.device(device).type == "cuda" else n_splits
    out, lse = dec.kernel_decode(q, inp.k_cache, inp.v_cache, inp.seqlens, k, v, case.causal, d ** -0.5,
                                 splits=splits, **call_kwargs(inp))
    o64, l64, o32, l32 = references(inp, n_splits)
    tag = f"decode {case.name}{' e4m3' if case.fp8 else ''} D{d} {str(dtype).replace('torch.', '')} {regime}"
    assert out.dtype == dtype and out.shape == q.shape, (tag, out.dtype, out.shape)
    got_o, got_l = packed(case, out, lse)
    KO.assert_accurate(f"{tag}: out", got_o, o64, o32.to(dtype), factor=KO._factor(regime),
                       report=report_key(dtype, d, case.fp8, regime),
                       blocks=sequence_blocks(case) if per_block else None)
    KO.assert_lse(f"{tag}: lse", got_l, l64, l32, report=f"decode lse {'e4m3' if case.fp8 else 'native'}")
    want_k, want_v = expected_caches(inp, k0, v0, case.append)
    for name, got, want in (("k_cache", inp.k_cache, want_k), ("v_cache", inp.v_cache, want_v)):
        diff = bytes_of(got) != bytes_of(want)
        assert not diff.any(), f"{tag}: {name} bytes differ at {diff.nonzero()[:4].tolist()}"


TWO_RANK_CASE = Case("two_ranks", (4, 4, 4), (700, 0, 300), 900, hq=16, hkv=2, splits=3)


def run_two_ranks(rank: int, world: int, fp8: bool, device_type: str):
    """A two-rank call (inside ``dist_utils.run_distributed``): rank 1 takes the append, each rank holds its own shard
    and descales.  The fp64 reference merges the per-shard fp64 results; the precision-matched one merges the per-rank
    fp32 partials in rank order, then rounds.  Both ranks must agree bitwise.  ``device_type="cpu"`` runs on
    ``tests/fake_ext.FakeDecodeExt``."""
    import torch.distributed as dist

    if device_type == "cpu":
        from fake_ext import FakeDecodeExt
        from ring_flash_attn_b200.ops import cuda_ext

        cuda_ext.load = FakeDecodeExt
    else:
        torch.backends.cuda.matmul.allow_tf32 = False
    case = dataclasses.replace(TWO_RANK_CASE, fp8=fp8)
    dtype, d, append_rank = torch.bfloat16, 128, 1
    dev = f"cuda:{rank}" if device_type == "cuda" else "cpu"
    shards = [build_inputs(case, dtype, d, "randn", dev, seed=3, cache_seed=10 + r) for r in range(world)]
    inp = shards[rank]
    q, k, v = call_views(inp, rank == append_rank)
    out, lse = dec.kernel_decode(q, inp.k_cache, inp.v_cache, inp.seqlens, k, v, case.causal, d ** -0.5,
                                 pg=dist.group.WORLD, world=world, splits=case.splits, **call_kwargs(inp))
    refs = [references(s, case.splits, appended_here=r == append_rank) for r, s in enumerate(shards)]
    o64, l64 = combine_ranks64([(a, b) for a, b, _, _ in refs])
    o32, l32 = combine_ranks32([(c, e) for _, _, c, e in refs])
    got_o, got_l = packed(case, out, lse)
    tag = f"decode two ranks {'e4m3' if fp8 else 'native'}"
    KO.assert_accurate(f"{tag}: out", got_o, o64, o32.to(dtype), report=f"{report_key(dtype, d, fp8)} two ranks")
    KO.assert_lse(f"{tag}: lse", got_l, l64, l32)
    both = torch.cat([out.float().reshape(-1), lse.reshape(-1)])
    got = [torch.empty_like(both) for _ in range(world)]
    dist.all_gather(got, both)
    for x in got:
        assert torch.equal(x.nan_to_num(7.0), both.nan_to_num(7.0)), "the ranks' results differ"
