"""cp_flash_attn_with_kvcache with paged shared prefixes (``prefix_block_table``), on CPU / gloo: bitwise the
contiguous prefix call on the same rows for pages of 16 to 256 rows in a seeded random page order with -1 past the
visible pages (uniform and varlen, causal and not, e4m3 caches, rotary, tree masks, cache slots and left pads on a
contiguous suffix, P in {1, 2, 6}), one pool shared by prefix and paged suffix, every guard, the dense range checks,
world-2/4 groups with a pool and table per rank, the arguments reaching the extension, torch.compile over the one-pool
layout and a dry run of the benchmark."""
import dataclasses
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist

import decode_cache_idx as CI
import decode_oracle as DO
import decode_prefix as DP
import decode_prefix_paged as PP
import decode_tree as DT
import ring_flash_attn_b200 as rfa
from dist_utils import run_distributed
from ring_flash_attn_b200.parallel import decode as dec
from test_decode_varlen import appended
from test_gpu_decode_fp8 import bytes_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = 64
P_CAP = 512  # a multiple of every page size tested
PAGE_SIZES = [16, 32, 64, 128, 256]
f = rfa.cp_flash_attn_with_kvcache

# (case, P): B = P * n
FEATURES = {
    "causal": (DO.Case("u6", (2,) * 6, (300, 0, 17, 128, 5, 250), 320), 2),
    "noncausal": (DO.Case("u6nc", (3,) * 6, (100, 31, 0, 129, 300, 2), 320, causal=False), 2),
    "varlen": (DO.Case("v6", (3, 0, 1, 5, 2, 1), (250, 9, 0, 200, 0, 33), 300, varlen=True), 2),
    "e4m3_cache": (DO.Case("u6f8", (2,) * 6, (200, 0, 60, 129, 7, 280), 300, fp8=True), 2),
    "rotary": (DO.Case("u6rot", (2,) * 6, (200, 0, 60, 129, 7, 280), 300, rotary=(16, True)), 2),
    "rotary_varlen": (DO.Case("v6rot", (3, 0, 1, 5, 2, 1), (250, 9, 0, 200, 0, 33), 300, varlen=True,
                              rotary=("full", True), causal=False), 2),
    "tree_rotary": (DO.Case("u6tree", (5,) * 6, (200, 0, 60, 129, 7, 280), 300, rotary=("half", False)), 2),
    "tree_varlen": (DO.Case("v6tree", (3, 0, 1, 5, 2, 4), (250, 9, 0, 200, 0, 33), 300, varlen=True), 2),
    "one_prefix": (DO.Case("u6p1", (1,) * 6, (30, 0, 17, 200, 5, 250), 300, hq=16), 1),
    "n1": (DO.Case("u6n1", (2,) * 6, (30, 0, 17, 200, 5, 250), 300, hq=4, hkv=1), 6),
}
MODES = (None, "slots", "leftpad", "both")


def _plens(n_prefix, rank=0):
    """Prefix lengths of a rank's shard: P_cap and 0 on rank 0."""
    pool = [P_CAP, 0, 271, 129, 1, 390, 257, 333]
    return [pool[(3 * rank + i) % len(pool)] for i in range(n_prefix)]


def _inputs(feature, mode=None, append=True, seed=3, cache_seed=10, prefix_seed=7, rank=0, device="cpu"):
    """(SlotInputs of the contiguous suffix, contiguous Prefix, tree mask or None)."""
    case, n_prefix = FEATURES[feature]
    if not append:
        case = dataclasses.replace(case, append=False)
    b = case.b
    idx = CI.slot_indices(b, 2 * b + 3, seed=100 + cache_seed) if mode in ("slots", "both") else None
    pads = CI.leftpads(case, seed=200 + cache_seed) if mode in ("leftpad", "both") else None
    si = CI.build(case, torch.bfloat16, D, device, idx=idx, n_slots=2 * b + 3, pads=pads, seed=seed,
                  cache_seed=cache_seed)
    pre = DP.make_prefix(case, torch.bfloat16, D, device, _plens(n_prefix, rank), P_CAP, seed=prefix_seed)
    mask = None
    if feature.startswith("tree"):
        gen = torch.Generator().manual_seed(seed)
        sq = max(max(case.counts), 1)
        mask = DT.packed_mask(DT.tree_masks(case.counts, gen), sq, gen, case.varlen).to(device)
    return si, pre, mask


def _public(si, prefix_kwargs, mask, append_rank=0, group=None, with_append=True):
    q, k, v, kw = CI.call_args(si, with_append)
    kw.update(prefix_kwargs)
    if mask is not None:
        kw["tree_mask"] = mask
    return f(q, si.k_pool, si.v_pool, si.seqlens, k, v, append_rank=append_rank if with_append else None,
             causal=si.plain.case.causal, return_softmax_lse=True, group=group, **kw)


@pytest.mark.parametrize("page_size", PAGE_SIZES)
@pytest.mark.parametrize("feature", list(FEATURES))
def test_paged_equals_contiguous_prefix(feature, page_size):
    """Bitwise: the paged prefix is the contiguous prefix on the same rows; the suffix's appended bytes match too."""
    mode = MODES[(list(FEATURES).index(feature) + PAGE_SIZES.index(page_size)) % len(MODES)]
    si, pre, mask = _inputs(feature, mode)
    si2, _, _ = _inputs(feature, mode)
    pp = PP.page(pre, page_size, seed=page_size)
    assert (pp.table == -1).any() or feature == "one_prefix"  # tables are padded past the visible pages
    out, lse = _public(si, pp.kwargs(), mask)
    ref_out, ref_lse = _public(si2, pre.kwargs(), mask)
    tag = f"{feature} {mode} pages of {page_size}"
    assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse), tag
    assert torch.equal(bytes_of(si.k_pool), bytes_of(si2.k_pool)), tag
    assert torch.equal(bytes_of(si.v_pool), bytes_of(si2.v_pool)), tag
    fresh = PP.page(DP.make_prefix(si.plain.case, torch.bfloat16, D, "cpu", pre.lens, P_CAP), page_size,
                    seed=page_size)
    assert torch.equal(bytes_of(pp.k), bytes_of(fresh.k)) and torch.equal(bytes_of(pp.v), bytes_of(fresh.v)), tag


def _one_pool(page_size, fp8=False, varlen=False, seed=0):
    """A paged suffix (S_cap 512) and a paged prefix in one pool: (inp, pre, k_pool, v_pool, table, prefix_table)."""
    if varlen:
        case = DO.Case("v6pool", (3, 0, 1, 5, 2, 4), (250, 9, 0, 200, 0, 33), 512, varlen=True, layout="paged",
                       page_size=page_size, fp8=fp8)
    else:
        case = DO.Case("u6pool", (2,) * 6, (300, 0, 17, 128, 5, 250), 512, layout="paged", page_size=page_size,
                       fp8=fp8)
    inp = DO.build_inputs(case, torch.bfloat16, D, "randn", "cpu", seed)
    pre = DP.make_prefix(case, torch.bfloat16, D, "cpu", _plens(2, seed), P_CAP, seed=seed + 7)
    pp = PP.page(pre, page_size, seed=seed + 1)
    k, v, table, ptable = PP.share_pool(inp.k_cache, inp.v_cache, inp.table, pp, seed=seed + 2)
    return inp, pre, k, v, table, ptable


@pytest.mark.parametrize("page_size", PAGE_SIZES)
def test_one_pool_shared_by_prefix_and_paged_suffix(page_size):
    """prefix_k_cache / prefix_v_cache are the very tensors k_cache / v_cache: bitwise the call with a contiguous
    prefix and a pool of the suffix's own; the appended rows land in the suffix's pages, the prompt pages stay."""
    for fp8, varlen in ((False, False), (True, False), (False, True)):
        inp, pre, k, v, table, ptable = _one_pool(page_size, fp8, varlen)
        q, kn, vn = DO.call_views(inp, True)
        kw = DO.call_kwargs(inp)
        kw.pop("block_table")
        pages = PP.prompt_pages(ptable)
        before_k, before_v = bytes_of(k[pages]).clone(), bytes_of(v[pages]).clone()
        k0, v0 = k.clone(), v.clone()
        out, lse = f(q, k, v, inp.seqlens, kn, vn, append_rank=0, return_softmax_lse=True, block_table=table,
                     prefix_k_cache=k, prefix_v_cache=v, prefix_block_table=ptable, prefix_seqlens=pre.seqlens,
                     prefix_k_descale=pre.k_descale, prefix_v_descale=pre.v_descale, **kw)
        sk, sv = inp.k_cache.clone(), inp.v_cache.clone()
        ref_out, ref_lse = f(q, sk, sv, inp.seqlens, kn, vn, append_rank=0, return_softmax_lse=True,
                             block_table=inp.table, **pre.kwargs(), **kw)
        tag = f"pages of {page_size} fp8={fp8} varlen={varlen}"
        assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse), tag
        assert torch.equal(bytes_of(k[pages]), before_k) and torch.equal(bytes_of(v[pages]), before_v), tag
        want_k = appended(k0, table, inp.case.seqlens, inp.stored_k, inp.case.counts)
        want_v = appended(v0, table, inp.case.seqlens, inp.stored_v, inp.case.counts)
        assert torch.equal(bytes_of(k), bytes_of(want_k)) and torch.equal(bytes_of(v), bytes_of(want_v)), tag


def test_guards():
    si, pre, _ = _inputs("causal")
    q, k, v, kw = CI.call_args(si, True)
    kc, vc, sl = si.k_pool, si.v_pool, si.seqlens
    pp = PP.page(pre, 32)
    good = pp.kwargs()
    f(q, kc, vc, sl, **good)  # the good call passes
    for drop in ("prefix_k_cache", "prefix_v_cache", "prefix_seqlens"):
        bad = dict(good)
        del bad[drop]
        with pytest.raises(ValueError, match="together"):
            f(q, kc, vc, sl, **bad)
    with pytest.raises(ValueError, match="together"):
        f(q, kc, vc, sl, prefix_block_table=pp.table)
    t = pp.table
    wide = torch.cat([t, t], dim=1)
    for bad, msg in (
            (t.long(), "prefix_block_table must be a \\(P, max_prefix_blocks\\) int32"),
            (t[0], "prefix_block_table must be a \\(P, max_prefix_blocks\\) int32"),
            (t[:0], "prefix_block_table must be a \\(P, max_prefix_blocks\\) int32"),
            (t[:, :0], "prefix_block_table must be a \\(P, max_prefix_blocks\\) int32"),
            (wide[:, ::2], "prefix_block_table must be a \\(P, max_prefix_blocks\\) int32"),  # stride(1) == 2
            ([[0, 1]], "prefix_block_table must be a \\(P, max_prefix_blocks\\) int32"),
            (t.to("meta"), "prefix_block_table must be on q's device"),
            (torch.zeros(4, t.shape[1], dtype=torch.int32), "multiple of the prefix count"),  # B = 6, P = 4
    ):
        with pytest.raises(ValueError, match=msg):
            f(q, kc, vc, sl, **dict(good, prefix_block_table=bad, prefix_seqlens=pre.seqlens[:1].repeat(
                bad.shape[0] if isinstance(bad, torch.Tensor) and bad.dim() == 2 else 2)))
    # the pool: page size, mergeable strides, dtype, device, shape, k / v strides, size
    n_pages = pp.k.shape[0]
    odd = torch.zeros(n_pages, 48, 2, D, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="page_size 48 is not supported"):
        f(q, kc, vc, sl, **dict(good, prefix_k_cache=odd, prefix_v_cache=odd))
    strided = torch.zeros(n_pages, 40, 2, D, dtype=torch.bfloat16)[:, :32]  # stride(0) != 32 * stride(1)
    with pytest.raises(ValueError, match="mergeable"):
        f(q, kc, vc, sl, **dict(good, prefix_k_cache=strided, prefix_v_cache=strided))
    with pytest.raises(ValueError, match="cache's dtype"):
        f(q, kc, vc, sl, **dict(good, prefix_k_cache=pp.k.half()))
    with pytest.raises(ValueError, match="on q's device"):
        f(q, kc, vc, sl, **dict(good, prefix_k_cache=pp.k.to("meta"), prefix_v_cache=pp.v.to("meta")))
    with pytest.raises(ValueError, match="must both be"):
        f(q, kc, vc, sl, **dict(good, prefix_v_cache=pp.v[:1]))
    with pytest.raises(ValueError, match="page pool"):
        f(q, kc, vc, sl, **dict(good, prefix_k_cache=pp.k[0]))
    kv = torch.zeros(n_pages, 32, 2, 2, D, dtype=torch.bfloat16)  # k and v interleaved per head: other strides
    with pytest.raises(ValueError, match="same strides"):
        f(q, kc, vc, sl, **dict(good, prefix_k_cache=kv[:, :, :, 0], prefix_v_cache=pp.v))
    huge = torch.empty((2 ** 22, 2 ** 9, 2, D), dtype=torch.bfloat16, device="meta")
    with pytest.raises(ValueError, match="num_blocks \\* page_size and max_prefix_blocks \\* page_size"):
        f(q.to("meta"), kc.to("meta"), vc.to("meta"), sl.to("meta"), prefix_k_cache=huge, prefix_v_cache=huge,
          prefix_block_table=pp.table.to("meta"), prefix_seqlens=pre.seqlens.to("meta"))
    # e4m3 pools: the descales are still (), (Hkv,) or (P, Hkv); an e4m3 q is still left out
    si8, pre8, _ = _inputs("e4m3_cache")
    q8, _, _, kw8 = CI.call_args(si8, False)
    base = dict(k_descale=kw8["k_descale"], v_descale=kw8["v_descale"])
    pp8 = PP.page(pre8, 64)
    f(q8, si8.k_pool, si8.v_pool, si8.seqlens, **base, **pp8.kwargs())
    with pytest.raises(ValueError, match="shape"):
        f(q8, si8.k_pool, si8.v_pool, si8.seqlens, **base, **dict(pp8.kwargs(), prefix_k_descale=torch.ones(3)))
    with pytest.raises(ValueError, match="bf16 / fp16 q"):
        f(q8.to(torch.float8_e4m3fn), si8.k_pool, si8.v_pool, si8.seqlens, **base, q_descale=torch.ones(()),
          **pp8.kwargs())


def test_dense_range_checks():
    """The dense path raises for a table entry outside the pool on a page it reads and for prefix_seqlens past
    P_cap, before anything is appended; -1 and out-of-pool entries past the visible pages are never read."""
    si, pre, _ = _inputs("causal")
    q, k, v, kw = CI.call_args(si, True)
    pp = PP.page(pre, 64)
    n_pages = pp.k.shape[0]
    bad = pp.table.clone()
    bad[0, 0] = n_pages
    with pytest.raises(ValueError, match="prefix_block_table\\[0\\] points outside the"):
        f(q, si.k_pool, si.v_pool, si.seqlens, k, v, append_rank=0, **kw, **dict(pp.kwargs(), prefix_block_table=bad))
    for x in (-1, P_CAP + 1):
        pl = pre.seqlens.clone()
        pl[1] = x
        with pytest.raises(ValueError, match=f"prefix_seqlens\\[1\\] = {x} is outside"):
            f(q, si.k_pool, si.v_pool, si.seqlens, k, v, append_rank=0, **kw,
              **dict(pp.kwargs(), prefix_seqlens=pl))
    fresh, _, _ = _inputs("causal")
    assert torch.equal(bytes_of(si.k_pool), bytes_of(fresh.k_pool))  # nothing appended by the refused calls
    # entries past the visible pages may hold anything
    junk = pp.table.clone()
    junk[junk < 0] = 10 ** 6
    si2, _, _ = _inputs("causal")
    out, lse = f(q, si.k_pool, si.v_pool, si.seqlens, k, v, append_rank=0, return_softmax_lse=True, **kw,
                 **dict(pp.kwargs(), prefix_block_table=junk))
    ref_out, ref_lse = f(q, si2.k_pool, si2.v_pool, si2.seqlens, k, v, append_rank=0, return_softmax_lse=True, **kw,
                         **pre.kwargs())
    assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse)


def _run_ranks(rank, world, scenarios):
    """Each rank holds its own suffix shard and its own prefix pool and table: bitwise the contiguous prefix call on
    the same shards, and bitwise equal on every rank."""
    torch.set_num_threads(1)
    for feature, mode, page_size in scenarios:
        append_rank = world - 1
        kw = dict(cache_seed=10 + rank, prefix_seed=20 + rank, rank=rank)
        si, pre, mask = _inputs(feature, mode, **kw)
        si2, _, _ = _inputs(feature, mode, **kw)
        pp = PP.page(pre, page_size, seed=30 + rank, spare=1 + 2 * rank)
        out, lse = _public(si, pp.kwargs(), mask, append_rank, dist.group.WORLD)
        ref_out, ref_lse = _public(si2, pre.kwargs(), mask, append_rank, dist.group.WORLD)
        tag = f"{feature} {mode} pages of {page_size} world {world} rank {rank}"
        assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse), tag
        assert torch.equal(bytes_of(si.k_pool), bytes_of(si2.k_pool)), tag
        both = torch.cat([out.float().reshape(-1), lse.reshape(-1)])
        got = [torch.empty_like(both) for _ in range(world)]
        dist.all_gather(got, both)
        for x in got:
            assert torch.equal(x.nan_to_num(7.0), both.nan_to_num(7.0)), f"{tag}: the ranks' results differ"


@pytest.mark.parametrize("world", [2, 4])
def test_ranks_with_their_own_pools(world):
    scenarios = [("causal", "both", 16), ("varlen", None, 128), ("e4m3_cache", "slots", 32),
                 ("rotary", None, 256), ("noncausal", "leftpad", 64), ("tree_rotary", None, 16)]
    run_distributed(_run_ranks, world, scenarios)


class _Recorder:
    """Stands in for the extension and records what kernel_decode passes to it."""

    def __init__(self):
        self.prefix = self.parts = None

    def decode_fwd(self, *args):
        pass

    def decode_prefix_fwd(self, *args):
        self.prefix = args

    def decode_combine(self, parts, out, lse):
        self.parts = parts
        out.zero_()
        lse.zero_()


def test_kernel_decode_passes_the_table(monkeypatch):
    from ring_flash_attn_b200.ops import cuda_ext

    rec = _Recorder()
    monkeypatch.setattr(cuda_ext, "load", lambda: rec)
    monkeypatch.setattr(dec, "_sm_count", lambda index: 132)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)  # q is on the CPU here
    si, pre, _ = _inputs("causal")
    q, k, v, kw = CI.call_args(si, True)
    pp = PP.page(pre, 16)
    dec.kernel_decode(q, si.k_pool, si.v_pool, si.seqlens, k, v, True, 0.1, splits=2, **kw, **pp.kwargs())
    args = rec.prefix
    assert len(args) == 17 and args[1] is pp.k and args[2] is pp.v and args[15] is None and args[16] is pp.table
    # the default prefix split count: from P = the table's rows and P_cap = max_prefix_blocks * page_size
    slots = dec.prefix_tile_slots(3, 2, 8, 2)
    assert rec.parts.shape[0] == 2 + dec.num_splits_prefix(2, slots, 2, P_CAP, 132)
    # a contiguous prefix keeps the form it had
    dec.kernel_decode(q, si.k_pool, si.v_pool, si.seqlens, k, v, True, 0.1, splits=2, **kw, **pre.kwargs())
    assert len(rec.prefix) == 15


def test_torch_compile_fullgraph_one_pool():
    """The one-pool layout under torch.compile: prefix_k_cache aliases the mutated k_cache, and the compiled call
    gives the eager result and the same pool."""
    inp, pre, k, v, table, ptable = _one_pool(16)
    q, kn, vn = DO.call_views(inp, True)

    def fn(q, kc, vc, sl, kn, vn, bt, pbt, pl):
        out, lse = f(q, kc, vc, sl, kn, vn, append_rank=0, return_softmax_lse=True, block_table=bt,
                     prefix_k_cache=kc, prefix_v_cache=vc, prefix_block_table=pbt, prefix_seqlens=pl)
        return out * 1.0, lse

    k2, v2 = k.clone(), v.clone()
    args = (inp.seqlens, kn, vn, table, ptable, pre.seqlens)
    out, lse = torch.compile(fn, backend="aot_eager", fullgraph=True)(q, k, v, *args)
    ref_out, ref_lse = fn(q, k2, v2, *args)
    assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse)
    assert torch.equal(bytes_of(k), bytes_of(k2)) and torch.equal(bytes_of(v), bytes_of(v2))


def test_bench_decode_dry_run_paged_prefix():
    cmd = [sys.executable, os.path.join(ROOT, "benchmark", "bench_decode.py"), "--dry-run", "--shared-prefix",
           "32768", "--samples", "4", "--prefix-page", "16"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:]
    rows = [json.loads(line) for line in r.stdout.splitlines() if line.startswith("{")]
    assert rows
    for x in rows:
        assert x["page_size"] == 16
        assert x["paged_prefix_bytes"] == x["prefix_bytes"] < x["paged_bytes"]
