"""cp_flash_attn_with_kvcache over paged caches (``block_table=``) on CPU / gloo (worlds 1-4) against the fp64
oracle over the gathered logical cache."""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist

import ring_flash_attn_b200 as rfa
from dist_utils import run_distributed
from test_decode import TOL, decode_oracle, make_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAGE_SIZES = (16, 128, 256)


def to_pool(kc, vc, lens, page_size, alloc=None, spare=3, seed=0):
    """A page pool and block table holding the contiguous cache ``kc`` / ``vc`` (B, S_cap, Hkv, D), with S_cap a
    multiple of ``page_size``.  Sequence b owns the pages of rows [0, alloc[b]) (default: lens[b]), drawn in a seeded
    random order from a pool with ``spare`` extra pages; its later table entries are -1.  Pool rows at or past
    lens[b], and the spare pages, are NaN.  Returns (k_pool, v_pool, block_table) on kc's device."""
    b, s_cap, hkv, d = kc.shape
    assert s_cap % page_size == 0
    alloc = lens if alloc is None else alloc
    n_pages = [-(-int(a) // page_size) for a in alloc]
    total = sum(n_pages) + spare
    perm = torch.randperm(total, generator=torch.Generator().manual_seed(seed)).tolist()
    pk = torch.full((total, page_size, hkv, d), float("nan"), dtype=kc.dtype, device=kc.device)
    pv = torch.full_like(pk, float("nan"))
    table = torch.full((b, s_cap // page_size), -1, dtype=torch.int32)
    nxt = 0
    for i in range(b):
        n = int(lens[i])
        for j in range(n_pages[i]):
            page = perm[nxt]
            nxt += 1
            table[i, j] = page
            lo, hi = j * page_size, min((j + 1) * page_size, n)
            if hi > lo:
                pk[page, :hi - lo] = kc[i, lo:hi]
                pv[page, :hi - lo] = vc[i, lo:hi]
    return pk, pv, table.to(kc.device)


def append_to_pool(pool, table, lens, new):
    """``pool`` after appending ``new`` (B, Sq, Hkv, D) at logical rows [lens[b], lens[b] + Sq) through ``table``."""
    want = pool.clone()
    ps = pool.shape[1]
    for i in range(new.shape[0]):
        for t in range(new.shape[1]):
            row = int(lens[i]) + t
            if row < table.shape[1] * ps:
                want[int(table[i, row // ps]), row % ps] = new[i, t]
    return want


def paged_case(world, sq, grp, page_size, seed, b=3, hkv=2, d=16, max_blocks=None):
    """make_case with S_cap = max_blocks * page_size, plus one sequence per rank holding page_size - 1 rows, so that
    an append of Sq > 1 rows crosses a page boundary."""
    if max_blocks is None:
        max_blocks = max(2, -(-48 // page_size))
    caches, lens, q, k, v = make_case(world, b, sq, hkv * grp, hkv, d, max_blocks * page_size, seed)
    for r in range(world):
        i = (r + seed + 1) % b
        lens[r][i] = page_size - 1
        for c in caches[r]:
            c[i, :page_size - 1].nan_to_num_(0.5)
    return caches, lens, q, k, v


CASES = [(sq, grp, causal, append) for sq in (1, 4) for grp in (1, 4, 8) for causal in (True, False)
         for append in (True, False)]


def _run_paged(rank, world, page_sizes, cases):
    for ps in page_sizes:
        for n, (sq, grp, causal, append) in enumerate(cases):
            seed = 1000 * world + 10 * ps + n
            caches, lens, q, k, v = paged_case(world, sq, grp, ps, seed)
            ar = (n % world) if append else None
            kc, vc = caches[rank]
            s_cap = kc.shape[1]
            alloc = (lens[rank] + sq).clamp(max=s_cap)
            pk, pv, table = to_pool(kc, vc, lens[rank], ps, alloc=alloc, seed=seed + rank)
            pk0, pv0 = pk.clone(), pv.clone()
            out, lse = rfa.cp_flash_attn_with_kvcache(q, pk, pv, lens[rank], k if append else None,
                                                      v if append else None, append_rank=ar, causal=causal,
                                                      return_softmax_lse=True, block_table=table)
            ref_out, ref_lse = decode_oracle(q, caches, lens, k if append else None, v if append else None, causal)
            torch.testing.assert_close(out, ref_out, **TOL)
            torch.testing.assert_close(lse, ref_lse, **TOL)
            # the pools: k / v at logical rows [len, len + Sq) of the append rank, every other row untouched
            want_k, want_v = pk0, pv0
            if append and rank == ar:
                want_k, want_v = append_to_pool(pk0, table, lens[rank], k), append_to_pool(pv0, table, lens[rank], v)
            assert torch.equal(pk.nan_to_num(7.0), want_k.nan_to_num(7.0))
            assert torch.equal(pv.nan_to_num(7.0), want_v.nan_to_num(7.0))
            if world == 1:  # the same logical cache, contiguous: bitwise the same result
                c_out, c_lse = rfa.cp_flash_attn_with_kvcache(q, kc.clone(), vc.clone(), lens[rank],
                                                              k if append else None, v if append else None,
                                                              append_rank=ar, causal=causal, return_softmax_lse=True)
                assert torch.equal(out, c_out) and torch.equal(lse, c_lse)
            if world > 1:  # bitwise the same on every rank
                both = torch.cat([out.reshape(-1), lse.reshape(-1)])
                got = [torch.empty_like(both) for _ in range(world)]
                dist.all_gather(got, both)
                for x in got:
                    assert torch.equal(x.nan_to_num(7.0), both.nan_to_num(7.0))


@pytest.mark.parametrize("page_size", PAGE_SIZES)
def test_paged_world1_matches_oracle(page_size):
    _run_paged(0, 1, (page_size,), CASES)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_paged_gloo_worlds_match_oracle(world):
    run_distributed(_run_paged, world, PAGE_SIZES, CASES)


def test_append_across_a_page_boundary():
    ps, sq = 16, 4
    caches, lens, q, k, v = paged_case(1, sq, 4, ps, seed=7, b=1)  # the one sequence holds ps - 1 rows
    assert int(lens[0][0]) == ps - 1
    kc, vc = caches[0]
    pk, pv, table = to_pool(kc, vc, lens[0], ps, alloc=lens[0] + sq, seed=7)
    pk0 = pk.clone()
    out = rfa.cp_flash_attn_with_kvcache(q, pk, pv, lens[0], k, v, append_rank=0, block_table=table)
    ref, _ = decode_oracle(q, caches, lens, k, v, True)
    torch.testing.assert_close(out, ref, **TOL)
    p0, p1 = int(table[0, 0]), int(table[0, 1])
    assert torch.equal(pk[p0, ps - 1], k[0, 0]) and torch.equal(pk[p1, :sq - 1], k[0, 1:])
    changed = (pk.nan_to_num(7.0) != pk0.nan_to_num(7.0)).any(-1).any(-1)  # (pages, rows)
    assert sorted(changed.nonzero().tolist()) == sorted([[p0, ps - 1]] + [[p1, r] for r in range(sq - 1)])


def test_block_table_guards():
    caches, lens, q, k, v = paged_case(1, 1, 2, 16, seed=0, b=2)
    kc, vc = caches[0]
    sl = lens[0]
    pk, pv, table = to_pool(kc, vc, sl, 16, alloc=sl + 1)
    f = rfa.cp_flash_attn_with_kvcache
    with pytest.raises(ValueError, match="int32"):
        f(q, pk, pv, sl, block_table=table.long())
    with pytest.raises(ValueError, match="max_blocks"):
        f(q, pk, pv, sl, block_table=table[:1])  # one row for two sequences
    with pytest.raises(ValueError, match="max_blocks"):
        f(q, pk, pv, sl, block_table=table[:, 0])
    with pytest.raises(ValueError, match="stride"):
        f(q, pk, pv, sl, block_table=table.t().contiguous().t())
    with pytest.raises(ValueError, match="q's device"):
        f(q, pk, pv, sl, block_table=table.to("meta"))
    for ps in (8, 24, 48, 96, 192):
        bad = torch.zeros(4, ps, *pk.shape[2:])
        with pytest.raises(ValueError, match=f"page_size {ps} is not supported"):
            f(q, bad, bad, sl, block_table=table)
    with pytest.raises(ValueError, match="mergeable"):
        wide = torch.zeros(pk.shape[0], 32, *pk.shape[2:])
        f(q, wide[:, :16], wide[:, :16], sl, block_table=table)
    with pytest.raises(ValueError, match="same"):  # pools of different shapes
        f(q, pk, pv[:-1], sl, block_table=table)
    with pytest.raises(ValueError, match="does not match"):  # pool head size differs from q's
        f(q, pk[..., :8], pv[..., :8], sl, block_table=table)


def test_torch_compile_fullgraph_paged():
    caches, lens, q, k, v = paged_case(1, 4, 4, 16, seed=1, b=2)
    kc, vc = caches[0]
    pk, pv, table = to_pool(kc, vc, lens[0], 16, alloc=lens[0] + 4)
    pk2, pv2 = pk.clone(), pv.clone()

    def f(q, pk, pv, sl, k, v, bt):
        out, lse = rfa.cp_flash_attn_with_kvcache(q, pk, pv, sl, k, v, append_rank=0, return_softmax_lse=True,
                                                  block_table=bt)
        return out * 1.0, lse

    out, lse = torch.compile(f, backend="aot_eager", fullgraph=True)(q, pk, pv, lens[0], k, v, table)
    ref_out, ref_lse = f(q, pk2, pv2, lens[0], k, v, table)
    torch.testing.assert_close(out, ref_out, **TOL)
    torch.testing.assert_close(lse, ref_lse, **TOL)
    assert torch.equal(pk.nan_to_num(7.0), pk2.nan_to_num(7.0))  # the compiled call appended too


def test_bench_decode_dry_run_paged():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "benchmark", "bench_decode.py"), "--dry-run",
                        "--page-size", "16", "--batch", "1", "8", "--cache", "32768"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:]
    rows = [json.loads(line) for line in r.stdout.splitlines() if line.startswith("{")]
    assert [(x["batch"], x["page_size"]) for x in rows] == [(1, 16), (8, 16)]
    assert rows[1]["block_table_bytes"] == 8 * (32768 // 16) * 4
