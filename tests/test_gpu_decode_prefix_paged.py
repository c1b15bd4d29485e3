"""The sm_90a split-KV decode kernel with paged shared prefixes (``prefix_block_table``): every prefix instantiation
(bf16 / fp16 x D 64 / 128 x native / e4m3 cache, with and without tree mask + rotary) against the fp64 oracle with
``kernel_oracle``'s precision-matched bound, at pages of 16, 64, 128 and 256 rows, split counts (1, 1), (3, 5) and the
default, on prefix tiles that pack sequences across a 64-row boundary; out / lse bitwise the contiguous prefix call on
the same rows at equal P_cap and split counts; one pool shared by prefix and paged suffix (prompt pages unchanged,
appended rows in the suffix pages); CUDA-graph replay with a new table and new prefix lengths; and per-rank pools and
tables on two GPUs."""
import dataclasses

import pytest
import torch
import torch.distributed as dist

import decode_oracle as DO
import decode_prefix as DP
import decode_prefix_paged as PP
import decode_tree as DT
import kernel_oracle as KO
from dist_utils import run_distributed
from ring_flash_attn_b200.parallel import decode as dec
from test_decode_varlen import appended
from test_gpu_decode_fp8 import bytes_of

pytestmark = pytest.mark.gpu

# B = P * n.  "rows80": n * Sq * G = 5 * 4 * 4 = 80 packed rows per prompt, so the second 64-row tile starts inside
# sequence 3 of each group
CASES = {
    "rows80": (DO.Case("rows80", (4,) * 10, (300, 0, 17, 128, 5, 250, 1, 129, 64, 200), 320, hq=8, hkv=2), 2),
    "varlen": (DO.Case("v9", (3, 0, 20, 5, 2, 1, 7, 0, 4), (250, 9, 0, 200, 0, 33, 1, 2, 300), 320, varlen=True,
                       hq=8, hkv=2), 3),
    "noncausal": (DO.Case("nc", (3,) * 6, (100, 31, 0, 129, 300, 2), 320, hq=8, hkv=2, causal=False), 3),
}
# with a tree mask (kTree instantiations: mask + rotary): causal cases with rotary
TREE_ROTARY = {"rows80": ("half", False), "varlen": ("full", True)}
P_CAP = 1536  # a multiple of every page size
PLENS = [P_CAP, 0, 1201, 129]
PAGE_SIZES = (16, 64, 128, 256)
SPLITS = ((1, 1), (3, 5), (None, None))
KINDS = [(torch.bfloat16, "native"), (torch.float16, "native"), (torch.bfloat16, "e4m3"), (torch.float16, "e4m3")]


@pytest.fixture(autouse=True)
def _exact_fp32_matmul():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


def _build(name, dtype, d, kind, tree, seed=0):
    case, n_prefix = CASES[name]
    case = dataclasses.replace(case, fp8=kind == "e4m3", rotary=TREE_ROTARY[name] if tree else None)
    inp = DO.build_inputs(case, dtype, d, "randn", "cuda", seed)
    pre = DP.make_prefix(case, dtype, d, "cuda", PLENS[:n_prefix], P_CAP, seed=seed + 7)
    return inp, pre


def _mask(case, tril, seed=0):
    gen = torch.Generator().manual_seed(seed)
    per = DT.tril_masks(case.counts) if tril else DT.tree_masks(case.counts, gen)
    return DT.packed_mask(per, max(max(case.counts), 1), gen, case.varlen).cuda()


def _default_prefix_splits(case, n_prefix):
    slots = dec.prefix_tile_slots(case.b // n_prefix, max(case.counts), case.hq, case.hkv,
                                  sum(case.counts) if case.varlen else None)
    return dec.num_splits_prefix(n_prefix, slots, case.hkv, P_CAP, dec._sm_count(torch.cuda.current_device()))


def _call(inp, prefix_kwargs, splits, prefix_splits, mask=None):
    """(out, lse, k_cache, v_cache) of kernel_decode with an append into fresh copies of the suffix caches."""
    q, k, v = DO.call_views(inp, True)
    kc, vc = inp.k_cache.clone(), inp.v_cache.clone()
    out, lse = dec.kernel_decode(q, kc, vc, inp.seqlens, k, v, inp.case.causal, inp.d ** -0.5, splits=splits,
                                 prefix_splits=prefix_splits, tree_mask=mask, **DO.call_kwargs(inp),
                                 **prefix_kwargs)
    return out, lse, kc, vc


@pytest.mark.parametrize("tree", [False, True], ids=["plain", "tree_rotary"])
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("dtype, kind", KINDS, ids=[f"{str(t)[6:]}-{k}" for t, k in KINDS])
def test_oracle_and_bitwise_contiguous(dtype, kind, d, tree):
    """A lower-triangular mask with rotary runs the kTree instantiation with exactly the causal call's positions, so
    the oracle of the causal rotary call holds it; random trees are held bitwise to the contiguous prefix call."""
    names = list(TREE_ROTARY) if tree else list(CASES)
    for i, name in enumerate(names):
        inp, pre = _build(name, dtype, d, kind, tree, seed=i)
        case = inp.case
        mask = _mask(case, tril=True) if tree else None
        for splits, prefix_splits in SPLITS:
            n_s = splits if splits is not None else DO.default_splits(case, "cuda")
            n_p = prefix_splits if prefix_splits is not None else _default_prefix_splits(case, pre.n)
            o64, l64, o32, l32 = DP.references(inp, pre, n_s, n_p)
            ref_out, ref_lse, _, _ = _call(inp, pre.kwargs(), splits, prefix_splits, mask)
            for ps in PAGE_SIZES:
                pp = PP.page(pre, ps, seed=ps + i)
                pool_k, pool_v = pp.k.clone(), pp.v.clone()
                out, lse, kc, vc = _call(inp, pp.kwargs(), splits, prefix_splits, mask)
                tag = f"{name} {kind} {dtype} D{d} tree={tree} pages of {ps} splits={splits}/{prefix_splits}"
                assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse), f"{tag}: differs from contiguous"
                got_o, got_l = DO.packed(case, out, lse)
                KO.assert_accurate(f"{tag}: out", got_o, o64, o32.to(dtype), factor=KO._factor("randn"),
                                   report=f"decode paged prefix {kind} D{d}")
                KO.assert_lse(f"{tag}: lse", got_l, l64, l32)
                want_k, want_v = DO.expected_caches(inp, inp.k_cache, inp.v_cache, True)
                assert torch.equal(bytes_of(kc), bytes_of(want_k)) and torch.equal(bytes_of(vc), bytes_of(want_v)), tag
                assert torch.equal(bytes_of(pp.k), bytes_of(pool_k)) and torch.equal(bytes_of(pp.v), bytes_of(pool_v))
        if tree:  # random trees: the same as the contiguous prefix under the same mask
            mask = _mask(case, tril=False, seed=d)
            ref_out, ref_lse, _, _ = _call(inp, pre.kwargs(), 3, 5, mask)
            for ps in PAGE_SIZES:
                out, lse, _, _ = _call(inp, PP.page(pre, ps, seed=ps).kwargs(), 3, 5, mask)
                assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse), (name, ps, "random tree")


def _one_pool(page_size, dtype, fp8, varlen, seed=0):
    if varlen:
        case = DO.Case("v9pool", (3, 0, 20, 5, 2, 1, 7, 0, 4), (250, 9, 0, 200, 0, 33, 1, 2, 300), 512, varlen=True,
                       layout="paged", page_size=page_size, fp8=fp8)
        n_prefix = 3
    else:
        case = DO.Case("rows80pool", (4,) * 10, (300, 0, 17, 128, 5, 250, 1, 129, 64, 200), 512, layout="paged",
                       page_size=page_size, fp8=fp8)
        n_prefix = 2
    inp = DO.build_inputs(case, dtype, 128, "randn", "cuda", seed)
    pre = DP.make_prefix(case, dtype, 128, "cuda", PLENS[:n_prefix], P_CAP, seed=seed + 7)
    pp = PP.page(pre, page_size, seed=seed + 1)
    k, v, table, ptable = PP.share_pool(inp.k_cache, inp.v_cache, inp.table, pp, seed=seed + 2)
    return inp, pre, k, v, table, ptable


@pytest.mark.parametrize("page_size", PAGE_SIZES)
def test_one_pool_shared_by_prefix_and_suffix(page_size):
    for dtype, fp8, varlen in ((torch.bfloat16, False, False), (torch.float16, True, False),
                               (torch.bfloat16, False, True), (torch.bfloat16, True, True)):
        inp, pre, k, v, table, ptable = _one_pool(page_size, dtype, fp8, varlen)
        q, kn, vn = DO.call_views(inp, True)
        kw = DO.call_kwargs(inp)
        kw.pop("block_table")
        pkw = dict(pre.kwargs(), prefix_k_cache=k, prefix_v_cache=v, prefix_block_table=ptable)
        pages = PP.prompt_pages(ptable)
        before_k, before_v = bytes_of(k[pages]).clone(), bytes_of(v[pages]).clone()
        k0, v0 = k.clone(), v.clone()
        for splits, prefix_splits in SPLITS:
            k.copy_(k0)
            v.copy_(v0)
            out, lse = dec.kernel_decode(q, k, v, inp.seqlens, kn, vn, True, 128 ** -0.5, splits=splits,
                                         prefix_splits=prefix_splits, block_table=table, **kw, **pkw)
            sk, sv = inp.k_cache.clone(), inp.v_cache.clone()
            ref_out, ref_lse = dec.kernel_decode(q, sk, sv, inp.seqlens, kn, vn, True, 128 ** -0.5, splits=splits,
                                                 prefix_splits=prefix_splits, block_table=inp.table, **kw,
                                                 **pre.kwargs())
            torch.cuda.synchronize()
            tag = f"pages of {page_size} {dtype} fp8={fp8} varlen={varlen} splits={splits}/{prefix_splits}"
            assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse), tag
            assert torch.equal(bytes_of(k[pages]), before_k) and torch.equal(bytes_of(v[pages]), before_v), tag
            want_k = appended(k0, table, inp.case.seqlens, inp.stored_k, inp.case.counts)
            want_v = appended(v0, table, inp.case.seqlens, inp.stored_v, inp.case.counts)
            assert torch.equal(bytes_of(k), bytes_of(want_k)) and torch.equal(bytes_of(v), bytes_of(want_v)), tag


def test_cuda_graph_replay_with_new_table_and_lengths():
    """A captured one-pool step picks up new prefix_block_table and prefix_seqlens contents on replay: the prompt's
    pages moved elsewhere in the pool give the same result as an eager call on the new table."""
    g = torch.Generator().manual_seed(5)
    n_prefix, n, hq, hkv, d, ps = 2, 5, 32, 8, 128, 64
    b, s_pages, p_pages = n_prefix * n, 4, 24  # own rows < 256, prompts of up to 1536 rows
    n_pool = b * s_pages + 2 * n_prefix * p_pages  # room to move the prompts
    k, v = (torch.randn(n_pool, ps, hkv, d, generator=g).bfloat16().cuda() for _ in range(2))
    q = torch.randn(b, 1, hq, d, generator=g).bfloat16().cuda()
    kn, vn = (torch.randn(b, 1, hkv, d, generator=g).bfloat16().cuda() for _ in range(2))
    own = torch.arange(b * s_pages, dtype=torch.int32).view(b, s_pages).cuda()
    ptable = (b * s_pages + torch.arange(n_prefix * p_pages, dtype=torch.int32)).view(n_prefix, p_pages).cuda()
    sl = torch.tensor([10, 0, 200, 7, 250, 3, 3, 3, 0, 64], dtype=torch.int32, device="cuda")
    pl = torch.tensor([1536, 1], dtype=torch.int32, device="cuda")

    def step(kc, vc):
        return dec.kernel_decode(q, kc, vc, sl, kn, vn, True, d ** -0.5, splits=2, block_table=own,
                                 prefix_k_cache=kc, prefix_v_cache=vc, prefix_block_table=ptable, prefix_seqlens=pl)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(k.clone(), v.clone())
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out, lse = step(k, v)
    free = b * s_pages + n_prefix * p_pages  # the second half of the prompt region
    perm = torch.randperm(n_prefix * p_pages, generator=torch.Generator().manual_seed(9)).view(n_prefix, p_pages)
    for moved, lens in ((False, [1536, 1]), (True, [0, 1535]), (True, [129, 700]), (False, [64, -5])):
        table_now = (free + perm).to(torch.int32).cuda() if moved else ptable.clone()
        if moved:  # the same prompt rows, in other pages
            k[table_now.view(-1).long()] = k[ptable.view(-1).long()]
            v[table_now.view(-1).long()] = v[ptable.view(-1).long()]
        ptable.copy_(table_now)
        pl.copy_(torch.tensor(lens, dtype=torch.int32))  # -5: clamped to 0
        ek, ev = k.clone(), v.clone()
        graph.replay()
        want_out, want_lse = step(ek, ev)
        torch.cuda.synchronize()
        assert torch.equal(out, want_out) and torch.equal(lse, want_lse), (moved, lens)
        assert torch.equal(bytes_of(k), bytes_of(ek)) and torch.equal(bytes_of(v), bytes_of(ev)), (moved, lens)


def _run_two_gpus(rank, world):
    """Per-rank suffix shards and per-rank prefix pools and tables (different page order and spare pages): out / lse
    bitwise equal on both ranks, and within fp32 summation order of the one-rank call on the gathered rows."""
    torch.cuda.set_device(rank)
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = f"cuda:{rank}"
    for name, ps in (("rows80", 16), ("varlen", 128), ("noncausal", 256)):
        case, n_prefix = CASES[name]
        case = dataclasses.replace(case, append=False)
        shards = []
        for r in range(world):
            inp = DO.build_inputs(case, torch.bfloat16, 128, "randn", dev, seed=3, cache_seed=10 + r)
            pre = DP.make_prefix(case, torch.bfloat16, 128, dev, PLENS[r:r + n_prefix], P_CAP, seed=20 + r)
            shards.append((inp, pre))
        inp, pre = shards[rank]
        pp = PP.page(pre, ps, seed=30 + rank, spare=1 + 2 * rank)
        q, _, _ = DO.call_views(inp, False)
        out, lse = dec.kernel_decode(q, inp.k_cache, inp.v_cache, inp.seqlens, None, None, case.causal,
                                     128 ** -0.5, pg=dist.group.WORLD, world=world, **DO.call_kwargs(inp),
                                     **pp.kwargs())
        both = torch.cat([out.float().reshape(-1), lse.reshape(-1)])
        got = [torch.empty_like(both) for _ in range(world)]
        dist.all_gather(got, both)
        for x in got:
            assert torch.equal(x.nan_to_num(7.0), both.nan_to_num(7.0)), f"{name}: the ranks' results differ"
        # one rank on the gathered rows: each prompt's rows of every rank, then each sequence's rows of every rank
        gk = torch.cat([s[1].k[:, :max(s[1].lens)] for s in shards], dim=1)
        gpre = DP.Prefix(gk.clone(), torch.cat([s[1].v[:, :max(s[1].lens)] for s in shards], dim=1).clone(),
                         [], torch.zeros(n_prefix, dtype=torch.int32, device=dev))
        gcases = []
        for p in range(n_prefix):
            rows_k = torch.cat([s[1].k[p, :s[1].lens[p]] for s in shards])
            rows_v = torch.cat([s[1].v[p, :s[1].lens[p]] for s in shards])
            gpre.k[p, :rows_k.shape[0]] = rows_k
            gpre.v[p, :rows_v.shape[0]] = rows_v
            gcases.append(rows_k.shape[0])
        gpre.seqlens.copy_(torch.tensor(gcases, dtype=torch.int32))
        sk = torch.cat([s[0].k_cache for s in shards], dim=1)
        sv = torch.cat([s[0].v_cache for s in shards], dim=1)
        lens = [sum(s[0].lens[i] for s in shards) for i in range(case.b)]
        for i in range(case.b):
            rows_k = torch.cat([s[0].k_cache[i, :s[0].lens[i]] for s in shards])
            rows_v = torch.cat([s[0].v_cache[i, :s[0].lens[i]] for s in shards])
            sk[i, :rows_k.shape[0]] = rows_k
            sv[i, :rows_v.shape[0]] = rows_v
        ref_out, ref_lse = dec.kernel_decode(q, sk, sv, torch.tensor(lens, dtype=torch.int32, device=dev), None, None,
                                             case.causal, 128 ** -0.5, **DO.call_kwargs(inp), **gpre.kwargs())
        torch.testing.assert_close(out.float(), ref_out.float(), atol=2e-2, rtol=2e-2, msg=lambda m: f"{name}: {m}")
        fin = torch.isfinite(ref_lse)
        assert torch.equal(fin, torch.isfinite(lse)), name
        assert ((lse - ref_lse)[fin].abs() <= 2e-4 * (1 + ref_lse[fin].abs())).all(), name


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_per_rank_pools_and_tables():
    run_distributed(_run_two_gpus, 2, backend="nccl")
