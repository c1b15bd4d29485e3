"""The sm_90a split-KV decode kernel over paged caches (``block_table=``): against the fp64 oracle, bitwise against
the contiguous kernel on the same logical data, the pool after appends, a 512K-token cache, CUDA-graph replay after
the table changes, and the cross-rank merge on two GPUs."""
import pytest
import torch
import torch.distributed as dist

import ring_flash_attn_b200 as rfa
from ring_flash_attn_b200.parallel import decode as dec
from dist_utils import run_distributed
from test_decode import decode_oracle, make_case
from test_decode_paged import append_to_pool, to_pool

pytestmark = pytest.mark.gpu

OUT_TOL = dict(atol=2e-2, rtol=2e-2)
LSE_TOL = dict(atol=2e-3, rtol=2e-3)


def _finite_valid_rows(kc, vc, lens):
    """Finite values in the valid rows, NaN past them (make_case leaves NaN only past its own lengths)."""
    for i in range(kc.shape[0]):
        n = int(lens[i])
        kc[i, :n].nan_to_num_(0.25)
        vc[i, :n].nan_to_num_(-0.5)
        kc[i, n:] = float("nan")
        vc[i, n:] = float("nan")


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("page_size", [16, 64, 128, 256])
@pytest.mark.parametrize("dtype,d,sq,grp", [(torch.bfloat16, 128, 4, 4), (torch.bfloat16, 64, 2, 8),
                                            (torch.float16, 128, 2, 1), (torch.float16, 64, 4, 4)])
def test_paged_kernel_matches_oracle_and_contiguous(dtype, d, sq, grp, page_size, causal):
    b, hkv = 3, 2
    s_cap = -(-1000 // page_size) * page_size
    seed = page_size + d + sq
    caches, lens, q, k, v = make_case(1, b, sq, hkv * grp, hkv, d, s_cap, seed=seed, dtype=dtype, device="cuda")
    sl = lens[0]
    sl[(seed + 1) % b] = s_cap - sq  # filled to the capacity by the append
    sl[(seed + 2) % b] = page_size - 1  # the append crosses a page boundary
    kc, vc = caches[0]
    _finite_valid_rows(kc, vc, sl)
    pk, pv, table = to_pool(kc, vc, sl, page_size, alloc=sl + sq, seed=seed)
    ref_caches = [(kc.float().cpu(), vc.float().cpu())]
    for splits in (None, 1, 3, 7):
        out, lse = dec.kernel_decode(q, pk, pv, sl, None, None, causal, d ** -0.5, splits=splits, block_table=table)
        c_out, c_lse = dec.kernel_decode(q, kc, vc, sl, None, None, causal, d ** -0.5, splits=splits)
        assert torch.equal(out, c_out) and torch.equal(lse, c_lse), splits
    ref_out, ref_lse = decode_oracle(q.float().cpu(), ref_caches, [sl.cpu()], None, None, causal)
    assert out.dtype == dtype and torch.isfinite(out).all()
    torch.testing.assert_close(out.float().cpu(), ref_out, **OUT_TOL)
    torch.testing.assert_close(lse.cpu(), ref_lse, **LSE_TOL)

    want_k, want_v = append_to_pool(pk, table, sl, k), append_to_pool(pv, table, sl, v)
    out, lse = dec.kernel_decode(q, pk, pv, sl, k, v, causal, d ** -0.5, splits=5, block_table=table)
    c_out, c_lse = dec.kernel_decode(q, kc, vc, sl, k, v, causal, d ** -0.5, splits=5)
    torch.cuda.synchronize()
    assert torch.equal(out, c_out) and torch.equal(lse, c_lse)
    ref_out, ref_lse = decode_oracle(q.float().cpu(), ref_caches, [sl.cpu()], k.float().cpu(), v.float().cpu(),
                                     causal)
    torch.testing.assert_close(out.float().cpu(), ref_out, **OUT_TOL)
    torch.testing.assert_close(lse.cpu(), ref_lse, **LSE_TOL)
    # only the addressed pool rows changed, across the page boundary too
    assert torch.equal(pk.nan_to_num(7.0), want_k.nan_to_num(7.0))
    assert torch.equal(pv.nan_to_num(7.0), want_v.nan_to_num(7.0))


def _shuffled_pool(kc, vc, page_size, spare, seed):
    """Every page of the contiguous (B, S_cap, Hkv, D) caches, in a seeded random order among ``spare`` extra NaN
    pages.  Returns (k_pool, v_pool, block_table)."""
    b, s_cap = kc.shape[:2]
    mb = s_cap // page_size
    perm = torch.randperm(b * mb + spare, generator=torch.Generator().manual_seed(seed)).to(kc.device)
    pools = []
    for c in (kc, vc):
        pool = c.new_full((b * mb + spare, page_size) + tuple(c.shape[2:]), float("nan"))
        pool[perm[:b * mb]] = c.reshape(b * mb, page_size, *c.shape[2:])
        pools.append(pool)
    return pools[0], pools[1], perm[:b * mb].to(torch.int32).view(b, mb)


def test_half_million_token_paged_cache():
    torch.manual_seed(0)
    s, hq, d, ps = 512 * 1024 + 77, 8, 128, 16
    s_cap = s + 128 - 77  # whole pages
    kc = torch.randn(1, s_cap, 1, d, device="cuda", dtype=torch.bfloat16)
    vc = torch.randn(1, s_cap, 1, d, device="cuda", dtype=torch.bfloat16)
    pk, pv, table = _shuffled_pool(kc, vc, ps, spare=5, seed=1)
    table[0, -(-s // ps):] = -1  # pages past the valid rows are never read
    q = torch.randn(1, 2, hq, d, device="cuda", dtype=torch.bfloat16) * 3
    sl = torch.tensor([s], dtype=torch.int32, device="cuda")
    out, lse = rfa.cp_flash_attn_with_kvcache(q, pk, pv, sl, return_softmax_lse=True, block_table=table)
    c_out, c_lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, sl, return_softmax_lse=True)
    assert torch.equal(out, c_out) and torch.equal(lse, c_lse)
    sc = torch.einsum("thd,jd->htj", q[0].float(), kc[0, :s, 0].float()) * d ** -0.5
    ref_lse = torch.logsumexp(sc, dim=-1)
    ref = torch.einsum("htj,jd->thd", torch.softmax(sc, dim=-1), vc[0, :s, 0].float())
    torch.testing.assert_close(out[0].float(), ref, **OUT_TOL)
    torch.testing.assert_close(lse[0], ref_lse, **LSE_TOL)


def test_cuda_graph_replay_after_table_changes():
    ps = 16
    caches, lens, q, k, v = make_case(1, 2, 1, 32, 8, 128, 3008, seed=5, dtype=torch.bfloat16, device="cuda")
    kc, vc = caches[0]
    kc.nan_to_num_(0.0)
    vc.nan_to_num_(0.0)
    pk, pv, table = _shuffled_pool(kc, vc, ps, spare=4, seed=5)
    pk.nan_to_num_(0.0)
    pv.nan_to_num_(0.0)
    spare = sorted(set(range(pk.shape[0])) - set(table.flatten().tolist()))  # page ids no sequence uses
    sl = torch.tensor([1000, 2500], dtype=torch.int32, device="cuda")
    f = rfa.cp_flash_attn_with_kvcache
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        f(q, pk.clone(), pv.clone(), sl, k, v, append_rank=0, block_table=table)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = f(q, pk, pv, sl, k, v, append_rank=0, block_table=table)
    for lens, seq, row in (([1000, 2500], None, None), ([1200, 1], 0, 1100), ([0, 2999], 1, 2999)):
        sl.copy_(torch.tensor(lens, dtype=torch.int32))
        if seq is not None:  # move a page that is read to a newly allocated page; the old one holds other data
            new = spare.pop()
            old = int(table[seq, row // ps])
            pk[new], pv[new] = pk[old], pv[old]
            pk[old].fill_(3.0)
            pv[old].fill_(-3.0)
            table[seq, row // ps] = new
        ek, ev = pk.clone(), pv.clone()
        g.replay()
        want = f(q, ek, ev, sl, k, v, append_rank=0, block_table=table)
        torch.cuda.synchronize()
        assert torch.equal(out, want), lens
        assert torch.equal(pk, ek) and torch.equal(pv, ev)
        # the logical cache the table now describes, contiguous, gives the same result (appending the same rows again
        # into the copy changes nothing)
        logical_k, logical_v = pk[table.long()].flatten(1, 2), pv[table.long()].flatten(1, 2)
        assert torch.equal(out, f(q, logical_k, logical_v, sl, k, v, append_rank=0)), lens


def _two_gpu_case(rank, world):
    caches, lens, q, k, v = make_case(world, 3, 4, 16, 2, 128, 896, seed=11, dtype=torch.bfloat16,
                                      device=f"cuda:{rank}")
    kc, vc = caches[rank]
    pk, pv, table = to_pool(kc, vc, lens[rank], 64, alloc=lens[rank] + 4, seed=rank)
    out, lse = rfa.cp_flash_attn_with_kvcache(q, pk, pv, lens[rank], k, v, append_rank=1, causal=True,
                                              return_softmax_lse=True, block_table=table)
    ref_out, ref_lse = decode_oracle(q.float().cpu(), [(a.float().cpu(), b.float().cpu()) for a, b in caches],
                                     [x.cpu() for x in lens], k.float().cpu(), v.float().cpu(), True)
    torch.testing.assert_close(out.float().cpu(), ref_out, **OUT_TOL)
    torch.testing.assert_close(lse.cpu(), ref_lse, **LSE_TOL)
    both = torch.cat([out.float().reshape(-1), lse.reshape(-1)])
    got = [torch.empty_like(both) for _ in range(world)]
    dist.all_gather(got, both)
    assert all(torch.equal(x, both) for x in got)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_paged_bitwise_equal_and_match_oracle():
    run_distributed(_two_gpu_case, 2, backend="nccl")
