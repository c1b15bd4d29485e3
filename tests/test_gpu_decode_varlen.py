"""The sm_90a split-KV decode kernel with variable-length query batches (``cu_seqlens_q``): against the per-sequence
fp64 oracle; bitwise against a uniform call on each sequence alone, against the uniform call at equal counts, between
paged and contiguous caches and, for e4m3 caches at power-of-two descales, against the bf16 / fp16 kernel on the
widened cache; the cache bytes after the append; CUDA-graph replay after the counts and lengths change; a 512K-token
cache in a mixed batch; and the cross-rank merge on two GPUs."""
import pytest
import torch
import torch.distributed as dist

import ring_flash_attn_b200 as rfa
from ring_flash_attn_b200.parallel import decode as dec
from dist_utils import run_distributed
from test_decode import make_case
from test_decode_paged import to_pool
from test_decode_varlen import appended, cu_of, pack, varlen_oracle
from test_gpu_decode_fp8 import assert_scaled, bytes_of, quantize

pytestmark = pytest.mark.gpu

OUT_TOL = dict(atol=2e-2, rtol=2e-2)
LSE_TOL = dict(atol=2e-3, rtol=2e-3)

# (dtype, head_dim, group, counts): several sequences' row tiles in adjacent slots, idle slots at the end, 0-token
# sequences, and chunks longer than one 64-row tile
KERNEL_CASES = [
    (torch.bfloat16, 128, 4, (1, 0, 40, 3, 1, 17, 0, 1)),  # 9 tiles in 11 slots
    (torch.bfloat16, 64, 1, (1, 70, 0, 2, 1)),  # 5 tiles in 6 slots
    (torch.float16, 128, 8, (1, 0, 9, 1, 3)),  # 5 tiles in 6 slots
    (torch.float16, 64, 4, (5, 16, 1, 1)),  # 4 tiles in 4 slots
]


def ragged_case(dtype, d, grp, counts, s_cap, seed, hkv=2):
    """make_case on the GPU with finite valid rows and NaN past them; sequence 1 is filled to the capacity by the
    append.  Returns caches, lens, the (B, Smax) q / k / v and their packed rows, and cu_seqlens_q."""
    b, smax = len(counts), max(counts)
    caches, lens, q4, k4, v4 = make_case(1, b, smax, hkv * grp, hkv, d, s_cap, seed=seed, dtype=dtype, device="cuda")
    sl = lens[0]
    sl[1] = s_cap - counts[1]
    kc, vc = caches[0]
    for i in range(b):
        n = int(sl[i])
        kc[i, :n].nan_to_num_(0.25)
        vc[i, :n].nan_to_num_(-0.5)
        kc[i, n:] = float("nan")
        vc[i, n:] = float("nan")
    return kc, vc, sl, q4, k4, v4, pack(q4, counts), pack(k4, counts), pack(v4, counts), cu_of(counts, "cuda")


def sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("dtype,d,grp,counts", KERNEL_CASES)
def test_varlen_kernel_matches_oracle_and_per_sequence_calls(dtype, d, grp, counts, causal):
    b, smax, hkv, s_cap = len(counts), max(counts), 2, 900
    kc, vc, sl, q4, k4, v4, q, k, v, cu = ragged_case(dtype, d, grp, counts, s_cap, seed=d + grp)
    hq, total_q = hkv * grp, sum(counts)
    assert dec.tile_slots(b, total_q, smax, hq, hkv) >= sum(-(-n * grp // 64) for n in counts)
    scale = d ** -0.5
    ref_caches = [(kc.float().cpu(), vc.float().cpu())]
    for append in (False, True):
        kn, vn = (k, v) if append else (None, None)
        ref_out, ref_lse = varlen_oracle(q4.float().cpu(), ref_caches, [sl.cpu()],
                                         k4.float().cpu() if append else None, v4.float().cpu() if append else None,
                                         counts, causal)
        for splits in (None, 1, 3, 7):
            sp = splits or dec.num_splits_varlen(b, total_q, smax, hq, hkv, s_cap, sm_count())
            ka, va = kc.clone(), vc.clone()
            out, lse = dec.kernel_decode(q, ka, va, sl, kn, vn, causal, scale, splits=splits, cu_seqlens_q=cu,
                                         max_seqlen_q=smax)
            torch.cuda.synchronize()
            assert out.shape == q.shape and lse.shape == (hq, total_q)
            assert out.dtype == dtype and torch.isfinite(out).all()
            torch.testing.assert_close(out.float().cpu(), ref_out, **OUT_TOL)
            torch.testing.assert_close(lse.cpu(), ref_lse, **LSE_TOL)
            # bitwise a uniform call on each sequence alone, with the same split count
            kb, vb = kc.clone(), vc.clone()
            lo = 0
            for i, n in enumerate(counts):
                if n:  # x[i, :n][None]: a (1, n) view with stride(0) = n * stride(1), as the kernel takes it
                    o, l = dec.kernel_decode(q4[i, :n][None], kb[i:i + 1], vb[i:i + 1], sl[i:i + 1],
                                             k4[i, :n][None] if append else None, v4[i, :n][None] if append else None,
                                             causal, scale, splits=sp)
                    assert torch.equal(out[lo:lo + n], o[0]), (i, splits)
                    assert torch.equal(lse[:, lo:lo + n], l[0]), (i, splits)
                lo += n
            torch.cuda.synchronize()
            assert torch.equal(bytes_of(ka), bytes_of(kb)) and torch.equal(bytes_of(va), bytes_of(vb))
            want_k = appended(kc, None, sl, k, counts) if append else kc
            want_v = appended(vc, None, sl, v, counts) if append else vc
            assert torch.equal(bytes_of(ka), bytes_of(want_k)) and torch.equal(bytes_of(va), bytes_of(want_v))


@pytest.mark.parametrize("causal", [True, False])
def test_equal_counts_are_the_uniform_call(causal):
    b, sq, grp, hkv, d = 5, 4, 4, 2, 128
    kc, vc, sl, q4, k4, v4, q, k, v, cu = ragged_case(torch.bfloat16, d, grp, (sq,) * b, 700, seed=9)
    for splits in (None, 3):
        ka, va, kb, vb = kc.clone(), vc.clone(), kc.clone(), vc.clone()
        u_out, u_lse = dec.kernel_decode(q4, ka, va, sl, k4, v4, causal, d ** -0.5, splits=splits)
        out, lse = dec.kernel_decode(q, kb, vb, sl, k, v, causal, d ** -0.5, splits=splits, cu_seqlens_q=cu,
                                     max_seqlen_q=sq)
        torch.cuda.synchronize()
        assert torch.equal(out, u_out.flatten(0, 1))
        assert torch.equal(lse, u_lse.permute(1, 0, 2).reshape(hkv * grp, b * sq))
        assert torch.equal(bytes_of(ka), bytes_of(kb)) and torch.equal(bytes_of(va), bytes_of(vb))


@pytest.mark.parametrize("page_size", [16, 128])
def test_paged_varlen_equals_contiguous_varlen(page_size):
    counts = (1, 0, 40, 3, 1, 17, 0, 1)
    s_cap = 1024
    kc, vc, sl, q4, k4, v4, q, k, v, cu = ragged_case(torch.bfloat16, 128, 4, counts, s_cap, seed=21)
    alloc = (sl + torch.tensor(counts, device="cuda")).clamp(max=s_cap)
    pk, pv, table = to_pool(kc, vc, sl, page_size, alloc=alloc, seed=21)
    for append in (False, True):
        kn, vn = (k, v) if append else (None, None)
        pk0, pv0 = pk.clone(), pv.clone()
        ka, va = kc.clone(), vc.clone()
        c_out, c_lse = dec.kernel_decode(q, ka, va, sl, kn, vn, True, 0.1, splits=5, cu_seqlens_q=cu, max_seqlen_q=40)
        p_out, p_lse = dec.kernel_decode(q, pk, pv, sl, kn, vn, True, 0.1, splits=5, block_table=table,
                                         cu_seqlens_q=cu, max_seqlen_q=40)
        torch.cuda.synchronize()
        assert torch.equal(c_out, p_out) and torch.equal(c_lse, p_lse), append
        if append:  # the pool bytes after the varlen append
            assert torch.equal(bytes_of(pk), bytes_of(appended(pk0, table, sl, k, counts)))
            assert torch.equal(bytes_of(pv), bytes_of(appended(pv0, table, sl, v, counts)))


@pytest.mark.parametrize("page_size", [None, 16])
@pytest.mark.parametrize("dtype,d", [(torch.bfloat16, 128), (torch.float16, 64)])
def test_fp8_varlen_equals_widened_kernel(dtype, d, page_size):
    counts = (2, 0, 33, 1, 5)
    s_cap = 1024
    b, hkv, grp, smax = len(counts), 2, 4, max(counts)
    kc, vc, sl, q4, k4, v4, q, k, v, cu = ragged_case(dtype, d, grp, counts, s_cap, seed=d)
    p2k, p2v = torch.full((b, hkv), 2.0 ** -3, device="cuda"), torch.full((b, hkv), 2.0 ** 5, device="cuda")
    # cache bytes of ordinary magnitude (V quantised at 2^5 would put fp16 outputs near the subnormal range)
    k8, v8 = quantize(kc, torch.full_like(p2k, 0.37)), quantize(vc, torch.full_like(p2v, 0.05))
    wk, wv = k8.to(dtype), v8.to(dtype)  # the widened cache (exact)
    pk, pv, table = k8, v8, None
    if page_size is not None:
        alloc = (sl + torch.tensor(counts, device="cuda")).clamp(max=s_cap)
        pk, pv, table = to_pool(k8, v8, sl, page_size, alloc=alloc, seed=d)
    scale = d ** -0.5
    vl = dict(cu_seqlens_q=cu, max_seqlen_q=smax)
    for causal in (True, False):
        e_out, e_lse = dec.kernel_decode(q, pk, pv, sl, None, None, causal, scale, splits=3, block_table=table,
                                         k_descale=p2k, v_descale=p2v, **vl)
        w_out, w_lse = dec.kernel_decode(q, wk, wv, sl, None, None, causal, scale * 2.0 ** -3, splits=3, **vl)
        assert_scaled(e_out, w_out, 2.0 ** 5)
        assert torch.equal(e_lse, w_lse)
    # append: the e4m3 bytes are torch's quantisation, and the result is the widened kernel's with the widened rows
    kq, vq = pack(quantize(k4, p2k), counts), pack(quantize(v4, p2v), counts)
    want_k, want_v = appended(pk, table, sl, kq, counts), appended(pv, table, sl, vq, counts)
    e_out, e_lse = dec.kernel_decode(q, pk, pv, sl, k, v, True, scale, splits=4, block_table=table, k_descale=p2k,
                                     v_descale=p2v, **vl)
    w_out, w_lse = dec.kernel_decode(q, wk, wv, sl, kq.to(dtype), vq.to(dtype), True, scale * 2.0 ** -3, splits=4,
                                     **vl)
    torch.cuda.synchronize()
    assert torch.equal(bytes_of(pk), bytes_of(want_k)) and torch.equal(bytes_of(pv), bytes_of(want_v))
    assert_scaled(e_out, w_out, 2.0 ** 5)
    assert torch.equal(e_lse, w_lse)


@pytest.mark.parametrize("page_size", [None, 16])
def test_cuda_graph_replay_after_counts_and_lengths_change(page_size):
    b, total_q, smax, hkv, grp, d, s_cap = 4, 8, 5, 8, 4, 128, 3008
    caches, lens, q4, k4, v4 = make_case(1, b, total_q, hkv * grp, hkv, d, s_cap, seed=5, dtype=torch.bfloat16,
                                         device="cuda")
    kc, vc = caches[0][0].nan_to_num(0.0), caches[0][1].nan_to_num(0.0)
    q, k, v = q4[0], k4[0], v4[0]  # total_q packed rows
    table = None
    if page_size is not None:
        kc, vc, table = to_pool(kc, vc, torch.full((b,), s_cap), page_size, seed=5)
    cu = cu_of((1, 5, 0, 2), "cuda")
    sl = torch.tensor([1000, 2500, 7, 0], dtype=torch.int32, device="cuda")
    f = rfa.cp_flash_attn_with_kvcache
    kw = dict(append_rank=0, block_table=table, cu_seqlens_q=cu, max_seqlen_q=smax, return_softmax_lse=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        f(q, kc.clone(), vc.clone(), sl, k, v, **kw)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out, lse = f(q, kc, vc, sl, k, v, **kw)
    for counts, lens_now in (((1, 5, 0, 2), [1000, 2500, 7, 0]), ((2, 2, 2, 2), [1200, 1, 0, 3000]),
                             ((0, 5, 3, 0), [0, 2999, 64, 5])):
        cu.copy_(cu_of(counts))
        sl.copy_(torch.tensor(lens_now, dtype=torch.int32))
        ek, ev = kc.clone(), vc.clone()
        g.replay()
        want_out, want_lse = f(q, ek, ev, sl, k, v, **kw)
        torch.cuda.synchronize()
        assert torch.equal(out, want_out) and torch.equal(lse, want_lse), counts
        assert torch.equal(bytes_of(kc), bytes_of(ek)) and torch.equal(bytes_of(vc), bytes_of(ev)), counts


def test_half_million_token_cache_in_a_mixed_batch():
    torch.manual_seed(0)
    s, hq, d = 512 * 1024 + 77, 8, 128
    counts = (64, 1, 1)
    kc = torch.randn(3, s + 128, 1, d, device="cuda", dtype=torch.bfloat16)
    vc = torch.randn(3, s + 128, 1, d, device="cuda", dtype=torch.bfloat16)
    q = torch.randn(sum(counts), hq, d, device="cuda", dtype=torch.bfloat16) * 3
    sl = torch.tensor([s, 1000, 0], dtype=torch.int32, device="cuda")
    out, lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, sl, return_softmax_lse=True,
                                              cu_seqlens_q=cu_of(counts, "cuda"), max_seqlen_q=64)
    for i, (lo, n) in enumerate(((0, 64), (64, 1))):
        keys = int(sl[i])
        sc = torch.einsum("thd,jd->htj", q[lo:lo + n].float(), kc[i, :keys, 0].float()) * d ** -0.5
        ref = torch.einsum("htj,jd->thd", torch.softmax(sc, dim=-1), vc[i, :keys, 0].float())
        torch.testing.assert_close(out[lo:lo + n].float(), ref, **OUT_TOL)
        torch.testing.assert_close(lse[:, lo:lo + n], torch.logsumexp(sc, dim=-1), **LSE_TOL)
    assert torch.equal(out[65:], torch.zeros_like(out[65:])) and torch.isneginf(lse[:, 65:]).all()  # empty shard


def _two_gpu_case(rank, world):
    counts = (1, 0, 20, 3)
    b, smax = len(counts), max(counts)
    caches, lens, q4, k4, v4 = make_case(world, b, smax, 16, 2, 128, 900, seed=11, dtype=torch.bfloat16,
                                         device=f"cuda:{rank}")
    q, k, v = pack(q4, counts), pack(k4, counts), pack(v4, counts)
    kc, vc = caches[rank][0].clone(), caches[rank][1].clone()
    out, lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, lens[rank], k, v, append_rank=1, causal=True,
                                              return_softmax_lse=True, cu_seqlens_q=cu_of(counts, q.device),
                                              max_seqlen_q=smax)
    ref_out, ref_lse = varlen_oracle(q4.float().cpu(), [(a.float().cpu(), c.float().cpu()) for a, c in caches],
                                     [x.cpu() for x in lens], k4.float().cpu(), v4.float().cpu(), counts, True)
    torch.testing.assert_close(out.float().cpu(), ref_out, **OUT_TOL)
    torch.testing.assert_close(lse.cpu(), ref_lse, **LSE_TOL)
    both = torch.cat([out.float().reshape(-1), lse.reshape(-1)])
    got = [torch.empty_like(both) for _ in range(world)]
    dist.all_gather(got, both)
    assert all(torch.equal(x, both) for x in got)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_varlen_bitwise_equal_and_match_oracle():
    run_distributed(_two_gpu_case, 2, backend="nccl")
