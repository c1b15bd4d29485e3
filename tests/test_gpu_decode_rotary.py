"""The sm_90a split-KV decode kernel with rotary embeddings fused into its query load and cache append: bitwise the
plain kernel on ``apply_rotary``-rotated q / k (out, lse and the cache bytes) and the fp64 oracle on those inputs, for
bf16 / fp16 x head_dim 64 / 128 over contiguous, paged and e4m3 caches, uniform and varlen queries, causal and not,
interleaved and not, rotary_dim in {D, D/2, 16}, with several splits; positions past the tables clamp; CUDA-graph
replay after the positions and lengths change; and the cross-rank merge on two GPUs."""
import pytest
import torch
import torch.distributed as dist

import ring_flash_attn_b200 as rfa
from ring_flash_attn_b200.parallel import decode as dec
from dist_utils import run_distributed
from test_decode import decode_oracle, make_case
from test_decode_paged import to_pool
from test_decode_rotary import rope_tables, rotate_grid
from test_decode_varlen import cu_of, pack, varlen_oracle
from test_gpu_decode_fp8 import bytes_of, dequantize, quantize
from test_gpu_decode_varlen import LSE_TOL, OUT_TOL, ragged_case

pytestmark = pytest.mark.gpu

S_CAP = 640
COUNTS = (1, 0, 40, 3, 17)  # varlen: a 0, and a chunk longer than one 64-row tile at G = 4


def _case(dtype, d, varlen, seed):
    counts = COUNTS if varlen else (4,) * 3
    kc, vc, sl, q4, k4, v4, q, k, v, cu = ragged_case(dtype, d, 4, counts, S_CAP, seed)
    return counts, kc, vc, sl, q4, k4, v4, cu


@pytest.mark.parametrize("layout", ["contiguous", "paged16", "e4m3"])
@pytest.mark.parametrize("dtype,d", [(torch.bfloat16, 128), (torch.bfloat16, 64), (torch.float16, 128),
                                     (torch.float16, 64)])
def test_rotary_kernel_is_the_plain_kernel_on_rotated_inputs(dtype, d, layout):
    n = 0
    for varlen in (False, True):
        counts, kc, vc, sl, q4, k4, v4, cu = _case(dtype, d, varlen, seed=d + len(layout) + varlen)
        b = len(counts)
        kw = {}
        if layout == "e4m3":
            kd, vd = torch.full((b, 2), 0.37, device="cuda"), torch.full((b, 2), 0.05, device="cuda")
            kc, vc = quantize(kc, kd), quantize(vc, vd)
            kw.update(k_descale=kd, v_descale=vd)
        table = None
        if layout == "paged16":
            alloc = (sl + torch.tensor(counts, device="cuda")).clamp(max=S_CAP)
            kc, vc, table = to_pool(kc, vc, sl, 16, alloc=alloc, seed=d)
            kw.update(block_table=table)
        if varlen:
            kw.update(cu_seqlens_q=cu, max_seqlen_q=max(counts))
        rs = (sl + 1000 + 7 * torch.arange(b, device="cuda", dtype=torch.int32)).contiguous()
        for causal in (True, False):
            for interleaved in (True, False):
                for rotary_dim in (d, d // 2, 16):
                    n += 1
                    cos, sin = rope_tables(S_CAP + 1200, rotary_dim, dtype, "cuda")
                    q4r, k4r = rotate_grid(q4, k4, cos, sin, rs, causal, interleaved)
                    q, k, v, qr, kr = ((pack(x, counts) for x in (q4, k4, v4, q4r, k4r)) if varlen
                                       else (q4, k4, v4, q4r, k4r))
                    splits = 3 + n % 3
                    ka, va, kb, vb = kc.clone(), vc.clone(), kc.clone(), vc.clone()
                    out, lse = dec.kernel_decode(q, ka, va, sl, k, v, causal, d ** -0.5, splits=splits,
                                                 rotary_cos=cos, rotary_sin=sin, rotary_seqlens=rs,
                                                 rotary_interleaved=interleaved, **kw)
                    p_out, p_lse = dec.kernel_decode(qr, kb, vb, sl, kr, v, causal, d ** -0.5, splits=splits, **kw)
                    torch.cuda.synchronize()
                    tag = (varlen, causal, interleaved, rotary_dim)
                    assert torch.equal(out, p_out) and torch.equal(lse, p_lse), tag
                    assert torch.equal(bytes_of(ka), bytes_of(kb)) and torch.equal(bytes_of(va), bytes_of(vb)), tag
                    # the fp64 oracle on the rotated inputs (the cache as this rank holds it before the append)
                    if layout == "e4m3":
                        ref_c = [(dequantize(kc, kw["k_descale"]).cpu(), dequantize(vc, kw["v_descale"]).cpu())]
                        kn = dequantize(quantize(k4r, kw["k_descale"]), kw["k_descale"]).cpu()
                        vn = dequantize(quantize(v4, kw["v_descale"]), kw["v_descale"]).cpu()
                    elif layout == "paged16":
                        continue  # bitwise the plain paged kernel, which is bitwise the contiguous one
                    else:
                        ref_c = [(kc.float().cpu(), vc.float().cpu())]
                        kn, vn = k4r.float().cpu(), v4.float().cpu()
                    oracle = varlen_oracle if varlen else decode_oracle
                    args = (counts, causal) if varlen else (causal,)
                    ref_out, ref_lse = oracle(q4r.float().cpu(), ref_c, [sl.cpu()], kn, vn, *args)
                    torch.testing.assert_close(out.float().cpu(), ref_out, **OUT_TOL)
                    torch.testing.assert_close(lse.cpu(), ref_lse, **LSE_TOL)


@pytest.mark.parametrize("causal", [True, False])
def test_positions_past_the_tables_clamp(causal):
    dtype, d, sq, seqlen_ro = torch.bfloat16, 128, 4, 50
    counts, kc, vc, sl, q4, k4, v4, cu = _case(dtype, d, False, seed=3)
    cos, sin = rope_tables(seqlen_ro, d, dtype, "cuda")
    rs = torch.tensor([48, 400, -9], dtype=torch.int32, device="cuda")  # partly, wholly and below the tables
    keys = (rs.long()[:, None] + torch.arange(sq, device="cuda")[None]).clamp(0, seqlen_ro - 1)
    queries = keys if causal else rs.long()[:, None].clamp(0, seqlen_ro - 1).expand_as(keys)
    qr, kr = dec.apply_rotary(q4, cos, sin, queries, False), dec.apply_rotary(k4, cos, sin, keys, False)
    ka, va, kb, vb = kc.clone(), vc.clone(), kc.clone(), vc.clone()
    out, lse = dec.kernel_decode(q4, ka, va, sl, k4, v4, causal, 0.1, splits=4, rotary_cos=cos, rotary_sin=sin,
                                 rotary_seqlens=rs, rotary_interleaved=False)
    p_out, p_lse = dec.kernel_decode(qr, kb, vb, sl, kr, v4, causal, 0.1, splits=4)
    torch.cuda.synchronize()
    assert torch.equal(out, p_out) and torch.equal(lse, p_lse)
    assert torch.equal(bytes_of(ka), bytes_of(kb))


@pytest.mark.parametrize("varlen", [False, True])
def test_cuda_graph_replay_after_positions_and_lengths_change(varlen):
    b, sq, hkv, grp, d, s_cap = 4, 2, 8, 4, 128, 3008
    caches, lens, q4, k4, v4 = make_case(1, b, sq, hkv * grp, hkv, d, s_cap, seed=5, dtype=torch.bfloat16,
                                         device="cuda")
    kc, vc = caches[0][0].nan_to_num(0.0), caches[0][1].nan_to_num(0.0)
    cos, sin = rope_tables(8192, d, torch.bfloat16, "cuda")
    sl = torch.tensor([1000, 2500, 7, 0], dtype=torch.int32, device="cuda")
    rs = torch.tensor([3000, 5000, 7, 1], dtype=torch.int32, device="cuda")
    kw = dict(append_rank=0, return_softmax_lse=True, rotary_cos=cos, rotary_sin=sin, rotary_seqlens=rs,
              rotary_interleaved=False)
    q, k, v = q4, k4, v4
    if varlen:
        counts = (1, 2, 0, 2)
        q, k, v = pack(q4, counts), pack(k4, counts), pack(v4, counts)
        kw.update(cu_seqlens_q=cu_of(counts, "cuda"), max_seqlen_q=sq)
    f = rfa.cp_flash_attn_with_kvcache
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        f(q, kc.clone(), vc.clone(), sl, k, v, **kw)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out, lse = f(q, kc, vc, sl, k, v, **kw)
    for lens_now, pos_now in (([1000, 2500, 7, 0], [3000, 5000, 7, 1]), ([1200, 1, 0, 3000], [1200, 8000, 0, 6000]),
                              ([0, 2999, 64, 5], [9000, 2999, 100, 0])):
        sl.copy_(torch.tensor(lens_now, dtype=torch.int32))
        rs.copy_(torch.tensor(pos_now, dtype=torch.int32))
        ek, ev = kc.clone(), vc.clone()
        g.replay()
        want_out, want_lse = f(q, ek, ev, sl, k, v, **kw)
        torch.cuda.synchronize()
        assert torch.equal(out, want_out) and torch.equal(lse, want_lse), pos_now
        assert torch.equal(bytes_of(kc), bytes_of(ek)) and torch.equal(bytes_of(vc), bytes_of(ev)), pos_now


def _two_gpu_case(rank, world):
    counts = (1, 0, 20, 3)
    b, smax, d = len(counts), max(counts), 128
    caches, lens, q4, k4, v4 = make_case(world, b, smax, 16, 2, d, 900, seed=11, dtype=torch.bfloat16,
                                         device=f"cuda:{rank}")
    cos, sin = rope_tables(4096, d, torch.bfloat16, q4.device)
    rs = sum(x for x in lens).to(torch.int32)  # the cached tokens of both ranks come first
    q4r, k4r = rotate_grid(q4, k4, cos, sin, rs, True, False)
    q, k, v = pack(q4, counts), pack(k4, counts), pack(v4, counts)
    kc, vc = caches[rank][0].clone(), caches[rank][1].clone()
    out, lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, lens[rank], k, v, append_rank=1, causal=True,
                                              return_softmax_lse=True, cu_seqlens_q=cu_of(counts, q.device),
                                              max_seqlen_q=smax, rotary_cos=cos, rotary_sin=sin, rotary_seqlens=rs,
                                              rotary_interleaved=False)
    ref_out, ref_lse = varlen_oracle(q4r.float().cpu(), [(a.float().cpu(), c.float().cpu()) for a, c in caches],
                                     [x.cpu() for x in lens], k4r.float().cpu(), v4.float().cpu(), counts, True)
    torch.testing.assert_close(out.float().cpu(), ref_out, **OUT_TOL)
    torch.testing.assert_close(lse.cpu(), ref_lse, **LSE_TOL)
    both = torch.cat([out.float().reshape(-1), lse.reshape(-1)])
    got = [torch.empty_like(both) for _ in range(world)]
    dist.all_gather(got, both)
    assert all(torch.equal(x, both) for x in got)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_rotary_bitwise_equal_and_match_oracle():
    run_distributed(_two_gpu_case, 2, backend="nccl")
