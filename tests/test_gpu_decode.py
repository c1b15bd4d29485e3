"""The sm_90a split-KV decode kernel (csrc/decode_sm90.cu) against the fp32 oracle, CUDA-graph replay, and the
cross-rank merge on two GPUs."""
import pytest
import torch
import torch.distributed as dist

import ring_flash_attn_b200 as rfa
from ring_flash_attn_b200.ops import cuda_ext
from ring_flash_attn_b200.parallel import decode as dec
from dist_utils import run_distributed
from test_decode import decode_oracle, make_case

pytestmark = pytest.mark.gpu

OUT_TOL = dict(atol=2e-2, rtol=2e-2)
LSE_TOL = dict(atol=2e-3, rtol=2e-3)

# (dtype, head_dim, batch, sq, group, s_cap, splits)
KERNEL_CASES = [
    (torch.bfloat16, 128, 1, 1, 4, 1000, None),
    (torch.bfloat16, 128, 8, 1, 8, 700, 3),
    (torch.bfloat16, 128, 2, 16, 8, 1300, 4),  # 128 packed rows: two row tiles
    (torch.bfloat16, 64, 3, 5, 1, 900, 5),
    (torch.float16, 128, 4, 4, 4, 1100, 2),
    (torch.float16, 64, 2, 2, 8, 517, None),
    (torch.float16, 128, 1, 16, 1, 2000, 8),
]


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("dtype,d,b,sq,grp,s_cap,splits", KERNEL_CASES)
def test_kernel_matches_oracle(dtype, d, b, sq, grp, s_cap, splits, causal):
    hkv = 2
    caches, lens, q, k, v = make_case(1, b, sq, hkv * grp, hkv, d, s_cap, seed=s_cap + sq, dtype=dtype,
                                      device="cuda")
    if b > 1:  # one sequence filled to the capacity after the append; make_case left sequence seed % b empty
        lens[0][(s_cap + sq + 1) % b] = s_cap - sq
    kc, vc = caches[0][0].clone(), caches[0][1].clone()
    for i in range(b):  # finite valid rows, garbage (NaN) past them, for the now longer sequence too
        kc[i, :int(lens[0][i])].nan_to_num_(0.25)
        vc[i, :int(lens[0][i])].nan_to_num_(-0.5)
        kc[i, int(lens[0][i]):] = float("nan")
        vc[i, int(lens[0][i]):] = float("nan")
    ref_caches = [(kc.clone().float().cpu(), vc.clone().float().cpu())]
    counter = cuda_ext.launch_counter()
    counter.reset()
    for append in (False, True):
        out, lse = dec.kernel_decode(q, kc, vc, lens[0], k if append else None, v if append else None, causal,
                                     d ** -0.5, splits=splits)
        torch.cuda.synchronize()
        ref_out, ref_lse = decode_oracle(q.float().cpu(), ref_caches, [lens[0].cpu()],
                                         k.float().cpu() if append else None, v.float().cpu() if append else None,
                                         causal)
        assert out.dtype == dtype and torch.isfinite(out).all()
        torch.testing.assert_close(out.float().cpu(), ref_out, **OUT_TOL)
        torch.testing.assert_close(lse.cpu(), ref_lse, **LSE_TOL)
    assert counter.value >= 5  # decode, combine; append, decode, combine
    for i in range(b):
        n0 = int(lens[0][i])
        assert torch.equal(kc[i, n0:n0 + sq], k[i]) and torch.equal(vc[i, n0:n0 + sq], v[i])


def test_public_function_runs_the_kernel_with_empty_shards():
    caches, lens, q, k, v = make_case(1, 4, 2, 16, 4, 128, 640, seed=3, dtype=torch.bfloat16, device="cuda")
    lens[0].zero_()
    kc, vc = caches[0]
    counter = cuda_ext.launch_counter()
    counter.reset()
    out, lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, lens[0], return_softmax_lse=True)
    torch.cuda.synchronize()
    assert counter.value == 2
    assert torch.equal(out, torch.zeros_like(out)) and torch.isneginf(lse).all()
    out = rfa.cp_flash_attn_with_kvcache(q, kc, vc, lens[0], k, v, append_rank=0, causal=True)
    ref_out, _ = decode_oracle(q.float().cpu(), [(kc.float().cpu(), vc.float().cpu())], [lens[0].cpu()],
                               k.float().cpu(), v.float().cpu(), True)
    torch.testing.assert_close(out.float().cpu(), ref_out, **OUT_TOL)


def test_half_million_token_cache():
    torch.manual_seed(0)
    s, hq, d = 512 * 1024 + 77, 8, 128
    kc = torch.randn(1, s + 128, 1, d, device="cuda", dtype=torch.bfloat16)
    vc = torch.randn(1, s + 128, 1, d, device="cuda", dtype=torch.bfloat16)
    q = torch.randn(1, 2, hq, d, device="cuda", dtype=torch.bfloat16) * 3
    sl = torch.tensor([s], dtype=torch.int32, device="cuda")
    out, lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, sl, return_softmax_lse=True)
    sc = torch.einsum("thd,jd->htj", q[0].float(), kc[0, :s, 0].float()) * d ** -0.5
    ref_lse = torch.logsumexp(sc, dim=-1)
    ref = torch.einsum("htj,jd->thd", torch.softmax(sc, dim=-1), vc[0, :s, 0].float())
    torch.testing.assert_close(out[0].float(), ref, **OUT_TOL)
    torch.testing.assert_close(lse[0], ref_lse, **LSE_TOL)


def test_cuda_graph_replay_after_seqlens_change():
    caches, lens, q, k, v = make_case(1, 2, 1, 32, 8, 128, 3000, seed=5, dtype=torch.bfloat16, device="cuda")
    kc, vc = caches[0]
    kc.nan_to_num_(0.0)
    vc.nan_to_num_(0.0)
    sl = torch.tensor([1000, 2500], dtype=torch.int32, device="cuda")
    f = rfa.cp_flash_attn_with_kvcache
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        f(q, kc.clone(), vc.clone(), sl, k, v, append_rank=0)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = f(q, kc, vc, sl, k, v, append_rank=0)
    for lens in ([1000, 2500], [1200, 1], [0, 2999]):
        sl.copy_(torch.tensor(lens, dtype=torch.int32))
        ek, ev = kc.clone(), vc.clone()
        g.replay()
        want = f(q, ek, ev, sl, k, v, append_rank=0)
        torch.cuda.synchronize()
        assert torch.equal(out, want), lens
        assert torch.equal(kc, ek) and torch.equal(vc, ev)


def _two_gpu_case(rank, world):
    caches, lens, q, k, v = make_case(world, 3, 4, 16, 2, 128, 900, seed=11, dtype=torch.bfloat16,
                                      device=f"cuda:{rank}")
    kc, vc = caches[rank][0].clone(), caches[rank][1].clone()
    out, lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, lens[rank], k, v, append_rank=1, causal=True,
                                              return_softmax_lse=True)
    ref_out, ref_lse = decode_oracle(q.float().cpu(), [(a.float().cpu(), b.float().cpu()) for a, b in caches],
                                     [x.cpu() for x in lens], k.float().cpu(), v.float().cpu(), True)
    torch.testing.assert_close(out.float().cpu(), ref_out, **OUT_TOL)
    torch.testing.assert_close(lse.cpu(), ref_lse, **LSE_TOL)
    both = torch.cat([out.float().reshape(-1), lse.reshape(-1)])
    got = [torch.empty_like(both) for _ in range(world)]
    dist.all_gather(got, both)
    assert all(torch.equal(x, both) for x in got)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_bitwise_equal_and_match_oracle():
    run_distributed(_two_gpu_case, 2, backend="nccl")
