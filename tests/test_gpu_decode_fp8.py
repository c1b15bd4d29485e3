"""The sm_90a split-KV decode kernel over fp8 (e4m3) caches: against the fp64 oracle on the dequantised cache, bitwise
against the bf16 / fp16 kernel on the widened cache (unit and power-of-two descales, before and after an append), the
cache bytes after the append kernel's quantisation (contiguous and paged), a 512K-token cache, CUDA-graph replay after
the lengths and descales change, and the cross-rank merge on two GPUs with per-rank descales."""
import pytest
import torch
import torch.distributed as dist

import ring_flash_attn_b200 as rfa
from ring_flash_attn_b200.parallel import decode as dec
from dist_utils import run_distributed
from test_decode import decode_oracle, make_case
from test_decode_paged import append_to_pool, to_pool

pytestmark = pytest.mark.gpu

E4M3 = torch.float8_e4m3fn
OUT_TOL = dict(atol=2e-2, rtol=2e-2)
LSE_TOL = dict(atol=2e-3, rtol=2e-3)


def quantize(x, descale):
    """Reference e4m3 storage of x (B, S, Hkv, D) with a (B, Hkv) descale."""
    return (x.float() / descale[:, None, :, None]).clamp(-448, 448).to(E4M3)


def dequantize(x8, descale):
    return x8.float() * descale[:, None, :, None]


def head_descales(b, hkv, base, device="cuda"):
    return (base * (1 + 0.1 * torch.arange(b * hkv, dtype=torch.float32, device=device))).view(b, hkv)


def assert_scaled(e_out, w_out, f):
    """e_out is the bf16 / fp16 kernel's w_out scaled by the power of two f (the fp8 kernel's v_descale): bitwise
    wherever w_out is a normal number.  A subnormal fp16 w_out was itself rounded to fewer bits than e_out, so there
    the two agree to 2^-18."""
    tiny = torch.finfo(w_out.dtype).tiny
    normal = w_out.float().abs() >= tiny
    assert torch.equal(e_out[normal], (w_out.float() * f).to(w_out.dtype)[normal])
    torch.testing.assert_close(e_out.float(), w_out.float() * f, atol=2.0 ** -18, rtol=0)


def bytes_of(x):
    return x.view(torch.uint8)


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("page_size", [None, 16, 128])
@pytest.mark.parametrize("dtype,d,sq,grp", [(torch.bfloat16, 128, 4, 4), (torch.bfloat16, 64, 2, 8),
                                            (torch.float16, 128, 2, 1), (torch.float16, 64, 4, 4)])
def test_fp8_kernel_matches_oracle_and_widened_kernel(dtype, d, sq, grp, page_size, causal):
    b, hkv = 3, 2
    ps = page_size or 128
    s_cap = -(-1000 // ps) * ps
    seed = (page_size or 0) + d + sq
    caches, lens, q, k, v = make_case(1, b, sq, hkv * grp, hkv, d, s_cap, seed=seed, dtype=dtype, device="cuda")
    sl = lens[0]
    sl[(seed + 1) % b] = s_cap - sq  # filled to the capacity by the append
    sl[(seed + 2) % b] = ps - 1  # the append crosses a page boundary
    kc, vc = caches[0]
    for i in range(b):  # finite valid rows, NaN (e4m3 byte 0x7F) past them
        n = int(sl[i])
        kc[i, :n].nan_to_num_(0.25)
        vc[i, :n].nan_to_num_(-0.5)
        kc[i, n:] = float("nan")
        vc[i, n:] = float("nan")
    kd, vd = head_descales(b, hkv, 0.37), head_descales(b, hkv, 0.05)
    k8, v8 = quantize(kc, kd), quantize(vc, vd)
    for i in range(b):
        assert (bytes_of(k8)[i, int(sl[i]):] == 0x7F).all() and (bytes_of(v8)[i, int(sl[i]):] == 0x7F).all()
    table = None
    pk, pv = k8, v8
    if page_size is not None:
        pk, pv, table = to_pool(k8, v8, sl, page_size, alloc=sl + sq, seed=seed)
    scale = d ** -0.5
    ones = torch.ones(b, hkv, device="cuda")
    p2k, p2v = torch.full((b, hkv), 2.0 ** -3, device="cuda"), torch.full((b, hkv), 2.0 ** 5, device="cuda")
    wk, wv = k8.to(dtype), v8.to(dtype)  # the widened cache (exact)

    ref_caches = [(dequantize(k8, kd).cpu(), dequantize(v8, vd).cpu())]
    ref_out, ref_lse = decode_oracle(q.float().cpu(), ref_caches, [sl.cpu()], None, None, causal)
    for splits in (None, 1, 3, 7):
        out, lse = dec.kernel_decode(q, pk, pv, sl, None, None, causal, scale, splits=splits, block_table=table,
                                     k_descale=kd, v_descale=vd)
        assert out.dtype == dtype and torch.isfinite(out).all()
        torch.testing.assert_close(out.float().cpu(), ref_out, **OUT_TOL)
        torch.testing.assert_close(lse.cpu(), ref_lse, **LSE_TOL)
        # bitwise the bf16 / fp16 kernel on the widened cache: unit descales, then powers of two
        w_out, w_lse = dec.kernel_decode(q, wk, wv, sl, None, None, causal, scale, splits=splits)
        u_out, u_lse = dec.kernel_decode(q, pk, pv, sl, None, None, causal, scale, splits=splits, block_table=table,
                                         k_descale=ones, v_descale=ones)
        assert torch.equal(u_out, w_out) and torch.equal(u_lse, w_lse), splits
        w_out, w_lse = dec.kernel_decode(q, wk, wv, sl, None, None, causal, scale * 2.0 ** -3, splits=splits)
        e_out, e_lse = dec.kernel_decode(q, pk, pv, sl, None, None, causal, scale, splits=splits, block_table=table,
                                         k_descale=p2k, v_descale=p2v)
        assert_scaled(e_out, w_out, 2.0 ** 5)
        assert torch.equal(e_lse, w_lse), splits

    # append (power-of-two descales): the kernel's bytes are torch's quantisation, and the result is the widened
    # kernel's over the widened cache plus the widened quantised rows
    kq, vq = quantize(k, p2k), quantize(v, p2v)
    if page_size is None:
        want_k, want_v = k8.clone(), v8.clone()
        for i in range(b):
            n0 = int(sl[i])
            m = min(sq, s_cap - n0)
            want_k[i, n0:n0 + m], want_v[i, n0:n0 + m] = kq[i, :m], vq[i, :m]
    else:
        want_k, want_v = append_to_pool(pk, table, sl, kq), append_to_pool(pv, table, sl, vq)
    e_out, e_lse = dec.kernel_decode(q, pk, pv, sl, k, v, causal, scale, splits=5, block_table=table, k_descale=p2k,
                                     v_descale=p2v)
    w_out, w_lse = dec.kernel_decode(q, wk, wv, sl, kq.to(dtype), vq.to(dtype), causal, scale * 2.0 ** -3, splits=5)
    torch.cuda.synchronize()
    assert torch.equal(bytes_of(pk), bytes_of(want_k)) and torch.equal(bytes_of(pv), bytes_of(want_v))
    assert_scaled(e_out, w_out, 2.0 ** 5)
    assert torch.equal(e_lse, w_lse)
    # after the append, attention only over the grown cache (descales that are not powers of two) against the oracle
    sl2 = (sl + sq).clamp(max=s_cap)
    out, lse = dec.kernel_decode(q, pk, pv, sl2, None, None, causal, scale, splits=3, block_table=table,
                                 k_descale=kd, v_descale=vd)
    logical_k = want_k if page_size is None else pk[table.clamp(min=0).long()].flatten(1, 2)
    logical_v = want_v if page_size is None else pv[table.clamp(min=0).long()].flatten(1, 2)
    ref_out, ref_lse = decode_oracle(q.float().cpu(), [(dequantize(logical_k, kd).cpu(),
                                                        dequantize(logical_v, vd).cpu())], [sl2.cpu()], None, None,
                                     causal)
    torch.testing.assert_close(out.float().cpu(), ref_out, **OUT_TOL)
    torch.testing.assert_close(lse.cpu(), ref_lse, **LSE_TOL)


def test_append_kernel_quantisation_bytes():
    """Saturation, +-inf, ties and subnormals through the append kernel, descale 0.37, both q dtypes, head dims."""
    vals = torch.tensor([1e6, -1e6, float("inf"), float("-inf"), 448 * 0.37, 460 * 0.37, 1e-3, -1e-3, 2.0 ** -9,
                         0.37 * 2.0 ** -10, 0.37 * 1.0625, 0.37 * 1.1875, 0.0, -0.0, 17.0, -3.3])
    for dtype in (torch.bfloat16, torch.float16):
        for d in (64, 128):
            b, sq, hkv = 2, 3, 2
            x = (vals.repeat(b * sq * hkv * d // 16) * torch.linspace(0.5, 2.0, b * sq * hkv * d)).view(b, sq, hkv, d)
            k, v = x.to(dtype).cuda(), (-x).to(dtype).cuda()
            q = torch.randn(b, sq, 2 * hkv, d, device="cuda", dtype=dtype)
            kc = torch.zeros(b, 256, hkv, d, device="cuda", dtype=E4M3)
            vc = torch.zeros_like(kc)
            ds = torch.full((b, hkv), 0.37, device="cuda")
            sl = torch.tensor([5, 254], dtype=torch.int32, device="cuda")  # the second drops a row past S_cap
            out = rfa.cp_flash_attn_with_kvcache(q, kc, vc, sl, k, v, append_rank=0, k_descale=ds, v_descale=ds)
            assert torch.isfinite(out).all()
            want_k, want_v = torch.zeros_like(kc), torch.zeros_like(vc)
            kq, vq = quantize(k, ds), quantize(v, ds)
            want_k[0, 5:8], want_v[0, 5:8] = kq[0], vq[0]
            want_k[1, 254:], want_v[1, 254:] = kq[1, :2], vq[1, :2]
            assert torch.equal(bytes_of(kc), bytes_of(want_k)), (dtype, d)
            assert torch.equal(bytes_of(vc), bytes_of(want_v)), (dtype, d)


def test_half_million_token_fp8_cache():
    torch.manual_seed(0)
    s, hq, d = 512 * 1024 + 77, 8, 128
    kc = torch.randn(1, s + 51, 1, d, device="cuda", dtype=torch.bfloat16)
    vc = torch.randn(1, s + 51, 1, d, device="cuda", dtype=torch.bfloat16)
    kd, vd = torch.tensor([[0.011]], device="cuda"), torch.tensor([[0.013]], device="cuda")
    k8, v8 = quantize(kc, kd), quantize(vc, vd)
    q = torch.randn(1, 2, hq, d, device="cuda", dtype=torch.bfloat16) * 3
    sl = torch.tensor([s], dtype=torch.int32, device="cuda")
    out, lse = rfa.cp_flash_attn_with_kvcache(q, k8, v8, sl, return_softmax_lse=True, k_descale=kd, v_descale=vd)
    kf, vf = dequantize(k8, kd)[0, :s, 0], dequantize(v8, vd)[0, :s, 0]
    sc = torch.einsum("thd,jd->htj", q[0].float(), kf) * d ** -0.5
    ref_lse = torch.logsumexp(sc, dim=-1)
    ref = torch.einsum("htj,jd->thd", torch.softmax(sc, dim=-1), vf)
    torch.testing.assert_close(out[0].float(), ref, **OUT_TOL)
    torch.testing.assert_close(lse[0], ref_lse, **LSE_TOL)


@pytest.mark.parametrize("page_size", [None, 16])
def test_cuda_graph_replay_after_lengths_and_descales_change(page_size):
    caches, lens, q, k, v = make_case(1, 2, 1, 32, 8, 128, 3008, seed=5, dtype=torch.bfloat16, device="cuda")
    kc, vc = caches[0]
    kd, vd = head_descales(2, 8, 0.02), head_descales(2, 8, 0.03)
    k8, v8 = quantize(kc.nan_to_num(0.0), kd), quantize(vc.nan_to_num(0.0), vd)
    table = None
    if page_size is not None:
        k8, v8, table = to_pool(k8, v8, torch.full((2,), 3008), page_size, seed=5)
    sl = torch.tensor([1000, 2500], dtype=torch.int32, device="cuda")
    kd_dev, vd_dev = kd.clone(), vd[0].clone()  # (B, Hkv) and (Hkv,) descales, read on the device at replay
    f = rfa.cp_flash_attn_with_kvcache
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        f(q, k8.clone(), v8.clone(), sl, k, v, append_rank=0, block_table=table, k_descale=kd_dev, v_descale=vd_dev)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = f(q, k8, v8, sl, k, v, append_rank=0, block_table=table, k_descale=kd_dev, v_descale=vd_dev)
    for lens, kmul, vmul in (([1000, 2500], 1.0, 1.0), ([1200, 1], 0.5, 3.0), ([0, 2999], 1.7, 0.37)):
        sl.copy_(torch.tensor(lens, dtype=torch.int32))
        kd_dev.copy_(kd * kmul)
        vd_dev.copy_(vd[0] * vmul)
        ek, ev = k8.clone(), v8.clone()
        g.replay()
        want = f(q, ek, ev, sl, k, v, append_rank=0, block_table=table, k_descale=kd_dev, v_descale=vd_dev)
        torch.cuda.synchronize()
        assert torch.equal(out, want), lens
        assert torch.equal(bytes_of(k8), bytes_of(ek)) and torch.equal(bytes_of(v8), bytes_of(ev))


def _two_gpu_case(rank, world):
    dev = f"cuda:{rank}"
    caches, lens, q, k, v = make_case(world, 3, 4, 16, 2, 128, 896, seed=11, dtype=torch.bfloat16, device=dev)
    ds = [(head_descales(3, 2, 0.3 + 0.2 * r, dev), head_descales(3, 2, 0.4 - 0.1 * r, dev)) for r in range(world)]
    f8 = [(quantize(kc, kd), quantize(vc, vd)) for (kc, vc), (kd, vd) in zip(caches, ds)]
    kd, vd = ds[rank]
    k8, v8 = f8[rank][0].clone(), f8[rank][1].clone()
    out, lse = rfa.cp_flash_attn_with_kvcache(q, k8, v8, lens[rank], k, v, append_rank=1, causal=True,
                                              return_softmax_lse=True, k_descale=kd, v_descale=vd)
    kd1, vd1 = ds[1]
    k_ref, v_ref = dequantize(quantize(k, kd1), kd1), dequantize(quantize(v, vd1), vd1)
    ref_out, ref_lse = decode_oracle(q.float().cpu(), [(dequantize(a, x).cpu(), dequantize(c, y).cpu())
                                                       for (a, c), (x, y) in zip(f8, ds)],
                                     [x.cpu() for x in lens], k_ref.cpu(), v_ref.cpu(), True)
    torch.testing.assert_close(out.float().cpu(), ref_out, **OUT_TOL)
    torch.testing.assert_close(lse.cpu(), ref_lse, **LSE_TOL)
    both = torch.cat([out.float().reshape(-1), lse.reshape(-1)])
    got = [torch.empty_like(both) for _ in range(world)]
    dist.all_gather(got, both)
    assert all(torch.equal(x, both) for x in got)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_fp8_bitwise_equal_and_match_oracle():
    run_distributed(_two_gpu_case, 2, backend="nccl")
