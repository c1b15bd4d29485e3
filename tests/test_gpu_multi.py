"""Multi-GPU context parallelism on real GPUs: the fused NVLink path (default) and the torch.distributed
fallback around the same kernels (RFA_B200_DISABLE_P2P=1), each against the dense fp32 oracle.
Needs >= 2 GPUs; run with `-m gpu`."""
import os

import pytest
import torch
import torch.distributed as dist

import ring_flash_attn_b200 as rfa
from ring_flash_attn_b200.ops.dense import attention_oracle, varlen_attention_oracle
from ring_flash_attn_b200.parallel import layouts
from dist_utils import run_distributed

pytestmark = pytest.mark.gpu


def _ngpu():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _close(got, want, name, rel=5e-2, abs_=2e-2):
    err = (got.float() - want.float()).abs().max().item()
    lim = rel * want.float().abs().max().item() + abs_
    assert err < lim, f"{name}: max err {err} > {lim}"


def _batch_case(rank, world, scheme, causal, p2p, hq, hkv, s_local, iters, d=128, dtype=torch.bfloat16):
    os.environ["RFA_B200_DISABLE_P2P"] = "0" if p2p else "1"
    dev = torch.device("cuda", rank)
    torch.manual_seed(0)
    s = s_local * world
    q = torch.randn(1, s, hq, d, device=dev)
    k = torch.randn(1, s, hkv, d, device=dev)
    v = torch.randn(1, s, hkv, d, device=dev)
    dout = torch.randn(1, s, hq, d, device=dev)
    for t in (q, k, v, dout):
        dist.broadcast(t, src=0)
    q, k, v, dout = (t.to(dtype) for t in (q, k, v, dout))
    rq, rk, rv = (t.float().requires_grad_(True) for t in (q, k, v))
    ref_out, ref_lse = attention_oracle(rq, rk, rv, causal)
    ref_out.backward(dout.float())
    shard = getattr(layouts, f"shard_{scheme}")
    prefix = {"ring": "ring", "zigzag": "zigzag_ring", "stripe": "stripe"}[scheme]
    fn = getattr(rfa, f"{prefix}_flash_attn_func")
    for _ in range(iters):  # several calls exercise epoch / staging-parity reuse
        lq, lk, lv = (shard(t, rank, world).detach().requires_grad_(True) for t in (q, k, v))
        out, lse, _ = fn(lq, lk, lv, causal=causal, return_attn_probs=True)
        out.backward(shard(dout, rank, world))
        torch.cuda.synchronize()
        _close(out, shard(ref_out, rank, world), "out")
        _close(lse, shard(ref_lse, rank, world, dim=2), "lse", rel=2e-3, abs_=2e-3)
        _close(lq.grad, shard(rq.grad, rank, world), "dq")
        _close(lk.grad, shard(rk.grad, rank, world), "dk")
        _close(lv.grad, shard(rv.grad, rank, world), "dv")


BATCH_CASES = [("zigzag", True, 4, 4, 512), ("zigzag", True, 4, 2, 600), ("ring", True, 4, 2, 384),
               ("ring", False, 2, 2, 300), ("stripe", True, 4, 1, 333)]


def _all_batch_cases(rank, world, p2p):
    # one process group for every case: spawning + NCCL init dominates the test time otherwise
    for scheme, causal, hq, hkv, s_local in BATCH_CASES:
        _batch_case(rank, world, scheme, causal, p2p, hq, hkv, s_local, 3 if p2p else 1)
    _batch_case(rank, world, "zigzag", True, p2p, 4, 2, 640, 2, d=64)  # kD = 64 instantiations, fused and fallback
    # fp16: the fused path's fp16 dK / dV reduction (reduce_dkv) and the fp16 delta / dq_finalize kernels
    _batch_case(rank, world, "zigzag", True, p2p, 4, 2, 512, 2, dtype=torch.float16)


@pytest.mark.parametrize("p2p", [True, False])
def test_batch_schemes_2gpu(p2p):
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    run_distributed(_all_batch_cases, 2, p2p, backend="nccl")


def _more_gpus(rank, world):
    _batch_case(rank, world, "zigzag", True, True, 4, 2, 512, 2)
    _batch_case(rank, world, "stripe", True, True, 4, 4, 300, 1)
    _batch_case(rank, world, "ring", False, True, 2, 1, 256, 1)
    for which in ("zigzag", "llama3"):
        _varlen_case(rank, world, which, True)


def _llama3_only(rank, world):
    _varlen_case(rank, world, "llama3", True)


@pytest.mark.parametrize("world", [8])
def test_llama3_fused_8gpu(world):
    if _ngpu() < world:
        pytest.skip(f"needs {world} GPUs")
    run_distributed(_llama3_only, world, backend="nccl")


@pytest.mark.parametrize("world", [4, 8])
def test_fused_more_gpus(world):
    if _ngpu() < world:
        pytest.skip(f"needs {world} GPUs")
    run_distributed(_more_gpus, world, backend="nccl")


def _varlen_case(rank, world, which, p2p):
    os.environ["RFA_B200_DISABLE_P2P"] = "0" if p2p else "1"
    dev = torch.device("cuda", rank)
    torch.manual_seed(0)
    unit = 2 * world
    cu = [0, 30 * unit, 130 * unit, 200 * unit]
    total = cu[-1]
    hq, hkv = 4, 2
    q = torch.randn(total, hq, 128, device=dev)
    k = torch.randn(total, hkv, 128, device=dev)
    v = torch.randn(total, hkv, 128, device=dev)
    dout = torch.randn(total, hq, 128, device=dev)
    for t in (q, k, v, dout):
        dist.broadcast(t, src=0)
    q, k, v, dout = (t.to(torch.bfloat16) for t in (q, k, v, dout))
    cu_t = torch.tensor(cu, dtype=torch.int32, device=dev)
    rq, rk, rv = (t.float().requires_grad_(True) for t in (q, k, v))
    ref_out, ref_lse = varlen_attention_oracle(rq, rk, rv, cu_t.cpu(), True)
    ref_out.backward(dout.float())
    if which == "llama3":
        sh = lambda t: layouts.shard_llama3(t, rank, world)  # noqa: E731
    elif which == "ring":
        sh = lambda t: layouts.shard_ring_varlen(t, cu, rank, world)  # noqa: E731
    else:
        sh = lambda t: layouts.shard_zigzag_varlen(t, cu, rank, world)  # noqa: E731
    for _ in range(2):
        lq, lk, lv = (sh(t).detach().requires_grad_(True) for t in (q, k, v))
        if which == "llama3":
            cq, ck, mq, mk, ks = rfa.llama3_flash_attn_prepare_cu_seqlens(cu_t, True, rank, world)
            cq, ck = cq.clone(), ck.clone()  # plain tensors: the fused path must not depend on prepare()'s objects
            out, lse, _ = rfa.llama3_flash_attn_varlen_func(lq, lk, lv, cq, ck, mq, mk, heads_k_stride=1,
                                                          local_k_slice=ks, causal=True, return_attn_probs=True)
        else:
            local_cu = cu_t // world
            fn = rfa.ring_flash_attn_varlen_func if which == "ring" else rfa.zigzag_ring_flash_attn_varlen_func
            out, lse, _ = fn(lq, lk, lv, local_cu, int((local_cu[1:] - local_cu[:-1]).max()), causal=True,
                             return_attn_probs=True)
        out.backward(sh(dout))
        torch.cuda.synchronize()
        _close(out, sh(ref_out), "out")
        _close(lse, sh(ref_lse.transpose(0, 1)).transpose(0, 1), "lse", rel=2e-3, abs_=2e-3)
        _close(lq.grad, sh(rq.grad), "dq")
        _close(lk.grad, sh(rk.grad), "dk")
        _close(lv.grad, sh(rv.grad), "dv")


def _all_varlen_cases(rank, world, p2p):
    for which in ("ring", "zigzag", "llama3"):
        _varlen_case(rank, world, which, p2p)


@pytest.mark.parametrize("p2p", [True, False])
def test_varlen_schemes_2gpu(p2p):
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    run_distributed(_all_varlen_cases, 2, p2p, backend="nccl")


def _zigzag_llama3_case(rank, world, p2p):
    os.environ["RFA_B200_DISABLE_P2P"] = "0" if p2p else "1"
    dev = torch.device("cuda", rank)
    torch.manual_seed(0)
    T, H, HK = 1024 * world, 8, 2
    cu = torch.tensor([0, 777, 900, T // 2 + 5, T], dtype=torch.int32)
    q = torch.randn(T, H, 128, device=dev)
    k = torch.randn(T, HK, 128, device=dev)
    v = torch.randn(T, HK, 128, device=dev)
    dout = torch.randn(T, H, 128, device=dev)
    for t in (q, k, v, dout):
        dist.broadcast(t, src=0)
    q, k, v, dout = (t.to(torch.bfloat16) for t in (q, k, v, dout))
    rq, rk, rv = (t.float().requires_grad_(True) for t in (q, k, v))
    ref, ref_lse = varlen_attention_oracle(rq, rk, rv, cu, True)
    ref.backward(dout.float())
    sh = lambda x: layouts.shard_zigzag_llama3(x, rank, world)  # noqa: E731
    for _ in range(2):
        lq, lk, lv = (sh(t).detach().requires_grad_(True) for t in (q, k, v))
        out, lse, _ = rfa.zigzag_llama3_flash_attn_varlen_func(lq, lk, lv, cu.to(dev), causal=True,
                                                               return_attn_probs=True)
        out.backward(sh(dout))
        torch.cuda.synchronize()
        _close(out, sh(ref), "out")
        _close(lse, sh(ref_lse.transpose(0, 1)).transpose(0, 1), "lse", rel=2e-3, abs_=2e-3)
        _close(lq.grad, sh(rq.grad), "dq")
        _close(lk.grad, sh(rk.grad), "dk")
        _close(lv.grad, sh(rv.grad), "dv")


@pytest.mark.parametrize("p2p", [True, False])
def test_zigzag_llama3_2gpu(p2p):
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    run_distributed(_zigzag_llama3_case, 2, p2p, backend="nccl")


def _window_fused_case(rank, world, p2p):
    os.environ.pop("RFA_B200_WINDOW_KERNEL", None)  # the kWindow kernel variants are the default
    os.environ["RFA_B200_DISABLE_P2P"] = "0" if p2p else "1"
    dev = torch.device("cuda", rank)
    torch.manual_seed(0)
    S, H, HK, d = 1024 * world, 8, 2, 128
    for scheme, window in (("zigzag", (300, 0)), ("ring", (1500, 0)), ("stripe", (77, 0))):
        q = torch.randn(1, S, H, d, device=dev).to(torch.bfloat16)
        kv = torch.randn(1, S, 2, HK, d, device=dev).to(torch.bfloat16)
        dout = torch.randn(1, S, H, d, device=dev).to(torch.bfloat16)
        for t in (q, kv, dout):
            dist.broadcast(t, src=0)
        rq, rkv = q.float().requires_grad_(True), kv.float().requires_grad_(True)
        ref, _ = attention_oracle(rq, rkv[:, :, 0], rkv[:, :, 1], True, window_size=window)
        ref.backward(dout.float())
        shard = getattr(layouts, f"shard_{scheme}")
        lq = shard(q, rank, world).detach().requires_grad_(True)
        lkv = shard(kv, rank, world).detach().requires_grad_(True)
        fn = getattr(rfa, {"ring": "ring", "zigzag": "zigzag_ring", "stripe": "stripe"}[scheme] + "_flash_attn_kvpacked_func")
        for _ in range(2):  # second call exercises buffer reuse / epochs
            lq.grad = lkv.grad = None
            out = fn(lq, lkv, causal=True, window_size=window)
            out.backward(shard(dout, rank, world))
        torch.testing.assert_close(out.float(), shard(ref, rank, world), atol=2e-2, rtol=2e-2)
        gq, gkv = shard(rq.grad, rank, world), shard(rkv.grad, rank, world)
        assert (lq.grad.float() - gq).abs().max().item() < 5e-2 * gq.abs().max().item() + 2e-2
        assert (lkv.grad.float() - gkv).abs().max().item() < 5e-2 * gkv.abs().max().item() + 2e-2


@pytest.mark.parametrize("p2p", [True, False])
def test_sliding_window_kernels_2gpu(p2p):
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    run_distributed(_window_fused_case, 2, p2p, backend="nccl")


def _subgroup_fused_case(rank, world):
    """Two fused context-parallel groups ({0,1} and {2,3}) side by side: separate peer contexts, staging buffers and
    signal pads per group."""
    os.environ["RFA_B200_DISABLE_P2P"] = "0"
    groups = [dist.new_group([0, 1]), dist.new_group([2, 3])]
    g = groups[rank // 2]
    grank, gworld = dist.get_rank(g), 2
    dev = torch.device("cuda", rank)
    torch.manual_seed(100 + rank // 2)
    qkv = torch.randn(1, 2048, 3, 4, 128, device=dev)
    dist.broadcast(qkv, src=(rank // 2) * 2, group=g)
    qkv = qkv.to(torch.bfloat16)
    ref, _ = attention_oracle(qkv[:, :, 0].float(), qkv[:, :, 1].float(), qkv[:, :, 2].float(), True)
    for _ in range(3):
        local = layouts.shard_zigzag(qkv, grank, gworld).detach().requires_grad_(True)
        out = rfa.zigzag_ring_flash_attn_qkvpacked_func(local, causal=True, group=g)
        out.sum().backward()
        torch.cuda.synchronize()
        _close(out, layouts.shard_zigzag(ref, grank, gworld), "out")


def test_fused_subgroups_4gpu():
    if _ngpu() < 4:
        pytest.skip("needs 4 GPUs")
    run_distributed(_subgroup_fused_case, 4, backend="nccl")


def _compiled_case(rank, world):
    """Every scheme once under torch.compile(fullgraph=True) on the fused path, against eager."""
    os.environ["RFA_B200_DISABLE_P2P"] = "0"
    dev = torch.device("cuda", rank)
    torch.manual_seed(3)
    s_l, h = 1024, 4
    qkv = torch.randn(1, s_l, 3, h, 128, device=dev).to(torch.bfloat16)
    dout = torch.randn(1, s_l, h, 128, device=dev).to(torch.bfloat16)
    cu_local = torch.tensor([0, 256, s_l], dtype=torch.int32)
    cu_global = torch.tensor([0, 300 * world, s_l * world], dtype=torch.int32)
    cq, ck, mq, mk, ks = rfa.llama3_flash_attn_prepare_cu_seqlens(cu_global, True, rank, world)

    def f(x):
        a = rfa.zigzag_ring_flash_attn_qkvpacked_func(x, causal=True)
        b = rfa.stripe_flash_attn_qkvpacked_func(x, causal=True)
        c = rfa.zigzag_ring_flash_attn_varlen_qkvpacked_func(x[0], cu_local, 768, causal=True)
        d = rfa.llama3_flash_attn_varlen_qkvpacked_func(x[0], cq, ck, mq, mk, heads_k_stride=1, local_k_slice=ks,
                                                        causal=True)
        return a + b + (c + d).unsqueeze(0)

    x = qkv.detach().requires_grad_(True)
    ref = f(x)
    ref.backward(dout)
    g_ref = x.grad.clone()
    y = qkv.detach().requires_grad_(True)
    out = torch.compile(f, backend="aot_eager", fullgraph=True)(y)
    out.backward(dout)
    torch.cuda.synchronize()
    torch.testing.assert_close(out.float(), ref.float(), atol=1e-2, rtol=1e-2)
    _close(y.grad, g_ref, "compiled grad", rel=2e-2, abs_=1e-2)


def test_compiled_schemes_2gpu():
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    run_distributed(_compiled_case, 2, backend="nccl")


def _headline_shape(rank, world):
    """The benchmark shape itself (zigzag qkvpacked, 4096 local tokens, 32 heads of 128, fwd + bwd) against the fp32
    oracle on sampled rows and heads (utils/verify.py) - a dense oracle of 32768 x 32768 x 32 does not fit.  Same
    check as ``bench.py --check``; here it fails the test tier instead of printing a flag."""
    from ring_flash_attn_b200.utils.verify import sampled_check

    os.environ["RFA_B200_DISABLE_P2P"] = "0"
    dev = torch.device("cuda", rank)
    torch.manual_seed(100 + rank)  # every rank owns different data: the oracle gathers the shards
    s_local, h = 4096, 32
    for _ in range(2):  # second call: other staging parity, epochs advanced
        qkv = torch.randn(1, s_local, 3, h, 128, device=dev).to(torch.bfloat16).requires_grad_(True)
        dout = torch.randn(1, s_local, h, 128, device=dev).to(torch.bfloat16)
        out, lse, _ = rfa.zigzag_ring_flash_attn_qkvpacked_func(qkv, causal=True, return_attn_probs=True)
        out.backward(dout)
        g = qkv.grad[0]
        x = qkv.detach()[0]
        res = sampled_check("zigzag", x[:, 0], x[:, 1], x[:, 2], dout[0], out.detach()[0], lse[0], g[:, 0], g[:, 1],
                            g[:, 2], kv_heads=[0, 13, 31])
        assert res["ok"], res


@pytest.mark.parametrize("world", [2, 8])
def test_headline_shape_sampled_oracle(world):
    if _ngpu() < world:
        pytest.skip(f"needs {world} GPUs")
    run_distributed(_headline_shape, world, backend="nccl")


def _llama3_strict_groups(rank, world):
    """heads_k_stride honoured literally (RFA_B200_LLAMA3_HEAD_GROUPS=strict): one fused launch per kv head, staging
    sized for one head; also a hand-built (cloned) cu_seqlens - no attribute of prepare()'s tensors is needed."""
    os.environ["RFA_B200_LLAMA3_HEAD_GROUPS"] = "strict"
    try:
        _varlen_case(rank, world, "llama3", True)
    finally:
        os.environ.pop("RFA_B200_LLAMA3_HEAD_GROUPS", None)


def test_llama3_head_groups_2gpu():
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    run_distributed(_llama3_strict_groups, 2, backend="nccl")


def _ring_schemes_head_groups(rank, world):
    """A staging budget smaller than one launch over all heads (RFA_B200_STAGE_BUDGET_MB=0): zigzag / ring / stripe
    run one fused launch per kv head, like llama3's head-group passes."""
    from ring_flash_attn_b200.ops import cuda_ext

    os.environ["RFA_B200_STAGE_BUDGET_MB"] = "0"
    try:
        before = cuda_ext.launch_counter().value
        _batch_case(rank, world, "zigzag", True, True, 4, 2, 512, 2)
        # per call: (fwd + delta + bwd + reduce + dq_finalize) x 2 head groups
        assert cuda_ext.launch_counter().value - before >= 2 * 2 * 4
        _batch_case(rank, world, "stripe", True, True, 4, 4, 384, 1)
        _batch_case(rank, world, "ring", False, True, 4, 2, 256, 1)
    finally:
        os.environ.pop("RFA_B200_STAGE_BUDGET_MB", None)


def test_ring_schemes_head_groups_2gpu():
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    run_distributed(_ring_schemes_head_groups, 2, backend="nccl")


def _fp8_block_scaled_fused(rank, world):
    """stripe attention on block-scaled e4m3 shards through the fused launch: e4m3 K/V rows on the NVLink wire, the
    sources' descale tables gathered on the device."""
    from ring_flash_attn_b200.ops import cuda_ext
    from ring_flash_attn_b200.utils import fp8

    os.environ["RFA_B200_DISABLE_P2P"] = "0"
    dev = torch.device("cuda", rank)
    torch.manual_seed(5)
    B, S, H = 2, 1024 * world, 4
    qkv = torch.randn(B, S, 3, H, 128, device=dev) * (1.0 + 3.0 * torch.rand(B, S, 1, 1, 1, device=dev))
    dist.broadcast(qkv, src=0)
    local = layouts.shard_stripe(qkv, rank, world)
    q8, scale = fp8.quantize_blockwise(local, [1, 128, 1, 1, 0])
    deq = fp8.dequantize(q8, scale, torch.float32)
    parts = [torch.empty_like(deq) for _ in range(world)]
    dist.all_gather(parts, deq)
    full = layouts.unshard("stripe", parts)
    ref, ref_lse = attention_oracle(full[:, :, 0], full[:, :, 1], full[:, :, 2], True)
    for _ in range(2):
        before = cuda_ext.launch_counter().value
        out, lse, _ = rfa.stripe_flash_attn_qkvpacked_func(q8, causal=True, descale=scale, return_attn_probs=True)
        torch.cuda.synchronize()
        assert cuda_ext.launch_counter().value == before + 1, "block-scaled fp8 did not take the fused fp8 launch"
        want = layouts.shard_stripe(ref, rank, world)
        err = (out.float() - want).abs().max().item()
        assert err < 6e-2 * want.abs().max().item() + 2e-2, err
        torch.testing.assert_close(lse, layouts.shard_stripe(ref_lse, rank, world, dim=2), atol=2e-2, rtol=2e-2)


def test_fp8_block_scaled_fused_2gpu():
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    run_distributed(_fp8_block_scaled_fused, 2, backend="nccl")
