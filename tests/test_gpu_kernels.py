"""sm_90a kernels through the public API against the fp64 oracle with a precision-matched error bound
(``tests/kernel_oracle.py``; the block-level sweep of every instantiation is ``test_gpu_kernel_accuracy.py``).
Run with -m gpu on an H100."""
import itertools

import pytest
import torch

import kernel_oracle as KO
import ring_flash_attn_b200 as rfa
from ring_flash_attn_b200.ops.dense import attention_oracle, varlen_attention_oracle

pytestmark = pytest.mark.gpu
DTYPES = (torch.bfloat16, torch.float16)  # the world-1 API tests run both: the fp16 delta / dq_finalize / dK-dV paths


@pytest.fixture(autouse=True)
def _exact_fp32_matmul():
    """The precision-matched reference needs true fp32 GEMMs."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


def _flat(x):
    """(B, S, ...) -> (B * S, ...)."""
    return x.reshape(-1, *x.shape[2:])


def _flat_lse(lse):
    """(B, H, S) -> (H, B * S)."""
    return lse.permute(1, 0, 2).reshape(lse.shape[1], -1)


def _batch_cu(b, s):
    return list(range(0, (b + 1) * s, s))


def _ext():
    from ring_flash_attn_b200.ops import cuda_ext

    return cuda_ext.load()


def test_extension_is_loaded_and_native():
    C = _ext()
    assert hasattr(C, "attn_fwd") and hasattr(C, "attn_bwd")
    assert torch.cuda.get_device_capability()[0] == 9, "these tests expect a Hopper (sm_90) GPU"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("sq,sk,hq,hkv,diag", [
    (128, 128, 1, 1, None), (128, 128, 1, 1, 0), (256, 256, 2, 1, 0), (384, 512, 4, 2, 128),
    (200, 333, 2, 2, 40), (77, 50, 1, 1, None), (300, 300, 2, 2, -1), (512, 1024, 2, 1, None),
])
def test_fwd_block_kernel(dtype, sq, sk, hq, hkv, diag):
    """One chunk x one segment through the wgmma forward kernel (head_dim 128) against the fp64 oracle.  These shapes
    are also rows of the geometry list that test_gpu_kernel_accuracy.py runs on every instantiation."""
    KO.run_forward(KO.single_segment(sq, sk, hq, hkv, diag), 128, dtype, False, "randn", "cuda")


@pytest.mark.parametrize("sq,sk,hq,hkv,diag", [
    (128, 128, 1, 1, None), (128, 128, 1, 1, 0), (256, 256, 2, 1, 0), (384, 512, 4, 2, 128),
    (200, 333, 2, 2, 40), (77, 50, 1, 1, None), (300, 300, 2, 2, -1),
])
def test_bwd_block_kernel(sq, sk, hq, hkv, diag):
    """The backward kernel (head_dim 128) on the same shapes, lse / delta from the fp64 oracle, in both dtypes and
    with fp32 and model-dtype dK / dV stores."""
    for dtype in DTYPES:
        for dkv_dtype in (torch.float32, dtype):
            KO.run_backward(KO.single_segment(sq, sk, hq, hkv, diag), 128, dtype, False, "randn", "cuda",
                            dkv_dtype=dkv_dtype)


def test_delta_kernel():
    """``bwd_delta_kernel`` and ``dq_finalize`` at bf16 / head_dim 128 (both dtypes and head sizes:
    test_gpu_kernel_accuracy.py::test_delta_and_dq_finalize)."""
    KO.run_delta_and_dq_finalize(torch.bfloat16, 128, "cuda")


def _qkv_case(name, qkv, dout, out, lse, cu, causal=True, window=(-1, -1)):
    """Check a qkv-packed call ((B, S, 3, H, D) or (T, 3, H, D)) after its backward."""
    x, g = qkv.detach(), qkv.grad
    if x.dim() == 5:
        x, g, dout, out = _flat(x), _flat(g), _flat(dout), _flat(out)
        lse = None if lse is None else _flat_lse(lse)
    ref64, reflp = KO.api_reference(x[:, 0], x[:, 1], x[:, 2], dout, cu, causal, window)
    got = dict(out=out.detach(), dq=g[:, 0], dk=g[:, 1], dv=g[:, 2])
    if lse is not None:
        got["lse"] = lse
    KO.assert_api(name, got, ref64, reflp)


def _kv_case(name, q, kv, dout, out, lse, cu, causal=True, window=(-1, -1)):
    """Check a kv-packed call (q (B, S, H, D) / kv (B, S, 2, Hkv, D), or without the batch dim) after its backward."""
    xq, xkv, gq, gkv = q.detach(), kv.detach(), q.grad, kv.grad
    if xq.dim() == 4:
        xq, xkv, gq, gkv, dout, out = _flat(xq), _flat(xkv), _flat(gq), _flat(gkv), _flat(dout), _flat(out)
        lse = None if lse is None else _flat_lse(lse)
    ref64, reflp = KO.api_reference(xq, xkv[:, 0], xkv[:, 1], dout, cu, causal, window)
    got = dict(out=out.detach(), dq=gq, dk=gkv[:, 0], dv=gkv[:, 1])
    if lse is not None:
        got["lse"] = lse
    KO.assert_api(name, got, ref64, reflp)


@pytest.mark.parametrize("fn_name", ["ring_flash_attn_qkvpacked_func", "zigzag_ring_flash_attn_qkvpacked_func",
                                     "stripe_flash_attn_qkvpacked_func"])
def test_world1_api_matches_oracle(fn_name):
    """world_size 1 through the public API: every scheme is causal flash attention (fwd + bwd)."""
    for dtype in DTYPES:
        torch.manual_seed(0)
        qkv = (torch.randn(2, 640, 3, 4, 128, device="cuda") * 0.7).to(dtype).requires_grad_(True)
        dout = torch.randn(2, 640, 4, 128, device="cuda").to(dtype)
        out, lse, _ = getattr(rfa, fn_name)(qkv, causal=True, return_attn_probs=True)
        out.backward(dout)
        _qkv_case(f"{fn_name} {dtype}", qkv, dout, out, lse, _batch_cu(2, 640))


def test_world1_gqa_kvpacked_noncausal():
    for dtype in DTYPES:
        torch.manual_seed(0)
        q = torch.randn(1, 500, 8, 128, device="cuda").to(dtype).requires_grad_(True)
        kv = torch.randn(1, 500, 2, 2, 128, device="cuda").to(dtype).requires_grad_(True)
        dout = torch.randn(1, 500, 8, 128, device="cuda").to(dtype)
        out = rfa.ring_flash_attn_kvpacked_func(q, kv, causal=False)
        out.backward(dout)
        _kv_case(f"gqa kvpacked {dtype}", q, kv, dout, out, None, [0, 500], causal=False)


def test_world1_varlen_and_llama3():
    cu = torch.tensor([0, 120, 1248, 2000], dtype=torch.int32, device="cuda")
    total = 2000
    for dtype, which in itertools.product(DTYPES, ("ring", "zigzag", "llama3")):
        torch.manual_seed(0)
        qkv = torch.randn(total, 3, 4, 128, device="cuda").to(dtype).requires_grad_(True)
        dout = torch.randn(total, 4, 128, device="cuda").to(dtype)
        if which == "llama3":
            cq, ck, mq, mk, ks = rfa.llama3_flash_attn_prepare_cu_seqlens(cu, True, 0, 1)
            out, lse, _ = rfa.llama3_flash_attn_varlen_qkvpacked_func(
                qkv, cq, ck, mq, mk, heads_k_stride=1, local_k_slice=ks, causal=True, return_attn_probs=True)
        else:
            fn = rfa.ring_flash_attn_varlen_qkvpacked_func if which == "ring" \
                else rfa.zigzag_ring_flash_attn_varlen_qkvpacked_func
            out, lse, _ = fn(qkv, cu, 1128, causal=True, return_attn_probs=True)
        out.backward(dout)
        _qkv_case(f"{which} {dtype}", qkv, dout, out, lse, cu.tolist())


def test_lse_layout_kernels_match_torch():
    from ring_flash_attn_b200.ops import lse_layout

    cu = torch.tensor([0, 5, 133, 400], dtype=torch.int32, device="cuda")
    lse = torch.randn(3, 4, 267, device="cuda")
    flat = lse_layout.flatten_varlen_lse(lse, cu)
    assert torch.equal(flat, lse_layout._flatten_torch(lse, cu))
    packed = torch.randn(400, 4, 1, device="cuda")
    un = lse_layout.unflatten_varlen_lse(packed, cu, 267)
    ref = lse_layout._unflatten_torch(packed, cu, 267)
    for b, (a, e) in enumerate(zip([0, 5, 133], [5, 133, 400])):
        assert torch.equal(un[b, :, : e - a], ref[b, :, : e - a])


def test_world1_sliding_window_on_device():
    """window_size on a GPU tensor: the plan carries the lower bound and (until the kernels learn it) the
    dense torch blocks run on the device - results must still match the oracle."""
    torch.manual_seed(0)
    q = torch.randn(1, 384, 4, 128, device="cuda").to(torch.bfloat16).requires_grad_(True)
    kv = torch.randn(1, 384, 2, 2, 128, device="cuda").to(torch.bfloat16).requires_grad_(True)
    dout = torch.randn(1, 384, 4, 128, device="cuda").to(torch.bfloat16)
    rq, rkv = q.detach().float().requires_grad_(True), kv.detach().float().requires_grad_(True)
    ref_out, _ = attention_oracle(rq, rkv[:, :, 0], rkv[:, :, 1], True, window_size=(100, 0))
    ref_out.backward(dout.float())
    out = rfa.zigzag_ring_flash_attn_kvpacked_func(q, kv, causal=True, window_size=(100, 0))
    out.backward(dout)
    torch.testing.assert_close(out.float(), ref_out, atol=2e-2, rtol=2e-2)
    assert (q.grad.float() - rq.grad).abs().max().item() < 5e-2 * rq.grad.abs().max().item() + 2e-2
    assert (kv.grad.float() - rkv.grad).abs().max().item() < 5e-2 * rkv.grad.abs().max().item() + 2e-2


@pytest.mark.parametrize("d", [32, 64, 96])
def test_world1_small_head_dim_runs_on_kernels(d):
    """head_dim 64 has its own kernel instantiations (template parameter kD); other sizes below 128 are zero-padded
    to the next instantiated size (parallel/api.py:_pad_head_dim) - still our launches (counter moves), still the
    oracle's numbers with the caller's 1/sqrt(d) scale."""
    from ring_flash_attn_b200.ops import cuda_ext

    for dtype in DTYPES:
        torch.manual_seed(0)
        qkv = (torch.randn(1, 512, 3, 4, d, device="cuda") * 0.8).to(dtype).requires_grad_(True)
        dout = torch.randn(1, 512, 4, d, device="cuda").to(dtype)
        before = cuda_ext.launch_counter().value
        out = rfa.zigzag_ring_flash_attn_qkvpacked_func(qkv, causal=True)
        out.backward(dout)
        assert cuda_ext.launch_counter().value > before
        assert out.shape == (1, 512, 4, d)
        _qkv_case(f"head_dim {d} {dtype}", qkv, dout, out, None, [0, 512])


def test_world1_zigzag_llama3():
    """Flat zigzag layout over packed documents of arbitrary lengths (beyond the reference): same kernels, the
    layout only changes the work tables."""
    T, H, HK = 2048, 8, 2
    cu = torch.tensor([0, 333, 420, 1500, T], dtype=torch.int32, device="cuda")
    for dtype in DTYPES:
        torch.manual_seed(0)
        q = torch.randn(T, H, 128, device="cuda").to(dtype).requires_grad_(True)
        kv = torch.randn(T, 2, HK, 128, device="cuda").to(dtype).requires_grad_(True)
        dout = torch.randn(T, H, 128, device="cuda").to(dtype)
        out, lse, _ = rfa.zigzag_llama3_flash_attn_varlen_kvpacked_func(q, kv, cu, causal=True,
                                                                        return_attn_probs=True)
        out.backward(dout)
        _kv_case(f"zigzag llama3 {dtype}", q, kv, dout, out, lse, cu.tolist())


@pytest.mark.parametrize("fn_name,causal,window", [
    ("zigzag_ring_flash_attn_kvpacked_func", True, (100, 0)),
    ("ring_flash_attn_kvpacked_func", True, (700, 0)),
    ("stripe_flash_attn_kvpacked_func", True, (33, 0)),
    ("ring_flash_attn_kvpacked_func", False, (150, 60)),
    ("ring_flash_attn_kvpacked_func", False, (-1, 200)),
])
def test_sliding_window_kernels(monkeypatch, fn_name, causal, window):
    """kWindow variants of both kernels (the default for windowed plans) against the windowed oracle."""
    from ring_flash_attn_b200.ops import cuda_ext

    monkeypatch.delenv("RFA_B200_WINDOW_KERNEL", raising=False)
    for dtype in DTYPES:
        torch.manual_seed(0)
        q = torch.randn(2, 1000, 8, 128, device="cuda").to(dtype).requires_grad_(True)
        kv = torch.randn(2, 1000, 2, 2, 128, device="cuda").to(dtype).requires_grad_(True)
        dout = torch.randn(2, 1000, 8, 128, device="cuda").to(dtype)
        before = cuda_ext.launch_counter().value
        out, lse, _ = getattr(rfa, fn_name)(q, kv, causal=causal, window_size=window, return_attn_probs=True)
        out.backward(dout)
        assert cuda_ext.launch_counter().value >= before + 2, "windowed call did not reach the kernels"
        _kv_case(f"{fn_name} {window} {dtype}", q, kv, dout, out, lse, _batch_cu(2, 1000), causal, window)


def _fp8_check(name, qd, kvd, out, lse):
    """fp8 forward (B, S, ...) against the oracle on the dequantised inputs, P and out rounded to bf16."""
    b, s = qd.shape[:2]
    ref64, reflp = KO.api_reference(_flat(qd), _flat(kvd[:, :, 0]), _flat(kvd[:, :, 1]), None, _batch_cu(b, s), True,
                                    dtype=torch.bfloat16)
    KO.assert_api(name, dict(out=_flat(out), lse=_flat_lse(lse)), ref64, reflp, fp8=True)


@pytest.mark.parametrize("per_head", [False, True])
def test_fp8_forward_kernel(monkeypatch, per_head):
    """Default for per-tensor / per-head descales: e4m3 q/k/v go straight into the forward kernel (e4m3 wgmma for Q K^T, V widened
    to bf16 in shared memory for P V); compared with the oracle on the dequantised tensors at fp8 tolerance."""
    from ring_flash_attn_b200.ops import cuda_ext
    from ring_flash_attn_b200.utils import fp8

    monkeypatch.delenv("RFA_B200_FP8_KERNEL", raising=False)
    torch.manual_seed(0)
    q = torch.randn(1, 900, 8, 128, device="cuda") * 1.5
    kv = torch.randn(1, 900, 2, 2, 128, device="cuda") * 1.5
    if per_head:
        q8, dq = fp8.quantize_blockwise(q, [0, 0, 1, 0])
        kv8, dkv = fp8.quantize_blockwise(kv, [0, 0, 1, 1, 0])
    else:
        q8, dq = fp8.quantize_blockwise(q, [0, 0, 0, 0])
        kv8, dkv = fp8.quantize_blockwise(kv, [0, 0, 1, 0, 0])
    qd = fp8.dequantize(q8, dq, torch.float32)
    kvd = fp8.dequantize(kv8, dkv, torch.float32)
    before = cuda_ext.launch_counter().value
    out, lse, _ = rfa.zigzag_ring_flash_attn_kvpacked_func(q8, kv8, causal=True, descale=(dq, dkv),
                                                           return_attn_probs=True)
    assert cuda_ext.launch_counter().value == before + 1 and out.dtype == torch.bfloat16
    _fp8_check("fp8 per-head" if per_head else "fp8 per-tensor", qd, kvd, out, lse)


def test_single_token_documents():
    """Degenerate packing (documents of one token, chunks of one row): covered by the CPU table tests, run on hardware
    with the other round-2 checks."""
    torch.manual_seed(0)
    T, H, HK = 1024, 4, 2
    cu = torch.tensor([0, 1, 2, 333, 334, 700, T], dtype=torch.int32, device="cuda")
    q = torch.randn(T, H, 128, device="cuda").to(torch.bfloat16).requires_grad_(True)
    kv = torch.randn(T, 2, HK, 128, device="cuda").to(torch.bfloat16).requires_grad_(True)
    dout = torch.randn(T, H, 128, device="cuda").to(torch.bfloat16)
    rq, rkv = q.detach().float().requires_grad_(True), kv.detach().float().requires_grad_(True)
    ref, _ = varlen_attention_oracle(rq, rkv[:, 0], rkv[:, 1], cu.cpu(), True)
    ref.backward(dout.float())
    out = rfa.zigzag_llama3_flash_attn_varlen_kvpacked_func(q, kv, cu, causal=True)
    out.backward(dout)
    torch.testing.assert_close(out.float(), ref, atol=2e-2, rtol=2e-2)
    assert (q.grad.float() - rq.grad).abs().max().item() < 5e-2 * rq.grad.abs().max().item() + 2e-2
    assert (kv.grad.float() - rkv.grad).abs().max().item() < 5e-2 * rkv.grad.abs().max().item() + 2e-2


@pytest.mark.parametrize("backend", ["aot_eager", "inductor"])
def test_compile_fullgraph_world1(backend):
    """torch.compile(fullgraph=True) through the public functions on the GPU: the CP op is a torch.library custom op
    (parallel/ops.py), so there is no graph break; the compiled function must launch OUR kernels and match eager.
    Mirrors the reference's `compile` test mode (/root/reference/test/test.sh:23-25)."""
    from ring_flash_attn_b200.ops import cuda_ext

    torch.manual_seed(0)
    qkv = torch.randn(1, 1024, 3, 4, 128, device="cuda").to(torch.bfloat16).requires_grad_(True)
    dout = torch.randn(1, 1024, 4, 128, device="cuda").to(torch.bfloat16)
    cu = torch.tensor([0, 300, 1024], dtype=torch.int32)  # CPU cu_seqlens: no device sync inside the op

    def f(x):
        a = rfa.zigzag_ring_flash_attn_qkvpacked_func(x, causal=True)
        b = rfa.ring_flash_attn_varlen_qkvpacked_func(x[0], cu, 724, causal=True)
        return a + b.unsqueeze(0)

    ref = f(qkv)
    ref.backward(dout)
    g_ref = qkv.grad.clone()
    qkv.grad = None
    try:
        cf = torch.compile(f, backend=backend, fullgraph=True)
        before = cuda_ext.launch_counter().value
        out = cf(qkv)
    except Exception as e:  # noqa: BLE001
        if backend == "inductor":
            pytest.skip(f"inductor toolchain unavailable on this box: {type(e).__name__}")
        raise
    out.backward(dout)
    assert cuda_ext.launch_counter().value >= before + 6, "compiled function did not reach the sm_90a kernels"
    torch.testing.assert_close(out.float(), ref.float(), atol=1e-2, rtol=1e-2)
    assert (qkv.grad.float() - g_ref.float()).abs().max().item() < 2e-2 * g_ref.float().abs().max().item() + 1e-2


@pytest.mark.parametrize("window", [(-1, -1), (200, 0)])
def test_head_dim_64_native(window):
    """kD = 64 instantiations of both kernels: GQA, packed varlen documents with ragged tiles, sliding window."""
    from ring_flash_attn_b200.ops import cuda_ext

    torch.manual_seed(1)
    T, H, HK, d = 1500, 8, 2, 64
    cu = torch.tensor([0, 100, 101, 900, T], dtype=torch.int32, device="cuda")
    for dtype in DTYPES:
        q = torch.randn(T, H, d, device="cuda").to(dtype).requires_grad_(True)
        kv = torch.randn(T, 2, HK, d, device="cuda").to(dtype).requires_grad_(True)
        dout = torch.randn(T, H, d, device="cuda").to(dtype)
        before = cuda_ext.launch_counter().value
        out, lse, _ = rfa.ring_flash_attn_varlen_kvpacked_func(q, kv, cu, 799, causal=True, window_size=window,
                                                             return_attn_probs=True)
        out.backward(dout)
        assert cuda_ext.launch_counter().value >= before + 3 and out.shape == (T, H, d)
        _kv_case(f"head_dim 64 {window} {dtype}", q, kv, dout, out, lse, cu.tolist(), True, window)


@pytest.mark.parametrize("q_block,kv_block", [(128, 128), (1, 256), (64, 128)])
def test_fp8_forward_block_scaled(q_block, kv_block):
    """Block-scaled e4m3 inputs (BASELINE.json config 5): one descale per token block x head for q, per 128-key
    tile (or a multiple) x kv head for k and v, applied INSIDE the forward kernel (fp32 scores / folded into P)."""
    from ring_flash_attn_b200.ops import cuda_ext
    from ring_flash_attn_b200.utils import fp8

    torch.manual_seed(0)
    B, S, H, HK = 2, 1024, 8, 2
    # token-dependent magnitudes, so that block scales actually differ
    amp = (1.0 + 3.0 * torch.rand(B, S, 1, 1, device="cuda"))
    q = torch.randn(B, S, H, 128, device="cuda") * amp
    kv = torch.randn(B, S, 2, HK, 128, device="cuda") * amp.unsqueeze(2)
    q8, dq = fp8.quantize_blockwise(q, [1, q_block, 1, 0])
    kv8, dkv = fp8.quantize_blockwise(kv, [1, kv_block, 1, 1, 0])
    qd, kvd = fp8.dequantize(q8, dq, torch.float32), fp8.dequantize(kv8, dkv, torch.float32)
    before = cuda_ext.launch_counter().value
    out, lse, _ = rfa.zigzag_ring_flash_attn_kvpacked_func(q8, kv8, causal=True, descale=(dq, dkv),
                                                           return_attn_probs=True)
    assert cuda_ext.launch_counter().value == before + 1 and out.dtype == torch.bfloat16, "not the fp8 kernel"
    _fp8_check(f"fp8 blocks {q_block} / {kv_block}", qd, kvd, out, lse)


def test_headline_shape_sampled_oracle_1gpu():
    """bench.py's shape at one GPU (S = 32768, 32 heads of 128, zigzag qkvpacked fwd + bwd) on sampled rows / heads
    against the fp32 oracle (utils/verify.py) - what ``bench.py --check`` prints, as a test."""
    from ring_flash_attn_b200.utils.verify import sampled_check

    torch.manual_seed(0)
    qkv = torch.randn(1, 32768, 3, 32, 128, device="cuda").to(torch.bfloat16).requires_grad_(True)
    dout = torch.randn(1, 32768, 32, 128, device="cuda").to(torch.bfloat16)
    out, lse, _ = rfa.zigzag_ring_flash_attn_qkvpacked_func(qkv, causal=True, return_attn_probs=True)
    out.backward(dout)
    g, x = qkv.grad[0], qkv.detach()[0]
    res = sampled_check("zigzag", x[:, 0], x[:, 1], x[:, 2], dout[0], out.detach()[0], lse[0], g[:, 0], g[:, 1], g[:, 2],
                        kv_heads=[0, 17, 31])
    assert res["ok"], res
