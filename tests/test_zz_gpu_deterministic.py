"""deterministic=True on the sm_90a path (H100): bitwise reproducible gradients, still equal to the fp32 oracle.

The file name sorts last so that the determinism checks run after every other GPU test file."""
import pytest
import torch

import ring_flash_attn_b200 as rfa
from ring_flash_attn_b200.ops.dense import attention_oracle, varlen_attention_oracle

pytestmark = pytest.mark.gpu


def _grads(fn, args, dout, **kw):
    xs = [a.detach().requires_grad_(True) for a in args]
    out = fn(*xs, deterministic=True, **kw)
    out.backward(dout)
    torch.cuda.synchronize()
    return out.detach(), [x.grad for x in xs]


@pytest.mark.filterwarnings("ignore:.*deterministic=True.*:RuntimeWarning")
@pytest.mark.parametrize("d,window", [(128, (-1, -1)), (64, (-1, -1)), (128, (300, 0))])
def test_deterministic_batch_is_bitwise_reproducible(d, window):
    torch.manual_seed(0)
    B, S, H, HK = 2, 1536, 4, 2
    q = torch.randn(B, S, H, d, device="cuda").to(torch.bfloat16)
    kv = torch.randn(B, S, 2, HK, d, device="cuda").to(torch.bfloat16)
    dout = torch.randn(B, S, H, d, device="cuda").to(torch.bfloat16)
    runs = [_grads(rfa.zigzag_ring_flash_attn_kvpacked_func, (q, kv), dout, causal=True, window_size=window)
            for _ in range(3)]
    for out, grads in runs[1:]:
        assert torch.equal(out, runs[0][0])
        for g, g0 in zip(grads, runs[0][1]):
            assert torch.equal(g, g0)
    rq, rkv = q.float().requires_grad_(True), kv.float().requires_grad_(True)
    ref, _ = attention_oracle(rq, rkv[:, :, 0], rkv[:, :, 1], True, window_size=window)
    ref.backward(dout.float())
    torch.testing.assert_close(runs[0][0].float(), ref, atol=2e-2, rtol=2e-2)
    for got, want in zip(runs[0][1], (rq.grad, rkv.grad)):
        assert (got.float() - want).abs().max().item() < 3e-2 * want.abs().max().item() + 1e-2


@pytest.mark.filterwarnings("ignore:.*deterministic=True.*:RuntimeWarning")
def test_deterministic_varlen_is_bitwise_reproducible():
    torch.manual_seed(1)
    cu = torch.tensor([0, 1, 130, 131, 900, 2048], dtype=torch.int32, device="cuda")
    T, H, HK, d = 2048, 8, 2, 128
    q = torch.randn(T, H, d, device="cuda").to(torch.bfloat16)
    k = torch.randn(T, HK, d, device="cuda").to(torch.bfloat16)
    v = torch.randn(T, HK, d, device="cuda").to(torch.bfloat16)
    dout = torch.randn(T, H, d, device="cuda").to(torch.bfloat16)
    max_len = int((cu[1:] - cu[:-1]).max())
    runs = [_grads(rfa.ring_flash_attn_varlen_func, (q, k, v), dout, cu_seqlens=cu, max_seqlen=max_len, causal=True)
            for _ in range(3)]
    for _out, grads in runs[1:]:
        for g, g0 in zip(grads, runs[0][1]):
            assert torch.equal(g, g0)
    rs = [t.float().requires_grad_(True) for t in (q, k, v)]
    ref, _ = varlen_attention_oracle(*rs, cu.cpu(), True)
    ref.backward(dout.float())
    for got, want in zip(runs[0][1], rs):
        assert (got.float() - want.grad).abs().max().item() < 3e-2 * want.grad.abs().max().item() + 1e-2
