"""The sm_90a kernels at the benchmarks' long-context shapes against the fp64 oracle, with the precision-matched bound
held within every unit of kernel work as well as tensor-wide (``kernel_oracle.assert_accurate(blocks=...)``).

At these lengths the tensor-wide baseline is set by the short rows near the start of a sequence, whose outputs are
tens of times larger than those of rows 30K keys long, so a lost key tile or a mis-scaled row block near the end
would hide under it; ``tests/test_kernel_oracle_cpu.py`` shows that on the references alone.  The cases reach what
only runs at scale: thousands of CTAs past the first wave, 256 online-softmax rescales per row, the backward's Q / dO
ring wrapping thousands of times in one CTA (MQA), dQ reduce-adds from 256 key tiles onto the same rows, decode
splits of hundreds of tiles, and buffers past 2^31 bytes.

* attention through the public API at world 1 (``bench.py --gpus 1`` and ``--config readme``), forward and backward;
* the per-rank plans of ``bench.py --gpus 2 / 8`` replayed on one GPU (``cp_oracle.replay``);
* split-KV decode at ``benchmark/bench_decode.py``'s shapes (``decode_oracle.run_decode``, ``decode_prefix``).

Each case prints its wall time, peak memory and worst global / per-block ratios."""
import time

import pytest
import torch

import cp_oracle as CP
import decode_oracle as DO
import decode_prefix as DP
import kernel_oracle as KO
import ring_flash_attn_b200 as rfa
from ring_flash_attn_b200.parallel import decode as dec

pytestmark = pytest.mark.gpu
BF16, FP16 = torch.bfloat16, torch.float16


@pytest.fixture(autouse=True)
def _exact_fp32_matmul():
    """The precision-matched reference needs true fp32 GEMMs."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.fixture(autouse=True)
def _measure(request):
    """Print the case's wall time, peak memory and the worst ratios it recorded in ``KO.WORST``."""
    before = dict(KO.WORST)
    KO.WORST.clear()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    secs, peak = time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 2 ** 30
    worst = ", ".join(f"{k} {v:.3f}" for k, v in sorted(KO.WORST.items()))
    print(f"\n[long context] {request.node.name}: {secs:.1f} s, peak {peak:.1f} GiB; {worst}")
    for k, v in before.items():
        KO.WORST[k] = max(KO.WORST.get(k, 0.0), v)


# ---------------------------------------------------------------------------------------------- attention, world 1

# name: run_api arguments
ATTENTION = {
    # bench.py --gpus 1: 8,192 forward CTAs, 256 key tiles per row; every head checked
    "headline": dict(fn_name="zigzag_ring_flash_attn_qkvpacked_func", b=1, s=32768, hq=32, hkv=32, d=128, dtype=BF16),
    # every key tile raises the running max: 256 rescales per row
    "headline_peaked": dict(fn_name="zigzag_ring_flash_attn_qkvpacked_func", b=1, s=32768, hq=32, hkv=32, d=128,
                            dtype=BF16, regime="peaked", backward=False),
    # bench.py --config readme at world 1
    "readme": dict(fn_name="zigzag_ring_flash_attn_kvpacked_func", b=1, s=8192, hq=32, hkv=8, d=128, dtype=FP16),
    # the fp32 dQ accumulator is 2.28 GB; every head runs, kv heads 0 and 7 (with their query heads) are checked
    "past_2e31_bytes": dict(fn_name="ring_flash_attn_kvpacked_func", b=1, s=139264, hq=32, hkv=8, d=128, dtype=BF16,
                            kv_heads=(0, 7)),
    # MQA: one backward CTA sweeps 32 heads x 512 query tiles; the D 64 instantiation
    "mqa_ring_wrap": dict(fn_name="ring_flash_attn_kvpacked_func", b=1, s=32768, hq=32, hkv=1, d=64, dtype=FP16),
    # lse_S indexing with B > 1, thousands of CTAs
    "batched_noncausal": dict(fn_name="ring_flash_attn_kvpacked_func", b=4, s=8192, hq=16, hkv=4, d=128, dtype=BF16,
                              causal=False),
    # kWindow kernels along a long band
    "window4096": dict(fn_name="zigzag_ring_flash_attn_kvpacked_func", b=1, s=32768, hq=32, hkv=8, d=128, dtype=BF16,
                       window=(4096, 0)),
}
# one-token documents, a document ending mid-tile, two long documents
VARLEN_CU = [0, 1, 129, 30000, 30001, 65536]


@pytest.mark.parametrize("name", list(ATTENTION))
def test_attention_world1(name):
    KO.run_api(**ATTENTION[name], device="cuda", seed=len(name), report=f"long {name}")


def _round_toward_zero(x64: torch.Tensor) -> torch.Tensor:
    """fp64 -> the fp32 value next to it toward zero."""
    f = x64.float()
    return torch.where(f.double().abs() > x64.abs(), torch.nextafter(f, torch.zeros_like(f)), f)


def test_mqa_dk_drift_is_the_accumulators_truncation():
    """The backward's dK / dV drift at MQA 32K (``kernel_oracle.ACCUM_ULP``) is the wgmma accumulator rounding toward
    zero: the dK of keys 0 .. 3 replayed as the kernel sweeps them (query heads in order, 64-row tiles in order, one
    addition per 16 rows, P and dS^T from the kernel's lse and out, dS^T rounded to fp16) lands on the kernel's fp16
    values when each addition truncates: on average at least twice as close as when it rounds to nearest, and within
    an ulp where round-to-nearest is furthest off (measured on an H100: key 1, column 28, kernel -9.13281,
    truncating -9.13166, nearest -9.15146)."""
    spec = ATTENTION["mqa_ring_wrap"]
    got, (q, k, v, dout) = KO.run_api(**spec, device="cuda", seed=len("mqa_ring_wrap"))
    t, hq, d = q.shape
    scale, keys = d ** -0.5, 4
    t2 = float(torch.tensor(scale * KO.LOG2E, dtype=torch.float32))
    lse2 = (got["lse"].float() * KO.LOG2E).float()  # (Hq, T), as the kernel forms lse in log2 units
    delta = (got["out"].float() * dout.float()).sum(-1).transpose(0, 1)  # (Hq, T) from the kernel's out
    s = torch.einsum("thd,kd->htk", q.float(), k[:keys, 0].float())  # (Hq, T, keys)
    p = KO._exp2_fma(s, t2, lse2.unsqueeze(-1))
    p = p.masked_fill(torch.arange(t, device="cuda").view(1, -1, 1) < torch.arange(keys, device="cuda"), 0.0)
    dp = torch.einsum("thd,kd->htk", dout.float(), v[:keys, 0].float())
    ds = (p * (dp - delta.unsqueeze(-1)) * scale).to(FP16).double()  # dS^T as the wgmma reads it
    # per addition: 16 rows of one head, summed exactly (fp64) -> (Hq * T / 16, keys, D)
    parts = torch.einsum("htk,thd->htkd", ds, q.double()).reshape(hq * t // 16, 16, keys, d).sum(1)
    rz = torch.zeros((keys, d), dtype=torch.float32, device="cuda")
    rn = torch.zeros_like(rz)
    for x in parts:
        rz = _round_toward_zero(rz.double() + x)
        rn = (rn.double() + x).float()
    kernel = got["dk"][:keys, 0].double()
    off_rz = (kernel - rz.to(FP16).double()).abs()
    off_rn = (kernel - rn.to(FP16).double()).abs()
    ulp = torch.finfo(FP16).eps * kernel.abs().amax(dim=1, keepdim=True)  # an fp16 ulp of each key's largest dK
    rz_u, rn_u = off_rz / ulp, off_rn / ulp
    i = int(off_rn.flatten().argmax())
    print(f"\nMQA dK keys 0..{keys - 1}, kernel - replay in fp16 ulps of the key's largest value: truncating mean "
          f"{rz_u.mean():.3f}, round-to-nearest mean {rn_u.mean():.3f}; where nearest is furthest off: kernel "
          f"{kernel.flatten()[i]:.5f}, truncating {rz.flatten()[i]:.5f}, nearest {rn.flatten()[i]:.5f}")
    assert rz_u.mean() <= 0.5 * rn_u.mean() and rz_u.flatten()[i] <= 1.0


def test_attention_world1_varlen():
    t, hq, hkv, d = VARLEN_CU[-1], 32, 8, 128
    q, k, v, dout = KO.make_inputs(dict(tq=t, tk=t, hq=hq, hkv=hkv), d, BF16, "randn", "cuda", seed=11)
    cu = torch.tensor(VARLEN_CU, dtype=torch.int32, device="cuda")
    xq = q.clone().requires_grad_(True)
    x = torch.stack([k, v], dim=1).requires_grad_(True)
    max_len = max(b - a for a, b in zip(VARLEN_CU[:-1], VARLEN_CU[1:]))
    out, lse, _ = rfa.ring_flash_attn_varlen_kvpacked_func(xq, x, cu, max_len, causal=True, return_attn_probs=True)
    out.backward(dout)
    got = dict(out=out.detach(), lse=lse.detach(), dq=xq.grad, dk=x.grad[:, 0], dv=x.grad[:, 1])
    del out, lse, x
    KO.check_api_heads("varlen", got, q, k, v, dout, VARLEN_CU, True, (-1, -1), report="long varlen")


# ---------------------------------------------------------------------------------------------- multi-GPU plans

REPLAY = [CP.Case("zigzag", 2, 16384, 32, 32, 128, BF16), CP.Case("zigzag", 8, 4096, 32, 32, 128, BF16),
          CP.Case("zigzag_llama3", 4, 8192, 32, 8, 128, BF16)]


@pytest.mark.parametrize("case", REPLAY, ids=lambda c: f"{c.scheme}-W{c.world}")
def test_benchmark_plans_replayed(case):
    """What each rank of ``bench.py --gpus W`` computes with the torch.distributed transports, 32K tokens in all."""
    plans = CP.build_plans(case)
    q, k, v, do = CP.make_inputs(case, case.world, "cuda")
    got = CP.replay(case, plans, q, k, v, do)
    refs = CP.references(case, plans, q, k, v, do, CP.FALLBACK_ORDER[case.scheme])
    for r in range(case.world):
        CP.check(f"{case.name()} rank {r}", got[r], *refs[r], report=f"long replay {case.scheme} W{case.world}",
                 per_block=True)


# ---------------------------------------------------------------------------------------------- decode

DECODE = [
    # the bf16 K cache is 2.28 GB; lengths full (the append is dropped), empty, 1, one tile, one past a tile, mid
    DO.Case("b8_139k", (1,) * 8, (139264, 0, 1, 128, 131073, 129, 65535, 139262), 139264, hq=32, hkv=8),
    DO.Case("b1_512k_e4m3", (1,), (524287,), 524288, hq=32, hkv=8, fp8=True),
    # pages of 16: each split's table window refills thousands of times
    DO.Case("b4_131k_paged16", (1,) * 4, (131071, 100000, 16, 77777), 131072, hq=32, hkv=8, layout="paged",
            page_size=16),
]


@pytest.mark.parametrize("case", DECODE, ids=lambda c: c.name)
def test_decode_at_benchmark_shapes(case):
    DO.run_decode(case, BF16, 128, "randn", "cuda", draw="cuda", per_block=True)


def test_decode_shared_prefix_131k():
    """One 131072-token prompt shared by 16 samples, each with a 256-row suffix (the last row appended here)."""
    p_cap, d = 131072, 128
    case = DO.Case("prefix_131k", (1,) * 16, (255,) * 16, 256, hq=32, hkv=8)
    inp = DO.build_inputs(case, BF16, d, "randn", "cuda", seed=3, draw="cuda")
    pre = DP.make_prefix(case, BF16, d, "cuda", [p_cap], p_cap, draw="cuda")
    q, k, v = DO.call_views(inp, True)
    # 4 prefix splits of 256 key tiles each; the suffix in one split
    out, lse = dec.kernel_decode(q, inp.k_cache, inp.v_cache, inp.seqlens, k, v, True, d ** -0.5, splits=1,
                                 prefix_splits=4, **DO.call_kwargs(inp), **pre.kwargs())
    o64, l64, o32, l32 = DP.references(inp, pre, 1, 4)
    got_o, got_l = DO.packed(case, out, lse)
    KO.assert_accurate("prefix 131k: out", got_o, o64, o32.to(BF16), report="long decode prefix",
                       blocks=DO.sequence_blocks(case))
    KO.assert_lse("prefix 131k: lse", got_l, l64, l32)
