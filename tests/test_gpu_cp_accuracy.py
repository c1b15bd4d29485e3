"""Every context-parallel scheme through the public API on 2 or more GPUs, held to the fp64 plan oracle's
precision-matched bound of its transport (``tests/cp_oracle.py``): the fused NVLink path and its variants (copy-engine
K/V transport, one push CTA, head-group passes, llama3's strict head groups, the block-scaled fp8 forward,
``deterministic=True``) and the torch.distributed fallback (``RFA_B200_DISABLE_P2P=1``).

Each test function is one process group.  Every call in it draws new seeded inputs and is checked against its own
references, and the sequence flips the staging parity, grows the staging and the dK/dV inbox with a longer shard and
shrinks back, interleaves schemes on one peer context and puts forward-only calls between training calls - so a
kernel that read the previous call's staging half, or reduced the inbox before a peer's partials landed, would see
stale data that differs from the fresh data.  Run with ``-m gpu``."""
import itertools
import os

import pytest
import torch
import torch.distributed as dist

import cp_oracle as CP
import kernel_oracle as KO
from dist_utils import run_distributed

pytestmark = pytest.mark.gpu

TRANSPORTS = ["fused", "fallback"]
DTYPES = [torch.bfloat16, torch.float16]
HEAD_DIMS = [64, 128]
WINDOWS = [False, True]
# (scheme, causal)
SCHEMES = [("ring", True), ("ring", False), ("zigzag", True), ("stripe", True), ("ring_varlen", True),
           ("ring_varlen", False), ("zigzag_varlen", True), ("llama3", True), ("zigzag_llama3", True)]
WORLDS = [2, 4, 8]
HEADS = [(8, 2), (4, 4), (4, 1), (8, 4), (6, 2)]  # (hq, hkv)


def _ngpu():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _need(world):
    if _ngpu() < world:
        pytest.skip(f"needs {world} GPUs")


def call_sequence(world: int, dtype, base_rows=None, head_dims=HEAD_DIMS, windows=WINDOWS):
    """[(case, train)] for one process group: every scheme x head dim x window, the scheme changing from call to call.
    Calls 4..8 run twice as many rows per rank (the staging and the inbox grow), later calls shrink back; two
    forward-only calls sit between training calls, and so do forward-only ``peaked`` calls."""
    base = base_rows or (512 if world == 2 else 256)
    calls = []
    for i, ((d, window), (scheme, causal)) in enumerate(itertools.product(
            itertools.product(head_dims, windows), SCHEMES)):
        rows = 2 * base if 4 <= i < 9 else base
        hq, hkv = HEADS[i % len(HEADS)]
        stride = hkv // 2 if scheme == "llama3" and hkv > 1 and i % 2 else 1
        case = CP.Case(scheme, world, rows, hq, hkv, d, dtype, causal, stride=stride,
                       batch=2 if scheme in CP.BATCH and i % 3 == 1 else 1)
        if window:
            case = case.with_(window=CP.window_for(causal, case.total))
        calls.append((case, True))
        if i % 7 == 3:
            calls.append((case.with_(regime="peaked"), False))
    calls.insert(2, (calls[5][0].with_(rows=base // 2), False))  # a shorter shard, forward only
    calls.insert(11, (calls[0][0], False))
    return calls


def _setup(rank, transport):
    torch.backends.cuda.matmul.allow_tf32 = False  # the autouse fixtures do not reach spawned processes
    os.environ["RFA_B200_DISABLE_P2P"] = "0" if transport == "fused" else "1"
    return torch.device("cuda", rank) if torch.cuda.is_available() else torch.device("cpu")


def _check_fused_available(dev):
    from ring_flash_attn_b200.parallel import fused

    assert fused.available(torch.empty(1, device=dev), None), "no peer access between the GPUs: the fused path is off"


def run_call(rank, case, train, seed, dev, transport, deterministic=False, bwd_transport=None, tag=""):
    """One API call on this rank against its own references.  ``transport``: ``fused`` or ``fallback``."""
    plans = CP.build_plans(case)
    q, k, v, do = CP.make_inputs(case, seed, dev)
    got = CP.api_train(case, rank, q[rank], k[rank], v[rank], do[rank], deterministic=deterministic, backward=train)
    ref_t = "fused" if transport == "fused" else CP.FALLBACK_ORDER[case.scheme]
    refs = CP.references(case, plans, q, k, v, do, ref_t, ranks=[rank], all_reduce=dist.all_reduce if train else None,
                         backward=train, bwd_transport=bwd_transport)
    name = f"{tag}{case.name()} seed {seed} rank {rank}{'' if train else ' (forward only)'}"
    CP.check(name, got, *refs[rank], report=CP.report_key(transport, case.world))
    return got


def _sequence_worker(rank, world, transport, dtype, calls=None):
    dev = _setup(rank, transport)
    if transport == "fused":
        _check_fused_available(dev)
    for i, (case, train) in enumerate(calls or call_sequence(world, dtype)):
        run_call(rank, case, train, 1000 * world + i, dev, transport)


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("transport", TRANSPORTS)
@pytest.mark.parametrize("world", WORLDS)
def test_every_scheme(world, transport, dtype):
    _need(world)
    run_distributed(_sequence_worker, world, transport, dtype, backend="nccl")


# ---------------------------------------------------------------------------------------------- fused variants

def variant_sequence(world: int, dtype):
    """Every scheme once on the fused path (head dims and windows alternating, two or more kv heads so that head
    groups split), growing and shrinking the shard, with a forward-only call in between."""
    base = 512 if world == 2 else 256
    calls = []
    for i, (scheme, causal) in enumerate(SCHEMES):
        hq, hkv = [(8, 2), (4, 4), (8, 4)][i % 3]
        case = CP.Case(scheme, world, 2 * base if i in (3, 4) else base, hq, hkv, HEAD_DIMS[i % 2], dtype, causal,
                       batch=2 if scheme in CP.BATCH and i % 2 else 1)
        if i % 3 == 2:
            case = case.with_(window=CP.window_for(causal, case.total))
        calls.append((case, True))
    calls.insert(3, (calls[1][0].with_(rows=base // 2), False))
    return calls


def _variant_worker(rank, world, env):
    os.environ.update(env)
    for dtype in DTYPES:
        _sequence_worker(rank, world, "fused", dtype, variant_sequence(world, dtype))


def _dma_available() -> bool:
    from ring_flash_attn_b200.ops import cuda_ext

    return bool(cuda_ext.load().dma_transport_available())


@pytest.mark.parametrize("env", [{"RFA_B200_KV_TRANSPORT": "dma"}, {"RFA_B200_PUSH_CTAS": "1"},
                                 {"RFA_B200_STAGE_BUDGET_MB": "0"}],
                         ids=["dma", "one_push_cta", "head_group_passes"])
def test_fused_variants_2gpu(env):
    _need(2)
    if env.get("RFA_B200_KV_TRANSPORT") == "dma" and not _dma_available():
        pytest.skip("the copy-engine K/V transport needs cuStreamWaitValue32 / cuStreamWriteValue32 (driver API)")
    run_distributed(_variant_worker, 2, env, backend="nccl")


def _llama3_strict_worker(rank, world):
    os.environ["RFA_B200_LLAMA3_HEAD_GROUPS"] = "strict"
    calls = []
    for i, (d, dtype) in enumerate(itertools.product(HEAD_DIMS, DTYPES)):
        case = CP.Case("llama3", world, 1024 if i == 1 else 512, 8, 4, d, dtype, stride=1 + i % 2)
        calls.append((case.with_(window=CP.window_for(True, case.total)) if i % 2 else case, True))
    calls.insert(2, (calls[0][0].with_(rows=256), False))
    for dtype in DTYPES:
        _sequence_worker(rank, world, "fused", dtype, [c for c in calls if c[0].dtype == dtype])


def test_llama3_strict_head_groups_2gpu():
    _need(2)
    run_distributed(_llama3_strict_worker, 2, backend="nccl")


def _fp8_worker(rank, world):
    """Block-scaled e4m3 stripe attention, forward only, through the fused fp8 launch: the references see the
    dequantised inputs and round P and out to bf16."""
    import ring_flash_attn_b200 as rfa
    from ring_flash_attn_b200.ops import cuda_ext
    from ring_flash_attn_b200.utils import fp8

    dev = _setup(rank, "fused")
    _check_fused_available(dev)
    B, H, D = 2, 4, 128
    for i, L in enumerate([512, 1024, 256, 512]):
        g = torch.Generator().manual_seed(7000 + i)
        # row-dependent magnitudes, so that the block descales differ
        amp = 1.0 + 3.0 * torch.rand(world, B, L, 1, 1, 1, generator=g)
        qkv = torch.randn(world, B, L, 3, H, D, generator=g) * amp
        quant = [fp8.quantize_blockwise(qkv[r], [1, 128, 1, 1, 0]) for r in range(world)]
        deq = [fp8.dequantize(x8, sc, torch.float32).to(dev) for x8, sc in quant]
        x8, sc = (t.to(dev) for t in quant[rank])
        before = cuda_ext.launch_counter().value
        out, lse, _ = rfa.stripe_flash_attn_qkvpacked_func(x8, causal=True, descale=sc, return_attn_probs=True)
        torch.cuda.synchronize()
        assert cuda_ext.launch_counter().value == before + 1, "block-scaled fp8 did not take the fused fp8 launch"
        case = CP.Case("stripe", world, B * L, H, H, D, torch.bfloat16, batch=B)
        q, k, v = ([x[:, :, j].reshape(B * L, H, D) for x in deq] for j in range(3))
        refs = CP.references(case, CP.build_plans(case), q, k, v, None, "fused", ranks=[rank], backward=False)
        got = dict(out=out.reshape(B * L, H, D), lse=lse.permute(1, 0, 2).reshape(H, B * L))
        CP.check(f"fp8 stripe {case.name()} rank {rank}", got, *refs[rank], report="cp fused e4m3",
                 factor=KO.FP8_RATIO, lse_rel=KO.FP8_LSE_REL)


def test_fp8_block_scaled_stripe_2gpu():
    _need(2)
    run_distributed(_fp8_worker, 2, backend="nccl")


def _deterministic_worker(rank, world):
    """``deterministic=True`` (strict): the fused forward and the fallback's ordered backward - bitwise repeatable,
    and within the bound of that pair of transports."""
    import warnings

    warnings.simplefilter("ignore")
    dev = _setup(rank, "fused")
    _check_fused_available(dev)
    for i, (case, train) in enumerate(variant_sequence(world, torch.bfloat16)):
        if not train:
            continue
        bwd = CP.FALLBACK_ORDER[case.scheme]
        first = run_call(rank, case, True, 9000 + i, dev, "fused", True, bwd, "deterministic ")
        again = run_call(rank, case, True, 9000 + i, dev, "fused", True, bwd, "deterministic ")
        for key in first:
            assert torch.equal(first[key], again[key]), f"{case.name()}: {key} not bitwise reproducible"


def test_deterministic_2gpu():
    _need(2)
    run_distributed(_deterministic_worker, 2, backend="nccl")
