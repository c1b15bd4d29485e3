"""The sm_90a split-KV decode kernel with shared prefixes: the fp64 oracle with ``kernel_oracle``'s precision-matched
bound for every prefix instantiation (bf16 / fp16 x D 64 / 128 x native / e4m3 cache; uniform and varlen, rotary,
appends, forced and default split counts, prefix tiles packing sequences across a 64-row boundary), agreement with
the plain call on the concatenated cache, appended and prefix bytes, CUDA-graph replay with new lengths, and per-rank
prefix shards on two GPUs."""
import dataclasses

import pytest
import torch

import decode_cache_idx as CI
import decode_oracle as DO
import decode_prefix as DP
import kernel_oracle as KO
from dist_utils import run_distributed
from ring_flash_attn_b200.parallel import decode as dec
from test_decode_prefix import _run_dense
from test_gpu_decode_fp8 import bytes_of

pytestmark = pytest.mark.gpu

# B = P * n.  "rows80": n * Sq * G = 5 * 4 * 4 = 80 packed rows per prompt, so the second 64-row tile starts inside
# sequence 3 of each group
CASES = {
    "rows80": (DO.Case("rows80", (4,) * 10, (300, 0, 17, 128, 5, 250, 1, 129, 64, 200), 320, hq=8, hkv=2), 2),
    "rows80_rotary": (DO.Case("rows80r", (4,) * 10, (300, 0, 17, 128, 5, 250, 1, 129, 64, 200), 320, hq=8, hkv=2,
                              rotary=("half", False)), 2),
    "g16_n16": (DO.Case("g16n16", (1,) * 16, tuple((37 * i) % 300 for i in range(16)), 300, hq=32, hkv=2), 1),
    "noncausal": (DO.Case("nc", (3,) * 6, (100, 31, 0, 129, 300, 2), 320, hq=8, hkv=2, causal=False), 3),
    "varlen": (DO.Case("v9", (3, 0, 20, 5, 2, 1, 7, 0, 4), (250, 9, 0, 200, 0, 33, 1, 2, 300), 320, varlen=True,
                       hq=8, hkv=2), 3),
    "varlen_rotary": (DO.Case("v9r", (3, 0, 20, 5, 2, 1, 7, 0, 4), (250, 9, 0, 200, 0, 33, 1, 2, 300), 320,
                              varlen=True, hq=8, hkv=2, rotary=("full", True), causal=False), 3),
}
P_CAP = 1500
PLENS = [P_CAP, 0, 1201, 129]
KINDS = [(torch.bfloat16, "native"), (torch.float16, "native"), (torch.bfloat16, "e4m3"), (torch.float16, "e4m3")]


@pytest.fixture(autouse=True)
def _exact_fp32_matmul():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


def _build(name, dtype, d, kind, append=True, seed=0):
    case, n_prefix = CASES[name]
    case = dataclasses.replace(case, fp8=kind == "e4m3", append=append)
    inp = DO.build_inputs(case, dtype, d, "randn", "cuda", seed)
    pre = DP.make_prefix(case, dtype, d, "cuda", PLENS[:n_prefix], P_CAP, seed=seed + 7)
    return inp, pre


def _default_prefix_splits(case, pre):
    slots = dec.prefix_tile_slots(case.b // pre.n, max(case.counts), case.hq, case.hkv,
                                  sum(case.counts) if case.varlen else None)
    return dec.num_splits_prefix(pre.n, slots, case.hkv, P_CAP, dec._sm_count(torch.cuda.current_device()))


def _call(inp, pre, splits, prefix_splits, with_append=True, caches=None, **over):
    q, k, v = DO.call_views(inp, with_append)
    kw = dict(DO.call_kwargs(inp), **pre.kwargs())
    kw.update(over)
    kc, vc = caches if caches is not None else (inp.k_cache, inp.v_cache)
    return dec.kernel_decode(q, kc, vc, inp.seqlens, k, v, inp.case.causal, inp.d ** -0.5, splits=splits,
                             prefix_splits=prefix_splits, **kw)


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("dtype, kind", KINDS, ids=[f"{str(t)[6:]}-{k}" for t, k in KINDS])
def test_oracle(dtype, kind, d):
    for i, name in enumerate(CASES):
        inp, pre = _build(name, dtype, d, kind, seed=i)
        case = inp.case
        for splits, prefix_splits in ((1, 1), (3, 5), (None, None)):
            pre_k, pre_v = pre.k.clone(), pre.v.clone()
            k0, v0 = inp.k_cache.clone(), inp.v_cache.clone()
            out, lse = _call(inp, pre, splits, prefix_splits, caches=(k0, v0))
            n_s = splits if splits is not None else DO.default_splits(case, "cuda")
            n_p = prefix_splits if prefix_splits is not None else _default_prefix_splits(case, pre)
            o64, l64, o32, l32 = DP.references(inp, pre, n_s, n_p)
            tag = f"{name} {kind} {dtype} D{d} splits={splits}/{prefix_splits}"
            got_o, got_l = DO.packed(case, out, lse)
            KO.assert_accurate(f"{tag}: out", got_o, o64, o32.to(dtype), factor=KO._factor("randn"),
                               report=f"decode prefix {kind} D{d}")
            KO.assert_lse(f"{tag}: lse", got_l, l64, l32)
            want_k, want_v = DO.expected_caches(inp, inp.k_cache, inp.v_cache, True)
            assert torch.equal(bytes_of(k0), bytes_of(want_k)) and torch.equal(bytes_of(v0), bytes_of(want_v)), tag
            assert torch.equal(bytes_of(pre.k), bytes_of(pre_k)) and torch.equal(bytes_of(pre.v), bytes_of(pre_v)), tag


@pytest.mark.parametrize("d", [64, 128])
def test_equals_plain_call_on_concatenated_cache(d):
    """The prefix call against the plain call on a cache holding the prefix rows, then the sequence's rows: the same
    result up to fp32 summation order (within the oracle's bound of each other), the same appended bytes."""
    for name in CASES:
        inp, pre = _build(name, torch.bfloat16, d, "native")
        case = inp.case
        kc, vc, lens = DP.concatenated(inp, pre)
        k0, v0 = inp.k_cache.clone(), inp.v_cache.clone()
        out, lse = _call(inp, pre, None, None, caches=(k0, v0))
        q, k, v = DO.call_views(inp, True)
        ref_out, ref_lse = dec.kernel_decode(q, kc, vc, lens, k, v, case.causal, d ** -0.5, **DO.call_kwargs(inp))
        o64, _, o32, _ = DP.references(inp, pre, DO.default_splits(case, "cuda"), _default_prefix_splits(case, pre))
        bound = 2 * (o32.to(torch.bfloat16).double() - o64).abs().max().item() + 1e-6
        got_o, got_l = DO.packed(case, out, lse)
        ref_o, ref_l = DO.packed(case, ref_out, ref_lse)
        assert (got_o.double() - ref_o.double()).abs().max().item() <= bound, name
        fin = torch.isfinite(ref_l)
        assert torch.equal(fin, torch.isfinite(got_l)), name
        assert ((got_l - ref_l)[fin].abs() <= 2e-4 * (1 + ref_l[fin].abs())).all(), name
        n = case.b // pre.n
        for b in range(case.b):
            pl = pre.lens[b // n]
            assert torch.equal(bytes_of(k0[b]), bytes_of(kc[b, pl:pl + case.s_cap])), (name, b)
            assert torch.equal(bytes_of(v0[b]), bytes_of(vc[b, pl:pl + case.s_cap])), (name, b)


def test_slots_and_left_pads_on_the_suffix():
    case = dataclasses.replace(CASES["rows80"][0], rotary=(16, True))
    si = CI.build(case, torch.bfloat16, 128, "cuda", idx=CI.slot_indices(case.b, 2 * case.b + 3, seed=4),
                  n_slots=2 * case.b + 3, pads=CI.leftpads(case, seed=5))
    pre = DP.make_prefix(case, torch.bfloat16, 128, "cuda", PLENS[:2], P_CAP)
    q, k, v, kw = CI.call_args(si, True)
    out, lse = dec.kernel_decode(q, si.k_pool, si.v_pool, si.seqlens, k, v, True, 128 ** -0.5, splits=2,
                                 prefix_splits=4, **kw, **pre.kwargs())
    o64, l64, o32, l32 = DP.references(CI.plain_inputs_for_reference(si), pre, 2, 4)
    got_o, got_l = DO.packed(case, out, lse)
    KO.assert_accurate("slots + pads: out", got_o, o64, o32.to(torch.bfloat16))
    KO.assert_lse("slots + pads: lse", got_l, l64, l32)
    want_k, want_v = CI.expected_pool(si, True)
    assert torch.equal(bytes_of(si.k_pool), bytes_of(want_k)) and torch.equal(bytes_of(si.v_pool), bytes_of(want_v))


def test_cuda_graph_replay_with_new_lengths():
    g = torch.Generator().manual_seed(5)
    n_prefix, n, sq, hq, hkv, d, s_cap, p_cap = 2, 5, 1, 32, 8, 128, 1000, 3000
    b = n_prefix * n
    kc, vc = (torch.randn(b, s_cap, hkv, d, generator=g).bfloat16().cuda() for _ in range(2))
    pk, pv = (torch.randn(n_prefix, p_cap, hkv, d, generator=g).bfloat16().cuda() for _ in range(2))
    q = torch.randn(b, sq, hq, d, generator=g).bfloat16().cuda()
    k, v = (torch.randn(b, sq, hkv, d, generator=g).bfloat16().cuda() for _ in range(2))
    sl = torch.tensor([10, 0, 500, 7, 999, 3, 3, 3, 0, 64], dtype=torch.int32, device="cuda")
    pl = torch.tensor([3000, 1], dtype=torch.int32, device="cuda")

    def step(kc_, vc_):
        return dec.kernel_decode(q, kc_, vc_, sl, k, v, True, d ** -0.5, splits=3, prefix_k_cache=pk,
                                 prefix_v_cache=pv, prefix_seqlens=pl)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(kc.clone(), vc.clone())
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out, lse = step(kc, vc)
    for lens_now, pre_now in (([10, 0, 500, 7, 999, 3, 3, 3, 0, 64], [3000, 1]),
                              ([0, 0, 0, 0, 0, 1, 2, 3, 4, 5], [0, 2999]),
                              ([998, 1, 2, 3, 4, 5, 6, 7, 8, 9], [129, -5]),  # -5: clamped to 0
                              ([5, 5, 5, 5, 5, 5, 5, 5, 5, 5], [4000, 128])):  # 4000: clamped to P_cap
        sl.copy_(torch.tensor(lens_now, dtype=torch.int32))
        pl.copy_(torch.tensor(pre_now, dtype=torch.int32))
        ek, ev = kc.clone(), vc.clone()
        graph.replay()
        want_out, want_lse = step(ek, ev)
        torch.cuda.synchronize()
        assert torch.equal(out, want_out) and torch.equal(lse, want_lse), (lens_now, pre_now)
        assert torch.equal(bytes_of(kc), bytes_of(ek)) and torch.equal(bytes_of(vc), bytes_of(ev))
    # clamping: the last replay equals a call with prefix_seqlens [P_cap, 128]
    pl.copy_(torch.tensor([p_cap, 128], dtype=torch.int32))
    ek, ev = kc.clone(), vc.clone()
    graph.replay()
    clamped_out, clamped_lse = out.clone(), lse.clone()
    pl.copy_(torch.tensor([4000, 128], dtype=torch.int32))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, clamped_out) and torch.equal(lse, clamped_lse)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_per_rank_prefix_shards():
    scenarios = [("causal", "both", True), ("varlen", None, True), ("e4m3_cache", "slots", True),
                 ("rotary", None, True), ("noncausal", None, False)]
    run_distributed(_run_dense, 2, scenarios, "cuda", backend="nccl")
