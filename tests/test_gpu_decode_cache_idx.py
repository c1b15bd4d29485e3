"""The sm_90a split-KV decode kernel with cache slots (``cache_batch_idx``) and left padding (``cache_leftpad``): the
fp64 oracle with ``kernel_oracle``'s precision-matched bound (bf16 / fp16 x D 64 / 128, e4m3 caches and e4m3
queries, forced split counts, varlen and rotary calls), bitwise relations to the plain call on the gathered / shifted
cache, out-of-range values inside a sentinel-guarded buffer, CUDA-graph replay with new slots, pads and lengths, and
per-rank left pads on two GPUs."""
import dataclasses

import pytest
import torch

import decode_cache_idx as CI
import decode_oracle as DO
import kernel_oracle as KO
from dist_utils import run_distributed
from ring_flash_attn_b200.parallel import decode as dec
from test_decode_cache_idx import _run_left_padded
from test_gpu_decode_fp8 import bytes_of

pytestmark = pytest.mark.gpu

HEAD_DIMS = [64, 128]
# geometry per feature; e4m3 kinds take the ones without rotary
FEATURES = {
    "causal": "split_edge_by_append",
    "noncausal": "rows64_g2",
    "varlen": "varlen44",
    "rows129": "rows129_g3",
    "rotary": "rotary16_interleaved",
    "rotary_varlen": "rotary_full_interleaved_varlen_noncausal",
}
MODES = ("slots", "leftpad", "both", "slots_dup")
SPLITS = (1, 3, None)


@pytest.fixture(autouse=True)
def _exact_fp32_matmul():
    """The precision-matched reference needs true fp32 GEMMs."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


def _build(name, mode, dtype, d, kind, append=True, seed=0):
    case = DO.geometry(name, fp8=kind != "native")
    if not append:
        case = dataclasses.replace(case, append=False)
    b = case.b
    idx = CI.slot_indices(b, 2 * b + 3, seed=100 + seed, duplicates=mode == "slots_dup") \
        if mode in ("slots", "both", "slots_dup") else None
    pads = CI.leftpads(case, seed=200 + seed) if mode in ("leftpad", "both") else None
    return CI.build(case, dtype, d, "cuda", idx=idx, n_slots=2 * b + 3, pads=pads, q8=kind == "q8", seed=seed)


def _call(si, splits, with_append, caches=None, **over):
    """kernel_decode of the slot / left-padded call on (by default) its own pool; returns (out, lse)."""
    case = si.plain.case
    q, k, v, kw = CI.call_args(si, with_append)
    kw.update(over)
    kc, vc = caches if caches is not None else (si.k_pool, si.v_pool)
    return dec.kernel_decode(q, kc, vc, si.seqlens, k, v, case.causal, si.plain.d ** -0.5, splits=splits, **kw)


def _check_oracle(si, splits, with_append, tag):
    case, d = si.plain.case, si.plain.d
    n_splits = splits if splits is not None else DO.default_splits(case, "cuda")
    out, lse = _call(si, n_splits, with_append)
    o64, l64, o32, l32 = DO.references(CI.plain_inputs_for_reference(si), n_splits)
    got_o, got_l = DO.packed(case, out, lse)
    q8, fp8 = si.q8 is not None, case.fp8
    out_dtype = torch.bfloat16 if q8 else si.plain.dtype
    assert out.dtype == out_dtype, tag
    KO.assert_accurate(f"{tag}: out", got_o, o64, o32.to(out_dtype),
                       factor=max(KO.FP8_RATIO, KO._factor("randn")) if q8 else KO._factor("randn"),
                       report=f"decode slots {'e4m3-q' if q8 else ('e4m3' if fp8 else 'native')} D{d}")
    KO.assert_lse(f"{tag}: lse", got_l, l64, l32, rel_limit=KO.FP8_LSE_REL if q8 else None)
    want_k, want_v = CI.expected_pool(si, with_append)
    for name, got, want in (("k", si.k_pool, want_k), ("v", si.v_pool, want_v)):
        diff = bytes_of(got) != bytes_of(want)
        assert not diff.any(), f"{tag}: {name} pool bytes differ at {diff.nonzero()[:4].tolist()}"


KINDS = [(torch.bfloat16, "native"), (torch.float16, "native"), (torch.bfloat16, "e4m3"), (torch.float16, "e4m3"),
         (torch.bfloat16, "q8")]


@pytest.mark.parametrize("d", HEAD_DIMS)
@pytest.mark.parametrize("dtype, kind", KINDS, ids=[f"{str(t)[6:]}-{k}" for t, k in KINDS])
def test_oracle(dtype, kind, d):
    i = 0
    for feature, name in FEATURES.items():
        if kind != "native" and feature.startswith("rotary"):
            continue
        for mode in MODES:
            if mode == "slots_dup" and feature.startswith("rotary"):  # rotary needs k / v
                continue
            append = mode != "slots_dup" and DO.geometry(name).append
            si = _build(name, mode, dtype, d, kind, append=append)
            splits = SPLITS[i % len(SPLITS)]
            i += 1
            _check_oracle(si, splits, append, f"{feature} {mode} {kind} {dtype} D{d} splits={splits}")


@pytest.mark.parametrize("kind", ["native", "e4m3", "q8"])
@pytest.mark.parametrize("d", HEAD_DIMS)
def test_equals_plain_call(d, kind):
    """A slot call is the call on ``pool[idx]`` and a left-padded one the call on the shifted cache, at the same split
    count (cache bytes after the append included); ``arange(B)`` / zero pads are the plain call; NaN pad rows change
    nothing."""
    for name in ("split_edge_by_append", "varlen44") + (("rotary16_interleaved",) if kind == "native" else ()):
        for mode in ("slots", "leftpad", "both"):
            si = _build(name, mode, torch.bfloat16, d, kind)
            for splits in (1, 4):
                caches = (si.k_pool.clone(), si.v_pool.clone())
                out, lse = _call(si, splits, True, caches=caches)
                plain = dataclasses.replace(si, k_pool=si.plain.k_cache.clone(), v_pool=si.plain.v_cache.clone(),
                                            idx=None, pads=None, seqlens=si.plain.seqlens)
                ref_out, ref_lse = _call(plain, splits, True)
                tag = f"{name} {mode} {kind} D{d} splits={splits}"
                assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse), tag
                s_cap = si.plain.case.s_cap
                for b in range(si.plain.case.b):
                    slot = b if si.idx is None else si.idx[b]
                    lp = 0 if si.pads is None else si.pads[b]
                    for got, ref in ((caches[0], plain.k_pool), (caches[1], plain.v_pool)):
                        assert torch.equal(bytes_of(got[slot, lp:]), bytes_of(ref[b, :s_cap - lp])), (tag, b)
                # pad rows holding zeros instead of NaN
                if si.pads is not None:
                    kz, vz = si.k_pool.clone(), si.v_pool.clone()
                    for b, lp in enumerate(si.pads):
                        slot = b if si.idx is None else si.idx[b]
                        CI.raw(kz)[slot, :lp] = 0
                        CI.raw(vz)[slot, :lp] = 0
                    zo, zl = _call(si, splits, True, caches=(kz, vz))
                    assert torch.equal(zo, out) and torch.equal(zl, lse), f"{tag}: NaN pad rows"
            # identity slots and zero pads are the plain call
            plain_si = _build(name, "slots", torch.bfloat16, d, kind)
            plain = dataclasses.replace(plain_si, k_pool=plain_si.plain.k_cache.clone(),
                                        v_pool=plain_si.plain.v_cache.clone(), idx=None, pads=None,
                                        seqlens=plain_si.plain.seqlens)
            b = plain_si.plain.case.b
            ident = dict(cache_batch_idx=torch.arange(b, dtype=torch.int32, device="cuda"),
                         cache_leftpad=torch.zeros(b, dtype=torch.int32, device="cuda"))
            c1 = (plain.k_pool.clone(), plain.v_pool.clone())
            c2 = (plain.k_pool.clone(), plain.v_pool.clone())
            o1, l1 = _call(plain, 3, True, caches=c1)
            o2, l2 = _call(plain, 3, True, caches=c2, **ident)
            assert torch.equal(o1, o2) and torch.equal(l1, l2), name
            assert torch.equal(bytes_of(c1[0]), bytes_of(c2[0])) and torch.equal(bytes_of(c1[1]), bytes_of(c2[1]))


@pytest.mark.parametrize("kind", ["native", "e4m3"])
def test_out_of_range_values_stay_in_bounds(kind):
    """An index outside [0, B_cache) sees no key and drops its append; pads below 0 or above cache_seqlens are
    clamped.  The pool is the middle of a sentinel-filled buffer: the sentinel bytes, the other sequences' results
    and every byte the call may not write stay as they were."""
    case = DO.Case("oob", (3,) * 6, (700, 300, 650, 200, 500, 129), 800, hq=8, hkv=2)
    si = CI.build(dataclasses.replace(case, fp8=kind != "native"), torch.bfloat16, 128, "cuda",
                  idx=[4, 0, 7, 2, 5, 1], n_slots=8, pads=[3, 5, 2, 9, 0, 11])
    n_slots = si.k_pool.shape[0]
    bufs = []
    for pool in (si.k_pool, si.v_pool):
        shape = (n_slots + 2,) + tuple(pool.shape[1:-1]) + (pool.shape[-1] * pool.element_size(),)
        buf = torch.full(shape, 0xA5, dtype=torch.uint8, device="cuda").view(pool.dtype)
        CI.raw(buf)[1:n_slots + 1] = CI.raw(pool)
        bufs.append(buf)
    sentinel = [CI.raw(x).clone() for x in bufs]
    kc, vc = bufs[0][1:n_slots + 1], bufs[1][1:n_slots + 1]
    q, k, v, kw = CI.call_args(si, True)
    bad_idx = kw["cache_batch_idx"].clone()
    bad_idx[0], bad_idx[1] = n_slots, -3
    bad_pad = kw["cache_leftpad"].clone()
    bad_pad[2], bad_pad[3] = -7, int(si.seqlens[3]) + 40
    out, lse = dec.kernel_decode(q, kc, vc, si.seqlens, k, v, True, 128 ** -0.5, splits=3,
                                 **dict(kw, cache_batch_idx=bad_idx, cache_leftpad=bad_pad))
    torch.cuda.synchronize()
    for i in (0, -1):  # the slots on either side of the pool
        assert torch.equal(CI.raw(bufs[0])[i], sentinel[0][i]) and torch.equal(CI.raw(bufs[1])[i], sentinel[1][i])
    # sequences 0 and 1: no key on this rank (out 0, lse -inf)
    assert (out[:2] == 0).all() and torch.isneginf(lse[:2]).all()
    # sequences 2 and 3 as with their pads clamped to [0, cache_seqlens], the others untouched
    ok_pad = bad_pad.clone()
    ok_pad[2], ok_pad[3] = 0, int(si.seqlens[3])
    ref_k, ref_v = si.k_pool.clone(), si.v_pool.clone()
    ref_out, ref_lse = dec.kernel_decode(q, ref_k, ref_v, si.seqlens, k, v, True, 128 ** -0.5, splits=3,
                                         **dict(kw, cache_leftpad=ok_pad))
    assert torch.equal(out[2:], ref_out[2:]) and torch.equal(lse[2:], ref_lse[2:])
    # the pool holds the appends of sequences 2.. only
    want_k, want_v = si.k_pool.clone(), si.v_pool.clone()
    inp = si.plain
    for b, (lo, n) in enumerate(DO.spans(case)):
        if b < 2:
            continue
        for t in range(n):
            row = int(si.seqlens[b]) + t
            if row < case.s_cap:
                CI.raw(want_k)[si.idx[b], row] = CI.raw(inp.stored_k)[lo + t]
                CI.raw(want_v)[si.idx[b], row] = CI.raw(inp.stored_v)[lo + t]
    assert torch.equal(bytes_of(kc), bytes_of(want_k)) and torch.equal(bytes_of(vc), bytes_of(want_v))


def test_cuda_graph_replay_with_new_slots_pads_and_lengths():
    g = torch.Generator().manual_seed(5)
    b, sq, hq, hkv, d, s_cap, n_slots = 4, 2, 32, 8, 128, 3008, 7
    kc = torch.randn(n_slots, s_cap, hkv, d, generator=g).bfloat16().cuda()
    vc = torch.randn(n_slots, s_cap, hkv, d, generator=g).bfloat16().cuda()
    q = torch.randn(b, sq, hq, d, generator=g).bfloat16().cuda()
    k, v = (torch.randn(b, sq, hkv, d, generator=g).bfloat16().cuda() for _ in range(2))
    sl = torch.tensor([1000, 2500, 7, 0], dtype=torch.int32, device="cuda")
    idx = torch.tensor([3, 0, 6, 2], dtype=torch.int32, device="cuda")
    lp = torch.tensor([10, 0, 7, 0], dtype=torch.int32, device="cuda")

    def step(kc_, vc_):
        return dec.kernel_decode(q, kc_, vc_, sl, k, v, True, d ** -0.5, splits=4, cache_batch_idx=idx,
                                 cache_leftpad=lp)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(kc.clone(), vc.clone())  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out, lse = step(kc, vc)
    for lens_now, idx_now, lp_now in (([1000, 2500, 7, 0], [3, 0, 6, 2], [10, 0, 7, 0]),
                                      ([1200, 1, 0, 3000], [1, 1, 5, 4], [0, 1, 0, 2999]),
                                      ([0, 2999, 64, 5], [6, 5, 4, 3], [0, 1000, 63, 5])):
        sl.copy_(torch.tensor(lens_now, dtype=torch.int32))
        idx.copy_(torch.tensor(idx_now, dtype=torch.int32))
        lp.copy_(torch.tensor(lp_now, dtype=torch.int32))
        ek, ev = kc.clone(), vc.clone()
        graph.replay()
        want_out, want_lse = step(ek, ev)
        torch.cuda.synchronize()
        assert torch.equal(out, want_out) and torch.equal(lse, want_lse), lens_now
        assert torch.equal(bytes_of(kc), bytes_of(ek)) and torch.equal(bytes_of(vc), bytes_of(ev)), lens_now


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("scheme", ["ring", "zigzag", "stripe"])
def test_two_gpus_per_rank_left_pads(scheme):
    run_distributed(_run_left_padded, 2, scheme, "cuda", backend="nccl")
