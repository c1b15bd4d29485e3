"""cp_flash_attn_with_kvcache with fp8 (e4m3) queries over e4m3 caches (``q_descale``), on CPU / gloo: the guards,
the dense path against the fp64 oracle on the dequantised inputs (worlds 1-3, contiguous / paged / varlen caches,
with and without an append, bitwise the same on every rank), the bytes of pre-quantised appends, the kernel path
through a stand-in extension, torch.compile and a dry run of the benchmark."""
import dataclasses
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist

import decode_oracle as DO
import decode_q8 as Q8
import ring_flash_attn_b200 as rfa
from dist_utils import run_distributed
from ring_flash_attn_b200.parallel import decode as dec
from test_gpu_decode_fp8 import bytes_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E4M3 = Q8.E4M3
D = 64


def _inputs(case, seed=3, cache_seed=None):
    inp = DO.build_inputs(dataclasses.replace(case, fp8=True), torch.bfloat16, D, "randn", "cpu", seed,
                          cache_seed=cache_seed)
    q8, qd, q64 = Q8.quantise_q(inp)
    return inp, q8, qd, q64


def test_q8_guards():
    inp, q8, qd, _ = _inputs(DO.geometry("rows1_g1"))
    q, k, v = DO.call_views(dataclasses.replace(inp, q=q8), True)
    kc, vc, sl = inp.k_cache, inp.v_cache, inp.seqlens
    kw = dict(k_descale=inp.k_descale, v_descale=inp.v_descale)
    f = rfa.cp_flash_attn_with_kvcache
    qb = q.float().bfloat16()
    with pytest.raises(ValueError, match="q_descale is only taken with an fp8"):
        f(qb, kc, vc, sl, q_descale=qd, **kw)
    with pytest.raises(ValueError, match="fp8 queries \\(e4m3\\) need q_descale"):
        f(q, kc, vc, sl, **kw)
    with pytest.raises(ValueError, match="need e4m3 caches"):
        f(q, kc.bfloat16(), vc.bfloat16(), sl, q_descale=qd)
    with pytest.raises(ValueError, match="must be torch.float8_e4m3fn"):
        f(q.float().to(torch.float8_e5m2), kc, vc, sl, q_descale=qd, **kw)
    cos = torch.ones(64, 8, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="the rotation belongs before quantisation"):
        f(q, kc, vc, sl, k, v, append_rank=0, rotary_cos=cos, rotary_sin=cos, q_descale=qd, **kw)
    with pytest.raises(ValueError, match="the rotation belongs before quantisation"):
        f(q, kc, vc, sl, k.to(E4M3), v.to(E4M3), append_rank=0, rotary_cos=cos, rotary_sin=cos, q_descale=qd, **kw)
    with pytest.raises(ValueError, match="k / v must both be float8_e4m3fn, bf16 or fp16"):
        f(q, kc, vc, sl, k.to(E4M3), v, append_rank=0, q_descale=qd, **kw)
    with pytest.raises(ValueError, match="k / v must both be float8_e4m3fn, bf16 or fp16"):
        f(q, kc, vc, sl, k.float(), v.float(), append_rank=0, q_descale=qd, **kw)
    for bad, match in ((qd.double(), "must be a float32"), (qd[:, :1].contiguous(), "must have shape"),
                       (qd.to("meta"), "must be on q's device")):
        with pytest.raises(ValueError, match=f"q_descale {match}"):
            f(q, kc, vc, sl, q_descale=bad, **kw)
    # e4m3 k / v over a bf16 cache keep the existing message; with a bf16 q they stay in q's dtype
    with pytest.raises(ValueError, match="q's dtype"):
        f(qb, kc.bfloat16(), vc.bfloat16(), sl, k.to(E4M3), v.to(E4M3), append_rank=0)
    with pytest.raises(ValueError, match="q's dtype"):
        f(qb, kc, vc, sl, k.to(E4M3), v.to(E4M3), append_rank=0, **kw)


DENSE_CASES = [("splits_default", "bf16"), ("paged16", "e4m3"), ("varlen44", "bf16"), ("varlen44_paged32", "e4m3"),
               ("append_overflow", "e4m3"), ("no_append_noncausal", "bf16")]


def _run_dense(rank, world, cases):
    for name, append_kind in cases:
        case = dataclasses.replace(DO.geometry(name), fp8=True)
        append_rank = world - 1
        shards = [_inputs(case, seed=3, cache_seed=10 + r) for r in range(world)]
        inp, q8, qd, _ = shards[rank]
        k0, v0 = inp.k_cache.clone(), inp.v_cache.clone()
        src = dataclasses.replace(inp, q=q8)
        if append_kind == "e4m3":
            src = dataclasses.replace(src, k_new=inp.stored_k, v_new=inp.stored_v)
        q, k, v = DO.call_views(src, case.append)
        out, lse = rfa.cp_flash_attn_with_kvcache(q, inp.k_cache, inp.v_cache, inp.seqlens, k, v,
                                                  append_rank=append_rank if case.append else None,
                                                  causal=case.causal, return_softmax_lse=True,
                                                  group=dist.group.WORLD, q_descale=qd, **DO.call_kwargs(inp))
        assert out.dtype == torch.bfloat16 and out.shape == q.shape
        refs = [DO.references(dataclasses.replace(s, q=s64), 1, appended_here=case.append and r == append_rank)
                for r, (s, _, _, s64) in enumerate(shards)]
        o64, l64 = DO.combine_ranks64([(a, b) for a, b, _, _ in refs])
        got_o, got_l = DO.packed(case, out, lse)
        tag = f"{name} append {append_kind} world {world}"
        torch.testing.assert_close(got_o.double(), o64, atol=2e-2, rtol=2e-2, msg=tag)
        torch.testing.assert_close(got_l.double(), l64, atol=1e-4, rtol=1e-4, msg=tag)
        want_k, want_v = DO.expected_caches(inp, k0, v0, case.append and rank == append_rank)
        assert torch.equal(bytes_of(inp.k_cache), bytes_of(want_k)), tag
        assert torch.equal(bytes_of(inp.v_cache), bytes_of(want_v)), tag
        both = torch.cat([out.float().reshape(-1), lse.reshape(-1)])
        got = [torch.empty_like(both) for _ in range(world)]
        dist.all_gather(got, both)
        for x in got:
            assert torch.equal(x.nan_to_num(7.0), both.nan_to_num(7.0)), f"{tag}: the ranks' results differ"


@pytest.mark.parametrize("world", [1, 2, 3])
def test_dense_path_matches_oracle(world):
    run_distributed(_run_dense, world, DENSE_CASES)


@pytest.mark.parametrize("name", ["append_overflow", "paged16", "varlen44_paged32", "paged_out_of_pool"])
def test_prequantised_append_bytes(name):
    """Cache rows [cache_seqlens[b], cache_seqlens[b] + n_b) hold exactly k / v's bytes; rows past S_cap, and rows
    whose page is outside the pool, are dropped; nothing else in the pool changes."""
    case = DO.geometry("paged16" if name == "paged_out_of_pool" else name)
    inp, q8, qd, _ = _inputs(case)
    table = inp.table
    if name == "paged_out_of_pool":  # the page of sequence 0's first new row points past the pool
        table = table.clone()
        table[0, inp.lens[0] // case.page_size] = inp.k_cache.shape[0]
    k8, v8 = torch.randn_like(inp.stored_k.float()).to(E4M3), torch.randn_like(inp.stored_v.float()).to(E4M3)
    want_k, want_v = inp.k_cache.clone(), inp.v_cache.clone()
    s_cap, ps = case.s_cap, case.page_size
    for b, (lo, n) in enumerate(DO.spans(case)):
        for t in range(n):
            row = inp.lens[b] + t
            if row >= s_cap:
                continue
            at = (b, row)
            if table is not None:
                page = int(table[b, row // ps])
                if not 0 <= page < inp.k_cache.shape[0]:
                    continue
                at = (page, row % ps)
            want_k[at], want_v[at] = k8[lo + t], v8[lo + t]
    q, k, v = DO.call_views(dataclasses.replace(inp, q=q8, k_new=k8, v_new=v8), True)
    kw = dict(DO.call_kwargs(inp), block_table=table)

    def call():
        rfa.cp_flash_attn_with_kvcache(q, inp.k_cache, inp.v_cache, inp.seqlens, k, v, append_rank=0, q_descale=qd,
                                       **kw)

    if name == "paged_out_of_pool":  # the dense path appends, then raises for the page attention must read
        with pytest.raises(ValueError, match="outside"):
            call()
    else:
        call()
    assert torch.equal(bytes_of(inp.k_cache), bytes_of(want_k))
    assert torch.equal(bytes_of(inp.v_cache), bytes_of(want_v))


@pytest.mark.parametrize("name, append_kind", [("paged16", "bf16"), ("paged16", "e4m3"), ("varlen44", "e4m3"),
                                               ("rows129_g3", "bf16"), ("empty_shard_no_append", "bf16")])
def test_kernel_path_through_stand_in_matches_dense(monkeypatch, name, append_kind):
    from ring_flash_attn_b200.ops import cuda_ext

    monkeypatch.setattr(cuda_ext, "load", Q8.FakeQ8DecodeExt)
    case = dataclasses.replace(DO.geometry(name), fp8=True)
    inp, q8, qd, _ = _inputs(case)
    src = dataclasses.replace(inp, q=q8)
    if append_kind == "e4m3":
        src = dataclasses.replace(src, k_new=inp.stored_k, v_new=inp.stored_v)
    q, k, v = DO.call_views(src, case.append)
    kd = DO.call_kwargs(inp)
    ka, va = inp.k_cache.clone(), inp.v_cache.clone()
    out, lse = dec.kernel_decode(q, ka, va, inp.seqlens, k, v, case.causal, D ** -0.5, splits=3, q_descale=qd, **kd)
    kb, vb = inp.k_cache.clone(), inp.v_cache.clone()
    d_out, d_lse = dec._dense_decode(q, kb, vb, inp.seqlens, k, v, case.causal, D ** -0.5, None, 1,
                                     kd["block_table"], inp.k_descale, inp.v_descale, kd.get("cu_seqlens_q"),
                                     kd.get("max_seqlen_q", 0), None, qd)
    assert out.dtype == d_out.dtype == torch.bfloat16
    torch.testing.assert_close(out.float(), d_out.float(), atol=2e-2, rtol=2e-2)
    torch.testing.assert_close(lse, d_lse, atol=1e-4, rtol=1e-4)
    assert torch.equal(bytes_of(ka), bytes_of(kb)) and torch.equal(bytes_of(va), bytes_of(vb))


@pytest.mark.parametrize("name", ["rows129_g3", "split_edge_by_append", "paged64", "varlen44", "saturating_append"])
def test_stand_in_holds_the_q8_oracle_bound(monkeypatch, name):
    """The fp64 / precision-matched references of the GPU sweep, on the stand-in extension."""
    from ring_flash_attn_b200.ops import cuda_ext

    monkeypatch.setattr(cuda_ext, "load", Q8.FakeQ8DecodeExt)
    for kind in ("bf16", "e4m3"):
        Q8.run_q8(DO.geometry(name), D, "randn", "cpu", append_kind=kind)


def test_two_ranks_on_stand_in():
    run_distributed(Q8.run_two_ranks_q8, 2, "cpu")


def test_torch_compile_fullgraph_q8():
    case = dataclasses.replace(DO.geometry("paged16"), fp8=True)
    inp, q8, qd, _ = _inputs(case)
    q, k, v = DO.call_views(dataclasses.replace(inp, q=q8, k_new=inp.stored_k, v_new=inp.stored_v), True)
    pk, pv = inp.k_cache, inp.v_cache
    pk2, pv2 = pk.clone(), pv.clone()

    def f(q, pk, pv, sl, k, v, bt, kd, vd, qd):
        out, lse = rfa.cp_flash_attn_with_kvcache(q, pk, pv, sl, k, v, append_rank=0, return_softmax_lse=True,
                                                  block_table=bt, k_descale=kd, v_descale=vd, q_descale=qd)
        return out * 1.0, lse

    args = (inp.seqlens, k, v, inp.table, inp.k_descale, inp.v_descale, qd)
    out, lse = torch.compile(f, backend="aot_eager", fullgraph=True)(q, pk, pv, *args)
    ref_out, ref_lse = f(q, pk2, pv2, *args)
    assert out.dtype == torch.bfloat16
    assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse)
    assert torch.equal(bytes_of(pk), bytes_of(pk2))  # the compiled call appended too


def test_bench_decode_dry_run_q8():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "benchmark", "bench_decode.py"), "--dry-run",
                        "--kv-dtype", "e4m3", "--q-dtype", "e4m3", "--batch", "1", "8", "--cache", "32768"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:]
    rows = [json.loads(line) for line in r.stdout.splitlines() if line.startswith("{")]
    assert [(x["batch"], x["cache_tokens"]) for x in rows] == [(1, 32768), (8, 32768)]
    for x in rows:
        assert x["q_dtype"] == "e4m3" and x["kv_dtype"] == "e4m3"
        assert x["q8_fields"] == ["q8_us", "q8_speedup_vs_bf16", "q8_speedup_vs_fp8", "q8_max_abs_diff_vs_bf16"]
    bad = subprocess.run([sys.executable, os.path.join(ROOT, "benchmark", "bench_decode.py"), "--dry-run",
                          "--q-dtype", "e4m3"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                         timeout=300, cwd=ROOT)
    assert bad.returncode != 0 and "--kv-dtype e4m3" in bad.stdout
