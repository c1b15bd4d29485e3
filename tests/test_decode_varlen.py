"""cp_flash_attn_with_kvcache with variable-length query batches (``cu_seqlens_q=``) on CPU / gloo (worlds 1-4):
against a per-sequence fp64 oracle, over contiguous, paged and e4m3 caches, the cache bytes after the append, bitwise
agreement across ranks and with the uniform call at equal counts, the guards, torch.compile, the varlen split count
and a dry run of the benchmark."""
import itertools
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist

import ring_flash_attn_b200 as rfa
from ring_flash_attn_b200.parallel import decode as dec
from dist_utils import run_distributed
from test_decode import TOL, decode_oracle, make_case
from test_decode_fp8 import LSE_TOL, OUT_TOL, dequantize, quantize
from test_decode_paged import to_pool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S_CAP = 128
# token counts per sequence: a 0, 1s, and chunks longer than one 64-row tile at every group size
COUNTS = [(1, 0, 70, 3), (2, 2, 2), (0, 5, 1, 1, 17, 9)]
CASES = [(grp, causal, append) for grp in (1, 4, 8) for causal in (True, False) for append in (True, False)]


def pack(x, counts):
    """(B, Smax, H, D) -> the (total_q, H, D) rows of the first counts[b] tokens of every sequence."""
    return torch.cat([x[i, :n] for i, n in enumerate(counts)])


def cu_of(counts, device="cpu"):
    return torch.tensor([0] + list(itertools.accumulate(counts)), dtype=torch.int32, device=device)


def varlen_oracle(q4, caches, lens, k4, v4, counts, causal):
    """test_decode.decode_oracle on every sequence's slice, packed: (out (total_q, Hq, D), lse (Hq, total_q))."""
    outs, lses = [], []
    for i, n in enumerate(counts):
        if n == 0:
            continue
        kn = None if k4 is None else k4[i:i + 1, :n]
        vn = None if v4 is None else v4[i:i + 1, :n]
        o, l = decode_oracle(q4[i:i + 1, :n], [(kc[i:i + 1], vc[i:i + 1]) for kc, vc in caches],
                             [x[i:i + 1] for x in lens], kn, vn, causal)
        outs.append(o[0])
        lses.append(l[0])
    return torch.cat(outs), torch.cat(lses, dim=1)


def appended(cache, table, lens, new_rows, counts):
    """``cache`` (contiguous, or a pool with ``table``) after sequence b's ``counts[b]`` rows of ``new_rows``
    (total_q, Hkv, D) go to logical rows [lens[b], lens[b] + counts[b]); rows past the capacity are dropped."""
    want = cache.clone()
    cu = cu_of(counts).tolist()
    ps = cache.shape[1]
    s_cap = cache.shape[1] if table is None else table.shape[1] * ps
    for i, n in enumerate(counts):
        for t in range(n):
            row = int(lens[i]) + t
            if row >= s_cap:
                continue
            if table is None:
                want[i, row] = new_rows[cu[i] + t]
            else:
                want[int(table[i, row // ps]), row % ps] = new_rows[cu[i] + t]
    return want


def _run_varlen(rank, world, kinds, cases):
    for kind in kinds:  # "contiguous", "paged16", "paged128", "fp8", "fp8paged16"
        fp8 = kind.startswith("fp8")
        ps = int(kind.split("paged")[1]) if "paged" in kind else None
        for n, (grp, causal, append) in enumerate(cases):
            counts = COUNTS[n % len(COUNTS)]
            seed = 1000 * world + 37 * len(kind) + n
            b, smax, hkv, d = len(counts), max(counts), 2, 16
            caches, lens, q4, k4, v4 = make_case(world, b, smax, hkv * grp, hkv, d, S_CAP, seed)
            ar = (n % world) if append else None
            ds = None
            if fp8:  # per-(sequence, kv head) descales, different on every rank and for K and V
                ds = [(0.37 * (1 + 0.25 * r) * (1 + 0.1 * torch.arange(b * hkv, dtype=torch.float32)).view(b, hkv),
                       0.55 * (1 + 0.1 * r) * (1 + 0.05 * torch.arange(b * hkv, dtype=torch.float32)).view(b, hkv))
                      for r in range(world)]
                caches = [(quantize(kc, kd), quantize(vc, vd)) for (kc, vc), (kd, vd) in zip(caches, ds)]
                q4, k4, v4 = q4.bfloat16(), k4.bfloat16(), v4.bfloat16()
            q, k, v = pack(q4, counts), pack(k4, counts), pack(v4, counts)
            cu = cu_of(counts)
            kc, vc = caches[rank][0].clone(), caches[rank][1].clone()
            table = None
            if ps is not None:
                alloc = (lens[rank] + torch.tensor(counts)).clamp(max=S_CAP)
                kc, vc, table = to_pool(kc, vc, lens[rank], ps, alloc=alloc, seed=seed + rank)
            kc0, vc0 = kc.clone(), vc.clone()
            extra = dict(k_descale=ds[rank][0], v_descale=ds[rank][1]) if fp8 else {}
            out, lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, lens[rank], k if append else None,
                                                      v if append else None, append_rank=ar, causal=causal,
                                                      return_softmax_lse=True, block_table=table, cu_seqlens_q=cu,
                                                      max_seqlen_q=smax, **extra)
            assert out.shape == q.shape and out.dtype == q.dtype and lse.shape == (q.shape[1], q.shape[0])
            if fp8:  # the oracle over the dequantised caches plus the rows as the append rank stores them
                ref_caches = [(dequantize(a, x), dequantize(c, y)) for (a, c), (x, y) in zip(caches, ds)]
                kr = vr = None
                if append:
                    kr = dequantize(quantize(k4, ds[ar][0]), ds[ar][0])
                    vr = dequantize(quantize(v4, ds[ar][1]), ds[ar][1])
                ref_out, ref_lse = varlen_oracle(q4.float(), ref_caches, lens, kr, vr, counts, causal)
                torch.testing.assert_close(out.float(), ref_out, **OUT_TOL)
                torch.testing.assert_close(lse, ref_lse, **LSE_TOL)
            else:
                ref_out, ref_lse = varlen_oracle(q4, caches, lens, k4 if append else None, v4 if append else None,
                                                 counts, causal)
                torch.testing.assert_close(out, ref_out, **TOL)
                torch.testing.assert_close(lse, ref_lse, **TOL)
            # the cache: sequence b's rows at [len, len + n_b) of the append rank, every other byte untouched
            want_k, want_v = kc0, vc0
            if append and rank == ar:
                nk, nv = (pack(quantize(k4, ds[rank][0]), counts), pack(quantize(v4, ds[rank][1]), counts)) if fp8 \
                    else (k, v)
                want_k, want_v = appended(kc0, table, lens[rank], nk, counts), appended(vc0, table, lens[rank], nv,
                                                                                        counts)
            if fp8:
                assert torch.equal(kc.view(torch.uint8), want_k.view(torch.uint8))
                assert torch.equal(vc.view(torch.uint8), want_v.view(torch.uint8))
            else:
                assert torch.equal(kc.nan_to_num(7.0), want_k.nan_to_num(7.0))
                assert torch.equal(vc.nan_to_num(7.0), want_v.nan_to_num(7.0))
            if world > 1:  # bitwise the same on every rank
                both = torch.cat([out.float().reshape(-1), lse.reshape(-1)])
                got = [torch.empty_like(both) for _ in range(world)]
                dist.all_gather(got, both)
                for x in got:
                    assert torch.equal(x.nan_to_num(7.0), both.nan_to_num(7.0))


KINDS = ("contiguous", "paged16", "paged128", "fp8", "fp8paged16")


@pytest.mark.parametrize("kind", KINDS)
def test_varlen_world1_matches_oracle(kind):
    _run_varlen(0, 1, (kind,), CASES)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_varlen_gloo_worlds_match_oracle(world):
    run_distributed(_run_varlen, world, KINDS, CASES)


@pytest.mark.parametrize("causal", [True, False])
def test_equal_counts_match_the_uniform_call(causal):
    """A varlen call whose counts are all Sq is the uniform call: out bitwise, lse after (B, Hq, Sq) -> (Hq, B*Sq)."""
    b, sq, hq, hkv, d = 3, 4, 8, 2, 16
    caches, lens, q, k, v = make_case(1, b, sq, hq, hkv, d, 40, seed=3)
    kc, vc = caches[0]
    kc2, vc2 = kc.clone(), vc.clone()
    u_out, u_lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, lens[0], k, v, append_rank=0, causal=causal,
                                                  return_softmax_lse=True)
    out, lse = rfa.cp_flash_attn_with_kvcache(q.flatten(0, 1), kc2, vc2, lens[0], k.flatten(0, 1), v.flatten(0, 1),
                                              append_rank=0, causal=causal, return_softmax_lse=True,
                                              cu_seqlens_q=cu_of([sq] * b), max_seqlen_q=sq)
    assert torch.equal(out, u_out.flatten(0, 1))
    assert torch.equal(lse, u_lse.permute(1, 0, 2).reshape(hq, b * sq))
    assert torch.equal(kc.nan_to_num(7.0), kc2.nan_to_num(7.0))


def test_all_counts_zero():
    caches, lens, q, k, v = make_case(1, 2, 1, 4, 2, 16, 8, seed=0)
    kc, vc = caches[0]
    kc0 = kc.clone()
    out, lse = rfa.cp_flash_attn_with_kvcache(q[:0, 0], kc, vc, lens[0], k[:0, 0], v[:0, 0], append_rank=0,
                                              return_softmax_lse=True, cu_seqlens_q=cu_of([0, 0]), max_seqlen_q=1)
    assert out.shape == (0, 4, 16) and lse.shape == (4, 0)
    assert torch.equal(kc.nan_to_num(7.0), kc0.nan_to_num(7.0))


def test_varlen_guards():
    caches, lens, q4, k4, v4 = make_case(1, 2, 3, 4, 2, 16, 8, seed=0)
    kc, vc = caches[0]
    sl = lens[0]
    q, k, v = q4.flatten(0, 1), k4.flatten(0, 1), v4.flatten(0, 1)  # total_q = 6
    cu = cu_of([3, 3])
    f = rfa.cp_flash_attn_with_kvcache
    with pytest.raises(ValueError, match="max_seqlen_q is required"):
        f(q, kc, vc, sl, cu_seqlens_q=cu)
    with pytest.raises(ValueError, match="max_seqlen_q is only taken with cu_seqlens_q"):
        f(q4, kc, vc, sl, max_seqlen_q=3)
    for bad in (0, -1, 2.0, True, torch.tensor(3)):
        with pytest.raises(ValueError, match="max_seqlen_q must be a host int"):
            f(q, kc, vc, sl, cu_seqlens_q=cu, max_seqlen_q=bad)
    with pytest.raises(ValueError, match="with cu_seqlens_q, q must be"):
        f(q4, kc, vc, sl, cu_seqlens_q=cu, max_seqlen_q=3)
    with pytest.raises(ValueError, match="needs cu_seqlens_q"):
        f(q, kc, vc, sl)
    for bad in (cu.long(), cu[:2], torch.zeros(4, dtype=torch.int32), cu.view(1, 3),
                torch.zeros(6, dtype=torch.int32)[::2], [0, 3, 6]):
        with pytest.raises(ValueError, match="cu_seqlens_q must be a contiguous"):
            f(q, kc, vc, sl, cu_seqlens_q=bad, max_seqlen_q=3)
    with pytest.raises(ValueError, match="cu_seqlens_q must be on q's device"):
        f(q, kc, vc, sl, cu_seqlens_q=cu.to("meta"), max_seqlen_q=3)
    with pytest.raises(ValueError, match=r"k / v must be \(total_q, Hkv, D\)"):
        f(q, kc, vc, sl, k4, v4, append_rank=0, cu_seqlens_q=cu, max_seqlen_q=3)
    with pytest.raises(ValueError, match=r"k / v must be \(total_q, Hkv, D\)"):
        f(q, kc, vc, sl, k[:5], v[:5], append_rank=0, cu_seqlens_q=cu, max_seqlen_q=3)
    with pytest.raises(ValueError, match=r"k / v must be \(total_q, Hkv, D\)"):
        f(q, kc, vc, sl, k, v.double(), append_rank=0, cu_seqlens_q=cu, max_seqlen_q=3)
    # malformed contents: the dense path checks them
    for bad, msg in (([1, 3, 6], "start at 0"), ([0, 3, 5], "end at total_q"), ([0, 7, 6], "not decrease"),
                     ([0, 6, 6], "above max_seqlen_q")):
        with pytest.raises(ValueError, match=msg):
            f(q, kc, vc, sl, cu_seqlens_q=torch.tensor(bad, dtype=torch.int32), max_seqlen_q=3)
    with pytest.raises(ValueError, match="above max_seqlen_q"):
        f(q, kc, vc, sl, cu_seqlens_q=cu, max_seqlen_q=2)


def test_torch_compile_fullgraph_varlen():
    counts = (1, 0, 6)
    caches, lens, q4, k4, v4 = make_case(1, 3, 6, 8, 2, 16, 32, seed=1)
    q, k, v = pack(q4, counts), pack(k4, counts), pack(v4, counts)
    kc, vc = caches[0]
    pk, pv, table = to_pool(kc, vc, lens[0], 16, alloc=(lens[0] + 6).clamp(max=32))
    pk2, pv2 = pk.clone(), pv.clone()
    cu = cu_of(counts)

    def f(q, pk, pv, sl, k, v, bt, cu):
        out, lse = rfa.cp_flash_attn_with_kvcache(q, pk, pv, sl, k, v, append_rank=0, return_softmax_lse=True,
                                                  block_table=bt, cu_seqlens_q=cu, max_seqlen_q=6)
        return out * 1.0, lse

    out, lse = torch.compile(f, backend="aot_eager", fullgraph=True)(q, pk, pv, lens[0], k, v, table, cu)
    ref_out, ref_lse = f(q, pk2, pv2, lens[0], k, v, table, cu)
    assert lse.shape == (8, 7)
    assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse)
    assert torch.equal(pk.nan_to_num(7.0), pk2.nan_to_num(7.0))  # the compiled call appended too


def test_varlen_split_count():
    # the bound: min(B * ceil(max * G / 64), (total_q * G + 63 B) // 64)
    assert dec.tile_slots(8, 71, 64, 32, 8) == min(8 * 4, (71 * 4 + 63 * 8) // 64) == 12
    assert dec.tile_slots(2, 2, 1, 32, 8) == 2
    assert dec.tile_slots(3, 0, 5, 8, 8) == 2  # no rows: only idle slots
    assert dec.tile_slots(1, 0, 5, 8, 8) == 0
    assert dec.num_splits_varlen(1, 1, 1, 32, 8, 512 * 1024, 132) == 16
    assert dec.num_splits_varlen(8, 71, 64, 32, 8, 512 * 1024, 132) == 1  # 12 slots x 8 kv heads
    assert dec.num_splits_varlen(3, 0, 5, 8, 8, 4096, 132) == 8
    assert dec.num_splits_varlen(1, 0, 5, 8, 8, 4096, 132) == 16  # no slots at all: still a valid count
    # equal counts: exactly the uniform call's split count, and the bound is the uniform grid
    for b, sq, hq, hkv, s_cap in itertools.product((1, 2, 3, 8, 33, 200), (1, 2, 5, 16, 64, 100), (8, 32, 64),
                                                   (1, 8), (200, 32768, 524288)):
        g = hq // hkv
        assert dec.tile_slots(b, b * sq, sq, hq, hkv) == b * -(-sq * g // 64)
        assert dec.num_splits_varlen(b, b * sq, sq, hq, hkv, s_cap, 132) == dec.num_splits(b, sq, hq, hkv, s_cap, 132)
    # the bound covers every ragged split of total_q into counts <= max
    g = 4
    for counts in ((1, 0, 70, 3), (16, 16, 15), (0, 0, 64), (1,) * 40, (17, 1, 1, 33)):
        tiles = sum(-(-n * g // 64) for n in counts)
        assert tiles <= dec.tile_slots(len(counts), sum(counts), max(counts), 4 * g, 4)


def test_bench_decode_dry_run_mixed_chunk():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "benchmark", "bench_decode.py"), "--dry-run",
                        "--mixed-chunk", "64", "--batch", "8", "32", "--cache", "32768"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:]
    rows = [json.loads(line) for line in r.stdout.splitlines() if line.startswith("{")]
    assert [(x["batch"], x["mixed_chunk"]) for x in rows] == [(8, 64), (32, 64)]
    x = rows[0]  # G = 4: the chunk is 4 row tiles, the 7 one-token sequences one each
    assert x["varlen_total_q"] == 71 and x["tile_slots"] == 12
    assert x["varlen_splits"] == dec.num_splits_varlen(8, 71, 64, 32, 8, 32768, 132)
    assert x["padded_splits"] == dec.num_splits(8, 64, 32, 8, 32768, 132)
    shard = 32768 * 8 * 128 * 2 * 2
    assert x["varlen_kv_bytes"] == 11 * shard and x["padded_kv_bytes"] == 32 * shard
    assert "splits" in x and x["kv_bytes"] == 8 * shard  # the default fields are still there
