"""cp_flash_attn_with_kvcache over fp8 (e4m3) caches with per-(sequence, kv head) descales, on CPU / gloo (worlds
1-4): against the fp64 oracle over the dequantised caches, the cache bytes after an append, the guards,
torch.compile and a dry run of the benchmark."""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist

import ring_flash_attn_b200 as rfa
from dist_utils import run_distributed
from test_decode import decode_oracle, make_case
from test_decode_paged import append_to_pool, to_pool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E4M3 = torch.float8_e4m3fn
OUT_TOL = dict(atol=1e-2, rtol=1e-2)  # out is rounded to bf16
LSE_TOL = dict(atol=1e-4, rtol=1e-4)
PAGE_SIZES = (None, 16, 128)


def quantize(x, descale):
    """Reference e4m3 storage of x (B, Sq, Hkv, D) with a (B, Hkv) descale."""
    return (x.float() / descale[:, None, :, None]).clamp(-448, 448).to(E4M3)


def dequantize(x8, descale):
    return x8.float() * descale[:, None, :, None]


def descales(b, hkv, rank, n, which):
    """Descales in one of the three accepted shapes (chosen by n), different on every rank and for K and V; the
    full (B, Hkv) values are returned too.  0.37 is not a power of two."""
    base = 0.37 * (1 + 0.25 * rank) * (1.5 if which == "v" else 1.0)
    full = base * (1 + 0.1 * torch.arange(b * hkv, dtype=torch.float32)).view(b, hkv)
    shape = n % 3
    if shape == 0:
        return torch.tensor(base), torch.full((b, hkv), base)
    if shape == 1:
        return full[0].clone(), full[0].expand(b, hkv).clone()
    return full, full


def fp8_case(world, sq, grp, seed, page_size, b=3, hkv=2, d=16):
    """make_case with e4m3 caches (NaN bytes past the valid rows) and bf16 q / k / v.  With a page size the capacity
    is a whole number of pages.  Inputs include saturating values and +-inf."""
    s_cap = 37 if page_size is None else max(2, -(-48 // page_size)) * page_size
    caches, lens, q, k, v = make_case(world, b, sq, hkv * grp, hkv, d, s_cap, seed)
    k[0, 0, 0, :4] = torch.tensor([1e6, -1e6, float("inf"), float("-inf")])
    v[-1, -1, -1, -3:] = torch.tensor([-1e5, float("inf"), 3e3])
    ds = [[descales(b, hkv, r, seed + r, w) for w in "kv"] for r in range(world)]
    f8 = [(quantize(kc, ds[r][0][1]), quantize(vc, ds[r][1][1])) for r, (kc, vc) in enumerate(caches)]
    return f8, lens, ds, q.bfloat16(), k.bfloat16(), v.bfloat16()


CASES = [(sq, grp, causal, append) for sq in (1, 4) for grp in (1, 4, 8) for causal in (True, False)
         for append in (True, False)]


def _run_fp8(rank, world, page_sizes, cases):
    for ps in page_sizes:
        for n, (sq, grp, causal, append) in enumerate(cases):
            seed = 1000 * world + n + (ps or 0)
            f8, lens, ds, q, k, v = fp8_case(world, sq, grp, seed, ps)
            (kd_arg, kd), (vd_arg, vd) = ds[rank]
            ar = (n % world) if append else None
            kn, vn = (k, v) if append else (None, None)
            kc, vc = f8[rank][0].clone(), f8[rank][1].clone()
            table = None
            if ps is not None:
                alloc = (lens[rank] + sq).clamp(max=kc.shape[1])
                kc, vc, table = to_pool(kc, vc, lens[rank], ps, alloc=alloc, seed=seed + rank)
            kc0, vc0 = kc.clone(), vc.clone()
            out, lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, lens[rank], kn, vn, append_rank=ar, causal=causal,
                                                      return_softmax_lse=True, block_table=table,
                                                      k_descale=kd_arg, v_descale=vd_arg)
            assert out.dtype == torch.bfloat16
            # the oracle over every rank's dequantised cache plus the appended rows as the append rank stores them
            deq = [(dequantize(a, ds[r][0][1]), dequantize(c, ds[r][1][1])) for r, (a, c) in enumerate(f8)]
            k_ref = v_ref = None
            if append:
                k_ref = dequantize(quantize(k, ds[ar][0][1]), ds[ar][0][1])
                v_ref = dequantize(quantize(v, ds[ar][1][1]), ds[ar][1][1])
            ref_out, ref_lse = decode_oracle(q.float(), deq, lens, k_ref, v_ref, causal)
            torch.testing.assert_close(out.float(), ref_out, **OUT_TOL)
            torch.testing.assert_close(lse, ref_lse, **LSE_TOL)
            # the cache bytes: the reference quantisation at the appended rows, every other byte untouched
            want_k, want_v = kc0, vc0
            if append and rank == ar:
                qk, qv = quantize(k, kd), quantize(v, vd)
                if ps is None:
                    want_k, want_v = kc0.clone(), vc0.clone()
                    for i in range(q.shape[0]):
                        n0 = int(lens[rank][i])
                        m = min(sq, kc.shape[1] - n0)
                        want_k[i, n0:n0 + m], want_v[i, n0:n0 + m] = qk[i, :m], qv[i, :m]
                else:
                    want_k, want_v = append_to_pool(kc0, table, lens[rank], qk), append_to_pool(vc0, table, lens[rank],
                                                                                                qv)
            assert torch.equal(kc.view(torch.uint8), want_k.view(torch.uint8))
            assert torch.equal(vc.view(torch.uint8), want_v.view(torch.uint8))
            if world > 1:  # bitwise the same on every rank
                both = torch.cat([out.float().reshape(-1), lse.reshape(-1)])
                got = [torch.empty_like(both) for _ in range(world)]
                dist.all_gather(got, both)
                for x in got:
                    assert torch.equal(x.nan_to_num(7.0), both.nan_to_num(7.0))


@pytest.mark.parametrize("page_size", PAGE_SIZES)
def test_fp8_world1_matches_oracle(page_size):
    _run_fp8(0, 1, (page_size,), CASES)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_fp8_gloo_worlds_match_oracle(world):
    run_distributed(_run_fp8, world, PAGE_SIZES, CASES)


def test_append_quantisation_bytes():
    """Saturation, +-inf, ties and subnormals with a descale that is not a power of two."""
    b, sq, hkv, d = 1, 1, 1, 16
    kc = torch.zeros(b, 4, hkv, d, dtype=E4M3)
    vc = kc.clone()
    vals = torch.tensor([1e6, -1e6, float("inf"), float("-inf"), 448 * 0.37, 460 * 0.37, 1e-3, -1e-3, 2.0 ** -9,
                         0.37 * 2.0 ** -10, 0.37 * 1.0625, 0.37 * 1.1875, 0.0, -0.0, 17.0, -3.3])
    k = vals.view(b, sq, hkv, d).bfloat16()
    v = (-vals).view(b, sq, hkv, d).bfloat16()
    q = torch.randn(b, sq, 2, d).bfloat16()
    ds = torch.tensor(0.37)
    sl = torch.tensor([2], dtype=torch.int32)
    rfa.cp_flash_attn_with_kvcache(q, kc, vc, sl, k, v, append_rank=0, k_descale=ds, v_descale=ds)
    want = quantize(k, ds.expand(1, 1))[0, 0].view(torch.uint8)
    assert torch.equal(kc[0, 2].view(torch.uint8), want)
    assert torch.equal(vc[0, 2].view(torch.uint8), quantize(v, ds.expand(1, 1))[0, 0].view(torch.uint8))
    assert kc[0, 2, 0, 2].float() == 448 and kc[0, 2, 0, 3].float() == -448  # +-inf saturate


def test_fp8_guards():
    f8, lens, ds, q, k, v = fp8_case(1, 1, 2, 0, None, b=2)
    kc, vc = f8[0]
    sl = lens[0]
    one = torch.tensor(1.0)
    f = rfa.cp_flash_attn_with_kvcache
    with pytest.raises(ValueError, match="fp8 queries"):
        f(q.to(E4M3), kc, vc, sl, k_descale=one, v_descale=one)
    with pytest.raises(ValueError, match="fp8 caches must be torch.float8_e4m3fn"):
        f(q, kc.to(torch.float8_e5m2), vc.to(torch.float8_e5m2), sl, k_descale=one, v_descale=one)
    with pytest.raises(ValueError, match="fp8 caches: k_cache"):
        f(q, kc, vc.bfloat16(), sl, k_descale=one, v_descale=one)
    with pytest.raises(ValueError, match="fp8 caches need a bf16 / fp16 q"):
        f(q.float(), kc, vc, sl, k_descale=one, v_descale=one)
    with pytest.raises(ValueError, match="fp8 caches need k_descale"):
        f(q, kc, vc, sl, v_descale=one)
    with pytest.raises(ValueError, match="fp8 caches need v_descale"):
        f(q, kc, vc, sl, k_descale=one)
    with pytest.raises(ValueError, match="fp8 k_descale must be a float32 tensor"):
        f(q, kc, vc, sl, k_descale=one.double(), v_descale=one)
    with pytest.raises(ValueError, match="fp8 v_descale must be a float32 tensor"):
        f(q, kc, vc, sl, k_descale=one, v_descale=1.0)
    with pytest.raises(ValueError, match="fp8 k_descale must be on q's device"):
        f(q, kc, vc, sl, k_descale=one.to("meta"), v_descale=one)
    for bad in (torch.ones(3), torch.ones(2, 3), torch.ones(1, 2), torch.ones(2, 2, 1)):
        with pytest.raises(ValueError, match="fp8 v_descale must have shape"):
            f(q, kc, vc, sl, k_descale=one, v_descale=bad)
    with pytest.raises(ValueError, match="only taken with fp8"):
        f(q, kc.bfloat16(), vc.bfloat16(), sl, k_descale=one, v_descale=one)
    with pytest.raises(ValueError, match="only taken with fp8"):
        f(q, kc.bfloat16(), vc.bfloat16(), sl, v_descale=one)
    with pytest.raises(ValueError, match="q's dtype"):  # new rows stay in q's dtype
        f(q, kc, vc, sl, k.to(E4M3), v.to(E4M3), append_rank=0, k_descale=one, v_descale=one)


def test_torch_compile_fullgraph_fp8():
    f8, lens, ds, q, k, v = fp8_case(1, 4, 4, 1, 16, b=2)
    kc, vc = f8[0]
    pk, pv, table = to_pool(kc, vc, lens[0], 16, alloc=lens[0] + 4)
    pk2, pv2 = pk.clone(), pv.clone()
    kd, vd = ds[0][0][0], ds[0][1][0]

    def f(q, pk, pv, sl, k, v, bt, kd, vd):
        out, lse = rfa.cp_flash_attn_with_kvcache(q, pk, pv, sl, k, v, append_rank=0, return_softmax_lse=True,
                                                  block_table=bt, k_descale=kd, v_descale=vd)
        return out * 1.0, lse

    out, lse = torch.compile(f, backend="aot_eager", fullgraph=True)(q, pk, pv, lens[0], k, v, table, kd, vd)
    ref_out, ref_lse = f(q, pk2, pv2, lens[0], k, v, table, kd, vd)
    assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse)
    assert torch.equal(pk.view(torch.uint8), pk2.view(torch.uint8))  # the compiled call appended too


def test_bench_decode_dry_run_fp8():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "benchmark", "bench_decode.py"), "--dry-run",
                        "--kv-dtype", "e4m3", "--batch", "1", "8", "--cache", "32768", "524288"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:]
    rows = [json.loads(line) for line in r.stdout.splitlines() if line.startswith("{")]
    assert [(x["batch"], x["cache_tokens"]) for x in rows] == [(1, 32768), (1, 524288), (8, 32768), (8, 524288)]
    for x in rows:
        assert x["kv_dtype"] == "e4m3" and 2 * x["fp8_kv_bytes"] == x["kv_bytes"]
    assert rows[-1]["fp8_kv_bytes"] == 8 * 524288 * 8 * 128 * 2
