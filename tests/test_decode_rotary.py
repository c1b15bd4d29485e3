"""cp_flash_attn_with_kvcache with rotary embeddings (``rotary_cos=`` / ``rotary_sin=`` / ``rotary_seqlens=``) on
CPU / gloo (worlds 1-4): bitwise a plain call on ``apply_rotary``-rotated q / k (out, lse and the cache bytes after
the append), bitwise the same on every rank, and the fp64 decode oracle on the rotated inputs, over contiguous, paged
and e4m3 caches, uniform and varlen queries, causal and not, interleaved and not, rotary_dim in {D, D/2, 16}; the
one-rank default, the dense path's range check, the guards, torch.compile and a dry run of the benchmark."""
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
from test_decode_varlen import COUNTS, cu_of, pack, varlen_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S_CAP, D, HKV, GRP = 128, 64, 2, 2
CASES = [(varlen, causal, interleaved, rotary_dim) for varlen in (False, True) for causal in (True, False)
         for interleaved in (True, False) for rotary_dim in (D, D // 2, 16)]


def rope_tables(seqlen_ro, rotary_dim, dtype, device="cpu", base=10000.0):
    """The usual RoPE cos / sin tables (seqlen_ro, rotary_dim / 2), computed in fp64 and rounded to dtype."""
    inv = base ** (-torch.arange(0, rotary_dim, 2, dtype=torch.float64) / rotary_dim)
    ang = torch.arange(seqlen_ro, dtype=torch.float64)[:, None] * inv[None]
    return ang.cos().to(dtype).to(device), ang.sin().to(dtype).to(device)


def grid_positions(rotary_seqlens, sq, causal):
    """(B, Sq) table rows of the new keys and of the query tokens (the first token's when not causal)."""
    rs = rotary_seqlens.long().cpu()[:, None]
    keys = rs + torch.arange(sq)[None]
    return keys, (keys if causal else rs.expand_as(keys))


def rotate_grid(q4, k4, cos, sin, rotary_seqlens, causal, interleaved):
    """q4 (B, Sq, Hq, D) / k4 (B, Sq, Hkv, D) as the rotary call sees them."""
    keys, queries = grid_positions(rotary_seqlens, q4.shape[1], causal)
    return (dec.apply_rotary(q4, cos, sin, queries.to(q4.device), interleaved),
            dec.apply_rotary(k4, cos, sin, keys.to(k4.device), interleaved))


def _run_rotary(rank, world, kinds, cases):
    for kind in kinds:  # "contiguous", "paged16", "fp8"
        fp8 = kind == "fp8"
        ps = int(kind.split("paged")[1]) if "paged" in kind else None
        for n, (varlen, causal, interleaved, rotary_dim) in enumerate(cases):
            counts = COUNTS[n % len(COUNTS)] if varlen else (3, 3, 3)
            seed = 2000 * world + 37 * len(kind) + n
            b, smax = len(counts), max(counts)
            caches, lens, q4, k4, v4 = make_case(world, b, smax, HKV * GRP, HKV, D, S_CAP, seed)
            dtype = torch.bfloat16 if fp8 else torch.float32
            q4, k4, v4 = q4.to(dtype), k4.to(dtype), v4.to(dtype)
            ar = n % world
            ds = None
            if fp8:
                ds = [(0.37 * (1 + 0.25 * r) * torch.ones(b, HKV), 0.55 * (1 + 0.1 * r) * torch.ones(b, HKV))
                      for r in range(world)]
                caches = [(quantize(kc, kd), quantize(vc, vd)) for (kc, vc), (kd, vd) in zip(caches, ds)]
            # global positions: the cached tokens of every rank come first
            rs = (sum(x.long() for x in lens) + 3 * torch.arange(b)).to(torch.int32)
            cos, sin = rope_tables(world * S_CAP + 100, rotary_dim, dtype)
            q4r, k4r = rotate_grid(q4, k4, cos, sin, rs, causal, interleaved)
            if varlen:
                q, k, v, qr, kr = (pack(x, counts) for x in (q4, k4, v4, q4r, k4r))
                vl = dict(cu_seqlens_q=cu_of(counts), max_seqlen_q=smax)
            else:
                q, k, v, qr, kr, vl = q4, k4, v4, q4r, k4r, {}
            kc, vc = caches[rank][0].clone(), caches[rank][1].clone()
            table = None
            if ps is not None:
                alloc = (lens[rank] + torch.tensor(counts)).clamp(max=S_CAP)
                kc, vc, table = to_pool(kc, vc, lens[rank], ps, alloc=alloc, seed=seed + rank)
            kc2, vc2 = kc.clone(), vc.clone()
            kw = dict(append_rank=ar, causal=causal, return_softmax_lse=True, block_table=table, **vl)
            if fp8:
                kw.update(k_descale=ds[rank][0], v_descale=ds[rank][1])
            out, lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, lens[rank], k, v, rotary_cos=cos, rotary_sin=sin,
                                                      rotary_interleaved=interleaved, rotary_seqlens=rs, **kw)
            p_out, p_lse = rfa.cp_flash_attn_with_kvcache(qr, kc2, vc2, lens[rank], kr, v, **kw)
            assert torch.equal(out, p_out) and torch.equal(lse, p_lse), (kind, n)
            for a, c in ((kc, kc2), (vc, vc2)):
                assert torch.equal(a.view(torch.uint8), c.view(torch.uint8)), (kind, n)
            # the oracle on the rotated inputs
            if fp8:
                ref_caches = [(dequantize(a, x), dequantize(c, y)) for (a, c), (x, y) in zip(caches, ds)]
                kn = dequantize(quantize(k4r, ds[ar][0]), ds[ar][0])
                vn = dequantize(quantize(v4, ds[ar][1]), ds[ar][1])
                qo, tol_out, tol_lse = q4r.float(), OUT_TOL, LSE_TOL
            else:
                ref_caches, kn, vn, qo, tol_out, tol_lse = caches, k4r, v4, q4r, TOL, TOL
            if varlen:
                ref_out, ref_lse = varlen_oracle(qo, ref_caches, lens, kn, vn, counts, causal)
            else:
                ref_out, ref_lse = decode_oracle(qo, ref_caches, lens, kn, vn, causal)
            torch.testing.assert_close(out.float(), ref_out, **tol_out)
            torch.testing.assert_close(lse, ref_lse, **tol_lse)
            if world > 1:  # bitwise the same on every rank
                both = torch.cat([out.float().reshape(-1), lse.reshape(-1)])
                got = [torch.empty_like(both) for _ in range(world)]
                dist.all_gather(got, both)
                for x in got:
                    assert torch.equal(x.nan_to_num(7.0), both.nan_to_num(7.0))


KINDS = ("contiguous", "paged16", "fp8")


@pytest.mark.parametrize("kind", KINDS)
def test_rotary_world1_is_the_plain_call_on_rotated_inputs(kind):
    _run_rotary(0, 1, (kind,), CASES)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_rotary_gloo_worlds_are_the_plain_call_on_rotated_inputs(world):
    run_distributed(_run_rotary, world, KINDS, CASES)


def test_apply_rotary_formula():
    """The helper against the formula written out element by element, in fp32 without FMA."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 3, 32, generator=g).bfloat16()
    cos, sin = rope_tables(10, 16, torch.bfloat16)
    pos = torch.tensor([[4, 9]])
    for interleaved in (True, False):
        y = dec.apply_rotary(x[None], cos, sin, pos, interleaved)[0]
        for r in range(2):
            c, s = cos[pos[0, r]].float(), sin[pos[0, r]].float()
            for hd in range(3):
                xr = x[r, hd].float()
                for i in range(8):
                    ia, ib = (2 * i, 2 * i + 1) if interleaved else (i, i + 8)
                    a = (xr[ia] * c[i]) - (xr[ib] * s[i])
                    bb = (xr[ib] * c[i]) + (xr[ia] * s[i])
                    assert y[r, hd, ia] == a.bfloat16() and y[r, hd, ib] == bb.bfloat16()
                assert torch.equal(y[r, hd, 16:], x[r, hd, 16:])


@pytest.mark.parametrize("causal", [True, False])
def test_one_rank_default_is_cache_seqlens(causal):
    caches, lens, q, k, v = make_case(1, 3, 2, 4, 2, 32, 40, seed=4)
    cos, sin = rope_tables(64, 32, torch.float32)
    kc, vc = caches[0]
    kc2, vc2 = kc.clone(), vc.clone()
    kw = dict(append_rank=0, causal=causal, return_softmax_lse=True, rotary_cos=cos, rotary_sin=sin,
              rotary_interleaved=False)
    out, lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, lens[0], k, v, **kw)
    out2, lse2 = rfa.cp_flash_attn_with_kvcache(q, kc2, vc2, lens[0], k, v, rotary_seqlens=lens[0].clone(), **kw)
    assert torch.equal(out, out2) and torch.equal(lse, lse2)
    assert torch.equal(kc.nan_to_num(7.0), kc2.nan_to_num(7.0))


def test_non_causal_queries_share_the_first_position():
    """Non-causal: every query token of a sequence is rotated at rotary_seqlens[b] (and the result differs from
    rotating them at rotary_seqlens[b] + t, so the check is not vacuous)."""
    caches, lens, q, k, v = make_case(1, 2, 3, 4, 2, 32, 40, seed=6)
    cos, sin = rope_tables(64, 32, torch.float32)
    rs = torch.tensor([5, 17], dtype=torch.int32)
    kc, vc = caches[0]
    out = rfa.cp_flash_attn_with_kvcache(q, kc.clone(), vc.clone(), lens[0], k, v, append_rank=0, causal=False,
                                         rotary_cos=cos, rotary_sin=sin, rotary_seqlens=rs)
    keys = rs.long()[:, None] + torch.arange(3)[None]
    kr = dec.apply_rotary(k, cos, sin, keys)
    first = dec.apply_rotary(q, cos, sin, rs.long()[:, None].expand(2, 3))
    per_token = dec.apply_rotary(q, cos, sin, keys)
    want = rfa.cp_flash_attn_with_kvcache(first, kc.clone(), vc.clone(), lens[0], kr, v, append_rank=0, causal=False)
    other = rfa.cp_flash_attn_with_kvcache(per_token, kc.clone(), vc.clone(), lens[0], kr, v, append_rank=0,
                                           causal=False)
    assert torch.equal(out, want) and not torch.equal(out, other)


def test_dense_path_raises_for_positions_past_the_tables():
    caches, lens, q, k, v = make_case(1, 2, 3, 4, 2, 32, 40, seed=2)
    cos, sin = rope_tables(20, 32, torch.float32)
    kc, vc = caches[0]
    f = rfa.cp_flash_attn_with_kvcache
    kw = dict(append_rank=0, rotary_cos=cos, rotary_sin=sin)
    f(q, kc.clone(), vc.clone(), lens[0], k, v, rotary_seqlens=torch.tensor([17, 0], dtype=torch.int32), **kw)
    for bad in ([18, 0], [0, -1]):
        with pytest.raises(ValueError, match="outside the 20-row rotary tables"):
            f(q, kc.clone(), vc.clone(), lens[0], k, v, rotary_seqlens=torch.tensor(bad, dtype=torch.int32), **kw)
    # varlen: only the sequence's own tokens count, and a sequence with no tokens has no position
    cu = cu_of([3, 0])
    f(q[0], kc.clone(), vc.clone(), lens[0], k[0], v[0], cu_seqlens_q=cu, max_seqlen_q=3,
      rotary_seqlens=torch.tensor([17, 99], dtype=torch.int32), **kw)


def test_rotary_guards():
    caches, lens, q, k, v = make_case(1, 2, 3, 4, 2, 32, 40, seed=0)
    kc, vc = caches[0]
    sl = lens[0]
    cos, sin = rope_tables(64, 32, torch.float32)
    rs = torch.tensor([3, 4], dtype=torch.int32)
    f = rfa.cp_flash_attn_with_kvcache

    def call(**kw):
        base = dict(rotary_cos=cos, rotary_sin=sin, rotary_seqlens=rs)
        base.update(kw)
        return f(q, kc.clone(), vc.clone(), sl, k, v, append_rank=0, **{x: y for x, y in base.items()
                                                                         if y is not _DROP})

    with pytest.raises(ValueError, match="need k / v"):
        f(q, kc, vc, sl, rotary_cos=cos, rotary_sin=sin, rotary_seqlens=rs)
    with pytest.raises(ValueError, match="pass both rotary_cos and rotary_sin"):
        call(rotary_sin=_DROP)
    with pytest.raises(ValueError, match="pass both rotary_cos and rotary_sin"):
        call(rotary_cos=_DROP)
    with pytest.raises(ValueError, match="must have the same shape"):
        call(rotary_sin=sin[:, :8].contiguous())
    with pytest.raises(ValueError, match="must have the same shape"):
        call(rotary_sin=sin[:10])
    for rotary_dim in (8, 24, 48):  # not a multiple of 16, or above D = 32
        c2, s2 = rope_tables(64, rotary_dim, torch.float32)
        with pytest.raises(ValueError, match="rotary_dim"):
            call(rotary_cos=c2, rotary_sin=s2)
    with pytest.raises(ValueError, match="rotary_dim"):
        call(rotary_cos=cos[:, :0].contiguous(), rotary_sin=sin[:, :0].contiguous())
    with pytest.raises(ValueError, match="between 1 and"):
        call(rotary_cos=cos[:0], rotary_sin=sin[:0])
    with pytest.raises(ValueError, match="rotary_cos must have q's dtype"):
        call(rotary_cos=cos.double())
    with pytest.raises(ValueError, match="rotary_sin must have q's dtype"):
        call(rotary_sin=sin.bfloat16())
    with pytest.raises(ValueError, match="rotary_cos must be on q's device"):
        call(rotary_cos=cos.to("meta"))
    for bad in (cos.t(), cos[None], cos[:, 0], cos.tolist()):
        with pytest.raises(ValueError, match="rotary_cos must be a contiguous"):
            call(rotary_cos=bad)
    for bad in (rs.long(), rs[:1], rs.view(1, 2), torch.zeros(4, dtype=torch.int32)[::2], [3, 4]):
        with pytest.raises(ValueError, match="rotary_seqlens must be a contiguous"):
            call(rotary_seqlens=bad)
    with pytest.raises(ValueError, match="rotary_seqlens must be on q's device"):
        call(rotary_seqlens=rs.to("meta"))
    with pytest.raises(ValueError, match="rotary_seqlens is only taken with rotary_cos"):
        call(rotary_cos=_DROP, rotary_sin=_DROP)
    call()  # and the well-formed call runs


_DROP = object()


def _missing_positions(rank, world):
    caches, lens, q, k, v = make_case(world, 2, 1, 4, 2, 32, 40, seed=1)
    cos, sin = rope_tables(128, 32, torch.float32)
    kc, vc = caches[rank]
    with pytest.raises(ValueError, match="rotary_seqlens is required in a group of more than one rank"):
        rfa.cp_flash_attn_with_kvcache(q, kc, vc, lens[rank], k, v, append_rank=0, rotary_cos=cos, rotary_sin=sin)


def test_rotary_seqlens_required_in_a_larger_group():
    run_distributed(_missing_positions, 2)


def test_torch_compile_fullgraph_rotary():
    counts = (1, 0, 6)
    caches, lens, q4, k4, v4 = make_case(1, 3, 6, 8, 2, 32, 32, seed=1)
    q, k, v = pack(q4, counts), pack(k4, counts), pack(v4, counts)
    kc, vc = caches[0]
    pk, pv, table = to_pool(kc, vc, lens[0], 16, alloc=(lens[0] + 6).clamp(max=32))
    pk2, pv2 = pk.clone(), pv.clone()
    cu = cu_of(counts)
    cos, sin = rope_tables(64, 16, torch.float32)
    rs = torch.tensor([7, 0, 30], dtype=torch.int32)

    def f(q, pk, pv, sl, k, v, bt, cu, cos, sin, rs):
        out, lse = rfa.cp_flash_attn_with_kvcache(q, pk, pv, sl, k, v, append_rank=0, return_softmax_lse=True,
                                                  block_table=bt, cu_seqlens_q=cu, max_seqlen_q=6, rotary_cos=cos,
                                                  rotary_sin=sin, rotary_seqlens=rs, rotary_interleaved=False)
        return out * 1.0, lse

    args = (q, pk, pv, lens[0], k, v, table, cu, cos, sin, rs)
    out, lse = torch.compile(f, backend="aot_eager", fullgraph=True)(*args)
    ref_out, ref_lse = f(q, pk2, pv2, *args[3:])
    assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse)
    assert torch.equal(pk.nan_to_num(7.0), pk2.nan_to_num(7.0))  # the compiled call appended the rotated keys


def test_bench_decode_dry_run_rotary():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "benchmark", "bench_decode.py"), "--dry-run", "--rotary",
                        "--batch", "1", "8", "--cache", "32768"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:]
    rows = [json.loads(line) for line in r.stdout.splitlines() if line.startswith("{")]
    assert [(x["batch"], x["rotary_dim"]) for x in rows] == [(1, 128), (8, 128)]
    assert rows[0]["rotary_interleaved"] is False and rows[0]["seqlen_ro"] == 32768
    assert "splits" in rows[0] and "kv_bytes" in rows[0]  # the default fields are still there
