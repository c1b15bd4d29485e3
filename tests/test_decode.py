"""cp_flash_attn_with_kvcache on CPU / gloo (worlds 1-4) against an fp32 oracle over the gathered cache."""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist

import ring_flash_attn_b200 as rfa
from ring_flash_attn_b200.ops.dense import attention_oracle
from ring_flash_attn_b200.parallel import decode as dec
from ring_flash_attn_b200.parallel import layouts
from dist_utils import run_distributed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = dict(atol=2e-5, rtol=2e-4)


def decode_oracle(q, caches, lens, k_new, v_new, causal, scale=None):
    """fp64 attention of q (B, Sq, Hq, D) over the valid rows of every rank's cache (``caches``: list of
    (k_cache, v_cache) before the append, ``lens``: per-rank lists of valid rows) plus the appended keys.
    Returns (out (B, Sq, Hq, D), lse (B, Hq, Sq)) in fp32."""
    b, sq, hq, d = q.shape
    scale = d ** -0.5 if scale is None else scale
    outs, lses = [], []
    for i in range(b):
        ks = [kc[i, :int(n[i])] for (kc, _), n in zip(caches, lens)]
        vs = [vc[i, :int(n[i])] for (_, vc), n in zip(caches, lens)]
        n_old = sum(x.shape[0] for x in ks)
        if k_new is not None:
            ks.append(k_new[i])
            vs.append(v_new[i])
        kk = torch.cat(ks).double()
        vv = torch.cat(vs).double()
        rep = hq // kk.shape[1]
        kk, vv = kk.repeat_interleave(rep, dim=1), vv.repeat_interleave(rep, dim=1)
        s = torch.einsum("thd,jhd->htj", q[i].double(), kk) * scale  # (Hq, Sq, keys)
        if k_new is not None and causal:
            t = torch.arange(sq).unsqueeze(1)
            j = torch.arange(kk.shape[0]).unsqueeze(0)
            s = s.masked_fill((j >= n_old + t + 1).unsqueeze(0), float("-inf"))
        lse = torch.logsumexp(s, dim=-1)
        p = torch.exp(s - torch.where(torch.isinf(lse), torch.zeros_like(lse), lse).unsqueeze(-1))
        outs.append(torch.einsum("htj,jhd->thd", p, vv))
        lses.append(lse)
    return torch.stack(outs).float(), torch.stack(lses).float()


def make_case(world, b, sq, hq, hkv, d, s_cap, seed, dtype=torch.float32, device="cpu"):
    """Per-rank caches (garbage past the valid rows), ragged valid lengths with zeros, q and the new k / v; the same
    on every rank for a given seed."""
    g = torch.Generator().manual_seed(seed)
    caches, lens = [], []
    for r in range(world):
        kc = torch.randn(b, s_cap, hkv, d, generator=g)
        vc = torch.randn(b, s_cap, hkv, d, generator=g)
        n = torch.randint(0, s_cap - sq + 1, (b,), generator=g)
        n[(r + seed) % b] = 0  # an empty shard for some sequence
        for i in range(b):
            kc[i, int(n[i]):] = float("nan")  # rows past the valid ones must never reach a result
            vc[i, int(n[i]):] = float("nan")
        caches.append((kc.to(dtype).to(device), vc.to(dtype).to(device)))
        lens.append(n.to(torch.int32).to(device))
    q = torch.randn(b, sq, hq, d, generator=g).to(dtype).to(device)
    k = torch.randn(b, sq, hkv, d, generator=g).to(dtype).to(device)
    v = torch.randn(b, sq, hkv, d, generator=g).to(dtype).to(device)
    return caches, lens, q, k, v


CASES = [(sq, grp, causal, append) for sq in (1, 4) for grp in (1, 4, 8) for causal in (True, False)
         for append in (True, False)]


def _run_cases(rank, world, cases):
    for n, (sq, grp, causal, append) in enumerate(cases):
        hkv = 2
        caches, lens, q, k, v = make_case(world, 3, sq, hkv * grp, hkv, 16, 37, seed=100 * world + n)
        ar = (n % world) if append else None
        kc, vc = caches[rank][0].clone(), caches[rank][1].clone()
        out, lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, lens[rank], k if append else None,
                                                  v if append else None, append_rank=ar, causal=causal,
                                                  return_softmax_lse=True)
        ref_out, ref_lse = decode_oracle(q, caches, lens, k if append else None, v if append else None, causal)
        torch.testing.assert_close(out, ref_out, **TOL)
        torch.testing.assert_close(lse, ref_lse, **TOL)
        # the cache: k / v at rows [len, len + Sq) of the append rank, every other row untouched
        want_k, want_v = caches[rank][0].clone(), caches[rank][1].clone()
        if append and rank == ar:
            for i in range(q.shape[0]):
                n0 = int(lens[rank][i])
                want_k[i, n0:n0 + sq], want_v[i, n0:n0 + sq] = k[i], v[i]
        assert torch.equal(kc.nan_to_num(7.0), want_k.nan_to_num(7.0))
        assert torch.equal(vc.nan_to_num(7.0), want_v.nan_to_num(7.0))
        if world > 1:  # bitwise the same on every rank
            both = torch.cat([out.reshape(-1), lse.reshape(-1)])
            got = [torch.empty_like(both) for _ in range(world)]
            dist.all_gather(got, both)
            for x in got:
                assert torch.equal(x.nan_to_num(7.0), both.nan_to_num(7.0))


def test_world1_matches_oracle():
    _run_cases(0, 1, CASES)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_gloo_worlds_match_oracle(world):
    run_distributed(_run_cases, world, CASES)


def test_argument_guards():
    caches, lens, q, k, v = make_case(1, 2, 1, 4, 2, 16, 8, seed=0)
    kc, vc = caches[0]
    sl = lens[0]
    f = rfa.cp_flash_attn_with_kvcache
    with pytest.raises(ValueError, match="sliding windows"):
        f(q, kc, vc, sl, window_size=(4, 0))
    with pytest.raises(ValueError, match="alibi"):
        f(q, kc, vc, sl, alibi_slopes=torch.ones(4))
    with pytest.raises(ValueError, match="fp8"):
        f(q, kc.to(torch.float8_e4m3fn), vc.to(torch.float8_e4m3fn), sl)
    big = torch.zeros(2, 1, 4, 192)
    with pytest.raises(ValueError, match="192 > 128"):
        f(big, torch.zeros(2, 8, 2, 192), torch.zeros(2, 8, 2, 192), sl)
    with pytest.raises(ValueError, match="multiple of kv heads"):
        f(torch.zeros(2, 1, 3, 16), kc, vc, sl)
    with pytest.raises(ValueError, match="append_rank is required"):
        f(q, kc, vc, sl, k, v)
    with pytest.raises(ValueError, match="append_rank must be None"):
        f(q, kc, vc, sl, append_rank=0)
    with pytest.raises(ValueError, match="both k and v"):
        f(q, kc, vc, sl, k, None, append_rank=0)
    with pytest.raises(ValueError, match="not a rank"):
        f(q, kc, vc, sl, k, v, append_rank=1)
    with pytest.raises(ValueError, match="int32"):
        f(q, kc, vc, sl.long())


def _prefill_then_decode(rank, world):
    torch.manual_seed(0)
    b, s, hq, hkv, d = 1, 8 * world * 2, 4, 2, 16
    q, k, v = (torch.randn(b, s + 1, h, d) for h in (hq, hkv, hkv))
    for t in (q, k, v):
        dist.broadcast(t, src=0)
    lq, lk, lv = (layouts.shard_zigzag(x[:, :s], rank, world) for x in (q, k, v))
    rfa.zigzag_ring_flash_attn_func(lq, lk, lv, causal=True)  # the prefill leaves lk / lv as this rank's shard
    s_loc = lk.shape[1]
    kc = torch.zeros(b, s_loc + 4, hkv, d)
    vc = torch.zeros(b, s_loc + 4, hkv, d)
    kc[:, :s_loc], vc[:, :s_loc] = lk, lv
    sl = torch.full((b,), s_loc, dtype=torch.int32)
    out = rfa.cp_flash_attn_with_kvcache(q[:, s:], kc, vc, sl, k[:, s:], v[:, s:], append_rank=world - 1)
    ref, _ = attention_oracle(q, k, v, causal=True)
    torch.testing.assert_close(out, ref[:, s:], **TOL)


def test_zigzag_prefill_then_decode_world2():
    run_distributed(_prefill_then_decode, 2)


def test_torch_compile_fullgraph():
    caches, lens, q, k, v = make_case(1, 2, 4, 8, 2, 16, 24, seed=1)
    kc, vc = caches[0][0].clone(), caches[0][1].clone()
    kc2, vc2 = kc.clone(), vc.clone()

    def f(q, kc, vc, sl, k, v):
        out, lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, sl, k, v, append_rank=0, return_softmax_lse=True)
        return out * 1.0, lse

    out, lse = torch.compile(f, backend="aot_eager", fullgraph=True)(q, kc, vc, lens[0], k, v)
    ref_out, ref_lse = f(q, kc2, vc2, lens[0], k, v)
    torch.testing.assert_close(out, ref_out, **TOL)
    torch.testing.assert_close(lse, ref_lse, **TOL)
    assert torch.equal(kc.nan_to_num(7.0), kc2.nan_to_num(7.0))  # the compiled call appended too


def test_num_splits_from_shapes():
    # one wave of one CTA per SM, never more splits than 128-key tiles
    assert dec.num_splits(1, 1, 32, 8, 512 * 1024, 132) == 16
    assert dec.num_splits(8, 1, 32, 8, 512 * 1024, 132) == 2
    assert dec.num_splits(64, 1, 32, 8, 512 * 1024, 132) == 1
    assert dec.num_splits(1, 1, 32, 8, 200, 132) == 2
    assert dec.num_splits(1, 16, 32, 4, 1 << 20, 132) == 132 // (4 * 2)  # 16 tokens x group 8 = two row tiles


def test_bench_decode_dry_run():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "benchmark", "bench_decode.py"), "--dry-run",
                        "--batch", "1", "8", "--cache", "32768", "524288"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:]
    rows = [json.loads(line) for line in r.stdout.splitlines() if line.startswith("{")]
    assert [(x["batch"], x["cache_tokens"]) for x in rows] == [(1, 32768), (1, 524288), (8, 32768), (8, 524288)]
    x = rows[-1]
    assert x["kv_bytes"] == 8 * 524288 * 8 * 128 * 2 * 2 and x["splits"] == 2
