"""Tree masks (``tree_mask=``) in context-parallel decoding on the dense path (CPU / gloo): the fp64 oracle on random
trees over every cache layout (uniform and varlen with an empty sequence, GQA, shared prefixes, slots and left pads,
pages, e4m3 caches and queries), rotary at the tree depths, a lower-triangular mask bitwise the causal call, every
``ValueError``, two ranks against one on the concatenated cache, torch.compile and a dry run of the benchmark."""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist

import decode_tree as DT
import ring_flash_attn_b200 as rfa
from dist_utils import run_distributed
from ring_flash_attn_b200.parallel import decode as dec
from test_decode_rotary import rope_tables

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f = rfa.cp_flash_attn_with_kvcache
OUT_TOL = dict(atol=1e-2, rtol=1e-2)  # out is rounded to bf16
LSE_TOL = dict(atol=1e-4, rtol=1e-4)
VARLEN = ((13, 0, 5, 9), (30, 41, 7, 12))  # counts, cached rows (S_cap 64 with pages of 16)
UNIFORM = ((6, 6, 6, 6), (30, 0, 41, 17))


def _call(call, mask, rotary=None):
    q, kc, vc, sl, k, v, kw = call.fresh()
    if rotary is not None:
        kw.update(rotary_cos=rotary[0], rotary_sin=rotary[1], rotary_seqlens=rotary[2],
                  rotary_interleaved=rotary[3])
    out, lse = f(q, kc, vc, sl, k, v, append_rank=0, return_softmax_lse=True, tree_mask=mask, **kw)
    return out, lse, kc, vc


def _masks(call, gen, tril=False):
    per = DT.tril_masks(call.counts) if tril else DT.tree_masks(call.counts, gen)
    sq = max(max(call.counts), 1)
    return DT.packed_mask(per, sq, gen, call.varlen)


@pytest.mark.parametrize("layout", DT.LAYOUTS)
@pytest.mark.parametrize("varlen", [False, True])
def test_dense_matches_oracle_on_random_trees(layout, varlen):
    counts, lens = VARLEN if varlen else UNIFORM
    gen = torch.Generator().manual_seed(3)
    for seed in range(2):
        call = DT.build(layout, torch.bfloat16, 32, counts, lens, 64, "cpu", seed=seed, varlen=varlen)
        mask = _masks(call, gen)
        out, lse, _, _ = _call(call, mask)
        ref_out, ref_lse = DT.oracle(call, mask, 32 ** -0.5)
        got_o, got_l = DT.packed(call, out, lse)
        torch.testing.assert_close(got_o.double(), ref_out, **OUT_TOL)
        torch.testing.assert_close(got_l.double(), ref_lse, **LSE_TOL)


@pytest.mark.parametrize("interleaved", [True, False])
@pytest.mark.parametrize("varlen", [False, True])
def test_rotary_at_tree_depths(varlen, interleaved):
    counts, lens = VARLEN if varlen else UNIFORM
    gen = torch.Generator().manual_seed(4)
    call = DT.build("contiguous", torch.bfloat16, 32, counts, lens, 64, "cpu", seed=5, varlen=varlen)
    cos, sin = rope_tables(200, 32, torch.bfloat16)
    rs = torch.tensor([100, 3, 60, 0], dtype=torch.int32)
    mask = _masks(call, gen)
    out, lse, _, _ = _call(call, mask, (cos, sin, rs, interleaved))
    ref_out, ref_lse = DT.oracle(call, mask, 32 ** -0.5, rotary=(cos, sin, rs, interleaved))
    got_o, got_l = DT.packed(call, out, lse)
    torch.testing.assert_close(got_o.double(), ref_out, **OUT_TOL)
    torch.testing.assert_close(got_l.double(), ref_lse, **LSE_TOL)


@pytest.mark.parametrize("layout", DT.LAYOUTS)
@pytest.mark.parametrize("varlen", [False, True])
def test_lower_triangular_mask_is_the_causal_call(layout, varlen):
    counts, lens = VARLEN if varlen else UNIFORM
    gen = torch.Generator().manual_seed(6)
    call = DT.build(layout, torch.bfloat16, 32, counts, lens, 64, "cpu", seed=1, varlen=varlen)
    rotaries = [None]
    if layout != "q8":
        cos, sin = rope_tables(200, 16, torch.bfloat16)
        rotaries.append((cos, sin, torch.tensor([9, 0, 77, 120], dtype=torch.int32), False))
    for rot in rotaries:
        out, lse, kc, vc = _call(call, _masks(call, gen, tril=True), rot)
        ref_out, ref_lse, ref_kc, ref_vc = _call(call, None, rot)
        assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse), (layout, rot is None)
        assert torch.equal(DT.raw(kc), DT.raw(ref_kc)) and torch.equal(DT.raw(vc), DT.raw(ref_vc))


def test_value_errors():
    call = DT.build("contiguous", torch.bfloat16, 32, (3, 3), (5, 9), 64, "cpu", varlen=False)
    q, kc, vc, sl, k, v, _ = call.fresh()
    good = torch.ones(2, 3, 3, dtype=torch.bool).tril()
    with pytest.raises(ValueError, match="needs k / v"):
        f(q, kc, vc, sl, tree_mask=good)
    with pytest.raises(ValueError, match="causal=True"):
        f(q, kc, vc, sl, k, v, append_rank=0, causal=False, tree_mask=good)
    with pytest.raises(ValueError, match="torch.bool"):
        f(q, kc, vc, sl, k, v, append_rank=0, tree_mask=good.to(torch.uint8))
    with pytest.raises(ValueError, match="shape"):
        f(q, kc, vc, sl, k, v, append_rank=0, tree_mask=good[:, :2])
    with pytest.raises(ValueError, match="shape"):
        f(q, kc, vc, sl, k, v, append_rank=0, tree_mask=good.reshape(6, 3))
    with pytest.raises(ValueError, match="contiguous"):
        f(q, kc, vc, sl, k, v, append_rank=0, tree_mask=good.transpose(1, 2))
    with pytest.raises(ValueError, match="device"):
        f(q, kc, vc, sl, k, v, append_rank=0, tree_mask=good.to("meta"))
    vcall = DT.build("contiguous", torch.bfloat16, 32, (3, 1), (5, 9), 64, "cpu")
    q, kc, vc, sl, k, v, kw = vcall.fresh()
    with pytest.raises(ValueError, match="shape"):  # varlen: (total_q, max_seqlen_q)
        f(q, kc, vc, sl, k, v, append_rank=0, tree_mask=torch.ones(4, 4, dtype=torch.bool), **kw)
    big = DT.build("contiguous", torch.bfloat16, 32, (129,), (5,), 256, "cpu", varlen=False)
    q, kc, vc, sl, k, v, _ = big.fresh()
    with pytest.raises(ValueError, match="at most 128"):
        f(q, kc, vc, sl, k, v, append_rank=0, tree_mask=torch.ones(1, 129, 129, dtype=torch.bool))


def _world2(rank, world, interleaved):
    """Rank 0 holds the first lens[b][0] rows of sequence b, rank 1 the next lens[b][1], and rank 1 appends.  Both
    ranks see bitwise the same out / lse, which match one rank on the concatenated cache and the oracle."""
    gen = torch.Generator().manual_seed(9)
    counts = (7, 0, 12)
    lens = [(20, 3), (0, 11), (17, 20)]  # per sequence: rows on rank 0, rank 1
    b, hq, hkv, d, cap = len(counts), 8, 2, 32, 40
    full = DT.build("contiguous", torch.float32, d, counts, [a + c for a, c in lens], 2 * cap, "cpu", seed=2,
                    hq=hq, hkv=hkv)
    mask = _masks(full, gen)
    cos, sin = rope_tables(200, d, torch.float32)
    rs = torch.tensor([a + c for a, c in lens], dtype=torch.int32)
    mine = torch.full((b, cap, hkv, d), float("nan")), torch.full((b, cap, hkv, d), float("nan"))
    for i, (a, c) in enumerate(lens):
        lo, n = (0, a) if rank == 0 else (a, c)
        mine[0][i, :n], mine[1][i, :n] = full.k_cache[i, lo:lo + n], full.v_cache[i, lo:lo + n]
    sl = torch.tensor([x[rank] for x in lens], dtype=torch.int32)
    kw = dict(full.kwargs, rotary_cos=cos, rotary_sin=sin, rotary_seqlens=rs, rotary_interleaved=interleaved)
    out, lse = f(full.q, mine[0], mine[1], sl, full.k, full.v, append_rank=1, return_softmax_lse=True,
                 tree_mask=mask, **kw)
    both = torch.cat([out.reshape(-1), lse.reshape(-1)])
    got = [torch.empty_like(both) for _ in range(world)]
    dist.all_gather(got, both)
    assert all(torch.equal(x, both) for x in got)
    ref_out, ref_lse = _single_rank(full, mask, kw)
    torch.testing.assert_close(out, ref_out, atol=2e-5, rtol=2e-5)
    torch.testing.assert_close(lse, ref_lse, atol=2e-5, rtol=2e-5)
    oo, ol = DT.oracle(full, mask, d ** -0.5, rotary=(cos, sin, rs, interleaved))
    torch.testing.assert_close(out.double(), oo, atol=2e-5, rtol=2e-5)
    torch.testing.assert_close(lse.double(), ol, atol=2e-5, rtol=2e-5)


def _single_rank(call, mask, kw):
    """The dense path of one rank on the concatenated cache (outside the two-rank group)."""
    q, kc, vc, sl, k, v, _ = call.fresh()
    rot = (kw["rotary_cos"], kw["rotary_sin"], kw["rotary_seqlens"], kw["rotary_interleaved"])
    return dec._dense_decode(q, kc, vc, sl, k, v, True, q.shape[-1] ** -0.5, None, 1,
                             cu_seqlens_q=kw["cu_seqlens_q"], max_seqlen_q=kw["max_seqlen_q"], rotary=rot,
                             tree_mask=mask)


@pytest.mark.parametrize("interleaved", [True, False])
def test_two_ranks_append_on_rank_1(interleaved):
    run_distributed(_world2, 2, interleaved)


def test_torch_compile_fullgraph():
    call = DT.build("paged16", torch.bfloat16, 32, (5, 5), (9, 30), 64, "cpu", varlen=False)
    mask = _masks(call, torch.Generator().manual_seed(1))

    def g(q, kc, vc, sl, k, v, bt, m):
        out, lse = f(q, kc, vc, sl, k, v, append_rank=0, return_softmax_lse=True, block_table=bt, tree_mask=m)
        return out * 1.0, lse

    q, kc, vc, sl, k, v, kw = call.fresh()
    out, lse = torch.compile(g, backend="aot_eager", fullgraph=True)(q, kc, vc, sl, k, v, kw["block_table"], mask)
    q, kc2, vc2, sl, k, v, kw = call.fresh()
    ref_out, ref_lse = g(q, kc2, vc2, sl, k, v, kw["block_table"], mask)
    assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse)
    assert torch.equal(DT.raw(kc), DT.raw(kc2))


def test_bench_decode_dry_run_tree():
    cmd = [sys.executable, os.path.join(ROOT, "benchmark", "bench_decode.py"), "--dry-run", "--tree", "4,2,2,1",
           "--batch", "1", "4", "--cache", "32768"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:]
    rows = [json.loads(line) for line in r.stdout.splitlines() if line.startswith("{")]
    assert [(x["batch"], x["tree_nodes"], x["tree_leaves"]) for x in rows] == [(1, 45, 16), (4, 45, 16)]
    assert rows[0]["per_path_calls"] == 16 and rows[0]["max_depth"] == 4
