"""The sm_90a split-KV decode kernel with tree masks (``tree_mask=``): a lower-triangular mask bitwise the causal call
(out, lse, appended bytes) and random trees against the fp64 oracle, for bf16 / fp16 x D 64 / 128 over contiguous,
paged (16-row pages), e4m3 caches, e4m3 queries, slots with left pads and shared prefixes, uniform and varlen, with
split and 128-key tile boundaries inside the new keys and trees spanning several 64-row tiles (Sq up to 61, G = 4);
rotary at the tree depths bitwise the call on rotated inputs; CUDA-graph replay with new trees, lengths and positions;
and two GPUs with the append on rank 1."""
import pytest
import torch
import torch.distributed as dist

import decode_tree as DT
import ring_flash_attn_b200 as rfa
from dist_utils import run_distributed
from ring_flash_attn_b200.parallel import decode as dec
from test_decode_rotary import rope_tables
from test_gpu_decode_varlen import LSE_TOL, OUT_TOL

pytestmark = pytest.mark.gpu

KINDS = [(torch.bfloat16, 64), (torch.bfloat16, 128), (torch.float16, 64), (torch.float16, 128)]
IDS = [f"{str(t)[6:]}-D{d}" for t, d in KINDS]
S_CAP = 640  # 5 key tiles: splits=5 puts a split boundary at every tile boundary
# counts, cached rows.  Cached 120: the new keys cross the 128-key tile (and, at splits=5, split) boundary; cached 250
# with 7 new keys crosses 256, a split boundary at splits=3.  61 x G=4 = 244 packed rows: four 64-row tiles.
UNIFORM = ((24,) * 4, (120, 0, 300, 500))
VARLEN = ((61, 0, 7, 33), (120, 5, 250, 0))
SPLITS = (1, 3, 5)


def _build(layout, dtype, d, varlen, seed):
    counts, lens = VARLEN if varlen else UNIFORM
    return DT.build(layout, dtype, d, counts, lens, S_CAP, "cuda", seed=seed, varlen=varlen)


def _masks(call, gen, tril=False):
    per = DT.tril_masks(call.counts) if tril else DT.tree_masks(call.counts, gen)
    return DT.packed_mask(per, max(call.counts), gen, call.varlen).cuda()


def _run(call, mask, splits, q=None, k=None, rotary=None):
    q0, kc, vc, sl, k0, v, kw = call.fresh()
    if rotary is not None:
        kw.update(rotary_cos=rotary[0], rotary_sin=rotary[1], rotary_seqlens=rotary[2], rotary_interleaved=rotary[3])
    out, lse = dec.kernel_decode(q0 if q is None else q, kc, vc, sl, k0 if k is None else k, v, True,
                                 call.q_rows.shape[-1] ** -0.5, splits=splits, tree_mask=mask, **kw)
    torch.cuda.synchronize()
    return out, lse, kc, vc


@pytest.mark.parametrize("layout", DT.LAYOUTS)
@pytest.mark.parametrize("dtype,d", KINDS, ids=IDS)
def test_lower_triangular_mask_is_the_causal_call(dtype, d, layout):
    gen = torch.Generator().manual_seed(d)
    for varlen in (False, True):
        call = _build(layout, dtype, d, varlen, seed=d + varlen)
        tril = _masks(call, gen, tril=True)
        for splits in SPLITS:
            out, lse, kc, vc = _run(call, tril, splits)
            ref_out, ref_lse, ref_kc, ref_vc = _run(call, None, splits)
            tag = (layout, varlen, splits)
            assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse), tag
            assert torch.equal(DT.raw(kc), DT.raw(ref_kc)) and torch.equal(DT.raw(vc), DT.raw(ref_vc)), tag


@pytest.mark.parametrize("layout", DT.LAYOUTS)
@pytest.mark.parametrize("dtype,d", KINDS, ids=IDS)
def test_random_trees_match_the_oracle(dtype, d, layout):
    gen = torch.Generator().manual_seed(7 * d)
    for varlen in (False, True):
        call = _build(layout, dtype, d, varlen, seed=3 + d + varlen)
        for splits in SPLITS:
            mask = _masks(call, gen)
            out, lse, kc, vc = _run(call, mask, splits)
            ref_out, ref_lse = DT.oracle(call, mask, d ** -0.5)
            got_o, got_l = DT.packed(call, out, lse)
            tag = f"{layout} varlen={varlen} splits={splits}"
            torch.testing.assert_close(got_o.double(), ref_out, **OUT_TOL, msg=lambda m: f"{tag}: {m}")
            torch.testing.assert_close(got_l.double(), ref_lse, **LSE_TOL, msg=lambda m: f"{tag}: {m}")
            # the append does not depend on the mask
            _, _, ref_kc, ref_vc = _run(call, None, splits)
            assert torch.equal(DT.raw(kc), DT.raw(ref_kc)) and torch.equal(DT.raw(vc), DT.raw(ref_vc)), tag


@pytest.mark.parametrize("layout", ["contiguous", "paged16", "e4m3", "prefix"])
@pytest.mark.parametrize("dtype,d", KINDS, ids=IDS)
def test_rotary_is_the_masked_call_on_rotated_inputs(dtype, d, layout):
    gen = torch.Generator().manual_seed(11 + d)
    for varlen in (False, True):
        call = _build(layout, dtype, d, varlen, seed=5 + d + varlen)
        b = len(call.counts)
        rs = torch.tensor([1000, 3, 77, 2500][:b], dtype=torch.int32, device="cuda")
        for interleaved in (True, False):
            for rotary_dim in (d, 16):
                cos, sin = rope_tables(3000, rotary_dim, dtype, "cuda")
                mask = _masks(call, gen)
                pos = []
                for (lo, n), start in zip(call.spans, rs.tolist()):
                    pos += [start + x for x in dec.tree_depths(mask.reshape(-1, mask.shape[-1]).cpu(), [(lo, n)])]
                pos = torch.tensor(pos, dtype=torch.long, device="cuda")
                qr = dec.apply_rotary(call.q_rows.cuda(), cos, sin, pos, interleaved)
                kr = dec.apply_rotary(call.k_rows.cuda(), cos, sin, pos, interleaved)
                q2, k2 = (x if varlen else x.view(b, -1, *x.shape[1:]) for x in (qr, kr))
                out, lse, kc, vc = _run(call, mask, 3, rotary=(cos, sin, rs, interleaved))
                p_out, p_lse, p_kc, p_vc = _run(call, mask, 3, q=q2, k=k2)
                tag = (layout, varlen, interleaved, rotary_dim)
                assert torch.equal(out, p_out) and torch.equal(lse, p_lse), tag
                assert torch.equal(DT.raw(kc), DT.raw(p_kc)) and torch.equal(DT.raw(vc), DT.raw(p_vc)), tag


@pytest.mark.parametrize("varlen", [False, True])
def test_cuda_graph_replay_with_new_trees(varlen):
    gen = torch.Generator().manual_seed(21)
    call = _build("contiguous", torch.bfloat16, 128, varlen, seed=2)
    cos, sin = rope_tables(4096, 128, torch.bfloat16, "cuda")
    b = len(call.counts)
    sl = call.seqlens.clone()
    rs = torch.tensor([500, 0, 1000, 7], dtype=torch.int32, device="cuda")
    mask = _masks(call, gen)
    kc, vc = call.k_cache.nan_to_num(0.25), call.v_cache.nan_to_num(-0.5)  # the lengths below grow into NaN rows
    kw = dict(call.kwargs, append_rank=0, return_softmax_lse=True, rotary_cos=cos, rotary_sin=sin,
              rotary_seqlens=rs, rotary_interleaved=False)
    f = rfa.cp_flash_attn_with_kvcache

    def step(k_cache, v_cache, m):
        return f(call.q, k_cache, v_cache, sl, call.k, call.v, tree_mask=m, **kw)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(kc.clone(), vc.clone(), mask)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out, lse = step(kc, vc, mask)
    for lens_now, pos_now in (([120, 0, 300, 0], [500, 0, 1000, 7]), ([7, 250, 0, 128], [9, 3000, 1, 64]),
                              ([500, 1, 2, 3], [0, 0, 0, 0])):
        new = _masks(call, gen)
        mask.copy_(new)
        sl.copy_(torch.tensor(lens_now[:b], dtype=torch.int32))
        rs.copy_(torch.tensor(pos_now[:b], dtype=torch.int32))
        ek, ev = kc.clone(), vc.clone()
        graph.replay()
        want_out, want_lse = step(ek, ev, new)
        torch.cuda.synchronize()
        assert torch.equal(out, want_out) and torch.equal(lse, want_lse), lens_now
        assert torch.equal(DT.raw(kc), DT.raw(ek)) and torch.equal(DT.raw(vc), DT.raw(ev)), lens_now


def _two_gpus(rank, world):
    gen = torch.Generator().manual_seed(9)
    counts = (37, 0, 12)
    lens = [(200, 3), (0, 111), (129, 120)]  # per sequence: rows on rank 0, rank 1
    b, hkv, d, cap = len(counts), 2, 128, 384
    dev = f"cuda:{rank}"
    full = DT.build("contiguous", torch.bfloat16, d, counts, [a + c for a, c in lens], 2 * cap, "cpu", seed=2,
                    hkv=hkv)
    mask = _masks(full, gen).to(dev)
    mine = [torch.full((b, cap, hkv, d), float("nan"), dtype=torch.bfloat16) for _ in range(2)]
    for i, (a, c) in enumerate(lens):
        lo, n = (0, a) if rank == 0 else (a, c)
        mine[0][i, :n], mine[1][i, :n] = full.k_cache[i, lo:lo + n], full.v_cache[i, lo:lo + n]
    sl = torch.tensor([x[rank] for x in lens], dtype=torch.int32, device=dev)
    kw = {k: (x.to(dev) if isinstance(x, torch.Tensor) else x) for k, x in full.kwargs.items()}
    out, lse = rfa.cp_flash_attn_with_kvcache(full.q.to(dev), mine[0].to(dev), mine[1].to(dev), sl, full.k.to(dev),
                                              full.v.to(dev), append_rank=1, return_softmax_lse=True, tree_mask=mask,
                                              **kw)
    both = torch.cat([out.float().reshape(-1), lse.reshape(-1)])
    got = [torch.empty_like(both) for _ in range(world)]
    dist.all_gather(got, both)
    assert all(torch.equal(x, both) for x in got)
    ref_out, ref_lse = DT.oracle(full, mask.cpu(), d ** -0.5)
    torch.testing.assert_close(out.cpu().double(), ref_out, **OUT_TOL)
    torch.testing.assert_close(lse.cpu().double(), ref_lse, **LSE_TOL)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_append_on_rank_1():
    run_distributed(_two_gpus, 2, backend="nccl")
