"""cp_flash_attn_with_kvcache with cache slots (``cache_batch_idx``) and left padding (``cache_leftpad``), on CPU /
gloo: the guards, the dense path against the fp64 oracle (worlds 1-4; contiguous, varlen, e4m3 caches, e4m3 queries,
rotary; causal and not; with and without an append; duplicate slots), bitwise relations to the plain call on the
gathered / shifted cache, a left-padded batch sharded with the ring, zigzag and stripe layouts, the dense range
checks, the arguments reaching the extension, torch.compile and a dry run of the benchmark."""
import dataclasses
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist

import decode_cache_idx as CI
import decode_oracle as DO
import ring_flash_attn_b200 as rfa
from dist_utils import run_distributed
from ring_flash_attn_b200.parallel import decode as dec
from ring_flash_attn_b200.parallel import layouts
from test_gpu_decode_fp8 import bytes_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = 64

# (geometry, overrides): causal / non-causal, varlen, e4m3 caches, e4m3 queries, rotary (causal, non-causal, varlen)
FEATURES = {
    "causal": ("split_edge_by_append", {}),
    "noncausal": ("rows64_g2", {}),
    "varlen": (DO.Case("varlen6", (3, 0, 1, 5, 2, 1), (350, 9, 0, 200, 600, 33), 700, varlen=True), {}),
    "e4m3_cache": ("splits3_of_10_tiles", dict(fp8=True)),
    "e4m3_q": ("rows129_g3", dict(fp8=True)),
    "rotary": ("rotary16_interleaved", {}),
    "rotary_noncausal": ("rotary_half_neox_noncausal", {}),
    "rotary_varlen": ("rotary_full_interleaved_varlen_noncausal", {}),
}
MODES = ("slots", "leftpad", "both")


def _case(feature, append=True):
    name, over = FEATURES[feature]
    case = DO.geometry(name, **over) if isinstance(name, str) else name
    return case if append else dataclasses.replace(case, append=False)


def _build(case, mode, feature, seed=0, cache_seed=None, device="cpu"):
    """Slot inputs of ``mode``: distinct seeded slots of a pool of 2B + 3, seeded pads, both, or (``slots_dup``)
    sequences sharing slots."""
    b = case.b
    idx = pads = None
    if mode in ("slots", "both", "slots_dup"):
        idx = CI.slot_indices(b, 2 * b + 3, seed=100 + (cache_seed or 0), duplicates=mode == "slots_dup")
    if mode in ("leftpad", "both"):
        pads = CI.leftpads(case, seed=200 + (cache_seed or 0))
    return CI.build(case, torch.bfloat16, D, device, idx=idx, n_slots=2 * b + 3, pads=pads,
                    q8=feature == "e4m3_q", seed=seed, cache_seed=cache_seed)


def _scenarios(world):
    """Every feature in every mode with one rank; with more ranks every feature in one mode, rotating with the
    world size, so that each (feature, mode) pair also runs across ranks."""
    out = []
    for i, feature in enumerate(FEATURES):
        for mode in MODES if world == 1 else (MODES[(i + world) % len(MODES)],):
            out.append((feature, mode, True))
            if not feature.startswith("rotary"):  # rotary needs k / v
                out.append((feature, mode, False))
        if not feature.startswith("rotary"):
            out.append((feature, "slots_dup", False))
    return out


def _public(si, with_append, append_rank, group=None):
    q, k, v, kw = CI.call_args(si, with_append)
    case = si.plain.case
    return rfa.cp_flash_attn_with_kvcache(q, si.k_pool, si.v_pool, si.seqlens, k, v,
                                          append_rank=append_rank if with_append else None, causal=case.causal,
                                          return_softmax_lse=True, group=group, **kw)


def _run_dense(rank, world, scenarios):
    torch.set_num_threads(1)  # one process per rank: keep them from oversubscribing the cores
    for feature, mode, append in scenarios:
        case = _case(feature, append)
        append_rank = world - 1
        shards = [_build(case, mode, feature, seed=3, cache_seed=10 + r) for r in range(world)]
        si = shards[rank]
        here = append and rank == append_rank
        out, lse = _public(si, append, append_rank, dist.group.WORLD)
        refs = [DO.references(CI.plain_inputs_for_reference(s), 1, appended_here=append and r == append_rank)
                for r, s in enumerate(shards)]
        o64, l64 = DO.combine_ranks64([(a, b) for a, b, _, _ in refs])
        got_o, got_l = DO.packed(case, out, lse)
        tag = f"{feature} {mode} append={append} world {world} rank {rank}"
        assert torch.isfinite(got_o.float()).all(), tag
        torch.testing.assert_close(got_o.double(), o64, atol=2e-2, rtol=2e-2, msg=tag)
        # the rotation rounds q and k to bf16 before the scores, which the fp64 reference does not
        lse_tol = 1e-2 if feature.startswith("rotary") else 1e-4
        torch.testing.assert_close(got_l.double(), l64, atol=lse_tol, rtol=lse_tol, msg=tag)
        want_k, want_v = CI.expected_pool(si, here)
        assert torch.equal(bytes_of(si.k_pool), bytes_of(want_k)), tag
        assert torch.equal(bytes_of(si.v_pool), bytes_of(want_v)), tag
        both = torch.cat([out.float().reshape(-1), lse.reshape(-1)])
        got = [torch.empty_like(both) for _ in range(world)]
        dist.all_gather(got, both)
        for x in got:
            assert torch.equal(x.nan_to_num(7.0), both.nan_to_num(7.0)), f"{tag}: the ranks' results differ"


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_dense_path_matches_oracle(world):
    run_distributed(_run_dense, world, _scenarios(world))


@pytest.mark.parametrize("feature", list(FEATURES))
@pytest.mark.parametrize("mode", MODES + ("slots_dup",))
def test_dense_equals_plain_call(feature, mode):
    """Bitwise: a slot call is the plain call on ``pool[idx]``, a left-padded one the plain call on the shifted
    cache (out, lse and the appended bytes); slots the call does not name keep their bytes."""
    append = mode != "slots_dup"
    if feature.startswith("rotary") and not append:
        pytest.skip("rotary needs k / v")
    case = _case(feature, append)
    si = _build(case, mode, feature)
    out, lse = _public(si, append, 0)
    plain = dataclasses.replace(si, k_pool=si.plain.k_cache.clone(), v_pool=si.plain.v_cache.clone(), idx=None,
                                pads=None, seqlens=si.plain.seqlens)
    ref_out, ref_lse = _public(plain, append, 0)
    assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse)
    for got, ref in ((si.k_pool, plain.k_pool), (si.v_pool, plain.v_pool)):
        for b in range(case.b):
            slot = b if si.idx is None else si.idx[b]
            lp = 0 if si.pads is None else si.pads[b]
            assert torch.equal(bytes_of(got[slot, lp:]), bytes_of(ref[b, :case.s_cap - lp])), b
    if si.idx is not None:
        untouched = sorted(set(range(si.k_pool.shape[0])) - set(si.idx))
        fresh = _build(case, mode, feature)
        assert torch.equal(bytes_of(si.k_pool[untouched]), bytes_of(fresh.k_pool[untouched]))
        assert torch.equal(bytes_of(si.v_pool[untouched]), bytes_of(fresh.v_pool[untouched]))


def _run_left_padded(rank, world, scheme, device_type="cpu"):
    """A left-padded batch, prefilled in ``scheme``'s layout: every rank derives its own ``cache_leftpad`` from the
    global positions of its rows, and the decode step must match the fp64 oracle on the unpadded sequences."""
    dev = f"cuda:{rank}" if device_type == "cuda" else "cpu"
    b, s_local, hq, hkv, sq = 3, 64, 4, 2, 2
    total = world * s_local
    left_pad = torch.tensor([0, 7, 2 * (s_local // 2) + 5])  # the last pad covers more than one zigzag chunk
    g = torch.Generator().manual_seed(0)
    kg, vg = (torch.randn(b, total, hkv, D, generator=g) for _ in range(2))
    q = torch.randn(b, sq, hq, D, generator=g).bfloat16()
    kn, vn = (torch.randn(b, sq, hkv, D, generator=g).bfloat16() for _ in range(2))
    kg, vg = kg.bfloat16(), vg.bfloat16()
    kp, vp = kg.clone(), vg.clone()
    for i, lp in enumerate(left_pad.tolist()):  # pad tokens hold anything
        kp[i, :lp] = float("nan")
        vp[i, :lp] = float("nan")
    shard = getattr(layouts, f"shard_{scheme}")
    s_cap = s_local + sq
    kc = torch.full((b, s_cap, hkv, D), float("nan"), dtype=torch.bfloat16)
    vc = kc.clone()
    kc[:, :s_local], vc[:, :s_local] = shard(kp, rank, world, dim=1), shard(vp, rank, world, dim=1)
    pos = layouts.positions(scheme, rank, world, s_local)
    cache_leftpad = (pos < left_pad[:, None]).sum(-1).to(torch.int32)
    sl = torch.full((b,), s_local, dtype=torch.int32)
    out, lse = rfa.cp_flash_attn_with_kvcache(*(x.to(dev) for x in (q, kc, vc, sl, kn, vn)), append_rank=world - 1,
                                              causal=True, return_softmax_lse=True, group=dist.group.WORLD,
                                              cache_leftpad=cache_leftpad.to(dev))
    out, lse = out.cpu(), lse.cpu()
    scale = D ** -0.5
    for i, lp in enumerate(left_pad.tolist()):
        keys = torch.cat([kg[i, lp:], kn[i]]).double()
        vals = torch.cat([vg[i, lp:], vn[i]]).double()
        n = total - lp
        for t in range(sq):
            qq = q[i, t].double().view(hkv, hq // hkv, D)
            s = torch.einsum("kgd,jkd->kgj", qq, keys[:n + t + 1]) * scale
            o = torch.einsum("kgj,jkd->kgd", s.softmax(-1), vals[:n + t + 1]).reshape(hq, D)
            torch.testing.assert_close(out[i, t].double(), o, atol=2e-2, rtol=2e-2, msg=f"{scheme} {i} {t}")
            torch.testing.assert_close(lse[i, :, t].double(), torch.logsumexp(s, -1).reshape(hq), atol=1e-4,
                                       rtol=1e-4)
    both = torch.cat([out.float().reshape(-1), lse.reshape(-1)]).to(dev)
    got = [torch.empty_like(both) for _ in range(world)]
    dist.all_gather(got, both)
    for x in got:
        assert torch.equal(x, both), "the ranks' results differ"


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("scheme", ["ring", "zigzag", "stripe"])
def test_left_padded_batch_sharded(scheme, world):
    run_distributed(_run_left_padded, world, scheme)


def test_guards():
    case = _case("causal")
    si = _build(case, "both", "causal")
    q, k, v, kw = CI.call_args(si, True)
    idx, lp = kw.pop("cache_batch_idx"), kw.pop("cache_leftpad")
    kc, vc, sl = si.k_pool, si.v_pool, si.seqlens
    f = rfa.cp_flash_attn_with_kvcache
    inp = DO.build_inputs(dataclasses.replace(case, layout="paged", page_size=16), torch.bfloat16, D, "randn", "cpu")
    with pytest.raises(ValueError, match="does not support cache_batch_idx"):
        f(q, inp.k_cache, inp.v_cache, sl, block_table=inp.table, cache_batch_idx=idx)
    with pytest.raises(ValueError, match="does not support cache_leftpad"):
        f(q, inp.k_cache, inp.v_cache, sl, block_table=inp.table, cache_leftpad=lp)
    for name, good in (("cache_batch_idx", idx), ("cache_leftpad", lp)):
        other = dict(cache_batch_idx=idx) if name == "cache_leftpad" else {}
        for bad in (good.long(), good.float(), torch.cat([good, good[:1]]), good[:, None], torch.stack([good] * 2,
                                                                                                       1)[:, 0], 3):
            with pytest.raises(ValueError, match=f"{name} must be a contiguous"):
                f(q, kc, vc, sl, **other, **{name: bad})
        with pytest.raises(ValueError, match=f"{name} must be on q's device"):
            f(q, kc, vc, sl, **other, **{name: good.to("meta")})
    # without cache_batch_idx the cache must still hold B sequences
    with pytest.raises(ValueError, match="does not match the cache"):
        f(q, kc, vc, sl, cache_leftpad=lp)
    huge = torch.empty((2 ** 16, 2 ** 15, case.hkv, D), dtype=torch.bfloat16, device="meta")
    with pytest.raises(ValueError, match="B_cache \\* S_cap"):
        f(q, huge, huge, sl, cache_batch_idx=idx)


def test_dense_range_checks():
    case = _case("causal")
    si = _build(case, "both", "causal")
    q, k, v, kw = CI.call_args(si, True)
    n_slots = si.k_pool.shape[0]
    f = rfa.cp_flash_attn_with_kvcache
    for bad in (-1, n_slots):
        idx = kw["cache_batch_idx"].clone()
        idx[1] = bad
        with pytest.raises(ValueError, match=f"cache_batch_idx\\[1\\] = {bad} is outside the {n_slots}-slot cache"):
            f(q, si.k_pool, si.v_pool, si.seqlens, k, v, append_rank=0, **dict(kw, cache_batch_idx=idx))
    for bad in (-1, int(si.seqlens[2]) + 1):
        lp = kw["cache_leftpad"].clone()
        lp[2] = bad
        with pytest.raises(ValueError, match=f"cache_leftpad\\[2\\] = {bad} is outside"):
            f(q, si.k_pool, si.v_pool, si.seqlens, k, v, append_rank=0, **dict(kw, cache_leftpad=lp))
    # nothing was appended by the refused calls
    fresh = _build(case, "both", "causal")
    assert torch.equal(bytes_of(si.k_pool), bytes_of(fresh.k_pool))


class _Recorder:
    """Stands in for the extension and records what kernel_decode passes to decode_fwd."""

    def __init__(self):
        self.args = None

    def decode_fwd(self, *args):
        self.args = args

    def decode_combine(self, parts, out, lse):
        out.zero_()
        lse.zero_()


def test_kernel_decode_passes_the_arguments(monkeypatch):
    from ring_flash_attn_b200.ops import cuda_ext

    rec = _Recorder()
    monkeypatch.setattr(cuda_ext, "load", lambda: rec)
    si = _build(_case("causal"), "both", "causal")
    q, k, v, kw = CI.call_args(si, True)
    dec.kernel_decode(q, si.k_pool, si.v_pool, si.seqlens, k, v, True, 0.1, splits=2, **kw)
    assert len(rec.args) == 21 and rec.args[-3] is None
    assert rec.args[-2] is kw["cache_batch_idx"] and rec.args[-1] is kw["cache_leftpad"]
    dec.kernel_decode(q, si.k_pool, si.v_pool, si.seqlens, k, v, True, 0.1, splits=2,
                      cache_leftpad=kw["cache_leftpad"])
    assert len(rec.args) == 21 and rec.args[-2] is None and rec.args[-1] is kw["cache_leftpad"]
    plain = dict(kw)
    del plain["cache_batch_idx"], plain["cache_leftpad"]
    dec.kernel_decode(q, si.plain.k_cache, si.plain.v_cache, si.plain.seqlens, k, v, True, 0.1, splits=2, **plain)
    assert len(rec.args) == 18  # calls without them keep the form they had


def test_torch_compile_fullgraph():
    case = _case("causal")
    si = _build(case, "both", "causal")
    si2 = _build(case, "both", "causal")
    q, k, v, kw = CI.call_args(si, True)

    def f(q, kc, vc, sl, k, v, idx, lp):
        out, lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, sl, k, v, append_rank=0, return_softmax_lse=True,
                                                  cache_batch_idx=idx, cache_leftpad=lp)
        return out * 1.0, lse

    args = (si.seqlens, k, v, kw["cache_batch_idx"], kw["cache_leftpad"])
    out, lse = torch.compile(f, backend="aot_eager", fullgraph=True)(q, si.k_pool, si.v_pool, *args)
    ref_out, ref_lse = f(q, si2.k_pool, si2.v_pool, *args)
    assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse)
    assert torch.equal(bytes_of(si.k_pool), bytes_of(si2.k_pool))  # the compiled call appended too


def test_bench_decode_dry_run_slots_and_leftpad():
    cmd = [sys.executable, os.path.join(ROOT, "benchmark", "bench_decode.py"), "--dry-run", "--cache-slots", "16",
           "--leftpad", "1000"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:]
    rows = [json.loads(line) for line in r.stdout.splitlines() if line.startswith("{")]
    assert len(rows) == 6
    for x in rows:
        assert x["cache_slots"] == 16 and x["leftpad"] == 1000
        assert x["pool_bytes"] == x["kv_bytes"] // x["batch"] * 16
        assert x["gather_scatter_bytes"] == 4 * x["kv_bytes"]
    r = subprocess.run(cmd + ["--kv-dtype", "e4m3", "--q-dtype", "e4m3", "--batch", "8", "--cache", "32768"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:]
    (x,) = [json.loads(line) for line in r.stdout.splitlines() if line.startswith("{")]
    assert x["pool_bytes"] == x["fp8_kv_bytes"] // 8 * 16
    bad = subprocess.run(cmd[:3] + ["4", "--batch", "8"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True, timeout=300, cwd=ROOT)
    assert bad.returncode != 0 and "--cache-slots" in bad.stdout
