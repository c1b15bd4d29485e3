"""cp_flash_attn_with_kvcache with shared prefixes (``prefix_k_cache`` / ``prefix_v_cache`` / ``prefix_seqlens``), on
CPU / gloo: the dense path against the fp64 oracle (worlds 1-4; uniform and varlen, causal and not, with and without
an append, rotary, e4m3 caches, cache slots and left pads on the suffix, P in {1, 2}, n in {1, 3}, prefixes of 0 and
P_cap rows, empty suffixes), bitwise equality with the plain call on the concatenated cache, the guards, the dense
range check, the arguments reaching the extension, torch.compile and a dry run of the benchmark."""
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
import decode_prefix as DP
import ring_flash_attn_b200 as rfa
from dist_utils import run_distributed
from ring_flash_attn_b200.parallel import decode as dec
from test_decode_rotary import rope_tables
from test_gpu_decode_fp8 import bytes_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = 64

# (case, prefix lens as a function of P_cap, P_cap): B = P * n
FEATURES = {
    # P = 2, n = 3; one empty suffix, one prefix of P_cap rows
    "causal": DO.Case("u6", (2,) * 6, (300, 0, 17, 128, 5, 250), 320, hq=8, hkv=2),
    "noncausal": DO.Case("u6nc", (3,) * 6, (100, 31, 0, 129, 300, 2), 320, hq=8, hkv=2, causal=False),
    # P = 2, n = 3, varlen with zero counts
    "varlen": DO.Case("v6", (3, 0, 1, 5, 2, 1), (250, 9, 0, 200, 0, 33), 300, varlen=True),
    "e4m3_cache": DO.Case("u6f8", (2,) * 6, (200, 0, 60, 129, 7, 280), 300, hq=8, hkv=2, fp8=True),
    "rotary": DO.Case("u6rot", (2,) * 6, (200, 0, 60, 129, 7, 280), 300, rotary=(16, True)),
    "rotary_varlen": DO.Case("v6rot", (3, 0, 1, 5, 2, 1), (250, 9, 0, 200, 0, 33), 300, varlen=True,
                             rotary=("full", True), causal=False),
    # P = 1 (n = 6) and P = 6 (n = 1)
    "one_prefix": DO.Case("u6p1", (1,) * 6, (30, 0, 17, 200, 5, 250), 300, hq=16, hkv=2),
    "n1": DO.Case("u6n1", (2,) * 6, (30, 0, 17, 200, 5, 250), 300, hq=4, hkv=1),
}
N_PREFIX = {"one_prefix": 1, "n1": 6}
P_CAP = 400


def _plens(feature, rank=0):
    """Prefix lengths of a rank's shard: P_cap and 0 on rank 0 (and with six prefixes)."""
    pool = [P_CAP, 0, 271, 129, 1, 390, 257, 333]
    return [pool[(3 * rank + i) % len(pool)] for i in range(N_PREFIX.get(feature, 2))]


def _inputs(feature, append=True, mode=None, seed=3, cache_seed=10, prefix_seed=7, rank=0, device="cpu"):
    """(SlotInputs of the suffix, Prefix): ``mode`` None, "slots", "leftpad" or "both" on the suffix."""
    case = FEATURES[feature]
    if not append:
        case = dataclasses.replace(case, append=False)
    b = case.b
    idx = CI.slot_indices(b, 2 * b + 3, seed=100 + cache_seed) if mode in ("slots", "both") else None
    pads = CI.leftpads(case, seed=200 + cache_seed) if mode in ("leftpad", "both") else None
    si = CI.build(case, torch.bfloat16, D, device, idx=idx, n_slots=2 * b + 3, pads=pads, seed=seed,
                  cache_seed=cache_seed)
    pre = DP.make_prefix(case, torch.bfloat16, D, device, _plens(feature, rank), P_CAP, seed=prefix_seed)
    return si, pre


def _public(si, pre, with_append, append_rank, group=None, **over):
    q, k, v, kw = CI.call_args(si, with_append)
    kw.update(pre.kwargs())
    kw.update(over)
    case = si.plain.case
    return rfa.cp_flash_attn_with_kvcache(q, si.k_pool, si.v_pool, si.seqlens, k, v,
                                          append_rank=append_rank if with_append else None, causal=case.causal,
                                          return_softmax_lse=True, group=group, **kw)


def _scenarios(world):
    out = []
    modes = (None, "slots", "leftpad", "both")
    for i, feature in enumerate(FEATURES):
        mode = modes[(i + world) % len(modes)]
        out.append((feature, mode, True))
        if not feature.startswith("rotary"):  # rotary needs k / v
            out.append((feature, None if world > 1 else "both", False))
    return out


def _run_dense(rank, world, scenarios, device_type="cpu"):
    """Each rank holds its own suffix shard and prefix shard (``device_type="cuda"``: on its GPU, through the
    kernel); the result must match the fp64 oracle of all shards and be bitwise equal on every rank."""
    torch.set_num_threads(1)
    dev = f"cuda:{rank}" if device_type == "cuda" else "cpu"
    if device_type == "cuda":
        torch.cuda.set_device(rank)
    for feature, mode, append in scenarios:
        append_rank = world - 1
        shards = [_inputs(feature, append, mode, cache_seed=10 + r, prefix_seed=20 + r, rank=r, device=dev)
                  for r in range(world)]
        si, pre = shards[rank]
        out, lse = _public(si, pre, append, append_rank, dist.group.WORLD)
        refs = []
        for r, (s, p) in enumerate(shards):
            inp = CI.plain_inputs_for_reference(s)
            refs.append(DO.references(inp, 1, appended_here=append and r == append_rank))
            refs.append(DO.references(DP.prefix_view(inp, p), 1, appended_here=False))
        o64, l64, _, _ = DP.parts_merged(refs)
        case = si.plain.case
        got_o, got_l = DO.packed(case, out, lse)
        tag = f"{feature} {mode} append={append} world {world} rank {rank}"
        assert torch.isfinite(got_o.float()).all(), tag
        torch.testing.assert_close(got_o.double(), o64, atol=2e-2, rtol=2e-2, msg=tag)
        lse_tol = 1e-2 if feature.startswith("rotary") else 1e-4
        torch.testing.assert_close(got_l.double(), l64, atol=lse_tol, rtol=lse_tol, msg=tag)
        want_k, want_v = CI.expected_pool(si, append and rank == append_rank)
        assert torch.equal(bytes_of(si.k_pool), bytes_of(want_k)), tag
        assert torch.equal(bytes_of(si.v_pool), bytes_of(want_v)), tag
        fresh = DP.make_prefix(case, torch.bfloat16, D, dev, _plens(feature, rank), P_CAP, seed=20 + rank)
        assert torch.equal(bytes_of(pre.k), bytes_of(fresh.k)) and torch.equal(bytes_of(pre.v), bytes_of(fresh.v))
        both = torch.cat([out.float().reshape(-1), lse.reshape(-1)])
        got = [torch.empty_like(both) for _ in range(world)]
        dist.all_gather(got, both)
        for x in got:
            assert torch.equal(x.nan_to_num(7.0), both.nan_to_num(7.0)), f"{tag}: the ranks' results differ"


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_dense_path_matches_oracle(world):
    run_distributed(_run_dense, world, _scenarios(world))


@pytest.mark.parametrize("feature", [f for f in FEATURES if f != "e4m3_cache"])
def test_dense_equals_plain_call_on_concatenated_cache(feature):
    """Bitwise: the prefix call is the plain call on a cache holding the prefix rows, then the sequence's rows (the
    dense path computes both with one softmax over the same keys), and the appended bytes match."""
    si, pre = _inputs(feature)
    inp = si.plain
    out, lse = _public(si, pre, True, 0)
    kc, vc, lens = DP.concatenated(inp, pre)
    q, k, v, kw = CI.call_args(si, True)
    ref_out, ref_lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, lens, k, v, append_rank=0, causal=inp.case.causal,
                                                      return_softmax_lse=True, **kw)
    assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse), feature
    n = inp.case.b // pre.n
    for b in range(inp.case.b):
        pl = pre.lens[b // n]
        assert torch.equal(bytes_of(si.k_pool[b]), bytes_of(kc[b, pl:pl + inp.case.s_cap])), b
        assert torch.equal(bytes_of(si.v_pool[b]), bytes_of(vc[b, pl:pl + inp.case.s_cap])), b


def test_rotary_default_positions_in_one_rank_group():
    """Without rotary_seqlens, a one-rank group rotates at prefix_seqlens[p] + cache_seqlens[b], as the plain call on
    the concatenated cache does at its cache_seqlens."""
    si, pre = _inputs("rotary")
    q, k, v, kw = CI.call_args(si, True)
    kw.pop("rotary_seqlens")
    kw["rotary_cos"], kw["rotary_sin"] = rope_tables(P_CAP + si.plain.case.s_cap + 8, 16, torch.bfloat16, "cpu")
    out = rfa.cp_flash_attn_with_kvcache(q, si.k_pool, si.v_pool, si.seqlens, k, v, append_rank=0, **kw,
                                         **pre.kwargs())
    kc, vc, lens = DP.concatenated(si.plain, pre)
    ref = rfa.cp_flash_attn_with_kvcache(q, kc, vc, lens, k, v, append_rank=0, **kw)
    assert torch.equal(out, ref)


def test_guards():
    si, pre = _inputs("causal")
    q, k, v, kw = CI.call_args(si, True)
    kc, vc, sl = si.k_pool, si.v_pool, si.seqlens
    f = rfa.cp_flash_attn_with_kvcache
    good = pre.kwargs()
    for drop in ("prefix_k_cache", "prefix_v_cache", "prefix_seqlens"):
        bad = dict(good)
        del bad[drop]
        with pytest.raises(ValueError, match="together"):
            f(q, kc, vc, sl, **bad)
    with pytest.raises(ValueError, match="only taken with prefix_k_cache"):
        f(q, kc, vc, sl, prefix_k_descale=torch.ones(()))
    pk = pre.k
    for name, bad, msg in (
            ("prefix_k_cache", pk.transpose(1, 2).contiguous().transpose(1, 2), "contiguous"),
            ("prefix_k_cache", pk[:, :, :, :32].contiguous(), "must both be"),
            ("prefix_v_cache", pre.v[:1], "must both be"),
            ("prefix_k_cache", pk.half(), "cache's dtype"),
            ("prefix_k_cache", pk.to("meta"), "on q's device"),
            ("prefix_k_cache", pk[0], "contiguous"),
            ("prefix_seqlens", pre.seqlens.long(), "prefix_seqlens must be a contiguous"),
            ("prefix_seqlens", pre.seqlens[:1], "prefix_seqlens must be a contiguous"),
            ("prefix_seqlens", torch.stack([pre.seqlens] * 2, 1)[:, 0], "prefix_seqlens must be a contiguous"),
            ("prefix_seqlens", pre.seqlens.to("meta"), "prefix_seqlens must be on q's device"),
    ):
        with pytest.raises(ValueError, match=msg):
            f(q, kc, vc, sl, **dict(good, **{name: bad}))
    # B % P != 0
    three = DP.make_prefix(si.plain.case, torch.bfloat16, D, "cpu", [1, 2, 3, 4], P_CAP)
    with pytest.raises(ValueError, match="multiple of the prefix count"):
        f(q, kc, vc, sl, **three.kwargs())
    huge = torch.empty((2 ** 16, 2 ** 15, 2, D), dtype=torch.bfloat16, device="meta")
    with pytest.raises(ValueError, match="P \\* P_cap < 2\\^31"):
        f(q, kc, vc, sl, prefix_k_cache=huge, prefix_v_cache=huge, prefix_seqlens=pre.seqlens)
    with pytest.raises(ValueError, match="only taken with fp8"):
        f(q, kc, vc, sl, **good, prefix_k_descale=torch.ones(()), prefix_v_descale=torch.ones(()))
    # e4m3 caches: the prefix descales are required and shaped like k_descale
    si8, pre8 = _inputs("e4m3_cache")
    q8, _, _, kw8 = CI.call_args(si8, False)
    base = dict(k_descale=kw8["k_descale"], v_descale=kw8["v_descale"])
    bad = pre8.kwargs()
    del bad["prefix_v_descale"]
    with pytest.raises(ValueError, match="need prefix_v_descale"):
        f(q8, si8.k_pool, si8.v_pool, si8.seqlens, **base, **bad)
    for x, msg in ((torch.ones(3), "shape"), (torch.ones(2, dtype=torch.float64), "float32"),
                   (torch.ones(6, 2), "shape")):
        with pytest.raises(ValueError, match=msg):
            f(q8, si8.k_pool, si8.v_pool, si8.seqlens, **base, **dict(pre8.kwargs(), prefix_k_descale=x))
    # an e4m3 q with a prefix is left out
    qq = q8.to(torch.float8_e4m3fn)
    with pytest.raises(ValueError, match="bf16 / fp16 q"):
        f(qq, si8.k_pool, si8.v_pool, si8.seqlens, **base, q_descale=torch.ones(()), **pre8.kwargs())


def test_dense_range_check():
    si, pre = _inputs("causal")
    q, k, v, kw = CI.call_args(si, True)
    for bad in (-1, P_CAP + 1):
        pl = pre.seqlens.clone()
        pl[1] = bad
        with pytest.raises(ValueError, match=f"prefix_seqlens\\[1\\] = {bad} is outside"):
            rfa.cp_flash_attn_with_kvcache(q, si.k_pool, si.v_pool, si.seqlens, k, v, append_rank=0, **kw,
                                           **dict(pre.kwargs(), prefix_seqlens=pl))
    fresh, _ = _inputs("causal")
    assert torch.equal(bytes_of(si.k_pool), bytes_of(fresh.k_pool))  # nothing appended by the refused calls


class _Recorder:
    """Stands in for the extension and records what kernel_decode passes to it."""

    def __init__(self):
        self.fwd = self.prefix = self.parts = None

    def decode_fwd(self, *args):
        self.fwd = args

    def decode_prefix_fwd(self, *args):
        self.prefix = args

    def decode_combine(self, parts, out, lse):
        self.parts = parts
        out.zero_()
        lse.zero_()


def test_kernel_decode_passes_the_arguments(monkeypatch):
    from ring_flash_attn_b200.ops import cuda_ext

    rec = _Recorder()
    monkeypatch.setattr(cuda_ext, "load", lambda: rec)
    si, pre = _inputs("rotary")
    q, k, v, kw = CI.call_args(si, True)
    counter = cuda_ext.launch_counter()
    counter.reset()
    dec.kernel_decode(q, si.k_pool, si.v_pool, si.seqlens, k, v, True, 0.1, splits=2, prefix_splits=3,
                      **kw, **pre.kwargs())
    assert counter.value == 4  # append, suffix pass, prefix pass, combine
    assert len(rec.fwd) == 18 and rec.fwd[8].shape[0] == 2  # the plain form, on the first two slabs
    assert rec.parts.shape[0] == 5
    args = rec.prefix
    assert args[0] is q and args[1] is pre.k and args[2] is pre.v and args[3] is pre.seqlens
    assert args[6].shape[0] == 3 and args[6].data_ptr() == rec.parts[2:].data_ptr()
    assert args[11] is kw["rotary_cos"] and args[13] is kw["rotary_seqlens"]
    # calls without a prefix keep the form they had
    rec.prefix = None
    dec.kernel_decode(q, si.k_pool, si.v_pool, si.seqlens, k, v, True, 0.1, splits=2, **kw)
    assert rec.prefix is None and rec.parts.shape[0] == 2


def test_prefix_splits_fill_one_wave():
    # P x Hkv x slots x splits <= the SM count, never more than the prefix's key tiles
    slots = dec.prefix_tile_slots(16, 1, 32, 8, None)
    assert slots == 1
    assert dec.num_splits_prefix(2, slots, 8, 128 * 1024, 132) == 8
    assert dec.num_splits_prefix(1, 1, 1, 300, 132) == 3
    assert dec.prefix_tile_slots(5, 4, 8, 2) == 2  # 80 rows
    assert dec.prefix_tile_slots(5, 4, 8, 2, total_q=9) == 1  # varlen: at most total_q rows


def test_torch_compile_fullgraph():
    si, pre = _inputs("causal")
    si2, _ = _inputs("causal")
    q, k, v, kw = CI.call_args(si, True)

    def f(q, kc, vc, sl, k, v, pk, pv, pl):
        out, lse = rfa.cp_flash_attn_with_kvcache(q, kc, vc, sl, k, v, append_rank=0, return_softmax_lse=True,
                                                  prefix_k_cache=pk, prefix_v_cache=pv, prefix_seqlens=pl)
        return out * 1.0, lse

    args = (si.seqlens, k, v, pre.k, pre.v, pre.seqlens)
    out, lse = torch.compile(f, backend="aot_eager", fullgraph=True)(q, si.k_pool, si.v_pool, *args)
    ref_out, ref_lse = f(q, si2.k_pool, si2.v_pool, *args)
    assert torch.equal(out, ref_out) and torch.equal(lse, ref_lse)
    assert torch.equal(bytes_of(si.k_pool), bytes_of(si2.k_pool))  # the compiled call appended too


def test_bench_decode_dry_run_shared_prefix():
    cmd = [sys.executable, os.path.join(ROOT, "benchmark", "bench_decode.py"), "--dry-run", "--shared-prefix",
           "32768", "--samples", "4"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:]
    rows = [json.loads(line) for line in r.stdout.splitlines() if line.startswith("{")]
    assert rows
    for x in rows:
        assert x["shared_prefix"] == 32768 and x["samples"] == 4
        assert x["prefix_bytes"] < x["copied_bytes"] and x["prefix_bytes"] < x["paged_bytes"]
