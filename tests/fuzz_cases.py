"""Randomised end-to-end cases for the table-driven launch contract, on CPU.

* ``world1_case(seed)``: the public API at world size 1 through ``tests/fake_ext.py`` (a torch implementation of each
  launch's contract, driven by the same work tables as the sm_90a kernels) against the dense fp32 oracle: random
  shapes, GQA ratios, head sizes, sliding windows, packed documents, causal or not, ordered (deterministic) launch
  groups.
* ``fused_case(seed)``: the fused multi-GPU launch replayed in one process (``tests/test_fused_emulation.py``) for a
  random scheme / world size / shard length / window / packing.

* ``dist_worker(...)``: the torch.distributed transports inside a spawned gloo world (per-source launches or dense
  blocks), every scheme incl. llama3 with ``heads_k_stride``.

``tests/test_fuzz.py`` runs a few fixed seeds; ``python tests/fuzz_cases.py world1|fused <first seed> <seconds>`` runs
until the time is up (round 2: 1591 world-1, 524 fused-replay, 430 distributed and 150 fp8 cases, no failure).
"""
import os
import random
import sys
import time
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)

import ring_flash_attn_b200 as rfa  # noqa: E402
from ring_flash_attn_b200.ops.dense import attention_oracle, varlen_attention_oracle  # noqa: E402
from ring_flash_attn_b200.parallel import api, layouts, ops, symm  # noqa: E402


def _close(a, b, name):
    err = (a.float() - b.float()).abs().max().item()
    ref = b.float().abs().max().item()
    assert err <= 3e-2 * ref + 2e-2, f"{name}: err {err} vs max {ref}"


def world1_case(seed: int):
    """One random world-1 call (needs ``fake_ext.install()``); returns a description of the case."""
    rnd = random.Random(seed)
    torch.manual_seed(seed)
    hkv = rnd.choice([1, 2, 3])
    hq = hkv * rnd.choice([1, 2, 4])
    d = rnd.choice([32, 64, 128])
    det = rnd.random() < 0.5
    window = rnd.choice([(-1, -1), (-1, -1), (rnd.randint(0, 500), 0), (rnd.randint(0, 300), rnd.randint(0, 300))])
    kind = rnd.choice(["ring", "zigzag", "stripe", "ring_varlen", "zigzag_varlen", "zzl3"])
    causal = True if kind in ("zigzag", "stripe", "zigzag_varlen", "zzl3") else rnd.random() < 0.6
    if causal and window[1] > 0:
        window = (window[0], 0)
    desc = (seed, kind, hq, hkv, d, window, causal, det)
    if kind in ("ring", "zigzag", "stripe"):
        B = rnd.choice([1, 2])
        S = rnd.choice([64, 128, 200, 256, 300, 514, 2 * rnd.randint(1, 400)])
        q = torch.randn(B, S, hq, d).to(torch.bfloat16)
        kv = torch.randn(B, S, 2, hkv, d).to(torch.bfloat16)
        dout = torch.randn(B, S, hq, d).to(torch.bfloat16)
        x, y = q.clone().requires_grad_(True), kv.clone().requires_grad_(True)
        prefix = {"ring": "ring", "zigzag": "zigzag_ring", "stripe": "stripe"}[kind]
        fn = getattr(rfa, prefix + "_flash_attn_kvpacked_func")
        out, lse, _ = fn(x, y, causal=causal, window_size=window, deterministic=det, return_attn_probs=True)
        out.backward(dout)
        rq, rkv = q.float().requires_grad_(True), kv.float().requires_grad_(True)
        ref, ref_lse = attention_oracle(rq, rkv[:, :, 0], rkv[:, :, 1], causal, window_size=window)
        ref.backward(dout.float())
        _close(out, ref, "out")
        _close(x.grad, rq.grad, "dq")
        _close(y.grad, rkv.grad, "dkv")
        m = torch.isfinite(ref_lse)
        assert (lse[m] - ref_lse[m]).abs().max() < 5e-3, "lse"
        return desc + (B, S)
    T = 2 * rnd.randint(8, 500)
    ndoc = rnd.randint(1, 5)
    if kind == "zzl3":  # documents of arbitrary lengths
        cuts = sorted(rnd.sample(range(1, T), min(ndoc - 1, T - 1)))
    else:  # every document is sharded on its own (zigzag: even lengths)
        cuts = sorted({2 * c for c in rnd.sample(range(1, T // 2), min(ndoc - 1, T // 2 - 1))})
    cu = torch.tensor([0] + cuts + [T], dtype=torch.int32)
    q, k, v = (torch.randn(T, h, d).to(torch.bfloat16) for h in (hq, hkv, hkv))
    dout = torch.randn(T, hq, d).to(torch.bfloat16)
    xs = [t.clone().requires_grad_(True) for t in (q, k, v)]
    if kind == "zzl3":
        out = rfa.zigzag_llama3_flash_attn_varlen_func(*xs, cu, causal=True, window_size=window, deterministic=det)
    else:
        fn = rfa.ring_flash_attn_varlen_func if kind == "ring_varlen" else rfa.zigzag_ring_flash_attn_varlen_func
        out = fn(*xs, cu, int((cu[1:] - cu[:-1]).max()), causal=causal, window_size=window, deterministic=det)
    out.backward(dout)
    rs = [t.float().requires_grad_(True) for t in (q, k, v)]
    ref, _ = varlen_attention_oracle(*rs, cu, causal, window_size=window)
    ref.backward(dout.float())
    _close(out, ref, "out")
    for a, b, nm in zip(xs, rs, "qkv"):
        _close(a.grad, b.grad, "d" + nm)
    return desc + (T, cu.tolist())


def fused_case(seed: int):
    """One random replay of the fused multi-GPU launch; returns a description of the case, or None when a llama3
    packing needs more row ranges per source than the device table holds (the library then uses the fallback)."""
    import test_fused_emulation as E

    rnd = random.Random(seed)
    world = rnd.choice([2, 3, 4, 5, 8])
    hkv = rnd.choice([1, 2])
    hq = hkv * rnd.choice([1, 2, 4])
    kind = rnd.choice(["ring", "zigzag", "stripe", "llama3", "zzl3"])
    window = rnd.choice([(-1, -1), (-1, -1), (rnd.randint(1, 700), 0)])
    L = rnd.choice([64, 128, 130, 192, 256, 300, 384, rnd.randint(2, 200) * 2])
    S = world * L
    torch.manual_seed(seed)
    desc = (seed, kind, world, L, hq, hkv, window)
    old_d, E.D = E.D, 32  # the tables do not depend on the head size
    try:
        D = E.D
        R = range(world)
        if kind in ("ring", "zigzag", "stripe"):
            q, k, v, dout = (torch.randn(1, S, h, D) for h in (hq, hkv, hkv, hq))
            rq, rk, rv = (t.clone().requires_grad_(True) for t in (q, k, v))
            ref, ref_lse = attention_oracle(rq, rk, rv, True, window_size=window)
            ref.backward(dout)
            shard = getattr(layouts, f"shard_{kind}")
            E._replay(E._plans(kind, world, L, window), world, L, hq, hkv,
                      [shard(q, r, world)[0] for r in R], [shard(k, r, world)[0] for r in R],
                      [shard(v, r, world)[0] for r in R], [shard(dout, r, world)[0] for r in R],
                      [shard(ref, r, world)[0] for r in R], [shard(ref_lse, r, world, dim=2)[0] for r in R],
                      [shard(rq.grad, r, world)[0] for r in R], [shard(rk.grad, r, world)[0] for r in R],
                      [shard(rv.grad, r, world)[0] for r in R])
            return desc
        ndoc = rnd.randint(1, 6)
        cu = tuple([0] + (sorted(rnd.sample(range(1, S), min(ndoc - 1, S - 1))) if ndoc > 1 else []) + [S])
        q, k, v, dout = (torch.randn(S, h, D) for h in (hq, hkv, hkv, hq))
        rq, rk, rv = (t.clone().requires_grad_(True) for t in (q, k, v))
        ref, ref_lse = varlen_attention_oracle(rq, rk, rv, torch.tensor(cu), True, window_size=window)
        ref.backward(dout)
        if kind == "llama3":
            plans = []
            for r in R:
                cq, ck, _mq, _mk, ks = api.llama3_flash_attn_prepare_cu_seqlens(torch.tensor(cu, dtype=torch.int32),
                                                                               True, r, world)
                plans.append(ops.llama3_plan(r, world, L, tuple(cq.tolist()), tuple(ck.tolist()), int(ks.start), True,
                                             window))
            if not all(symm.dynamic_ok(p) for p in plans):
                return None

            def sh(x, r):
                return layouts.shard_llama3(x, r, world)
        else:
            plans = [ops.zigzag_llama3_plan(r, world, cu, True, window) for r in R]

            def sh(x, r):
                return layouts.shard_zigzag_llama3(x, r, world)
        E._replay(plans, world, L, hq, hkv, [sh(q, r) for r in R], [sh(k, r) for r in R], [sh(v, r) for r in R],
                  [sh(dout, r) for r in R], [sh(ref, r) for r in R],
                  [sh(ref_lse.transpose(0, 1), r).transpose(0, 1) for r in R], [sh(rq.grad, r) for r in R],
                  [sh(rk.grad, r) for r in R], [sh(rv.grad, r) for r in R])
        return desc + (cu,)
    finally:
        E.D = old_d


def dist_worker(rank: int, world: int, seed0: int, ncases: int, use_fake: bool):
    """Random cases over the torch.distributed transports inside a spawned world (``dist_utils.run_distributed``):
    per-source launches of the table-driven contract (``use_fake``, bf16) or the dense fp32 blocks; batch schemes,
    varlen, llama3 (with ``heads_k_stride``), zigzag-llama3; windows; ordered mode."""
    warnings.simplefilter("ignore")
    os.environ["RFA_B200_DISABLE_P2P"] = "1"
    if use_fake:
        import fake_ext

        fake_ext.install()
    dt = torch.bfloat16 if use_fake else torch.float32
    for seed in range(seed0, seed0 + ncases):
        rnd = random.Random(seed)
        torch.manual_seed(seed)
        hkv = rnd.choice([1, 2])
        hq = hkv * rnd.choice([1, 2, 4])
        d = rnd.choice([32, 64, 128]) if use_fake else rnd.choice([16, 32])
        det = rnd.random() < 0.5
        window = rnd.choice([(-1, -1), (-1, -1), (rnd.randint(0, 400), 0)])
        kind = rnd.choice(["ring", "zigzag", "stripe", "ring_varlen", "zigzag_varlen", "llama3", "zzl3"])
        causal = True if kind not in ("ring", "ring_varlen") else rnd.random() < 0.6
        if not causal:
            window = (-1, -1) if rnd.random() < 0.5 else (rnd.randint(0, 300), rnd.randint(0, 300))
        if kind in ("ring", "zigzag", "stripe"):
            B = rnd.choice([1, 2])
            S = world * rnd.choice([32, 64, 130, 2 * rnd.randint(1, 150)])
            q, kv, dout = torch.randn(B, S, hq, d).to(dt), torch.randn(B, S, 2, hkv, d).to(dt), torch.randn(B, S, hq, d).to(dt)
            shard = getattr(layouts, f"shard_{kind}")
            x = shard(q, rank, world).clone().requires_grad_(True)
            y = shard(kv, rank, world).clone().requires_grad_(True)
            prefix = {"ring": "ring", "zigzag": "zigzag_ring", "stripe": "stripe"}[kind]
            out = getattr(rfa, prefix + "_flash_attn_kvpacked_func")(x, y, causal=causal, window_size=window,
                                                                     deterministic=det)
            out.backward(shard(dout, rank, world))
            rq, rkv = q.clone().float().requires_grad_(True), kv.clone().float().requires_grad_(True)
            ref, _ = attention_oracle(rq, rkv[:, :, 0], rkv[:, :, 1], causal, window_size=window)
            ref.backward(dout.float())
            _close(out, shard(ref, rank, world), f"{seed} out")
            _close(x.grad, shard(rq.grad, rank, world), f"{seed} dq")
            _close(y.grad, shard(rkv.grad, rank, world), f"{seed} dkv")
            continue
        ndoc = rnd.randint(1, 4)
        if kind in ("llama3", "zzl3"):
            T = 2 * world * rnd.randint(4, 120)
            cuts = sorted(rnd.sample(range(1, T), min(ndoc - 1, T - 1)))
        else:
            unit, nunits = 2 * world, rnd.randint(ndoc, 60)
            T = unit * nunits
            cuts = sorted({unit * c for c in rnd.sample(range(1, nunits), min(ndoc - 1, nunits - 1))}) if nunits > 1 else []
        cu = [0] + cuts + [T]
        cu_t = torch.tensor(cu, dtype=torch.int32)
        q, k, v = (torch.randn(T, h, d).to(dt) for h in (hq, hkv, hkv))
        dout = torch.randn(T, hq, d).to(dt)
        rs = [t.clone().float().requires_grad_(True) for t in (q, k, v)]
        ref, _ = varlen_attention_oracle(*rs, cu_t, causal, window_size=window)
        ref.backward(dout.float())
        if kind == "zzl3":
            def sh(t):
                return layouts.shard_zigzag_llama3(t, rank, world)

            xs = [sh(t).clone().requires_grad_(True) for t in (q, k, v)]
            out = rfa.zigzag_llama3_flash_attn_varlen_func(*xs, cu_t, causal=True, window_size=window, deterministic=det)
        elif kind == "llama3":
            def sh(t):
                return layouts.shard_llama3(t, rank, world)

            xs = [sh(t).clone().requires_grad_(True) for t in (q, k, v)]
            cq, ck, mq, mk, ks = rfa.llama3_flash_attn_prepare_cu_seqlens(cu_t, True, rank, world)
            out = rfa.llama3_flash_attn_varlen_func(*xs, cq, ck, mq, mk, heads_k_stride=rnd.choice([1, hkv]),
                                                    local_k_slice=ks, causal=True, window_size=window, deterministic=det)
        else:
            which = "ring" if kind == "ring_varlen" else "zigzag"

            def sh(t):
                return getattr(layouts, f"shard_{which}_varlen")(t, cu, rank, world)

            xs = [sh(t).clone().requires_grad_(True) for t in (q, k, v)]
            lcu = cu_t // world
            fn = rfa.ring_flash_attn_varlen_func if which == "ring" else rfa.zigzag_ring_flash_attn_varlen_func
            out = fn(*xs, lcu, int((lcu[1:] - lcu[:-1]).max()), causal=causal, window_size=window, deterministic=det)
        out.backward(sh(dout))
        _close(out, sh(ref), f"{seed} out")
        for a, b, nm in zip(xs, rs, "qkv"):
            _close(a.grad, sh(b.grad), f"{seed} d{nm}")


def fp8_worker(rank, world, seed0, n):
    """Random fp8 descale layouts (per tensor / head / token block / MX along head_dim) x schemes x entry points:
    either the fp8 launch contract (``attn_fwd_fp8`` with its scale tables) or the dequantise-to-bf16 path must match
    attention on the dequantised values of every rank.  Returns how many cases took which path."""
    import torch.distributed as dist

    import fake_ext
    from ring_flash_attn_b200.utils import fp8

    warnings.simplefilter("ignore")
    os.environ["RFA_B200_DISABLE_P2P"] = "1"
    fake = fake_ext.install()
    counts = {"kernel": 0, "dequant": 0}
    prefixes = {"ring": "ring", "zigzag": "zigzag_ring", "stripe": "stripe"}

    def gather(t, scheme):
        parts = [torch.empty_like(t.contiguous()) for _ in range(world)]
        dist.all_gather(parts, t.contiguous())
        return layouts.unshard(scheme, parts, dim=1)

    for seed in range(seed0, seed0 + n):
        rnd = random.Random(seed)
        torch.manual_seed(seed)
        os.environ["RFA_B200_FP8_KERNEL"] = rnd.choice(["1", "2", "2", "0"])
        hkv = rnd.choice([1, 2])
        hq = hkv * rnd.choice([1, 2])
        d = rnd.choice([128, 128, 64])
        scheme = rnd.choice(["ring", "zigzag", "stripe"])
        B = rnd.choice([1, 2])
        L = rnd.choice([128, 256, 384, 200, 512])
        S = L * world
        entry = rnd.choice(["func", "kvpacked", "qkvpacked"])
        if entry == "qkvpacked":
            hq = hkv
        tb = rnd.choice([0, 128, 64, L, 1 if L <= 256 else 128, 256 if L % 256 == 0 else 128])  # tokens per block, 0 = all
        if tb and L % tb:
            tb = 0
        per_head = rnd.choice([0, 1])      # 0: one scale for all heads, 1: one per head
        dblk = rnd.choice([0, 0, 0, 32])   # sometimes MX-style blocks along head_dim
        per_batch = 1 if tb else 0
        q = torch.randn(B, S, hq, d) * (1 + 2 * torch.rand(B, S, 1, 1))
        kv = torch.randn(B, S, 2, hkv, d) * (1 + torch.rand(B, S, 1, 1, 1))
        dist.broadcast(q, src=0)
        dist.broadcast(kv, src=0)
        shard = getattr(layouts, f"shard_{scheme}")
        lq, lkv = shard(q, rank, world), shard(kv, rank, world)
        desc = (seed, scheme, world, entry, B, L, hq, hkv, d, tb, per_head, dblk, os.environ["RFA_B200_FP8_KERNEL"])
        fake.calls.clear()
        if entry == "qkvpacked":
            x8, sc = fp8.quantize_blockwise(torch.cat([lq.unsqueeze(2), lkv], dim=2), [per_batch, tb, 1, per_head, dblk])
            deq = fp8.dequantize(x8, sc, torch.float32)
            dq_, dk_, dv_ = deq[:, :, 0], deq[:, :, 1], deq[:, :, 2]
            out = getattr(rfa, prefixes[scheme] + "_flash_attn_qkvpacked_func")(x8, causal=True, descale=sc)
        else:
            q8, sq = fp8.quantize_blockwise(lq, [per_batch, tb, per_head, dblk])
            kv8, skv = fp8.quantize_blockwise(lkv, [per_batch, tb, 1, per_head, dblk])
            dq_ = fp8.dequantize(q8, sq, torch.float32)
            dkv_ = fp8.dequantize(kv8, skv, torch.float32)
            dk_, dv_ = dkv_[:, :, 0], dkv_[:, :, 1]
            if entry == "kvpacked":
                out = getattr(rfa, prefixes[scheme] + "_flash_attn_kvpacked_func")(q8, kv8, causal=True, descale=(sq, skv))
            else:
                out = getattr(rfa, prefixes[scheme] + "_flash_attn_func")(
                    q8, kv8[:, :, 0], kv8[:, :, 1], causal=True, descale=(sq, skv[:, :, 0], skv[:, :, 1]))
        counts["kernel" if "attn_fwd_fp8" in fake.calls else "dequant"] += 1
        ref, _ = attention_oracle(gather(dq_, scheme), gather(dk_, scheme), gather(dv_, scheme), True)
        want = shard(ref, rank, world)
        err, mag = (out.float() - want).abs().max().item(), want.abs().max().item()
        assert out.dtype == torch.bfloat16 and err <= 3e-2 * mag + 2e-2, f"{desc}: err {err} vs {mag}, {set(fake.calls)}"
    return counts


def main():
    which, seed0, budget = sys.argv[1], int(sys.argv[2]), float(sys.argv[3])
    warnings.simplefilter("ignore")
    if which == "world1":
        import fake_ext

        fake_ext.install()
    case = world1_case if which == "world1" else fused_case
    t0, n, fails = time.time(), 0, 0
    while time.time() - t0 < budget:
        try:
            case(seed0 + n)
        except Exception as e:  # noqa: BLE001 - report and go on
            fails += 1
            print("FAIL seed", seed0 + n, type(e).__name__, str(e).splitlines()[0][:200], flush=True)
        n += 1
    print(f"done: {n} cases, {fails} failures", flush=True)


if __name__ == "__main__":
    main()
