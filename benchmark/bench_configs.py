#!/usr/bin/env python
"""The four GPU configurations BASELINE.json names, one JSON line each, for this library or the reference.

    torchrun --nproc-per-node 8 benchmark/bench_configs.py [--impl reference] [--only zigzag,varlen,...]

  zigzag  : zigzag_ring_flash_attn_qkvpacked_func         bs=1 seq=32768 nheads=32 d=128 causal (headline)
  varlen  : zigzag_ring_flash_attn_varlen_qkvpacked_func  total_seq=32768 packed as 3 documents, causal
  llama3  : llama3_flash_attn_varlen_func                 GQA 32/8 heads, total_seq=65536, heads_k_stride=1
  stripe8 : stripe_flash_attn_qkvpacked_func              block-scaled fp8 inputs, bs=2 seq=16384 nheads=16

Every line carries the achieved fraction of the path's roofline: the slower of (attention FLOPs of one rank at
the H100 SXM data-sheet dense bf16 rate) and (bytes the rank must receive over NVLink at the data-sheet NVLink 4
bandwidth per direction).  Both are data-sheet figures for a 700 W card, not measured rates; a card with a lower
power limit or lower clocks will not reach them.  Timing: CUDA events per step, L2 flushed between steps, max over ranks.
The reference has no fp8 entry point, so ``stripe8`` runs its bf16 function on the dequantised tensors.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NVLINK_GBS = 450.0  # NVLink 4 per direction per GPU, H100 SXM data sheet (not a measured rate)
BF16_TFLOPS = 989.0  # dense bf16 tensor-core rate, H100 SXM data sheet at 700 W (not a measured rate)


def causal_flops(doc_lens, hq, d, fwd_only):
    f = sum(2.0 * n * n * hq * d for n in doc_lens)  # 4*n^2*H*d / 2 (causal)
    return f * (1.0 if fwd_only else 3.5)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--only", default="zigzag,varlen,llama3,stripe8")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--forward-only", action="store_true")
    ap.add_argument("--tiny", action="store_true", help="CPU/gloo dry run of the script itself (shapes / 64)")
    ap.add_argument("--fp8-per-head", action="store_true",
                    help="stripe8: per-head instead of per-128-token descales (the granularity the fp8 forward kernel "
                         "takes natively with RFA_B200_FP8_KERNEL=1; finer scales are dequantised to bf16 first)")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29517")
    if args.tiny:
        dev = torch.device("cpu")
        dist.init_process_group("gloo", rank=rank, world_size=world)
    else:
        dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
        torch.cuda.set_device(dev)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    shrink = 64 if args.tiny else 1
    if args.impl == "reference":
        sys.path.insert(0, ROOT)
        import bench as headline_bench

        mod = headline_bench.load_reference()
    else:
        import ring_flash_attn_b200 as mod
    from ring_flash_attn_b200.parallel import layouts
    from ring_flash_attn_b200.utils import fp8

    bf16 = torch.float32 if args.tiny else torch.bfloat16
    flush = torch.empty((1 if args.tiny else 256) * 1024 * 1024, dtype=torch.uint8, device=dev)
    gen = torch.Generator(device=dev).manual_seed(1234)

    def rnd(*shape):
        return torch.randn(*shape, device=dev, dtype=bf16, generator=gen)

    def bcast(t):
        dist.broadcast(t, src=0)
        return t

    def measure(step):
        if args.tiny:
            import time

            step()
            dist.barrier()
            t0 = time.perf_counter()
            step()
            ms = (time.perf_counter() - t0) * 1e3
            return ms, ms
        for _ in range(args.warmup):
            step()
        dist.barrier()
        torch.cuda.synchronize()
        evs = []
        for _ in range(args.steps):
            flush.fill_(1)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step()
            b.record()
            evs.append((a, b))
        dist.barrier()
        torch.cuda.synchronize()
        per = sorted(a.elapsed_time(b) for a, b in evs)
        t = torch.tensor([sum(per) / len(per), per[len(per) // 2]], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t[0]), float(t[1])

    def run_fb(call, leaves, dout):
        def step():
            if args.forward_only:
                with torch.no_grad():
                    call()
                return
            for t in leaves:
                t.grad = None
            call().backward(dout)
        return step

    def report(name, api, ms, med, flops_rank, rx_bytes, extra):
        if rank != 0:
            return
        t_flops = flops_rank / (BF16_TFLOPS * 1e12) * 1e3
        t_link = rx_bytes / (NVLINK_GBS * 1e9) * 1e3
        bound = max(t_flops, t_link)
        print(json.dumps({
            "config": name, "api": api, "impl": args.impl, "n_gpus": world,
            "mode": "fwd" if args.forward_only else "fwd_bwd", "ms_per_step": ms, "ms_median": med,
            "iter_per_s": 1000.0 / ms, "tflops_per_gpu": flops_rank / (ms * 1e-3) / 1e12,
            "roofline": {"compute_ms": t_flops, "nvlink_ms": t_link, "bound": "compute" if t_flops >= t_link else "nvlink",
                         "fraction": bound / ms, "peaks": "H100 SXM data sheet (989 TFLOP/s bf16, 450 GB/s NVLink)"},
            "steps": args.steps, "warmup": args.warmup, "l2": "flushed between steps", **extra}), flush=True)

    fwd = args.forward_only
    d = 16 if args.tiny else 128
    from ring_flash_attn_b200.parallel import ops as _ops
    from ring_flash_attn_b200.parallel.symm import _ranges

    def link_bytes(plan, hkv, batch=1):
        """NVLink bytes of the busiest rank, per direction: K/V rows of other shards this rank's queries can see (model
        dtype, received in the forward and again in the backward) plus the dK/dV partials for the same rows (model
        dtype since round 2; round 1 and the reference send fp32, i.e. twice these bytes).  The links are full duplex:
        what a rank receives (K/V in, dK/dV of its own shard in) and what it sends are of the same size."""
        rows = sum(hi - lo for src in range(world) if src != rank for lo, hi in _ranges(plan, src))
        kv = rows * hkv * d * 2 * 2
        total = kv * (1 if fwd else 2) + (0 if fwd else kv)
        t = torch.tensor([float(total)], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t[0])
    for name in args.only.split(","):
        if name == "zigzag":
            S, H = 32768 // shrink, 32 // min(shrink, 8)
            L = S // world
            qkv = rnd(1, L, 3, H, d).requires_grad_(True)
            dout = rnd(1, L, H, d)
            fn = mod.zigzag_ring_flash_attn_qkvpacked_func
            ms, med = measure(run_fb(lambda: fn(qkv, causal=True), [qkv], dout))
            rx = link_bytes(_ops.batch_plan("zigzag", rank, world, 1, L, True), H)
            report(name, "zigzag_ring_flash_attn_qkvpacked_func", ms, med, causal_flops([S], H, d, fwd) / world, rx,
                   {"seq_len": S, "nheads": H})
        elif name == "varlen":
            S, H = 32768 // shrink, 32 // min(shrink, 8)
            unit = S // 16  # three documents, each divisible by 2*world for world <= 8
            lens = [3 * unit, 8 * unit, 5 * unit]
            cu = [0, lens[0], lens[0] + lens[1], S]
            local_cu = torch.tensor([c // world for c in cu], dtype=torch.int32, device=dev)
            max_s = max(lens) // world
            L = S // world
            qkv = rnd(L, 3, H, d).requires_grad_(True)
            dout = rnd(L, H, d)
            fn = mod.zigzag_ring_flash_attn_varlen_qkvpacked_func
            ms, med = measure(run_fb(lambda: fn(qkv, local_cu, max_s, causal=True), [qkv], dout))
            rx = link_bytes(_ops.varlen_plan("zigzag", rank, world, tuple(c // world for c in cu), True), H)
            report(name, "zigzag_ring_flash_attn_varlen_qkvpacked_func", ms, med,
                   causal_flops(lens, H, d, fwd) / world, rx, {"total_seq": S, "docs": lens, "nheads": H})
        elif name == "llama3":
            S, HQ, HK = 65536 // shrink, 32 // min(shrink, 4), 8 // min(shrink, 4)
            unit = S // 16
            lens = [5 * unit, 4 * unit, 7 * unit]
            cu = torch.tensor([0, lens[0], lens[0] + lens[1], S], dtype=torch.int32, device=dev)
            L = S // world
            q = rnd(L, HQ, d).requires_grad_(True)
            k = rnd(L, HK, d).requires_grad_(True)
            v = rnd(L, HK, d).requires_grad_(True)
            dout = rnd(L, HQ, d)
            cq, ck, mq, mk, ks = mod.llama3_flash_attn_prepare_cu_seqlens(cu, True, rank, world)
            fn = mod.llama3_flash_attn_varlen_func
            ms, med = measure(run_fb(lambda: fn(q, k, v, cq, ck, mq, mk, heads_k_stride=1, local_k_slice=ks,
                                                causal=True), [q, k, v], dout))
            # this rank's share of the causal work: its queries against the keys of their documents up to them
            rx = link_bytes(_ops.llama3_plan(rank, world, L, tuple(cq.tolist()), tuple(ck.tolist()), int(ks.start),
                                              True), HK)
            lo, hi = rank * L, (rank + 1) * L
            pairs, start = 0.0, 0
            for n in lens:
                a, b = max(lo, start), min(hi, start + n)
                if b > a:
                    pairs += sum(range(a - start + 1, b - start + 1)) if b - a < 4096 else \
                        ((a - start + 1) + (b - start)) * (b - a) / 2.0
                start += n
            fl = 4.0 * pairs * HQ * d * (1.0 if fwd else 3.5)
            flt = torch.tensor([fl], dtype=torch.float64, device=dev)
            dist.all_reduce(flt, op=dist.ReduceOp.MAX)  # the slowest rank's work bounds the step
            report(name, "llama3_flash_attn_varlen_func", ms, med, float(flt[0]), rx,
                   {"total_seq": S, "docs": lens, "nheads_q": HQ, "nheads_kv": HK, "heads_k_stride": 1})
        elif name == "stripe8":
            B, S, H = 2, 16384 // shrink, 16 // min(shrink, 8)
            L = S // world
            full = bcast(rnd(B, S, 3, H, d)) if world <= 8 else None
            local = layouts.shard_stripe(full, rank, world).contiguous()
            del full
            if args.fp8_per_head:
                q8, scale = fp8.quantize_blockwise(local, [0, 0, 1, 1, 0])
            else:
                q8, scale = fp8.quantize_blockwise(local, [1, 128 // min(shrink, 16), 1, 1, 0])  # 128-token block x head
            dout = rnd(B, L, H, d)
            if args.impl == "ours":
                fn = mod.stripe_flash_attn_qkvpacked_func
                call = lambda: fn(q8, causal=True, descale=scale)  # noqa: E731
                leaves = []
                step = run_fb(call, leaves, dout) if fwd else None
                if not fwd:
                    # fp8 leaves carry no gradient: differentiate with respect to the dequantised tensor, which is
                    # what a training step does (the quantised copy is an activation, not a parameter)
                    deq = fp8.dequantize(q8, scale).to(bf16).requires_grad_(True)
                    step = run_fb(lambda: fn(deq, causal=True), [deq], dout)
            else:
                deq = fp8.dequantize(q8, scale).to(bf16).requires_grad_(True)
                fn = mod.stripe_flash_attn_qkvpacked_func
                step = run_fb(lambda: fn(deq, causal=True), [deq], dout)
            ms, med = measure(step)
            rx = link_bytes(_ops.batch_plan("stripe", rank, world, B, L, True), H)
            report(name, "stripe_flash_attn_qkvpacked_func", ms, med, B * causal_flops([S], H, d, fwd) / world, rx,
                   {"batch": B, "seq_len": S, "nheads": H, "inputs": "e4m3 + per-128-token scales" if fwd and
                    args.impl == "ours" else "bf16 (dequantised)"})
        else:
            raise SystemExit(f"unknown config {name}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
