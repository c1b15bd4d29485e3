"""Time the sm_90a attention backward kernel alone at the headline shape (world 1, zigzag, causal).

    python benchmark/bench_bwd.py [--seq 32768] [--heads 32/32,32/8] [--dims 128,64] [--iters 20] [--warmup 5]
                                  [--deterministic] [--dump DIR]

For every (heads, head_dim) case: one forward, then two rounds of ``--iters`` backward passes through the public API,
each after a 256 MiB L2 flush.  The first round runs under ``torch.profiler`` (CUDA activity) and gives the
``attn_bwd_kernel`` time, summed over the kernel launches of one backward; the second, with the profiler off, gives
the whole backward (delta kernel, dq accumulator and casts included) from CUDA events.  Rates are over the kernel
time: FLOPs = 2.5 x the causal forward's 2 S^2 Hq D.  ``--deterministic`` runs the backward with a fixed dq reduction
order.  ``--dump DIR`` writes dq / dk / dv of the last pass as ``DIR/<case>_{dq,dk,dv}.npy`` (float32) for a bitwise
comparison of two builds.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEAK_BF16_TFLOPS = 989.0  # H100 SXM data sheet, dense bf16


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, default=32768)
    ap.add_argument("--heads", default="32/32,32/8", help="comma-separated q/kv head counts")
    ap.add_argument("--dims", default="128,64", help="comma-separated head dims")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--deterministic", action="store_true", help="fixed dq reduction order")
    ap.add_argument("--dump", metavar="DIR", default=None)
    args = ap.parse_args(argv)
    heads = []
    for h in args.heads.split(","):
        hq, hkv = (int(x) for x in h.split("/"))
        if hq <= 0 or hkv <= 0 or hq % hkv:
            ap.error(f"--heads {h}: q heads must be a positive multiple of kv heads")
        heads.append((hq, hkv))
    dims = [int(d) for d in args.dims.split(",")]
    if any(d not in (64, 128) for d in dims):
        ap.error("--dims: the kernels take head_dim 64 or 128")
    # the headline case (first heads entry at the first dim) plus every other head layout / dim at the headline dim
    cases = [(hq, hkv, dims[0]) for hq, hkv in heads] + [(heads[0][0], heads[0][1], d) for d in dims[1:]]
    return args, cases


def bwd_flops(seq: int, hq: int, d: int) -> float:
    """Causal backward FLOPs: 2.5 x the causal forward (4 S^2 Hq D / 2)."""
    return 2.5 * 2.0 * seq * seq * hq * d


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        return out.strip().splitlines()[0] if out.strip() else None
    except (OSError, subprocess.TimeoutExpired):
        return None


def per_pass_times(kernel_us, iters):
    """Kernel time of each pass (ms) from the recorded launches of ``iters`` passes, which must all be there."""
    if not kernel_us or len(kernel_us) % iters:
        raise SystemExit(f"recorded {len(kernel_us)} attn_bwd_kernel launches for {iters} passes")
    n = len(kernel_us) // iters
    return [sum(kernel_us[i * n:(i + 1) * n]) / 1000.0 for i in range(iters)], n


def run_case(torch, rfa, seq, hq, hkv, d, iters, warmup, dump, deterministic):
    from torch.profiler import ProfilerActivity, profile

    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(1234)
    q = torch.randn(1, seq, hq, d, device=dev, generator=g).to(torch.bfloat16).requires_grad_(True)
    k = torch.randn(1, seq, hkv, d, device=dev, generator=g).to(torch.bfloat16).requires_grad_(True)
    v = torch.randn(1, seq, hkv, d, device=dev, generator=g).to(torch.bfloat16).requires_grad_(True)
    dout = torch.randn(1, seq, hq, d, device=dev, generator=g).to(torch.bfloat16)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    out = rfa.zigzag_ring_flash_attn_func(q, k, v, causal=True, deterministic=deterministic)

    def bwd():
        q.grad = k.grad = v.grad = None
        out.backward(dout, retain_graph=True)

    for _ in range(warmup):
        bwd()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            flush.fill_(1)
            bwd()
        torch.cuda.synchronize()
    kern = [e.device_time for e in prof.events() if e.device_type.name == "CUDA" and "attn_bwd_kernel" in e.name]
    times, per_pass = per_pass_times(kern, iters)
    kernel_ms = statistics.median(times)
    events = []
    for _ in range(iters):
        flush.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        bwd()
        b.record()
        events.append((a, b))
    torch.cuda.synchronize()
    bwd_ms = statistics.median(a.elapsed_time(b) for a, b in events)
    flops = bwd_flops(seq, hq, d)
    name = f"s{seq}_h{hq}-{hkv}_d{d}" + ("_det" if deterministic else "")
    if dump:
        import numpy as np

        os.makedirs(dump, exist_ok=True)
        for t, n in ((q.grad, "dq"), (k.grad, "dk"), (v.grad, "dv")):
            np.save(os.path.join(dump, f"{name}_{n}.npy"), t.detach().float().cpu().numpy())
    return {"case": name, "kernel_ms": kernel_ms, "kernel_ms_min": min(times), "kernel_ms_max": max(times),
            "backward_ms": bwd_ms, "kernel_tflops": flops / (kernel_ms * 1e-3) / 1e12,
            "kernel_peak_fraction": flops / (kernel_ms * 1e-3) / 1e12 / PEAK_BF16_TFLOPS,
            "launches_per_pass": per_pass}


def main():
    args, cases = parse()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_bwd.py needs a CUDA device")
    sys.path.insert(0, ROOT)
    import ring_flash_attn_b200 as rfa

    info = {"card": card(), "peak_bf16_tflops_datasheet": PEAK_BF16_TFLOPS}
    for hq, hkv, d in cases:
        res = run_case(torch, rfa, args.seq, hq, hkv, d, args.iters, args.warmup, args.dump, args.deterministic)
        print(json.dumps({**res, **info}))


if __name__ == "__main__":
    main()
