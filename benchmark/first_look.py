"""Single-GPU kernel timings: sm_90a kernels vs flash_attn 2.8 (the kernel the reference calls)."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ring_flash_attn_b200 as rfa  # noqa: E402


def timeit(fn, iters=20, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    res = {}
    try:
        if os.environ.get("RFA_FIRST_LOOK_SKIP_FA2", "0") == "1":  # variant sweeps only need our side
            raise ImportError("skipped")
        from flash_attn import flash_attn_func
    except Exception as e:  # noqa: BLE001
        flash_attn_func = None
        res["flash_attn_import_error"] = str(e)
    for (s, hq, hkv) in [(4096, 32, 32), (8192, 32, 8), (16384, 32, 8)]:
        q = torch.randn(1, s, hq, 128, device="cuda", dtype=torch.bfloat16, requires_grad=True)
        k = torch.randn(1, s, hkv, 128, device="cuda", dtype=torch.bfloat16, requires_grad=True)
        v = torch.randn(1, s, hkv, 128, device="cuda", dtype=torch.bfloat16, requires_grad=True)
        do = torch.randn(1, s, hq, 128, device="cuda", dtype=torch.bfloat16)
        fl_f = 2.0 * s * s * hq * 128  # causal fwd
        row = {}

        def ours_f():
            with torch.no_grad():
                return rfa.zigzag_ring_flash_attn_func(q, k, v, causal=True)

        def ours_fb():
            q.grad = k.grad = v.grad = None
            rfa.zigzag_ring_flash_attn_func(q, k, v, causal=True).backward(do)

        try:
            t = timeit(ours_f)
            row["ours_fwd_ms"] = t
            row["ours_fwd_tflops"] = fl_f / t / 1e9
            t = timeit(ours_fb)
            row["ours_fwdbwd_ms"] = t
            row["ours_fwdbwd_tflops"] = 3.5 * fl_f / t / 1e9
        except Exception as e:  # noqa: BLE001
            row["ours_error"] = str(e)[:400]
        if flash_attn_func is not None:
            def fa_f():
                with torch.no_grad():
                    return flash_attn_func(q, k, v, causal=True)

            def fa_fb():
                q.grad = k.grad = v.grad = None
                flash_attn_func(q, k, v, causal=True).backward(do)

            t = timeit(fa_f)
            row["fa2_fwd_ms"] = t
            row["fa2_fwd_tflops"] = fl_f / t / 1e9
            t = timeit(fa_fb)
            row["fa2_fwdbwd_ms"] = t
            row["fa2_fwdbwd_tflops"] = 3.5 * fl_f / t / 1e9
        res[f"s{s}_hq{hq}_hkv{hkv}"] = row
        print(s, hq, hkv, json.dumps(row))
    os.makedirs("gpurun_out", exist_ok=True)
    with open(os.environ.get("RFA_FIRST_LOOK_OUT", "gpurun_out/first_look.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
