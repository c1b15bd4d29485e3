"""Dump the clock64 timeline of CTA 0 of the backward kernel (needs a build with RFA_TRACE=1).

    RFA_TRACE=1 python -c "import __graft_entry__ as g; g.build()"
    python benchmark/trace_bwd.py [--seq 32768] [--heads 32/32] [--dim 128]

Prints the stamps of query tiles 6-25 and, over every traced tile past the first few, the median cycles of the
per-tile intervals: where the tensor pipe of the thread-0 warpgroup waits between GEMMs.
"""
import argparse
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ring_flash_attn_b200 as rfa  # noqa: E402
from ring_flash_attn_b200.ops import cuda_ext  # noqa: E402

# slots written by thread 0 of CTA 0 per query tile (attn_bwd_sm90.cu, RFA_STAMP)
NAMES = ["S^T ready", "dP^T ready", "dS^T staged", "dQ issued", "dQ complete", "dQ reduced", "S^T issued",
         "dV/dK issued"]
# (label, (tile offset, slot) from, (tile offset, slot) to): intervals inside tile i or from tile i to tile i + 1
# (the next tile's S^T is issued right after this tile's dQ GEMM, before the wait for dQ and the dQ staging)
INTERVALS = [
    ("dQ issued -> next S^T issued", (0, 3), (1, 6)),
    ("next S^T issued -> dQ complete", (1, 6), (0, 4)),
    ("dQ complete -> dQ reduce-add issued", (0, 4), (0, 5)),
    ("dQ reduce-add issued -> next S^T ready", (0, 5), (1, 0)),
    ("S^T issued -> S^T ready", (0, 6), (0, 0)),
    ("dP^T ready -> dV/dK issued", (0, 1), (0, 7)),
    ("cycles per tile (S^T ready -> next S^T ready)", (0, 0), (1, 0)),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, default=32768)
    ap.add_argument("--heads", default="32/32", help="q/kv head counts")
    ap.add_argument("--dim", type=int, default=128)
    args = ap.parse_args()
    hq, hkv = (int(x) for x in args.heads.split("/"))
    C = cuda_ext.load()
    S, D = args.seq, args.dim
    q = torch.randn(1, S, hq, D, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    k = torch.randn(1, S, hkv, D, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    v = torch.randn(1, S, hkv, D, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    do = torch.randn(1, S, hq, D, device="cuda", dtype=torch.bfloat16)
    for _ in range(3):
        rfa.zigzag_ring_flash_attn_func(q, k, v, causal=True).backward(do)
    out = rfa.zigzag_ring_flash_attn_func(q, k, v, causal=True)
    trace = torch.zeros(64 * 16, dtype=torch.int64, device="cuda")
    C.set_trace(trace)
    out.backward(do)
    torch.cuda.synchronize()
    C.set_trace(None)
    t = trace.cpu().view(64, 16)
    base = int(t[t > 0].min())
    print(f"seq {S}, heads {hq}/{hkv}, d {D}: CTA 0, thread 0, clock64 cycles from its first stamp")
    print("tile " + " ".join(f"{n:>13s}" for n in NAMES))
    for i in range(6, 26):
        print(f"{i:4d} " + " ".join(f"{(int(x) - base) if x > 0 else -1:13d}" for x in t[i][:len(NAMES)]))
    for label, (da, sa), (db, sb) in INTERVALS:
        d = [int(t[i + db][sb]) - int(t[i + da][sa]) for i in range(4, 62)
             if t[i + da][sa] > 0 and t[i + db][sb] > 0]
        if d:
            print(f"{label:48s} median {statistics.median(d):8.0f}  min {min(d):8d}  max {max(d):8d}  (n={len(d)})")


if __name__ == "__main__":
    main()
