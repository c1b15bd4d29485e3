"""Dump the clock64 timeline of CTA 0 of the backward kernel (needs a build with RFA_TRACE=1)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ring_flash_attn_b200 as rfa  # noqa: E402
from ring_flash_attn_b200.ops import cuda_ext  # noqa: E402

C = cuda_ext.load()
S, HQ, HKV = 8192, 32, 8
q = torch.randn(1, S, HQ, 128, device="cuda", dtype=torch.bfloat16, requires_grad=True)
k = torch.randn(1, S, HKV, 128, device="cuda", dtype=torch.bfloat16, requires_grad=True)
v = torch.randn(1, S, HKV, 128, device="cuda", dtype=torch.bfloat16, requires_grad=True)
do = torch.randn(1, S, HQ, 128, device="cuda", dtype=torch.bfloat16)
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
# slots written by thread 0 of CTA 0 per query tile (attn_bwd_sm90.cu, RFA_STAMP)
names = ["S^T ready", "dP^T ready", "dS^T staged", "dQ issued"]
print("tile " + " ".join(f"{n:>12s}" for n in names))
for i in range(6, 26):
    print(f"{i:4d} " + " ".join(f"{(int(x) - base) if x > 0 else -1:12d}" for x in t[i][:len(names)]))
per = [(int(t[i + 1][0]) - int(t[i][0])) for i in range(8, 40) if t[i + 1][0] > 0 and t[i][0] > 0]
print("cycles per tile (S^T ready deltas):", per[:16], "mean", sum(per) / max(1, len(per)))
