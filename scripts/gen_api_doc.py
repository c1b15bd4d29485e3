#!/usr/bin/env python
"""Regenerate docs/API.md from the docstrings and signatures of the public surface."""
import inspect
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ring_flash_attn_b200 as rfa  # noqa: E402
from ring_flash_attn_b200 import utils  # noqa: E402
from ring_flash_attn_b200.models import hf_adapter  # noqa: E402
from ring_flash_attn_b200.parallel import api, layouts  # noqa: E402

lines = ["# API reference (generated from the docstrings: `python scripts/gen_api_doc.py`)", "",
         "Names, argument order and defaults of the 19 attention functions and 2 adapter functions are those of",
         "zhuzilin/ring-flash-attention; everything else is marked *(extension)*.", ""]


def section(title):
    lines.extend(["", f"## {title}", ""])


def entry(name, obj, ext=False):
    try:
        sig = str(inspect.signature(obj))
    except (TypeError, ValueError):
        sig = "(...)"
    lines.append(f"### `{name}{sig}`" + (" *(extension)*" if ext else ""))
    lines.append("")
    doc = inspect.getdoc(obj)
    if doc:
        lines.extend([doc, ""])


section("Attention functions (`ring_flash_attn_b200`)")
for n in api.__all__:
    entry(n, getattr(rfa, n), ext=n.startswith("zigzag_llama3"))
lines += ["All functions additionally accept the keyword-only `descale=` *(extension)*: block-scaled fp8 inputs, see",
          "`ring_flash_attn_b200.utils.fp8`.", "",
          "Shared keyword arguments:", "",
          "* `causal`: on GLOBAL positions of the sharded sequence; zigzag / stripe require `True` (as in the reference).",
          "* `window_size=(left, right)`: sliding window on global positions, every scheme; `-1` = unbounded.",
          "* `softmax_scale`: default `head_dim ** -0.5` of the unpadded head size.",
          "* `dropout_p`, `alibi_slopes`: must be `0.0` / `None` (`NotImplementedError` otherwise).",
          "* `deterministic=True`: out / lse / dQ / dK / dV bitwise reproducible. On the sm_90a path the backward then",
          "  launches its key tiles in groups with disjoint query rows and, across GPUs, uses the fixed-order",
          "  torch.distributed transport (several times slower; a one-time `RuntimeWarning` says so).",
          "  `RFA_B200_DETERMINISTIC=fast` keeps the fused schedule: dK / dV reproducible, dQ an unordered fp32 sum.",
          "* `return_attn_probs=True`: returns `(out, softmax_lse, None)`; lse is fp32, `(B, H, S_local)` (batch) or",
          "  `(H, T_local)` (varlen).",
          "* `group`: the context-parallel process group (`None` = world). Every rank of the group must make the same",
          "  calls in the same order: on H100s the launches contain the K/V exchange.",
          "* packed inputs (`qkv`, `kv`): sliced as views; their gradient is written as one concatenation.", ""]
section("Decoding over a sharded KV cache (`ring_flash_attn_b200`, implemented in `parallel/decode.py`)")
entry("cp_flash_attn_with_kvcache", rfa.cp_flash_attn_with_kvcache, ext=True)
section("Hugging Face adapter (`ring_flash_attn_b200`, implemented in `models/hf_adapter.py`)")
for n in ("substitute_hf_flash_attn", "update_ring_flash_attn_params", "use_ring_attn"):
    entry(n, getattr(hf_adapter, n))
entry("restore_hf_flash_attn", hf_adapter.restore_hf_flash_attn, ext=True)
section("Reference-compatible helpers (`ring_flash_attn_b200.utils`)")
for n in sorted(getattr(utils, "__all__", [])):
    entry(n, getattr(utils, n))
section("Layouts (`ring_flash_attn_b200.parallel.layouts`) *(extension)*")
for n, o in inspect.getmembers(layouts, inspect.isfunction):
    if not n.startswith("_") and o.__module__ == layouts.__name__:
        entry(n, o, ext=True)
section("Verification and the op boundary *(extension)*")
from ring_flash_attn_b200.parallel import ops  # noqa: E402
from ring_flash_attn_b200.utils import verify  # noqa: E402

entry("ring_flash_attn_b200.utils.verify.sampled_check", verify.sampled_check, ext=True)
lines += ["### `torch.ops.rfa_b200.cp_attn_fwd` / `cp_attn_bwd` *(extension)*", "", inspect.getdoc(ops), ""]
with open(os.path.join(ROOT, "docs", "API.md"), "w") as f:
    f.write("\n".join(lines) + "\n")
print("wrote docs/API.md:", len(lines), "lines")
