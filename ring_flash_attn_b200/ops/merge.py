"""Online-softmax merge of partial attention results.

Capability parity with the reference's ``update_out_and_lse`` (/root/reference/ring_flash_attn/utils.py:32-73).
The fused sm_90a path never calls this - the accumulator stays in registers across key
shards - but the torch.distributed fallback path and the tests do.

Layout here is token-major: out ``(T, H, D)`` fp32, lse ``(H, T)`` fp32.  ``-inf`` lse (a row that
has seen no key yet) is the identity element.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch


def merge_partial(
    out: Optional[torch.Tensor],
    lse: Optional[torch.Tensor],
    block_out: torch.Tensor,
    block_lse: torch.Tensor,
    rows: Optional[slice] = None,
) -> Tuple[torch.Tensor, torch.Tensor]:
    """Merge ``(block_out, block_lse)`` into the running ``(out, lse)``.

    ``rows`` restricts the update to a row range of the running state (the reference's ``slice_``
    argument, utils.py:65-70); the block tensors then cover only that range.  The first call
    (``out is None``) must cover all rows, mirroring the reference's guard (utils.py:61-62).
    """
    block_out = block_out.float()
    block_lse = block_lse.float()
    if out is None:
        if rows is not None:
            raise RuntimeError("the first merge must cover every row (no row slice)")
        return block_out.clone(), block_lse.clone()
    if rows is None:
        o, l = out, lse
    else:
        o, l = out[rows], lse[:, rows]
    new_lse = torch.logaddexp(l, block_lse)
    # weights; guard the (-inf, -inf) case where logaddexp gives -inf and exp(nan) would appear
    safe = torch.where(torch.isinf(new_lse), torch.zeros_like(new_lse), new_lse)
    w_old = torch.exp(l - safe).transpose(0, 1).unsqueeze(-1)  # (T, H, 1)
    w_new = torch.exp(block_lse - safe).transpose(0, 1).unsqueeze(-1)
    new_out = o * w_old + block_out * w_new
    if rows is None:
        return new_out, new_lse
    out[rows] = new_out
    lse[:, rows] = new_lse
    return out, lse


def update_out_and_lse(out, lse, block_out, block_lse, slice_=None):
    """Drop-in for the reference primitive, in the reference's layouts.

    out ``(B,S,H,D)`` fp32, lse ``(B,S,H,1)`` fp32 running state; block_out ``(B,S,H,D)``,
    block_lse ``(B,H,S)`` (/root/reference/ring_flash_attn/utils.py:53-73).  ``slice_`` is a tuple
    of slices indexing the running state."""
    block_out = block_out.float()
    block_lse = block_lse.float().transpose(-2, -1).unsqueeze(-1)
    if out is None:
        if slice_ is not None:
            raise RuntimeError("first update_out_and_lse should not pass slice_ args")
        return block_out, block_lse
    if slice_ is not None:
        o, l = out[slice_], lse[slice_]
    else:
        o, l = out, lse
    new_lse = torch.logaddexp(l, block_lse)
    safe = torch.where(torch.isinf(new_lse), torch.zeros_like(new_lse), new_lse)
    new_out = o * torch.exp(l - safe) + block_out * torch.exp(block_lse - safe)
    if slice_ is not None:
        out[slice_], lse[slice_] = new_out, new_lse
        return out, lse
    return new_out, new_lse
