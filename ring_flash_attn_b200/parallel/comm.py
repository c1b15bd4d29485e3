"""torch.distributed transports used by the fallback (CPU/gloo, or GPUs without peer access).

Capability parity with the reference's ``RingComm`` and ``AllGatherComm``
(/root/reference/ring_flash_attn/utils.py:98-168).  The fused sm_90a path does not use these: the
attention kernels' own communication CTAs push K/V rows into the peers' memory over NVLink
(``parallel/symm.py``, ``csrc/comm_device.cuh``).
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.distributed as dist


def _wire(t: torch.Tensor) -> torch.Tensor:
    """One-byte float tensors (fp8 K/V of the experimental fp8 forward) travel as uint8: same bytes, and every
    backend knows the type."""
    return t.view(torch.uint8) if t.element_size() == 1 and t.dtype != torch.uint8 else t


def group_info(group: Optional[dist.ProcessGroup]):
    """(rank, world) of ``group``; (0, 1) when torch.distributed is not initialised."""
    if not (dist.is_available() and dist.is_initialized()):
        return 0, 1
    return dist.get_rank(group), dist.get_world_size(group)


class RingComm:
    """Neighbour exchange on a ring: send to ``rank+1``, receive from ``rank-1``.

    ``send_recv`` only *queues* the two point-to-point ops; ``commit`` launches everything queued
    as one batch and ``wait`` blocks (stream-wise on NCCL) until it has landed.  Misuse raises, as
    in the reference (utils.py:129-140)."""

    def __init__(self, group: Optional[dist.ProcessGroup]):
        self.group = group
        self.rank, self.world = group_info(group)
        self._queued: List[dist.P2POp] = []
        self._inflight = None
        nxt = (self.rank + 1) % self.world
        prv = (self.rank - 1) % self.world
        if group is not None and self.world > 1:
            nxt = dist.get_global_rank(group, nxt)
            prv = dist.get_global_rank(group, prv)
        self.send_rank, self.recv_rank = nxt, prv

    def send_recv(self, to_send: torch.Tensor, recv_buf: Optional[torch.Tensor] = None) -> torch.Tensor:
        out = torch.empty_like(to_send) if recv_buf is None else recv_buf
        if self.world == 1:
            out.copy_(to_send)
            return out
        self._queued.append(dist.P2POp(dist.isend, _wire(to_send), self.send_rank, group=self.group))
        self._queued.append(dist.P2POp(dist.irecv, _wire(out), self.recv_rank, group=self.group))
        return out

    def commit(self) -> None:
        if self._inflight is not None:
            raise RuntimeError("commit called twice")
        self._inflight = dist.batch_isend_irecv(self._queued) if self._queued else []

    def wait(self) -> None:
        if self._inflight is None:
            raise RuntimeError("wait called before commit")
        for req in self._inflight:
            req.wait()
        self._inflight = None
        self._queued = []

    def send_recv_kv(self, k, v, k_buf=None, v_buf=None):
        nk, nv = self.send_recv(k, k_buf), self.send_recv(v, v_buf)
        self.commit()
        return nk, nv


class AllGatherComm:
    """Asynchronous all-gather with a handle list (utils.py:154-168)."""

    def __init__(self, group: Optional[dist.ProcessGroup] = None):
        self.group = group
        self.rank, self.world = group_info(group)
        self._handles = []

    def all_gather(self, output: torch.Tensor, inp: torch.Tensor) -> None:
        if self.world == 1:
            output.copy_(inp.reshape(output.shape))
            return
        self._handles.append(dist.all_gather_into_tensor(_wire(output), _wire(inp), group=self.group, async_op=True))

    def wait(self) -> None:
        for h in self._handles:
            h.wait()
        self._handles = []
