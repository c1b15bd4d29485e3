#!/usr/bin/env python
"""The functional API in thirty lines: shard a sequence, run context-parallel attention, check it.

Same flow as the reference's test scripts (/root/reference/test/test_zigzag_ring_flash_attn_func.py:9-92: broadcast a
full qkv, cut out this rank's shard by hand, compare with single-device flash attention and print the differences),
with the hand-written slicing replaced by ``parallel.layouts`` and the printed differences by an assertion.

    torchrun --nproc-per-node 2 examples/ring_attention_minimal.py                  # CPU, gloo
    torchrun --nproc-per-node 8 examples/ring_attention_minimal.py --cuda           # H100s, fused NVLink path
    torchrun --nproc-per-node 8 examples/ring_attention_minimal.py --cuda --scheme stripe --seqlen 65536
"""
import argparse
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ring_flash_attn_b200 as rfa  # noqa: E402
from ring_flash_attn_b200.parallel import layouts  # noqa: E402
from ring_flash_attn_b200.utils.verify import sampled_check  # noqa: E402

FUNCS = {"ring": rfa.ring_flash_attn_qkvpacked_func, "zigzag": rfa.zigzag_ring_flash_attn_qkvpacked_func,
         "stripe": rfa.stripe_flash_attn_qkvpacked_func}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cuda", action="store_true")
    ap.add_argument("--scheme", default="zigzag", choices=sorted(FUNCS))
    ap.add_argument("--seqlen", type=int, default=0, help="global sequence length (default 256 per rank on CPU, 4096 on GPU)")
    ap.add_argument("--heads", type=int, default=4)
    ap.add_argument("--head-dim", type=int, default=128)
    args = ap.parse_args()
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29533")
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    dist.init_process_group("nccl" if args.cuda else "gloo", rank=rank, world_size=world)
    if args.cuda:
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dev = torch.device("cuda", torch.cuda.current_device()) if args.cuda else torch.device("cpu")
    dtype = torch.bfloat16
    S = args.seqlen or (4096 if args.cuda else 256) * world

    # every rank draws the same full tensors (a real job only ever holds its shard)
    torch.manual_seed(0)
    qkv = torch.randn(1, S, 3, args.heads, args.head_dim).to(dtype).to(dev)
    dout = torch.randn(1, S, args.heads, args.head_dim).to(dtype).to(dev)
    shard = getattr(layouts, f"shard_{args.scheme}")
    local = shard(qkv, rank, world).detach().requires_grad_(True)       # (1, S / world, 3, H, D)
    positions = layouts.positions(args.scheme, rank, world, S // world)  # global index of every local token (RoPE)

    out, lse, _ = FUNCS[args.scheme](local, causal=True, return_attn_probs=True)
    out.backward(shard(dout, rank, world))

    # fp32 oracle on sampled rows (collective: every rank calls it)
    g = local.grad[0]
    res = sampled_check(args.scheme, local[0, :, 0], local[0, :, 1], local[0, :, 2], shard(dout, rank, world)[0],
                        out[0], lse[0], g[:, 0], g[:, 1], g[:, 2], n_rows=64)
    if rank == 0:
        print(f"{args.scheme}: world {world}, S {S}, local tokens {S // world}, first positions "
              f"{positions[:4].tolist()}, max errors {res['max_err']}, ok={res['ok']}")
    assert res["ok"], res
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
