#!/usr/bin/env python
"""Context-parallel training step of a Hugging Face Llama with packed documents (llama3-style CP).

The flow is the one the reference documents for its adapter (/root/reference/README.md:35-61,
ring_flash_attn/adapters/hf_adapter.py): patch transformers once, publish the batch's global ``cu_seqlens`` once
per step, then feed every rank its contiguous slice of the token stream.  Runs on CPU/gloo (dense fp32 blocks) or
on GPUs (sm_90a kernels, fused NVLink path):

    torchrun --nproc-per-node 2 examples/train_hf_llama_cp.py            # CPU, gloo
    torchrun --nproc-per-node 8 examples/train_hf_llama_cp.py --cuda     # one process per GPU

Each rank holds tokens [rank*L, (rank+1)*L) of the packed stream and the matching position ids (positions restart
at every document); the loss is the sum over local tokens, gradients are all-reduced like any data-parallel model
because the weights are replicated across the context-parallel group.
"""
import argparse
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ring_flash_attn_b200 as rfa  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cuda", action="store_true")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--tokens", type=int, default=0, help="packed tokens per step (default: 64 per rank on CPU)")
    ap.add_argument("--layout", default="llama3", choices=["llama3", "zigzag"],
                    help="llama3: contiguous slice per rank (the reference's layout); zigzag: chunks r and 2W-1-r of the "
                         "packed stream (balanced causal work, extension)")
    args = ap.parse_args()
    from transformers import LlamaConfig, LlamaForCausalLM

    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29531")
    if args.cuda:
        dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
        torch.cuda.set_device(dev)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
        dtype, head_dim, hidden = torch.bfloat16, 128, 1024
    else:
        dev = torch.device("cpu")
        dist.init_process_group("gloo", rank=rank, world_size=world)
        dtype, head_dim, hidden = torch.float32, 16, 64
    heads = hidden // head_dim
    cfg = LlamaConfig(vocab_size=1024, hidden_size=hidden, intermediate_size=2 * hidden, num_hidden_layers=2,
                      num_attention_heads=heads, num_key_value_heads=max(1, heads // 2),
                      max_position_embeddings=1 << 17, attn_implementation="sdpa")
    torch.manual_seed(0)  # same weights on every rank
    model = LlamaForCausalLM(cfg).to(dev, dtype)
    # route every attention layer through the context-parallel kernels
    rfa.substitute_hf_flash_attn(process_group=None, heads_k_stride=1, layout=args.layout)
    from ring_flash_attn_b200.parallel import layouts

    def shard(x):  # (1, total) -> this rank's (1, L) tokens
        if args.layout == "zigzag":
            return layouts.shard_zigzag_llama3(x[0], rank, world).unsqueeze(0)
        return x[:, rank * (x.shape[1] // world):(rank + 1) * (x.shape[1] // world)]
    model.config._attn_implementation = "flash_attention_2"
    for layer in model.model.layers:
        layer.self_attn.config._attn_implementation = "flash_attention_2"
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3)

    total = args.tokens or (64 if not args.cuda else 8192) * world
    gen = torch.Generator().manual_seed(1)
    for step in range(args.steps):
        # a packed batch: three documents of uneven length, identical on every rank
        cut1 = int(torch.randint(total // 8, total // 2, (1,), generator=gen))
        cut2 = int(torch.randint(cut1 + 1, total - 1, (1,), generator=gen))
        cu = torch.tensor([0, cut1, cut2, total], dtype=torch.int32)
        ids = torch.randint(0, cfg.vocab_size, (1, total), generator=gen)
        pos = torch.cat([torch.arange(b - a) for a, b in zip(cu[:-1].tolist(), cu[1:].tolist())]).unsqueeze(0)
        labels = torch.roll(ids, -1, dims=1)
        labels[0, (cu[1:] - 1).long()] = -100  # the last token of a document has no target

        rfa.update_ring_flash_attn_params(cu.to(dev), None)  # once per batch, GLOBAL cu_seqlens
        logits = model(input_ids=shard(ids).to(dev), position_ids=shard(pos).to(dev)).logits
        loss_sum = torch.nn.functional.cross_entropy(logits.float().view(-1, cfg.vocab_size),
                                                     shard(labels).to(dev).reshape(-1), ignore_index=-100,
                                                     reduction="sum")
        n_targets = int((labels != -100).sum())
        (loss_sum / n_targets).backward()
        for p in model.parameters():  # weights are replicated over the CP group: sum the partial gradients
            dist.all_reduce(p.grad)
        opt.step()
        opt.zero_grad(set_to_none=True)
        dist.all_reduce(loss_sum)
        if rank == 0:
            print(f"step {step}: docs {cu.tolist()}  loss {float(loss_sum) / n_targets:.4f}", flush=True)
    if args.cuda:
        from ring_flash_attn_b200.parallel.symm import destroy_peer_contexts

        destroy_peer_contexts()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
