"""The code paths that normally need an H100 - work tables, launch dispatch (plain / sliding window / fp8), per-source
ring steps, autograd bridge - run on CPU against the dense oracle, with the extension replaced by
``tests/fake_ext.py`` (a torch implementation of each launch's contract, driven by the same tables)."""
import os

import pytest
import torch
import torch.distributed as dist

import ring_flash_attn_b200 as rfa
from ring_flash_attn_b200.ops.dense import attention_oracle, varlen_attention_oracle
from ring_flash_attn_b200.parallel import layouts
from dist_utils import run_distributed

BF16 = dict(atol=3e-2, rtol=3e-2)


def _grad_close(got, want):
    assert (got.float() - want).abs().max().item() < 5e-2 * want.abs().max().item() + 2e-2


def _case(rank, world, window, expect):
    import fake_ext

    os.environ["RFA_B200_DISABLE_P2P"] = "1"  # no CUDA IPC here: per-source launches around the ring transport
    fake = fake_ext.install()
    torch.manual_seed(0)
    S, H, HK, d = 320 * world, 4, 2, 128
    q = torch.randn(1, S, H, d).to(torch.bfloat16)
    kv = torch.randn(1, S, 2, HK, d).to(torch.bfloat16)
    dout = torch.randn(1, S, H, d).to(torch.bfloat16)
    if world > 1:
        for t in (q, kv, dout):
            dist.broadcast(t, src=0)
    rq, rkv = q.float().requires_grad_(True), kv.float().requires_grad_(True)
    for scheme, prefix in (("ring", "ring"), ("zigzag", "zigzag_ring"), ("stripe", "stripe")):
        rq.grad = rkv.grad = None
        ref, ref_lse = attention_oracle(rq, rkv[:, :, 0], rkv[:, :, 1], True, window_size=window)
        ref.backward(dout.float())
        shard = getattr(layouts, f"shard_{scheme}")
        lq = shard(q, rank, world).detach().requires_grad_(True)
        lkv = shard(kv, rank, world).detach().requires_grad_(True)
        fake.calls.clear()
        out, lse, _ = getattr(rfa, f"{prefix}_flash_attn_kvpacked_func")(lq, lkv, causal=True, window_size=window,
                                                                      return_attn_probs=True)
        out.backward(shard(dout, rank, world))
        assert set(expect) <= set(fake.calls), (scheme, fake.calls)
        torch.testing.assert_close(out.float(), shard(ref, rank, world), **BF16)
        torch.testing.assert_close(lse, shard(ref_lse, rank, world, dim=2), atol=2e-3, rtol=2e-3)
        _grad_close(lq.grad, shard(rq.grad, rank, world))
        _grad_close(lkv.grad, shard(rkv.grad, rank, world))
    # packed documents (varlen) through the same launches
    cu = [0, 96 * world, 224 * world, S]
    cu_t = torch.tensor(cu, dtype=torch.int32)
    q2, k2, v2 = q[0], kv[0, :, 0], kv[0, :, 1]
    r2 = [t.float().requires_grad_(True) for t in (q2, k2, v2)]
    ref, _ = varlen_attention_oracle(*r2, cu_t, True, window_size=window)
    ref.backward(dout[0].float())
    sh = lambda x: layouts.shard_zigzag_varlen(x, cu, rank, world)  # noqa: E731
    l2 = [sh(t).detach().requires_grad_(True) for t in (q2, k2, v2)]
    local_cu = cu_t // world
    out = rfa.zigzag_ring_flash_attn_varlen_func(*l2, local_cu, int((local_cu[1:] - local_cu[:-1]).max()), causal=True,
                                                 window_size=window)
    out.backward(sh(dout[0]))
    torch.testing.assert_close(out.float(), sh(ref), **BF16)
    for g, r in zip(l2, r2):
        _grad_close(g.grad, sh(r.grad))
    # flat zigzag layout, documents of arbitrary lengths
    gcu = torch.tensor([0, 77, 78, S // 2 + 9, S], dtype=torch.int32)
    r3 = [t.float().requires_grad_(True) for t in (q2, k2, v2)]
    ref, _ = varlen_attention_oracle(*r3, gcu, True, window_size=window)
    ref.backward(dout[0].float())
    sh3 = lambda x: layouts.shard_zigzag_llama3(x, rank, world)  # noqa: E731
    l3 = [sh3(t).detach().requires_grad_(True) for t in (q2, k2, v2)]
    out = rfa.zigzag_llama3_flash_attn_varlen_func(*l3, gcu, causal=True, window_size=window)
    out.backward(sh3(dout[0]))
    torch.testing.assert_close(out.float(), sh3(ref), **BF16)
    for g, r in zip(l3, r3):
        _grad_close(g.grad, sh3(r.grad))


@pytest.mark.parametrize("world", [1, 2])
def test_plain_launch_path(world):
    # the single-GPU path also launches the delta kernel; the ring transport computes delta with torch
    run_distributed(_case, world, (-1, -1), ("attn_fwd", "attn_bwd") + (("attn_bwd_delta",) if world == 1 else ()))


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("window", [(70, 0), (250, 0)])
def test_window_launch_path(world, window, monkeypatch):
    monkeypatch.setenv("RFA_B200_WINDOW_KERNEL", "1")
    run_distributed(_case, world, window, ("attn_fwd_window", "attn_bwd_window"))


def _fp8_case(rank, world):
    import fake_ext
    from ring_flash_attn_b200.utils import fp8

    os.environ["RFA_B200_DISABLE_P2P"] = "1"
    os.environ["RFA_B200_FP8_KERNEL"] = "1"
    fake = fake_ext.install()
    torch.manual_seed(0)
    S, H, HK, d = 256 * world, 4, 2, 128
    q = torch.randn(1, S, H, d)
    kv = torch.randn(1, S, 2, HK, d)
    if world > 1:
        dist.broadcast(q, src=0)
        dist.broadcast(kv, src=0)
    q8, dq = fp8.quantize_blockwise(q, [0, 0, 1, 0])  # per head
    kv8, dkv = fp8.quantize_blockwise(kv, [0, 0, 1, 1, 0])
    qd, kvd = fp8.dequantize(q8, dq, torch.float32), fp8.dequantize(kv8, dkv, torch.float32)
    ref, ref_lse = attention_oracle(qd, kvd[:, :, 0], kvd[:, :, 1], True)
    for scheme, fn in (("zigzag", rfa.zigzag_ring_flash_attn_kvpacked_func), ("ring", rfa.ring_flash_attn_kvpacked_func)):
        shard = getattr(layouts, f"shard_{scheme}")
        fake.calls.clear()
        out, lse, _ = fn(shard(q8.view(torch.uint8), rank, world).view(torch.float8_e4m3fn),
                         shard(kv8.view(torch.uint8), rank, world).view(torch.float8_e4m3fn), causal=True,
                         descale=(dq, dkv), return_attn_probs=True)
        assert fake.calls and set(fake.calls) == {"attn_fwd_fp8"}, fake.calls
        assert out.dtype == torch.bfloat16
        torch.testing.assert_close(out.float(), shard(ref, rank, world), **BF16)
        torch.testing.assert_close(lse, shard(ref_lse, rank, world, dim=2), atol=2e-3, rtol=2e-3)
    # block-scaled: one descale per 128 LOCAL tokens and head (BASELINE.json config 5).  The shard is quantised
    # locally (what a training step does with its activations), so every rank has different K / V tables and the
    # transports have to bring the source's table along with its rows.
    for scheme, fn in (("ring", rfa.ring_flash_attn_kvpacked_func), ("stripe", rfa.stripe_flash_attn_kvpacked_func)):
        shard = getattr(layouts, f"shard_{scheme}")
        lq8, ldq = fp8.quantize_blockwise(shard(q, rank, world), [1, 128, 1, 0])
        lkv8, ldkv = fp8.quantize_blockwise(shard(kv, rank, world), [1, 128, 1, 1, 0])
        parts_q = [torch.empty_like(lq8.view(torch.uint8)) for _ in range(world)]
        deq_q, deq_kv = fp8.dequantize(lq8, ldq, torch.float32), fp8.dequantize(lkv8, ldkv, torch.float32)
        if world > 1:
            gq = [torch.empty_like(deq_q) for _ in range(world)]
            gkv = [torch.empty_like(deq_kv) for _ in range(world)]
            dist.all_gather(gq, deq_q)
            dist.all_gather(gkv, deq_kv)
        else:
            gq, gkv = [deq_q], [deq_kv]
        fq, fkv = layouts.unshard(scheme, gq), layouts.unshard(scheme, gkv)
        ref_b, ref_lse_b = attention_oracle(fq, fkv[:, :, 0], fkv[:, :, 1], True)
        fake.calls.clear()
        out, lse, _ = fn(lq8, lkv8, causal=True, descale=(ldq, ldkv), return_attn_probs=True)
        assert set(fake.calls) == {"attn_fwd_fp8"}, fake.calls
        torch.testing.assert_close(out.float(), shard(ref_b, rank, world), **BF16)
        torch.testing.assert_close(lse, shard(ref_lse_b, rank, world, dim=2), atol=2e-3, rtol=2e-3)
        del parts_q
    # llama3 entry point: the all-gather transport slices the descales per head group
    cu = torch.tensor([0, S // 2 + 3, S], dtype=torch.int32)
    refv, _ = varlen_attention_oracle(qd[0], kvd[0, :, 0], kvd[0, :, 1], cu, True)
    cq, ck, mq, mk, ks = rfa.llama3_flash_attn_prepare_cu_seqlens(cu, True, rank, world)
    sh = lambda x: layouts.shard_llama3(x, rank, world)  # noqa: E731
    fake.calls.clear()
    out = rfa.llama3_flash_attn_varlen_kvpacked_func(
        sh(q8[0].view(torch.uint8)).view(torch.float8_e4m3fn), sh(kv8[0].view(torch.uint8)).view(torch.float8_e4m3fn),
        cq, ck, mq, mk, heads_k_stride=1, local_k_slice=ks, causal=True, descale=(dq[0], dkv[0]))
    assert set(fake.calls) == {"attn_fwd_fp8"}
    torch.testing.assert_close(out.float(), sh(refv), **BF16)


@pytest.mark.parametrize("world", [1, 2])
def test_fp8_launch_path(world):
    run_distributed(_fp8_case, world)


def test_ordered_dq_groups_are_conflict_free():
    """deterministic=True: key tiles of one launch group never reach the same query rows; every tile is launched once."""
    from ring_flash_attn_b200.ops import attn_cuda
    from ring_flash_attn_b200.parallel import ops as O

    def spans(it, qsegs):
        return [(r0 + max(0, -d), r0 + n) for r0, n, d, _ in qsegs[it[2]:it[2] + it[3]] if max(0, -d) < n]

    def check(plan, window=False):
        if window:
            items, qsegs = attn_cuda.bwd_tables_window_host(plan, plan.segments, {plan.rank: 0})
        else:
            items, qsegs = attn_cuda.bwd_tables_host(plan, plan.segments, {plan.rank: 0})
        ordered, bounds = attn_cuda.ordered_dq_groups(items, qsegs)
        assert sorted(map(tuple, ordered)) == sorted(map(tuple, items)) and bounds[0] == 0 and bounds[-1] == len(items)
        for a, b in zip(bounds[:-1], bounds[1:]):
            assert b > a
            taken = sorted(s for it in ordered[a:b] for s in spans(it, qsegs))
            assert all(x[1] <= y[0] for x, y in zip(taken[:-1], taken[1:])), (a, b, taken)
        return len(items), len(bounds) - 1

    n, g = check(O.batch_plan("zigzag", 0, 1, 1, 1024, True))
    assert n == 8 and g == 8  # one causal sequence: every key tile reaches the last query rows
    n, g = check(O.batch_plan("zigzag", 0, 1, 4, 512, True))
    assert n == 16 and g == 4  # four batch elements side by side
    n, g = check(O.batch_plan("ring", 0, 1, 1, 1024, True, (200, 0)), window=True)
    assert n == 8 and 2 <= g <= 3  # a 200-token window: a query row is reached by at most 3 key tiles
    n, g = check(O.varlen_plan("ring", 0, 1, (0, 100, 700, 701, 1500), True))
    assert g == 7  # the longest document (799 keys) has 7 key tiles; the other documents ride along


def _deterministic_case(rank, world):
    import fake_ext

    os.environ["RFA_B200_DISABLE_P2P"] = "1"
    fake = fake_ext.install()
    torch.manual_seed(1)
    S, H, d = 384 * world, 2, 64
    qkv = torch.randn(2, S, 3, H, d).to(torch.bfloat16)
    dout = torch.randn(2, S, H, d).to(torch.bfloat16)
    if world > 1:
        dist.broadcast(qkv, src=0)
        dist.broadcast(dout, src=0)
    local = layouts.shard_zigzag(qkv, rank, world)
    grads, launches = [], []
    for det in (False, True):
        x = local.detach().requires_grad_(True)
        fake.calls.clear()
        with pytest.warns(RuntimeWarning, match="deterministic=True") if det and not _deterministic_case.warned \
                else __import__("contextlib").nullcontext():
            out = rfa.zigzag_ring_flash_attn_qkvpacked_func(x, causal=True, deterministic=det)
            out.backward(layouts.shard_zigzag(dout, rank, world))
        _deterministic_case.warned |= det
        grads.append(x.grad.clone())
        launches.append(fake.calls.count("attn_bwd"))
    torch.testing.assert_close(grads[0].float(), grads[1].float(), atol=2e-2, rtol=2e-2)
    # world 1: 2 x 384 local rows = 3 key tiles per batch element -> 3 groups of 2 tiles instead of one launch;
    # world 2: one launch per source before, one per group and source now
    assert launches[0] == world and launches[1] > launches[0], launches
    os.environ["RFA_B200_DETERMINISTIC"] = "fast"
    try:
        x = local.detach().requires_grad_(True)
        fake.calls.clear()
        rfa.zigzag_ring_flash_attn_qkvpacked_func(x, causal=True, deterministic=True).backward(
            layouts.shard_zigzag(dout, rank, world))
        assert fake.calls.count("attn_bwd") == world
    finally:
        os.environ.pop("RFA_B200_DETERMINISTIC", None)


_deterministic_case.warned = False


@pytest.mark.parametrize("world", [1, 2])
def test_deterministic_backward_launch_groups(world):
    run_distributed(_deterministic_case, world)
