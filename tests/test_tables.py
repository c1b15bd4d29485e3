"""Host-side work tables consumed by the sm_90a kernels (no GPU needed): coverage and exclusivity invariants."""
import pytest
import torch

from ring_flash_attn_b200.ops import attn_cuda, plan as P
from ring_flash_attn_b200.parallel import api, symm


def _plans(scheme, world, L=600):
    if scheme == "ring":
        return [P.plan_ring(r, world, 1, L, True) for r in range(world)]
    if scheme == "zigzag":
        return [P.plan_zigzag(r, world, 2, L) for r in range(world)]
    if scheme == "stripe":
        return [P.plan_stripe(r, world, 1, L) for r in range(world)]
    cu = [0, 200, 520, 600]
    if scheme == "ring_varlen":
        return [P.plan_ring_varlen(r, world, cu, True) for r in range(world)]
    return [P.plan_zigzag_varlen(r, world, cu) for r in range(world)]


@pytest.mark.parametrize("scheme", ["ring", "zigzag", "stripe", "ring_varlen", "zigzag_varlen"])
@pytest.mark.parametrize("world", [1, 4])
def test_forward_items_cover_every_query_row_once(scheme, world):
    for plan in _plans(scheme, world):
        offsets = {s: (0 if s == plan.rank else s * plan.kv_rows) for s in range(world)}
        items, segs, covered = attn_cuda.fwd_tables_host(plan, plan.segments, offsets, {s: s for s in range(world)})
        assert covered
        seen = torch.zeros(plan.q_rows, dtype=torch.int32)
        for q_row0, q_rows, q_off, seg_begin, seg_count, *_ in items:
            assert 1 <= q_rows <= attn_cuda.Q_ITEM_ROWS and seg_count >= 1
            seen[q_row0:q_row0 + q_rows] += 1
            for kv_row0, kv_len, diag, flag in segs[seg_begin:seg_begin + seg_count]:
                assert kv_len > 0 and kv_row0 >= 0
        assert torch.all(seen == 1)


def _visible_pairs_from_plan(plan):
    total = 0
    for s in plan.segments:
        total += P.visible_area(plan.q_chunks[s.chunk].rows, s.kv_len, s.diag)
    return total


@pytest.mark.parametrize("scheme", ["ring", "zigzag", "stripe", "ring_varlen", "zigzag_varlen"])
@pytest.mark.parametrize("world", [1, 4])
def test_backward_tiles_are_exclusive_and_complete(scheme, world):
    for plan in _plans(scheme, world):
        offsets = {s: s * plan.kv_rows for s in range(world)}
        items, qsegs = attn_cuda.bwd_tables_host(plan, plan.segments, offsets)
        owner_rows = torch.zeros(world * plan.kv_rows, dtype=torch.int32)
        pairs = 0
        for kv_row0, kv_rows, seg_begin, seg_count, flag, *_ in items:
            assert 1 <= kv_rows <= attn_cuda.K_TILE_ROWS
            owner_rows[kv_row0:kv_row0 + kv_rows] += 1
            for q_row0, q_len, diag, _pad in qsegs[seg_begin:seg_begin + seg_count]:
                d = None if diag >= attn_cuda.DIAG_FULL else diag
                pairs += P.visible_area(q_len, kv_rows, d)
        assert int(owner_rows.max()) <= 1, "a key row has two writers in one launch"
        # every (query, key) pair of the plan is visited exactly once by the backward tiles
        assert pairs == _visible_pairs_from_plan(plan)


@pytest.mark.parametrize("scheme", ["zigzag", "ring"])
def test_fused_tables_push_and_reduce_are_consistent(scheme):
    world = 4
    plans = _plans(scheme, world, L=512)
    for r, p in enumerate(plans):
        p.peer = (lambda rr, _ps=plans: _ps[rr])

    class Ctx:
        group = None

    per = {}
    for p in plans:
        t, per_dst = symm.push_tasks(p, Ctx(), 1024, torch.device("cpu"))
        per[p.rank] = per_dst
        assert per_dst[p.rank] == 0
        for src_row, dst_off, packed, which in t.tolist():
            rows, dst = packed & 0xFFFFFFFF, packed >> 32
            assert 0 < rows and 0 <= dst < world and dst != p.rank and which in (0, 1)
            assert dst_off % 16 == 0
    for p in plans:
        offsets = {s: (0 if s == p.rank else s * p.kv_rows) for s in range(world)}
        flags = {s: s for s in range(world) if s != p.rank}
        _items, segs, _c = attn_cuda.fwd_tables_host(p, p.segments, offsets, flags)
        for s in {g[3] for g in segs if g[3] >= 0}:
            assert per[s][p.rank] > 0, f"rank {p.rank} waits for {s} but {s} pushes nothing to it"
        items, qsegs, per_owner = attn_cuda.bwd_tables_fused(p, offsets, torch.device("cpu"), flags)
        tasks = symm.reduce_tasks(p, Ctx(), torch.device("cpu")).tolist()
        covered = sorted((row0, row0 + rows) for row0, rows, _m, _p in tasks)
        assert covered[0][0] == 0 and covered[-1][1] == p.kv_rows
        assert all(a[1] == b[0] for a, b in zip(covered[:-1], covered[1:])), "reduce tasks must tile the shard"
        for row0, rows, mask, _p in tasks:
            for s in range(world):
                contributes = any(lo <= row0 and row0 + rows <= hi for lo, hi in symm._ranges(plans[s], p.rank))
                assert bool((mask >> s) & 1) == contributes
        assert sum(per_owner) == items.shape[0]


def test_llama3_needs_are_exchanged_not_derived():
    """Two global packings can give a rank the same local description while its peers' needs differ: llama3 plans
    therefore carry no ``peer`` function and the fused path gathers every rank's needs table on the device at each
    launch (parallel/symm.py:needs_gathered).  The local table is exactly the row ranges the plan reads."""
    from ring_flash_attn_b200.parallel import ops

    world, T = 8, 64
    a = torch.tensor([0, 8 * T], dtype=torch.int32)
    b = torch.tensor([0, 5 * T, 8 * T], dtype=torch.int32)
    pa = api.llama3_flash_attn_prepare_cu_seqlens(a, True, 0, world)
    pb = api.llama3_flash_attn_prepare_cu_seqlens(b, True, 0, world)
    assert pa[0].tolist() == pb[0].tolist() and pa[1].tolist() == pb[1].tolist()  # identical for rank 0
    plans = {}
    for name, cu in (("a", a), ("b", b)):
        cq, ck, _mq, _mk, ks = api.llama3_flash_attn_prepare_cu_seqlens(cu, True, 6, world)
        plans[name] = ops.llama3_plan(6, world, T, tuple(cq.tolist()), tuple(ck.tolist()), int(ks.start), True)
    for p in plans.values():
        assert symm.is_dynamic(p) and symm.dynamic_ok(p) and not hasattr(p, "peer")
    assert symm._ranges(plans["a"], 0) and not symm._ranges(plans["b"], 0)  # rank 6 needs rank 0's keys only in a

    class Ctx:
        group = None

    tasks = symm.reduce_tasks(plans["a"], Ctx(), torch.device("cpu")).tolist()
    assert tasks[0][0] == 0 and sum(t[1] for t in tasks) == T  # fixed row blocks; masks are computed on the device


# ----------------------------------------------------------------------------------------------
# sliding window: replay the kernels' index arithmetic on the host tables and compare with the plan
# ----------------------------------------------------------------------------------------------

def _plan_visibility(plan, world):
    """(q_rows, world * kv_rows) 0/1 matrix straight from the plan's segment semantics."""
    vis = torch.zeros(plan.q_rows, world * plan.kv_rows, dtype=torch.int32)
    for s in plan.segments:
        ch = plan.q_chunks[s.chunk]
        i = torch.arange(ch.rows).unsqueeze(1)
        j = torch.arange(s.kv_len).unsqueeze(0)
        m = torch.ones(ch.rows, s.kv_len, dtype=torch.bool)
        if s.diag is not None:
            m &= j <= i + s.diag
        if s.lo is not None:
            m &= j >= i + s.lo
        c0 = s.src * plan.kv_rows + s.kv_row0
        vis[ch.row0:ch.row0 + ch.rows, c0:c0 + s.kv_len] += m.int()
    return vis


def _replay_forward(items, segs, seg_lo, q_rows, kv_cols):
    """attn_fwd_sm90.cu: seg_geom / wg_active / wg_needs_mask / wg_needs_lower_mask / the column limits, per 64-row
    compute warpgroup of a work item."""
    T, W = 128, 64  # keys per K/V tile, query rows per warpgroup
    vis = torch.zeros(q_rows, kv_cols, dtype=torch.int32)
    for q_row0, n_rows, q_off, seg_begin, seg_count, *_ in items:
        for si in range(seg_begin, seg_begin + seg_count):
            kv_row0, kv_len, diag, _flag = segs[si]
            lo = seg_lo[si]
            last_row = q_off + n_rows - 1
            reach = min(max(last_row + diag + 1, 0), kv_len)
            n_tiles = (reach + T - 1) // T
            for w in range((n_rows + W - 1) // W):
                n_w = min(n_rows - w * W, W)
                first_row = q_off + w * W
                for jj in range(n_tiles):
                    if not jj * T <= first_row + n_w - 1 + diag:  # wg_active
                        continue
                    masked = (jj + 1) * T > kv_len or jj * T + T - 1 > first_row + diag  # wg_needs_mask
                    masked = masked or (first_row + W - 1 + lo > jj * T)  # wg_needs_lower_mask
                    for r in range(n_w):
                        chunk_row = first_row + r
                        c_lo, c_hi = 0, T - 1
                        if masked:
                            c_hi = max(-1, min(T - 1, min(chunk_row + diag, kv_len - 1) - jj * T))
                            c_lo = max(0, min(T, chunk_row + lo - jj * T))
                        if c_hi >= c_lo:
                            a = kv_row0 + jj * T
                            vis[q_row0 + w * W + r, a + c_lo:a + c_hi + 1] += 1
    return vis


def _replay_backward(items, qsegs, q_rows, kv_cols):
    """attn_bwd_sm90.cu: q_geom, the lse=+inf rows behind q_len, q_lo / q_hi per key."""
    TQ = 64
    vis = torch.zeros(q_rows, kv_cols, dtype=torch.int32)
    owner = torch.zeros(kv_cols, dtype=torch.int32)
    for kv_row0, kv_rows, seg_begin, seg_count, *_ in items:
        owner[kv_row0:kv_row0 + kv_rows] += 1
        for q_row0, q_len, diag, lo in qsegs[seg_begin:seg_begin + seg_count]:
            first = 0 if diag >= 0 else -diag
            t_end = (q_len + TQ - 1) // TQ
            t_begin = min(first // TQ, t_end)
            for ti in range(t_begin, t_end):
                for key in range(kv_rows):
                    q_lo = max(0, min(TQ, key - diag - ti * TQ))
                    last_q = key - lo - ti * TQ
                    q_hi = 0 if last_q < 0 else (TQ if last_q >= TQ else last_q + 1)
                    q_hi = min(q_hi, q_len - ti * TQ)  # rows behind q_len get lse = +inf from the stats warp
                    if q_hi > q_lo:
                        vis[q_row0 + ti * TQ + q_lo:q_row0 + ti * TQ + q_hi, kv_row0 + key] += 1
    return vis, owner


def _window_plans(scheme, world, window):
    L = 600
    if scheme == "zigzag_llama3":
        cu = [0, 100, 101, (L * world * 13) // 24, L * world]
        return [P.plan_zigzag_llama3(r, world, cu, True, window) for r in range(world)]
    if scheme == "ring":
        return [P.plan_ring(r, world, 1, L, window[1] == 0, window) for r in range(world)]
    if scheme == "zigzag":
        return [P.plan_zigzag(r, world, 2, L, window) for r in range(world)]
    if scheme == "stripe":
        return [P.plan_stripe(r, world, 1, L, window) for r in range(world)]
    cu = [0, 200, 520, 600]
    if scheme == "ring_varlen":
        return [P.plan_ring_varlen(r, world, cu, window[1] == 0, window) for r in range(world)]
    return [P.plan_zigzag_varlen(r, world, cu, window) for r in range(world)]


@pytest.mark.parametrize("scheme", ["ring", "zigzag", "stripe", "ring_varlen", "zigzag_varlen", "zigzag_llama3"])
@pytest.mark.parametrize("world", [1, 4])
@pytest.mark.parametrize("window", [(37, 0), (300, 0), (1000, 0)])
def test_window_tables_replay_matches_plan(scheme, world, window):
    for plan in _window_plans(scheme, world, window):
        want = _plan_visibility(plan, world)
        assert int(want.max()) <= 1
        got_f = torch.zeros_like(want)
        got_b = torch.zeros_like(want)
        for src, segs in plan.by_src().items():
            c0 = src * plan.kv_rows
            if attn_cuda.has_window(segs):
                items, seg_rows, seg_lo, covered = attn_cuda.fwd_tables_window_host(plan, segs, {src: 0})
                b_items, b_qsegs = attn_cuda.bwd_tables_window_host(plan, segs, {src: 0})
            else:
                items, seg_rows, covered = attn_cuda.fwd_tables_host(plan, segs, {src: 0})
                seg_lo = [attn_cuda.LO_NONE] * len(seg_rows)
                b_items, b_qsegs = attn_cuda.bwd_tables_host(plan, segs, {src: 0})
                b_qsegs = [[a, b, c, attn_cuda.LO_NONE] for a, b, c, _ in b_qsegs]
            got_f[:, c0:c0 + plan.kv_rows] += _replay_forward(items, seg_rows, seg_lo, plan.q_rows, plan.kv_rows)
            vb, owner = _replay_backward(b_items, b_qsegs, plan.q_rows, plan.kv_rows)
            assert int(owner.max()) <= 1
            got_b[:, c0:c0 + plan.kv_rows] += vb
            # rows the forward items do not touch must be exactly the rows that see nothing from this source
            touched = torch.zeros(plan.q_rows, dtype=torch.bool)
            for q_row0, n_rows, *_ in items:
                touched[q_row0:q_row0 + n_rows] = True
            sees = want[:, c0:c0 + plan.kv_rows].sum(1) > 0
            assert not bool((sees & ~touched).any())
            assert covered == bool(touched.all())
        assert torch.equal(got_f, want), "forward tables + kernel masks disagree with the plan"
        assert torch.equal(got_b, want), "backward tables + kernel masks disagree with the plan"


def test_window_two_sided_noncausal_replay():
    for window in [(20, 9), (-1, 50), (130, -1)]:
        for plan in [P.plan_ring(r, 4, 1, 300, False, window) for r in range(4)]:
            want = _plan_visibility(plan, 4)
            got_f, got_b = torch.zeros_like(want), torch.zeros_like(want)
            for src, segs in plan.by_src().items():
                c0 = src * plan.kv_rows
                if attn_cuda.has_window(segs):
                    items, seg_rows, seg_lo, _ = attn_cuda.fwd_tables_window_host(plan, segs, {src: 0})
                    b_items, b_qsegs = attn_cuda.bwd_tables_window_host(plan, segs, {src: 0})
                else:
                    items, seg_rows, _ = attn_cuda.fwd_tables_host(plan, segs, {src: 0})
                    seg_lo = [attn_cuda.LO_NONE] * len(seg_rows)
                    b_items, b_qsegs = attn_cuda.bwd_tables_host(plan, segs, {src: 0})
                    b_qsegs = [[a, b, c, attn_cuda.LO_NONE] for a, b, c, _ in b_qsegs]
                got_f[:, c0:c0 + plan.kv_rows] += _replay_forward(items, seg_rows, seg_lo, plan.q_rows, plan.kv_rows)
                got_b[:, c0:c0 + plan.kv_rows] += _replay_backward(b_items, b_qsegs, plan.q_rows, plan.kv_rows)[0]
            assert torch.equal(got_f, want) and torch.equal(got_b, want)


@pytest.mark.parametrize("scheme", ["zigzag", "ring", "stripe", "zigzag_varlen"])
@pytest.mark.parametrize("window", [(90, 0), (700, 0)])
def test_window_fused_tables(scheme, window):
    """Fused multi-GPU layout of the windowed tables: one launch over all sources (local tensor for flag -1,
    staging slot of the source otherwise), backward tiles for every key row a peer will reduce, per-owner counts."""
    world = 4
    plans = _window_plans(scheme, world, window)
    for p in plans:
        rows = p.kv_rows
        offsets = {s: (0 if s == p.rank else s * rows) for s in range(world)}
        flags = {s: s for s in range(world) if s != p.rank}
        want = _plan_visibility(p, world)
        items, seg_rows, seg_lo, _cov = attn_cuda.fwd_tables_window_host(p, p.segments, offsets, flags)
        glob = []
        for kv_row0, kv_len, d, flag in seg_rows:
            src = p.rank if flag < 0 else flag
            assert offsets[src] <= kv_row0 and kv_row0 + kv_len <= offsets[src] + rows
            glob.append([src * rows + kv_row0 - offsets[src], kv_len, d, flag])
        assert torch.equal(_replay_forward(items, glob, seg_lo, p.q_rows, world * rows), want)

        b_items, b_qsegs, per_owner = attn_cuda.bwd_tables_window_host(p, p.segments, offsets, flags, fused=True)
        assert sum(per_owner) == len(b_items)
        g_items = []
        for kv_row0, kv_rows, b, c, flag, owner, out_row0, z in b_items:
            assert (flag < 0) == (owner == p.rank) and kv_row0 - offsets[owner] == out_row0
            g_items.append([owner * rows + out_row0, kv_rows, b, c, flag, owner, out_row0, z])
        vb, owner_rows = _replay_backward(g_items, b_qsegs, p.q_rows, world * rows)
        assert torch.equal(vb, want) and int(owner_rows.max()) <= 1
        # every key row that an owner's reduction will read from this rank's slot is written by exactly one tile
        expect = torch.zeros(world * rows, dtype=torch.int32)
        for s in range(world):
            for lo, hi in symm._ranges(p, s):
                expect[s * rows + lo:s * rows + hi] = 1
        assert torch.equal(owner_rows, expect)
