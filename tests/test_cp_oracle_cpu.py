"""CPU self-test of ``tests/cp_oracle.py`` and of the GPU files built on it (``test_gpu_cp_replay.py``,
``test_gpu_cp_accuracy.py``): the fp64 reference agrees with dense attention over the whole sequence, the
torch.distributed fallback (gloo, per-source launches of ``tests/fake_ext.py``) and a bf16 replay of the fused launch
(staging buffers and dK/dV inboxes in the model dtype) meet the precision-matched bound, and planted transport errors
- a dropped remote key tile, a stale staging slot, a merge that skips a source, an inbox slot reduced twice or not
at all - fail it, although the dropped tile passes the dense-oracle tolerance of ``test_gpu_multi.py``."""
import itertools

import pytest
import torch

import cp_oracle as CP
import test_gpu_cp_accuracy as ACC
import test_gpu_cp_replay as REP
from dist_utils import run_distributed
from fake_ext import FakeExt
from ring_flash_attn_b200.ops import attn_cuda, cuda_ext
from ring_flash_attn_b200.ops import plan as P
from ring_flash_attn_b200.ops.dense import attention_oracle, varlen_attention_oracle
from ring_flash_attn_b200.parallel import engine, layouts, symm

# what the GPU files must cover
SCHEMES = {("ring", True), ("ring", False), ("zigzag", True), ("stripe", True), ("ring_varlen", True),
           ("zigzag_varlen", True), ("llama3", True), ("zigzag_llama3", True)}
DTYPES = {torch.bfloat16, torch.float16}
HEAD_DIMS = {64, 128}


@pytest.fixture
def fake(monkeypatch):
    ext = FakeExt()
    monkeypatch.setattr(cuda_ext, "load", lambda: ext)
    monkeypatch.setattr(engine, "_use_cuda_kernels", lambda q, k=None: True)
    return ext


def _install_fake():
    ext = FakeExt()
    cuda_ext.load = lambda: ext
    engine._use_cuda_kernels = lambda q, k=None: True


# ---------------------------------------------------------------------------------------------- the fp64 reference

@pytest.mark.parametrize("scheme,causal,window", [("zigzag", True, (-1, -1)), ("stripe", True, (70, 0)),
                                                  ("ring", False, (100, 60)), ("zigzag_llama3", True, (-1, -1)),
                                                  ("llama3", True, (90, 0))])
def test_fp64_reference_is_dense_attention(scheme, causal, window):
    """Plans over the concatenated source shards give dense attention on the whole sequence (out, lse, dq, dk, dv):
    the segments' rebased ``kv_row0`` and every rank's dK / dV partials summed by owner."""
    case = CP.Case(scheme, 3, 128, 4, 2, 32, torch.float32, causal, window)
    plans = CP.build_plans(case)
    q, k, v, do = CP.make_inputs(case, 0)
    refs = CP.references(case, plans, q, k, v, do, "fused")
    if scheme in CP.BATCH:
        def unshard(xs):
            return layouts.unshard(scheme, [x.unsqueeze(0) for x in xs])

        def shard(x, r):
            return getattr(layouts, f"shard_{scheme}")(x, r, 3)[0]
        gq, gk, gv, gdo = (unshard(t).double().requires_grad_(True) for t in (q, k, v, do))
        out, lse = attention_oracle(gq, gk, gv, causal, window_size=window)
        lse = lse[0]
        shard_lse = lambda x, r: getattr(layouts, f"shard_{scheme}")(x, r, 3, dim=1)  # noqa: E731
    else:
        sh = layouts.shard_llama3 if scheme == "llama3" else layouts.shard_zigzag_llama3

        def unshard(xs):
            if scheme == "llama3":
                return torch.cat(xs)
            return layouts.unshard("zigzag", [x.unsqueeze(0) for x in xs])[0]

        def shard(x, r):
            return sh(x, r, 3)
        gq, gk, gv, gdo = (unshard(t).double().requires_grad_(True) for t in (q, k, v, do))
        out, lse = varlen_attention_oracle(gq, gk, gv, torch.tensor(CP.global_cu(case)), causal, window_size=window)
        shard_lse = lambda x, r: sh(x.transpose(0, 1), r, 3).transpose(0, 1)  # noqa: E731
    out.backward(gdo.detach())
    for r in range(3):
        ref64 = refs[r][0]
        want = dict(out=shard(out.detach(), r), lse=shard_lse(lse.detach(), r), dq=shard(gq.grad, r),
                    dk=shard(gk.grad, r), dv=shard(gv.grad, r))
        for key, w in want.items():
            # (the dense oracle computes in fp32)
            torch.testing.assert_close(ref64[key].double(), w.double(), atol=2e-5, rtol=1e-5)


# ---------------------------------------------------------------------------------------------- fallback on gloo

def _fallback_worker(rank, world, dtype):
    torch.set_num_threads(1)  # small tensors; the ranks share the machine's cores
    _install_fake()
    calls = ACC.call_sequence(world, dtype, base_rows=128 // world, head_dims=[64])
    ACC._sequence_worker(rank, world, "fallback", dtype, calls)


@pytest.mark.parametrize("world", [2, 4])
def test_fallback_meets_reference(world):
    """The API's torch.distributed transports (ring / all-gather) around the kernels' contract, through the same call
    sequence as the GPU test, within the fallback reference's bound."""
    run_distributed(_fallback_worker, world, torch.bfloat16 if world == 2 else torch.float16)


# ---------------------------------------------------------------------------------------------- fused launch replay

class _Ctx:
    group = None


def fused_replay(case, plans, q, k, v, dout, stale=None, inbox_fault=None):
    """The fused launch of every rank in one process, in the model dtype: push tables fill staging buffers, forward
    and backward tables run on :class:`FakeExt` over [local rows | staging rows], dK/dV tiles are stored into the
    owners' inboxes in the model dtype and the reduce tables sum the slots in fp32.

    Planted errors: ``stale`` = (k, v) of a previous call, left in rank 0's staging slot of source 1;
    ``inbox_fault`` = ``"twice"`` / ``"none"``: rank 0 reduces the slot of source 1 twice / not at all."""
    ext = FakeExt()
    W, L, hq, hkv, d, dt = case.world, case.rows, case.hq, case.hkv, case.d, case.dtype
    row_bytes = hkv * d * torch.empty((), dtype=dt).element_size()
    region = W * L * row_bytes
    stage = [torch.full((2, W * L, hkv, d), float("nan"), dtype=dt) for _ in range(W)]
    dynamic = symm.is_dynamic(plans[0])
    needs_all = torch.stack([symm.local_needs_table(p) for p in plans]).tolist() if dynamic else None
    for me, p in enumerate(plans):
        if dynamic:
            chunk = symm.push_chunk_rows(row_bytes)
            chunks = -(-L // chunk)
            tasks = []
            for ti in range((W - 1) * 2 * symm.NEED_RANGES * chunks):
                r0, off, rows, dst, which = symm.dynamic_push_task(needs_all, me, W, ti, chunk, chunks, L, row_bytes,
                                                                   region)
                if rows:
                    tasks.append([r0, off, rows | (dst << 32), which])
        else:
            tasks = symm.push_tasks(p, _Ctx(), row_bytes, torch.device("cpu"))[0].tolist()
        for src_row, dst_off, packed, which in tasks:
            rows, dst = packed & 0xFFFFFFFF, packed >> 32
            dst_row = (dst_off - which * region) // row_bytes
            stage[dst][which, dst_row:dst_row + rows] = (k, v)[which][me][src_row:src_row + rows]
    if stale is not None:
        stage[0][0, L:2 * L], stage[0][1, L:2 * L] = stale[0][1], stale[1][1]
    got, inbox = {}, [torch.full((W, 2, L, hkv, d), float("nan"), dtype=dt) for _ in range(W)]
    for me, p in enumerate(plans):
        offsets = {s: (0 if s == me else s * L) for s in range(W)}
        flags = {s: s for s in range(W) if s != me}
        kk, vv = torch.cat([k[me], stage[me][0]]), torch.cat([v[me], stage[me][1]])
        window = attn_cuda.has_window(p.segments)
        if window:
            items, segs, seg_lo, _ = attn_cuda.fwd_tables_window_host(p, p.segments, offsets, flags)
        else:
            (items, segs, _), seg_lo = attn_cuda.fwd_tables_host(p, p.segments, offsets, flags), None
        segs = [[r0 if f < 0 else L + r0, n, dg, f] for r0, n, dg, f in segs]
        out = torch.zeros((L, hq, d), dtype=dt)
        lse = torch.full((hq, L), float("-inf"))
        ext._fwd(q[me], kk, vv, torch.tensor(items), torch.tensor(segs), seg_lo, out, lse, case.scale)
        assert not torch.isnan(out).any(), "a forward segment read staging rows nobody pushed"
        if window:
            items, qsegs, _ = attn_cuda.bwd_tables_window_host(p, p.segments, offsets, flags, fused=True)
        else:
            it_t, qs_t, _ = attn_cuda.bwd_tables_fused(p, offsets, torch.device("cpu"), flags)
            items, qsegs = it_t.tolist(), qs_t.tolist()
        delta = (out.float() * dout[me].float()).sum(-1).transpose(0, 1).contiguous()
        dq = torch.zeros((L, hq, d))
        for kv_row0, kv_rows, b, c, flag, owner, out_row0, _z in items:
            src_row = kv_row0 if flag < 0 else L + kv_row0
            tile = torch.zeros((2, L + W * L, hkv, d))
            if c:
                one = torch.tensor([[src_row, kv_rows, 0, c, flag, owner, out_row0, 0]])
                ext._bwd(q[me], dout[me], kk, vv, dq, one,
                         torch.tensor(qsegs[b:b + c]), lse, delta, tile[0], tile[1], case.scale, window)
            inbox[owner][me, :, out_row0:out_row0 + kv_rows] = tile[:, src_row:src_row + kv_rows].to(dt)
        got[me] = dict(out=out, lse=lse, dq=dq.to(dt))
    for me, p in enumerate(plans):
        tasks = symm.reduce_tasks(p, _Ctx(), torch.device("cpu")).tolist()
        if dynamic:
            tasks = [[r, 1, symm.dynamic_row_mask(needs_all, me, W, r), 0]
                     for row0, rows, _m, _p in tasks for r in range(row0, row0 + rows)]
        acc = torch.zeros((2, L, hkv, d))
        for row0, rows, mask, _pad in tasks:
            for s in range(W):
                if not (mask >> s) & 1:
                    continue
                times = 1
                if me == 0 and s == 1 and inbox_fault is not None:
                    times = 2 if inbox_fault == "twice" else 0
                for _ in range(times):
                    acc[:, row0:row0 + rows] += inbox[me][s, :, row0:row0 + rows].float()
        assert not torch.isnan(acc).any(), "the reduction read inbox rows no peer wrote"
        got[me]["dk"], got[me]["dv"] = acc[0].to(dt), acc[1].to(dt)
    return got


FUSED_CASES = [CP.Case("zigzag", 2, 256, 4, 2, 64, torch.bfloat16),
               CP.Case("stripe", 4, 128, 4, 1, 64, torch.float16, window=(90, 0)),
               CP.Case("ring", 3, 128, 2, 2, 128, torch.bfloat16, causal=False, batch=2),
               CP.Case("zigzag_varlen", 2, 192, 4, 2, 64, torch.float16, regime="peaked"),
               CP.Case("llama3", 4, 96, 4, 2, 64, torch.bfloat16, window=(100, 0)),
               CP.Case("zigzag_llama3", 3, 128, 4, 4, 64, torch.bfloat16)]


def _check_all(case, got, refs, report):
    for r in range(case.world):
        CP.check(f"{case.name()} rank {r}", got[r], *refs[r], report=report)


@pytest.mark.parametrize("case", FUSED_CASES, ids=lambda c: c.name())
def test_fused_replay_meets_reference(case):
    plans = CP.build_plans(case)
    q, k, v, do = CP.make_inputs(case, 3)
    got = fused_replay(case, plans, q, k, v, do)
    if case.regime not in CP.BACKWARD_REGIMES:
        got = {r: dict(out=g["out"], lse=g["lse"]) for r, g in got.items()}
    _check_all(case, got, CP.references(case, plans, q, k, v, do, "fused"), "cpu fused")


@pytest.mark.parametrize("fault", ["stale_staging", "inbox_twice", "inbox_none"])
def test_fused_mutants_fail(fault):
    case = CP.Case("zigzag", 2, 256, 4, 2, 64, torch.bfloat16)
    plans = CP.build_plans(case)
    prev = CP.make_inputs(case, 4)
    q, k, v, do = CP.make_inputs(case, 5)
    refs = CP.references(case, plans, q, k, v, do, "fused")
    kw = dict(stale=(prev[1], prev[2])) if fault == "stale_staging" else dict(inbox_fault=fault[len("inbox_"):])
    with pytest.raises(AssertionError):
        _check_all(case, fused_replay(case, plans, q, k, v, do, **kw), refs, "cpu mutant")


# ---------------------------------------------------------------------------------------------- fallback mutants

def _drop_last_remote_tile(victim: int, src: int):
    """``engine.step_forward`` that leaves the last 128 keys of ``src``'s shard out of rank ``victim``'s forward."""
    def step(plan, segs, *args):
        if plan.rank == victim and segs and segs[0].src == src:
            segs = [P.Segment(s.chunk, s.src, s.kv_row0, plan.kv_rows - 128 - s.kv_row0, s.diag, s.lo)
                    if s.kv_row0 + s.kv_len == plan.kv_rows and s.diag is None else s for s in segs]
            # a fresh plan object: launch tables are cached on the (lru-cached) plan
            plan = P.CPPlan(plan.world, plan.rank, plan.q_rows, plan.kv_rows, plan.q_chunks, segs)
        return engine.step_forward(plan, segs, *args)
    return step


def _skip_source(victim: int, src: int):
    def step(plan, segs, q, k, v, scale, out, lse):
        if plan.rank == victim and segs and segs[0].src == src:
            return out, lse
        return engine.step_forward(plan, segs, q, k, v, scale, out, lse)
    return step


def test_dropped_remote_tile_fails_bound_but_passes_old_tolerance(fake):
    """zigzag, world 2, 512 rows per rank, 4 heads of 128, bf16: rank 0's forward without the last 128-key tile of
    rank 1's shard.  The dense-oracle tolerance of ``test_gpu_multi.py`` accepts it; the precision-matched bound does
    not."""
    from test_gpu_multi import _close

    case = CP.Case("zigzag", 2, 512, 4, 4, 128, torch.bfloat16)
    plans = CP.build_plans(case)
    q, k, v, do = CP.make_inputs(case, 0)
    refs = CP.references(case, plans, q, k, v, do, "ring", backward=False)
    got = CP.replay(case, plans, q, k, v, do, backward=False, step_forward=_drop_last_remote_tile(0, 1))
    _close(got[0]["out"], refs[0][0]["out"], "out")  # the old tolerance lets the missing tile through
    with pytest.raises(AssertionError, match="out"):
        CP.check("dropped tile", got[0], *refs[0], report="cpu mutant")
    clean = CP.replay(case, plans, q, k, v, do, backward=False)
    CP.check("clean", clean[0], *refs[0], report="cpu replay")


@pytest.mark.parametrize("case", [CP.Case("ring", 4, 128, 4, 2, 64, torch.bfloat16, causal=False),
                                  CP.Case("llama3", 3, 128, 4, 2, 64, torch.float16)], ids=lambda c: c.scheme)
def test_merge_skipping_a_source_fails(fake, case):
    plans = CP.build_plans(case)
    q, k, v, do = CP.make_inputs(case, 1)
    refs = CP.references(case, plans, q, k, v, do, CP.FALLBACK_ORDER[case.scheme], backward=False)
    victim, src = case.world - 1, 0
    _check_all(case, CP.replay(case, plans, q, k, v, do, backward=False), refs, "cpu replay")
    got = CP.replay(case, plans, q, k, v, do, backward=False, step_forward=_skip_source(victim, src))
    with pytest.raises(AssertionError):
        CP.check("skipped source", got[victim], *refs[victim], report="cpu mutant")


@pytest.mark.parametrize("scheme,causal", sorted(SCHEMES))
def test_replay_meets_reference(fake, scheme, causal):
    """The GPU replay's host side (plans, per-source steps, fp32 merges and sums) on the kernels' contract."""
    case = CP.Case(scheme, 4 if scheme == "llama3" else 3, 96, 4, 2, 64, torch.bfloat16, causal,
                   window=(50, 0) if scheme == "stripe" else (-1, -1),
                   regime="peaked" if scheme == "zigzag" else "randn")
    plans = CP.build_plans(case)
    q, k, v, do = CP.make_inputs(case, 2)
    train = case.regime in CP.BACKWARD_REGIMES
    _check_all(case, CP.replay(case, plans, q, k, v, do, backward=train),
               CP.references(case, plans, q, k, v, do, CP.FALLBACK_ORDER[scheme], backward=train), "cpu replay")


# ---------------------------------------------------------------------------------------------- coverage

def _params(fn):
    out = {}
    for mark in getattr(fn, "pytestmark", []):
        if mark.name == "parametrize":
            names = [n.strip() for n in mark.args[0].split(",")]
            vals = list(mark.args[1])
            if len(names) == 1:
                out[names[0]] = vals
            else:
                out[tuple(names)] = vals
    return out


def _combos(cases):
    return {(c.scheme, c.causal, c.dtype, c.d, c.window != (-1, -1)) for c in cases}


def test_gpu_files_cover_every_combination():
    want = {(s, c, dt, d, w) for (s, c), dt, d, w in itertools.product(SCHEMES, DTYPES, HEAD_DIMS, [False, True])}
    # multi-GPU: every combination through the API on both transports, in one call sequence per (transport, dtype)
    p = _params(ACC.test_every_scheme)
    assert set(p["transport"]) == {"fused", "fallback"} and set(p["dtype"]) == DTYPES and 2 in p["world"]
    seq = {dt: ACC.call_sequence(2, dt) for dt in p["dtype"]}
    assert want <= _combos(c for calls in seq.values() for c, train in calls if train)
    for calls in seq.values():
        cases = [c for c, _ in calls]
        assert any(c.hq != c.hkv for c in cases) and any(c.regime == "peaked" for c in cases)
        assert max(c.rows for c in cases) > cases[0].rows and cases[-1].rows < max(c.rows for c in cases)
        trains = [t for _, t in calls]
        assert any(not t and a and b for a, t, b in zip(trains, trains[1:], trains[2:]))  # forward-only in between
        changes = [(a.scheme, a.causal) != (b.scheme, b.causal) for a, b in zip(cases, cases[1:])]
        assert sum(changes) >= len(changes) - 6  # schemes interleave on one peer context
        assert all(c.rows <= 1024 and c.hq <= 8 for c in cases)
    p = _params(ACC.test_fused_variants_2gpu)
    assert {next(iter(e)) for e in p["env"]} == {"RFA_B200_KV_TRANSPORT", "RFA_B200_PUSH_CTAS",
                                                 "RFA_B200_STAGE_BUDGET_MB"}
    for fn in ("test_llama3_strict_head_groups_2gpu", "test_fp8_block_scaled_stripe_2gpu", "test_deterministic_2gpu"):
        assert callable(getattr(ACC, fn))
    assert {c.scheme for c, _ in ACC.variant_sequence(2, torch.bfloat16)} == {s for s, _ in SCHEMES}
    # one GPU: every combination replayed at worlds 2, 3, 4 and 8, GQA and the peaked regime included
    p = _params(REP.test_replay_matches_fallback_reference)
    cases = [c for (s, causal), dt in itertools.product(p[("scheme", "causal")], p["dtype"])
             for c in REP.replay_cases(s, causal, dt)]
    assert want <= _combos(cases)
    assert {c.world for c in cases} == {2, 3, 4, 8}
    assert any(c.hq != c.hkv for c in cases) and sum(c.regime == "peaked" for c in cases) >= 4
    p = _params(REP.test_deterministic_api_world1)
    assert set(p["mode"]) == {"strict", "fast"}
    p = _params(REP.test_ordered_backward_sweep)
    assert set(p["dtype"]) == DTYPES and set(p["d"]) == HEAD_DIMS and set(p["window"]) == {False, True}
