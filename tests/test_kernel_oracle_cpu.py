"""CPU self-test of ``tests/kernel_oracle.py`` and of the GPU sweep built on it (``test_gpu_kernel_accuracy.py``):
the fp64 oracle agrees with ``ops.dense``, the sweep covers every kernel instantiation, ``tests/fake_ext.py`` (the
kernels' contract on the same work tables) passes it, and mutated copies of the fake - each a plausible kernel bug -
fail it."""
import itertools
import math

import pytest
import torch

import kernel_oracle as KO
import test_gpu_kernel_accuracy as GPU_SWEEP
from fake_ext import DIAG_FULL, LO_NONE, FakeExt
from ring_flash_attn_b200.ops import cuda_ext
from ring_flash_attn_b200.ops.dense import block_bwd, block_fwd

# a reduced geometry list keeps the CPU runtime to seconds; it still has multi-segment, windowed and GQA plans
CPU_GEOMETRIES = ["q1_k1", "q64_k65_gqa2", "q127_k128_diag-1", "q129_k129_gqa8", "q200_k333",
                  "diag-200_and_blind_chunk", "zigzag_adjacent", "overlapping_segments", "window_lo-10",
                  "window_rows_past_keys"]
CPU_REGIME_GEOMETRIES = ["q64_k65_gqa2", "zigzag_adjacent"]
CPU_CASES = KO.sweep_cases(CPU_GEOMETRIES, CPU_REGIME_GEOMETRIES)
INSTANTIATIONS = list(itertools.product([torch.bfloat16, torch.float16], [64, 128], [False, True], ["fwd", "bwd"]))


@pytest.fixture
def use_ext(monkeypatch):
    def install(ext):
        monkeypatch.setattr(cuda_ext, "load", lambda: ext)
        return ext

    return install


def _run(case, inst):
    (name, regime), (dtype, d, window, direction) = case, inst
    geom = KO.geometry(name)
    if direction == "fwd":
        KO.run_forward(geom, d, dtype, window, regime, "cpu")
    else:
        KO.run_backward(geom, d, dtype, window, regime, "cpu", dkv_dtype=dtype if len(name) % 2 else torch.float32)


# ---------------------------------------------------------------------------------------------- oracle vs dense

@pytest.mark.parametrize("name", ["zigzag_adjacent", "overlapping_segments", "chunks_row0_kvrow0", "window_two_segs",
                                  "diag-200_and_blind_chunk"])
@pytest.mark.parametrize("window", [False, True])
def test_oracle_matches_dense(name, window):
    """Per-segment ``dense.block_fwd`` partials merged by lse, and summed ``dense.block_bwd`` contributions."""
    geom = KO.geometry(name)
    plan = KO.build_plan(geom, window)
    q, k, v, do = KO.make_inputs(geom, 64, torch.float32, "randn", "cpu")
    scale = 64 ** -0.5
    o64, l64 = KO.plan_forward(plan, plan.segments, q, k, v, scale)
    delta = (o64 * do.double()).sum(-1).transpose(0, 1)
    dq64, dk64, dv64 = KO.plan_backward(plan, plan.segments, q, k, v, do, l64, delta, scale)
    out = torch.zeros_like(q)
    lse = torch.full((q.shape[1], q.shape[0]), float("-inf"))
    dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
    for ci, ch in enumerate(plan.q_chunks):
        rows = slice(ch.row0, ch.row0 + ch.rows)
        parts = [(s, *block_fwd(q[rows], k[s.kv_row0:s.kv_row0 + s.kv_len], v[s.kv_row0:s.kv_row0 + s.kv_len], scale,
                                s.diag, s.lo)) for s in plan.segments if s.chunk == ci]
        if not parts:
            continue
        l = torch.logsumexp(torch.stack([p[2] for p in parts]), dim=0)
        lse[:, rows] = l
        l_safe = torch.where(torch.isinf(l), torch.zeros_like(l), l)
        out[rows] = sum(o * torch.exp(ls - l_safe).transpose(0, 1).unsqueeze(-1) for _, o, ls in parts)
        for s, _, _ in parts:
            keys = slice(s.kv_row0, s.kv_row0 + s.kv_len)
            g = block_bwd(do[rows], q[rows], k[keys], v[keys], l64[:, rows].float(), delta[:, rows].float(), scale,
                          s.diag, s.lo)
            dq[rows] += g[0]
            dk[keys] += g[1]
            dv[keys] += g[2]
    tol = dict(atol=1e-5, rtol=1e-4)
    torch.testing.assert_close(out.double(), o64, **tol)
    torch.testing.assert_close(lse.double(), l64, **tol)
    for got, want in ((dq, dq64), (dk, dk64), (dv, dv64)):
        torch.testing.assert_close(got.double(), want, **tol)


def test_precision_matched_reference_is_between():
    """The fp32 / rounded reference is much closer to fp64 than a bf16 one and no closer than fp32 itself."""
    geom = KO.geometry("q200_k333")
    plan = KO.build_plan(geom, False)
    q, k, v, _ = KO.make_inputs(geom, 64, torch.bfloat16, "randn", "cpu")
    o64, _ = KO.plan_forward(plan, plan.segments, q, k, v, 0.125)
    olp, _ = KO.plan_forward(plan, plan.segments, q, k, v, 0.125, p_dtype=torch.bfloat16)
    o32, _ = KO.plan_forward(plan, plan.segments, q, k, v, 0.125, p_dtype=torch.float32)
    e_lp, e_32 = (olp.double() - o64).abs().max(), (o32.double() - o64).abs().max()
    assert 1e-4 < e_lp < 2e-2 and e_32 < e_lp / 50


# ---------------------------------------------------------------------------------------------- coverage

def _params(fn):
    out = {}
    for mark in fn.pytestmark:
        if mark.name == "parametrize":
            out[mark.args[0]] = list(mark.args[1])
    return out


def test_sweep_covers_every_instantiation():
    p = _params(GPU_SWEEP.test_kernel_sweep)
    grid = set(itertools.product(p["dtype"], p["d"], p["window"], p["direction"]))
    assert grid == set(INSTANTIATIONS)
    p = _params(GPU_SWEEP.test_invisible_rows_change_nothing)
    assert set(itertools.product(p["dtype"], p["d"], p["window"], p["direction"])) == set(INSTANTIATIONS)
    p = _params(GPU_SWEEP.test_delta_and_dq_finalize)
    assert set(p["dtype"]) == {torch.bfloat16, torch.float16} and set(p["d"]) == {64, 128}
    p = _params(GPU_SWEEP.test_fp8_forward_sweep)
    assert p["name"] and set(p["blocks"]) == {"per_head", "block_scaled"}


def test_geometries_reach_the_edges():
    geoms = KO.GEOMETRIES
    rows = {n for g in geoms for _, n in g["chunks"]}
    keys = {s[2] for g in geoms for s in g["segs"]}
    assert {1, 63, 64, 65, 127, 128, 129} <= rows and any(380 <= r <= 390 for r in rows)
    assert {1, 64, 65, 127, 128, 129, 333, 1024} <= keys
    assert {5, 77} <= {s[1] for g in geoms for s in g["segs"]}
    assert any(r0 != 0 for g in geoms if len(g["chunks"]) > 1 for r0, _ in g["chunks"])
    assert {1, 2, 4, 8} <= {g["hq"] // g["hkv"] for g in geoms}
    diags = [(s[3], s[2]) for g in geoms for s in g["segs"]]
    assert any(d is None for d, _ in diags) and {0, -1} <= {d for d, _ in diags}
    assert any(d is not None and d <= -128 for d, _ in diags)  # whole 64-row backward query tiles skipped
    assert any(d is not None and d > n for d, n in diags)
    multi = [g for g in geoms if any(sum(s[0] == c for s in g["segs"]) > 1 for c in range(len(g["chunks"])))]
    adjacent = overlapping = False
    for g in multi:
        for a, b in itertools.combinations(g["segs"], 2):
            if a[0] == b[0]:
                adjacent |= a[1] + a[2] == b[1] or b[1] + b[2] == a[1]
                overlapping |= a[1] < b[1] + b[2] and b[1] < a[1] + a[2]
    assert adjacent and overlapping
    assert any(s[4] is not None and s[4] > 0 for g in geoms for s in g["segs"])
    for g, r in itertools.product(KO.REGIME_GEOMETRIES, KO.REGIMES):
        assert (g, r) in KO.sweep_cases()


# ---------------------------------------------------------------------------------------------- the contract passes

@pytest.mark.parametrize("inst", INSTANTIATIONS, ids=lambda i: KO.report_key(i[3], i[1], i[0], i[2]))
def test_fake_ext_passes_sweep(use_ext, inst):
    use_ext(FakeExt())
    for case in CPU_CASES:
        _run(case, inst)


@pytest.mark.parametrize("direction", ["fwd", "bwd"])
@pytest.mark.parametrize("window", [False, True])
def test_fake_ext_passes_invisibility(use_ext, window, direction):
    use_ext(FakeExt())
    KO.run_invisibility(64, torch.bfloat16, window, direction == "bwd", "cpu")


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_fake_ext_passes_delta_and_dq_finalize(use_ext, dtype, d):
    use_ext(FakeExt())
    KO.run_delta_and_dq_finalize(dtype, d, "cpu")


@pytest.mark.parametrize("blocks", ["per_head", "block_scaled"])
def test_fake_ext_passes_fp8(use_ext, blocks):
    use_ext(FakeExt())
    for name in GPU_SWEEP.FP8_GEOMETRIES:
        KO.run_fp8_forward(KO.geometry(name), blocks, "cpu")


# ---------------------------------------------------------------------------------------------- planted errors

class DiagPlus1(FakeExt):
    def _mask(self, n_rows, q_off, kv_len, diag, lo):
        return super()._mask(n_rows, q_off, kv_len, diag + 1 if diag < DIAG_FULL else diag, lo)


class LoMinus1(FakeExt):
    def _mask(self, n_rows, q_off, kv_len, diag, lo):
        return super()._mask(n_rows, q_off, kv_len, diag, lo - 1 if lo > LO_NONE else lo)


class LastKeyDropped(FakeExt):
    def _mask(self, n_rows, q_off, kv_len, diag, lo):
        m = super()._mask(n_rows, q_off, kv_len, diag, lo)
        m[:, -1] = False
        return m


class KvHeadModulo(FakeExt):
    def _kv_heads(self, x, rep):  # query head h reads kv head h % hkv
        return x.repeat(1, rep, 1)


class PInE4M3(FakeExt):
    def _p_for_pv(self, p, dtype):
        return p.to(torch.float8_e4m3fn).float()


class LseShifted(FakeExt):
    def _fwd(self, q, k, v, items, segs, seg_lo, out, lse, scale, sqk=None, sv=None):
        super()._fwd(q, k, v, items, segs, seg_lo, out, lse, scale, sqk, sv)
        lse.add_(1e-3)


class FirstHeadOfGroup(FakeExt):
    def _group_sum(self, x, hkv, rep):
        return x.view(x.shape[0], hkv, rep, x.shape[2])[:, :, 0].clone()


MUTANTS = [DiagPlus1, LoMinus1, LastKeyDropped, KvHeadModulo, PInE4M3, LseShifted, FirstHeadOfGroup]


@pytest.mark.parametrize("mutant", MUTANTS, ids=lambda m: m.__name__)
def test_sweep_catches_planted_error(use_ext, mutant):
    use_ext(mutant())
    caught = []
    for inst in INSTANTIATIONS:
        for case in CPU_CASES:
            try:
                _run(case, inst)
            except AssertionError as e:
                caught.append(str(e))
                break
        if caught:
            break
    assert caught, f"{mutant.__name__} passed the whole sweep"


# ---------------------------------------------------------------------------------------------- long contexts

def _unchunked_forward(plan, segs, q, k, v, scale, p_dtype=None):
    """``plan_forward`` as it was before it worked in blocks: one (Hq, rows, keys) score tensor per chunk."""
    lowp = p_dtype is not None
    cd = torch.float32 if lowp else torch.float64
    tq, hq, d = q.shape
    rep = hq // k.shape[1]
    out = torch.zeros((tq, hq, d), dtype=cd)
    lse = torch.full((hq, tq), float("-inf"), dtype=cd)
    t2 = float(torch.tensor(scale * KO.LOG2E, dtype=torch.float32))
    for ci, cs in KO._by_chunk(segs).items():
        ch = plan.q_chunks[ci]
        rows = slice(ch.row0, ch.row0 + ch.rows)
        qc = q[rows].to(cd)
        sc = torch.cat([KO._scores(qc, k[s.kv_row0:s.kv_row0 + s.kv_len].to(cd).repeat_interleave(rep, 1), s, 0, 0)
                        for s in cs], dim=-1)
        vv = torch.cat([v[s.kv_row0:s.kv_row0 + s.kv_len].to(cd).repeat_interleave(rep, 1) for s in cs])
        mx = sc.amax(dim=-1, keepdim=True)
        empty = torch.isinf(mx)
        if lowp:
            m2 = torch.where(empty, torch.zeros_like(mx), mx * t2)
            p = KO._exp2_fma(sc, t2, m2)
            l = p.sum(dim=-1, keepdim=True)
            row_lse = (m2 + torch.log2(l)) * math.log(2.0)
            p = p.to(p_dtype).to(cd)
        else:
            m = torch.where(empty, torch.zeros_like(mx), mx)
            p = torch.exp((sc - m) * scale)
            l = p.sum(dim=-1, keepdim=True)
            row_lse = m * scale + torch.log(l)
        o = torch.einsum("hnk,khd->nhd", p, vv) / torch.where(empty, torch.ones_like(l), l).permute(1, 0, 2)
        out[rows] = torch.where(empty.permute(1, 0, 2), torch.zeros_like(o), o)
        lse[:, rows] = torch.where(empty, torch.full_like(row_lse, float("-inf")), row_lse).squeeze(-1)
    return out, lse


def _unchunked_backward(plan, segs, q, k, v, dout, lse, delta, scale, mm_dtype=None):
    """``plan_backward`` as it was before it worked in blocks (dq, dk, dv in fp32 / fp64)."""
    lowp = mm_dtype is not None
    cd = torch.float32 if lowp else torch.float64
    tq, hq, d = q.shape
    tk, hkv, _ = k.shape
    rep = hq // hkv
    dq, dk = torch.zeros((tq, hq, d), dtype=cd), torch.zeros((tk, hkv, d), dtype=cd)
    dv = torch.zeros_like(dk)
    lse, delta = lse.to(cd), delta.to(cd)
    t2 = float(torch.tensor(scale * KO.LOG2E, dtype=torch.float32))
    rnd = (lambda x: x.to(mm_dtype).to(cd)) if lowp else (lambda x: x)
    for ci, cs in KO._by_chunk(segs).items():
        ch = plan.q_chunks[ci]
        rows = slice(ch.row0, ch.row0 + ch.rows)
        qc, doc = q[rows].to(cd), dout[rows].to(cd)
        lr = lse[:, rows].unsqueeze(-1)
        lr = torch.where(torch.isinf(lr), torch.full_like(lr, float("inf")), lr)
        for s in cs:
            keys = slice(s.kv_row0, s.kv_row0 + s.kv_len)
            kk, vv = k[keys].to(cd).repeat_interleave(rep, 1), v[keys].to(cd).repeat_interleave(rep, 1)
            sc = KO._scores(qc, kk, s, 0, 0)
            p = KO._exp2_fma(sc, t2, (lr * KO.LOG2E).float()) if lowp else torch.exp(sc * scale - lr)
            ds = p * (torch.einsum("nhd,khd->hnk", doc, vv) - delta[:, rows].unsqueeze(-1)) * scale
            p, ds = rnd(p), rnd(ds)
            dq[rows] += torch.einsum("hnk,khd->nhd", ds, kk)
            dk[keys] += torch.einsum("hnk,nhd->khd", ds, qc).reshape(s.kv_len, hkv, rep, d).sum(2)
            dv[keys] += torch.einsum("hnk,nhd->khd", p, doc).reshape(s.kv_len, hkv, rep, d).sum(2)
    return dq, dk, dv


@pytest.mark.parametrize("window", [False, True])
@pytest.mark.parametrize("row_block,block_elems", [(64, 1 << 12), (50, 1 << 16), (1024, 1 << 27)])
def test_blocked_references_match_unchunked(monkeypatch, row_block, block_elems, window):
    """Row blocks (64, and 50: off the kernels' tile grid), head groups down to one head and parts of a GQA group, and
    the skipped key ranges past the diagonal / before the window change nothing but summation order: fp64 to 1e-12,
    the precision-matched arithmetic in fp32 (P and dS unrounded, so that an fp32 score one ulp off cannot flip a bf16
    rounding) to fp32 summation order."""
    monkeypatch.setattr(KO, "ROW_BLOCK", row_block)
    monkeypatch.setattr(KO, "BLOCK_ELEMS", block_elems)
    f32 = torch.float32
    for geom in KO.GEOMETRIES + [KO.INVISIBLE_GEOMETRY]:
        plan = KO.build_plan(geom, window)
        segs = plan.segments
        q, k, v, do = KO.make_inputs(geom, 64, torch.bfloat16, "randn", "cpu")
        scale = 64 ** -0.5
        o64, l64 = KO.plan_forward(plan, segs, q, k, v, scale)
        delta = (o64 * do.double()).sum(-1).transpose(0, 1)
        lse32, delta32 = l64.float(), delta.float()
        pairs = {
            "fp64": ((o64, l64) + KO.plan_backward(plan, segs, q, k, v, do, l64, delta, scale),
                     _unchunked_forward(plan, segs, q, k, v, scale)
                     + _unchunked_backward(plan, segs, q, k, v, do, l64, delta, scale)),
            "fp32": (KO.plan_forward(plan, segs, q, k, v, scale, p_dtype=f32)
                     + KO.plan_backward(plan, segs, q, k, v, do, lse32, delta32, scale, mm_dtype=f32),
                     _unchunked_forward(plan, segs, q, k, v, scale, p_dtype=f32)
                     + _unchunked_backward(plan, segs, q, k, v, do, lse32, delta32, scale, f32)),
        }
        for kind, (got, want) in pairs.items():
            rel = 1e-12 if kind == "fp64" else 2e-5
            for what, a, b in zip(("out", "lse", "dq", "dk", "dv"), got, want):
                torch.testing.assert_close(a, b, rtol=rel, atol=rel * max(b.abs().nan_to_num(0, 0, 0).max(), 1),
                                           msg=lambda m: f"{geom['name']} {kind} {what}: {m}")


def test_per_block_bound_catches_a_tile_lost_at_32k():
    """S = 32768, one head, causal, bf16: the precision-matched out with key tile 100 dropped for the last 64 rows.
    The tensor-wide bound (its baseline set by the short rows at the start) and ``sampled_check``'s tolerance both
    accept it; the per-(head, 64-row block) bound rejects it.  Only the rows involved are computed: the first 1024,
    which set the baseline, and the last 64."""
    from ring_flash_attn_b200.ops import plan as P
    from ring_flash_attn_b200.utils.verify import sampled_check

    S, d, tile = 32768, 128, 100
    q, k, v, _ = KO.make_inputs(dict(tq=S, tk=S, hq=1, hkv=1), d, torch.bfloat16, "randn", "cpu")
    r0 = S - 64
    chunks = [P.QChunk(0, 1024), P.QChunk(r0, 64)]
    plan = P.CPPlan(1, 0, S, S, chunks, [P.Segment(0, 0, 0, S, 0), P.Segment(1, 0, 0, S, r0)])
    lost = P.CPPlan(1, 0, S, S, chunks, [P.Segment(0, 0, 0, S, 0), P.Segment(1, 0, 0, tile * 128, r0),
                                         P.Segment(1, 0, tile * 128 + 128, S - tile * 128 - 128,
                                                   r0 - tile * 128 - 128)])
    scale = d ** -0.5
    rows = KO.chunk_rows(plan, "cpu")
    o64 = KO.plan_forward(plan, plan.segments, q, k, v, scale)[0][rows]
    olp = KO.plan_forward(plan, plan.segments, q, k, v, scale, p_dtype=torch.bfloat16)[0][rows]
    bad = KO.plan_forward(lost, lost.segments, q, k, v, scale, p_dtype=torch.bfloat16)[0][rows]
    assert torch.equal(bad[:1024], olp[:1024]) and not torch.equal(bad[1024:], olp[1024:])
    ratio = KO.assert_accurate("tile lost", bad, o64, olp, row_ids=rows)
    assert ratio < KO.MAX_RATIO
    err = (bad.double() - o64).abs().max().item()
    tol = sampled_check("ring", q, k, v, None, torch.zeros_like(q), None, None, None, None)["tol"]["out"]
    assert err < tol, (err, tol)
    with pytest.raises(AssertionError, match=f"block rows {r0}..{S - 1}, head 0: "):
        KO.assert_accurate("tile lost", bad, o64, olp, row_ids=rows, blocks=(64, 1, None))


class _LateItem(FakeExt):
    """Base of mutants that break the forward's last work item only (the highest query rows)."""
    late = False

    def _fwd(self, q, k, v, items, segs, seg_lo, out, lse, scale, sqk=None, sv=None):
        last = int(items[:, 0].argmax())
        for i in range(items.shape[0]):
            self.late = i == last
            super()._fwd(q, k, v, items[i:i + 1], segs, seg_lo, out, lse, scale, sqk, sv)
        self.late = False


class LateKeyTileDropped(_LateItem):
    def _mask(self, n_rows, q_off, kv_len, diag, lo):
        m = super()._mask(n_rows, q_off, kv_len, diag, lo)
        if self.late:
            m[:, 10 * 128:11 * 128] = False
        return m


class LateTileStaleMax(_LateItem):
    """Key tile 2's P left relative to the running maximum after that tile (a missed rescale when later tiles raise
    it)."""

    def _p_for_pv(self, p, dtype):
        if not self.late:
            return p
        p = p.clone()
        p[..., 256:384] *= p.amax(-1, keepdim=True) / p[..., :384].amax(-1, keepdim=True).clamp_min(1e-30)
        return p


class DqTileLost(FakeExt):
    """Key tile 10's dQ contribution to query rows 6400 .. 6463 never lands."""

    def _dq_part(self, x, q_row0, kv_row0):
        a = 6400 - q_row0
        if kv_row0 == 1280 and 0 <= a < x.shape[0]:
            x = x.clone()
            x[a:a + 64] = 0
        return x


class DkvModelDtype(FakeExt):
    """dK / dV rounded to the model dtype after every 64-row query tile instead of once."""

    def _bwd(self, q, dout, k, v, dq, items, qsegs, lse, delta, dk, dv, scale, window):
        tiles, per_item, segs = [], [], qsegs.tolist()
        for kv_row0, kv_rows, seg_begin, seg_count, *rest in items.tolist():
            first = len(tiles)
            for q_row0, q_len, diag, lo in segs[seg_begin:seg_begin + seg_count]:
                for i in range(0, q_len, 64):
                    tiles.append([q_row0 + i, min(64, q_len - i), diag + i if diag < DIAG_FULL else diag,
                                  lo + i if lo > LO_NONE else lo])
            per_item.append([kv_row0, kv_rows, first, len(tiles) - first, *rest])
        super()._bwd(q, dout, k, v, dq, torch.tensor(per_item), torch.tensor(tiles), lse, delta, dk, dv, scale,
                     window)

    def _accumulate(self, acc, x, dtype):
        return (acc + x).to(dtype).float()


# one kv head at 8192 tokens: 64 forward items of 128 rows, 64 backward key tiles
LONG_CASE = dict(fn_name="zigzag_ring_flash_attn_kvpacked_func", b=1, s=8192, hq=1, hkv=1, d=64, dtype=torch.bfloat16)


@pytest.fixture
def long_path(monkeypatch):
    def install(ext):
        monkeypatch.setattr(cuda_ext, "load", lambda: ext)
        monkeypatch.setattr(cuda_ext, "available_for", lambda t: True)

    return install


def test_fake_ext_passes_long_path(long_path):
    long_path(FakeExt())
    KO.run_api(**LONG_CASE, device="cpu")


@pytest.mark.parametrize("mutant,where", [
    (LateKeyTileDropped, r"out: block rows (80[6-9]|81[0-9])[0-9]\.\.(80|81)[0-9]{2}, head 0: "),
    (LateTileStaleMax, r"out: block rows (80[6-9]|81[0-9])[0-9]\.\.(80|81)[0-9]{2}, head 0: "),
    (DqTileLost, r"dq: block rows 6400\.\.6463, head 0: "),
    (DkvModelDtype, r"d[kv]: block keys \d+\.\.\d+, kv head 0: "),
], ids=lambda x: getattr(x, "__name__", ""))
def test_long_path_catches_planted_error(long_path, mutant, where):
    """Each mutant breaks one unit of work, or rounds where the kernels do not, and the per-block bound names it."""
    long_path(mutant())
    with pytest.raises(AssertionError, match=where):
        KO.run_api(**LONG_CASE, device="cpu")


class RoundedP(FakeExt):
    """A legitimate kernel-like forward: P rounded to the model dtype before P V, as the sm_90a forward does, but
    formed as exp(s - lse) in fp32 rather than exp2 relative to the running maximum."""

    def _p_for_pv(self, p, dtype):
        return p.to(dtype).float()


def test_legitimate_per_block_ratio_exceeds_2x(long_path):
    """Why the per-block factor is ``BLOCK_RATIO`` and not 2: a correct implementation that rounds in the same places
    as the reference, differing only in fp32 detail, passes the tensor-wide bound at 1.6x and reaches 2.4x in its worst
    64-row block (the H100 kernels measured up to 2.46x).  The weakest planted error above is 15x."""
    long_path(RoundedP())
    KO.WORST.pop("legit per-block", None)
    KO.run_api(**dict(LONG_CASE, dtype=torch.float16), backward=False, device="cpu", report="legit")
    worst = KO.WORST.pop("legit per-block")
    assert 2.0 < worst < KO.BLOCK_RATIO, worst
