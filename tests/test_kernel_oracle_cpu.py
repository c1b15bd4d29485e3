"""CPU self-test of ``tests/kernel_oracle.py`` and of the GPU sweep built on it (``test_gpu_kernel_accuracy.py``):
the fp64 oracle agrees with ``ops.dense``, the sweep covers every kernel instantiation, ``tests/fake_ext.py`` (the
kernels' contract on the same work tables) passes it, and mutated copies of the fake - each a plausible kernel bug -
fail it."""
import itertools

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
