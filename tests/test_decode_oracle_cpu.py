"""CPU self-test of ``tests/decode_oracle.py`` and of the GPU decode sweep built on it
(``test_gpu_decode_accuracy.py``): the fp64 reference agrees with the existing decode oracles and with the dense torch
path, the sweep covers every kernel instantiation and reaches every edge of the split-KV kernel, the decode contract in
torch (``fake_ext.FakeDecodeExt``) passes it, and mutated copies of the contract - each a plausible kernel bug -
fail it."""
import itertools

import pytest
import torch

import decode_oracle as DO
import test_gpu_decode_accuracy as GPU_SWEEP
from dist_utils import run_distributed
from fake_ext import FakeDecodeExt
from ring_flash_attn_b200.ops import cuda_ext
from ring_flash_attn_b200.parallel import decode as dec
from test_decode import decode_oracle
from test_decode_varlen import varlen_oracle

INSTANTIATIONS = list(itertools.product([torch.bfloat16, torch.float16], [64, 128], [False, True]))
# a reduced geometry list keeps the CPU runtime to seconds; it still has every kind of edge the mutants below need
CPU_GEOMETRIES = ["rows63_g1", "rows65_g1_one_live_row", "rows129_g3", "keys_0_1_127_128_129", "split_edge_by_append",
                  "splits1", "splits3_of_10_tiles", "splits8_of_3_tiles", "append_overflow", "paged16",
                  "paged256_mid_page_split", "packed_kv", "head_strided", "saturating_append", "varlen44",
                  "rotary_half_neox_noncausal", "rotary_full_interleaved_varlen_noncausal"]
CPU_REGIME_GEOMETRIES = ["splits3_of_10_tiles", "varlen44"]
CPU_CASES = DO.sweep_cases(CPU_GEOMETRIES, CPU_REGIME_GEOMETRIES)


@pytest.fixture
def use_ext(monkeypatch):
    def install(ext):
        monkeypatch.setattr(cuda_ext, "load", lambda: ext)
        return ext

    return install


def _inst_id(inst):
    dtype, d, fp8 = inst
    return DO.report_key(dtype, d, fp8).replace("decode ", "")


def _sweep(inst, cases=CPU_CASES):
    dtype, d, fp8 = inst
    for name, regime in cases:
        DO.run_decode(DO.geometry(name, fp8=fp8), dtype, d, regime, "cpu")


# ---------------------------------------------------------------------------------------------- the fp64 reference

def _grid(inp, x):
    """Packed (rows, H, D) -> (B, Sq, H, D) of a uniform case."""
    return x.view(inp.case.b, inp.case.counts[0], *x.shape[1:])


@pytest.mark.parametrize("name", ["rows64_g16", "keys_0_1_127_128_129", "split_edge_by_append", "splits1",
                                  "empty_shard_append", "no_append_noncausal"])
def test_reference_matches_decode_oracle(name):
    """Uniform cases without rotary, e4m3 or dropped rows: ``test_decode.decode_oracle`` on the same fp32 inputs."""
    case = DO.geometry(name)
    inp = DO.build_inputs(case, torch.float32, 64, "randn", "cpu")
    o64, l64, _, _ = DO.references(inp, 2)
    lens = [torch.tensor(inp.lens)]
    kn = _grid(inp, inp.k_new) if case.append else None
    vn = _grid(inp, inp.v_new) if case.append else None
    out, lse = decode_oracle(_grid(inp, inp.q), [(inp.kc0, inp.vc0)], lens, kn, vn, case.causal)
    got_o, got_l = DO.packed(case, out, lse)
    torch.testing.assert_close(o64.float(), got_o, atol=1e-5, rtol=1e-5)
    torch.testing.assert_close(l64.float(), got_l, atol=1e-5, rtol=1e-5)


def test_reference_matches_varlen_oracle():
    case = DO.geometry("varlen44")
    inp = DO.build_inputs(case, torch.float32, 64, "randn", "cpu")
    o64, l64, _, _ = DO.references(inp, 3)
    smax = max(case.counts)

    def grid(x):  # packed rows -> (B, Smax, H, D), zero past each count
        g = x.new_zeros(case.b, smax, *x.shape[1:])
        for i, (lo, n) in enumerate(DO.spans(case)):
            g[i, :n] = x[lo:lo + n]
        return g

    out, lse = varlen_oracle(grid(inp.q), [(inp.kc0, inp.vc0)], [torch.tensor(inp.lens)], grid(inp.k_new),
                             grid(inp.v_new), case.counts, case.causal)
    torch.testing.assert_close(o64.float(), out, atol=1e-5, rtol=1e-5)
    torch.testing.assert_close(l64.float(), lse, atol=1e-5, rtol=1e-5)


@pytest.mark.parametrize("name,fp8", [("append_overflow", False), ("scap300_filled", False), ("paged64", False),
                                      ("varlen44_paged32", False), ("rotary16_interleaved", False),
                                      ("rotary_full_neox_paged64", False), ("rotary_half_neox_varlen", False),
                                      ("paged32", True), ("saturating_append", True), ("varlen44", True)])
def test_reference_matches_dense_path(name, fp8):
    """``parallel.decode._dense_decode`` on the same inputs (fp32, or bf16 with an e4m3 cache), which also appends:
    its cache afterwards holds the bytes the reference expects."""
    case = DO.geometry(name, fp8=fp8)
    dtype = torch.bfloat16 if fp8 else torch.float32
    inp = DO.build_inputs(case, dtype, 64, "randn", "cpu")
    o64, l64, o32, _ = DO.references(inp, 2)
    q, k, v = DO.call_views(inp, case.append)
    kw = DO.call_kwargs(inp)
    rotary = None
    if inp.rotary is not None:
        rotary = (kw["rotary_cos"], kw["rotary_sin"], kw["rotary_seqlens"], kw["rotary_interleaved"])
    kc, vc = inp.k_cache.clone(), inp.v_cache.clone()
    k0, v0 = kc.clone(), vc.clone()
    out, lse = dec._dense_decode(q, kc, vc, inp.seqlens, k, v, case.causal, 64 ** -0.5, None, 1, inp.table,
                                 inp.k_descale, inp.v_descale, kw.get("cu_seqlens_q"), kw.get("max_seqlen_q", 0),
                                 rotary)
    got_o, got_l = DO.packed(case, out, lse)
    tol = dict(atol=1e-2, rtol=1e-2) if fp8 else dict(atol=1e-5, rtol=1e-5)  # e4m3: out rounded to bf16
    torch.testing.assert_close(got_o.double(), o64, **tol)
    torch.testing.assert_close(got_l.double(), l64, atol=1e-4, rtol=1e-4)
    want_k, want_v = DO.expected_caches(inp, k0, v0, case.append)
    assert torch.equal(DO.bytes_of(kc), DO.bytes_of(want_k)) and torch.equal(DO.bytes_of(vc), DO.bytes_of(want_v))


def test_precision_matched_error_is_small_but_not_zero():
    """The matched reference rounds P and out to bf16: it is well off the fp64 result, yet more than ten times closer
    than the atol / rtol of 2e-2 the older decode tests used."""
    case = DO.geometry("splits3_of_10_tiles")
    inp = DO.build_inputs(case, torch.bfloat16, 128, "randn", "cpu")
    o64, l64, o32, l32 = DO.references(inp, 3)
    e_lp = (o32.to(torch.bfloat16).double() - o64).abs().max()
    assert 1e-5 < e_lp < 2e-3
    assert ((l32.double() - l64).abs() / (1 + l64.abs())).max() < 1e-6


# ---------------------------------------------------------------------------------------------- coverage

def _params(fn):
    return {m.args[0]: list(m.args[1]) for m in fn.pytestmark if m.name == "parametrize"}


def test_sweep_covers_every_instantiation():
    p = _params(GPU_SWEEP.test_decode_sweep)
    assert set(itertools.product(p["dtype"], p["d"], p["fp8"])) == set(INSTANTIATIONS)
    assert set(_params(GPU_SWEEP.test_two_gpus_combine_matches_oracle)["fp8"]) == {False, True}
    assert set(DO.sweep_cases()) >= {(g, "randn") for g in DO.GEOMETRY_NAMES}
    assert {r for _, r in DO.sweep_cases()} == set(DO.REGIMES)


def _limits(c):
    """Per sequence: (clamped length, visible-key limit of every token)."""
    out = []
    for n, cnt in zip(c.seqlens, c.counts):
        n = min(max(n, 0), c.s_cap)
        vis = [0 if not c.append else (t + 1 if c.causal else cnt) for t in range(cnt)]
        out.append((n, [min(n + x, c.s_cap) for x in vis]))
    return out


def _splits(c):
    return c.splits if c.splits is not None else DO.default_splits(c, "cpu")


def test_geometries_reach_the_edges():
    geoms = DO.GEOMETRIES
    uniform = [c for c in geoms if not c.varlen]
    rows = {c.counts[0] * c.group for c in uniform}
    assert {1, 63, 64, 65, 128, 129} <= rows
    assert {1, 2, 4, 8, 16} <= {c.group for c in geoms}
    assert any(r % 64 == 1 and r > 64 for r in rows)  # a row tile with a single live row
    visible = {x for c in geoms for _, lims in _limits(c) for x in lims}
    assert {0, 1, 127, 128, 129} <= visible
    tps = lambda c: -(-max(1, -(-c.s_cap // 128)) // _splits(c))  # noqa: E731
    for off in (-1, 0, 1):  # one below, at and above a split boundary other than 0
        assert any(tps(c) * 128 + off in {x for _, lims in _limits(c) for x in lims} for c in geoms
                   if _splits(c) > 1), off
    tiles = lambda c: -(-c.s_cap // 128)  # noqa: E731
    assert any(c.splits == 1 for c in geoms) and any(c.splits is None for c in geoms)
    assert any(c.splits and c.splits < tiles(c) and tiles(c) % c.splits for c in geoms)
    assert any(c.splits and c.splits > tiles(c) for c in geoms)
    # S_cap: not a multiple of 128 and filled; appends that drop some rows and all rows; seqlens past S_cap; empty
    assert any(c.s_cap % 128 and any(max(lims) == c.s_cap for _, lims in _limits(c)) for c in geoms)
    assert any(c.append and n < c.s_cap < n + cnt for c in geoms for n, cnt in zip(c.seqlens, c.counts))
    assert any(c.append and n == c.s_cap and cnt for c in geoms for n, cnt in zip(c.seqlens, c.counts))
    assert any(n > c.s_cap for c in geoms for n in c.seqlens)
    assert any(c.append and 0 in c.seqlens for c in geoms) and any(not c.append and 0 in c.seqlens for c in geoms)
    assert {(c.causal, c.append) for c in geoms} == set(itertools.product((True, False), (True, False)))
    # paged: every page size; one split over more than 64 pages of 16; page 256 with a split starting mid-page
    paged = [c for c in geoms if c.layout == "paged"]
    assert {16, 32, 64, 128, 256} <= {c.page_size for c in paged}
    assert any(c.page_size == 16 and c.splits == 1 and max(c.seqlens) >= 1100 for c in paged)
    assert any(c.page_size == 256 and (tps(c) * 128) % 256 for c in paged)
    assert {"packed_kv", "head_strided"} <= {c.layout for c in geoms}
    assert any(c.saturate for c in geoms)
    # varlen: >= 40 sequences with zero and one counts and a chunk past one row tile, contiguous and paged
    var = [c for c in geoms if c.varlen and c.b >= 40]
    assert {"contiguous", "paged"} <= {c.layout for c in var}
    for c in var:
        assert 0 in c.counts and 1 in c.counts and any(n * c.group > 64 for n in c.counts)
        assert any(n * c.group > 64 for n in c.counts[32:]) and c.counts[-1] == 0
    rot = [c for c in geoms if c.rotary]
    assert {c.rotary[1] for c in rot} == {True, False} and {c.causal for c in rot} == {True, False}
    assert {c.rotary[0] for c in rot} == {16, "half", "full"} and any(c.varlen for c in rot)
    assert any(c.splits is None and 16384 <= c.s_cap <= 32768 and max(c.seqlens) >= 16384 for c in geoms)
    assert any(_splits(DO.geometry(g)) > 1 for g in DO.REGIME_GEOMETRIES)


# ---------------------------------------------------------------------------------------------- the contract passes

@pytest.mark.parametrize("inst", INSTANTIATIONS, ids=_inst_id)
def test_fake_decode_passes_sweep(use_ext, inst):
    fake = use_ext(FakeDecodeExt())
    _sweep(inst)
    assert {"decode_fwd", "decode_combine"} == set(fake.calls)


@pytest.mark.parametrize("fp8", [False, True], ids=["native", "e4m3"])
def test_fake_decode_passes_two_ranks(fp8):
    """The rank combine of ``kernel_decode`` (``decode_combine`` into fp32, the gather, the second combine) over gloo."""
    run_distributed(DO.run_two_ranks, 2, fp8, "cpu")


# ---------------------------------------------------------------------------------------------- planted errors

class CausalNVisT(FakeDecodeExt):  # causal n_vis = t: a token misses its own appended key
    def _n_vis(self, t, n_q, causal, appended):
        return t if appended and causal else super()._n_vis(t, n_q, causal, appended)


class CausalSeesNextKey(FakeDecodeExt):  # causal token t also sees appended key t + 1 (a finite row)
    def _n_vis(self, t, n_q, causal, appended):
        return min(t + 2, n_q) if appended and causal else super()._n_vis(t, n_q, causal, appended)


class TilesPerSplitFloor(FakeDecodeExt):
    def _tiles_per_split(self, tiles, n_splits):
        return max(1, tiles // n_splits)


class KvHeadModulo(FakeDecodeExt):
    def _kv_head(self, h, group, hkv):
        return h % hkv


class PInBf16(FakeDecodeExt):  # P rounded to bf16 whatever q's dtype
    def _p_for_pv(self, p, dtype):
        return p.to(torch.bfloat16).float()


class VDescaleByHeadOnly(FakeDecodeExt):
    def _v_descale(self, ds, b, kv_head):
        return ds.view(-1)[kv_head]


class NonCausalQueryRotatedPerToken(FakeDecodeExt):
    def _q_position(self, start, t, causal):
        return start + t


class BigPageFromRow0(FakeDecodeExt):  # a tile of a page_size > 128 page read from row 0, not key0 % page_size
    def _page_row(self, key, page_size):
        return key % 128 if page_size > 128 else key % page_size


class VarlenBaseNotCarried(FakeDecodeExt):  # sequences 32 and up mapped without the tiles of the first 32
    def _carry(self, base, step_tiles):
        return base


class CombineDropsLastPartial(FakeDecodeExt):
    def _combine_parts(self, parts):
        return parts[:-1] if parts.shape[0] > 1 else parts[:0]


class EmptySplitLseZero(FakeDecodeExt):
    def _empty_lse(self):
        return 0.0


class LseShifted(FakeDecodeExt):
    def _finish_lse(self, lse):
        return lse + 1e-3


MUTANTS = [CausalNVisT, CausalSeesNextKey, TilesPerSplitFloor, KvHeadModulo, PInBf16, VDescaleByHeadOnly,
           NonCausalQueryRotatedPerToken, BigPageFromRow0, VarlenBaseNotCarried, CombineDropsLastPartial,
           EmptySplitLseZero, LseShifted]


@pytest.mark.parametrize("mutant", MUTANTS, ids=lambda m: m.__name__)
def test_sweep_catches_planted_error(use_ext, mutant):
    use_ext(mutant())
    caught = None
    for inst in INSTANTIATIONS:
        try:
            _sweep(inst)
        except AssertionError as e:
            caught = str(e)
            break
    assert caught, f"{mutant.__name__} passed the whole sweep"
