"""Every context-parallel scheme's per-rank plans on the sm_90a kernels of ONE GPU, against the fp64 plan oracle with
the precision-matched bound of the torch.distributed fallback (``tests/cp_oracle.py``).

``cp_oracle.replay`` runs what the fallback runs on each rank - one ``engine.step_forward`` / ``step_backward`` launch
per source shard, the partials merged in fp32 in the transport's source order, dK / dV summed over the ranks in fp32
- at worlds 2, 3, 4 and 8 without a process group.  ``deterministic=True`` (ordered launch groups) is held to the
same bound at world 1: over the kernel sweep's geometries and through the public API in both modes."""
import itertools

import pytest
import torch

import cp_oracle as CP
import kernel_oracle as KO
from ring_flash_attn_b200.parallel import engine

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
HEAD_DIMS = [64, 128]
WINDOWS = [False, True]
# (scheme, causal)
SCHEMES = [("ring", True), ("ring", False), ("zigzag", True), ("stripe", True), ("ring_varlen", True),
           ("ring_varlen", False), ("zigzag_varlen", True), ("llama3", True), ("zigzag_llama3", True)]
WORLDS = [2, 3, 4, 8]
HEADS = [(4, 2), (4, 4), (8, 2), (2, 1)]  # (hq, hkv): GQA groups of 2, 1, 4, 2


@pytest.fixture(autouse=True)
def _exact_fp32_matmul():
    """The precision-matched reference needs true fp32 GEMMs."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


def replay_cases(scheme: str, causal: bool, dtype):
    """Head dim x window for one scheme, worlds and head layouts rotating; the first D 128 plain case also runs the
    ``peaked`` regime (row maximum in a remote source's last tile)."""
    cases = []
    for i, (d, window) in enumerate(itertools.product(HEAD_DIMS, WINDOWS)):
        world = WORLDS[(i + SCHEMES.index((scheme, causal))) % len(WORLDS)]
        rows = 256 if world < 8 else 128
        hq, hkv = HEADS[(i + DTYPES.index(dtype)) % len(HEADS)]
        base = CP.Case(scheme, world, rows, hq, hkv, d, dtype, causal, batch=2 if scheme in CP.BATCH and i % 2 else 1)
        if window:
            base = base.with_(window=CP.window_for(causal, base.total))
        cases.append(base)
        if d == 128 and not window:
            cases.append(base.with_(regime="peaked"))
    return cases


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("scheme,causal", SCHEMES, ids=[f"{s}{'' if c else '-noncausal'}" for s, c in SCHEMES])
def test_replay_matches_fallback_reference(scheme, causal, dtype):
    for seed, case in enumerate(replay_cases(scheme, causal, dtype)):
        plans = CP.build_plans(case)
        q, k, v, do = CP.make_inputs(case, seed, "cuda")
        assert engine._use_cuda_kernels(q[0], k[0]), "the replay must run the sm_90a kernels"
        train = case.regime in CP.BACKWARD_REGIMES
        got = CP.replay(case, plans, q, k, v, do, backward=train)
        refs = CP.references(case, plans, q, k, v, do, CP.FALLBACK_ORDER[scheme], backward=train)
        for r in range(case.world):
            CP.check(f"{case.name()} rank {r}", got[r], *refs[r], report=CP.report_key("replay", case.world))


# ---------------------------------------------------------------------------------------------- deterministic=True

@pytest.mark.parametrize("window", [False, True], ids=["plain", "window"])
@pytest.mark.parametrize("d", HEAD_DIMS)
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_ordered_backward_sweep(dtype, d, window):
    """The ordered launch groups (one launch per group of key tiles with disjoint query rows) over the kernel sweep's
    geometries: within the bound, and bitwise equal when run again."""
    for i, (name, regime) in enumerate(KO.sweep_cases()):
        geom = KO.geometry(name)
        dkv = torch.float32 if i % 2 else dtype
        first = KO.run_backward(geom, d, dtype, window, regime, "cuda", dkv_dtype=dkv, deterministic=True)
        again = KO.run_backward(geom, d, dtype, window, regime, "cuda", dkv_dtype=dkv, deterministic=True)
        for a, b in zip(first, again):
            assert torch.equal(a, b), f"{name} {regime}: ordered backward not bitwise reproducible"


@pytest.mark.filterwarnings("ignore:.*deterministic=True.*:RuntimeWarning")
@pytest.mark.parametrize("mode", ["strict", "fast"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_deterministic_api_world1(monkeypatch, mode, dtype):
    """``deterministic=True`` through the public API at world size 1 in both ``RFA_B200_DETERMINISTIC`` modes: within
    the bound; dK / dV (and, strict, dQ) bitwise reproducible."""
    monkeypatch.setenv("RFA_B200_DETERMINISTIC", mode)
    cases = [CP.Case("zigzag", 1, 1536, 4, 2, 128, dtype, batch=2),
             CP.Case("zigzag", 1, 1024, 8, 2, 64, dtype, window=(300, 0)),
             CP.Case("ring_varlen", 1, 1000, 4, 1, 128, dtype),
             CP.Case("ring", 1, 768, 4, 4, 64, dtype, causal=False, window=(200, 100))]
    for seed, case in enumerate(cases):
        plans = CP.build_plans(case)
        q, k, v, do = CP.make_inputs(case, 100 + seed, "cuda")
        runs = [CP.api_train(case, 0, q[0], k[0], v[0], do[0], deterministic=True) for _ in range(2)]
        torch.cuda.synchronize()
        keys = ("out", "lse", "dq", "dk", "dv") if mode == "strict" else ("out", "lse", "dk", "dv")
        for key in keys:
            assert torch.equal(runs[0][key], runs[1][key]), f"{case.name()} {mode}: {key} not bitwise reproducible"
        refs = CP.references(case, plans, q, k, v, do, "fused")
        CP.check(f"{case.name()} deterministic {mode}", runs[0], *refs[0], report=CP.report_key("fused", 1))
