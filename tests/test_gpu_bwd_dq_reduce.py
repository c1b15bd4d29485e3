"""The sm_90a backward's per-warpgroup dQ reduce-add against the fp64 plan oracle (``tests/kernel_oracle.py``).

Each warpgroup stages and adds its own dQ columns, and the loader's tile iterator lives in shared memory.  These
cases walk the edges of that schedule: key-tile CTAs whose sweep has 1 to kStages + 1 query tiles (so the Q / dO ring
wraps), sweeps across query segments and across the query heads of a GQA group, ragged query and key lengths, both
head dims, with and without a sliding window; and ``deterministic=True`` runs that must agree bitwise."""
import pytest
import torch

import kernel_oracle as KO
import ring_flash_attn_b200 as rfa

pytestmark = pytest.mark.gpu

GEOMETRIES = [
    # one key tile, one query head: 1, 2, 3 (= kStages) and 4 query tiles in the sweep
    KO._one("tiles1", 64, 128, 1, 1, None),
    KO._one("tiles2", 128, 128, 2, 2, None),
    KO._one("tiles3", 192, 128, 1, 1, None),
    KO._one("tiles4", 256, 128, 2, 2, None),
    # ragged q_len and kv_rows
    KO._one("ragged_q65_k100", 65, 100, 1, 1, None),
    KO._one("ragged_q250_k300_causal", 250, 300, 2, 1, 60),
    # a GQA group of 4 query heads (32 / 8) in one sweep, ragged rows
    KO._one("gqa32_8_q130_k200", 130, 200, 32, 8, 90),
    # sweeps that cross query segments
    KO._g("two_segments", 300, 256, 4, 2, [(0, 150), (150, 150)],
          [(0, 0, 256, None, None), (1, 0, 256, 40, -100)]),
]


@pytest.fixture(autouse=True)
def _exact_fp32_matmul():
    """The precision-matched reference needs true fp32 GEMMs."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.mark.parametrize("window", [False, True], ids=["plain", "window"])
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("geom", GEOMETRIES, ids=[g["name"] for g in GEOMETRIES])
def test_backward_sweep_edges(geom, d, window):
    KO.run_backward(geom, d, torch.bfloat16, window, "randn", "cuda")


@pytest.mark.filterwarnings("ignore:.*deterministic=True.*:RuntimeWarning")
@pytest.mark.parametrize("d", [64, 128])
def test_deterministic_gqa_is_bitwise_reproducible(d):
    torch.manual_seed(1)
    B, S, H, HK = 1, 704, 32, 8
    q = torch.randn(B, S, H, d, device="cuda").to(torch.bfloat16)
    kv = torch.randn(B, S, 2, HK, d, device="cuda").to(torch.bfloat16)
    dout = torch.randn(B, S, H, d, device="cuda").to(torch.bfloat16)
    runs = []
    for _ in range(3):
        xs = [q.clone().requires_grad_(True), kv.clone().requires_grad_(True)]
        rfa.zigzag_ring_flash_attn_kvpacked_func(*xs, causal=True, deterministic=True).backward(dout)
        torch.cuda.synchronize()
        runs.append([x.grad for x in xs])
    for grads in runs[1:]:
        for g, g0 in zip(grads, runs[0]):
            assert torch.equal(g, g0)
