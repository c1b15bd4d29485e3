"""Every sm_90a attention kernel instantiation against the fp64 plan oracle, with a precision-matched error bound
(``tests/kernel_oracle.py``).  Hand-built plans go straight through ``attn_cuda.segments_forward`` /
``segments_backward``; the backward takes lse and delta from the fp64 oracle, so it is tested apart from the forward."""
import pytest
import torch

import kernel_oracle as KO
from ring_flash_attn_b200.ops import attn_cuda

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
HEAD_DIMS = [64, 128]


@pytest.fixture(autouse=True)
def _exact_fp32_matmul():
    """The precision-matched reference needs true fp32 GEMMs."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.mark.parametrize("direction", ["fwd", "bwd"])
@pytest.mark.parametrize("window", [False, True], ids=["plain", "window"])
@pytest.mark.parametrize("d", HEAD_DIMS)
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_kernel_sweep(dtype, d, window, direction):
    """One instantiation ({bf16, fp16} x head_dim x {plain, window} x {forward, backward}) over every geometry and
    value regime.  Backward cases alternate between fp32 and model-dtype dK / dV stores."""
    for i, (name, regime) in enumerate(KO.sweep_cases()):
        geom = KO.geometry(name)
        if direction == "fwd":
            KO.run_forward(geom, d, dtype, window, regime, "cuda")
        else:
            KO.run_backward(geom, d, dtype, window, regime, "cuda", dkv_dtype=torch.float32 if i % 2 else dtype)


@pytest.mark.parametrize("direction", ["fwd", "bwd"])
@pytest.mark.parametrize("window", [False, True], ids=["plain", "window"])
@pytest.mark.parametrize("d", HEAD_DIMS)
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_invisible_rows_change_nothing(dtype, d, window, direction):
    KO.run_invisibility(d, dtype, window, direction == "bwd", "cuda")


@pytest.mark.parametrize("d", HEAD_DIMS)
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_delta_and_dq_finalize(dtype, d):
    KO.run_delta_and_dq_finalize(dtype, d, "cuda")


FP8_GEOMETRIES = ["q65_k127_gqa8", "q384_k512_gqa2", "q512_k1024", "zigzag_adjacent", "diag-200_and_blind_chunk"]


@pytest.mark.parametrize("blocks", ["per_head", "block_scaled"])
@pytest.mark.parametrize("name", FP8_GEOMETRIES)
def test_fp8_forward_sweep(name, blocks):
    """e4m3 forward (head_dim 128, bf16 out) against the oracle on the dequantised inputs, P rounded to bf16."""
    KO.run_fp8_forward(KO.geometry(name), blocks, "cuda")
