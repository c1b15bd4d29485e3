"""Every sm_90a split-KV decode kernel instantiation ({bf16, fp16} x head_dim {64, 128} x {native, e4m3 cache})
against the fp64 decode oracle, with the precision-matched error bound of ``tests/kernel_oracle.py``, over the
geometries and value regimes of ``tests/decode_oracle.py``; the append kernels' cache bytes on the way; and the
cross-rank combine on two GPUs."""
import pytest
import torch

import decode_oracle as DO
from dist_utils import run_distributed

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


@pytest.mark.parametrize("fp8", [False, True], ids=["native", "e4m3"])
@pytest.mark.parametrize("d", HEAD_DIMS)
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
def test_decode_sweep(dtype, d, fp8):
    """One instantiation of ``decode_kernel`` (and of the append kernel for its cache dtype) over every geometry and
    value regime."""
    for name, regime in DO.sweep_cases():
        DO.run_decode(DO.geometry(name, fp8=fp8), dtype, d, regime, "cuda")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("fp8", [False, True], ids=["native", "e4m3"])
def test_two_gpus_combine_matches_oracle(fp8):
    """The rank-partial combine (``decode_combine`` into fp32, then over the gathered partials) under the same bound,
    and bitwise the same result on both ranks."""
    run_distributed(DO.run_two_ranks, 2, fp8, "cuda", backend="nccl")
