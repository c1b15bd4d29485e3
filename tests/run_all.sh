#!/bin/bash
# Counterpart of the reference's test/test.sh (one torchrun per script on 8 GPUs): here everything is pytest.
#   CPU (no GPU needed): plans, host tables, gloo world 1/2/4/8, HF adapter, training example
#   GPU (H100):          kernels vs the fp32 oracle, fused NVLink path on 2/4/8 GPUs, fallback transports
set -e
cd "$(dirname "$0")/.."
python -c "import __graft_entry__ as g; g.build()"
python -m pytest tests -q -m "not gpu" "$@"
if python -c "import torch,sys; sys.exit(0 if torch.cuda.is_available() else 1)"; then
  python -m pytest tests -q -m gpu "$@"
fi
