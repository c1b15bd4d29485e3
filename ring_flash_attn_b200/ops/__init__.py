"""Compute ops: dense oracle, merge, plans, and the sm_90a kernels' Python bindings."""
from .merge import merge_partial, update_out_and_lse  # noqa: F401
from .lse_layout import flatten_varlen_lse, unflatten_varlen_lse  # noqa: F401
