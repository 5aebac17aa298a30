"""Python entry points of the sm_90a kernels (csrc/kernels).  All ops fail loudly
if the native extension is missing — there is no eager/PyTorch fallback."""
from .p2p import copy, fill_pattern, verify_pattern  # noqa: F401
from .fused import triad_put, triad_reference  # noqa: F401
from .gemm import (allgather_gemm, gemm_all_to_all, gemm_put, gemm_reduce_scatter,  # noqa: F401
                   gemm_reference)
from .halo import stencil_step, stencil_step_reference  # noqa: F401
