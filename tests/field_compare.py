"""The comparison rules of the on-device checks, on the host.

``same_bits`` / ``count_wrong`` are the rule of the halo checks (``Elem<T>::differs`` in csrc/kernels/halo_stencil.cu,
``host_same`` in csrc/miniapps/halo.cu): an element is wrong iff its bit pattern differs from the reference's, unless
both are NaN, of any sign or payload (the GPU's and the host's canonical NaNs differ).  So a wrong sign of zero or a
flushed subnormal is wrong, and a NaN where a NaN is due is right.  ``torch.equal`` and ``!=`` get both cases wrong.

``count_far`` is the rule of ``count_mismatch`` (csrc/kernels/ring_allreduce.cu), the reference's
``|x - expected| < 1e-6`` check: the value widened to double, NaN counted.
"""
import numpy as np
import torch

_INT = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def wrong_mask(got: torch.Tensor, want: torch.Tensor) -> torch.Tensor:
    """Boolean mask of the wrong elements of ``got`` against ``want`` (same dtype and shape)."""
    if got.dtype != want.dtype or got.shape != want.shape:
        raise ValueError(f"compare like with like: {got.dtype}{tuple(got.shape)} vs {want.dtype}{tuple(want.shape)}")
    bits = _INT[got.element_size()]
    got, want = got.contiguous(), want.contiguous()
    differ = got.view(bits) != want.view(bits)
    if got.is_floating_point():
        differ &= ~(torch.isnan(got) & torch.isnan(want))
    return differ


def count_wrong(got: torch.Tensor, want: torch.Tensor) -> int:
    return int(wrong_mask(got, want).sum())


def same_bits(got: torch.Tensor, want: torch.Tensor) -> bool:
    return count_wrong(got, want) == 0


def count_far(values, expected: float) -> int:
    """Elements of ``values`` (array-like, any type that widens exactly or by rounding to double) that are not within
    1e-6 of ``expected``."""
    d = np.asarray(values, dtype=np.float64) - np.float64(expected)
    return int((~((d < 1e-6) & (d > -1e-6))).sum())
