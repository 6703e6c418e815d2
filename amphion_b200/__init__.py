"""amphion_b200 — H100-native (sm_90a) vocoder-inference hot path for Amphion recipes.

Host code is Python with PyTorch tensors at the boundary; all arithmetic runs
in hand-written CUDA behind the C ABI declared in ``include/amphion_b200.h``
(``amphion_b200/libamphion_b200.so``).  There is no CPU path: every op raises
if the tensor is not on a CUDA device or the library is missing.
"""
__version__ = "0.1.0"

from . import _capi  # noqa: F401  (fails loudly if the CUDA library cannot be loaded/built)
