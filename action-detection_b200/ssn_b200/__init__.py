"""ssn_b200 — host package of the H100-native SSN hot path (see DESIGN.md).

Importing this package loads libssn_b200.so; it raises ImportError if the CUDA extension has not
been built (there is deliberately no fallback path)."""
from . import _lib  # noqa: F401  (fails loudly when the .so is missing)
from ._lib import EXACT_FP32, FAST_FP16, EXACT_TC  # noqa: F401
