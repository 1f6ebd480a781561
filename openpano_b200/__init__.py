"""openpano_b200 — H100-native SIFT + match + blend engine behind the call
surface of ppwwyyxx/OpenPano's hot path.  The compute lives in
libpano_b200.so (hand-written sm_90a CUDA, C ABI in include/pano_b200.h);
this package is the ctypes binding plus the synthetic-input generator.
Importing `openpano_b200.capi` fails loudly when the library is not built."""
from ._abi import PanoParams, default_params  # noqa: F401

__all__ = ["PanoParams", "default_params"]
