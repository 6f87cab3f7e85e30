"""madstereo — Python host of the H100-native self-adaptive stereo engine (libmadstereo.so).

The public, reference-compatible API lives in the sibling packages `Nets`, `Sampler`, `Losses`,
`Data_utils` (same module and function names as the reference repo); this package holds the ctypes
binding (`_lib`), the engine handle (`engine`), eager ops (`ops`), the adaptation loop (`adaptation`)
and synthetic data (`synthetic`).
"""
from ._lib import MadStereoError, LIB_PATH  # noqa: F401
