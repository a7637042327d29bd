"""fastga_b200 -- H100-native (sm_90a) implementation of FastGA's seed-and-extend hot path.

The product is the C-ABI shared library ``libfastga_b200.so`` (include/fastga_b200.h); this
package is the thin Python host side used by tests and bench.py: a ctypes binding (``lib``),
readers for the reference's on-disk formats (``formats``) and the synthetic-genome generator
(``synth``).  There is no CPU fallback: every op raises if the CUDA library is missing.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# FGB_LIB: an alternative build of the SAME library (tuning variants made by profiles/build_variant.sh)
LIB_PATH = os.environ.get("FGB_LIB") or os.path.join(_HERE, "libfastga_b200.so")
_lib = None


class LibraryMissing(RuntimeError):
    pass


def load_library():
    """Loads the in-tree CUDA library; fails loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise LibraryMissing(
                "fastga_b200: %s not found -- run `python __graft_entry__.py` (build()) first; "
                "there is no CPU fallback" % LIB_PATH)
        from .lib import bind
        L = ctypes.CDLL(LIB_PATH)
        bind(L)
        _lib = L
    return _lib
