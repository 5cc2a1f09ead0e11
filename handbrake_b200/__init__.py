"""handbrake_b200 -- H100-native (sm_90a) implementation of libhb's per-pixel
video-filter hot path (NLMeans, comb-detect, decomb/EEDI2, lapsharp) behind
libhb's own filter plugin interface.

The product is native code: `lib/libhbcu.so` (CUDA kernels + the C-ABI of
include/hbcu.h) and `lib/libhbcu_filters.so` (the hb_filter_object_t drop-ins in
C).  Python is only the test/bench harness around them.  There is no CPU
fallback anywhere: loading fails loudly when the libraries are missing.
"""
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
LIB_DIR = PKG_DIR / "lib"
LIBHBCU = LIB_DIR / "libhbcu.so"
LIBHBCU_FILTERS = LIB_DIR / "libhbcu_filters.so"


class NativeLibraryMissing(RuntimeError):
    pass


def require_native():
    for p in (LIBHBCU, LIBHBCU_FILTERS):
        if not p.exists():
            raise NativeLibraryMissing(
                f"{p} is missing: run `python -m handbrake_b200.build` (or __graft_entry__.build()). "
                "There is no CPU fallback.")
    return LIBHBCU, LIBHBCU_FILTERS


def filters():
    """FilterLib over the CUDA filter objects (hb_filter_nlmeans_cuda, ...)."""
    from .hblib import FilterLib
    require_native()
    return FilterLib(LIBHBCU_FILTERS)
