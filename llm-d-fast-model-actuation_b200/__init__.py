"""H100-native sleep / wake / hot-swap weight-movement engine (host-side Python mirror).

The directory name follows the repo layout contract; import it as ``fma_b200`` (the loader
``fma_b200.py`` at the repo root registers this directory under that name).

Everything here sits ABOVE the C-ABI of ``libfma_b200.so`` (``include/fma_engine.h``).  There is
no CPU fallback: on a machine without a CUDA driver, creating an engine raises.
"""
from ._lib import (  # noqa: F401
    FMA_FLAG_KEEP_BACKUP,
    FMA_FLAG_VERIFY,
    FMA_KERNEL_LDG,
    FMA_KERNEL_TMA,
    FMA_MODE_AUTO,
    FMA_MODE_DIRECT,
    FMA_MODE_KERNEL,
    FMA_MODE_STAGED,
    FMA_PAGE_BYTES,
    FMA_TIER_HOST,
    FMA_TIER_LOCAL,
    FMA_TIER_PEER,
    FmaError,
    lib_path,
    load_library,
)
from .engine import Engine, EngineConfig, ParkingBuffer  # noqa: F401

__all__ = [
    "Engine",
    "EngineConfig",
    "ParkingBuffer",
    "FmaError",
    "lib_path",
    "load_library",
]
