"""khronos_b200 — H100-native active-window volumetric integrator for Khronos.

The product is the CUDA library ``khronos_b200/csrc/libkhronos_b200.so`` behind the C ABI of
``include/khronos_b200.h``; this package is the thin Python host mirror used by tests and bench.
There is no CPU fallback: creating a map without a CUDA device raises.
"""
from . import capi
from .capi import (Camera, Frame, FrameStats, IntegratorConfig, KbError, MapConfig, MapHandle,
                   MotionConfig, TrackingConfig, default_integrator_config, default_map_config,
                   default_motion_config, default_tracking_config, load_product_library)

_LIB = None


def lib():
    """The loaded product library (raises ImportError if it has not been built)."""
    global _LIB
    if _LIB is None:
        _LIB = load_product_library()
    return _LIB


def create_map(map_cfg, integ_cfg, tracking_cfg=None, motion_cfg=None, device=0) -> MapHandle:
    """Create a GPU map handle (kb_create). Raises KbError(KB_ERR_NO_DEVICE) without a GPU."""
    return MapHandle(lib(), "kb_", map_cfg, integ_cfg, tracking_cfg, motion_cfg, device)
