"""H100-native MLS-MPM substep engine: drop-in for the P2G / grid update / G2P + constitutive hot
path of yuanming-hu/taichi_mpm behind a C-ABI (include/mpmb.h).  See DESIGN.md."""
from . import bgeo, capi, scenes  # noqa: F401
from .capi import Engine, MpmbError  # noqa: F401
from .mpm import MPM, MPM2D, LevelSet  # noqa: F401
from .async_mpm import AsyncMPM  # noqa: F401

__all__ = ["bgeo", "capi", "scenes", "Engine", "MpmbError", "MPM", "MPM2D", "LevelSet", "AsyncMPM"]
