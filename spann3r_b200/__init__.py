"""spann3r_b200 -- H100-native (sm_90a) implementation of Spann3R's per-frame forward path.

Public surface mirrors the reference: `Spann3R`, `SpatialMemory`, `AsymmetricCroCo3DStereo`
(spann3r/model.py, dust3r/model.py).  Importing the package does not need a GPU; running it does.
"""
from .model import AsymmetricCroCo3DStereo, SpatialMemory, Spann3R  # noqa: F401

__all__ = ["Spann3R", "SpatialMemory", "AsymmetricCroCo3DStereo"]
