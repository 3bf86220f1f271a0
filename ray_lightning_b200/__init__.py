"""ray_lightning_b200 — an H100-native (sm_90a) DDP gradient-sync path behind ray_lightning's plugin API.

Public surface == the reference's (ray_lightning/__init__.py:1-5)."""
from .ray_ddp import RayStrategy
from .ray_ddp_sharded import RayShardedStrategy
from .ray_horovod import HorovodRayStrategy

__all__ = ["RayStrategy", "HorovodRayStrategy", "RayShardedStrategy"]
__version__ = "0.1.0"
