"""RayHorovodLauncher — surface parity only.

The reference's Horovod launcher (ray_lightning/launchers/ray_horovod_launcher.py:37-277) drives
``horovod.ray.RayExecutor`` and calls ``hvd.init()`` in each worker (:192).  Horovod is not
installable in this image and is OUT OF SCOPE for the GPU data path (SURVEY.md §2.1 row 5b):
its gradient sync is a per-parameter allreduce-average — the same arithmetic contract
``RayStrategy``'s libb2d hook implements — so a Horovod user switches to ``RayStrategy``.  The
class keeps the reference's constructor and ``launch`` signature and fails loudly if used
without Horovod.
"""
from typing import Any, Callable

from .._compat import _Launcher, ray


class RayHorovodLauncher(_Launcher):
    def __init__(self, strategy) -> None:
        self._strategy = strategy
        self._executor = getattr(strategy, "executor", None)
        self._start_method = "ray"
        self.tune_queue = None
        if not ray.is_initialized():
            ray.init()

    def is_interactive_compatible(self) -> bool:
        return True

    @property
    def global_rank(self) -> int:
        return self._strategy.global_rank

    @property
    def local_rank(self) -> int:
        return self._strategy.local_rank

    @property
    def world_size(self) -> int:
        return self._strategy.world_size

    def launch(self, function: Callable, *args: Any, trainer=None, **kwargs: Any) -> Any:
        raise RuntimeError("Please intall Horovod to use this strategy. (Horovod is not available in this build; "
                           "RayStrategy(use_gpu=True) provides the same allreduce-average semantics on libb2d.)")
