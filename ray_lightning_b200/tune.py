"""Ray Tune integration surface (ray_lightning/tune.py:13-241).

OUT OF SCOPE for the GPU data path (HPO control plane; SURVEY.md §2.1 row 9).  ``ray.tune`` is
not installable here, so — like the reference when Tune is missing (ray_lightning/tune.py:13-27,
238-241) — the callbacks resolve to ``Unavailable`` and ``is_session_enabled()`` is False.  The
worker->driver queue they would use (session.py, util.process_results) is implemented and tested.
"""
from .util import Unavailable

try:  # pragma: no cover - ray.tune is not installable here
    from ray import tune
    from ray.tune import is_session_enabled
    from ray.tune.integration.pytorch_lightning import TuneCallback
    TUNE_INSTALLED = True
except ImportError:
    tune = None
    TuneCallback = Unavailable

    def is_session_enabled():
        return False

    get_tune_resources = Unavailable
    TUNE_INSTALLED = False

if TUNE_INSTALLED:  # pragma: no cover
    import os
    from .session import get_actor_rank, put_queue
    from .util import to_state_stream

    def get_tune_resources(num_workers: int = 1, num_cpus_per_worker: int = 1, use_gpu: bool = False,
                           cpus_per_worker=None):
        """1 head CPU bundle + one bundle per worker, PACKed (ray_lightning/tune.py:32-56)."""
        from ray.tune import PlacementGroupFactory
        if cpus_per_worker is not None:
            num_cpus_per_worker = cpus_per_worker
        bundles = [{"CPU": 1}] + [{"CPU": num_cpus_per_worker, "GPU": int(use_gpu)} for _ in range(num_workers)]
        return PlacementGroupFactory(bundles, strategy="PACK")

    class TuneReportCallback(TuneCallback):
        """Rank 0 queues ``tune.report(**metrics)`` for the driver (ray_lightning/tune.py:59-134)."""

        def __init__(self, metrics=None, on="validation_end"):
            super().__init__(on)
            self._metrics = [metrics] if isinstance(metrics, str) else metrics

        def _get_report_dict(self, trainer, pl_module):
            if trainer.sanity_checking:
                return None
            if not self._metrics:
                return {k: v.item() for k, v in trainer.callback_metrics.items()}
            names = self._metrics.items() if isinstance(self._metrics, dict) else ((k, k) for k in self._metrics)
            return {out: trainer.callback_metrics[src].item() for out, src in names}

        def _handle(self, trainer, pl_module):
            if get_actor_rank() == 0:
                report = self._get_report_dict(trainer, pl_module)
                if report is not None:
                    put_queue(lambda: tune.report(**report))

    class _TuneCheckpointCallback(TuneCallback):
        def __init__(self, filename="checkpoint", on="validation_end"):
            super().__init__(on)
            self._filename = filename

        @staticmethod
        def _create_checkpoint(stream, global_step, filename):
            with tune.checkpoint_dir(step=global_step) as d:
                with open(os.path.join(d, filename), "wb") as f:
                    f.write(stream)

        def _handle(self, trainer, pl_module):
            if trainer.sanity_checking:
                return
            stream = to_state_stream(trainer._checkpoint_connector.dump_checkpoint())
            step = trainer.global_step
            if get_actor_rank() == 0:
                put_queue(lambda: self._create_checkpoint(stream, step, self._filename))

    class TuneReportCheckpointCallback(TuneCallback):
        def __init__(self, metrics=None, filename="checkpoint", on="validation_end"):
            super().__init__(on)
            self._checkpoint = _TuneCheckpointCallback(filename, on)
            self._report = TuneReportCallback(metrics, on)

        def _handle(self, trainer, pl_module):
            self._checkpoint._handle(trainer, pl_module)
            self._report._handle(trainer, pl_module)
else:
    TuneReportCallback = Unavailable
    TuneReportCheckpointCallback = Unavailable
