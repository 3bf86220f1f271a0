"""A minimal Lightning-shaped trainer: the slice of pytorch_lightning 1.6 that the strategies,
the launcher and the examples of this repo touch.

``pytorch_lightning`` is not installable in this image.  The reference's strategies subclass
PL's ``DDPSpawnStrategy`` and are driven by ``pl.Trainer`` (ray_lightning/ray_ddp.py:23,112-116);
what they need from PL is small and well defined: a Trainer whose ``fit`` goes through
``strategy.launcher.launch(trainer._fit_impl, model, trainer=trainer)``, a strategy base that keeps
``**ddp_kwargs`` / ``ddp_comm_hook`` / ``ddp_comm_state`` and builds
``DistributedDataParallel(model, device_ids=..., **ddp_kwargs)`` then registers the hook when the
root device is CUDA, samplers from ``strategy.distributed_sampler_kwargs``, callbacks, metrics,
checkpoints.  That is what this file provides — nothing else of Lightning (no loggers, no
precision plugins beyond bf16 autocast, no tuner, no CLI).  With the real package installed
``ray_lightning_b200._compat`` prefers it.
"""
import copy
import os
import random
from enum import Enum

import numpy as np
import torch
import torch.distributed as dist
from torch import nn
from torch.nn.parallel import DistributedDataParallel
from torch.utils.data import DataLoader, DistributedSampler


# ---- utilities ---------------------------------------------------------------------------------
class _RankZeroOnly:
    rank = 0

    def __call__(self, fn):
        def wrapped(*a, **k):
            if _RankZeroOnly.rank == 0:
                return fn(*a, **k)
        return wrapped


rank_zero_only = _RankZeroOnly()


def rank_zero_info(msg):
    if _RankZeroOnly.rank == 0 and os.environ.get("B2D_VERBOSE"):
        print(msg, flush=True)


rank_zero_debug = rank_zero_info
rank_zero_warn = rank_zero_info


def seed_everything(seed=None, workers=False):
    seed = int(seed if seed is not None else os.environ.get("PL_GLOBAL_SEED", 0))
    os.environ["PL_GLOBAL_SEED"] = str(seed)
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    return seed


def reset_seed():
    seed = os.environ.get("PL_GLOBAL_SEED")
    if seed is not None:
        seed_everything(int(seed))


def apply_to_collection(data, dtype, fn):
    if isinstance(data, dtype):
        return fn(data)
    if isinstance(data, dict):
        return {k: apply_to_collection(v, dtype, fn) for k, v in data.items()}
    if isinstance(data, (list, tuple)):
        return type(data)(apply_to_collection(v, dtype, fn) for v in data)
    return data


def move_data_to_device(batch, device):
    return apply_to_collection(batch, torch.Tensor, lambda t: t.to(device, non_blocking=True))


class TrainerStatus(str, Enum):
    INITIALIZING = "initializing"
    RUNNING = "running"
    FINISHED = "finished"
    INTERRUPTED = "interrupted"


class TrainerFn(str, Enum):
    FITTING = "fit"
    VALIDATING = "validate"
    TESTING = "test"
    PREDICTING = "predict"


class TrainerState:
    def __init__(self):
        self.status = TrainerStatus.INITIALIZING
        self.fn = None

    @property
    def finished(self):
        return self.status == TrainerStatus.FINISHED

    def __repr__(self):
        return "TrainerState(status=%s, fn=%s)" % (self.status, self.fn)


# ---- callbacks ---------------------------------------------------------------------------------
class Callback:
    def setup(self, trainer, pl_module, stage=None): pass
    def on_fit_start(self, trainer, pl_module): pass
    def on_train_start(self, trainer, pl_module): pass
    def on_train_epoch_start(self, trainer, pl_module): pass
    def on_train_batch_start(self, trainer, pl_module, batch, batch_idx): pass
    def on_train_batch_end(self, trainer, pl_module, outputs, batch, batch_idx): pass
    def on_train_epoch_end(self, trainer, pl_module): pass
    def on_validation_start(self, trainer, pl_module): pass
    def on_validation_end(self, trainer, pl_module): pass
    def on_test_start(self, trainer, pl_module): pass
    def on_test_end(self, trainer, pl_module): pass
    def on_train_end(self, trainer, pl_module): pass
    def on_fit_end(self, trainer, pl_module): pass
    def teardown(self, trainer, pl_module, stage=None): pass


class EarlyStopping(Callback):
    def __init__(self, monitor="val_loss", min_delta=0.0, patience=3, verbose=False, mode="min"):
        self.monitor, self.min_delta, self.patience, self.mode = monitor, min_delta, patience, mode
        self.wait_count, self.best = 0, None
        self.stopped_epoch = 0

    def on_validation_end(self, trainer, pl_module):
        if trainer.sanity_checking or self.monitor not in trainer.callback_metrics:
            return
        cur = float(trainer.callback_metrics[self.monitor])
        better = self.best is None or (cur < self.best - self.min_delta if self.mode == "min" else cur > self.best + self.min_delta)
        stop = False
        if better:
            self.best, self.wait_count = cur, 0
        else:
            self.wait_count += 1
            stop = self.wait_count >= self.patience
        # The monitored metric is per rank (the validation set is sharded by DistributedSampler and logged values
        # are not reduced), so ranks may disagree; a rank that left the loop alone would strand the others in
        # their next collective.  PL settles it with strategy.reduce_boolean_decision: stop if ANY rank wants to.
        stop = trainer.strategy.reduce_boolean_decision(stop, all=False)
        if stop:
            trainer.should_stop = True
            self.stopped_epoch = trainer.current_epoch


class ModelCheckpoint(Callback):
    """Saves one checkpoint (the latest, or the best by ``monitor``) at the end of every epoch."""

    def __init__(self, dirpath=None, filename=None, monitor=None, mode="min", save_top_k=1):
        self.dirpath, self.filename, self.monitor, self.mode = dirpath, filename, monitor, mode
        self.best_model_path = ""
        self.best_model_score = None

    def _path(self, trainer):
        d = self.dirpath or os.path.join(trainer.default_root_dir, "checkpoints")
        name = self.filename or "epoch=%d-step=%d" % (trainer.current_epoch, trainer.global_step)
        return os.path.join(d, name + ".ckpt")

    def on_train_epoch_end(self, trainer, pl_module):
        score = None
        save = True
        if self.monitor is not None and self.monitor in trainer.callback_metrics:
            score = float(trainer.callback_metrics[self.monitor])
            if self.best_model_score is not None:
                save = not (score >= self.best_model_score if self.mode == "min" else score <= self.best_model_score)
        # saving is collective (the sharded strategy consolidates optimizer state on every rank): rank 0 decides
        save = bool(trainer.strategy.broadcast(save, src=0))
        if not save:
            return
        path = self._path(trainer)
        if trainer.is_global_zero:
            old = self.best_model_path
            trainer.save_checkpoint(path)
            if old and old != path and os.path.exists(old):
                os.remove(old)
        else:
            trainer.strategy.optimizer_state_for_checkpoint(trainer)  # collective on every rank
        self.best_model_path, self.best_model_score = path, score


def _clip_algorithm(algorithm):
    """PL's GradClipAlgorithmType: "norm" (the default) or "value"."""
    if algorithm is None:
        return "norm"
    if algorithm not in ("norm", "value"):
        raise ValueError("gradient_clip_algorithm %r is invalid: allowed values are 'norm' and 'value'" % (algorithm,))
    return algorithm


# ---- module / datamodule ---------------------------------------------------------------------------
class LightningModule(nn.Module):
    def __init__(self):
        super().__init__()
        self.trainer = None
        self._hparams = {}
        self._current_fx = None

    # hooks users override
    def training_step(self, batch, batch_idx): raise NotImplementedError
    def configure_optimizers(self): raise NotImplementedError
    def on_save_checkpoint(self, checkpoint): pass

    def configure_gradient_clipping(self, optimizer, optimizer_idx, gradient_clip_val=None, gradient_clip_algorithm=None):
        """PL 1.6 hook, called after backward and before each optimizer step when the Trainer clips."""
        self.clip_gradients(optimizer, gradient_clip_val=gradient_clip_val, gradient_clip_algorithm=gradient_clip_algorithm)

    def clip_gradients(self, optimizer, gradient_clip_val=None, gradient_clip_algorithm=None):
        if gradient_clip_val is None or gradient_clip_val <= 0:
            return
        algorithm = _clip_algorithm(gradient_clip_algorithm)
        self.trainer.strategy.clip_gradients(optimizer, float(gradient_clip_val), algorithm)
    def on_load_checkpoint(self, checkpoint): pass
    def prepare_data(self): pass
    def setup(self, stage=None): pass

    @property
    def hparams(self):
        return self._hparams

    def save_hyperparameters(self, *args, **kw):
        import inspect
        frame = inspect.currentframe().f_back
        params = inspect.signature(type(self).__init__).parameters
        self._hparams = {k: frame.f_locals[k] for k in params if k != "self" and k in frame.f_locals}

    @property
    def device(self):
        try:
            return next(self.parameters()).device
        except StopIteration:
            return torch.device("cpu")

    @property
    def global_rank(self):
        return self.trainer.global_rank if self.trainer else 0

    def log(self, name, value, prog_bar=False, logger=True, on_step=None, on_epoch=None, sync_dist=False, **_kw):
        if self.trainer is not None:
            self.trainer._log(self._current_fx, name, value, on_step, on_epoch)

    def log_dict(self, d, **kw):
        for k, v in d.items():
            self.log(k, v, **kw)

    @classmethod
    def load_from_checkpoint(cls, checkpoint_path, map_location="cpu", **kwargs):
        ckpt = torch.load(checkpoint_path, map_location=map_location, weights_only=False)
        hp = dict(ckpt.get("hyper_parameters", {}))
        hp.update(kwargs)
        model = cls(**hp)
        model.load_state_dict(ckpt["state_dict"])
        model.on_load_checkpoint(ckpt)
        return model

    def __getstate__(self):
        d = dict(self.__dict__)
        d["trainer"] = None  # the trainer travels separately (ray_launcher.py:234-237)
        return d


class LightningDataModule:
    def prepare_data(self): pass
    def setup(self, stage=None): pass
    def train_dataloader(self): return None
    def val_dataloader(self): return None
    def test_dataloader(self): return None


# ---- strategies --------------------------------------------------------------------------------------
class _Launcher:
    def launch(self, function, *args, trainer=None, **kwargs):
        raise NotImplementedError

    @property
    def is_interactive_compatible(self):
        return False


class Strategy:
    strategy_name = "single"

    def __init__(self, accelerator=None, parallel_devices=None, cluster_environment=None, **_kw):
        self.accelerator = accelerator
        self.parallel_devices = parallel_devices
        self.cluster_environment = cluster_environment
        self._launcher = None
        self.model = None
        self.lightning_module = None
        self.optimizers, self.lr_schedulers = [], []
        self.precision = 32

    @property
    def launcher(self):
        return self._launcher

    def _configure_launcher(self):
        self._launcher = None

    @property
    def root_device(self):
        return torch.device("cpu")

    @property
    def is_global_zero(self):
        return self.global_rank == 0

    global_rank = 0
    local_rank = 0
    world_size = 1
    node_rank = 0

    @property
    def distributed_sampler_kwargs(self):
        return None

    def setup_environment(self):
        pass

    def connect(self, model):
        self.lightning_module = model
        self.model = model

    def model_to_device(self):
        self.lightning_module.to(self.root_device)

    def setup_optimizers(self, trainer):
        opt = self.lightning_module.configure_optimizers()
        scheds = []
        if isinstance(opt, tuple) and len(opt) == 2:
            opt, scheds = opt
        if isinstance(opt, dict):
            scheds = [opt["lr_scheduler"]] if "lr_scheduler" in opt else []
            opt = opt["optimizer"]
        self.optimizers = list(opt) if isinstance(opt, (list, tuple)) else [opt]
        self.lr_schedulers = list(scheds) if isinstance(scheds, (list, tuple)) else [scheds]

    def setup(self, trainer):
        self.model_to_device()
        if trainer.state.fn == TrainerFn.FITTING:
            self.setup_optimizers(trainer)

    def _autocast(self):
        if self.precision in ("bf16", "bf16-mixed"):
            return torch.autocast(self.root_device.type, dtype=torch.bfloat16)
        import contextlib
        return contextlib.nullcontext()

    def training_step(self, *args):
        with self._autocast():
            return self.model(*args) if self.model is not self.lightning_module else self.lightning_module.training_step(*args)

    def validation_step(self, *args):
        with self._autocast():
            return self.lightning_module.validation_step(*args)

    def test_step(self, *args):
        with self._autocast():
            return self.lightning_module.test_step(*args)

    def backward(self, loss):
        loss.backward()

    def optimizer_step(self, optimizer):
        optimizer.step()

    def clip_gradients(self, optimizer, clip_val, algorithm="norm"):
        """torch's clip_grad_norm_ (norm_type 2) or clip_grad_value_ over the parameters of the optimizer's groups."""
        params = [p for g in optimizer.param_groups for p in g["params"]]
        if algorithm == "value":
            torch.nn.utils.clip_grad_value_(params, clip_val)
        else:
            torch.nn.utils.clip_grad_norm_(params, clip_val)

    def barrier(self, name=None):
        pass

    def broadcast(self, obj, src=0):
        return obj

    def reduce_boolean_decision(self, decision, all=True):
        """PL's Strategy.reduce_boolean_decision: every rank leaves with the same answer (all / any)."""
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
            return bool(decision)
        t = torch.tensor([int(bool(decision))], device=self.root_device)
        dist.all_reduce(t)
        return bool(int(t) == dist.get_world_size()) if all else bool(int(t) > 0)

    def reduce(self, tensor, group=None, reduce_op="mean"):
        return tensor

    def optimizer_state_for_checkpoint(self, trainer):
        return [o.state_dict() for o in self.optimizers]

    def teardown(self):
        pass


class ParallelStrategy(Strategy):
    pass


class _LightningDistributedModule(nn.Module):
    """What DDP wraps: forward == LightningModule.training_step (PL's LightningDistributedModule)."""

    def __init__(self, pl_module):
        super().__init__()
        self.module = pl_module

    def forward(self, *args):
        return self.module.training_step(*args)


class DDPSpawnStrategy(ParallelStrategy):
    """PL-1.6 DDPSpawnStrategy, reduced to what sits between RayStrategy and torch DDP."""

    strategy_name = "ddp_spawn"

    def __init__(self, accelerator=None, parallel_devices=None, cluster_environment=None, checkpoint_io=None,
                 precision_plugin=None, ddp_comm_state=None, ddp_comm_hook=None, ddp_comm_wrapper=None, **kwargs):
        super().__init__(accelerator=accelerator, parallel_devices=parallel_devices,
                         cluster_environment=cluster_environment)
        self._ddp_kwargs = kwargs
        self._ddp_comm_state = ddp_comm_state
        self._ddp_comm_hook = ddp_comm_hook
        self._ddp_comm_wrapper = ddp_comm_wrapper
        self._process_group_backend = None

    @property
    def torch_distributed_backend(self):
        return self._process_group_backend or self._get_process_group_backend()

    def _get_process_group_backend(self):
        return os.environ.get("PL_TORCH_DISTRIBUTED_BACKEND") or ("nccl" if self.root_device.type == "cuda" else "gloo")

    def set_world_ranks(self, process_idx=0):
        pass

    def determine_ddp_device_ids(self):
        return None if self.root_device.type == "cpu" else [self.root_device.index]

    def pre_configure_ddp(self):
        # PL 1.6 defaults find_unused_parameters to True (ray_lightning/tests/test_ddp.py:311-323)
        self._ddp_kwargs["find_unused_parameters"] = self._ddp_kwargs.get("find_unused_parameters", True)

    def configure_ddp(self):
        self.pre_configure_ddp()
        self.model = DistributedDataParallel(_LightningDistributedModule(self.lightning_module),
                                             device_ids=self.determine_ddp_device_ids(), **self._ddp_kwargs)
        self._register_ddp_hooks()

    def _register_ddp_hooks(self):
        if self.root_device.type == "cuda" and self._ddp_comm_hook is not None:
            hook = self._ddp_comm_hook
            if self._ddp_comm_wrapper is not None:
                hook = self._ddp_comm_wrapper(hook)
            self.model.register_comm_hook(self._ddp_comm_state, hook)

    def configure_sync_batchnorm(self, model):
        return torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)

    def setup(self, trainer):
        self.model_to_device()
        # PL 1.6 order: convert after moving the model, before wrapping it
        if getattr(self, "sync_batchnorm", False):
            self.model = self.configure_sync_batchnorm(self.model)
        if trainer.state.fn == TrainerFn.FITTING:
            self.configure_ddp()
            self.setup_optimizers(trainer)

    def training_step(self, *args):
        with self._autocast():
            return self.model(*args)

    def barrier(self, name=None):
        if dist.is_available() and dist.is_initialized():
            dist.barrier()

    def broadcast(self, obj, src=0):
        if not (dist.is_available() and dist.is_initialized()):
            return obj
        box = [obj]
        dist.broadcast_object_list(box, src=src)
        return box[0]

    def reduce_boolean_decision(self, decision, all=True):
        """PL's Strategy.reduce_boolean_decision: every rank leaves with the same answer (all / any)."""
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
            return bool(decision)
        t = torch.tensor([int(bool(decision))], device=self.root_device)
        dist.all_reduce(t)
        return bool(int(t) == dist.get_world_size()) if all else bool(int(t) > 0)

    def reduce(self, tensor, group=None, reduce_op="mean"):
        if not (dist.is_available() and dist.is_initialized()) or not isinstance(tensor, torch.Tensor):
            return tensor
        t = tensor.detach().clone().to(self.root_device)
        dist.all_reduce(t)
        return t / dist.get_world_size() if reduce_op in ("mean", "avg") else t

    def teardown(self):
        self.model = None
        if dist.is_available() and dist.is_initialized() and getattr(self, "_is_remote", False):
            dist.destroy_process_group()


class DDPSpawnShardedStrategy(DDPSpawnStrategy):
    strategy_name = "ddp_sharded_spawn"


class HorovodStrategy(ParallelStrategy):
    strategy_name = "horovod"

    def join(self):
        pass


# ---- trainer ------------------------------------------------------------------------------------------
class _DataConnector:
    def __init__(self, trainer):
        self.trainer = trainer

    def prepare_data(self):
        t = self.trainer
        if t.datamodule is not None:
            t.datamodule.prepare_data()
        if t.lightning_module is not None:
            t.lightning_module.prepare_data()


class _CheckpointConnector:
    def __init__(self, trainer):
        self.trainer = trainer

    def dump_checkpoint(self):
        t = self.trainer
        m = t.lightning_module
        ckpt = {"epoch": t.current_epoch, "global_step": t.global_step,
                "state_dict": {k: v.detach().cpu() for k, v in m.state_dict().items()},
                "hyper_parameters": dict(getattr(m, "_hparams", {})),
                "optimizer_states": t.strategy.optimizer_state_for_checkpoint(t),
                "lr_schedulers": [s.state_dict() for s in t.strategy.lr_schedulers]}
        m.on_save_checkpoint(ckpt)
        return ckpt


class Trainer:
    def __init__(self, default_root_dir=None, callbacks=None, strategy=None, max_epochs=1, max_steps=-1,
                 limit_train_batches=1.0, limit_val_batches=1.0, limit_test_batches=1.0, enable_progress_bar=False,
                 checkpoint_callback=None, enable_checkpointing=True, precision=32, num_sanity_val_steps=0,
                 resume_from_checkpoint=None, reload_dataloaders_every_n_epochs=0, gpus=None, logger=None,
                 progress_bar_refresh_rate=None, log_every_n_steps=50, sync_batchnorm=False, gradient_clip_val=None,
                 gradient_clip_algorithm=None, **_ignored):
        self.default_root_dir = str(default_root_dir) if default_root_dir is not None else os.getcwd()
        self.callbacks = list(callbacks or [])
        if checkpoint_callback is not None:
            enable_checkpointing = bool(checkpoint_callback)
        if enable_checkpointing and not any(isinstance(c, ModelCheckpoint) for c in self.callbacks):
            self.callbacks.append(ModelCheckpoint())
        self.strategy = strategy if strategy is not None else Strategy()
        self.strategy.precision = precision
        self.strategy.sync_batchnorm = bool(sync_batchnorm)
        self.gradient_clip_algorithm = _clip_algorithm(gradient_clip_algorithm)
        self.gradient_clip_val = gradient_clip_val
        self.max_epochs, self.max_steps = max_epochs, max_steps
        self.limit_train_batches, self.limit_val_batches, self.limit_test_batches = \
            limit_train_batches, limit_val_batches, limit_test_batches
        self.precision = precision
        self.resume_from_checkpoint = resume_from_checkpoint
        self.state = TrainerState()
        self.callback_metrics, self.logged_metrics = {}, {}
        self.current_epoch, self.global_step = 0, 0
        self.should_stop = False
        self.sanity_checking = False
        self.model = None
        self.datamodule = None
        self.train_dataloader = None
        self.val_dataloaders, self.test_dataloaders = None, None
        self._epoch_acc = {}
        self._data_connector = _DataConnector(self)
        self._checkpoint_connector = _CheckpointConnector(self)
        self._ckpt_path = None
        self.strategy._configure_launcher()

    # -- properties
    @property
    def lightning_module(self):
        m = self.model
        if isinstance(m, LightningModule) or m is None:
            return m if m is not None else self.strategy.lightning_module
        return self.strategy.lightning_module

    @property
    def checkpoint_callback(self):
        for c in self.callbacks:
            if isinstance(c, ModelCheckpoint):
                return c
        return None

    @property
    def global_rank(self):
        return self.strategy.global_rank

    @property
    def local_rank(self):
        return self.strategy.local_rank

    @property
    def world_size(self):
        return self.strategy.world_size

    @property
    def is_global_zero(self):
        return self.strategy.global_rank == 0

    @property
    def optimizers(self):
        return self.strategy.optimizers

    # -- logging (names fork into _step/_epoch like PL's ResultCollection)
    def _log(self, fx, name, value, on_step, on_epoch):
        v = value.detach().float().cpu() if isinstance(value, torch.Tensor) else torch.tensor(float(value))
        if on_step is None:
            on_step = fx == "training_step"
        if on_epoch is None:
            on_epoch = fx != "training_step"
        if on_step and on_epoch:
            self.logged_metrics[name + "_step"] = v
            self._epoch_acc.setdefault(name, {"vals": [], "fork": True})["vals"].append(v)
        elif on_step:
            self.logged_metrics[name] = v
            self.callback_metrics[name] = v
        elif on_epoch:
            if fx is not None and fx.endswith("epoch_end"):
                self.logged_metrics[name] = v
                self.callback_metrics[name] = v
            else:
                self._epoch_acc.setdefault(name, {"vals": [], "fork": False})["vals"].append(v)

    def _flush_epoch_metrics(self):
        for name, acc in self._epoch_acc.items():
            mean = torch.stack(acc["vals"]).mean()
            if acc["fork"]:
                self.logged_metrics[name + "_epoch"] = mean
                self.callback_metrics[name + "_epoch"] = mean
                self.callback_metrics[name] = mean
            else:
                self.logged_metrics[name] = mean
                self.callback_metrics[name] = mean
        self._epoch_acc = {}

    # -- entry points
    def _call_and_handle_interrupt(self, fn, *args, **kwargs):
        if self.strategy.launcher is not None:
            return self.strategy.launcher.launch(fn, *args, trainer=self, **kwargs)
        return fn(*args, **kwargs)

    def fit(self, model, train_dataloaders=None, val_dataloaders=None, datamodule=None, ckpt_path=None):
        if isinstance(train_dataloaders, LightningDataModule):
            datamodule, train_dataloaders = train_dataloaders, None
        self.model = model
        self.strategy.lightning_module = model
        self.state.fn, self.state.status = TrainerFn.FITTING, TrainerStatus.RUNNING
        return self._call_and_handle_interrupt(self._fit_impl, model, train_dataloaders, val_dataloaders, datamodule,
                                               ckpt_path or self.resume_from_checkpoint)

    def test(self, model=None, dataloaders=None, datamodule=None, ckpt_path=None):
        model = model if model is not None else self.lightning_module
        self.model = model
        self.strategy.lightning_module = model
        self.state.fn, self.state.status = TrainerFn.TESTING, TrainerStatus.RUNNING
        return self._call_and_handle_interrupt(self._test_impl, model, dataloaders, datamodule, ckpt_path)

    def save_checkpoint(self, path):
        ckpt = self._checkpoint_connector.dump_checkpoint()
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        torch.save(ckpt, path)

    # -- implementation (runs inside the worker when a launcher is configured)
    def _attach(self, model, datamodule):
        self.model = model
        self.datamodule = datamodule
        model.trainer = self
        self.strategy.connect(model)

    def _loader(self, fn_name, model, datamodule, explicit, shuffle):
        dl = explicit
        if dl is None and datamodule is not None:
            dl = getattr(datamodule, fn_name)()
        if dl is None and hasattr(model, fn_name):
            dl = getattr(model, fn_name)()
        if dl is None:
            return None
        kw = self.strategy.distributed_sampler_kwargs
        if kw is not None and isinstance(dl, DataLoader) and not isinstance(dl.sampler, DistributedSampler):
            sampler = DistributedSampler(dl.dataset, shuffle=shuffle, **kw)
            dl = DataLoader(dl.dataset, batch_size=dl.batch_size, sampler=sampler, num_workers=dl.num_workers,
                            collate_fn=dl.collate_fn, pin_memory=dl.pin_memory, drop_last=dl.drop_last)
        return dl

    @staticmethod
    def _limit(limit, loader):
        if isinstance(limit, float):
            try:
                return max(1, int(len(loader) * limit)) if limit < 1.0 else None
            except TypeError:
                return None
        return int(limit)

    def _call(self, hook, *args):
        for c in self.callbacks:
            getattr(c, hook)(self, self.lightning_module, *args)

    def _fit_impl(self, model, train_dataloaders=None, val_dataloaders=None, datamodule=None, ckpt_path=None):
        self._attach(model, datamodule)
        if datamodule is not None:
            datamodule.setup("fit")
        model.setup("fit")
        self.strategy.setup_environment()
        self.strategy.setup(self)
        if ckpt_path:
            self._restore(ckpt_path)
        for c in self.callbacks:
            c.setup(self, model, "fit")
        self.train_dataloader = self._loader("train_dataloader", model, datamodule, train_dataloaders, True)
        vdl = self._loader("val_dataloader", model, datamodule, val_dataloaders, False)
        self.val_dataloaders = [vdl] if vdl is not None else []
        self._call("on_fit_start")
        self._call("on_train_start")
        dev = self.strategy.root_device
        start_epoch = self.current_epoch
        for epoch in range(start_epoch, self.max_epochs):
            self.current_epoch = epoch
            model.train()
            self._call("on_train_epoch_start")
            sampler = getattr(self.train_dataloader, "sampler", None)
            if isinstance(sampler, DistributedSampler):
                sampler.set_epoch(epoch)
            outputs = []
            lim = self._limit(self.limit_train_batches, self.train_dataloader)
            for batch_idx, batch in enumerate(self.train_dataloader):
                if lim is not None and batch_idx >= lim:
                    break
                batch = move_data_to_device(batch, dev)
                self._call("on_train_batch_start", batch, batch_idx)
                for opt in self.strategy.optimizers:
                    opt.zero_grad()
                model._current_fx = "training_step"
                out = self.strategy.training_step(batch, batch_idx)
                loss = out["loss"] if isinstance(out, dict) else out
                self.strategy.backward(loss)
                if self.gradient_clip_val is not None and self.gradient_clip_val > 0:
                    for i, opt in enumerate(self.strategy.optimizers):
                        model.configure_gradient_clipping(opt, i, gradient_clip_val=self.gradient_clip_val,
                                                          gradient_clip_algorithm=self.gradient_clip_algorithm)
                for opt in self.strategy.optimizers:
                    self.strategy.optimizer_step(opt)
                self.global_step += 1
                outputs.append({"loss": loss.detach()} if not isinstance(out, dict) else
                               {k: (v.detach() if isinstance(v, torch.Tensor) else v) for k, v in out.items()})
                self._call("on_train_batch_end", outputs[-1], batch, batch_idx)
                if 0 < self.max_steps <= self.global_step:
                    self.should_stop = True
                    break
            if self.val_dataloaders:
                self._eval_loop(model, self.val_dataloaders[0], "validation", self.limit_val_batches, dev)
            if hasattr(model, "training_epoch_end"):
                model._current_fx = "training_epoch_end"
                model.training_epoch_end(outputs)
            self._flush_epoch_metrics()
            for s in self.strategy.lr_schedulers:
                s.step()
            self._call("on_train_epoch_end")
            if self.should_stop:
                break
        self._call("on_train_end")
        self._call("on_fit_end")
        self.state.status = TrainerStatus.FINISHED
        return None

    def _eval_loop(self, model, loader, kind, limit, dev):
        model.eval()
        self._call("on_%s_start" % kind)
        outputs = []
        lim = self._limit(limit, loader)
        with torch.no_grad():
            for batch_idx, batch in enumerate(loader):
                if lim is not None and batch_idx >= lim:
                    break
                batch = move_data_to_device(batch, dev)
                model._current_fx = "%s_step" % kind
                step = self.strategy.validation_step if kind == "validation" else self.strategy.test_step
                outputs.append(step(batch, batch_idx))
            end = "%s_epoch_end" % kind
            if hasattr(model, end):
                model._current_fx = end
                getattr(model, end)(outputs)
        self._flush_epoch_metrics()
        self._call("on_%s_end" % kind)
        model.train()
        return outputs

    def _test_impl(self, model, dataloaders=None, datamodule=None, ckpt_path=None):
        self._attach(model, datamodule)
        if datamodule is not None:
            datamodule.setup("test")
        self.strategy.setup_environment()
        self.strategy.setup(self)
        if ckpt_path:
            self._restore(ckpt_path, weights_only=True)
        tdl = self._loader("test_dataloader", model, datamodule, dataloaders, False)
        self.test_dataloaders = [tdl]
        self._eval_loop(model, tdl, "test", self.limit_test_batches, self.strategy.root_device)
        self.state.status = TrainerStatus.FINISHED
        return [dict(self.callback_metrics)]

    def _restore(self, path, weights_only=False):
        ckpt = torch.load(path, map_location="cpu", weights_only=False)
        self.lightning_module.load_state_dict(ckpt["state_dict"])
        self.lightning_module.on_load_checkpoint(ckpt)
        if weights_only:
            return
        self.current_epoch = int(ckpt.get("epoch", -1)) + 1
        self.global_step = int(ckpt.get("global_step", 0))
        self.strategy.load_optimizer_state(ckpt.get("optimizer_states"))


def _load_optimizer_state(self, states):
    if not states:
        return
    for opt, st in zip(self.optimizers, states):
        try:
            opt.load_state_dict(copy.deepcopy(st))
        except Exception as e:   # never silently: a resume that drops the optimizer state trains differently
            import warnings
            warnings.warn("optimizer state of %s could not be restored from the checkpoint (%r): weights resume, "
                          "optimizer state restarts" % (type(opt).__name__, e))


Strategy.load_optimizer_state = _load_optimizer_state
