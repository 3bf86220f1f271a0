"""Gradient clipping on the H100: the global-norm entry points on loopback ranks against the NumPy restatement (bit for
bit) and torch's clip_grad_norm_ (tolerance), the scaled fused step, clip + step without host synchronisation, worker
processes against torch on the averaged gradients, and Trainer.fit(gradient_clip_val=...) through both strategies."""
import os
import socket
import warnings
from contextlib import closing

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import clip_ref as ref
from ray_lightning_b200 import RayShardedStrategy, RayStrategy
from ray_lightning_b200._compat import Callback, ray
from utils import BoringModel, RandomDataset, get_trainer

pytestmark = pytest.mark.gpu


def _bits(x):
    return np.asarray(x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else x, np.float32).view(np.uint32)


def _shards(world, seed, special=None):
    """Rank 0 has more tiles than the library's block cap (257 x 4096 + 5 elements), the last rank owns nothing."""
    g = torch.Generator().manual_seed(seed)
    sizes = [257 * 4096 + 5] + [1000 * r + 8 for r in range(1, world)]
    sizes[-1] = 0
    xs = [torch.randn(n, generator=g) * 2.0 ** -r for r, n in enumerate(sizes)]
    if special is not None:
        xs[0][3] = special
    return [x.cuda() for x in xs]


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_loopback_clip_norm_matches_the_restatement(world):
    from ray_lightning_b200.comm import LoopbackGroup
    g = LoopbackGroup(world, 0, arena_bytes=16 << 20, timeout_ms=20000)
    try:
        off = g.clip_register()
        assert g.clip_register() == off                       # idempotent
        for call, (max_norm, special) in enumerate([(1.0, None), (1e9, None), (0.5, float("inf")), (1.0, float("nan"))]):
            xs = _shards(world, seed=call, special=special)
            norms = [torch.full((1,), -1.0, device="cuda") for _ in range(world)]
            coefs = [torch.full((1,), -1.0, device="cuda") for _ in range(world)]
            g.clip_norm_(xs, max_norm, norms, coefs)           # two calls in a row without a step use both generations
            g.synchronize()
            want_n, want_c = ref.norm_coef([ref.partial(x.cpu().numpy()) for x in xs], max_norm)
            for r in range(world):
                assert _bits(norms[r]) == _bits(norms[0]) and _bits(coefs[r]) == _bits(coefs[0]), (call, r)
                if special is not None and np.isnan(special):    # the device's NaN payload is not numpy's
                    assert torch.isnan(norms[r]).all() and torch.isnan(coefs[r]).all()
                else:
                    assert _bits(norms[r]) == _bits([want_n]) and _bits(coefs[r]) == _bits([want_c]), (call, r)
            if special is None:
                full = torch.cat(xs).requires_grad_()
                full.grad = full.detach().clone()
                torch_norm = torch.nn.utils.clip_grad_norm_([full], max_norm)
                torch.testing.assert_close(norms[0][0], torch_norm, rtol=1e-5, atol=0)
                torch.testing.assert_close(full.grad, torch.cat(xs) * coefs[0], rtol=1e-6, atol=0)
            elif special == float("inf"):
                assert torch.isinf(norms[0]).all() and float(coefs[0]) == 0.0
            else:
                assert torch.isnan(norms[0]).all() and torch.isnan(coefs[0]).all()
    finally:
        g.close()


@pytest.mark.parametrize("world", [2, 4])
def test_scaled_fused_step_equals_the_fused_step_on_premultiplied_gradients(world):
    from ray_lightning_b200.comm import LoopbackGroup
    shard = [0]
    for r in range(world):
        shard.append(shard[-1] + 4096 * (r + 1))
    total = shard[-1]
    n_own = [shard[r + 1] - shard[r] for r in range(world)]
    gen = torch.Generator().manual_seed(7)
    p0 = torch.randn(total, generator=gen).cuda()
    grads = [torch.randn(n, generator=gen).cuda() for n in n_own]
    coef = torch.tensor([0.3712], device="cuda")
    results = []
    for scaled in (True, False):
        g = LoopbackGroup(world, 0, arena_bytes=16 << 20, timeout_ms=20000)
        try:
            params = [rk.arena_tensor(total) for rk in g.ranks]
            for p in params:
                p.copy_(p0)
            m = [torch.full((n,), 0.01, device="cuda") for n in n_own]
            v = [torch.full((n,), 0.02, device="cuda") for n in n_own]
            red = [x.clone() if scaled else x * coef for x in grads]
            groups = [[(0, n, dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, step=3, adamw=1))]
                      for n in n_own]
            torch.cuda.synchronize()
            g.adam_push_(params, m, v, red, shard, groups, grad_scale=[coef] * world if scaled else None)
            g.synchronize()
            results.append([t.clone() for t in params + m + v])
        finally:
            g.close()
    for a, b in zip(*results):
        assert torch.equal(a, b)


def test_clip_and_step_need_no_host_synchronisation():
    """One rank of a loopback group as the ShardedOptimizer's communicator: after the first (registering) clip, a
    backward + clip_grad_norm + step raises nothing under set_sync_debug_mode("error")."""
    from ray_lightning_b200.comm import LoopbackGroup
    from ray_lightning_b200.sharded import FlatShards, ShardedOptimizer
    g = LoopbackGroup(1, 0, arena_bytes=16 << 20, timeout_ms=20000)
    try:
        torch.manual_seed(0)
        model = torch.nn.Sequential(torch.nn.Linear(64, 256), torch.nn.Tanh(), torch.nn.Linear(256, 8)).cuda()
        shards = FlatShards(model, g.ranks[0], wire="fp32", reduce_bucket_mb=0.01)
        sopt = ShardedOptimizer(torch.optim.Adam(model.parameters(), lr=1e-3), shards, wire="fp32",
                                stream=torch.cuda.Stream(priority=-1))
        x, y = torch.randn(32, 64, device="cuda"), torch.randn(32, 8, device="cuda")

        def step():
            sopt.zero_grad()
            torch.nn.functional.mse_loss(model(x), y).backward()
            n = sopt.clip_grad_norm(1e-3)
            sopt.step()
            return n

        step()
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            norm = step()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert float(norm) > 1e-3
    finally:
        g.close()


# ---- worker processes, gloo control plane -------------------------------------------------------------------------
def _port():
    with closing(socket.socket(socket.AF_INET, socket.SOCK_STREAM)) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _net():
    return torch.nn.Sequential(torch.nn.Linear(24, 300), torch.nn.Tanh(), torch.nn.Linear(300, 40), torch.nn.Tanh(),
                               torch.nn.Linear(40, 5))


_MK = {"adam": lambda ps: torch.optim.Adam(ps, lr=1e-2),
       "adamw": lambda ps: torch.optim.AdamW(ps, lr=1e-2, weight_decay=0.05),
       "sgd_momentum": lambda ps: torch.optim.SGD(ps, lr=0.05, momentum=0.9)}


def _mp_worker(rank, world, port, ret):
    import torch.distributed as dist
    from ray_lightning_b200.comm import Communicator
    from ray_lightning_b200.sharded import FlatShards, ShardedOptimizer
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world, init_method="env://")
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    res = {}
    try:
        data = [(torch.randn(16, 24, generator=torch.Generator().manual_seed(10 + r)),
                 torch.randn(16, 5, generator=torch.Generator().manual_seed(20 + r))) for r in range(world)]
        max_norm = 0.02
        for name, mk in _MK.items():
            torch.manual_seed(0)
            ref_model = _net().to(dev)
            torch.manual_seed(0)
            model = _net().to(dev)
            ref_opt = mk(ref_model.parameters())
            for r in range(world):
                x, y = data[r]
                (torch.nn.functional.mse_loss(ref_model(x.to(dev)), y.to(dev)) / world).backward()
            ref_norm = torch.nn.utils.clip_grad_norm_(ref_model.parameters(), max_norm)
            ref_opt.step()
            comm = Communicator(rank, world, dev.index, 64 << 20, mem="ipc", timeout_ms=60000)
            shards = FlatShards(model, comm, wire="fp32", reduce_bucket_mb=0.02)
            sopt = ShardedOptimizer(mk(model.parameters()), shards, wire="fp32", stream=torch.cuda.Stream(priority=-1))
            sopt.zero_grad()
            x, y = data[rank]
            torch.nn.functional.mse_loss(model(x.to(dev)), y.to(dev)).backward()
            norm = sopt.clip_grad_norm(max_norm)
            sopt.step()
            torch.cuda.synchronize()
            ok = all(torch.allclose(p, q, rtol=2e-5, atol=2e-6) for p, q in zip(model.parameters(), ref_model.parameters()))
            allv = [None] * world
            dist.all_gather_object(allv, (float(norm), torch.cat([p.detach().flatten() for p in model.parameters()]).cpu()))
            res[name] = dict(ok=ok, norm=float(norm), ref_norm=float(ref_norm),
                             same_norm=len({v[0] for v in allv}) == 1,
                             same_params=all(torch.equal(v[1], allv[0][1]) for v in allv))
            for p in shards.params:          # parameters were views of the arena: ordinary storage before it goes
                p.data = p.data.clone()
                p.grad = None
            del sopt, shards
            comm.close()
        ret[rank] = res
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_worker_processes_match_torch_clipping(world):
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_mp_worker, args=(world, _port(), ret), nprocs=world, join=True)
    assert sorted(ret.keys()) == list(range(world))
    for r in range(world):
        for name, res in ret[r].items():
            assert res["ok"] and res["same_norm"] and res["same_params"], (r, name, res)
            assert res["ref_norm"] > 0.02                                  # the clip was active (coef < 1)
            np.testing.assert_allclose(res["norm"], res["ref_norm"], rtol=1e-5)


# ---- end to end through the strategies ---------------------------------------------------------------------------
class ClipProbe(Callback):
    """In the workers: did the sharded optimizer clip on the device?"""

    def on_train_end(self, trainer, pl_module):
        from ray_lightning_b200.sharded import ShardedOptimizer
        opt = trainer.strategy.optimizers[0]
        pl_module._current_fx = "training_step"
        pl_module.log("probe_sharded_clip", float(isinstance(opt, ShardedOptimizer) and opt._clip_bufs is not None),
                      on_step=True, on_epoch=False)


class WideBoring(BoringModel):
    def __init__(self):
        super().__init__()
        self.layer = torch.nn.Sequential(torch.nn.Linear(32, 256), torch.nn.Tanh(), torch.nn.Linear(256, 2))

    def train_dataloader(self):
        return torch.utils.data.DataLoader(RandomDataset(32, 64, 0), batch_size=8)

    def val_dataloader(self):
        return torch.utils.data.DataLoader(RandomDataset(32, 64, 1), batch_size=8)


class AdamWide(WideBoring):
    def configure_optimizers(self):
        return torch.optim.Adam(self.layer.parameters(), lr=0.01)


@pytest.fixture
def ray_gpu():
    n = torch.cuda.device_count()
    ray.init(num_cpus=4, num_gpus=n)
    yield n
    ray.shutdown()
    os.environ.pop("PL_TORCH_DISTRIBUTED_BACKEND", None)


def _fit(tmpdir, sub, strategy, model_cls, **kw):
    torch.manual_seed(0)
    model = model_cls()
    trainer = get_trainer(os.path.join(str(tmpdir), sub), strategy=strategy, limit_train_batches=6, limit_val_batches=1,
                          callbacks=[ClipProbe()], checkpoint_callback=False, **kw)
    trainer.fit(model)
    return [p.detach().clone() for p in model.parameters()], trainer.logged_metrics


def test_fit_with_gradient_clipping(tmpdir, ray_gpu):
    n = ray_gpu
    share = {"GPU": 1} if n >= 2 else {"GPU": 0.5}
    if n < 2:
        os.environ["PL_TORCH_DISTRIBUTED_BACKEND"] = "gloo"   # two workers on one device: NCCL refuses
    common = dict(num_workers=2, use_gpu=True, resources_per_worker=dict(share), find_unused_parameters=False)
    clip = dict(gradient_clip_val=0.05)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref_adam, _ = _fit(tmpdir, "ref_adam", RayStrategy(b200_enable=False, **common), AdamWide, **clip)
        sharded, m_sh = _fit(tmpdir, "sharded", RayShardedStrategy(b200_wire="fp32", **common), AdamWide, **clip)
        plain, _ = _fit(tmpdir, "plain", RayShardedStrategy(b200_wire="fp32", **common), AdamWide)
        loose, _ = _fit(tmpdir, "loose", RayShardedStrategy(b200_wire="fp32", **common), AdamWide, gradient_clip_val=1e6)
        ref_sgd, _ = _fit(tmpdir, "ref_sgd", RayStrategy(b200_enable=False, **common), WideBoring, **clip)
        hook_sgd, _ = _fit(tmpdir, "hook_sgd", RayStrategy(b200_wire="fp32", **common), WideBoring, **clip)
        value = dict(gradient_clip_val=0.01, gradient_clip_algorithm="value")
        ref_val, _ = _fit(tmpdir, "ref_val", RayStrategy(b200_enable=False, **common), AdamWide, **value)
        sh_val, _ = _fit(tmpdir, "sh_val", RayShardedStrategy(b200_wire="fp32", **common), AdamWide, **value)
        hook_val, _ = _fit(tmpdir, "hook_val", RayStrategy(b200_wire="fp32", **common), WideBoring, **value)
        ref_sgd_val, _ = _fit(tmpdir, "ref_sgd_val", RayStrategy(b200_enable=False, **common), WideBoring, **value)
    assert m_sh["probe_sharded_clip"] == 1.0
    # Sharded vs DDP + torch clipping over 6 Adam steps: the averaged gradients agree to a few ulp (rank-ordered sum of
    # g / W vs. DDP's allreduce) and the norms to ~1e-7 relative (fp64 partials vs. torch's fp32 foreach norms); Adam's
    # update is bounded by lr per step, so the weights drift apart by far less than 6 x lr x 1e-4.
    for a, b in zip(sharded, ref_adam):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)
    assert any(not torch.allclose(a, b, rtol=1e-3, atol=1e-4) for a, b in zip(sharded, plain))   # the clip was active
    for a, b in zip(loose, plain):                       # coef exactly 1.0: the scaled step is the plain step
        assert torch.equal(a, b)
    for a, b in zip(hook_sgd, ref_sgd):                  # replicated path: torch's own clip on identical gradients
        assert torch.equal(a, b)
    for a, b in zip(sh_val, ref_val):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)
    for a, b in zip(hook_val, ref_sgd_val):
        assert torch.equal(a, b)


def test_fit_refuses_clipping_with_optimizer_in_backward(tmpdir, ray_gpu):
    n = ray_gpu
    share = {"GPU": 1} if n >= 2 else {"GPU": 0.5}
    if n < 2:
        os.environ["PL_TORCH_DISTRIBUTED_BACKEND"] = "gloo"
    s = RayStrategy(num_workers=2, use_gpu=True, resources_per_worker=dict(share), b200_optimizer_in_backward=True)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(Exception, match="b200_optimizer_in_backward"):
            _fit(tmpdir, "oib", s, WideBoring, gradient_clip_val=1.0)
