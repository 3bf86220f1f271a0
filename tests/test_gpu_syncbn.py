"""Synchronised BatchNorm over libb2d on the H100: the exchange entry points on loopback ranks against the float32
restatement (bit for bit) and torch's gather op (tolerance), the module without host synchronisation, worker
processes against torch.nn.SyncBatchNorm over the same gloo group, and Trainer.fit(sync_batchnorm=True) through
RayStrategy and RayShardedStrategy."""
import os
import socket
import warnings
from contextlib import closing

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp
import torch.nn.functional as F

import syncbn_ref as ref
from ray_lightning_b200 import RayShardedStrategy, RayStrategy
from ray_lightning_b200._compat import Callback, ray
from utils import BoringModel, RandomDataset, get_trainer

pytestmark = pytest.mark.gpu

EPS, MOM = 1e-5, 0.1


def _bits(t):
    return np.asarray(t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else t, np.float32).view(np.uint32)


def _rank_input(r, n, channels, dtype, channels_last, seed):
    g = torch.Generator().manual_seed(seed + r)
    x = (torch.randn(n, channels, 5, 4, generator=g) * (1 + 0.5 * r) + 0.3 * r).to("cuda", dtype)
    return x.contiguous(memory_format=torch.channels_last) if channels_last else x


@pytest.mark.parametrize("dtype,channels_last", [(torch.float32, False), (torch.float32, True), (torch.bfloat16, False),
                                                 (torch.bfloat16, True)])
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_loopback_exchange_matches_the_restatement(world, dtype, channels_last):
    from ray_lightning_b200.comm import LoopbackGroup
    from ray_lightning_b200.syncbn import syncbn_arena_bytes
    C = 67
    g = LoopbackGroup(world, 0, arena_bytes=16 << 20, timeout_ms=20000)
    try:
        off0 = g.bn_register(0, C)
        assert g.bn_register(1, 5) - off0 == syncbn_arena_bytes([C], world)
        for step, empty in enumerate((-1, world - 1)):          # the second exchange has an empty rank
            xs = [_rank_input(r, 0 if r == empty else 3 + r, C, dtype, channels_last, 10 * step) for r in range(world)]
            stats = [torch.batch_norm_stats(x, EPS) if x.numel() > 0 else (None, None) for x in xs]
            counts = [float(x.numel() // C) for x in xs]
            rm = [torch.linspace(-1, 1, C, device="cuda") for _ in range(world)]
            rv = [torch.linspace(0.5, 2, C, device="cuda") for _ in range(world)]
            rm0, rv0 = rm[0].clone(), rv[0].clone()
            mo = [torch.empty(C, device="cuda") for _ in range(world)]
            io = [torch.empty(C, device="cuda") for _ in range(world)]
            co = [torch.empty(world, dtype=torch.int32, device="cuda") for _ in range(world)]
            g.bn_stats_exchange(0, [s[0] for s in stats], [s[1] for s in stats], counts, EPS, MOM, mo, io, co, rm, rv)
            g.synchronize()
            npm = [None if s[0] is None else s[0].cpu().numpy() for s in stats]
            npi = [None if s[1] is None else s[1].cpu().numpy() for s in stats]
            wm, wi, wc, wrm, wrv = ref.combine_stats(npm, npi, counts, EPS, MOM, rm0.cpu().numpy(), rv0.cpu().numpy())
            for r in range(world):
                assert np.array_equal(_bits(mo[r]), _bits(wm)) and np.array_equal(_bits(io[r]), _bits(wi)), r
                assert co[r].cpu().tolist() == wc.tolist()
                assert np.array_equal(_bits(rm[r]), _bits(wrm)) and np.array_equal(_bits(rv[r]), _bits(wrv)), r
            # torch's own gather op on the same rows, masked as torch.nn.SyncBatchNorm masks them
            keep = [r for r in range(world) if counts[r] > 0]
            x_any = xs[keep[0]]
            trm, trv = rm0.clone(), rv0.clone()
            tm, ti = torch.batch_norm_gather_stats_with_counts(
                x_any, torch.stack([stats[r][0] for r in keep]), torch.stack([stats[r][1] for r in keep]), trm, trv, MOM, EPS,
                torch.tensor([counts[r] for r in keep], device="cuda"))
            for a, b in ((mo[0], tm), (io[0], ti), (rm[0], trm), (rv[0], trv)):
                torch.testing.assert_close(a, b.float(), rtol=1e-5, atol=1e-6)
            # backward rows: rank-ordered fp32 sums
            gg = torch.Generator().manual_seed(99 + step)
            dys = [None if r == empty else torch.randn(C, generator=gg).cuda() for r in range(world)]
            dxs = [None if r == empty else torch.randn(C, generator=gg).cuda() for r in range(world)]
            so = [torch.empty(C, device="cuda") for _ in range(world)]
            xo = [torch.empty(C, device="cuda") for _ in range(world)]
            g.bn_grad_exchange(0, dys, dxs, so, xo)
            g.synchronize()
            want_dy = ref.sum_rows([None if t is None else t.cpu().numpy() for t in dys])
            want_dx = ref.sum_rows([None if t is None else t.cpu().numpy() for t in dxs])
            for r in range(world):
                assert np.array_equal(_bits(so[r]), _bits(want_dy)) and np.array_equal(_bits(xo[r]), _bits(want_dx)), r
            if world == 2 and empty < 0:      # what torch's all_reduce of two rows computes
                assert torch.equal(so[0], dys[0] + dys[1]) and torch.equal(xo[0], dxs[0] + dxs[1])
    finally:
        g.close()


def test_module_runs_without_host_synchronisation_and_matches_one_big_batch():
    """Two loopback ranks, each with its own module on its own stream: forward and backward inside
    set_sync_debug_mode("error") (torch's SyncBatchNorm synchronises the host once per forward, for its mask).
    Outputs and all three gradients against F.batch_norm on the concatenated batch in float64."""
    from ray_lightning_b200.comm import LoopbackGroup
    from ray_lightning_b200.syncbn import convert_sync_batchnorm, register_sync_batchnorm
    C, world = 24, 2
    g = LoopbackGroup(world, 0, arena_bytes=16 << 20, timeout_ms=20000)
    try:
        torch.manual_seed(3)
        proto = torch.nn.BatchNorm2d(C)
        with torch.no_grad():
            proto.weight.uniform_(0.5, 1.5)
            proto.bias.uniform_(-0.5, 0.5)
        mods = []
        for rk in g.ranks:
            m = torch.nn.Sequential(torch.nn.BatchNorm2d(C))
            m[0].load_state_dict(proto.state_dict())
            m = convert_sync_batchnorm(m, (lambda rk=rk: rk)).cuda()
            register_sync_batchnorm(m, rk)
            mods.append(m)
        xs = [(torch.randn(4 + r, C, 6, 6, generator=torch.Generator().manual_seed(r)) + r).cuda().requires_grad_()
              for r in range(world)]
        ws = [torch.randn(4 + r, C, 6, 6, generator=torch.Generator().manual_seed(50 + r)).cuda() for r in range(world)]
        # Load torch's BatchNorm and elementwise kernels first: CUDA loads a kernel on its first launch, and the load
        # waits for the device to drain, which it never does while rank 0's combine spins for a push that this same
        # thread has yet to issue for rank 1.  (Separate processes only wait for their peers there.)
        for x, w in zip(xs, ws):
            x2 = x.detach().clone().requires_grad_()
            wt, bs = mods[0][0].weight.detach(), mods[0][0].bias.detach()
            mean, invstd = torch.batch_norm_stats(x2.detach(), EPS)
            y = torch.batch_norm_elemt(x2.detach(), wt, bs, mean, invstd, EPS)
            sdy, sdx, _, _ = torch.batch_norm_backward_reduce(y, x2.detach(), mean, invstd, wt, True, True, True)
            torch.batch_norm_backward_elemt(y, x2.detach(), mean, invstd, wt, sdy, sdx,
                                            torch.tensor([x.numel() // C], dtype=torch.int32, device="cuda"))
            (x2 * w).sum().backward()
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            outs = []
            for r, rk in enumerate(g.ranks):
                with torch.cuda.stream(rk.stream):
                    outs.append(mods[r](xs[r]))
            for r, rk in enumerate(g.ranks):
                with torch.cuda.stream(rk.stream):
                    (outs[r] * ws[r]).sum().backward()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()
        x64 = torch.cat([x.detach().double() for x in xs]).requires_grad_()
        w64 = proto.weight.detach().double().cuda().requires_grad_()
        b64 = proto.bias.detach().double().cuda().requires_grad_()
        y64 = F.batch_norm(x64, None, None, w64, b64, True, MOM, EPS)
        (y64 * torch.cat(ws).double()).sum().backward()
        torch.testing.assert_close(torch.cat(outs).double(), y64, rtol=1e-4, atol=1e-4)
        torch.testing.assert_close(torch.cat([x.grad for x in xs]).double(), x64.grad, rtol=1e-4, atol=1e-4)
        torch.testing.assert_close(sum(m[0].weight.grad for m in mods).double(), w64.grad, rtol=1e-4, atol=1e-3)
        torch.testing.assert_close(sum(m[0].bias.grad for m in mods).double(), b64.grad, rtol=1e-4, atol=1e-3)
        assert torch.equal(mods[0][0].running_mean, mods[1][0].running_mean)
        assert torch.equal(mods[0][0].running_var, mods[1][0].running_var)
    finally:
        g.close()


# ---- worker processes, gloo control plane -------------------------------------------------------------------------
def _port():
    with closing(socket.socket(socket.AF_INET, socket.SOCK_STREAM)) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


class _ConvBnNet(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 8, 3)
        self.bn2 = torch.nn.BatchNorm2d(8)
        self.fc = torch.nn.Linear(8 * 6 * 6, 16)
        self.bn1 = torch.nn.BatchNorm1d(16)
        self.out = torch.nn.Linear(16, 4)

    def forward(self, x):
        x = F.relu(self.bn2(self.conv(x)))
        x = F.relu(self.bn1(self.fc(x.flatten(1))))
        return self.out(x)


def _mp_worker(rank, world, port, ret):
    import torch.distributed as dist
    from ray_lightning_b200.comm import Communicator
    from ray_lightning_b200.syncbn import convert_sync_batchnorm, register_sync_batchnorm
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world, init_method="env://")
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    comm = Communicator(rank, world, dev.index, 32 << 20, mem="ipc", timeout_ms=60000)
    res = {"ok": True, "why": []}
    try:
        torch.manual_seed(0)
        proto = _ConvBnNet()
        ours = convert_sync_batchnorm(_ConvBnNet(), lambda: comm)
        ours.load_state_dict(proto.state_dict())
        theirs = torch.nn.SyncBatchNorm.convert_sync_batchnorm(_ConvBnNet())
        theirs.load_state_dict(proto.state_dict())
        ours, theirs = ours.to(dev), theirs.to(dev)
        register_sync_batchnorm(ours, comm)
        # torch's module first in every iteration: if it fails, it fails on every rank before any libb2d exchange waits
        opts = [torch.optim.SGD(m.parameters(), lr=0.05) for m in (theirs, ours)]
        for it in range(4):
            gen = torch.Generator().manual_seed(1000 * it + rank)
            x = torch.randn(3 + rank, 3, 8, 8, generator=gen).to(dev)
            y = torch.randint(0, 4, (3 + rank,), generator=gen).to(dev)
            outs = []
            for m, opt in zip((theirs, ours), opts):
                opt.zero_grad(set_to_none=True)
                o = m(x)
                F.cross_entropy(o, y).backward()
                for p in m.parameters():        # what DDP would do with the local gradients
                    dist.all_reduce(p.grad)
                    p.grad /= world
                outs.append(o.detach())
                opt.step()
            if not torch.allclose(outs[1], outs[0], rtol=1e-4, atol=1e-5):
                res["ok"] = False; res["why"].append(("out", it, float((outs[1] - outs[0]).abs().max())))
            for (n, p), q in zip(ours.named_parameters(), theirs.parameters()):
                if not torch.allclose(p, q, rtol=1e-4, atol=1e-5):
                    res["ok"] = False; res["why"].append(("param", it, n, float((p - q).abs().max())))
            for (n, b), c in zip(ours.named_buffers(), theirs.buffers()):
                if b.dtype.is_floating_point and not torch.allclose(b, c, rtol=1e-4, atol=1e-5):
                    res["ok"] = False; res["why"].append(("buffer", it, n))
        torch.cuda.synchronize()
        mine = {n: b.cpu() for n, b in ours.named_buffers()}
        allb = [None] * world
        dist.all_gather_object(allb, mine)
        res["buffers_identical"] = all(torch.equal(allb[r][n], mine[n]) for r in range(world) for n in mine)
        ret[rank] = res
    finally:
        comm.close()
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_worker_processes_match_torch_syncbatchnorm(world):
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_mp_worker, args=(world, _port(), ret), nprocs=world, join=True)
    assert sorted(ret.keys()) == list(range(world))
    for r in range(world):
        assert ret[r]["ok"], (r, ret[r]["why"])
        assert ret[r]["buffers_identical"], r


# ---- end to end through the strategies ---------------------------------------------------------------------------
class BnBoringModel(BoringModel):
    def __init__(self):
        super().__init__()
        self.layer = torch.nn.Sequential(torch.nn.Linear(32, 16), torch.nn.BatchNorm1d(16), torch.nn.ReLU(),
                                         torch.nn.Linear(16, 2))

    def train_dataloader(self):
        return torch.utils.data.DataLoader(RandomDataset(32, 64, 0), batch_size=8)

    def val_dataloader(self):
        return torch.utils.data.DataLoader(RandomDataset(32, 64, 1), batch_size=8)


class AdamBnBoringModel(BnBoringModel):
    def configure_optimizers(self):
        return torch.optim.Adam(self.layer.parameters(), lr=0.05)


class BnProbe(Callback):
    """In the workers: do the BatchNorm buffers agree across ranks, and which module ran?"""

    def on_train_end(self, trainer, pl_module):
        import torch.distributed as dist
        from ray_lightning_b200.syncbn import B200SyncBatchNorm
        bufs = torch.cat([b.detach().float().flatten().cpu() for n, b in pl_module.named_buffers() if "running" in n])
        allb = [None] * dist.get_world_size()
        dist.all_gather_object(allb, bufs)
        pl_module._current_fx = "training_step"
        pl_module.log("probe_bn_equal", float(all(torch.equal(b, bufs) for b in allb)), on_step=True, on_epoch=False)
        pl_module.log("probe_b200_bn", float(any(isinstance(m, B200SyncBatchNorm) for m in pl_module.modules())),
                      on_step=True, on_epoch=False)


@pytest.fixture
def ray_gpu():
    n = torch.cuda.device_count()
    ray.init(num_cpus=4, num_gpus=n)
    yield n
    ray.shutdown()
    os.environ.pop("PL_TORCH_DISTRIBUTED_BACKEND", None)


def _fit(tmpdir, sub, strategy, model_cls):
    torch.manual_seed(0)
    model = model_cls()
    trainer = get_trainer(os.path.join(str(tmpdir), sub), strategy=strategy, limit_train_batches=6, limit_val_batches=1,
                          callbacks=[BnProbe()], sync_batchnorm=True)
    trainer.fit(model)
    return [p.detach().clone() for p in model.parameters()], trainer.logged_metrics


def test_fit_with_sync_batchnorm_matches_torch_syncbatchnorm(tmpdir, ray_gpu):
    n = ray_gpu
    share = {"GPU": 1} if n >= 2 else {"GPU": 0.5}
    if n < 2:
        os.environ["PL_TORCH_DISTRIBUTED_BACKEND"] = "gloo"   # two workers on one device: NCCL refuses
    common = dict(num_workers=2, use_gpu=True, resources_per_worker=dict(share), find_unused_parameters=False)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        theirs, m_ref = _fit(tmpdir, "ref", RayStrategy(b200_enable=False, **common), BnBoringModel)
        ours, m = _fit(tmpdir, "ours", RayStrategy(**common), BnBoringModel)
        sharded, m_sh = _fit(tmpdir, "sharded", RayShardedStrategy(b200_wire="fp32", **common), AdamBnBoringModel)
    assert m["probe_b200_bn"] == 1.0 and m_ref["probe_b200_bn"] == 0.0 and m_sh["probe_b200_bn"] == 1.0
    for a, b in zip(ours, theirs):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)
    # no DDP wrapper broadcasts buffers on the sharded path: synchronised statistics keep them equal
    assert m_sh["probe_bn_equal"] == 1.0 and m["probe_bn_equal"] == 1.0

