#!/usr/bin/env python
"""syncbn_bench.py — what synchronised BatchNorm costs on this box, libb2d's exchange against torch's SyncBatchNorm.

    python tools/syncbn_bench.py --out DIR [--iters 200] [--steps 20] [--warmup 5] [--repeats 2]

Writes DIR/syncbn_bench.json with
  * gpu: card name, power limit and clocks (read-only nvidia-smi query, in this call);
  * layer: per-layer exchange latency (CUDA events over --iters exchanges after warm-up) for C in {64, 256, 1024, 2048}:
      forward   libb2d push + combine                vs  torch: cat + all_gather_into_tensor + mask + gather op
      backward  libb2d push + sum                    vs  torch: cat + all_reduce + split
    one process per GPU; with one GPU, two processes share it and the torch / NCCL arm is "not measured" (NCCL
    refuses two ranks on one device);
  * resnet50: step time of bench.py's workload (ResNet-50, bf16 autocast, channels_last, batch 64 per process) under
    RayStrategy with sync_batchnorm off / on with libb2d / on with torch's SyncBatchNorm (b200_enable=False), the three
    alternated --repeats times, at the largest process count the box has (two processes sharing the GPU on a one-GPU
    box, where the torch arm's collectives run over gloo).  Median and spread over the repeats.
"""
import argparse
import json
import os
import socket
import statistics
import subprocess
import sys
import time
from contextlib import closing

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = (64, 256, 1024, 2048)


def free_port():
    with closing(socket.socket(socket.AF_INET, socket.SOCK_STREAM)) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=60)
    return [dict(zip(q.split(","), (v.strip() for v in line.split(",")))) for line in out.stdout.strip().splitlines()]


def _init(rank, world, port, backend):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    kw = {"device_id": torch.device("cuda", dev)} if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, init_method="env://", **kw)
    return torch.device("cuda", dev)


def _layer_worker(rank, world, port, iters, warmup, nccl, ret):
    import torch
    import torch.distributed as dist
    from ray_lightning_b200.comm import Communicator
    dev = _init(rank, world, port, "nccl" if nccl else "gloo")
    comm = Communicator(rank, world, dev.index, 32 << 20, mem="ipc")
    res = {}
    try:
        for lid, C in enumerate(SIZES):
            comm.bn_register_all([(lid, C)])
            x = torch.randn(64, C, 7, 7, device=dev)
            mean, invstd = torch.batch_norm_stats(x, 1e-5)
            count = float(x.numel() // C)
            mo, io = torch.empty(C, device=dev), torch.empty(C, device=dev)
            co = torch.empty(world, dtype=torch.int32, device=dev)
            rm, rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
            dy, dxmu = torch.randn(C, device=dev), torch.randn(C, device=dev)
            so, xo = torch.empty(C, device=dev), torch.empty(C, device=dev)

            def b2d_fwd():
                comm.bn_stats_exchange(lid, mean, invstd, count, 1e-5, 0.1, mo, io, co, rm, rv)

            def b2d_bwd():
                comm.bn_grad_exchange(lid, dy, dxmu, so, xo)

            def torch_fwd():   # torch/nn/modules/_functions.py:65-115
                cnt = torch.full((1,), count, dtype=mean.dtype, device=dev)
                combined = torch.cat([mean, invstd, cnt], dim=0)
                flat = torch.empty(world * combined.numel(), dtype=combined.dtype, device=dev)
                dist.all_gather_into_tensor(flat, combined)
                allc = flat.view(world, -1)
                m_all, i_all, c_all = torch.split(allc, C, dim=1)
                mask = c_all.squeeze(-1) >= 1
                counts = c_all[mask]
                torch.batch_norm_gather_stats_with_counts(x, m_all[mask], i_all[mask], rm, rv, 0.1, 1e-5, counts.view(-1))

            def torch_bwd():   # :155-165
                combined = torch.cat([dy, dxmu], dim=0)
                dist.all_reduce(combined)
                torch.split(combined, C)

            arms = [("b2d_fwd", b2d_fwd), ("b2d_bwd", b2d_bwd)] + ([("torch_fwd", torch_fwd), ("torch_bwd", torch_bwd)] if nccl else [])
            for name, fn in arms:
                for _ in range(warmup):
                    fn()
                torch.cuda.synchronize()
                dist.barrier()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(iters):
                    fn()
                b.record()
                b.synchronize()
                res.setdefault(C, {})[name] = a.elapsed_time(b) * 1e3 / iters
        ret[rank] = res
    finally:
        comm.close()
        dist.destroy_process_group()


def _step_worker(rank, world, port, mode, steps, warmup, ret):
    import torch
    import torch.distributed as dist
    import torch.nn.functional as F
    import torchvision
    from ray_lightning_b200 import RayStrategy
    from ray_lightning_b200._compat import LightningModule
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = torch.device("cuda", rank % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    torch.backends.cudnn.benchmark = True
    torch.manual_seed(0)

    class Net(LightningModule):
        def __init__(self):
            super().__init__()
            self.net = torchvision.models.resnet50()

        def training_step(self, batch, batch_idx):
            x, y = batch
            return F.cross_entropy(self.net(x), y)

        def configure_optimizers(self):
            return torch.optim.SGD(self.parameters(), lr=0.05, momentum=0.9)

    # the worker-side call sequence of RayLauncher._wrapping_function, with PL's sync_batchnorm conversion
    strategy = RayStrategy(num_workers=world, use_gpu=True, b200_enable=(mode != "torch"), find_unused_parameters=False,
                           gradient_as_bucket_view=True, bucket_cap_mb=25)
    strategy.precision = "bf16"
    strategy.set_remote(True)
    strategy.set_global_to_local([(i, 0) for i in range(world)])
    strategy.root_device = dev
    strategy._worker_setup(process_idx=rank)
    model = Net().to(memory_format=torch.channels_last)
    strategy.connect(model)
    strategy.model_to_device()
    if mode != "off":
        strategy.model = strategy.configure_sync_batchnorm(strategy.model)
    strategy.configure_ddp()

    class _T:
        pass
    strategy.setup_optimizers(_T())
    opt = strategy.optimizers[0]
    g = torch.Generator().manual_seed(1000 + rank)
    batch = (torch.randn(64, 3, 224, 224, generator=g).contiguous(memory_format=torch.channels_last).to(dev),
             torch.randint(0, 1000, (64,), generator=g).to(dev))

    def step(i):
        opt.zero_grad(set_to_none=True)
        loss = strategy.training_step(batch, i)
        strategy.backward(loss)
        opt.step()

    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    dist.barrier()
    t0 = time.perf_counter()
    for i in range(steps):
        step(warmup + i)
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / steps
    ret[rank] = dt
    strategy.teardown_worker()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    import torch
    import torch.multiprocessing as mp
    if not torch.cuda.is_available():
        raise SystemExit("syncbn_bench.py measures on a GPU: none is visible")
    os.makedirs(args.out, exist_ok=True)
    ngpu = torch.cuda.device_count()
    shared = ngpu < 2
    world = 2 if shared else ngpu
    out = {"gpu": gpu_info(), "world": world,
           "placement": "2 processes sharing one GPU" if shared else "one process per GPU"}

    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_layer_worker, args=(world, free_port(), args.iters, 20, not shared, ret), nprocs=world, join=True)
    layer = {}
    for C in SIZES:
        row = {"C": C}
        for arm in ("b2d_fwd", "b2d_bwd", "torch_fwd", "torch_bwd"):
            vals = [ret[r][C][arm] for r in range(world) if arm in ret[r][C]]
            row[arm + "_us"] = max(vals) if vals else "not measured"
        layer[str(C)] = row
    out["layer"] = layer
    out["layer_note"] = ("microseconds per exchange, slowest rank; " +
                         ("2 processes sharing one GPU, whose contexts the driver time-slices: a combine kernel waits for the other "
                          "process's time slice, so these figures measure context switching, not the exchange; torch/NCCL "
                          "arm not measured" if shared else "torch arm over NCCL"))

    if shared:
        os.environ["PL_TORCH_DISTRIBUTED_BACKEND"] = "gloo"
    times = {m: [] for m in ("off", "b2d", "torch")}
    for _ in range(args.repeats):
        for mode in times:
            ret = mgr.dict()
            mp.spawn(_step_worker, args=(world, free_port(), mode, args.steps, args.warmup, ret), nprocs=world, join=True)
            times[mode].append(max(ret[r] for r in range(world)) * 1e3)
    out["resnet50_step_ms"] = {m: {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}
                               for m, v in times.items()}
    out["resnet50_note"] = ("ResNet-50, bf16 autocast, channels_last, batch 64 per process, %d processes (%s); "
                            "off / on with libb2d / on with torch SyncBatchNorm (b200_enable=False%s)"
                            % (world, out["placement"], ", collectives over gloo" if shared else ", NCCL"))
    path = os.path.join(args.out, "syncbn_bench.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
