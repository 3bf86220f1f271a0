"""Kernel micro-benchmarks (CUDA events, L2-flush between iterations); the training benchmark is bench.py.

  python tools/microbench.py k0            # world=1 cast/scale kernel, HBM roofline
  python tools/microbench.py loopback      # W ranks on one GPU (protocol overhead only, no NVLink)
  torchrun --nproc-per-node N tools/microbench.py sweep   # real multi-GPU sweep vs NCCL
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ray_lightning_b200 import _b2d  # noqa: E402
from ray_lightning_b200.comm import LoopbackGroup  # noqa: E402


def peaks():
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    try:
        return json.load(open(p))
    except Exception:
        return {"hbm_gbs": 3350.0, "fallback": True}   # H100 SXM data sheet


def time_ms(fn, iters, flush=None):
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.add_(1.0)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def k0():
    hbm = peaks()["hbm_gbs"]
    ctx = _b2d.Context(0, 1, 0, 1 << 20)
    flush = torch.empty(256 << 20, dtype=torch.float32, device="cuda")  # 1 GiB > 50 MB L2
    st = torch.cuda.current_stream()
    for mib in (1, 8, 30, 98, 418, 1354):
        n = mib * (1 << 20) // 4
        buf = torch.randn(n, device="cuda")
        for wire in ("bf16", "fp32"):
            f = lambda: ctx.allreduce_bucket(0, buf.data_ptr(), n, _b2d.WIRE_NAMES[wire], 1.0, 0, st, st)
            for _ in range(3):
                f()
            med, best = time_ms(f, 10, flush)
            print(json.dumps({"bench": "k0", "wire": wire, "MiB": mib, "ms_med": round(med, 4), "ms_best": round(best, 4),
                              "GBps_med": round(8 * n / med / 1e6, 1), "frac_of_measured_hbm": round(8 * n / med / 1e6 / hbm, 3),
                              "grid": ctx.plan(n, 1)[1]}), flush=True)
        del buf
    ctx.destroy()


def loopback():
    for world in (2, 4, 8):
        g = LoopbackGroup(world, 0, arena_bytes=512 << 20, timeout_ms=20000)
        for mib in (0.0625, 1, 30):
            n = int(mib * (1 << 20)) // 4
            bufs = [torch.randn(n, device="cuda") for _ in range(world)]
            for algo in ("one_shot", "two_shot"):
                def f():
                    g.allreduce_(bufs, bucket_idx=int(mib * 100) + (algo == "one_shot"), wire="bf16", algo=algo)
                    g.join_current_stream()
                for _ in range(3):
                    f()
                med, best = time_ms(f, 10)
                print(json.dumps({"bench": "loopback", "world": world, "MiB": mib, "algo": algo,
                                  "ms_med": round(med, 4), "ms_best": round(best, 4)}), flush=True)
        g.close()


def _comm():
    import torch.distributed as dist
    from ray_lightning_b200.comm import Communicator
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    env = os.environ.get
    comm = Communicator(rank, world, local, int(env("B2D_ARENA_MB", "3072")) << 20, mem=env("B2D_MEM", "vmm"),
                        max_ctas=int(env("B2D_MAX_CTAS", "128")), timeout_ms=20000, nvls="auto",
                        chunk_bytes=(int(env("B2D_CHUNK_MB")) << 20) if env("B2D_CHUNK_MB") else None,
                        exch_ctas=int(env("B2D_EXCH_CTAS")) if env("B2D_EXCH_CTAS") else None)
    return dist, comm, rank, world


def sweep():
    """Real multi-GPU sweep (one process per GPU, launched by torchrun): libb2d (every algorithm) vs ncclAllReduce,
    the reference's bf16 hook sequence and torch.ops.symm_mem.*; link probe; parity vs NCCL."""
    from bench import allreduce_sweep, link_probe
    dist, comm, rank, world = _comm()
    if rank == 0:
        print(json.dumps({"bench": "sweep_setup", "world": world, "nvls": comm.nvls, "stats": {k: comm.stats()[k] for k in ("arena_bytes", "mc_bound")}}), flush=True)
    link = link_probe(comm, dist, torch, world, rank)
    if rank == 0:
        print(json.dumps({"bench": "link_probe", **link}), flush=True)
    sizes = [64 << 10, 256 << 10, 1 << 20, 4 << 20, 16 << 20, 64 << 20, 256 << 20]  # bytes of WIRE payload (bf16)
    rows = allreduce_sweep(comm, dist, torch, world, rank, sizes, iters=int(os.environ.get("B2D_ITERS", "30")))
    if rank == 0:
        for row in rows:
            print(json.dumps({"bench": "sweep", "world": world, **row}), flush=True)
    # correctness against NCCL on the same inputs
    g = torch.randn(1 << 20, device="cuda", generator=torch.Generator("cuda").manual_seed(rank))
    out = {"bench": "sweep_parity_vs_nccl"}
    theirs = g / world
    dist.all_reduce(theirs)
    c = g.to(torch.bfloat16).div_(world)
    parts = [torch.empty_like(c) for _ in range(world)]
    dist.all_gather(parts, c)
    exact = sum(p.double() for p in parts)
    dist.all_reduce(c)
    torch.cuda.synchronize()
    out["bf16_max_err_vs_exact_nccl"] = float((c.double() - exact).abs().max())
    for ai, algo in enumerate(["two_shot", "staged"] + (["nvls"] if comm.nvls else [])):
        mine = g.clone()
        comm.allreduce_(mine, bucket_idx=990 + ai, wire="fp32", algo=algo)
        mine2 = g.clone()
        comm.allreduce_(mine2, bucket_idx=980 + ai, wire="bf16", algo=algo)
        torch.cuda.synchronize()
        out[algo + "_fp32_allclose_rtol1e-3_atol1e-5"] = bool(torch.allclose(mine, theirs, rtol=1e-3, atol=1e-5))
        out[algo + "_bf16_max_err_vs_exact"] = float((mine2.double() - exact).abs().max())
        out[algo + "_bf16_max_abs_diff_vs_nccl"] = float((mine2 - c.float()).abs().max())
    if rank == 0:
        print(json.dumps(out), flush=True)
    comm.close()
    dist.destroy_process_group()


def tune():
    """Chunk size x exchange-CTA grid for the staged algorithms (isolated, back to back)."""
    dist, comm, rank, world = _comm()
    sizes = [4 << 20, 16 << 20, 64 << 20, 256 << 20]
    iters = 20

    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        dist.barrier()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        t = torch.tensor([a.elapsed_time(b) / iters], device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t)

    bufs = {w: torch.randn(w // 2, device="cuda") * 0.01 for w in sizes}
    chunks = [int(x) for x in os.environ.get("B2D_TUNE_CHUNKS", "4,8,16,32,64").split(",")]
    ctass = [int(x) for x in os.environ.get("B2D_TUNE_CTAS", "8,16,32,64").split(",")]
    for chunk_mb in chunks:
        for ctas in ctass:
            torch.cuda.synchronize()
            dist.barrier()
            comm.ctx.set_chunk_bytes(chunk_mb << 20)
            comm.ctx.set_exch_ctas(ctas)
            row = {"bench": "tune", "world": world, "chunk_mb": chunk_mb, "exch_ctas": ctas}
            for si, w in enumerate(sizes):
                for algo in ["staged"] + (["nvls"] if comm.nvls else []):
                    ms = timed(lambda: comm.allreduce_(bufs[w], bucket_idx=100 + si, wire="bf16", algo=algo))
                    row["%s_%dMiB_us" % (algo, w >> 20)] = round(ms * 1e3, 1)
            if rank == 0:
                print(json.dumps(row), flush=True)
    comm.close()
    dist.destroy_process_group()


def ncu_target():
    """A tiny multi-rank workload meant to run with EVERY rank under its own ncu (single-pass metrics, no kernel
    replay): a few allreduce calls of one size."""
    import torch.distributed as dist
    from ray_lightning_b200.comm import Communicator
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")          # control plane only; keeps NCCL kernels out of the capture
    wire_bytes = int(os.environ.get("B2D_NCU_WIRE_BYTES", str(16 << 20)))
    algos = os.environ.get("B2D_NCU_ALGO", "staged").split(",")
    comm = Communicator(rank, world, local, 1 << 30, mem="vmm", timeout_ms=8000, nvls="auto",
                        max_ctas=int(os.environ.get("B2D_MAX_CTAS", "64")))
    buf = torch.randn(wire_bytes // 2, device="cuda") * 0.01
    for ai, algo in enumerate(algos):
        if algo.startswith("nvls") and not comm.nvls:
            continue
        for i in range(4):
            comm.allreduce_(buf, bucket_idx=ai, wire="bf16", algo=algo)
            torch.cuda.synchronize()
            dist.barrier()
    comm.close()
    dist.destroy_process_group()


def ncu_loopback():
    """Single-GPU target for `ncu --set full`: W loopback ranks run the staged exchange of one ResNet-50-sized bucket
    (7 564 264 elements) phase-major, so every kernel (stage | exchange | wait | write-back, bf16 and fp32 wire, in place)
    can be profiled one at a time.  Peer accesses stay on the device here; HBM-side behaviour is what this shows."""
    world = int(os.environ.get("B2D_NCU_WORLD", "2"))
    n = int(os.environ.get("B2D_NCU_ELEMS", "7564264"))
    g = LoopbackGroup(world, 0, arena_bytes=1 << 30, timeout_ms=20000)
    flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
    for wire in ("bf16", "fp32"):
        bufs = [torch.randn(n, device="cuda") * 0.01 for _ in range(world)]
        for it in range(3):
            flush.add_(1.0)
            torch.cuda.synchronize()
            g.allreduce_(bufs, bucket_idx=1 + (wire == "fp32"), wire=wire, algo="staged")
            g.synchronize()
    abufs = []
    for rk in g.ranks:
        a = rk.arena_tensor(n)
        a.normal_()
        abufs.append(a)
    for it in range(3):
        flush.add_(1.0)
        torch.cuda.synchronize()
        g.allreduce_(abufs, bucket_idx=9, wire="fp32", algo="staged")
        g.synchronize()
    g.close()


def ncu_loopback_sharded():
    """Single-GPU target for ncu: the sharded path's kernels (K11 seg_stage, K12 seg_reduce, K13 adam_push) on W loopback
    ranks, one reduce bucket of 8.4 M elements made of 12 parameter segments, bf16 wire; then K14 (optimizer step of one
    DDP bucket with parameters in separate allocations)."""
    from ray_lightning_b200._b2d import AdamParams
    world = int(os.environ.get("B2D_NCU_WORLD", "2"))
    seg = 699_904                                   # 12 segments ~ one GPT-2-medium reduce bucket
    nseg = 12
    total = seg * nseg
    g = LoopbackGroup(world, 0, arena_bytes=1 << 30, timeout_ms=20000)
    segs = [(i * seg, seg, i % world) for i in range(nseg)]
    # a flat layout grouped by owner: owner r holds the segments with i % world == r, contiguously
    order = sorted(range(nseg), key=lambda i: (i % world, i))
    offs = {i: k * seg for k, i in enumerate(order)}
    segs = [(offs[i], seg, i % world) for i in range(nseg)]
    shard_off = [0]
    for r in range(world):
        shard_off.append(shard_off[-1] + seg * len([i for i in range(nseg) if i % world == r]))
    g.register_bucket(0, segs, "bf16")
    grads = [torch.randn(total, device="cuda") * 0.01 for _ in range(world)]
    reduced = [torch.zeros(shard_off[r + 1] - shard_off[r], device="cuda") for r in range(world)]
    params = []
    for rk in g.ranks:
        p = rk.arena_tensor(total)
        p.normal_()
        params.append(p)
    ms = [torch.zeros_like(t) for t in reduced]
    vs = [torch.zeros_like(t) for t in reduced]
    flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
    for it in range(3):
        for gr in grads:
            gr.normal_()
        flush.add_(1.0)
        torch.cuda.synchronize()
        g.reduce_to_owner(0, grads, reduced, shard_off, zero_grads=True)
        g.synchronize()
        groups = [[(0, shard_off[r + 1] - shard_off[r], dict(lr=1e-4, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, step=it + 1, adamw=0))]
                  for r in range(world)]
        flush.add_(1.0)
        torch.cuda.synchronize()
        g.adam_push_(params, ms, vs, reduced, shard_off, groups)
        g.synchronize()
    # K14
    ctx = g.ranks[0].ctx
    ps = [torch.randn(seg, device="cuda") for _ in range(nseg)]
    s1 = [torch.zeros_like(p) for p in ps]
    bucket = torch.randn(total, device="cuda") * 0.01
    ctx.optim_register(5, [p.data_ptr() for p in ps], [t.data_ptr() for t in s1], None, [i * seg for i in range(nseg)], [seg] * nseg)
    hp = AdamParams(lr=0.05, beta1=0.0, beta2=0.0, eps=0.0, weight_decay=0.0, step=1, adamw=0, zero_grads=0)
    for it in range(3):
        flush.add_(1.0)
        torch.cuda.synchronize()
        ctx.bucket_optim(5, bucket.data_ptr(), total, 0, hp, 0.9, torch.cuda.current_stream())
        torch.cuda.synchronize()
    g.close()


if __name__ == "__main__":
    {"k0": k0, "loopback": loopback, "sweep": sweep, "tune": tune, "ncu_target": ncu_target, "ncu_loopback": ncu_loopback, "ncu_loopback_sharded": ncu_loopback_sharded}[sys.argv[1]]()
