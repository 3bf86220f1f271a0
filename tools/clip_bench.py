#!/usr/bin/env python
"""clip_bench.py — what gradient clipping costs on the sharded path, on one GPU.

    python tools/clip_bench.py --out DIR [--world 2] [--iters 50] [--warmup 5]

Writes DIR/clip_bench.json with
  * gpu: card name, power limit and clocks (read-only nvidia-smi query, in this call);
  * norm: for an own shard of 1 M, 4 M, 16 M and 64 M fp32 elements per rank, through --world loopback ranks on the
    one device (phase-major: every K18, then every K19), the time of one clip call (K18 + K19 of every rank, CUDA events
    over --iters calls) and K18's HBM rate (4 B per owned element, all ranks' elements over that time); as a baseline,
    ``torch.linalg.vector_norm(shard)`` followed by ``shard.mul_(coef)`` on one shard of the same size;
  * step: a ResNet-50-sized model (torchvision resnet50's parameters, Adam) on a one-rank ShardedOptimizer: the step
    (reduce of the gradients + fused Adam + push) without and with ``clip_grad_norm`` in front, CUDA events over --iters
    steps, the two alternated.
Multi-GPU figures are not measured by this tool.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES_M = (1, 4, 16, 64)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=60)
    return [dict(zip(q.split(","), (v.strip() for v in line.split(",")))) for line in out.stdout.strip().splitlines()]


def _time(fn, iters, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def bench_norm(world, iters, warmup):
    import torch
    from ray_lightning_b200.comm import LoopbackGroup
    out = []
    for m in SIZES_M:
        n = m << 20
        g = LoopbackGroup(world, 0, arena_bytes=16 << 20, timeout_ms=60000)
        try:
            g.clip_register()
            xs = [torch.randn(n, device="cuda") for _ in range(world)]
            norms = [torch.zeros(1, device="cuda") for _ in range(world)]
            coefs = [torch.zeros(1, device="cuda") for _ in range(world)]

            def clip():
                g.clip_norm_(xs, 1.0, norms, coefs)
                g.join_current_stream()
            ms = _time(clip, iters, warmup)
        finally:
            g.close()
        x = torch.randn(n, device="cuda")

        def baseline():
            norm = torch.linalg.vector_norm(x)
            x.mul_(torch.clamp(1.0 / (norm + 1e-6), max=1.0))
        base_ms = _time(baseline, iters, warmup)
        out.append(dict(elements_per_rank=n, world=world, clip_call_ms=ms,
                        k18_hbm_gbps=world * n * 4 / (ms * 1e-3) / 1e9,
                        torch_norm_mul_ms=base_ms, torch_norm_mul_hbm_gbps=3 * n * 4 / (base_ms * 1e-3) / 1e9))
        print(json.dumps(out[-1]), flush=True)
    return out


def bench_step(iters, warmup):
    import torch
    import torchvision
    from ray_lightning_b200.comm import LoopbackGroup
    from ray_lightning_b200.sharded import FlatShards, ShardedOptimizer
    g = LoopbackGroup(1, 0, arena_bytes=640 << 20, timeout_ms=60000)
    try:
        model = torchvision.models.resnet50().cuda()
        shards = FlatShards(model, g.ranks[0], wire="fp32")
        sopt = ShardedOptimizer(torch.optim.Adam(model.parameters(), lr=1e-4), shards, wire="fp32",
                                stream=torch.cuda.Stream(priority=-1))
        grads = torch.randn(shards.total, device="cuda") * 1e-2

        def step(clip):
            sopt.zero_grad()
            shards.flat_grads.copy_(grads)        # what backward leaves behind; the step reduces it
            if clip:
                sopt.clip_grad_norm(1.0)
            sopt.step()
        res = {"params": shards.total}
        for rep in range(2):                      # alternated: no arm gets the warmer clocks
            for clip in (False, True):
                res.setdefault("clip" if clip else "plain", []).append(_time(lambda: step(clip), iters, warmup))
        res["plain_ms"] = min(res["plain"])
        res["clip_ms"] = min(res["clip"])
        return res
    finally:
        g.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--world", type=int, default=2)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("clip_bench.py measures on the GPU; no CUDA device is visible")
    res = {"gpu": gpu_info(), "torch": torch.__version__, "norm": bench_norm(a.world, a.iters, a.warmup),
           "step": bench_step(a.iters, a.warmup), "multi_gpu": "not measured"}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "clip_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["step"]))


if __name__ == "__main__":
    main()
