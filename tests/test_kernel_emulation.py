"""The libb2d KERNEL SOURCES, compiled for the host and executed on CPU threads (one OS thread per CUDA
thread, all ranks of a job concurrently in one process), checked bit for bit against the oracle.

This is not a CPU fallback of the product — csrc/emu/ is test infrastructure that only this file builds — it is
a way to execute the real index mappings, phase structure, per-block epoch barriers and double buffering of
b2d_kernels.cuh without a GPU, under whatever interleaving the OS scheduler produces.  It cannot see GPU memory-
ordering bugs or performance; the `-m gpu` tests and the model in test_protocol_model.py cover those angles."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import ddp_oracle

EMU_DIR = os.path.join(ROOT, "ray_lightning_b200", "csrc", "emu")
FP = ctypes.POINTER(ctypes.c_float)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu") / "libb2d_emu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-fPIC", "-shared", "-DB2D_EMU", "-ffp-contract=off",
                    "-o", out, os.path.join(EMU_DIR, "emu_harness.cpp")], check=True)
    lib = ctypes.CDLL(out)
    lib.emu_group_create.restype = ctypes.c_void_p
    lib.emu_group_create.argtypes = [ctypes.c_int, ctypes.c_size_t]
    lib.emu_group_destroy.argtypes = [ctypes.c_void_p]
    lib.emu_signal_bytes.restype = ctypes.c_size_t
    lib.emu_allreduce.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(FP), ctypes.c_size_t,
                                  ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.emu_staged_allreduce.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(FP),
                                         ctypes.c_size_t, ctypes.c_float, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int,
                                         ctypes.c_int, ctypes.c_uint, ctypes.c_int, ctypes.c_int]
    UP = ctypes.POINTER(ctypes.c_uint)
    LP = ctypes.POINTER(ctypes.c_longlong)
    lib.emu_reduce_to_owner.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(FP), ctypes.POINTER(FP), LP, LP, UP,
                                        ctypes.c_int, UP, ctypes.c_size_t, ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_uint,
                                        ctypes.c_int, ctypes.c_int]
    lib.emu_adam_push.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.POINTER(FP), ctypes.POINTER(FP), ctypes.POINTER(FP),
                                  ctypes.c_size_t, LP, ctypes.c_int, LP, LP, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                  ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_uint, ctypes.c_int, ctypes.c_int]
    lib.emu_bucket_optim.argtypes = [ctypes.POINTER(FP), ctypes.POINTER(FP), ctypes.POINTER(FP), UP, ctypes.c_int, FP, ctypes.c_size_t,
                                     ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                     ctypes.c_float, ctypes.c_int, ctypes.c_int]
    lib.emu_k0.argtypes = [FP, ctypes.c_size_t, ctypes.c_float, ctypes.c_int, ctypes.c_int]
    lib.emu_sharded_step.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(FP), ctypes.c_size_t, ctypes.POINTER(FP),
                                     ctypes.POINTER(FP), ctypes.c_size_t, ctypes.POINTER(ctypes.c_longlong), ctypes.c_float,
                                     ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                     ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.emu_reduce_scatter.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(FP), ctypes.POINTER(FP), ctypes.c_size_t,
                                       ctypes.POINTER(ctypes.c_longlong), ctypes.c_float, ctypes.c_size_t, ctypes.c_int, ctypes.c_int]
    lib.emu_allgather.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t, ctypes.POINTER(ctypes.c_longlong), ctypes.c_int]
    lib.emu_owner_table.argtypes = [LP, ctypes.c_int, ctypes.c_int, ctypes.c_int, LP, UP, UP]
    D = ctypes.c_double
    lib.emu_adam_push64.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.POINTER(FP), ctypes.POINTER(FP),
                                    ctypes.POINTER(FP), ctypes.c_size_t, LP, ctypes.c_int, LP, LP, D, D, D, D, D, ctypes.c_int,
                                    ctypes.c_int, ctypes.c_uint, ctypes.c_int, ctypes.c_int]
    lib.emu_sharded_step64.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(FP), ctypes.c_size_t, ctypes.POINTER(FP),
                                       ctypes.POINTER(FP), ctypes.c_size_t, LP, ctypes.c_float, D, D, D, D, D, ctypes.c_int,
                                       ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.emu_arena_ptr.restype = FP
    lib.emu_arena_ptr.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t]
    return lib


def inputs(world, n, seed):
    return [(torch.randn(n, generator=torch.Generator().manual_seed(1000 * seed + r)) * 2.0 ** -4) for r in range(world)]


def ptrs(arrs):
    return (FP * len(arrs))(*[a.ctypes.data_as(FP) for a in arrs])


def same_bits(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


@pytest.mark.parametrize("bf16", [1, 0])
def test_k0_on_cpu_threads(emu, bf16):
    for n in (1, 7, 1000, 4099):
        x = inputs(1, n, 5)[0]
        buf = x.numpy().copy()
        assert emu.emu_k0(buf.ctypes.data_as(FP), n, 1.0, bf16, 2) == 0
        want = (ddp_oracle.allreduce_bf16_wire if bf16 else ddp_oracle.allreduce_fp32_wire)([x])
        assert same_bits(buf, want.numpy()), n


@pytest.mark.parametrize("world,grid,generic", [(2, 2, 0), (4, 2, 0), (8, 1, 0), (3, 2, 1)])
@pytest.mark.parametrize("algo", [1, 2, 3])
def test_allreduce_kernels_on_cpu_threads(emu, world, grid, generic, algo):
    """K1 (one-shot), K2 (two-shot) and K3 (NVLS, the switch emulated) for both wires; consecutive launches
    alternate the slot half and keep the epoch counters, as in the real call sequence."""
    g = emu.emu_group_create(world, 4 << 20)
    try:
        step = 0
        for bf16 in (1, 0):
            for n in (1, 9, 1000, 4099, 20011):
                per_rank = inputs(world, n, 10 * step + algo)
                bufs = [t.numpy().copy() for t in per_rank]
                scale = float(np.float32(1.0) / np.float32(world))
                assert emu.emu_allreduce(g, algo, bf16, ptrs(bufs), n, scale, grid, step & 1, generic, 4) == 0
                want = (ddp_oracle.allreduce_bf16_wire if bf16 else ddp_oracle.allreduce_fp32_wire)(per_rank).numpy()
                for r in range(world):
                    assert same_bits(bufs[r], want), (world, algo, bf16, n, r)
                step += 1
    finally:
        emu.emu_group_destroy(g)


@pytest.mark.parametrize("world,generic", [(2, 0), (4, 0), (3, 1)])
@pytest.mark.parametrize("bf16", [0, 1])
def test_sharded_step_on_cpu_threads(emu, world, generic, bf16):
    """K4+K5+K6: three consecutive fused steps; every rank ends with the same, whole parameter vector ==
    Adam on the oracle-averaged gradients (uneven, 8-aligned owner shards)."""
    rng = np.random.default_rng(3)
    numels = [int(x) for x in rng.integers(1, 700, size=9)] + [3000]
    owner = ddp_oracle.partition_fairscale(numels, world)
    _, shard_off, total = ddp_oracle.shard_layout(numels, owner, world)
    sig = emu.emu_signal_bytes()
    g = emu.emu_group_create(world, 4 << 20)
    try:
        p0 = torch.randn(total, generator=torch.Generator().manual_seed(9))
        views = []
        for r in range(world):
            v = np.ctypeslib.as_array(emu.emu_arena_ptr(g, r, sig), shape=(total,))
            v[:] = p0.numpy()
            views.append(v)
        ms = [np.zeros(max(shard_off[r + 1] - shard_off[r], 8), np.float32) for r in range(world)]
        vs = [np.zeros(max(shard_off[r + 1] - shard_off[r], 8), np.float32) for r in range(world)]
        ref = torch.nn.Parameter(p0.clone())
        opt = torch.optim.Adam([ref], lr=1e-2)
        scale = float(np.float32(1.0) / np.float32(world))
        off = (ctypes.c_longlong * (world + 1))(*shard_off)
        for step in range(1, 4):
            per_rank = [torch.randn(total, generator=torch.Generator().manual_seed(100 * step + r)) * 0.1 for r in range(world)]
            grads = [t.numpy().copy() for t in per_rank]
            rc = emu.emu_sharded_step(g, bf16, ptrs(grads), sig, ptrs(ms), ptrs(vs), total, off, scale, 1e-2, 0.9, 0.999, 1e-8,
                                      0.0, step, 0, int(step == 2), 2, step & 1, generic)
            assert rc == 0
            avg = ddp_oracle.allreduce_fp32_wire(per_rank, scale) if not bf16 else sum(ddp_oracle.wire_bf16(t, scale) for t in per_rank)
            ref.grad = avg.clone()
            opt.step()
            for r in range(1, world):
                assert same_bits(views[r], views[0]), (step, r)
            np.testing.assert_allclose(views[0], ref.detach().numpy(), rtol=2e-5, atol=2e-6)
            if step == 2:
                assert all(float(np.abs(gr).max()) == 0.0 for gr in grads)
    finally:
        emu.emu_group_destroy(g)


@pytest.mark.parametrize("world,generic", [(2, 0), (4, 0), (8, 0), (3, 1)])
@pytest.mark.parametrize("nvls", [0, 1])
@pytest.mark.parametrize("order", [0, 1, 2])
def test_staged_exchange_on_cpu_threads(emu, world, generic, nvls, order):
    """K7-K10 (stage | exchange | wait + write back as separate kernels, b2d_staged.cuh), P2P and NVLS (switch
    emulated), both wires, one to several chunks, ragged sizes; consecutive calls keep the monotone epochs and
    alternate the staging half.  order 1 runs every kernel of every rank strictly one after the other, phase-major:
    the schedule a serialising profiler imposes on the loopback ranks must complete too."""
    sig = emu.emu_signal_bytes()
    g = emu.emu_group_create(world, 4 << 20)
    try:
        epoch, step = 1, 0
        chunk = 1024 * world if world != 3 else 1026
        for bf16 in (1, 0):
            for n in (1, 9, 4099, 20011, 40003):
                per_rank = inputs(world, n, 70 * step + nvls)
                bufs = [t.numpy().copy() for t in per_rank]
                scale = float(np.float32(1.0) / np.float32(world))
                npacks = -(-n // (8 if bf16 else 4))
                half = (step & 1) * (1 << 20)
                rc = emu.emu_staged_allreduce(g, nvls, bf16, 0, ptrs(bufs), n, scale, sig + half, chunk, 1, 1, epoch, order, generic)
                assert rc == 0
                epoch += -(-npacks // chunk)
                want = (ddp_oracle.allreduce_bf16_wire if bf16 else ddp_oracle.allreduce_fp32_wire)(per_rank).numpy()
                for r in range(world):
                    assert same_bits(bufs[r], want), (world, nvls, bf16, n, r, order)
                step += 1
    finally:
        emu.emu_group_destroy(g)


@pytest.mark.parametrize("world,generic", [(2, 0), (4, 0), (3, 1)])
@pytest.mark.parametrize("nvls", [0, 1])
def test_staged_exchange_in_place_on_cpu_threads(emu, world, generic, nvls):
    """fp32 buckets that LIVE in the arena (f-1): no stage, no write back; the exchange scales and reduces the
    bucket where it is, ragged last pack included (element-wise path)."""
    sig = emu.emu_signal_bytes()
    g = emu.emu_group_create(world, 4 << 20)
    try:
        epoch = 1
        for step, n in enumerate((1, 2, 7, 4099, 4100, 20011)):
            per_rank = inputs(world, n, 33 * step + nvls)
            views = []
            for r in range(world):
                v = np.ctypeslib.as_array(emu.emu_arena_ptr(g, r, sig + 4096), shape=(n + 8,))
                v[:] = 777.0                       # a neighbour's bytes past the end must survive
                v[:n] = per_rank[r].numpy()
                views.append(v)
            scale = float(np.float32(1.0) / np.float32(world))
            chunk = 1024 * world if world != 3 else 1026
            assert emu.emu_staged_allreduce(g, nvls, 0, 1, None, n, scale, sig + 4096, chunk, 1, 1, epoch, 2 if step % 2 else 0, generic) == 0
            epoch += -(-(-(-n // 4)) // chunk)
            want = ddp_oracle.allreduce_fp32_wire(per_rank, scale).numpy()
            for r in range(world):
                if nvls and world & (world - 1):
                    # the switch adds the RAW values and the kernel scales the sum: (sum g) / W rounds differently from
                    # sum (g / W) unless W is a power of two — the NVLS tolerance contract (north star: rtol 1e-3 / atol 1e-5)
                    np.testing.assert_allclose(views[r][:n], want, rtol=1e-5, atol=1e-7)
                    assert same_bits(views[r][:n], views[0][:n])
                else:
                    assert same_bits(views[r][:n], want), (world, nvls, n, r)
                assert float(views[r][n]) == 777.0 and float(views[r][n + 3]) == 777.0
    finally:
        emu.emu_group_destroy(g)


@pytest.mark.parametrize("algo", [2, 5])
def test_kernels_with_scheduling_jitter(emu, algo, monkeypatch):
    """Random 0-300 us sleeps at 2 % of all barrier entries (B2D_EMU_JITTER): blocks and ranks drift far apart;
    six consecutive launches on alternating halves must still match the oracle bit for bit (5 = staged exchange,
    three flag-coupled streams per rank)."""
    monkeypatch.setenv("B2D_EMU_JITTER", "20")
    world, grid = 4, 2
    sig = emu.emu_signal_bytes()
    g = emu.emu_group_create(world, 8 << 20)
    try:
        epoch = 1
        for step in range(6):
            n = 30011 + 997 * step
            per_rank = inputs(world, n, 900 + step)
            bufs = [t.numpy().copy() for t in per_rank]
            if algo == 5:
                chunk = 1024 * world
                assert emu.emu_staged_allreduce(g, 0, 1, 0, ptrs(bufs), n, 0.25, sig + (step & 1) * (1 << 20), chunk, 2, 2,
                                                epoch, 2, 0) == 0
                epoch += -(-(-(-n // 8)) // chunk)
            else:
                assert emu.emu_allreduce(g, algo, 1, ptrs(bufs), n, 0.25, grid, step & 1, 0, 1) == 0
            want = ddp_oracle.allreduce_bf16_wire(per_rank).numpy()
            for r in range(world):
                assert same_bits(bufs[r], want), (algo, step, r)
    finally:
        emu.emu_group_destroy(g)


@pytest.mark.parametrize("world", [2, 3])
def test_reduce_scatter_and_allgather_alone_on_cpu_threads(emu, world):
    """K4 and K6 as separate launches (the path of optimizers other than Adam): reduce-scatter bit-exact for both
    wires, then an all-gather of a flat arena buffer whose shards were filled by their owners."""
    rng = np.random.default_rng(5)
    numels = [int(x) for x in rng.integers(1, 900, size=7)]
    owner = ddp_oracle.partition_fairscale(numels, world)
    _, shard_off, total = ddp_oracle.shard_layout(numels, owner, world)
    off = (ctypes.c_longlong * (world + 1))(*shard_off)
    sig = emu.emu_signal_bytes()
    g = emu.emu_group_create(world, 4 << 20)
    try:
        scale = float(np.float32(1.0) / np.float32(world))
        for step, bf16 in enumerate((0, 1, 0)):
            per_rank = [torch.randn(total, generator=torch.Generator().manual_seed(31 * step + r)) * 0.1 for r in range(world)]
            grads = [t.numpy().copy() for t in per_rank]
            outs = [np.zeros(max(shard_off[r + 1] - shard_off[r], 8), np.float32) for r in range(world)]
            assert emu.emu_reduce_scatter(g, bf16, ptrs(grads), ptrs(outs), total, off, scale, sig + (1 << 20), 2, step & 1) == 0
            if bf16:
                want = None
                for t in per_rank:
                    c = ddp_oracle.wire_bf16(t, scale)
                    want = c if want is None else want + c
            else:
                want = ddp_oracle.allreduce_fp32_wire(per_rank, scale)
            for r in range(world):
                n_own = shard_off[r + 1] - shard_off[r]
                assert same_bits(outs[r][:n_own], want[shard_off[r]:shard_off[r + 1]].numpy()), (step, r)
        full = torch.randn(total, generator=torch.Generator().manual_seed(77)).numpy()
        views = []
        for r in range(world):
            v = np.ctypeslib.as_array(emu.emu_arena_ptr(g, r, sig), shape=(total,))
            v[:] = 0
            v[shard_off[r]:shard_off[r + 1]] = full[shard_off[r]:shard_off[r + 1]]
            views.append(v)
        assert emu.emu_allgather(g, sig, total, off, 2) == 0
        for r in range(world):
            assert same_bits(views[r], full), r
    finally:
        emu.emu_group_destroy(g)


def _seg_table(emu, segs, world, epp):
    """What b2d_bucket_register builds (segments sorted by (owner, offset), touching runs merged, cumulative pack starts),
    from the library's own table builder."""
    flat = (ctypes.c_longlong * len(segs))()
    start = (ctypes.c_uint * (len(segs) + 1))()
    owner_pack = (ctypes.c_uint * (world + 1))()
    triples = (ctypes.c_longlong * (3 * len(segs)))(*[x for seg in segs for x in seg])
    nseg = emu.emu_owner_table(triples, len(segs), world, int(epp == 8), flat, start, owner_pack)
    assert nseg > 0
    return list(flat[:nseg]), list(start[:nseg + 1]), list(owner_pack)


@pytest.mark.parametrize("world,generic", [(2, 0), (4, 0), (3, 1)])
@pytest.mark.parametrize("bf16", [0, 1])
@pytest.mark.parametrize("nvls", [0, 1])
def test_reduce_to_owner_and_adam_push_on_cpu_threads(emu, world, generic, bf16, nvls):
    """K11 + K12 + K13: two reduce buckets of scattered parameter segments go to their owners (second pass accumulates),
    then Adam on every owner's shard and the push of the new parameters; serialised phase-major order included."""
    rng = np.random.default_rng(7)
    numels = [int(x) for x in rng.integers(1, 900, size=11)] + [2500]
    owner = ddp_oracle.partition_fairscale(numels, world)
    offs, shard_off, total = ddp_oracle.shard_layout(numels, owner, world)
    epp = 8 if bf16 else 4
    idx = list(reversed(range(len(numels))))
    buckets = [[(offs[i], -(-numels[i] // 8) * 8, owner[i]) for i in part] for part in (idx[:6], idx[6:])]
    sig = emu.emu_signal_bytes()
    g = emu.emu_group_create(world, 4 << 20)
    off = (ctypes.c_longlong * (world + 1))(*shard_off)
    mask = np.zeros(total, bool)
    for o, n in zip(offs, numels):
        mask[o:o + n] = True
    try:
        scale = float(np.float32(1.0) / np.float32(world))
        n_own = [shard_off[r + 1] - shard_off[r] for r in range(world)]
        reduced = [np.full(max(n, 8), 5.0, np.float32) for n in n_own]
        epoch = 1
        total_want = None
        for rep in range(2):
            per_rank = [torch.randn(total, generator=torch.Generator().manual_seed(31 * rep + r)) * 0.1 for r in range(world)]
            grads = [t.numpy().copy() for t in per_rank]
            wire_off = sig + (1 << 20)
            for b, segs in enumerate(buckets):
                flat, start, opack = _seg_table(emu, segs, world, epp)
                rc = emu.emu_reduce_to_owner(g, bf16, nvls, ptrs(grads), ptrs(reduced), off, (ctypes.c_longlong * len(flat))(*flat),
                                             (ctypes.c_uint * len(start))(*start), len(flat), (ctypes.c_uint * len(opack))(*opack),
                                             wire_off, scale, 1, rep, epoch, (rep + b) % 2, generic)
                assert rc == 0
                epoch += 1
                wire_off += start[-1] * 16
            if bf16 and nvls:
                want = ddp_oracle.allreduce_bf16_wire(per_rank)      # the switch hands back a bf16 sum: one rounding more
            elif bf16:
                want = None
                for t in per_rank:
                    c = ddp_oracle.wire_bf16(t, scale)
                    want = c if want is None else want + c
            else:
                want = ddp_oracle.allreduce_fp32_wire(per_rank, scale)
            total_want = want.numpy() if rep == 0 else total_want + want.numpy()
            for r in range(world):
                lo, hi = shard_off[r], shard_off[r + 1]
                m = mask[lo:hi]
                assert same_bits(reduced[r][:hi - lo][m], total_want[lo:hi][m]), (world, bf16, nvls, rep, r)
                assert float(np.abs(grads[r][mask]).max()) == 0.0
        # Adam on the owners' shards + push
        p0 = torch.randn(total, generator=torch.Generator().manual_seed(9)).numpy()
        poff = sig + (2 << 20)
        views = []
        for r in range(world):
            v = np.ctypeslib.as_array(emu.emu_arena_ptr(g, r, poff), shape=(total,))
            v[:] = p0
            views.append(v)
        ms = [np.zeros(max(n, 8), np.float32) for n in n_own]
        vs = [np.zeros(max(n, 8), np.float32) for n in n_own]
        glo = (ctypes.c_longlong * world)(*[0] * world)
        ghi = (ctypes.c_longlong * world)(*n_own)
        ref = torch.nn.Parameter(torch.from_numpy(p0.copy()))
        opt = torch.optim.Adam([ref], lr=1e-2)
        for step in (1, 2):
            assert emu.emu_adam_push(g, nvls, poff, ptrs(ms), ptrs(vs), ptrs(reduced), total, off, 1, glo, ghi, 1e-2, 0.9, 0.999, 1e-8, 0.0,
                                     step, 0, epoch, step % 2, generic) == 0
            epoch += 1
            full = np.zeros(total, np.float32)
            for r in range(world):
                full[shard_off[r]:shard_off[r + 1]] = reduced[r][:n_own[r]]
            ref.grad = torch.from_numpy(full.copy())
            opt.step()
            for r in range(world):
                assert same_bits(views[r], views[0]), (step, r)
            np.testing.assert_allclose(views[0], ref.detach().numpy(), rtol=2e-5, atol=2e-6)
    finally:
        emu.emu_group_destroy(g)


@pytest.mark.parametrize("opt_name", ["sgd", "sgd_plain", "adam", "adamw"])
def test_bucket_optimizer_kernel_on_cpu_threads(emu, opt_name):
    """K14 (optimizer step of one DDP bucket, parameters in separate allocations of odd sizes) against torch.optim over
    three steps."""
    sizes = [5, 1, 37, 1000, 3]
    torch.manual_seed(3)
    ref = [torch.nn.Parameter(torch.randn(n)) for n in sizes]
    mk = {"sgd": lambda ps: torch.optim.SGD(ps, lr=0.05, momentum=0.9, weight_decay=1e-2),
          "sgd_plain": lambda ps: torch.optim.SGD(ps, lr=0.05),
          "adam": lambda ps: torch.optim.Adam(ps, lr=1e-2, weight_decay=1e-2),
          "adamw": lambda ps: torch.optim.AdamW(ps, lr=1e-2, weight_decay=0.05)}[opt_name]
    opt = mk(ref)
    params = [p.detach().numpy().copy() for p in ref]
    s1 = [np.zeros(n, np.float32) for n in sizes]
    s2 = [np.zeros(n, np.float32) for n in sizes]
    start = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    g = opt.param_groups[0]
    for step in (1, 2, 3):
        grads = torch.randn(sum(sizes), generator=torch.Generator().manual_seed(step)) * 0.1
        off = 0
        for p, n in zip(ref, sizes):
            p.grad = grads[off:off + n].clone()
            off += n
        opt.step()
        gb = grads.numpy().copy()
        kind = 0 if opt_name.startswith("sgd") else 1
        betas = g.get("betas", (0.0, 0.0))
        rc = emu.emu_bucket_optim(ptrs(params), ptrs(s1), ptrs(s2), start.ctypes.data_as(ctypes.POINTER(ctypes.c_uint)), len(sizes),
                                  gb.ctypes.data_as(FP), sum(sizes), kind, g["lr"], g.get("momentum", 0.0), g["weight_decay"],
                                  betas[0], betas[1], g.get("eps", 0.0), step, int(opt_name == "adamw"))
        assert rc == 0
        for mine, p in zip(params, ref):
            np.testing.assert_allclose(mine, p.detach().numpy(), rtol=2e-5, atol=2e-6)
    if opt_name == "sgd":
        for mine, p in zip(s1, ref):
            np.testing.assert_allclose(mine, opt.state[p]["momentum_buffer"].numpy(), rtol=2e-5, atol=2e-6)


def test_owner_path_with_ranks_that_own_nothing(emu):
    """Edge cases of K12 / K13: a reduce bucket in which one rank owns no segment at all (empty staging range), and a
    parameter push from a rank whose shard is empty — every other rank's result must be unaffected."""
    world = 4
    sig = emu.emu_signal_bytes()
    g = emu.emu_group_create(world, 4 << 20)
    try:
        # three parameters, owners 0, 1 and 3: rank 2 owns nothing, in the bucket and in the flat space
        numels = [504, 1000, 256]
        owner = [0, 1, 3]
        offs, cur = [], 0
        shard_off = [0]
        for r in range(world):
            for i, n in enumerate(numels):
                if owner[i] == r:
                    offs.append((i, cur))
                    cur += n
            shard_off.append(cur)
        offs = [o for _, o in sorted(offs)]
        total = cur
        segs = [(offs[i], numels[i], owner[i]) for i in range(3)]
        flat, start, opack = _seg_table(emu, segs, world, 4)
        assert opack[2] == opack[3]                      # rank 2's range of the staging region is empty
        per_rank = [torch.randn(total, generator=torch.Generator().manual_seed(r)) * 0.1 for r in range(world)]
        grads = [t.numpy().copy() for t in per_rank]
        n_own = [shard_off[r + 1] - shard_off[r] for r in range(world)]
        reduced = [np.full(max(n, 8), 9.0, np.float32) for n in n_own]
        off = (ctypes.c_longlong * (world + 1))(*shard_off)
        scale = 0.25
        rc = emu.emu_reduce_to_owner(g, 0, 0, ptrs(grads), ptrs(reduced), off, (ctypes.c_longlong * len(flat))(*flat),
                                     (ctypes.c_uint * len(start))(*start), len(flat), (ctypes.c_uint * len(opack))(*opack),
                                     sig + (1 << 20), scale, 1, 0, 1, 0, 0)
        assert rc == 0
        want = ddp_oracle.allreduce_fp32_wire(per_rank, scale).numpy()
        for r in range(world):
            assert same_bits(reduced[r][:n_own[r]], want[shard_off[r]:shard_off[r + 1]]), r
        assert float(reduced[2][0]) == 9.0               # untouched
        # push: every rank's copy of every shard becomes its owner's; rank 2 pushes nothing
        poff = sig + (2 << 20)
        views = []
        for r in range(world):
            v = np.ctypeslib.as_array(emu.emu_arena_ptr(g, r, poff), shape=(total,))
            v[:] = -1.0
            v[shard_off[r]:shard_off[r + 1]] = float(r + 1)
            views.append(v)
        assert emu.emu_adam_push(g, 0, poff, None, None, None, total, off, 0, None, None, 0, 0, 0, 0, 0, 1, 0, 2, 0, 0) == 0
        for r in range(world):
            for o in range(world):
                assert (views[r][shard_off[o]:shard_off[o + 1]] == float(o + 1)).all(), (r, o)
    finally:
        emu.emu_group_destroy(g)


# ---- index math at every world size, at non-default grids, with guard bytes around every output ------------------------
# The specialisations W = 2, 4, 8 and the generic build (W = 0: B2D_MAX_WORLD-wide arrays masked by r < world, one pack
# per batch) cut the buckets differently; the sizes below are derived from each kernel's geometry (slices, grid-stride
# batches, pipeline chunks) rather than listed, so that every tail a grid can meet is hit.  Every output sits between
# two GUARD-float margins of a NaN canary (payload + a per-rank salt: a reduction of the neighbours' canaries then
# changes some rank's margin even on the host, where NaN arithmetic keeps the first payload), compared as bits.
CANARY = 0x7fc0beef
GUARD = 16          # 64 bytes: a view behind the margin keeps the 16-byte alignment of its buffer


def guarded(values, salt=0):
    """(whole buffer, view of `values` inside it) with canary margins on both sides."""
    values = np.asarray(values, np.float32)
    whole = np.empty(values.size + 2 * GUARD, np.float32)
    whole.view(np.uint32)[:] = CANARY + salt
    whole[GUARD:GUARD + values.size] = values
    return whole, whole[GUARD:GUARD + values.size]


def guards_intact(whole, n, salt=0):
    u = whole.view(np.uint32)
    return bool((u[:GUARD] == CANARY + salt).all() and (u[GUARD + n:] == CANARY + salt).all())


def packs_per_batch(per_pack):
    """b2d_kernels.cuh: packs a thread handles per batch when every pack costs `per_pack` loads (W = 0: one)."""
    return 16 // per_pack if per_pack > 0 and 16 // per_pack > 1 else 1


def specialisation(world):
    """b2d_launch.cuh's dispatch_world: the W a world size runs."""
    return world if world in (2, 4, 8) else 0


def chunk_packs(world, chunk_bytes):
    """b2d.cu's staged_chunk_packs: the chunk in packs, rounded down to a multiple of W x 1024, at least one such unit."""
    unit = world * 1024
    return max(chunk_bytes // 16 // unit * unit, unit)


def ragged(npacks, epp, i):
    """A bucket of `npacks` packs whose last pack holds 1, epp - 1 or epp elements, by turns."""
    return npacks * epp - (epp - 1, 1, 0)[i % 3]


@pytest.mark.parametrize("grid", [1, 3])
def test_k0_grid_stride_tails_and_guard_bytes(emu, grid):
    """K0 (world 1): one grid-stride batch covers grid x 512 threads x U = 4 vectors of 4 elements; below, at and past
    it, several batches, and the scalar tail of 1-3 elements."""
    per_pass = grid * 512 * 4 * 4
    for bf16 in (1, 0):
        for k, n in enumerate((1, 2, 3, 5, per_pass - 1, per_pass, per_pass + 2, 3 * per_pass + 3)):
            x = inputs(1, n, 40 + k)[0]
            whole, buf = guarded(x.numpy())
            assert emu.emu_k0(buf.ctypes.data_as(FP), n, 1.0, bf16, grid) == 0
            want = (ddp_oracle.allreduce_bf16_wire if bf16 else ddp_oracle.allreduce_fp32_wire)([x])
            assert same_bits(buf, want.numpy()), (grid, bf16, n)
            assert guards_intact(whole, n), (grid, bf16, n)


@pytest.mark.parametrize("world,grid", [(5, 1), (6, 1), (7, 1), (2, 3), (2, 5), (3, 3), (3, 5)])
@pytest.mark.parametrize("algo", [1, 2])
def test_allreduce_kernels_at_any_world_and_grid(emu, world, grid, algo):
    """K1 / K2 at the world sizes only the generic build runs (5, 6, 7) and at grids of 3 and 5 blocks: fewer packs
    than ranks (empty slices), a slice (K2) or a bucket (K1) of exactly one grid-stride batch and one pack either side
    (k x W - 1, k x W, k x W + 1 packs), several batches; both wires, ragged last packs, guard bytes."""
    g = emu.emu_group_create(world, 8 << 20)
    try:
        per_pass = grid * 512 * packs_per_batch(specialisation(world))
        counts = sorted({1, world - 1, per_pass, per_pass + 1, world * per_pass - 1, world * per_pass, world * per_pass + 1,
                         3 * world * per_pass + 2})
        step = 0
        for bf16 in (1, 0):
            epp = 8 if bf16 else 4
            for i, npacks in enumerate(counts):
                n = ragged(npacks, epp, i)
                per_rank = inputs(world, n, 500 + step)
                held = [guarded(t.numpy(), r) for r, t in enumerate(per_rank)]
                scale = float(np.float32(1.0) / np.float32(world))
                assert emu.emu_allreduce(g, algo, bf16, ptrs([b for _, b in held]), n, scale, grid, step & 1, 0, 4) == 0
                want = (ddp_oracle.allreduce_bf16_wire if bf16 else ddp_oracle.allreduce_fp32_wire)(per_rank).numpy()
                for r, (whole, buf) in enumerate(held):
                    assert same_bits(buf, want), (world, grid, algo, bf16, n, r)
                    assert guards_intact(whole, n, r), (world, grid, algo, bf16, n, r)
                step += 1
    finally:
        emu.emu_group_destroy(g)


@pytest.mark.parametrize("world", [5, 6, 7])
@pytest.mark.parametrize("nvls", [0, 1])
def test_staged_exchange_at_any_world(emu, world, nvls):
    """K7-K10 through the generic build with one-block stage and exchange grids: empty slices, a slice of exactly one
    grid-stride batch of the exchange kernel and one pack past it, one chunk and one pack, and six chunks with a ragged last pack (the library's chunk of 64 KiB + 16 bytes, rounded to W x 1024 packs); the three
    schedules of emu_staged_allreduce by turns; guard bytes around every bucket."""
    sig = emu.emu_signal_bytes()
    g = emu.emu_group_create(world, 16 << 20)
    try:
        cp = chunk_packs(world, (64 << 10) + 16)
        per_pass = 256 * packs_per_batch(specialisation(world))
        counts = (1, world + 1, world * per_pass, world * per_pass + 1, cp + 1, 5 * cp + world * per_pass + 3)
        epoch, step = 1, 0
        for bf16 in (1, 0):
            epp = 8 if bf16 else 4
            for i, npacks in enumerate(counts):
                n = ragged(npacks, epp, i)
                per_rank = inputs(world, n, 600 + 10 * step + nvls)
                held = [guarded(t.numpy(), r) for r, t in enumerate(per_rank)]
                scale = float(np.float32(1.0) / np.float32(world))
                half = (step & 1) * (4 << 20)
                rc = emu.emu_staged_allreduce(g, nvls, bf16, 0, ptrs([b for _, b in held]), n, scale, sig + half, cp, 1, 1, epoch,
                                              step % 3, 0)
                assert rc == 0
                epoch += -(-npacks // cp)
                want = (ddp_oracle.allreduce_bf16_wire if bf16 else ddp_oracle.allreduce_fp32_wire)(per_rank).numpy()
                for r, (whole, buf) in enumerate(held):
                    assert same_bits(buf, want), (world, nvls, bf16, n, r)
                    assert guards_intact(whole, n, r), (world, nvls, bf16, n, r)
                step += 1
    finally:
        emu.emu_group_destroy(g)


@pytest.mark.parametrize("world", [5, 6, 7])
@pytest.mark.parametrize("nvls", [0, 1])
def test_staged_exchange_in_place_at_any_world_next_to_a_neighbour(emu, world, nvls):
    """In-place fp32 buckets (n % 4 = 1, 2, 3, 0) of one to six chunks, two of them side by side in the arena with a
    canary margin before, between and after: exchanging the second must leave the first one's result and every
    margin alone, and the ragged last pack of each must stop at its last element."""
    sig = emu.emu_signal_bytes()
    g = emu.emu_group_create(world, 16 << 20)
    try:
        cp = chunk_packs(world, 64 << 10)
        scale = float(np.float32(1.0) / np.float32(world))
        epoch = 1
        for step, (pa, pb, rag) in enumerate(((1, world - 1, 1), (cp - 1, cp + 1, 2), (5 * cp + 7, 2 * cp, 3), (3, 5 * cp + 1, 0))):
            na, nb = pa * 4 - (4 - rag) % 4, pb * 4 - rag
            a0 = GUARD
            b0 = -(-(a0 + na) // 4) * 4 + GUARD
            size = b0 + nb + GUARD
            base = sig + 4096
            per_a = inputs(world, na, 700 + step + 10 * nvls)
            per_b = inputs(world, nb, 800 + step + 10 * nvls)
            views = []
            for r in range(world):
                v = np.ctypeslib.as_array(emu.emu_arena_ptr(g, r, base), shape=(size,))
                v.view(np.uint32)[:] = CANARY + r
                v[a0:a0 + na] = per_a[r].numpy()
                v[b0:b0 + nb] = per_b[r].numpy()
                views.append(v)
            for off, n in ((a0, na), (b0, nb)):
                assert emu.emu_staged_allreduce(g, nvls, 0, 1, None, n, scale, base + 4 * off, cp, 1, 1, epoch, step % 3, 0) == 0
                epoch += -(-(-(-n // 4)) // cp)
            mask = np.ones(size, bool)
            mask[a0:a0 + na] = mask[b0:b0 + nb] = False
            for off, n, per_rank in ((a0, na, per_a), (b0, nb, per_b)):
                want = ddp_oracle.allreduce_fp32_wire(per_rank, scale).numpy()
                for r in range(world):
                    got = views[r][off:off + n]
                    if nvls and world & (world - 1):
                        # the emulated switch adds the raw values and the kernel scales the sum (tolerance contract)
                        np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-7)
                        assert same_bits(got, views[0][off:off + n])
                    else:
                        assert same_bits(got, want), (world, nvls, n, r)
            for r in range(world):
                assert bool((views[r].view(np.uint32)[mask] == CANARY + r).all()), (world, nvls, step, r)
    finally:
        emu.emu_group_destroy(g)


def _owner_buckets(world, kind):
    """(numels, owner, flat offsets, shard_off, total, buckets): "empty" has W - 1 parameters, so owner W - 1 owns
    nothing, and a first bucket holding owner 1's parameters only; "deep" has 4000 eight-element parameters and a first
    bucket of 2000 segments that do not touch (every other parameter of each owner), so seg_find searches a deep table."""
    if kind == "empty":
        numels = [3001, 1203, 805, 640, 96, 51, 9][:world - 1]
    else:
        numels = [8] * 4000
    owner = ddp_oracle.partition_fairscale(numels, world)
    offs, shard_off, total = ddp_oracle.shard_layout(numels, owner, world)
    if kind == "empty":
        first = [i for i in range(len(numels)) if owner[i] == 1]
    else:
        first = [i for i in range(len(numels)) if (i // world) % 2 == 0]
    rest = [i for i in range(len(numels)) if i not in set(first)]
    buckets = [[(offs[i], -(-numels[i] // 8) * 8, owner[i]) for i in part] for part in (first, rest)]
    return numels, owner, offs, shard_off, total, buckets


@pytest.mark.parametrize("world", [5, 7])
@pytest.mark.parametrize("kind", ["empty", "deep"])
@pytest.mark.parametrize("bf16", [0, 1])
def test_owner_path_at_any_world(emu, world, kind, bf16):
    """K11 + K12 at W = 5 and 7 (generic build): an owner with an empty shard, a bucket whose segments all belong to one
    owner (every other owner's staging range is empty), a deep segment table; then K13 (Adam + push) bit for bit
    against torch's CUDA foreach Adam as restated in optim_ref.  Guard bytes around the gradients K11 zeroes, the
    reduced shards K12 writes, exp_avg / exp_avg_sq and the flat parameters K13 writes; K11 must zero exactly the
    bucket's segments, and reducing the second bucket must leave the first one's results alone."""
    import optim_ref
    numels, owner, offs, shard_off, total, buckets = _owner_buckets(world, kind)
    if kind == "empty":
        assert shard_off[world - 1] == shard_off[world]
        assert {owner_of for _, _, owner_of in buckets[0]} == {1}
    epp = 8 if bf16 else 4
    sig = emu.emu_signal_bytes()
    g = emu.emu_group_create(world, 8 << 20)
    off = (ctypes.c_longlong * (world + 1))(*shard_off)
    n_own = [shard_off[r + 1] - shard_off[r] for r in range(world)]
    try:
        scale = float(np.float32(1.0) / np.float32(world))
        per_rank = [torch.randn(total, generator=torch.Generator().manual_seed(90 + r)) * 0.1 for r in range(world)]
        grads = [guarded(t.numpy(), r) for r, t in enumerate(per_rank)]
        reduced = [guarded(np.full(n, 5.0, np.float32), r) for r, n in enumerate(n_own)]
        if bf16:
            want = None
            for t in per_rank:
                c = ddp_oracle.wire_bf16(t, scale)
                want = c if want is None else want + c
            want = want.numpy()
        else:
            want = ddp_oracle.allreduce_fp32_wire(per_rank, scale).numpy()
        done = np.zeros(total, bool)
        epoch, wire_off = 1, sig + (1 << 20)
        for b, segs in enumerate(buckets):
            flat, start, opack = _seg_table(emu, segs, world, epp)
            if kind == "deep" and b == 0:
                assert len(flat) >= 2000
            rc = emu.emu_reduce_to_owner(g, bf16, 0, ptrs([v for _, v in grads]), ptrs([v for _, v in reduced]), off,
                                         (ctypes.c_longlong * len(flat))(*flat), (ctypes.c_uint * len(start))(*start), len(flat),
                                         (ctypes.c_uint * len(opack))(*opack), wire_off, scale, 1, 0, epoch, b % 2, 0)
            assert rc == 0
            epoch += 1
            wire_off += start[-1] * 16
            for o, n, _ in segs:
                done[o:o + n] = True
            for r in range(world):
                lo, hi = shard_off[r], shard_off[r + 1]
                whole, red = reduced[r]
                m = done[lo:hi]
                assert same_bits(red[m], want[lo:hi][m]), (world, kind, bf16, b, r)
                assert bool((red[~m] == 5.0).all()), (world, kind, bf16, b, r)
                assert guards_intact(whole, hi - lo, r), (world, kind, bf16, b, r)
                gw, gv = grads[r]
                assert bool((gv[done] == 0.0).all()) and same_bits(gv[~done], per_rank[r].numpy()[~done]), (world, kind, b, r)
                assert guards_intact(gw, total, r), (world, kind, bf16, b, r)
        assert done.all()

        # K13: one Adam group per owner over its whole shard, two steps, parameters pushed into every arena
        hp = dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, adamw=True)
        p = torch.randn(total, generator=torch.Generator().manual_seed(91)).numpy()
        poff = sig + (4 << 20) + 4 * GUARD
        views = []
        for r in range(world):
            v = np.ctypeslib.as_array(emu.emu_arena_ptr(g, r, poff - 4 * GUARD), shape=(total + 2 * GUARD,))
            v.view(np.uint32)[:] = CANARY + r
            v[GUARD:GUARD + total] = p
            views.append(v)
        ms = [guarded(np.zeros(n, np.float32), r) for r, n in enumerate(n_own)]
        vs = [guarded(np.zeros(n, np.float32), r) for r, n in enumerate(n_own)]
        gl = (ctypes.c_longlong * world)(*[0] * world)
        gh = (ctypes.c_longlong * world)(*n_own)
        m_ref, v_ref = np.zeros(total, np.float32), np.zeros(total, np.float32)
        for step in (1, 2):
            assert emu.emu_adam_push64(g, 0, poff, ptrs([x for _, x in ms]), ptrs([x for _, x in vs]), ptrs([x for _, x in reduced]),
                                       total, off, 1, gl, gh, hp["lr"], hp["beta1"], hp["beta2"], hp["eps"], hp["weight_decay"],
                                       step, 1, epoch, step % 2, 0) == 0
            epoch += 1
            p, m_ref, v_ref = optim_ref.adam_step32(p, want, m_ref, v_ref, step=step, path="foreach", **hp)
            for r in range(world):
                lo, hi = shard_off[r], shard_off[r + 1]
                assert same_bits(views[r][GUARD:GUARD + total], p), (world, kind, bf16, step, r)
                assert guards_intact(views[r], total, r), (world, kind, bf16, step, r)
                assert same_bits(ms[r][1], m_ref[lo:hi]) and same_bits(vs[r][1], v_ref[lo:hi]), (world, kind, bf16, step, r)
                assert guards_intact(ms[r][0], hi - lo, r) and guards_intact(vs[r][0], hi - lo, r), (world, kind, bf16, step, r)
    finally:
        emu.emu_group_destroy(g)


@pytest.mark.parametrize("world,grid", [(5, 1), (7, 1), (3, 3), (2, 5)])
@pytest.mark.parametrize("bf16", [0, 1])
def test_sharded_step_at_any_world_and_grid(emu, world, grid, bf16):
    """K4 + K5 + K6 (fused) and K4 alone at W = 5 and 7 with one block, and at grids of 3 and 5 blocks, with an owner
    whose shard is empty: parameters bit for bit against optim_ref's restatement of torch's CUDA foreach Adam on the
    oracle's reduced gradients, reduce-scatter outputs bit-exact, guard bytes around exp_avg / exp_avg_sq, the
    reduce-scatter outputs, the gradients the step zeroes and the flat parameters."""
    import optim_ref
    numels = [4099, 1500, 9, 777, 2048, 3, 8200][:world - 1]
    owner = ddp_oracle.partition_fairscale(numels, world)
    _, shard_off, total = ddp_oracle.shard_layout(numels, owner, world)
    n_own = [shard_off[r + 1] - shard_off[r] for r in range(world)]
    assert 0 in n_own
    sig = emu.emu_signal_bytes()
    g = emu.emu_group_create(world, 8 << 20)
    off = (ctypes.c_longlong * (world + 1))(*shard_off)
    scale = float(np.float32(1.0) / np.float32(world))
    try:
        hp = dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, adamw=False)
        p = torch.randn(total, generator=torch.Generator().manual_seed(12)).numpy()
        views = []
        for r in range(world):
            v = np.ctypeslib.as_array(emu.emu_arena_ptr(g, r, sig), shape=(total + 2 * GUARD,))
            v.view(np.uint32)[:] = CANARY + r
            v[GUARD:GUARD + total] = p
            views.append(v)
        ms = [guarded(np.zeros(n, np.float32), r) for r, n in enumerate(n_own)]
        vs = [guarded(np.zeros(n, np.float32), r) for r, n in enumerate(n_own)]
        m_ref, v_ref = np.zeros(total, np.float32), np.zeros(total, np.float32)
        for step in (1, 2):
            per_rank = [torch.randn(total, generator=torch.Generator().manual_seed(100 * step + r)) * 0.1 for r in range(world)]
            grads = [guarded(t.numpy(), r) for r, t in enumerate(per_rank)]
            rc = emu.emu_sharded_step64(g, bf16, ptrs([x for _, x in grads]), sig + 4 * GUARD, ptrs([x for _, x in ms]),
                                        ptrs([x for _, x in vs]), total, off, scale, hp["lr"], hp["beta1"], hp["beta2"], hp["eps"],
                                        hp["weight_decay"], step, 0, 1, grid, step & 1, 0)
            assert rc == 0
            if bf16:
                avg = None
                for t in per_rank:
                    c = ddp_oracle.wire_bf16(t, scale)
                    avg = c if avg is None else avg + c
                avg = avg.numpy()
            else:
                avg = ddp_oracle.allreduce_fp32_wire(per_rank, scale).numpy()
            p, m_ref, v_ref = optim_ref.adam_step32(p, avg, m_ref, v_ref, step=step, path="foreach", **hp)
            for r in range(world):
                lo, hi = shard_off[r], shard_off[r + 1]
                assert same_bits(views[r][GUARD:GUARD + total], p), (world, grid, bf16, step, r)
                assert guards_intact(views[r], total, r), (world, grid, bf16, step, r)
                assert same_bits(ms[r][1], m_ref[lo:hi]) and same_bits(vs[r][1], v_ref[lo:hi]), (world, grid, bf16, step, r)
                assert guards_intact(ms[r][0], hi - lo, r) and guards_intact(vs[r][0], hi - lo, r), (world, grid, bf16, step, r)
                assert bool((grads[r][1] == 0.0).all()) and guards_intact(grads[r][0], total, r), (world, grid, bf16, step, r)
        # K4 alone into guarded outputs
        per_rank = [torch.randn(total, generator=torch.Generator().manual_seed(300 + r)) * 0.1 for r in range(world)]
        grads = [t.numpy().copy() for t in per_rank]
        outs = [guarded(np.zeros(n, np.float32), r) for r, n in enumerate(n_own)]
        assert emu.emu_reduce_scatter(g, bf16, ptrs(grads), ptrs([x for _, x in outs]), total, off, scale, sig + (2 << 20), grid, 0) == 0
        if bf16:
            want = None
            for t in per_rank:
                c = ddp_oracle.wire_bf16(t, scale)
                want = c if want is None else want + c
        else:
            want = ddp_oracle.allreduce_fp32_wire(per_rank, scale)
        for r in range(world):
            lo, hi = shard_off[r], shard_off[r + 1]
            assert same_bits(outs[r][1], want[lo:hi].numpy()), (world, grid, bf16, r)
            assert guards_intact(outs[r][0], hi - lo, r), (world, grid, bf16, r)
    finally:
        emu.emu_group_destroy(g)
