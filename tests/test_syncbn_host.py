"""Synchronised BatchNorm without a GPU: the float32 restatement against float64 batch statistics, the exchange
kernels (csrc/b2d_syncbn.cuh) on CPU threads bit for bit against it, a model of the exchange protocol, and the
module conversion / strategy plumbing."""
import ctypes
import os
import pickle
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT
import syncbn_ref as ref

EMU_DIR = os.path.join(ROOT, "ray_lightning_b200", "csrc", "emu")
FP = ctypes.POINTER(ctypes.c_float)
IP = ctypes.POINTER(ctypes.c_int32)
SIGNAL_BYTES = 64 * 1024


def _rank_inputs(world, channels, sizes, seed, shape_tail=(3,)):
    g = torch.Generator().manual_seed(seed)
    out = []
    for r in range(world):
        x = torch.randn((sizes[r], channels) + shape_tail, generator=g, dtype=torch.float64) * (1 + r) + 0.5 * r
        out.append(x)
    return out


# ---- the restatement against float64 statistics of the concatenated batch ------------------------------------
@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("empty", [False, True])
def test_restatement_matches_float64_batch_statistics(world, empty):
    C, eps, mom = 37, 1e-5, 0.1
    sizes = [4 + r for r in range(world)]
    if empty and world > 1:
        sizes[1] = 0
    xs = _rank_inputs(world, C, sizes, seed=world)
    means, invstds, counts = [], [], []
    for x in xs:
        if x.shape[0] == 0:
            means.append(None); invstds.append(None); counts.append(0)
        else:
            m, s, n = ref.local_stats(x.numpy(), eps)
            means.append(m); invstds.append(s); counts.append(n)
    rm0 = np.linspace(-1, 1, C).astype(np.float32)
    rv0 = np.linspace(0.5, 2, C).astype(np.float32)
    mean, invstd, cnt, rm, rv = ref.combine_stats(means, invstds, counts, eps, mom, rm0, rv0)
    full = torch.cat(xs).numpy()
    fc = np.moveaxis(full, 1, 0).reshape(C, -1)
    want_mean, want_var = fc.mean(1), fc.var(1)
    np.testing.assert_allclose(mean, want_mean, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(invstd, 1 / np.sqrt(want_var + eps), rtol=1e-5, atol=1e-6)
    assert cnt.tolist() == counts
    np.testing.assert_allclose(rm, (1 - mom) * rm0 + mom * want_mean, rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(rv, (1 - mom) * rv0 + mom * fc.var(1, ddof=1), rtol=1e-5, atol=1e-6)


# ---- the kernels on CPU threads ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu_bn") / "libb2d_emu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-fPIC", "-shared", "-DB2D_EMU", "-ffp-contract=off",
                    "-o", out, os.path.join(EMU_DIR, "emu_harness.cpp")], check=True)
    lib = ctypes.CDLL(out)
    lib.emu_group_create.restype = ctypes.c_void_p
    lib.emu_group_create.argtypes = [ctypes.c_int, ctypes.c_size_t]
    lib.emu_group_destroy.argtypes = [ctypes.c_void_p]
    lib.emu_bn_exchange.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(FP), ctypes.POINTER(FP), FP,
                                    ctypes.c_float, ctypes.c_float, ctypes.POINTER(FP), ctypes.POINTER(FP), ctypes.POINTER(IP),
                                    ctypes.POINTER(FP), ctypes.POINTER(FP), ctypes.c_size_t, ctypes.c_uint, ctypes.c_int,
                                    ctypes.c_int]
    return lib


def _arr(arrs, P=FP):
    return (P * len(arrs))(*[(ctypes.cast(0, P) if a is None else a.ctypes.data_as(P)) for a in arrs])


def _rows(layout_off, world, channels):
    """Region offsets of one layer as b2d.cu lays it out: forward gen 0 | gen 1 | backward gen 0 | gen 1."""
    f, b = (2 * channels + 1 + 3) // 4 * 4, (2 * channels + 3) // 4 * 4
    return [layout_off + g * world * f * 4 for g in (0, 1)], [layout_off + 2 * world * f * 4 + g * world * b * 4 for g in (0, 1)]


def _same_bits(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


@pytest.mark.parametrize("order", [0, 1])
@pytest.mark.parametrize("channels", [1, 3, 37, 2048])
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_bn_exchange_kernels_on_cpu_threads(emu, world, channels, order):
    """K15 + K16 and K15 + K17, all ranks concurrently (order 0) or fully serialised phase-major (order 1); two
    generations back to back on the same epoch words, the second with an empty rank; running statistics carried
    over.  Every rank's outputs equal the restatement bit for bit."""
    eps, mom = 1e-5, 0.1
    g = emu.emu_group_create(world, 2 << 20)
    try:
        fwd_off, bwd_off = _rows(SIGNAL_BYTES, world, channels)
        rng = np.random.default_rng(world * 1000 + channels)
        rm = [np.linspace(-1, 1, channels).astype(np.float32) for _ in range(world)]
        rv = [np.linspace(0.5, 2, channels).astype(np.float32) for _ in range(world)]
        want_rm, want_rv = rm[0].copy(), rv[0].copy()
        epoch = 0
        grid = 1 if channels < 1024 else 2
        for gen in (0, 1):
            empty = world - 1 if gen == 1 else -1
            counts = np.array([0 if r == empty else 5 + 3 * r for r in range(world)], np.float32)
            means = [None if r == empty else rng.standard_normal(channels).astype(np.float32) for r in range(world)]
            invstds = [None if r == empty else rng.uniform(0.5, 2, channels).astype(np.float32) for r in range(world)]
            mo = [np.zeros(channels, np.float32) for _ in range(world)]
            io = [np.zeros(channels, np.float32) for _ in range(world)]
            co = [np.full(world, -1, np.int32) for _ in range(world)]
            epoch += 1
            assert emu.emu_bn_exchange(g, 1, channels, _arr(means), _arr(invstds), counts.ctypes.data_as(FP), eps, mom,
                                       _arr(mo), _arr(io), _arr(co, IP), _arr(rm), _arr(rv), fwd_off[gen], epoch, grid,
                                       order) == 0
            wm, wi, wc, want_rm, want_rv = ref.combine_stats(means, invstds, counts, eps, mom, want_rm, want_rv)
            for r in range(world):
                assert _same_bits(mo[r], wm) and _same_bits(io[r], wi), (gen, r)
                assert co[r].tolist() == wc.tolist(), (gen, r)
                assert _same_bits(rm[r], want_rm) and _same_bits(rv[r], want_rv), (gen, r)
            # backward of the same layer
            dy = [None if r == empty else rng.standard_normal(channels).astype(np.float32) for r in range(world)]
            dx = [None if r == empty else rng.standard_normal(channels).astype(np.float32) for r in range(world)]
            so = [np.zeros(channels, np.float32) for _ in range(world)]
            xo = [np.zeros(channels, np.float32) for _ in range(world)]
            epoch += 1
            assert emu.emu_bn_exchange(g, 0, channels, _arr(dy), _arr(dx), counts.ctypes.data_as(FP), 0.0, 0.0,
                                       _arr(so), _arr(xo), None, None, None, bwd_off[gen], epoch, grid, order) == 0
            for r in range(world):
                assert _same_bits(so[r], ref.sum_rows(dy)) and _same_bits(xo[r], ref.sum_rows(dx)), (gen, r)
    finally:
        emu.emu_group_destroy(g)


# ---- protocol model -----------------------------------------------------------------------------------------------
def _check_protocol(world, program, generations=2, staged=2, shared_flags=False):
    """Explicit-state exploration of every interleaving of W ranks, each running two streams:

      * the compute stream issues the BN exchanges of ``program`` ([(layer, direction)], the same on every rank) as
        push (write the row into region (layer, direction, call parity) of every rank, then bn[rank] = epoch) and
        combine (enabled once bn[src] >= epoch for every src; reads the W rows);
      * an internal stream runs ``staged`` bucket exchanges (arrive: staged[rank] = e; wait: staged[src] >= e).

    A combine that reads a row another exchange has overwritten, or a state without successors in which some stream
    has not finished, is returned as (kind, trace).  ``generations=1`` removes the double buffer; ``shared_flags=True``
    lets the BN exchanges and the bucket exchanges signal through the same words."""
    n_bn = 2 * len(program)
    calls, gen_of = {}, []
    for layer, d in program:
        k = calls.get((layer, d), 0)
        calls[(layer, d)] = k + 1
        gen_of.append(k % generations)

    start = (tuple([0] * world), tuple([0] * world), tuple([0] * world), tuple([0] * world), frozenset())
    seen = set()
    stack = [(start, ())]
    while stack:
        state, trace = stack.pop()
        if state in seen:
            continue
        seen.add(state)
        pc_bn, pc_st, bn, st, mem = state
        mem_d = dict(mem)
        succ = []
        for r in range(world):
            p = pc_bn[r]
            if p < n_bn:
                e = p // 2
                layer, d = program[e]
                region = (layer, d, gen_of[e])
                flags = st if shared_flags else bn
                if p % 2 == 0:     # push: rows into every arena, then the flags
                    m2 = dict(mem_d)
                    for dst in range(world):
                        m2[(region, dst, r)] = e
                    f2 = list(flags)
                    f2[r] = max(f2[r], e + 1)      # epochs are monotone: a word never goes back
                    nb, ns = (bn, tuple(f2)) if shared_flags else (tuple(f2), st)
                    succ.append(((pc_bn[:r] + (p + 1,) + pc_bn[r + 1:], pc_st, nb, ns, frozenset(m2.items())),
                                 (r, "push", e)))
                elif all(flags[s] >= e + 1 for s in range(world)):
                    for s in range(world):
                        if mem_d.get((region, r, s)) != e:
                            return "bad_row", trace + ((r, "combine", e, "row of", s, "holds", mem_d.get((region, r, s))),)
                    succ.append(((pc_bn[:r] + (p + 1,) + pc_bn[r + 1:], pc_st, bn, st, mem), (r, "combine", e)))
            q = pc_st[r]
            if q < 2 * staged:
                e = q // 2
                # a bucket exchange's epochs are its own counter; with shared flags they land in the same words
                target = e + 1 + (n_bn if shared_flags else 0)
                if q % 2 == 0:
                    s2 = list(st)
                    s2[r] = max(s2[r], target)
                    succ.append(((pc_bn, pc_st[:r] + (q + 1,) + pc_st[r + 1:], bn, tuple(s2), mem), (r, "arrive", e)))
                elif all(st[s] >= target for s in range(world)):
                    succ.append(((pc_bn, pc_st[:r] + (q + 1,) + pc_st[r + 1:], bn, st, mem), (r, "wait", e)))
        if not succ:
            if any(p < n_bn for p in pc_bn) or any(q < 2 * staged for q in pc_st):
                return "deadlock", trace
            continue
        for s, step in succ:
            stack.append((s, trace + (step,)))
    return None


# one training step and the next: layer 0 is a shared module applied twice in a row, layer 1 once
_PROGRAM = [(0, "f"), (0, "f"), (1, "f"), (1, "b"), (0, "b"), (0, "b")] * 2


@pytest.mark.parametrize("world", [2, 3])
def test_protocol_model_is_safe_and_deadlock_free(world):
    assert _check_protocol(world, _PROGRAM if world == 2 else _PROGRAM[:6], staged=2 if world == 2 else 1) is None


def test_protocol_model_finds_the_overwrite_without_the_double_buffer():
    """A fast rank pushes the second application of the shared layer into the row a slow rank has not combined."""
    res = _check_protocol(2, _PROGRAM[:6], generations=1)
    assert res is not None and res[0] == "bad_row", res


def test_protocol_model_needs_its_own_flag_words():
    """Signalling through the bucket exchange's words lets a bucket arrival satisfy a BN wait early."""
    res = _check_protocol(2, _PROGRAM[:6], shared_flags=True)
    assert res is not None and res[0] == "bad_row", res


# ---- conversion and plumbing ------------------------------------------------------------------------------------
class _Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 5, 3)
        self.bn2 = torch.nn.BatchNorm2d(5)
        self.inner = torch.nn.Sequential(torch.nn.Linear(5, 7), torch.nn.BatchNorm1d(7, affine=False))
        self.bn3 = torch.nn.BatchNorm3d(2, momentum=None)
        self.sync = torch.nn.SyncBatchNorm(4)
        self.ln = torch.nn.LayerNorm(4)


def test_conversion_keeps_parameters_and_buffers_and_numbers_layers():
    from ray_lightning_b200.syncbn import B200SyncBatchNorm, convert_sync_batchnorm, sync_batchnorm_layers
    net = _Net()
    before = {n: m for n, m in net.named_modules()}
    params = {n: p for n, p in net.named_parameters()}
    buffers = {n: b for n, b in net.named_buffers()}
    getter = lambda: None
    out = convert_sync_batchnorm(net, getter)
    assert out is net
    layers = sync_batchnorm_layers(out)
    assert [type(before[n]).__name__ for n, m in out.named_modules() if isinstance(m, B200SyncBatchNorm)] == \
        ["BatchNorm2d", "BatchNorm1d", "BatchNorm3d", "SyncBatchNorm"]
    assert [m.layer_id for m in layers] == [0, 1, 2, 3]
    assert all(isinstance(m, torch.nn.SyncBatchNorm) for m in layers)
    assert type(out.conv) is torch.nn.Conv2d and type(out.ln) is torch.nn.LayerNorm
    for n, p in out.named_parameters():
        assert p is params[n], n
    for n, b in out.named_buffers():
        assert b is buffers[n], n
    assert out.inner[1].weight is None and out.bn3.momentum is None


def test_state_dict_interchanges_with_torch_modules():
    from ray_lightning_b200.syncbn import convert_sync_batchnorm
    torch.manual_seed(0)
    plain = _Net()
    with torch.no_grad():
        for b in plain.buffers():
            if b.dtype == torch.float32:
                b.uniform_(0.5, 1.5)
    ours = convert_sync_batchnorm(_Net(), lambda: None)
    ours.load_state_dict(plain.state_dict())
    torch_sync = torch.nn.SyncBatchNorm.convert_sync_batchnorm(_Net())
    torch_sync.load_state_dict(ours.state_dict())
    assert ours.state_dict().keys() == plain.state_dict().keys() == torch_sync.state_dict().keys()
    for k, v in plain.state_dict().items():
        assert torch.equal(ours.state_dict()[k], v) and torch.equal(torch_sync.state_dict()[k], v), k
    # a pickled module (a checkpoint of the whole module) does not carry the worker's communicator
    back = pickle.loads(pickle.dumps(ours))
    assert back.bn2._comm_getter is None and back.bn2.layer_id == 0


def test_without_a_communicator_it_is_batchnorm():
    """World 1 / no communicator: plain batch norm, running statistics and the batch counter updated as torch does."""
    from ray_lightning_b200.syncbn import convert_sync_batchnorm
    torch.manual_seed(1)
    a = torch.nn.Sequential(torch.nn.BatchNorm2d(6))
    b = convert_sync_batchnorm(torch.nn.Sequential(torch.nn.BatchNorm2d(6)), lambda: None)
    x = torch.randn(4, 6, 5, 5)
    for m in (a, b):
        m.train()
    ya, yb = a(x), b(x)
    assert torch.equal(ya, yb)
    for (n, u), (_, v) in zip(a.state_dict().items(), b.state_dict().items()):
        assert torch.equal(u, v), n
    a.eval(); b.eval()
    assert torch.equal(a(x), b(x))


def test_conversion_refuses_what_it_cannot_synchronise():
    from ray_lightning_b200.syncbn import convert_sync_batchnorm
    half = torch.nn.BatchNorm1d(3).to(torch.float16)
    with pytest.raises(ValueError, match="float32"):
        convert_sync_batchnorm(torch.nn.Sequential(half), lambda: None)
    sub = torch.nn.SyncBatchNorm(3)
    sub.process_group = object()     # a subgroup (no process group is initialised here)
    with pytest.raises(ValueError, match="whole world"):
        convert_sync_batchnorm(torch.nn.Sequential(sub), lambda: None)


def test_arena_bytes_for_resnet50():
    """About 32 x W x sum(C) bytes: 6.8 MB for ResNet-50's 26 560 BN channels at W = 8."""
    import torchvision
    from ray_lightning_b200.syncbn import syncbn_arena_bytes
    chans = [m.num_features for m in torchvision.models.resnet50().modules() if isinstance(m, torch.nn.BatchNorm2d)]
    assert len(chans) == 53 and sum(chans) == 26560
    nbytes = syncbn_arena_bytes(chans, 8)
    assert 32 * 8 * 26560 <= nbytes <= 32 * 8 * 26560 + 53 * (256 + 2 * 8 * 64)


def test_strategies_pick_the_conversion():
    """libb2d's module on the libb2d path; torch's SyncBatchNorm with b200_enable=False, use_gpu=False, or a comm hook
    of the user's (the reference behaviour)."""
    import warnings
    from torch.distributed.algorithms.ddp_comm_hooks import default_hooks
    from ray_lightning_b200 import RayShardedStrategy, RayStrategy
    from ray_lightning_b200.syncbn import B200SyncBatchNorm

    def kind(strategy, cuda):
        if cuda:
            strategy.root_device = torch.device("cuda", 0)     # what a GPU worker sees; conversion itself needs no GPU
        m = strategy.configure_sync_batchnorm(torch.nn.Sequential(torch.nn.BatchNorm2d(3)))
        return type(m[0])

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        assert kind(RayStrategy(num_workers=2, use_gpu=True), True) is B200SyncBatchNorm
        assert kind(RayShardedStrategy(num_workers=2, use_gpu=True), True) is B200SyncBatchNorm
        assert kind(RayStrategy(num_workers=2, use_gpu=True, b200_enable=False), True) is torch.nn.SyncBatchNorm
        assert kind(RayStrategy(num_workers=2, use_gpu=False), False) is torch.nn.SyncBatchNorm
        assert kind(RayShardedStrategy(num_workers=2, use_gpu=False), False) is torch.nn.SyncBatchNorm
        hooked = RayStrategy(num_workers=2, use_gpu=True, ddp_comm_hook=default_hooks.allreduce_hook)
        assert kind(hooked, True) is torch.nn.SyncBatchNorm


def test_trainer_flag_reaches_configure_sync_batchnorm():
    from ray_lightning_b200._runtime import minipl
    from utils import BoringModel

    class Recording(minipl.DDPSpawnStrategy):
        calls = []

        def configure_sync_batchnorm(self, model):
            Recording.calls.append(type(model).__name__)
            return super().configure_sync_batchnorm(model)

        def configure_ddp(self):
            Recording.calls.append("configure_ddp")

    for flag in (False, True):
        Recording.calls = []
        model = BoringModel()
        model.norm = torch.nn.BatchNorm1d(2)
        s = Recording(accelerator="cpu", parallel_devices=[])
        t = minipl.Trainer(strategy=s, sync_batchnorm=flag, enable_checkpointing=False)
        s.connect(model)
        t.state.fn = minipl.TrainerFn.FITTING
        s.setup(t)
        if flag:
            assert Recording.calls == ["BoringModel", "configure_ddp"]
            assert type(model.norm) is torch.nn.SyncBatchNorm
        else:
            assert Recording.calls == ["configure_ddp"] and type(model.norm) is torch.nn.BatchNorm1d
