"""libb2d's exchange kernels at every world size from 2 to 8, at non-default launch geometry, with guard bytes around
every output, on loopback ranks of one H100.

The arithmetic of these kernels is pinned elsewhere; this file pins their index math: which thread touches which pack
for a given world size, grid and chunking.  W = 2, 4 and 8 run specialisations, every other W the generic build
(dispatch_world).  The sizes are derived from each kernel's geometry at the grid `ctx.plan()` reports (empty slices,
k x W +- 1 packs, a slice of exactly one grid-stride batch and one pack either side, many batches per thread, the
macro tiles of K2T, ragged last packs and chunks), and every configuration first asserts that plan() returns the grid
the test expects, so that a knob which stopped applying cannot leave the sweep vacuous.  Results are bit-exact against
oracle/ddp_oracle.py on every rank, and the optimizer steps bit-exact against torch's foreach Adam on CUDA.

Every output sits between two GUARD-float margins of a NaN canary (0x7fc0beef plus a per-rank salt) compared as bits:
a store one element past a bucket, a shard or a segment fails the test even where the values inside are right.

Co-residency: on one GPU the loopback ranks of the single-kernel algorithms (K1, K2, K2T, K5) spin on each other's
blocks, so W x grid must fit on the device at once, or the kernels wait until the watchdog traps.  `knobs` asserts
W x max_ctas, W x tma_ctas and W x exch_ctas <= BUDGET (LoopbackGroup's 128 CTAs) before it sets anything; the
exchange kernel of the staged path outranks the stage kernels it waits for, so its grid is held to the same budget.
Larger grids run on CPU threads only (test_kernel_emulation.py)."""
import contextlib
import itertools

import numpy as np
import pytest
import torch

from oracle import ddp_oracle

pytestmark = pytest.mark.gpu

BUDGET = 128
CANARY = 0x7fc0beef
GUARD = 16                  # 64 bytes: a view behind the margin keeps the allocation's 16-byte alignment
WORLDS = [2, 3, 4, 5, 6, 7, 8]
ADAM = dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, adamw=True)
_groups = {}
_ids = itertools.count(1)   # a fresh bucket id per call: no slot ever changes geometry (which would add a barrier launch)


def default_knobs(world):
    return dict(max_ctas=BUDGET // world, tma_ctas=min(48, BUDGET // world), exch_ctas=min(64, BUDGET // world),
                chunk_bytes=64 << 20)


def _apply(g, max_ctas=None, tma_ctas=None, exch_ctas=None, chunk_bytes=None):
    for name, v in (("max_ctas", max_ctas), ("tma_ctas", tma_ctas), ("exch_ctas", exch_ctas)):
        assert v is None or g.world * v <= BUDGET, \
            "%s = %d at W = %d: %d CTAs do not fit the co-residency budget of %d" % (name, v, g.world, g.world * v, BUDGET)
    for rk in g.ranks:
        if max_ctas is not None:
            rk.ctx.set_max_ctas(max_ctas)            # caps tma_ctas too: set it first
        if tma_ctas is not None:
            rk.ctx.set_tma_ctas(tma_ctas)
        if exch_ctas is not None:
            rk.ctx.set_exch_ctas(exch_ctas)
        if chunk_bytes is not None:
            rk.ctx.set_chunk_bytes(chunk_bytes)


@contextlib.contextmanager
def knobs(g, **kw):
    """Set launch knobs on every rank (co-residency checked first), restore the defaults afterwards."""
    try:
        _apply(g, **kw)
        yield {**default_knobs(g.world), **kw}
    finally:
        _apply(g, **default_knobs(g.world))


def group(world):
    """A fresh loopback group per test, at the default knobs of this file: every call takes a bucket slot of its own,
    and closing the previous group gives its arena back."""
    from ray_lightning_b200.comm import LoopbackGroup
    teardown_module(None)
    g = LoopbackGroup(world, 0, arena_bytes=(512 if world <= 4 else 256) << 20, timeout_ms=20000)
    _apply(g, **default_knobs(world))
    _groups[world] = g
    return g


def teardown_module(module):
    for g in _groups.values():
        g.close()
    _groups.clear()


# ---- geometry the library computes (b2d.cu / b2d_kernels.cuh), restated ----------------------------------------------
def packs_per_batch(per_pack):
    return 16 // per_pack if per_pack > 0 and 16 // per_pack > 1 else 1


def specialisation(world):
    return world if world in (2, 4, 8) else 0


def clamp_grid(work, per_cta, cap):
    return min(max(-(-work // per_cta), 1), cap)


def chunk_packs(world, chunk_bytes):
    unit = world * 1024
    return max(chunk_bytes // 16 // unit * unit, unit)


def exch_per_thread(world):
    return 16 // world if 16 // world > 1 else 1


def expected_plan(world, n, wire, algo, kn):
    """(algo, grid) that b2d_plan must report for this bucket at knobs `kn`."""
    from ray_lightning_b200 import _b2d
    epp = 8 if wire == "bf16" else 4
    npacks = -(-n // epp)
    slice_ = -(-npacks // world)
    if algo == "staged":
        chunk = min(npacks, chunk_packs(world, kn["chunk_bytes"]))
        return _b2d.ALGO_STAGED, clamp_grid(-(-chunk // world), 256 * exch_per_thread(world), kn["exch_ctas"])
    if algo == "two_shot_tma":
        if wire == "bf16" and n % 8 == 0:
            return _b2d.ALGO_TWO_SHOT_TMA, clamp_grid(slice_, 256, kn["tma_ctas"])
        algo = "two_shot"                                          # the documented fall-back
    if algo == "two_shot":
        return _b2d.ALGO_TWO_SHOT, clamp_grid(slice_, 512, kn["max_ctas"])
    return _b2d.ALGO_ONE_SHOT, clamp_grid(npacks, 512, kn["max_ctas"])


def tma_mt(slice_, grid):
    mt = -(-slice_ // grid)
    return min(max(-(-mt // 8) * 8, 8), 4096)


# ---- buffers and comparisons --------------------------------------------------------------------------------------
def rank_inputs(world, n, seed):
    return [torch.randn(n, generator=torch.Generator().manual_seed(7919 * seed + r)) * 2.0 ** -4 for r in range(world)]


def oracle(per_rank, wire):
    return (ddp_oracle.allreduce_bf16_wire if wire == "bf16" else ddp_oracle.allreduce_fp32_wire)(per_rank)


def wire_sum(per_rank, wire, scale):
    """The reduced gradient an owner receives: fp32 sum in rank order of the wire values, not rounded again."""
    if wire == "fp32":
        return ddp_oracle.allreduce_fp32_wire(per_rank, scale)
    out = None
    for t in per_rank:
        c = ddp_oracle.wire_bf16(t, scale)
        out = c if out is None else out + c
    return out


def guarded(values, salt, whole=None):
    """(whole, view): `values` (a CPU tensor) on the GPU between two canary margins.  `whole` may be given (an arena
    tensor of at least values.numel() + 2 * GUARD elements)."""
    n = values.numel()
    if whole is None:
        whole = torch.empty(n + 2 * GUARD, device="cuda")
    whole = whole[:n + 2 * GUARD]
    whole.view(torch.int32).fill_(CANARY + salt)
    view = whole[GUARD:GUARD + n]
    view.copy_(values)
    return whole, view


def args(pairs):
    """The views of guarded buffers as kernel arguments.  An empty view has no data pointer, and the library refuses a
    NULL buffer (after the other ranks launched, which would leave them waiting): an empty shard passes a pointer into
    its own margin instead, which the kernels must leave alone like any other margin."""
    return [view if view.numel() else whole[GUARD:GUARD + 1] for whole, view in pairs]


def guards_intact(whole, n, salt):
    u = whole.view(torch.int32)
    return bool((u[:GUARD] == CANARY + salt).all()) and bool((u[GUARD + n:] == CANARY + salt).all())


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.to(a.device).contiguous().view(torch.int32))


def ragged(npacks, epp, i):
    """A bucket of `npacks` packs whose last pack holds 1, epp - 1 or epp elements, by turns."""
    return npacks * epp - (epp - 1, 1, 0)[i % 3]


def run_allreduce(g, algo, wire, n, kn, seed, salt0=0):
    """One allreduce of guarded buckets; checks the plan, the launch, every rank's bits and every margin."""
    from ray_lightning_b200 import _b2d
    world = g.world
    a, grid = expected_plan(world, n, wire, algo, kn)
    got = g.ranks[0].ctx.plan(n, _b2d.WIRE_NAMES[wire], _b2d.ALGO_NAMES[algo])
    assert got[:2] == (a, grid), (world, algo, wire, n, kn, got, (a, grid))
    per_rank = rank_inputs(world, n, seed)
    held = [guarded(t, salt0 + r) for r, t in enumerate(per_rank)]
    torch.cuda.synchronize()
    before = g.ranks[0].ctx.stats()["launches"]
    g.allreduce_([v for _, v in held], bucket_idx=next(_ids), wire=wire, algo=algo)
    g.synchronize()
    st = g.ranks[0].ctx.stats()
    last_grid = grid
    if algo == "staged":                     # 4 launches per chunk; stats report the last chunk's exchange grid
        npacks, cp = -(-n // (8 if wire == "bf16" else 4)), chunk_packs(world, kn["chunk_bytes"])
        nchunks = -(-npacks // cp)
        assert st["launches"] - before == 4 * nchunks, (world, wire, n, kn, st)
        last_grid = clamp_grid(-(-(npacks - (nchunks - 1) * cp) // world), 256 * exch_per_thread(world), kn["exch_ctas"])
    assert (st["last_algo"], st["last_grid"]) == (a, last_grid), (world, algo, wire, n, st)
    want = oracle(per_rank, wire).cuda()
    for r, (whole, view) in enumerate(held):
        assert same_bits(view, want), (world, algo, wire, n, kn, r)
        assert guards_intact(whole, n, salt0 + r), (world, algo, wire, n, kn, r)
    return a, grid


# ---- 1. worlds 2-8 x every P2P algorithm x a grid sweep ----------------------------------------------------------------
def _sweep(world, algo):
    w = BUDGET // world
    if algo == "two_shot_tma":
        return [dict(tma_ctas=c) for c in sorted({1, 3, 5, w})]
    if algo == "staged":
        return [dict(exch_ctas=c) for c in sorted({1, 2, 3, 5, w})]
    return [dict(max_ctas=c) for c in sorted({1, 2, 3, 7, w})]


def _counts(world, algo, grid):
    """Pack counts at `grid` blocks: fewer than W, k x W - 1 / k x W / k x W + 1, a bucket (K1) or a slice (K2, the
    staged exchange) of exactly one grid-stride batch and one pack either side, and many batches per thread (several
    MiB of bucket at grid 1)."""
    if algo == "staged":
        batch = grid * 256 * exch_per_thread(world)     # a multiple of grid x 256 threads x U of the exchange kernel
    else:
        batch = grid * 512 * packs_per_batch(specialisation(world))
    many = [40] if grid == 1 else ([3] if grid < 8 else [])
    if algo == "one_shot":
        return sorted({1, max(world - 1, 1), 2 * world - 1, 2 * world + 1, batch - 1, batch, batch + 1} |
                      {k * batch + 5 for k in many})
    return sorted({1, max(world - 1, 1), 2 * world - 1, 2 * world, 2 * world + 1, world * batch - 1, world * batch,
                   world * batch + 1, world * (batch + 1)} | {k * world * batch + 5 for k in many})


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("algo", ["one_shot", "two_shot", "staged"])
def test_allreduce_grid_sweep(world, algo):
    """K1, K2 and the staged exchange (K7-K10) at every grid of the sweep, both wires, ragged last packs."""
    g = group(world)
    for cfg in _sweep(world, algo):
        with knobs(g, **cfg) as kn:
            grid = list(cfg.values())[0]
            for i, npacks in enumerate(_counts(world, algo, grid)):
                for wire in ("bf16", "fp32"):
                    n = ragged(npacks, 8 if wire == "bf16" else 4, i)
                    run_allreduce(g, algo, wire, n, kn, seed=i)


@pytest.mark.parametrize("world", WORLDS)
def test_tma_two_shot_macro_tiles(world):
    """K2T at every TMA grid of the sweep: mt = 8 (slices of up to 8 packs, empty slices), an mt that is not a multiple
    of W (phase 1 then has part x W < mt), mt = 4096 with several macro tiles per block and, at one block, a bucket
    whose phase-1 job list wraps the 3-slot mbarrier ring at least 10 times; n % 8 != 0 falls back to K2."""
    from ray_lightning_b200 import _b2d
    g = group(world)
    seen = set()
    for cfg in _sweep(world, "two_shot_tma"):
        with knobs(g, **cfg) as kn:
            t = cfg["tma_ctas"]
            slices = [1, 8, 1020 * t + 1] + ([8192 * t + 24] if t <= 5 else [])
            if t == 1:
                slices.append(15 * 4096 + 24)
            for i, s in enumerate(slices):
                for npacks in sorted({world * s, world * s - 1, max(world * (s - 1) + 1, 1)}):
                    n = 8 * npacks
                    a, grid = run_allreduce(g, "two_shot_tma", "bf16", n, kn, seed=100 + i)
                    assert a == _b2d.ALGO_TWO_SHOT_TMA
                    sl = -(-npacks // world)
                    mt = tma_mt(sl, grid)
                    seen.add(mt)
                    if s == 15 * 4096 + 24:
                        part = mt // world
                        parts = -(-mt // part)
                        assert grid == 1 and -(-sl // mt) * parts >= 30        # >= 10 wraps of the ring in phase 1
                for n in (8 * world * s + 1, 8 * world * s + 7):
                    a, _ = run_allreduce(g, "two_shot_tma", "bf16", n, kn, seed=200 + i)
                    assert a == _b2d.ALGO_TWO_SHOT
    assert 8 in seen and 4096 in seen
    if world in (3, 5, 6, 7):
        assert any(m % world for m in seen)
    # the fp32 wire falls back too
    run_allreduce(g, "two_shot_tma", "fp32", 8 * 4096, default_knobs(world), seed=300)


@pytest.mark.parametrize("world", WORLDS)
def test_staged_in_place_next_to_a_neighbour(world):
    """fp32 buckets that live in the arena (n % 4 = 1, 2, 3), two side by side with canary margins before, between and
    after them, at every exchange grid of the sweep: the second exchange must leave the first result and every margin
    alone, and each ragged last pack stops at its last element.  3 launches (arrive, exchange, wait) per bucket."""
    g = group(world)
    scale = float(np.float32(1.0) / np.float32(world))
    sweep = []
    for cfg in _sweep(world, "staged"):
        batch = cfg["exch_ctas"] * 256 * exch_per_thread(world)
        sweep.append((cfg, [1, max(world - 1, 1), 2 * world + 1, world * batch - 1, world * batch, world * batch + 1] +
                      ([20 * world * batch + 5] if cfg["exch_ctas"] == 1 else [])))
    arena = [rk.arena_tensor(8 * max(max(c) for _, c in sweep) + 8 * GUARD) for rk in g.ranks]
    for cfg, counts in sweep:
        with knobs(g, **cfg) as kn:
            for i, npacks in enumerate(counts):
                nb = npacks * 4 - (3, 2, 1)[i % 3]
                na = max(counts[(i + 3) % len(counts)] * 4 - (1, 3, 2)[i % 3], 1)
                a0 = GUARD
                b0 = -(-(a0 + na) // 4) * 4 + GUARD
                size = b0 + nb + GUARD
                assert size <= arena[0].numel()
                per_a, per_b = rank_inputs(world, na, 400 + i), rank_inputs(world, nb, 500 + i)
                for r in range(world):
                    arena[r][:size].view(torch.int32).fill_(CANARY + r)
                    arena[r][a0:a0 + na].copy_(per_a[r])
                    arena[r][b0:b0 + nb].copy_(per_b[r])
                torch.cuda.synchronize()
                for off, n in ((a0, na), (b0, nb)):
                    before = g.ranks[0].ctx.stats()["launches"]
                    g.allreduce_([t[off:off + n] for t in arena], bucket_idx=next(_ids), wire="fp32", algo="staged")
                    g.synchronize()
                    assert g.ranks[0].ctx.stats()["launches"] - before == 3, (world, kn, n)
                mask = torch.ones(size, dtype=torch.bool, device="cuda")
                mask[a0:a0 + na] = False
                mask[b0:b0 + nb] = False
                wa = ddp_oracle.allreduce_fp32_wire(per_a, scale).cuda()
                wb = ddp_oracle.allreduce_fp32_wire(per_b, scale).cuda()
                for r in range(world):
                    assert same_bits(arena[r][a0:a0 + na], wa), (world, kn, na, r)
                    assert same_bits(arena[r][b0:b0 + nb], wb), (world, kn, nb, r)
                    assert bool((arena[r][:size].view(torch.int32)[mask] == CANARY + r).all()), (world, kn, na, nb, r)


@pytest.mark.parametrize("world", WORLDS)
def test_staged_chunk_pipeline(world):
    """Chunks of 64 KiB and of 64 KiB + 16 bytes of wire (rounded by the library to W x 1024 packs): 1, 2 and 6 chunks
    with the ragged pack in the last one, both wires through the stage / write-back kernels (4 launches per chunk)
    and fp32 in place (an arrive, then an exchange and a wait per chunk)."""
    g = group(world)
    arena = [rk.arena_tensor(1 << 21) for rk in g.ranks]
    scale = float(np.float32(1.0) / np.float32(world))
    for cb in (64 << 10, (64 << 10) + 16):
        with knobs(g, chunk_bytes=cb) as kn:
            cp = chunk_packs(world, cb)
            for i, npacks in enumerate((cp - 3, cp + 5, 5 * cp + cp // 2 + 1)):
                nchunks = -(-npacks // cp)
                for wire in ("bf16", "fp32"):
                    run_allreduce(g, "staged", wire, ragged(npacks, 8 if wire == "bf16" else 4, i), kn, seed=600 + i)
                n = npacks * 4 - (1 + i % 3)
                assert n + 2 * GUARD <= arena[0].numel()
                per_rank = rank_inputs(world, n, 700 + i)
                held = [guarded(t, r, whole=arena[r]) for r, t in enumerate(per_rank)]
                torch.cuda.synchronize()
                before = g.ranks[0].ctx.stats()["launches"]
                g.allreduce_([v for _, v in held], bucket_idx=next(_ids), wire="fp32", algo="staged")
                g.synchronize()
                assert g.ranks[0].ctx.stats()["launches"] - before == 1 + 2 * nchunks, (world, cb, n)
                want = ddp_oracle.allreduce_fp32_wire(per_rank, scale).cuda()
                for r, (whole, view) in enumerate(held):
                    assert same_bits(view, want), (world, cb, n, r)
                    assert guards_intact(whole, n, r), (world, cb, n, r)


@pytest.mark.parametrize("wire", ["bf16", "fp32"])
def test_k0_world1_guard_bytes(wire):
    """K0 (world 1): the scalar tail of 1-3 elements and the grid-stride vectors stop at the bucket's end."""
    from ray_lightning_b200 import _b2d
    ctx = _b2d.Context(0, 1, 0, 1 << 20)
    try:
        st = torch.cuda.current_stream()
        for i, n in enumerate((1, 2, 3, 5, 4099, 65537, (1 << 20) + 2, (1 << 22) + 3)):
            x = rank_inputs(1, n, 800 + i)[0]
            whole, view = guarded(x, 0)
            ctx.allreduce_bucket(0, view.data_ptr(), n, _b2d.WIRE_NAMES[wire], 1.0, 0, st, st)
            torch.cuda.synchronize()
            assert same_bits(view, oracle([x], wire)), (wire, n)
            assert guards_intact(whole, n, 0), (wire, n)
    finally:
        ctx.destroy()


# ---- 2. the sharded path at W = 2 ... 8 ------------------------------------------------------------------------------
def torch_adam_steps(p0, grads):
    """torch.optim.AdamW (foreach, CUDA) from a fresh state over the given flat gradients: [(p, exp_avg, exp_avg_sq)]."""
    prm = torch.nn.Parameter(p0.cuda().clone())
    opt = torch.optim.AdamW([prm], lr=ADAM["lr"], betas=(ADAM["beta1"], ADAM["beta2"]), eps=ADAM["eps"],
                            weight_decay=ADAM["weight_decay"], foreach=True)
    out = []
    for gr in grads:
        prm.grad = gr.cuda().clone()
        opt.step()
        st = opt.state[prm]
        out.append((prm.detach().clone(), st["exp_avg"].clone(), st["exp_avg_sq"].clone()))
    return out


def layouts(world):
    """Owner layouts: FairScale's partition of random sizes; W - 1 parameters, so the last owner's shard is empty."""
    rng = np.random.default_rng(world)
    fair = [int(x) for x in rng.integers(1, 3000, size=23)] + [40000, 8, 1]
    return {"fairscale": fair, "empty_owner": [30011, 1203, 805, 640, 96, 51, 9][:world - 1]}


def guarded_shards(shard_off, fill, salt0=0):
    return [guarded(torch.full((shard_off[r + 1] - shard_off[r],), fill), salt0 + r) for r in range(len(shard_off) - 1)]


def arena_params(g, p0):
    """The flat parameters in every rank's arena, between canary margins."""
    out = []
    for r, rk in enumerate(g.ranks):
        out.append(guarded(p0, r, whole=rk.arena_tensor(p0.numel() + 2 * GUARD)))
    return out


@pytest.mark.parametrize("world", WORLDS)
def test_sharded_step_geometry(world):
    """K4 + K5 + K6 (sharded_step_) at max_ctas 1, 3 and the default, both wires, two steps: every rank's parameters
    and every owner's exp_avg / exp_avg_sq bit for bit against torch's foreach AdamW on CUDA on the oracle's reduced
    gradients; then K4 alone (reduce_scatter) and K6 alone (allgather).  Guard bytes around every output."""
    g = group(world)
    scale = float(np.float32(1.0) / np.float32(world))
    for name, numels in layouts(world).items():
        owner = ddp_oracle.partition_fairscale(numels, world)
        _, shard_off, total = ddp_oracle.shard_layout(numels, owner, world)
        if name == "empty_owner":
            assert shard_off[world - 1] == shard_off[world]
        max_len = max(shard_off[r + 1] - shard_off[r] for r in range(world))
        for mc in sorted({1, 3, BUDGET // world}):
            with knobs(g, max_ctas=mc):
                for wire in ("fp32", "bf16"):
                    epp = 8 if wire == "bf16" else 4
                    p0 = torch.randn(total, generator=torch.Generator().manual_seed(mc))
                    params = arena_params(g, p0)
                    ms, vs = guarded_shards(shard_off, 0.0), guarded_shards(shard_off, 0.0)
                    per_step = [[torch.randn(total, generator=torch.Generator().manual_seed(100 * s + r)) * 0.1 for r in range(world)]
                                for s in (1, 2)]
                    want = torch_adam_steps(p0, [wire_sum(pr, wire, scale) for pr in per_step])
                    slot = next(_ids)
                    for s, per_rank in enumerate(per_step):
                        grads = [guarded(t, r) for r, t in enumerate(per_rank)]
                        torch.cuda.synchronize()
                        g.sharded_step_(args(grads), args(params), args(ms), args(vs),
                                        shard_off, step=s + 1, lr=ADAM["lr"], betas=(ADAM["beta1"], ADAM["beta2"]), eps=ADAM["eps"],
                                        weight_decay=ADAM["weight_decay"], adamw=True, zero_grads=True, wire=wire, slot=slot)
                        g.synchronize()
                        assert g.ranks[0].ctx.stats()["last_grid"] == clamp_grid(max_len // epp, 512, mc)
                        wp, wm, wv = want[s]
                        for r in range(world):
                            lo, hi = shard_off[r], shard_off[r + 1]
                            what = (world, name, mc, wire, s, r)
                            assert same_bits(params[r][1], wp) and guards_intact(params[r][0], total, r), what
                            assert same_bits(ms[r][1], wm[lo:hi]) and guards_intact(ms[r][0], hi - lo, r), what
                            assert same_bits(vs[r][1], wv[lo:hi]) and guards_intact(vs[r][0], hi - lo, r), what
                            assert bool((grads[r][1] == 0).all()) and guards_intact(grads[r][0], total, r), what
                    # K4 alone
                    per_rank = rank_inputs(world, total, 900 + mc)
                    grads = [t.cuda() for t in per_rank]
                    outs = guarded_shards(shard_off, 7.0)
                    torch.cuda.synchronize()
                    g.reduce_scatter(grads, args(outs), shard_off, wire=wire, slot=next(_ids))
                    g.synchronize()
                    red = wire_sum(per_rank, wire, scale).cuda()
                    for r in range(world):
                        lo, hi = shard_off[r], shard_off[r + 1]
                        assert same_bits(outs[r][1], red[lo:hi]) and guards_intact(outs[r][0], hi - lo, r), (world, name, mc, wire, r)
                # K6 alone
                full = torch.randn(total, generator=torch.Generator().manual_seed(950 + mc))
                bufs = arena_params(g, torch.zeros(total))
                for r in range(world):
                    bufs[r][1][shard_off[r]:shard_off[r + 1]] = full[shard_off[r]:shard_off[r + 1]].cuda()
                torch.cuda.synchronize()
                g.allgather_([v for _, v in bufs], shard_off)
                g.synchronize()
                assert g.ranks[0].ctx.stats()["last_grid"] == clamp_grid(max_len // 4, 512, mc)
                for r in range(world):
                    assert same_bits(bufs[r][1], full) and guards_intact(bufs[r][0], total, r), (world, name, mc, r)


def owner_buckets(world, kind):
    """(numels, owner, offsets, shard_off, total, [bucket0, bucket1]).  "empty_owner": W - 1 parameters (the last owner
    has an empty shard) and a first bucket whose segments all belong to owner 0 (every other owner has none in it);
    "deep": 4000 eight-element parameters and a first bucket of >= 2000 segments that do not touch (every other
    parameter of each owner), so that seg_find searches a deep table."""
    numels = [30011, 1203, 805, 640, 96, 51, 9][:world - 1] if kind == "empty_owner" else [8] * 4000
    owner = ddp_oracle.partition_fairscale(numels, world)
    offs, shard_off, total = ddp_oracle.shard_layout(numels, owner, world)
    if kind == "empty_owner":
        first = [i for i in range(len(numels)) if owner[i] == 0]
    else:
        first = [i for i in range(len(numels)) if (i // world) % 2 == 0]
    rest = [i for i in range(len(numels)) if i not in set(first)]
    buckets = [[(offs[i], -(-numels[i] // 8) * 8, owner[i]) for i in part] for part in (first, rest) if part]   # W = 2: one
    return numels, owner, offs, shard_off, total, buckets


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("kind", ["empty_owner", "deep"])
def test_owner_path_geometry(world, kind):
    """K11 + K12 (register_bucket / reduce_to_owner) at exch_ctas 1, 3 and the default, both wires, then K13
    (adam_push_) bit for bit against torch's foreach AdamW on CUDA on the oracle's reduced gradients.  K11 zeroes
    exactly the bucket's segments; K12 writes exactly the bucket's part of each owner's shard, and reducing the second
    bucket leaves the first one's results alone; guard bytes around the gradients, the reduced shards, exp_avg /
    exp_avg_sq and the flat parameters on every rank."""
    g = group(world)
    scale = float(np.float32(1.0) / np.float32(world))
    numels, owner, offs, shard_off, total, buckets = owner_buckets(world, kind)
    if kind == "empty_owner":
        assert shard_off[world - 1] == shard_off[world] and {o for _, _, o in buckets[0]} == {0}
    else:
        assert len(buckets[0]) >= 2000
    n_own = [shard_off[r + 1] - shard_off[r] for r in range(world)]
    for ec in sorted({1, 3, min(64, BUDGET // world)}):
        with knobs(g, exch_ctas=ec):
            for wire in ("bf16", "fp32"):
                epp = 8 if wire == "bf16" else 4
                ids = [next(_ids) for _ in buckets]
                for bid, segs in zip(ids, buckets):
                    g.register_bucket(bid, segs, wire)
                per_rank = [torch.randn(total, generator=torch.Generator().manual_seed(40 + r + ec)) * 0.1 for r in range(world)]
                grads = [guarded(t, r) for r, t in enumerate(per_rank)]
                reduced = guarded_shards(shard_off, 5.0)
                want = wire_sum(per_rank, wire, scale).cuda()
                done = torch.zeros(total, dtype=torch.bool, device="cuda")
                torch.cuda.synchronize()
                for bid, segs in zip(ids, buckets):
                    g.reduce_to_owner(bid, args(grads), args(reduced), shard_off, zero_grads=True)
                    g.synchronize()
                    for o, n, _ in segs:
                        done[o:o + n] = True
                    for r in range(world):
                        mine = sum(n // epp for _, n, o in segs if o == r)
                        assert g.ranks[r].ctx.stats()["last_grid"] == clamp_grid(mine, 256 * exch_per_thread(world), ec)
                        lo, hi = shard_off[r], shard_off[r + 1]
                        m = done[lo:hi]
                        red = reduced[r][1]
                        what = (world, kind, ec, wire, bid, r)
                        assert same_bits(red[m], want[lo:hi][m]) and bool((red[~m] == 5.0).all()), what
                        assert guards_intact(reduced[r][0], hi - lo, r), what
                        gv = grads[r][1]
                        assert bool((gv[done] == 0).all()) and same_bits(gv[~done], per_rank[r].cuda()[~done]), what
                        assert guards_intact(grads[r][0], total, r), what
                assert bool(done.all())
            # K13: one AdamW group per owner over its whole shard, two steps on the reduced gradients of the fp32 wire
            p0 = torch.randn(total, generator=torch.Generator().manual_seed(60 + ec))
            want_steps = torch_adam_steps(p0, [want.cpu(), want.cpu()])
            params = arena_params(g, p0)
            ms, vs = guarded_shards(shard_off, 0.0), guarded_shards(shard_off, 0.0)
            for s in (1, 2):
                groups = [[(0, n_own[r], dict(ADAM, step=s))] if n_own[r] else [] for r in range(world)]
                torch.cuda.synchronize()
                g.adam_push_(args(params), args(ms), args(vs), args(reduced), shard_off, groups)
                g.synchronize()
                wp, wm, wv = want_steps[s - 1]
                for r in range(world):
                    lo, hi = shard_off[r], shard_off[r + 1]
                    what = (world, kind, ec, s, r)
                    assert same_bits(params[r][1], wp) and guards_intact(params[r][0], total, r), what
                    assert same_bits(ms[r][1], wm[lo:hi]) and guards_intact(ms[r][0], hi - lo, r), what
                    assert same_bits(vs[r][1], wv[lo:hi]) and guards_intact(vs[r][0], hi - lo, r), what
