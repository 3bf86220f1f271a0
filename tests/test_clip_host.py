"""Gradient clipping without a GPU: the NumPy restatement of the global-norm kernels against exact norms and torch's
coefficient, the kernels themselves (csrc/b2d_clip.cuh, the scaled K13) on CPU threads bit for bit against it, a model
of the clip exchange next to reduce-to-owner and the step, the ShardedOptimizer host logic over a threaded test double,
and the Trainer plumbing on gloo workers."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import clip_ref as ref
from conftest import ROOT
from test_protocol_model import explore_owner
from test_sharded_host import FakeComm, _Net, make_model, run_ranks

EMU_DIR = os.path.join(ROOT, "ray_lightning_b200", "csrc", "emu")
FP = ctypes.POINTER(ctypes.c_float)
LP = ctypes.POINTER(ctypes.c_longlong)
SIGNAL_BYTES = 64 * 1024


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


# ---- the restatement -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 5, 4096, 4097, 3 * 4096 + 100, 300_001])
def test_restatement_is_the_exact_sum_of_squares(n):
    x = (np.random.default_rng(n).standard_normal(n) * 3).astype(np.float32)
    exact = math.fsum(float(v) * float(v) for v in x)
    p = ref.partial(x)
    assert abs(p - exact) <= 1e-13 * max(exact, 1.0)
    # the block cap changes only the order of exact-enough float64 adds
    assert abs(ref.partial(x, gmax=3) - exact) <= 1e-13 * max(exact, 1.0)
    norm, _ = ref.norm_coef([p], 1.0)
    assert norm == np.float32(math.sqrt(exact))


def test_restatement_coefficient_is_torchs():
    """K19's coefficient == torch's clip_grads_with_norm_ (max_norm / (norm + 1e-6), clamped to 1) on the same norm."""
    rng = np.random.default_rng(5)
    for i in range(3000):
        total = float(rng.uniform(0, 50)) ** 2 if i % 10 else float(rng.uniform(0, 1e-6))
        max_norm = float(rng.choice([rng.uniform(0, 10), 1.0, 0.0]))
        norm, coef = ref.norm_coef([total], max_norm)
        p = torch.nn.Parameter(torch.zeros(1))
        p.grad = torch.ones(1)
        torch.nn.utils.clip_grads_with_norm_([p], max_norm, torch.tensor(norm))
        assert _bits(p.grad.numpy()) == _bits([coef]), (total, max_norm)


def test_restatement_non_finite():
    norm, coef = ref.norm_coef([ref.partial(np.array([1.0, np.inf], np.float32))], 1.0)
    assert np.isinf(norm) and coef == 0.0
    norm, coef = ref.norm_coef([ref.partial(np.array([1.0, np.nan], np.float32))], 1.0)
    assert np.isnan(norm) and np.isnan(coef)


# ---- the kernels on CPU threads --------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu_clip") / "libb2d_emu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-fPIC", "-shared", "-DB2D_EMU", "-ffp-contract=off",
                    "-o", out, os.path.join(EMU_DIR, "emu_harness.cpp")], check=True)
    lib = ctypes.CDLL(out)
    lib.emu_group_create.restype = ctypes.c_void_p
    lib.emu_group_create.argtypes = [ctypes.c_int, ctypes.c_size_t]
    lib.emu_group_destroy.argtypes = [ctypes.c_void_p]
    lib.emu_clip_gmax.restype = ctypes.c_uint
    lib.emu_clip_norm.argtypes = [ctypes.c_void_p, ctypes.POINTER(FP), ctypes.POINTER(ctypes.c_size_t), ctypes.c_float,
                                  ctypes.POINTER(FP), ctypes.POINTER(FP), ctypes.c_size_t, ctypes.c_int, ctypes.c_uint,
                                  ctypes.c_uint, ctypes.c_int]
    push = [ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.POINTER(FP), ctypes.POINTER(FP), ctypes.POINTER(FP),
            ctypes.c_size_t, LP, ctypes.c_int, LP, LP, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float,
            ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_uint, ctypes.c_int, ctypes.c_int]
    lib.emu_adam_push.argtypes = push
    lib.emu_adam_push_scaled.argtypes = push + [ctypes.POINTER(FP)]
    lib.emu_arena_ptr.restype = FP
    lib.emu_arena_ptr.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t]
    return lib


def _ptrs(arrs):
    return (FP * len(arrs))(*[a.ctypes.data_as(FP) for a in arrs])


def test_library_block_cap_is_the_restatements(emu):
    assert emu.emu_clip_gmax() == ref.G_MAX


def _clip(emu, g, xs, max_norm, gen, epoch, order, gmax):
    world = len(xs)
    norms = [np.full(1, -1, np.float32) for _ in range(world)]
    coefs = [np.full(1, -1, np.float32) for _ in range(world)]
    ns = (ctypes.c_size_t * world)(*[len(x) for x in xs])
    rc = emu.emu_clip_norm(g, _ptrs(xs), ns, max_norm, _ptrs(norms), _ptrs(coefs), SIGNAL_BYTES, gen, gmax, epoch, order)
    assert rc == 0
    return [float(n[0]) for n in norms], [float(c[0]) for c in coefs], norms, coefs


def _shards(world, seed, special=None):
    """Rank sizes with an empty rank, a ragged last tile and (rank 0) more tiles than the small block cap."""
    rng = np.random.default_rng(seed)
    sizes = [3 * 4096 + 100] + [(4096 + 37 * r) if r % 3 else 517 * r for r in range(1, world)]
    if world > 1:
        sizes[world - 1] = 0
    xs = [(rng.standard_normal(n) * (1 + r)).astype(np.float32) for r, n in enumerate(sizes)]
    if special is not None:
        xs[0][7] = special
    return xs


@pytest.mark.parametrize("order", [0, 1])
@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_clip_kernels_on_cpu_threads(emu, world, order):
    """K18 + K19, all ranks concurrently (order 0) or fully serialised phase-major (order 1); three calls back to back
    without a step (generations 0, 1, 0 on the same epoch word); a small block cap so that rank 0 has more tiles than
    blocks; an empty rank.  Every rank's norm and coefficient equal the restatement bit for bit."""
    gmax = 3
    g = emu.emu_group_create(world, 1 << 20)
    try:
        for call, max_norm in enumerate((1.0, 1e4, 0.5)):
            xs = _shards(world, seed=10 * world + call)
            norms, coefs, nb, cb = _clip(emu, g, xs, max_norm, call % 2, call + 1, order, gmax)
            want_n, want_c = ref.norm_coef([ref.partial(x, gmax) for x in xs], max_norm)
            for r in range(world):
                assert _bits(nb[r]) == _bits([want_n]) and _bits(cb[r]) == _bits([want_c]), (call, r)
            exact = math.sqrt(math.fsum(float(v) * float(v) for x in xs for v in x))
            assert abs(norms[0] - exact) <= 1e-6 * exact
    finally:
        emu.emu_group_destroy(g)


@pytest.mark.parametrize("special", [np.inf, -np.inf, np.nan])
def test_clip_kernels_non_finite(emu, special):
    world = 3
    g = emu.emu_group_create(world, 1 << 20)
    try:
        xs = _shards(world, seed=1, special=special)
        norms, coefs, _, _ = _clip(emu, g, xs, 1.0, 0, 1, 0, ref.G_MAX)
        if np.isnan(special):
            assert all(np.isnan(n) and np.isnan(c) for n, c in zip(norms, coefs))
        else:
            assert all(np.isinf(n) and c == 0.0 for n, c in zip(norms, coefs))
    finally:
        emu.emu_group_destroy(g)


@pytest.mark.parametrize("world", [1, 2, 3])
def test_scaled_adam_push_on_cpu_threads(emu, world):
    """The scaled K13 with coef 1.0 is the unscaled K13 bit for bit; with coef c it is the unscaled K13 on c * g."""
    shard = [0]
    for r in range(world):
        shard.append(shard[-1] + 64 * (r + 1))
    total = shard[-1]
    off = (ctypes.c_longlong * (world + 1))(*shard)
    n_own = [shard[r + 1] - shard[r] for r in range(world)]
    glo = (ctypes.c_longlong * world)(*[0] * world)
    ghi = (ctypes.c_longlong * world)(*n_own)
    rng = np.random.default_rng(world)
    p0 = rng.standard_normal(total).astype(np.float32)
    grads = [rng.standard_normal(n).astype(np.float32) for n in n_own]

    def run(scale, premultiply):
        g = emu.emu_group_create(world, 1 << 20)
        try:
            poff = SIGNAL_BYTES
            views = []
            for r in range(world):
                v = np.ctypeslib.as_array(emu.emu_arena_ptr(g, r, poff), shape=(total,))
                v[:] = p0
                views.append(v)
            ms = [np.full(n, 0.01, np.float32) for n in n_own]
            vs = [np.full(n, 0.02, np.float32) for n in n_own]
            red = [(x * np.float32(premultiply)).astype(np.float32) if premultiply is not None else x.copy() for x in grads]
            args = (g, 0, poff, _ptrs(ms), _ptrs(vs), _ptrs(red), total, off, 1, glo, ghi, 1e-2, 0.9, 0.999, 1e-8, 0.01,
                    3, 1, 1, 0, 0)
            if scale is None:
                assert emu.emu_adam_push(*args) == 0
            else:
                sc = [np.full(1, scale, np.float32) for _ in range(world)]
                assert emu.emu_adam_push_scaled(*args, _ptrs(sc)) == 0
            return [v.copy() for v in views], ms, vs
        finally:
            emu.emu_group_destroy(g)

    plain = run(None, None)
    one = run(1.0, None)
    c = np.float32(0.3712)
    scaled = run(float(c), None)
    pre = run(None, c)
    for a, b in ((plain, one), (pre, scaled)):
        for xa, xb in zip(a, b):
            for u, v in zip(xa, xb):
                assert np.array_equal(u.view(np.uint32), v.view(np.uint32))
    assert not np.array_equal(plain[0][0], scaled[0][0])


# ---- protocol model ------------------------------------------------------------------------------------------------
def _clip_model(world, steps=2, buckets=1, calls=2, bn=2, generations=2, clip_word="clip"):
    """Every interleaving of W ranks, each running four streams (DESIGN.md §5):

      S  stage every reduce bucket into its own staging region, then staged[rank] = idx; a step's first stage waits for
         the rank's U of the step before (backward follows optimizer.step())
      X  (the internal stream) per bucket: wait staged of every rank, read every rank's staging region; then ``calls``
         clip calls: K18 writes the partial into slot `rank` of generation (call parity) in every arena and sets the clip
         word, K19 waits for every rank's clip word and reads the W slots; then the step pushes the parameters and sets
         published
      U  wait published of every rank, read every rank's parameters
      B  (the compute stream) ``bn`` BatchNorm exchanges on their own word and double buffer

    Returns None, or (kind, trace).  ``generations=1`` removes the clip double buffer; ``clip_word`` = "staged" / "bn"
    lets the clip exchange signal through another exchange's word (each keeps its own epoch counter)."""
    S, X, U, B = [], [], [], []
    cid = 0
    for k in range(steps):
        for b in range(buckets):
            idx = k * buckets + b + 1
            S += ([("after", ("U", 2 * k))] if b == 0 and k > 0 else []) + [("write_own", ("stg", b), k), ("set", "staged", idx)]
            X += [("wait", "staged", idx), ("read_own_of_all", ("stg", b), k)]
        for _ in range(calls):
            cid += 1
            gen = cid % generations
            X += [("write_all", ("clip", gen), cid), ("set", clip_word, cid), ("wait", clip_word, cid),
                  ("read_all", ("clip", gen), cid)]
        X += [("write_all", ("par",), k), ("set", "published", k + 1)]
        U += [("wait", "published", k + 1), ("read_all", ("par",), k)]
    for j in range(bn):
        B += [("write_all", ("bn", j % 2), j), ("set", "bn", j + 1), ("wait", "bn", j + 1), ("read_all", ("bn", j % 2), j)]
    progs = {"S": S, "X": X, "U": U, "B": B}
    names = ("S", "X", "U", "B")
    words = ("staged", "published", "clip", "bn")
    init = (tuple(tuple(0 for _ in names) for _ in range(world)),
            tuple(tuple(tuple(0 for _ in range(world)) for _ in words) for _ in range(world)),
            frozenset())
    seen = set()
    stack = [(init, ())]
    while stack:
        state, trace = stack.pop()
        if state in seen:
            continue
        seen.add(state)
        pcs, flags, mem = state
        memd = dict(mem)
        succ = []
        for r in range(world):
            for si, name in enumerate(names):
                pc = pcs[r][si]
                if pc == len(progs[name]):
                    continue
                op, a, *v = progs[name][pc]
                nflags, nmem = flags, mem
                if op == "after":
                    if pcs[r][names.index(a[0])] < a[1]:
                        continue
                elif op == "wait":
                    w = words.index(a)
                    if any(flags[r][w][s] < v[0] for s in range(world)):
                        continue
                elif op == "set":
                    w = words.index(a)
                    fl = [[list(x) for x in f] for f in flags]
                    for dst in range(world):
                        fl[dst][w][r] = max(fl[dst][w][r], v[0])       # monotone words
                    nflags = tuple(tuple(tuple(x) for x in f) for f in fl)
                elif op == "write_own":
                    m2 = dict(memd)
                    m2[(r, a, r)] = v[0]
                    nmem = frozenset(m2.items())
                elif op == "write_all":
                    m2 = dict(memd)
                    for dst in range(world):
                        m2[(dst, a, r)] = v[0]
                    nmem = frozenset(m2.items())
                elif op in ("read_all", "read_own_of_all"):
                    for s in range(world):
                        key = (r, a, s) if op == "read_all" else (s, a, s)
                        if memd.get(key) != v[0]:
                            return "bad_read", trace + ((r, name, op, a, "from", s, "holds", memd.get(key), "wants", v[0]),)
                row = list(pcs[r])
                row[si] = pc + 1
                succ.append(((pcs[:r] + (tuple(row),) + pcs[r + 1:], nflags, nmem), (r, name, op, a)))
        if not succ:
            if any(pcs[r][si] < len(progs[n]) for r in range(world) for si, n in enumerate(names)):
                return "deadlock", trace
            continue
        for s, step in succ:
            stack.append((s, trace + (step,)))
    return None


@pytest.mark.parametrize("world,buckets", [(2, 2), (3, 1)])
def test_clip_protocol_is_safe_and_deadlock_free(world, buckets):
    # the owner path the clip exchange is inserted into, as test_protocol_model checks it
    assert explore_owner(world, 2, buckets) is None
    assert _clip_model(world, buckets=buckets, bn=2 if world == 2 else 0) is None


def test_clip_protocol_model_finds_the_overwrite_without_the_double_buffer():
    """Two clip calls without a step: a fast rank pushes the second partial into the slot a slow rank has not read."""
    res = _clip_model(2, steps=1, generations=1, bn=0)
    assert res is not None and res[0] == "bad_read", res


@pytest.mark.parametrize("word", ["staged", "bn"])
def test_clip_protocol_needs_its_own_word(word):
    """Signalling through the bucket exchange's or the BatchNorm exchange's word lets their arrivals satisfy a clip wait
    before the partials are there."""
    res = _clip_model(2, steps=1, calls=1, bn=2 if word == "bn" else 0, clip_word=word)
    assert res is not None and res[0] == "bad_read", res


# ---- ShardedOptimizer host logic over the threaded test double ----------------------------------------------------------
class ClipComm(FakeComm):
    """FakeComm plus the clip exchange (the restatement between threads) and the scaled fused step."""

    def clip_register(self):
        self.clip_registered = getattr(self, "clip_registered", 0) + 1
        return 0

    def clip_norm_(self, x, max_norm, norm_out, coef_out, wait_stream=None, comm_stream=None, phases=3):
        assert self.clip_registered == 1
        parts = self._exchange(ref.partial(x.numpy()))
        norm, coef = ref.norm_coef(parts, max_norm)
        norm_out.fill_(float(norm))
        coef_out.fill_(float(coef))

    def adam_push_(self, params, exp_avg, exp_avg_sq, reduced, shard_off, groups, nvls=False, wait_stream=None,
                   comm_stream=None, phases=6, grad_scale=None):
        if grad_scale is not None:
            reduced = reduced * grad_scale
        super().adam_push_(params, exp_avg, exp_avg_sq, reduced, shard_off, groups, nvls, wait_stream, comm_stream, phases)


_OPTS = {"adam": lambda ps: torch.optim.Adam(ps, lr=1e-2),
         "adamw": lambda ps: torch.optim.AdamW(ps, lr=1e-2, weight_decay=0.05),
         "sgd_momentum": lambda ps: torch.optim.SGD(ps, lr=0.05, momentum=0.9),
         "rmsprop": lambda ps: torch.optim.RMSprop(ps, lr=1e-3)}


def _groups(model):
    decay = [p for n, p in model.named_parameters() if n.endswith("weight")]
    no_decay = [p for n, p in model.named_parameters() if not n.endswith("weight")]
    return [{"params": no_decay, "weight_decay": 0.0}, {"params": decay, "weight_decay": 0.01}]


@pytest.mark.parametrize("algo", ["norm", "value"])
@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("opt_name", ["adam", "adamw", "sgd_momentum", "rmsprop"])
def test_sharded_clipping_equals_torch_on_averaged_grads(world, opt_name, algo):
    """W ranks + ShardedOptimizer.clip_grad_norm / clip_grad_value + step == one replica clipping the mean gradient
    with torch and stepping; two parameter groups; the last step accumulates two backward passes."""
    net = _Net(world)
    mk = _OPTS[opt_name]
    steps = 4
    data = [[[(torch.randn(6, 13, generator=torch.Generator().manual_seed(1000 * s + 10 * a + r)),
               torch.randn(6, 3, generator=torch.Generator().manual_seed(7 + 1000 * s + 10 * a + r)))
              for r in range(world)] for a in range(2 if s == steps - 1 else 1)] for s in range(steps)]
    max_norm, clip_value = 0.05, 0.004
    ref_model = make_model()
    ref_opt = mk(_groups(ref_model))
    norms_ref = []
    for s in range(steps):
        ref_opt.zero_grad()
        for batch in data[s]:
            for r in range(world):
                x, y = batch[r]
                (torch.nn.functional.mse_loss(ref_model(x), y) / world).backward()
        if algo == "norm":
            norms_ref.append(float(torch.nn.utils.clip_grad_norm_(ref_model.parameters(), max_norm)))
        else:
            torch.nn.utils.clip_grad_value_(ref_model.parameters(), clip_value)
        ref_opt.step()
    models = [make_model() for _ in range(world)]

    def rank_fn(r):
        from ray_lightning_b200.sharded import FlatShards, ShardedOptimizer, group_index_of
        model = models[r]
        base = mk(_groups(model))
        params = [p for p in model.parameters() if p.requires_grad]
        shards = FlatShards(model, ClipComm(net, r), wire="fp32", group_of=group_index_of(params, base),
                            reduce_bucket_mb=0.001)
        sopt = ShardedOptimizer(base, shards, wire="fp32")
        norms = []
        for s in range(steps):
            sopt.zero_grad()
            for batch in data[s]:
                x, y = batch[r]
                torch.nn.functional.mse_loss(model(x), y).backward()
            if algo == "norm":
                norms.append(float(sopt.clip_grad_norm(max_norm)))
            else:
                sopt.clip_grad_value(clip_value)
            sopt.step()
        return [p.detach().clone() for p in model.parameters()], norms

    outs = run_ranks(world, rank_fn)
    for params, norms in outs:
        for a, b in zip(params, ref_model.parameters()):
            # the mean gradient differs in its last bits (sum of g / W vs. accumulated (loss / W) gradients); RMSprop's
            # division by sqrt(v) of small clipped gradients turns that into a few 1e-6 over four steps
            torch.testing.assert_close(a, b.detach(), rtol=2e-5, atol=5e-6)
        for a, b in zip(params, outs[0][0]):
            assert torch.equal(a, b)
        if algo == "norm":
            assert norms == outs[0][1]
            np.testing.assert_allclose(norms, norms_ref, rtol=1e-5)
            assert max(norms_ref) > max_norm        # the clip was active


def test_sharded_backward_after_clip_raises_and_zero_grad_drops_the_coefficient():
    net = _Net(1)
    model = make_model()
    from ray_lightning_b200.sharded import FlatShards, ShardedOptimizer
    comm = ClipComm(net, 0)
    sopt = ShardedOptimizer(torch.optim.SGD(model.parameters(), lr=0.1), FlatShards(model, comm, wire="fp32"), wire="fp32")
    x, y = torch.randn(4, 13), torch.randn(4, 3)
    torch.nn.functional.mse_loss(model(x), y).backward()
    sopt.clip_grad_norm(1e-3)
    assert sopt._coef is not None
    with pytest.raises(RuntimeError, match="after the gradients were clipped"):
        torch.nn.functional.mse_loss(model(x), y).backward()
    sopt.zero_grad()
    assert sopt._coef is None
    torch.nn.functional.mse_loss(model(x), y).backward()    # a new step's backward is fine again
    sopt.clip_grad_norm(1e-3)
    sopt.step()
    assert comm.clip_registered == 1                       # registered once, at the first clip
    with pytest.raises(ValueError, match="norm_type"):
        sopt.clip_grad_norm(1.0, norm_type=1)


# ---- Trainer plumbing ------------------------------------------------------------------------------------------------
def test_trainer_validates_the_algorithm():
    from ray_lightning_b200._runtime import minipl
    with pytest.raises(ValueError, match="'norm' and 'value'"):
        minipl.Trainer(gradient_clip_val=1.0, gradient_clip_algorithm="l1", enable_checkpointing=False)
    assert minipl.Trainer(enable_checkpointing=False).gradient_clip_algorithm == "norm"


def test_configure_gradient_clipping_is_called_once_per_step_with_the_trainers_values(tmpdir):
    from utils import BoringModel, get_trainer

    class Recording(BoringModel):
        def __init__(self):
            super().__init__()
            self.calls = []

        def configure_gradient_clipping(self, optimizer, optimizer_idx, gradient_clip_val=None, gradient_clip_algorithm=None):
            self.calls.append((optimizer_idx, gradient_clip_val, gradient_clip_algorithm))
            super().configure_gradient_clipping(optimizer, optimizer_idx, gradient_clip_val, gradient_clip_algorithm)

    model = Recording()
    trainer = get_trainer(tmpdir, strategy=None, limit_train_batches=3, limit_val_batches=1, checkpoint_callback=False,
                          gradient_clip_val=0.5, gradient_clip_algorithm="value")
    trainer.fit(model)
    assert model.calls == [(0, 0.5, "value")] * 3
    model = Recording()
    get_trainer(tmpdir, strategy=None, limit_train_batches=3, limit_val_batches=1, checkpoint_callback=False,
                gradient_clip_val=0).fit(model)
    assert model.calls == []                               # no clipping: the hook is not reached


def test_optimizer_in_backward_refuses_clipping():
    from ray_lightning_b200 import RayStrategy
    from ray_lightning_b200._runtime import minipl
    s = RayStrategy(num_workers=2, use_gpu=False, b200_optimizer_in_backward=True)
    t = minipl.Trainer(strategy=s, gradient_clip_val=1.0, enable_checkpointing=False)
    with pytest.raises(ValueError, match="b200_optimizer_in_backward.*gradient_clip_val"):
        s.setup_optimizers(t)


def _reference_run(model_cls, world, steps, clip_val, algo):
    """One process, full batch: every step averages the W ranks' batches (DistributedSampler order), clips with torch."""
    from torch.utils.data import DistributedSampler
    from utils import RandomDataset
    torch.manual_seed(0)
    model = model_cls()
    opt = model.configure_optimizers()
    opt = opt[0][0] if isinstance(opt, tuple) else opt
    ds = RandomDataset(32, 64, 0)
    order = []
    for r in range(world):
        smp = DistributedSampler(ds, num_replicas=world, rank=r, shuffle=True)
        smp.set_epoch(0)
        order.append(list(smp))
    for s in range(steps):
        opt.zero_grad()
        batch = torch.stack([ds[order[r][s]] for r in range(world)])
        model.training_step(batch, s)["loss"].backward()
        if clip_val:
            if algo == "value":
                torch.nn.utils.clip_grad_value_(model.parameters(), clip_val)
            else:
                torch.nn.utils.clip_grad_norm_(model.parameters(), clip_val)
        opt.step()
    return [p.detach() for p in model.parameters()]


@pytest.fixture
def ray_start_2_cpus():
    from ray_lightning_b200._compat import ray
    ray.init(num_cpus=2)
    yield
    ray.shutdown()


@pytest.mark.parametrize("sharded", [False, True])
@pytest.mark.parametrize("algo", ["norm", "value"])
def test_strategies_clip_on_gloo_workers(tmpdir, ray_start_2_cpus, sharded, algo):
    """RayStrategy / RayShardedStrategy(use_gpu=False) with gradient_clip_val == one process clipping the averaged
    gradient with torch; and the clip was active (the weights differ from the unclipped run)."""
    from ray_lightning_b200 import RayShardedStrategy, RayStrategy
    from utils import AdamBoringModel, BoringModel, get_trainer
    model_cls = AdamBoringModel if sharded else BoringModel
    clip_val = 0.05 if algo == "norm" else 0.01
    steps = 4
    torch.manual_seed(0)
    model = model_cls()
    strategy = (RayShardedStrategy if sharded else RayStrategy)(num_workers=2, use_gpu=False)
    trainer = get_trainer(tmpdir, strategy=strategy, limit_train_batches=steps, limit_val_batches=1,
                          checkpoint_callback=False, gradient_clip_val=clip_val, gradient_clip_algorithm=algo)
    trainer.fit(model)
    want = _reference_run(model_cls, 2, steps, clip_val, algo)
    unclipped = _reference_run(model_cls, 2, steps, None, algo)
    got = [p.detach() for p in model.parameters()]
    for a, b in zip(got, want):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
    assert any(not torch.allclose(a, b, rtol=1e-4, atol=1e-5) for a, b in zip(got, unclipped))
