"""The optimizer epilogues of libb2d on an H100, bit for bit against torch.optim on CUDA.

Three layers, each pinned separately so that a failure names its cause:
1. torch's own CUDA element-wise operations (lerp_, mul_, addcmul_, sqrt, div_, add_, addcdiv_, add(alpha=) and
   their _foreach_ forms) against their one-rounding restatements in tests/optim_ref.py;
2. torch.optim.Adam / AdamW / SGD, both paths, against the restated update (the foreach path is what the kernels
   reproduce; the single-tensor path divides by sqrt(bias_correction2) as a multiply by its reciprocal, so it rounds
   differently);
3. K13 (and the clip-scaled K13), K5 and K14 through the C ABI on loopback ranks against torch's default (foreach)
   Adam / AdamW / SGD on CUDA, one step from identical state and along a 2000-step trajectory, plus the float64
   bound of optim_ref.adam_step64 for every single step."""
import numpy as np
import pytest
import torch

import optim_ref as ref
from oracle import ddp_oracle

pytestmark = pytest.mark.gpu

f32 = np.float32
GRID = ref.adam_grid()
STEPS = (1, 2, 10, 1000, 10000)
_groups = {}


def group(world, tag="k13"):
    """Loopback ranks on one GPU; K5 runs on a group of its own."""
    from ray_lightning_b200.comm import LoopbackGroup
    if (world, tag) not in _groups:
        _groups[(world, tag)] = LoopbackGroup(world, 0, arena_bytes=64 << 20, timeout_ms=20000)
    return _groups[(world, tag)]


def teardown_module(module):
    for g in _groups.values():
        g.close()
    _groups.clear()


def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x, f32)).cuda()


def host(t):
    return t.detach().float().cpu().numpy()


def assert_same_bits(got, want, what):
    got, want = np.asarray(got, f32), np.asarray(want, f32)
    # NaN where torch has NaN; its sign and payload are not part of the contract (the device's canonical NaN is not
    # NumPy's)
    both_nan = np.isnan(got) & np.isnan(want)
    got, want = np.where(both_nan, f32(np.nan), got), np.where(both_nan, f32(np.nan), want)
    bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
    assert bad.size == 0, "%s: %d of %d differ, first at %d: %r != %r" % (what, bad.size, got.size, bad[0], got[bad[0]],
                                                                          want[bad[0]])


# ---- 1. torch's element-wise CUDA operations ------------------------------------------------------------------------
N_PROBE = 1 << 20
EDGES = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, -1.1754942e-38, 1e-20, 1e-9, 1.0, -1.0, 3.4028235e38, -3.4028235e38,
                  1e18, 1e21, np.inf, -np.inf, np.nan], f32)


def _probe_values(seed, lo=-45, hi=45):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal(N_PROBE) * 2.0 ** rng.integers(lo, hi, N_PROBE)).astype(f32)
    idx = rng.permutation(N_PROBE)[:64 * len(EDGES)]
    x[idx] = np.resize(EDGES, idx.size)
    return x


def _fe(op):
    """The _foreach_ form of an in-place op on a one-tensor list."""
    def run(x, *args):
        xs = [x]
        op(xs, *args)
        return xs[0]
    return run


# name -> (torch on CUDA tensors, restatement on numpy arrays); a, b, c are wide-range values with edges, q >= 0
PROBES = {}
for w in (0.1, 0.05, 0.49999997, 0.5, 0.7, 1.0):
    PROBES["lerp_%r" % w] = (lambda a, b, c, q, w=w: a.clone().lerp_(b, w), lambda a, b, c, q, w=w: ref.lerp(a, b, w))
    PROBES["foreach_lerp_%r" % w] = (lambda a, b, c, q, w=w: _fe(torch._foreach_lerp_)(a.clone(), [b], w),
                                     lambda a, b, c, q, w=w: ref.lerp(a, b, w))
for s in (0.999, 0.95, 1 - 1e-3 * 0.1):
    PROBES["mul_%g" % s] = (lambda a, b, c, q, s=s: a.clone().mul_(s), lambda a, b, c, q, s=s: ref.mul_scalar(a, s))
    PROBES["foreach_mul_%g" % s] = (lambda a, b, c, q, s=s: _fe(torch._foreach_mul_)(a.clone(), s),
                                    lambda a, b, c, q, s=s: ref.mul_scalar(a, s))
for v in (1 - 0.999, 1 - 0.95, 0.3):
    PROBES["addcmul_sq_%g" % v] = (lambda a, b, c, q, v=v: a.clone().addcmul_(b, b, value=v),
                                   lambda a, b, c, q, v=v: ref.addcmul(a, b, b, v))
    PROBES["addcmul_%g" % v] = (lambda a, b, c, q, v=v: a.clone().addcmul_(b, c, value=v),
                                lambda a, b, c, q, v=v: ref.addcmul(a, b, c, v))
    PROBES["foreach_addcmul_sq_%g" % v] = (lambda a, b, c, q, v=v: _fe(torch._foreach_addcmul_)(a.clone(), [b], [b], v),
                                           lambda a, b, c, q, v=v: ref.addcmul(a, b, b, v))
PROBES["sqrt"] = (lambda a, b, c, q: q.sqrt(), lambda a, b, c, q: ref.sqrt(q))
PROBES["foreach_sqrt"] = (lambda a, b, c, q: torch._foreach_sqrt([q])[0], lambda a, b, c, q: ref.sqrt(q))
for s in ((1 - 0.999 ** 3) ** 0.5, 0.7, 3.0):
    PROBES["div_%g" % s] = (lambda a, b, c, q, s=s: a.clone().div_(s), lambda a, b, c, q, s=s: ref.div_scalar(a, s))
    PROBES["foreach_div_scalar_%g" % s] = (lambda a, b, c, q, s=s: _fe(torch._foreach_div_)(a.clone(), s),
                                           lambda a, b, c, q, s=s: ref.div_scalar(a, s))
    PROBES["foreach_div_scalarlist_%g" % s] = (lambda a, b, c, q, s=s: _fe(torch._foreach_div_)(a.clone(), [s]),
                                               lambda a, b, c, q, s=s: ref.div_scalar_list(a, s))
for e in ref.EPS:
    PROBES["add_%g" % e] = (lambda a, b, c, q, e=e: a.clone().add_(e), lambda a, b, c, q, e=e: ref.add_scalar(a, e))
    PROBES["foreach_add_%g" % e] = (lambda a, b, c, q, e=e: _fe(torch._foreach_add_)(a.clone(), e),
                                    lambda a, b, c, q, e=e: ref.add_scalar(a, e))
for s in (-1e-3, -0.3, -1.0 / (1 - 0.9 ** 2)):
    PROBES["addcdiv_%g" % s] = (lambda a, b, c, q, s=s: a.clone().addcdiv_(b, c, value=s),
                                lambda a, b, c, q, s=s: ref.addcdiv(a, b, c, s))
    PROBES["foreach_addcdiv_scalarlist_%g" % s] = (
        lambda a, b, c, q, s=s: _fe(torch._foreach_addcdiv_)(a.clone(), [b], [c], [s]),
        lambda a, b, c, q, s=s: ref.addcdiv(a, b, c, s))
for al in (0.01, -1e-3, 1.0):
    PROBES["add_alpha_%g" % al] = (lambda a, b, c, q, al=al: a.add(b, alpha=al), lambda a, b, c, q, al=al: ref.add_alpha(a, b, al))
    PROBES["foreach_add_alpha_%g" % al] = (lambda a, b, c, q, al=al: torch._foreach_add([a], [b], alpha=al)[0],
                                           lambda a, b, c, q, al=al: ref.add_alpha(a, b, al))


@pytest.fixture(scope="module")
def probe_inputs():
    a, b, c = _probe_values(1), _probe_values(2), _probe_values(3)
    q = np.abs(_probe_values(4))
    return (a, b, c, q), tuple(dev(x) for x in (a, b, c, q))


@pytest.mark.parametrize("name", sorted(PROBES))
def test_torch_cuda_operation_rounds_as_restated(probe_inputs, name):
    """If a torch build ever rounds one of these differently, this names the operation before anything else fails."""
    (a, b, c, q), (ta, tb, tc, tq) = probe_inputs
    t_op, r_op = PROBES[name]
    got = host(t_op(ta, tb, tc, tq))
    with np.errstate(all="ignore"):
        want = r_op(a, b, c, q)
    assert_same_bits(got, want, name)


# ---- 2. torch.optim against the restatement ----------------------------------------------------------------------------
def torch_adam(p, g, m, v, hp, step, foreach=True):
    """One step of torch.optim.Adam / AdamW on CUDA from state (m, v) after step - 1 steps; returns numpy (p, m, v)."""
    prm = torch.nn.Parameter(dev(p))
    cls = torch.optim.AdamW if hp["adamw"] else torch.optim.Adam
    opt = cls([prm], lr=hp["lr"], betas=(hp["beta1"], hp["beta2"]), eps=hp["eps"], weight_decay=hp["weight_decay"],
              foreach=foreach)
    opt.state[prm] = {"step": torch.tensor(float(step - 1)), "exp_avg": dev(m), "exp_avg_sq": dev(v)}
    prm.grad = dev(g)
    opt.step()
    st = opt.state[prm]
    return host(prm), host(st["exp_avg"]), host(st["exp_avg_sq"])


@pytest.mark.parametrize("hp", GRID, ids=ref.grid_id)
def test_torch_adam_is_the_restatement(hp):
    """torch.optim.Adam / AdamW on CUDA, foreach and single-tensor, three steps from a fresh state and then single
    steps from random states at steps 1000 and 10000, bit for bit against optim_ref on the matching path."""
    n = 1 << 14
    for foreach, path in ((True, "foreach"), (False, "single")):
        p, m, v = ref.state(n, 3)
        m[:], v[:] = 0.0, 0.0
        prm = torch.nn.Parameter(dev(p))
        cls = torch.optim.AdamW if hp["adamw"] else torch.optim.Adam
        opt = cls([prm], lr=hp["lr"], betas=(hp["beta1"], hp["beta2"]), eps=hp["eps"], weight_decay=hp["weight_decay"],
                  foreach=foreach)
        for step in (1, 2, 3):
            g = ref.grads(n, 10 + step)
            prm.grad = dev(g)
            opt.step()
            p, m, v = ref.adam_step32(p, g, m, v, step=step, path=path, **hp)
            st = opt.state[prm]
            for name, t, want in (("p", prm, p), ("m", st["exp_avg"], m), ("v", st["exp_avg_sq"], v)):
                assert_same_bits(host(t), want, "%s %s step %d" % (path, name, step))
        for step in (1000, 10000):
            p, m, v = ref.state(n, step)
            g = ref.grads(n, step)
            got = torch_adam(p, g, m, v, hp, step, foreach)
            want = ref.adam_step32(p, g, m, v, step=step, path=path, **hp)
            for name, x, y in zip("pmv", got, want):
                assert_same_bits(x, y, "%s %s step %d" % (path, name, step))


def test_torch_adam_paths_differ_only_by_the_reciprocal():
    """The two torch paths are not interchangeable: they round sqrt(v) / sqrt(bc2) differently."""
    hp = GRID[0]
    n = 1 << 16
    p, m, v = ref.state(n, 1)
    g = ref.grads(n, 2, edges=False)
    a = torch_adam(p, g, m, v, hp, 10, foreach=True)
    b = torch_adam(p, g, m, v, hp, 10, foreach=False)
    assert not np.array_equal(a[0], b[0])
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


@pytest.mark.parametrize("foreach", [True, False])
@pytest.mark.parametrize("lr,momentum,wd", [(1e-3, 0.9, 0.01), (0.05, 0.9, 0.0), (1.0, 0.0, 0.01), (0.1, 0.0, 0.0)])
def test_torch_sgd_is_the_restatement(foreach, lr, momentum, wd):
    n = 1 << 14
    p, _, _ = ref.state(n, 4)
    prm = torch.nn.Parameter(dev(p))
    opt = torch.optim.SGD([prm], lr=lr, momentum=momentum, weight_decay=wd, foreach=foreach)
    buf = None
    for step in range(1, 5):
        g = ref.grads(n, 20 + step)
        prm.grad = dev(g)
        opt.step()
        p, buf = ref.sgd_step32(p, g, buf, lr=lr, momentum=momentum, weight_decay=wd)
        assert_same_bits(host(prm), p, "p step %d" % step)
        if momentum:
            assert_same_bits(host(opt.state[prm]["momentum_buffer"]), buf, "buf step %d" % step)


# ---- 3. the kernels against torch ------------------------------------------------------------------------------------
def bound_excess(got, out64, tol, ok):
    """Per result: how many elements of ``got`` lie outside ``out64 ± tol`` (plus half an fp32 ulp) where ``ok``, and
    the largest error in units of the bound."""
    res = []
    for x32, x64, t in zip(got, out64, tol):
        with np.errstate(all="ignore"):
            err = np.abs(np.asarray(x32, np.float64) - x64)
            lim = t + np.spacing(np.abs(np.asarray(x32, f32))).astype(np.float64) / 2
            bad = ok & ~(err <= lim)
            res.append((int(bad.sum()), float(np.max(np.where(ok, err / lim, 0.0), initial=0.0))))
    return res


def _check_bound(p, g, m, v, hp, step, got, what):
    """The float64 bound of optim_ref.adam_step64 on the elements whose update stays in fp32's finite range."""
    out64, tol = ref.adam_step64(p, g, m, v, step=step, **hp)
    ok = np.isfinite(g) & (np.abs(g) < 1e15)
    for x in out64:
        ok &= np.isfinite(x) & (np.abs(x) < 1e30)
    for name, (bad, _) in zip("pmv", bound_excess(got, out64, tol, ok)):
        assert not bad, "%s %s: %d elements outside the float64 bound" % (what, name, bad)


def _k13_layout(world, n_groups):
    """Owner shards (multiples of 8, an empty rank at W >= 3) and per rank up to n_groups parameter groups with
    edges at multiples of 4 (not 8), an empty group and gaps the kernel must leave alone."""
    lens = [8 * (300 + 37 * r) for r in range(world)]
    if world >= 3:
        lens[world - 2] = 0
    shard = [0]
    for x in lens:
        shard.append(shard[-1] + x)
    groups = []
    for r in range(world):
        cuts = sorted({min(lens[r], 4 * k) for k in (0, 1, 3, 3, 50, 51, 130, 200, 301)})
        windows = [(cuts[i], cuts[i + 1]) for i in range(len(cuts) - 1)][::-1][:n_groups]
        if lens[r] and len(windows) < n_groups:
            windows.append((cuts[1], cuts[1]))            # an empty group
        groups.append(windows[:n_groups] if lens[r] else [])
    return shard, groups


def _run_k13(world, hps, step, coef, seed):
    """One K13 step on every rank; group k of every rank uses hps[k % len(hps)].  Returns per element the torch
    reference and what the kernel left, for params (whole vector, every rank) and the owned m, v."""
    g = group(world)
    shard, groups = _k13_layout(world, 8)
    total = shard[-1]
    p, m, v = ref.state(total, seed)
    gr = ref.grads(total, seed + 1)
    params, ms, vs, red = [], [], [], []
    for r, rk in enumerate(g.ranks):
        t = rk.arena_tensor(total)
        t.copy_(dev(p))
        params.append(t)
        lo, hi = shard[r], shard[r + 1]
        ms.append(dev(np.resize(m[lo:hi], max(hi - lo, 8))))
        vs.append(dev(np.resize(v[lo:hi], max(hi - lo, 8))))
        red.append(dev(np.resize(gr[lo:hi], max(hi - lo, 8))))
    gs = [[(lo, hi, dict(hps[k % len(hps)], step=step)) for k, (lo, hi) in enumerate(groups[r])] for r in range(world)]
    torch.cuda.synchronize()
    scale = None if coef is None else [torch.full((1,), coef, device="cuda") for _ in range(world)]
    g.adam_push_(params, ms, vs, red, shard, gs, grad_scale=scale)
    g.synchronize()
    want_p, want_m, want_v = p.copy(), m.copy(), v.copy()
    for r in range(world):
        for k, (lo, hi) in enumerate(groups[r]):
            if hi == lo:
                continue
            a, b = shard[r] + lo, shard[r] + hi
            hp = hps[k % len(hps)]
            gg = gr[a:b] if coef is None else host(dev(gr[a:b]).mul_(coef))      # torch's grad.mul_(clip_coef)
            out = torch_adam(p[a:b], gg, m[a:b], v[a:b], hp, step)
            want_p[a:b], want_m[a:b], want_v[a:b] = out
            _check_bound(p[a:b], gg, m[a:b], v[a:b], hp, step, (params[0][a:b].cpu().numpy(), host(ms[r][lo:hi]),
                                                                host(vs[r][lo:hi])), "K13 %s" % ref.grid_id(hp))
    for r in range(world):
        assert_same_bits(host(params[r]), want_p, "p on rank %d" % r)
        lo, hi = shard[r], shard[r + 1]
        assert_same_bits(host(ms[r])[:hi - lo], want_m[lo:hi], "m of rank %d" % r)
        assert_same_bits(host(vs[r])[:hi - lo], want_v[lo:hi], "v of rank %d" % r)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("step", STEPS)
def test_k13_matches_torch_over_grid(world, step):
    """K13 with eight parameter groups per rank: the 90 grid points spread over the groups of twelve launches."""
    for i in range(0, len(GRID), 8):
        _run_k13(world, GRID[i:i + 8], step, None, seed=1000 * step + i)


@pytest.mark.parametrize("coef", [0.37, 1.0, 0.0])
@pytest.mark.parametrize("world", [2, 3])
def test_scaled_k13_matches_torch(world, coef):
    for step in (1, 10, 10000):
        _run_k13(world, GRID[::11], step, coef, seed=77 * step)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_k5_matches_torch(world):
    """K5 (through sharded_step_, fp32 wire) on the oracle average of the ranks' gradients, every step of a short
    run per grid slice, against torch's Adam / AdamW with state carried over."""
    g = group(world, "k5")
    rng = np.random.default_rng(world)
    numels = [int(x) for x in rng.integers(1, 3000, size=17)] + [8, 1, 20000]
    owner = ddp_oracle.partition_fairscale(numels, world)
    _, shard_off, total = ddp_oracle.shard_layout(numels, owner, world)
    scale = float(f32(1.0) / f32(world))
    slot = 0
    for k, hp in enumerate(GRID[::7]):
        p, _, _ = ref.state(total, 500 + k)
        params, ms, vs = [], [], []
        for r, rk in enumerate(g.ranks):
            t = rk.arena_tensor(total)
            t.copy_(dev(p))
            params.append(t)
            n_own = shard_off[r + 1] - shard_off[r]
            ms.append(torch.zeros(max(n_own, 8), device="cuda"))
            vs.append(torch.zeros(max(n_own, 8), device="cuda"))
        prm = torch.nn.Parameter(dev(p))
        cls = torch.optim.AdamW if hp["adamw"] else torch.optim.Adam
        opt = cls([prm], lr=hp["lr"], betas=(hp["beta1"], hp["beta2"]), eps=hp["eps"], weight_decay=hp["weight_decay"])
        for step in (1, 2, 3):
            per_rank = [torch.from_numpy(ref.grads(total, 100 * k + 10 * step + r, edges=(r == 0))) for r in range(world)]
            grads = [t.cuda() for t in per_rank]
            torch.cuda.synchronize()
            g.sharded_step_(grads, params, ms, vs, shard_off, step=step, lr=hp["lr"], betas=(hp["beta1"], hp["beta2"]),
                            eps=hp["eps"], weight_decay=hp["weight_decay"], adamw=hp["adamw"], wire="fp32", slot=slot)
            slot ^= 1
            g.synchronize()
            prm.grad = ddp_oracle.allreduce_fp32_wire(per_rank, scale).cuda()
            opt.step()
            what = "%s step %d" % (ref.grid_id(hp), step)
            want = host(prm)
            st = opt.state[prm]
            for r in range(world):
                assert_same_bits(host(params[r]), want, "p rank %d %s" % (r, what))
                sl = slice(shard_off[r], shard_off[r + 1])
                n_own = sl.stop - sl.start
                assert_same_bits(host(ms[r])[:n_own], host(st["exp_avg"][sl]), "m rank %d %s" % (r, what))
                assert_same_bits(host(vs[r])[:n_own], host(st["exp_avg_sq"][sl]), "v rank %d %s" % (r, what))


class _Bucket:
    """A DDP-like bucket for K14: separate parameter tensors (1-element ones, sizes not multiples of 4, a
    channels_last weight and ~2000 small ones so that the segment search runs deep), their state tensors, and the
    bucket's flat gradient in parameters' memory order."""

    def __init__(self, ctx, bucket_id, kind, momentum, seed, n_small=2000):
        rng = np.random.default_rng(seed)
        shapes = [(1,), (3,), (5,), (1,), (37,), (1000,), (8, 3, 3, 5)] + [(int(x),) for x in rng.integers(1, 10, n_small)]
        shapes += [(4099,), (1,)]
        self.params = []
        for s in shapes:
            t = dev(rng.standard_normal(int(np.prod(s))).astype(f32)).view(s)
            if len(s) == 4:
                t = t.contiguous(memory_format=torch.channels_last)
            self.params.append(torch.nn.Parameter(t))
        self.numel = [p.numel() for p in self.params]
        self.n = sum(self.numel)
        self.offs = np.concatenate([[0], np.cumsum(self.numel)[:-1]]).tolist()
        need1 = kind == 1 or momentum != 0
        self.s1 = [torch.zeros_like(p) for p in self.params] if need1 else None
        self.s2 = [torch.zeros_like(p) for p in self.params] if kind == 1 else None
        self.ctx, self.id, self.kind, self.momentum = ctx, bucket_id, kind, momentum
        ctx.optim_register(bucket_id, [p.data_ptr() for p in self.params], None if self.s1 is None else [s.data_ptr() for s in self.s1],
                           None if self.s2 is None else [s.data_ptr() for s in self.s2], self.offs, self.numel)

    @staticmethod
    def mem(t):
        """A tensor's elements in memory order."""
        if t.dim() == 4 and not t.is_contiguous():
            return t.permute(0, 2, 3, 1).reshape(-1)
        return t.reshape(-1)

    def grads_for(self, flat):
        """The flat bucket as each parameter's gradient tensor, laid out like the parameter."""
        out = []
        for p, o, k in zip(self.params, self.offs, self.numel):
            x = flat[o:o + k]
            if p.dim() == 4 and not p.is_contiguous():
                n, c, h, w = p.shape
                x = x.view(n, h, w, c).permute(0, 3, 1, 2)
            else:
                x = x.view(p.shape)
            out.append(x.clone())
        return out

    def flat(self, ts):
        return torch.cat([self.mem(t.detach()) for t in ts])

    def step(self, flat_grad, hp, step):
        from ray_lightning_b200._b2d import AdamParams
        a = AdamParams(lr=hp["lr"], beta1=hp.get("beta1", 0.0), beta2=hp.get("beta2", 0.0), eps=hp.get("eps", 0.0),
                       weight_decay=hp["weight_decay"], step=step, adamw=int(hp.get("adamw", False)), zero_grads=0)
        s = torch.cuda.current_stream()
        self.ctx.bucket_optim(self.id, flat_grad.data_ptr(), self.n, self.kind, a, self.momentum, s)


def _mirror(bucket):
    """Independent copies of the bucket's parameters for torch's optimizer."""
    return [torch.nn.Parameter(p.detach().clone(memory_format=torch.preserve_format)) for p in bucket.params]


@pytest.mark.parametrize("hp", GRID, ids=ref.grid_id)
def test_k14_adam_matches_torch(hp):
    """K14 one step from identical state at steps 1, 2, 10, 1000 and 10000, every parameter of an awkward bucket
    (about 2000 parameters at every fifteenth grid point, 100 small ones elsewhere)."""
    ctx = group(1).ranks[0].ctx
    i = GRID.index(hp)
    b = _Bucket(ctx, 100 + i, 1, 0.0, seed=i, n_small=2000 if i % 15 == 0 else 100)
    for step in STEPS:
        p, m, v = ref.state(b.n, step)
        g = ref.grads(b.n, 3 * step + 1)
        with torch.no_grad():
            for t, src in ((b.params, p), (b.s1, m), (b.s2, v)):
                for x, y in zip(t, b.grads_for(dev(src))):
                    x.copy_(y)
        torch.cuda.synchronize()
        b.step(dev(g), hp, step)
        torch.cuda.synchronize()
        want = torch_adam(p, g, m, v, hp, step)      # element-wise: memory order is all that matters
        got = (host(b.flat(b.params)), host(b.flat(b.s1)), host(b.flat(b.s2)))
        for name, x, y in zip("pmv", got, want):
            assert_same_bits(x, y, "K14 %s step %d" % (name, step))
        _check_bound(p, g, m, v, hp, step, got, "K14 step %d" % step)


def test_fp32_entry_point_is_the_double_one_on_widened_values():
    """b2d_bucket_optim (fp32 b2d_adam) runs the update of b2d_bucket_optim64 on the widened fp32 values: bit-identical
    to it when the hyper-parameters are the fp32 values themselves, and off torch's foreach Adam in the last bits when
    they are not (beta2 = 0.999), which is why the library's Python side passes doubles."""
    import ctypes
    from ray_lightning_b200._b2d import AdamParams, AdamParams32
    ctx = group(1).ranks[0].ctx
    hp = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, adamw=False)
    narrowed = {k: (float(f32(x)) if isinstance(x, float) else x) for k, x in hp.items()}
    step = 10
    outs = {}
    for name in ("fp32", "double_narrowed", "double"):
        b = _Bucket(ctx, 500 + len(outs), 1, 0.0, seed=11, n_small=20)
        p, m, v = ref.state(b.n, 12)
        g = ref.grads(b.n, 13, edges=False)
        with torch.no_grad():
            for t, src in ((b.params, p), (b.s1, m), (b.s2, v)):
                for x, y in zip(t, b.grads_for(dev(src))):
                    x.copy_(y)
        flat = dev(g)
        torch.cuda.synchronize()
        h = hp if name == "double" else narrowed
        fields = dict(lr=h["lr"], beta1=h["beta1"], beta2=h["beta2"], eps=h["eps"], weight_decay=h["weight_decay"], step=step,
                      adamw=0, zero_grads=0)
        s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        if name == "fp32":
            a = AdamParams32(**dict(fields, **{k: hp[k] for k in ("lr", "beta1", "beta2", "eps", "weight_decay")}))
            rc = ctx._lib.b2d_bucket_optim(ctx._ctx, b.id, ctypes.c_void_p(flat.data_ptr()), b.n, 1, ctypes.byref(a), 0.0, s)
        else:
            a = AdamParams(**fields)
            rc = ctx._lib.b2d_bucket_optim64(ctx._ctx, b.id, ctypes.c_void_p(flat.data_ptr()), b.n, 1, ctypes.byref(a), 0.0, s)
        assert rc == 0
        torch.cuda.synchronize()
        outs[name] = [host(b.flat(x)) for x in (b.params, b.s1, b.s2)]
        if name == "double":
            want = torch_adam(p, g, m, v, hp, step)
            for x, y, what in zip(outs[name], want, "pmv"):
                assert_same_bits(x, y, "K14 through b2d_bucket_optim64: " + what)
    for x, y, what in zip(outs["fp32"], outs["double_narrowed"], "pmv"):
        assert_same_bits(x, y, "b2d_bucket_optim vs b2d_bucket_optim64 on the fp32 values: " + what)
    assert not np.array_equal(outs["fp32"][2], outs["double"][2])      # exp_avg_sq: 1 - beta2 from the narrowed beta2


SGD_CASES = [(1e-3, 0.9, 0.01), (0.05, 0.9, 0.0), (1.0, 0.0, 0.01), (0.1, 0.0, 0.0)]


@pytest.mark.parametrize("lr,momentum,wd", SGD_CASES)
def test_k14_sgd_matches_torch(lr, momentum, wd):
    """K14's SGD with and without momentum and weight decay, five steps; the first starts the momentum buffer as a
    copy of the gradient, as torch does."""
    ctx = group(1).ranks[0].ctx
    b = _Bucket(ctx, 300 + SGD_CASES.index((lr, momentum, wd)), 0, momentum, seed=5)
    mirror = _mirror(b)
    opt = torch.optim.SGD(mirror, lr=lr, momentum=momentum, weight_decay=wd)
    for step in range(1, 6):
        flat = dev(ref.grads(b.n, 40 + step))
        for p, gt in zip(mirror, b.grads_for(flat)):
            p.grad = gt
        opt.step()
        b.step(flat, dict(lr=lr, weight_decay=wd), step)
        torch.cuda.synchronize()
        assert_same_bits(host(b.flat(b.params)), host(b.flat(mirror)), "K14 SGD p step %d" % step)
        if momentum:
            assert_same_bits(host(b.flat(b.s1)), host(b.flat([opt.state[p]["momentum_buffer"] for p in mirror])),
                             "K14 SGD momentum_buffer step %d" % step)


# ---- 3(b). 2000-step trajectories ---------------------------------------------------------------------------------------
TRAJ = 2000


def test_trajectories_match_torch_for_2000_steps():
    """K14, K13 (W = 2) and K5 (W = 2) each run 2000 steps next to torch's default Adam / AdamW; parameters and
    state stay bit-identical at every 100th step and at the end."""
    hp = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, adamw=True)
    cls = torch.optim.AdamW
    kw = dict(lr=hp["lr"], betas=(hp["beta1"], hp["beta2"]), eps=hp["eps"], weight_decay=hp["weight_decay"])
    # K14
    b = _Bucket(group(1).ranks[0].ctx, 400, 1, 0.0, seed=9, n_small=50)
    mirror = _mirror(b)
    opt = cls(mirror, **kw)
    # K13 and K5 at W = 2 on one flat vector
    world = 2
    g2, g5 = group(world), group(world, "k5")
    total = 8 * 4000
    shard = [0, 8 * 1500, total]
    p0, _, _ = ref.state(total, 10)
    flat13, flat5, m13, v13, m5, v5 = [], [], [], [], [], []
    for r in range(world):
        for lst, grp in ((flat13, g2), (flat5, g5)):
            t = grp.ranks[r].arena_tensor(total)
            t.copy_(dev(p0))
            lst.append(t)
        n_own = shard[r + 1] - shard[r]
        for lst in (m13, v13, m5, v5):
            lst.append(torch.zeros(n_own, device="cuda"))
    prm = torch.nn.Parameter(dev(p0))
    opt2 = cls([prm], **kw)
    gen = torch.Generator(device="cuda").manual_seed(0)
    slot = 0
    for step in range(1, TRAJ + 1):
        scale_exp = float(np.random.default_rng(step).integers(-12, 2))
        flat = torch.randn(b.n, device="cuda", generator=gen) * 2.0 ** scale_exp
        for p, gt in zip(mirror, b.grads_for(flat)):
            p.grad = gt
        opt.step()
        b.step(flat, hp, step)
        full = torch.randn(total, device="cuda", generator=gen) * 2.0 ** scale_exp
        prm.grad = full.clone()
        opt2.step()
        red = [full[shard[r]:shard[r + 1]].contiguous() for r in range(world)]
        groups = [[(0, shard[r + 1] - shard[r], dict(hp, step=step))] for r in range(world)]
        g2.adam_push_(flat13, m13, v13, red, shard, groups)
        grads5 = [full.clone(), torch.zeros_like(full)]             # fp32 wire: g * 1 + 0 * 1 == g exactly
        g5.sharded_step_(grads5, flat5, m5, v5, shard, step=step, lr=hp["lr"], betas=(hp["beta1"], hp["beta2"]),
                         eps=hp["eps"], weight_decay=hp["weight_decay"], adamw=True, wire="fp32", scale=1.0, slot=slot)
        slot ^= 1
        g2.synchronize()
        g5.synchronize()
        if step % 100 == 0 or step == TRAJ:
            torch.cuda.synchronize()
            what = "step %d" % step
            assert_same_bits(host(b.flat(b.params)), host(b.flat(mirror)), "K14 p " + what)
            assert_same_bits(host(b.flat(b.s1)), host(b.flat([opt.state[p]["exp_avg"] for p in mirror])), "K14 m " + what)
            assert_same_bits(host(b.flat(b.s2)), host(b.flat([opt.state[p]["exp_avg_sq"] for p in mirror])), "K14 v " + what)
            st = opt2.state[prm]
            for r in range(world):
                sl = slice(shard[r], shard[r + 1])
                for name, flats, ms_, vs_ in (("K13", flat13, m13, v13), ("K5", flat5, m5, v5)):
                    assert_same_bits(host(flats[r]), host(prm), "%s p rank %d %s" % (name, r, what))
                    assert_same_bits(host(ms_[r]), host(st["exp_avg"][sl]), "%s m rank %d %s" % (name, r, what))
                    assert_same_bits(host(vs_[r]), host(st["exp_avg_sq"][sl]), "%s v rank %d %s" % (name, r, what))
