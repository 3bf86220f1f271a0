"""The optimizer epilogues of libb2d (K5 `k456_sharded_kernel`, K13 `adam_push_kernel`, the clip-scaled K13 and K14
`bucket_optim_kernel`) on CPU threads, bit for bit against the NumPy restatement of torch's CUDA Adam / AdamW / SGD
(tests/optim_ref.py), and the restatement itself against libm and against float64.

The kernels are compiled for the host through csrc/emu/ with -ffp-contract=off; every operation of adam_update is
spelled out (__f*_rn), so the host build rounds exactly as the sm_90a build.  test_gpu_optim.py ties the restatement
to torch on an H100."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import optim_ref as ref
from conftest import ROOT
from oracle import ddp_oracle

EMU_DIR = os.path.join(ROOT, "ray_lightning_b200", "csrc", "emu")
FP = ctypes.POINTER(ctypes.c_float)
LP = ctypes.POINTER(ctypes.c_longlong)
UP = ctypes.POINTER(ctypes.c_uint)
D, F, I = ctypes.c_double, ctypes.c_float, ctypes.c_int
GRID = ref.adam_grid()
f32 = np.float32


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu_optim") / "libb2d_emu.so")
    subprocess.run(["g++", "-std=c++20", "-O1", "-pthread", "-fPIC", "-shared", "-DB2D_EMU", "-ffp-contract=off",
                    "-o", out, os.path.join(EMU_DIR, "emu_harness.cpp")], check=True)
    lib = ctypes.CDLL(out)
    lib.emu_group_create.restype = ctypes.c_void_p
    lib.emu_group_create.argtypes = [I, ctypes.c_size_t]
    lib.emu_group_destroy.argtypes = [ctypes.c_void_p]
    lib.emu_signal_bytes.restype = ctypes.c_size_t
    push = [ctypes.c_void_p, I, ctypes.c_size_t, ctypes.POINTER(FP), ctypes.POINTER(FP), ctypes.POINTER(FP), ctypes.c_size_t, LP, I,
            LP, LP, D, D, D, D, D, I, I, ctypes.c_uint, I, I]
    lib.emu_adam_push64.argtypes = push
    lib.emu_adam_push_scaled64.argtypes = push + [ctypes.POINTER(FP)]
    lib.emu_bucket_optim64.argtypes = [ctypes.POINTER(FP), ctypes.POINTER(FP), ctypes.POINTER(FP), UP, I, FP, ctypes.c_size_t, I,
                                     D, F, D, D, D, D, I, I]
    lib.emu_sharded_step64.argtypes = [ctypes.c_void_p, I, ctypes.POINTER(FP), ctypes.c_size_t, ctypes.POINTER(FP),
                                     ctypes.POINTER(FP), ctypes.c_size_t, LP, F, D, D, D, D, D, I, I, I, I, I, I]
    lib.emu_arena_ptr.restype = FP
    lib.emu_arena_ptr.argtypes = [ctypes.c_void_p, I, ctypes.c_size_t]
    return lib


def ptrs(arrs):
    return (FP * len(arrs))(*[a.ctypes.data_as(FP) for a in arrs])


def bits(x):
    return np.asarray(x, f32).view(np.uint32)


def assert_same_bits(got, want, what):
    got, want = np.asarray(got, f32), np.asarray(want, f32)
    # NaN where torch has NaN; its sign and payload are not part of the contract (the device's canonical NaN is not
    # NumPy's)
    both_nan = np.isnan(got) & np.isnan(want)
    got, want = np.where(both_nan, f32(np.nan), got), np.where(both_nan, f32(np.nan), want)
    bad = np.nonzero(bits(got) != bits(want))[0]
    assert bad.size == 0, "%s: %d of %d differ, first at %d: %r != %r" % (what, bad.size, got.size, bad[0], got[bad[0]],
                                                                          want[bad[0]])


# ---- fma32 -------------------------------------------------------------------------------------------------------------
def _libm_fmaf():
    libm = ctypes.CDLL("libm.so.6")
    libm.fmaf.restype = F
    libm.fmaf.argtypes = [F, F, F]
    return libm.fmaf


def _fma_cases(rng, n):
    """Random triples over the whole exponent range, near-cancellations, products that put the float64 sum exactly
    on an fp32 rounding midpoint (the double-rounding trap), subnormal results and every combination of edges."""
    def wide(k, lo, hi):
        with np.errstate(over="ignore"):
            return (rng.standard_normal(k) * 2.0 ** rng.integers(lo, hi, k)).astype(f32)
    a, b, c = wide(n, -75, 64), wide(n, -75, 64), wide(n, -150, 127)
    # c close to -a*b: massive cancellation
    a2, b2 = wide(n // 4, -40, 40), wide(n // 4, -40, 40)
    with np.errstate(over="ignore"):
        c2 = (-(a2.astype(np.float64) * b2) * (1 + rng.standard_normal(n // 4) * 2.0 ** -20)).astype(f32)
    # a*b = half an ulp of c times (1 - k^2 2^-46): the float64 sum is a midpoint, the exact value is not
    c3 = wide(n // 4, -120, 120)
    e = np.frexp(c3.astype(np.float64))[1]
    k = rng.integers(1, 1 << 11, n // 4)
    a3 = (np.ldexp(1.0, e - 25) * (1 + k * 2.0 ** -23)).astype(f32)
    b3 = ((1 - k * 2.0 ** -23) * rng.choice([-1.0, 1.0], n // 4)).astype(f32)
    # subnormal and overflowing results
    a4, b4, c4 = wide(n // 4, -80, -60), wide(n // 4, -80, -60), wide(n // 4, -149, -126)
    a5, b5, c5 = wide(n // 8, 60, 64), wide(n // 8, 60, 66), wide(n // 8, 120, 128)
    edges = np.array([0.0, -0.0, 1.0, -1.0, 1e-45, -1e-45, 1.1754942e-38, -1.1754942e-38, 3.4028235e38, -3.4028235e38,
                      np.inf, -np.inf, np.nan, 0.5, 3.0, 2.0 ** -24, 1 + 2.0 ** -23], f32)
    ea, eb, ec = (x.ravel() for x in np.meshgrid(edges, edges, edges, indexing="ij"))
    return (np.concatenate(x) for x in ((a, a2, a3, a4, a5, ea), (b, b2, b3, b4, b5, eb), (c, c2, c3, c4, c5, ec)))


def test_fma32_matches_libm_fmaf():
    """fma32 against the C library's fmaf on about four million triples, the hard cases for a float64 emulation
    included; the plain float64 expression a * b + c rounded to fp32 must differ on the midpoint cases."""
    fmaf = _libm_fmaf()
    a, b, c = _fma_cases(np.random.default_rng(11), 1 << 21)
    got = ref.fma32(a, b, c)
    want = np.fromiter(map(fmaf, a.tolist(), b.tolist(), c.tolist()), f32, count=a.size)
    same = (bits(got) == bits(want)) | (np.isnan(got) & np.isnan(want))
    assert same.all(), "fma32 != fmaf at %s" % ((a[~same][:3], b[~same][:3], c[~same][:3]),)
    with np.errstate(all="ignore"):
        naive = (a.astype(np.float64) * b + c).astype(f32)
    assert (bits(naive) != bits(want)).sum() > 1000          # the cases do exercise the tie-break


# ---- the restatement against float64 ------------------------------------------------------------------------------------
def _finite_region(out64, g, hp):
    """Elements whose float64 update stays well inside fp32's range (v overflows fp32 for |g| >~ 1e19)."""
    ok = np.isfinite(g) & (np.abs(g) < 1e15)
    for x in out64:
        ok &= np.isfinite(x) & (np.abs(x) < 1e30)
    return ok


def _within_bound(out32, out64, tol, ok, what):
    for name, x32, x64, t in zip(("p", "m", "v"), out32, out64, tol):
        x32 = np.asarray(x32, np.float64)
        with np.errstate(invalid="ignore"):
            err = np.abs(x32 - x64)
        half_ulp = np.spacing(np.abs(np.asarray(out32[("p", "m", "v").index(name)], f32))).astype(np.float64) / 2
        bad = ok & ~(err <= t + half_ulp)
        assert not bad.any(), "%s %s: %d elements outside the float64 bound, e.g. got %r want %r (tol %r)" % (
            what, name, bad.sum(), x32[bad][:2], x64[bad][:2], t[bad][:2])


@pytest.mark.parametrize("hp", GRID, ids=ref.grid_id)
def test_restatement_within_float64_bound(hp):
    """Both of torch's paths, as restated, stay within the float64 reference's bound at steps 1, 2, 10, 1000 and
    10000, from a fresh state and from a random one."""
    n = 4096
    for step in (1, 2, 10, 1000, 10000):
        p, m, v = ref.state(n, step)
        if step == 1:
            m[:], v[:] = 0.0, 0.0
        g = ref.grads(n, 7 * step)
        out64, tol = ref.adam_step64(p, g, m, v, step=step, **hp)
        ok = _finite_region(out64, g, hp)
        assert ok.sum() > n // 2
        for path in ("foreach", "single"):
            out32 = ref.adam_step32(p, g, m, v, step=step, path=path, **hp)
            _within_bound(out32, out64, tol, ok, "%s step %d" % (path, step))


def _narrowed_1_minus_beta2(p, g, m, v, *, beta2, **kw):
    """The defect the bound exists for: beta2 rounded to fp32 before `1 - beta2` is formed."""
    b2 = float(f32(beta2))
    pn, mn, vn = ref.adam_step32(p, g, m, v, beta2=beta2, **kw)
    vn = ref.addcmul(ref.mul_scalar(v, beta2), g, g, f32(1.0 - b2))
    return pn, mn, vn


def _eps_inside_sqrt(p, g, m, v, *, lr, beta1, beta2, eps, step, **kw):
    pn, mn, vn = ref.adam_step32(p, g, m, v, lr=lr, beta1=beta1, beta2=beta2, eps=eps, step=step, **kw)
    _, bc2, step_size, _ = ref.adam_consts(lr, beta1, beta2, step)
    denom = ref.sqrt(((vn / f32(bc2)) + f32(eps)).astype(f32))
    return ref.addcdiv(p, mn, denom, -step_size), mn, vn


@pytest.mark.parametrize("defect", [_narrowed_1_minus_beta2, _eps_inside_sqrt])
def test_float64_bound_catches_known_defects(defect):
    """The bound is tight enough to fail on the mistakes the test-suite used to let through at rtol 2e-5."""
    hp = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, adamw=False)
    n = 4096
    p, m, v = ref.state(n, 1)
    m[:], v[:] = 0.0, 0.0
    g = ref.grads(n, 3, edges=False)
    out64, tol = ref.adam_step64(p, g, m, v, step=1, **hp)
    with pytest.raises(AssertionError, match="outside the float64 bound"):
        _within_bound(defect(p, g, m, v, step=1, **{k: x for k, x in hp.items()}), out64, tol,
                      _finite_region(out64, g, hp), "defect")


def test_sgd_restatement_within_float64_bound():
    n = 4096
    p, _, _ = ref.state(n, 5)
    buf = None
    for step in range(3):
        g = ref.grads(n, 40 + step, edges=False)
        for lr, mom, wd in ((1e-3, 0.9, 0.01), (1.0, 0.0, 0.0)):
            p32, b32 = ref.sgd_step32(p, g, buf, lr=lr, momentum=mom, weight_decay=wd)
            p64, _ = ref.sgd_step64(p, g, buf, lr=lr, momentum=mom, weight_decay=wd)
            gmag = np.abs(g).astype(np.float64) + wd * np.abs(p) + (0 if buf is None else mom * np.abs(buf))
            tol = 2.0 ** -24 * (4 * np.abs(p) + 4 * lr * gmag) + np.spacing(np.abs(p32)) / 2
            assert (np.abs(p32 - p64) <= tol).all()
        p, buf = ref.sgd_step32(p, g, buf, lr=1e-3, momentum=0.9, weight_decay=0.01)


# ---- K14 over the whole grid ---------------------------------------------------------------------------------------------
SIZES = [1, 3, 5, 4, 37, 1000, 2, 8, 515, 7]


def _k14(emu, params, s1, s2, grads, kind, hp, step, momentum=0.0):
    start = np.concatenate([[0], np.cumsum([x.size for x in params])]).astype(np.uint32)
    rc = emu.emu_bucket_optim64(ptrs(params), ptrs(s1), ptrs(s2), start.ctypes.data_as(UP), len(params), grads.ctypes.data_as(FP),
                              grads.size, kind, hp["lr"], momentum, hp["weight_decay"], hp.get("beta1", 0.0), hp.get("beta2", 0.0),
                              hp.get("eps", 0.0), step, int(hp.get("adamw", False)))
    assert rc == 0


def _split(x):
    return [a.copy() for a in np.split(x, np.cumsum(SIZES)[:-1])]


@pytest.mark.parametrize("hp", GRID, ids=ref.grid_id)
def test_k14_adam_bit_exact_over_grid(emu, hp):
    """K14 (parameters in separate allocations of sizes 1 .. 1000, none a multiple of 8 in total) equals torch's
    foreach Adam / AdamW bit for bit: three steps from a fresh state, then single steps from random states at
    steps 10, 1000 and 10000; gradients with every edge value."""
    n = sum(SIZES)
    p, m, v = ref.state(n, 1)
    m[:], v[:] = 0.0, 0.0
    P, M, V = _split(p), _split(m), _split(v)
    for step in (1, 2, 3, 10, 1000, 10000):
        if step >= 10:
            p, m, v = ref.state(n, step)
            P, M, V = _split(p), _split(m), _split(v)
        g = ref.grads(n, 100 + step)
        _k14(emu, P, M, V, g, 1, hp, step)
        p, m, v = ref.adam_step32(p, g, m, v, step=step, **hp)
        for name, got, want in (("p", P, p), ("m", M, m), ("v", V, v)):
            assert_same_bits(np.concatenate(got), want, "%s step %d" % (name, step))


@pytest.mark.parametrize("lr,momentum,wd", [(1e-3, 0.9, 0.01), (0.05, 0.9, 0.0), (1.0, 0.0, 0.01), (0.1, 0.0, 0.0),
                                            (1e-3, 0.5, 1e-4)])
def test_k14_sgd_bit_exact(emu, lr, momentum, wd):
    """K14's SGD equals torch's over four steps; the first step starts the momentum buffer as a copy of the
    gradient (-0.0 and NaN gradients included)."""
    n = sum(SIZES)
    p, _, _ = ref.state(n, 2)
    P = _split(p)
    B = _split(np.full(n, 123.0, f32))          # the first step must not read the buffer
    buf = None
    hp = dict(lr=lr, weight_decay=wd)
    for step in (1, 2, 3, 4):
        g = ref.grads(n, 300 + step)
        _k14(emu, P, B, [np.zeros(1, f32)] * len(P), g, 0, hp, step, momentum)
        p, buf = ref.sgd_step32(p, g, buf, lr=lr, momentum=momentum, weight_decay=wd)
        assert_same_bits(np.concatenate(P), p, "p step %d" % step)
        if momentum:
            assert_same_bits(np.concatenate(B), buf, "momentum_buffer step %d" % step)


# ---- K13 and the scaled K13 ----------------------------------------------------------------------------------------------
# a representative slice of the grid: both lerp branches, both weight-decay forms, the eps extremes, lr 1
K13_GRID = [GRID[i] for i in (0, 13, 29, 34, 47, 55, 70, 88)]


def _layout(world):
    """Owner shards (multiples of 8) with one empty rank at W >= 3, and a group window inside each shard whose
    edges are multiples of 4 but not of 8."""
    lens = [8 * (60 + 13 * r) for r in range(world)]
    if world >= 3:
        lens[1] = 0
    shard = [0]
    for x in lens:
        shard.append(shard[-1] + x)
    glo = [min(4, x) for x in lens]
    ghi = [max(lo, x - 12) for lo, x in zip(glo, lens)]
    return shard, glo, ghi


@pytest.mark.parametrize("world", [1, 2, 3, 4])
@pytest.mark.parametrize("order", [0, 1])
@pytest.mark.parametrize("coef", [None, 0.37, 1.0, 0.0], ids=["K13", "scaled0.37", "scaled1", "scaled0"])
def test_k13_bit_exact(emu, world, order, coef):
    """K13 (and K13 with a clip coefficient applied on the device) on every rank's own shard equals torch's foreach
    Adam on the shard's gradients (times the coefficient, one fp32 rounding), inside the group window; outside it
    nothing changes; every rank ends with the same whole parameter vector."""
    shard, glo, ghi = _layout(world)
    total = shard[-1]
    lens = [shard[r + 1] - shard[r] for r in range(world)]
    sig = emu.emu_signal_bytes()
    g = emu.emu_group_create(world, 2 << 20)
    off = (ctypes.c_longlong * (world + 1))(*shard)
    try:
        epoch = 1
        for k, hp in enumerate(K13_GRID):
            p, m, v = ref.state(total, 50 + k)
            gr = ref.grads(total, 60 + k)
            step = (1, 2, 10, 1000)[k % 4]
            views = []
            for r in range(world):
                x = np.ctypeslib.as_array(emu.emu_arena_ptr(g, r, sig), shape=(total,))
                x[:] = p
                views.append(x)
            ms = [np.resize(m[shard[r]:shard[r + 1]], max(lens[r], 8)).astype(f32) for r in range(world)]
            vs = [np.resize(v[shard[r]:shard[r + 1]], max(lens[r], 8)).astype(f32) for r in range(world)]
            red = [np.resize(gr[shard[r]:shard[r + 1]], max(lens[r], 8)).astype(f32) for r in range(world)]
            args = (g, 0, sig, ptrs(ms), ptrs(vs), ptrs(red), total, off, 1, (ctypes.c_longlong * world)(*glo),
                    (ctypes.c_longlong * world)(*ghi), hp["lr"], hp["beta1"], hp["beta2"], hp["eps"], hp["weight_decay"],
                    step, int(hp["adamw"]), epoch, order, 0)
            if coef is None:
                assert emu.emu_adam_push64(*args) == 0
            else:
                sc = [np.full(1, coef, f32) for _ in range(world)]
                assert emu.emu_adam_push_scaled64(*args, ptrs(sc)) == 0
            epoch += 1
            want_p = p.copy()
            for r in range(world):
                lo, hi = shard[r] + glo[r], shard[r] + ghi[r]
                gg = gr[lo:hi] if coef is None else ref.mul_scalar(gr[lo:hi], coef)
                pn, mn, vn = ref.adam_step32(p[lo:hi], gg, m[lo:hi], v[lo:hi], step=step, **hp)
                want_p[lo:hi] = pn
                want_m, want_v = m[shard[r]:shard[r + 1]].copy(), v[shard[r]:shard[r + 1]].copy()
                want_m[glo[r]:ghi[r]], want_v[glo[r]:ghi[r]] = mn, vn
                what = "%s rank %d" % (ref.grid_id(hp), r)
                assert_same_bits(ms[r][:lens[r]], want_m, "m " + what)
                assert_same_bits(vs[r][:lens[r]], want_v, "v " + what)
            for r in range(world):
                assert_same_bits(views[r], want_p, "p %s on rank %d" % (ref.grid_id(hp), r))
    finally:
        emu.emu_group_destroy(g)


# ---- K5 --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world,generic", [(1, 1), (2, 0), (3, 1), (4, 0)])
def test_k5_bit_exact(emu, world, generic):
    """The fused sharded step (reduce-scatter, Adam in registers, all-gather) equals torch's foreach Adam on the
    fp32-wire average of the ranks' gradients, over a slice of the grid and three consecutive steps each."""
    rng = np.random.default_rng(world)
    numels = [int(x) for x in rng.integers(1, 400, size=7)] + [900]
    owner = ddp_oracle.partition_fairscale(numels, world)
    _, shard_off, total = ddp_oracle.shard_layout(numels, owner, world)
    lens = [shard_off[r + 1] - shard_off[r] for r in range(world)]
    off = (ctypes.c_longlong * (world + 1))(*shard_off)
    sig = emu.emu_signal_bytes()
    scale = float(f32(1.0) / f32(world))
    g = emu.emu_group_create(world, 4 << 20)
    try:
        parity = 0
        for k, hp in enumerate(K13_GRID[::2]):
            p, _, _ = ref.state(total, 80 + k)
            m, v = np.zeros(total, f32), np.zeros(total, f32)
            views = []
            for r in range(world):
                x = np.ctypeslib.as_array(emu.emu_arena_ptr(g, r, sig), shape=(total,))
                x[:] = p
                views.append(x)
            ms = [np.zeros(max(x, 8), f32) for x in lens]
            vs = [np.zeros(max(x, 8), f32) for x in lens]
            for step in (1, 2, 3):
                per_rank = [torch.from_numpy(ref.grads(total, 1000 * k + 10 * step + r, edges=(r == 0))) for r in range(world)]
                grads = [t.numpy().copy() for t in per_rank]
                rc = emu.emu_sharded_step64(g, 0, ptrs(grads), sig, ptrs(ms), ptrs(vs), total, off, scale, hp["lr"], hp["beta1"],
                                          hp["beta2"], hp["eps"], hp["weight_decay"], step, int(hp["adamw"]), 0, 2, parity, generic)
                assert rc == 0
                parity ^= 1
                avg = ddp_oracle.allreduce_fp32_wire(per_rank, scale).numpy()
                p, m, v = ref.adam_step32(p, avg, m, v, step=step, **hp)
                what = "%s step %d" % (ref.grid_id(hp), step)
                for r in range(world):
                    assert_same_bits(views[r], p, "p rank %d %s" % (r, what))
                    assert_same_bits(ms[r][:lens[r]], m[shard_off[r]:shard_off[r + 1]], "m rank %d %s" % (r, what))
                    assert_same_bits(vs[r][:lens[r]], v[shard_off[r]:shard_off[r + 1]], "v rank %d %s" % (r, what))
    finally:
        emu.emu_group_destroy(g)


def test_grid_covers_both_lerp_branches_and_all_decay_forms():
    seen = {(abs(f32(1 - hp["beta1"])) < f32(0.5), hp["adamw"], hp["weight_decay"] != 0) for hp in K13_GRID}
    assert len({s[0] for s in seen}) == 2 and len({s[1:] for s in seen}) == 3
    assert len(GRID) == 90 and math.prod([len(ref.BETAS), len(ref.EPS), len(ref.LRS), len(ref.DECAY)]) == 90
