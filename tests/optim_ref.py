"""NumPy restatement of torch.optim.Adam / AdamW / SGD as torch runs them on CUDA, for fp32 parameters.

Every ATen operation of `_single_tensor_*` ("single", foreach=False) and `_multi_tensor_*` ("foreach", the default
for CUDA parameters) rounds once to fp32, in the order torch issues them; the functions below spell out that order
with exactly rounded fp32 NumPy arithmetic and an exact fp32 fused multiply-add (`fma32`).  Where an ATen CUDA kernel
computes `a + b * c` the compiler contracts it into one fused multiply-add, and so does this file; test_gpu_optim.py
checks each operation against torch on the device, one by one.

Host constants follow Python: float64 arithmetic (`beta ** step`, `bc2 ** 0.5`, `lr / bc1`), one cast to fp32
where the value becomes a kernel argument.

`adam_step64` / `sgd_step64` are the same updates in float64 from the same fp32 inputs: the high-precision
reference that error bounds are measured against, independent of any rounding choice."""
import numpy as np

f32, f64 = np.float32, np.float64
_INF = np.float64(np.inf)


def _quiet(fn):
    """IEEE arithmetic on purpose: overflow, inf - inf and 0 * inf are part of what is restated."""
    def run(*args, **kw):
        with np.errstate(all="ignore"):
            return fn(*args, **kw)
    run.__name__, run.__doc__ = fn.__name__, fn.__doc__
    return run


def fma32(a, b, c):
    """fp32 fused multiply-add a * b + c with one rounding (round to nearest even), element-wise.

    The float64 product of two fp32 values is exact; the float64 sum p + c is rounded once and its TwoSum residual
    holds what was lost.  Rounding that sum to fp32 gives the correctly rounded result unless it landed exactly on an
    fp32 rounding midpoint while the exact value did not: then one float64 step towards the residual breaks the tie.
    fp32 midpoints, subnormal ones and the overflow threshold included, are float64 values, so no other case exists."""
    a, b, c = np.broadcast_arrays(np.asarray(a, f32), np.asarray(b, f32), np.asarray(c, f32))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a.astype(f64) * b.astype(f64)
        cc = c.astype(f64)
        s = p + cc
        bb = s - p
        err = (p - (s - bb)) + (cc - bb)
        r = s.astype(f32)
        rd = r.astype(f64)
        # the fp32 neighbour of r on the other side of s; past FLT_MAX the grid continues with 2^128
        over = np.isinf(r) & np.isfinite(s)
        rd = np.where(over, np.copysign(2.0 ** 128, s), rd)
        other = np.nextafter(np.where(over, np.copysign(np.finfo(f32).max, s), r).astype(f32),
                             np.where(s > rd, f32(np.inf), f32(-np.inf))).astype(f64)
        other = np.where(over, np.copysign(np.finfo(f32).max, s).astype(f64), other)
        tie = np.isfinite(s) & (s != rd) & (s == (rd + other) * 0.5) & (err != 0) & np.isfinite(err)
        if tie.any():
            nudged = np.nextafter(s[tie], np.where(err[tie] > 0, _INF, -_INF))
            r = r.copy()
            r[tie] = nudged.astype(f32)
    return r


# ---- ATen's CUDA kernels, one rounding each ------------------------------------------------------------------------
@_quiet
def mul_scalar(x, s):
    """x.mul_(s) / _foreach_mul_(x, s): the Python float becomes fp32 first."""
    return (np.asarray(x, f32) * f32(s)).astype(f32)


@_quiet
def add_scalar(x, s):
    """x.add_(s) / _foreach_add_(x, s)."""
    return (np.asarray(x, f32) + f32(s)).astype(f32)


@_quiet
def add_alpha(x, y, alpha):
    """x.add(y, alpha=a) / _foreach_add(x, y, alpha=a): x + a * y, contracted; alpha == 1 is a plain sum."""
    return fma32(f32(alpha), y, x)


@_quiet
def lerp(x, end, w):
    """x.lerp_(end, w) / _foreach_lerp_ with a scalar weight (ATen/native/Lerp.h): the weight becomes fp32; below
    |w| < 0.5 the result is x + w * (end - x), otherwise end - (end - x) * (1 - w), each contracted."""
    w = f32(w)
    x, end = np.asarray(x, f32), np.asarray(end, f32)
    d = (end - x).astype(f32)
    if abs(w) < f32(0.5):
        return fma32(w, d, x)
    return fma32(-d, f32(f32(1) - w), end)


@_quiet
def addcmul(x, t1, t2, value):
    """x.addcmul_(t1, t2, value=v) / _foreach_addcmul_(x, t1, t2, v): x + v * (t1 * t2), contracted."""
    return fma32(f32(value), (np.asarray(t1, f32) * np.asarray(t2, f32)).astype(f32), x)


@_quiet
def addcdiv(x, t1, t2, value):
    """x.addcdiv_(t1, t2, value=v) / _foreach_addcdiv_ with a scalar or a scalar list: x + v * (t1 / t2), contracted."""
    with np.errstate(divide="ignore", invalid="ignore"):
        q = (np.asarray(t1, f32) / np.asarray(t2, f32)).astype(f32)
    return fma32(f32(value), q, x)


@_quiet
def div_scalar(x, s):
    """tensor / python_float on CUDA (div_true_kernel_cuda with a CPU scalar): a multiply by the reciprocal, formed in
    float64 and rounded to fp32 once."""
    inv = f32(1.0 / float(s))
    return (np.asarray(x, f32) * inv).astype(f32)


@_quiet
def div_scalar_list(x, s):
    """_foreach_div_(xs, [s, ...]): a true fp32 division by the fp32 scalar."""
    return (np.asarray(x, f32) / f32(s)).astype(f32)


@_quiet
def sqrt(x):
    with np.errstate(invalid="ignore"):
        return np.sqrt(np.asarray(x, f32)).astype(f32)


# ---- the optimizers ---------------------------------------------------------------------------------------------------
def adam_consts(lr, beta1, beta2, step):
    """Python's float64 host arithmetic of torch/optim/adam.py (non-capturable): bc1, bc2, lr / bc1, sqrt(bc2)."""
    bc1 = 1 - beta1 ** step
    bc2 = 1 - beta2 ** step
    return bc1, bc2, lr / bc1, bc2 ** 0.5


@_quiet
def adam_step32(p, g, m, v, *, lr, beta1, beta2, eps, weight_decay=0.0, adamw=False, step, path="foreach"):
    """One step of torch.optim.Adam (adamw=False) / AdamW on CUDA fp32 tensors; returns new (p, m, v).
    `step` is the count after the increment.  path: "single" (foreach=False) or "foreach" (the CUDA default)."""
    assert path in ("single", "foreach")
    p, g, m, v = (np.asarray(x, f32).copy() for x in (p, g, m, v))
    if weight_decay != 0:
        if adamw:
            p = mul_scalar(p, 1 - lr * weight_decay)
        else:
            g = add_alpha(g, p, weight_decay)
    m = lerp(m, g, 1 - beta1)
    v = addcmul(mul_scalar(v, beta2), g, g, 1 - beta2)
    _, _, step_size, bc2_sqrt = adam_consts(lr, beta1, beta2, step)
    s = sqrt(v)
    s = div_scalar(s, bc2_sqrt) if path == "single" else div_scalar_list(s, bc2_sqrt)
    denom = add_scalar(s, eps)
    p = addcdiv(p, m, denom, -step_size if path == "single" else (lr / (1 - beta1 ** step)) * -1)
    return p, m, v


@_quiet
def sgd_step32(p, g, buf, *, lr, momentum=0.0, weight_decay=0.0, path="foreach"):
    """One step of torch.optim.SGD (dampening 0, no nesterov) on CUDA fp32 tensors; returns new (p, buf).
    buf is None before the first step with momentum (torch then clones the gradient into it).  Both paths issue
    the same element-wise operations."""
    assert path in ("single", "foreach")
    p, g = np.asarray(p, f32).copy(), np.asarray(g, f32).copy()
    if weight_decay != 0:
        g = add_alpha(g, p, weight_decay)
    if momentum != 0:
        if buf is None:
            buf = g.copy()
        else:
            buf = (mul_scalar(buf, momentum) + g).astype(f32)
        g = buf
    p = add_alpha(p, g, -lr)
    return p, buf


def adam_step64(p, g, m, v, *, lr, beta1, beta2, eps, weight_decay=0.0, adamw=False, step):
    """The Adam / AdamW update in float64 from fp32 inputs.  Returns float64 (p, m, v) and the error each fp32
    result may carry: a small multiple of 2^-24 times the magnitudes of the terms of its update (the error of the
    quantities it is computed from included), plus a subnormal-sized floor.  A correct fp32 implementation of
    torch's operation order, on either path, stays inside; a constant narrowed to fp32 before the float64 arithmetic
    (1.3e-5 relative for 1 - beta2 = 0.001) or eps moved inside the square root does not.  Meaningful where the
    float64 values stay in fp32's finite range; the non-finite patterns are pinned bit for bit elsewhere."""
    e, floor = 2.0 ** -24, 2.0 ** -148
    p, g, m, v = (np.asarray(x, f32).astype(f64) for x in (p, g, m, v))
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        gmag = np.abs(g)
        if weight_decay != 0 and not adamw:
            gmag = gmag + np.abs(weight_decay * p)
            g = g + weight_decay * p
        pmag = np.abs(p)
        if weight_decay != 0 and adamw:
            p = p * (1 - lr * weight_decay)
        tol_m = 4 * e * (np.abs(m) + gmag) + floor
        m = m + (1 - beta1) * (g - m)
        tv = beta2 * v + (1 - beta2) * gmag * gmag
        tol_v = 6 * e * tv + floor
        v = beta2 * v + (1 - beta2) * g * g
        bc1, bc2, step_size, _ = adam_consts(lr, beta1, beta2, step)
        sv = np.sqrt(v)
        tol_s = np.minimum(np.where(sv > 0, tol_v / (2 * sv), np.inf), np.sqrt(tol_v)) + 2 * e * sv
        denom = sv / np.sqrt(bc2) + eps
        tol_d = tol_s / np.sqrt(bc2) + 4 * e * denom
        upd = step_size * m / denom
        tol_u = step_size * (tol_m / denom + np.abs(m) * tol_d / (denom * denom)) + 4 * e * np.abs(upd)
        p = p - upd
        tol_p = tol_u + 2 * e * pmag + 2 * e * np.abs(p) + floor
    return (p, m, v), (tol_p, tol_m, tol_v)


def sgd_step64(p, g, buf, *, lr, momentum=0.0, weight_decay=0.0):
    """The SGD update in float64 from fp32 inputs; returns float64 (p, buf)."""
    p, g = np.asarray(p, f32).astype(f64), np.asarray(g, f32).astype(f64)
    with np.errstate(invalid="ignore", over="ignore"):
        if weight_decay != 0:
            g = g + weight_decay * p
        if momentum != 0:
            buf = g if buf is None else momentum * np.asarray(buf, f32).astype(f64) + g
            g = buf
        p = p - lr * g
    return p, buf


def sgd_bound64(p, g, buf, *, lr, momentum=0.0, weight_decay=0.0):
    """The error an fp32 SGD step may carry against sgd_step64, for (p, buf): a few roundings of 2^-24 times the
    magnitudes of the terms of each update (the decayed gradient, the momentum buffer, the parameter), plus a
    subnormal-sized floor.  An fp32 implementation of torch's order of operations stays inside whether or not it
    contracts `a + b * c` into a fused multiply-add (torch's single-tensor, foreach and fused kernels differ there).
    `buf` is the buffer before the step (None on the first step with momentum); the buffer's bound is None without
    momentum."""
    e, floor = 2.0 ** -24, 2.0 ** -148
    p, g = np.asarray(p, f32).astype(f64), np.asarray(g, f32).astype(f64)
    with np.errstate(invalid="ignore", over="ignore"):
        gmag = np.abs(g) + np.abs(weight_decay * p)
        tol_g = 2 * e * gmag + floor
        tol_b = None
        if momentum != 0:
            bmag = gmag if buf is None else momentum * np.abs(np.asarray(buf, f32).astype(f64)) + gmag
            tol_b = tol_g + 3 * e * bmag + floor
            tol_g, gmag = tol_b, bmag
        pn, _ = sgd_step64(p.astype(f32), g.astype(f32), buf, lr=lr, momentum=momentum, weight_decay=weight_decay)
        tol_p = lr * tol_g + 2 * e * (np.abs(p) + lr * gmag + np.abs(pn)) + floor
    return tol_p, tol_b


# ---- the grid the tests run ------------------------------------------------------------------------------------------
BETAS = [(0.9, 0.999), (0.9, 0.95), (0.0, 0.99), (0.5, 0.9), (0.3, 0.999)]
EPS = [1e-8, 1e-6, 1e-12]
LRS = [1e-3, 1.0]
DECAY = [(False, 0.0), (False, 0.01), (True, 0.1)]     # (adamw, weight_decay)


def adam_grid():
    """Every hyper-parameter set of the grid, as keyword arguments of adam_step32 (without `step`)."""
    return [dict(lr=lr, beta1=b1, beta2=b2, eps=eps, weight_decay=wd, adamw=aw)
            for (b1, b2) in BETAS for eps in EPS for lr in LRS for (aw, wd) in DECAY]


def grid_id(hp):
    return "%s-b%g,%g-eps%g-lr%g-wd%g" % ("adamw" if hp["adamw"] else "adam", hp["beta1"], hp["beta2"], hp["eps"],
                                          hp["lr"], hp["weight_decay"])


# gradients where kernels go wrong: zero (m = v = 0, denominator eps), -0.0, eps-dominated, subnormal (g * g
# underflows), overflowing v, non-finite
GRAD_EDGES = np.array([0.0, -0.0, 1e-9, -1e-9, 1e-20, 1e-42, -3e-39, 2e-23, 1e18, -1e18, 1e21, -1e21,
                       np.inf, -np.inf, np.nan], f32)


def grads(n, seed, edges=True):
    """n fp32 gradients: N(0, 0.1) scaled by 2^U(-20, 4), with every edge value at many places when `edges`."""
    rng = np.random.default_rng(seed)
    g = (rng.standard_normal(n) * 0.1 * 2.0 ** rng.integers(-20, 5, n)).astype(f32)
    if edges:
        idx = rng.permutation(n)[:min(n, 8 * len(GRAD_EDGES))]
        g[idx] = np.resize(GRAD_EDGES, len(idx))
    return g


def state(n, seed, kind="adam"):
    """Random optimizer state as it looks some steps in: p ~ N(0, 1), m ~ N(0, 0.01), v >= 0 (a few zeros)."""
    rng = np.random.default_rng(seed)
    p = rng.standard_normal(n).astype(f32)
    m = (rng.standard_normal(n) * 0.01 * 2.0 ** rng.integers(-10, 3, n)).astype(f32)
    v = (np.abs(rng.standard_normal(n)) * 1e-4 * 2.0 ** rng.integers(-20, 3, n)).astype(f32)
    z = rng.permutation(n)[:max(1, n // 50)]
    m[z], v[z] = 0.0, 0.0
    return p, m, v
