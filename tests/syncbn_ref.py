"""Float32 restatement of libb2d's synchronised-BatchNorm exchange (csrc/b2d_syncbn.cuh), one rounding per
operation, for the CPU and GPU SyncBN tests.  numpy float32 arithmetic rounds every elementwise operation once, as
the kernels' __fadd_rn / __fmul_rn / __fdiv_rn / __fsqrt_rn do, so the kernels must match it bit for bit."""
import numpy as np

f32 = np.float32


def combine_stats(means, invstds, counts, eps, momentum, running_mean=None, running_var=None):
    """Rank-ordered Chan merge of the W forward rows, rows with count 0 skipped (K16).

    means / invstds: per rank a float32 [C] array, or None for an empty rank; counts: per rank elements per channel.
    Returns (mean, invstd, counts int32 [W], running_mean, running_var) — the last two None when not given."""
    C = next(len(m) for m in means if m is not None)
    eps, mom = f32(eps), f32(momentum)
    avg = np.zeros(C, f32)
    var_n = np.zeros(C, f32)
    n = f32(0)
    for m, s, c in zip(means, invstds, counts):
        c = f32(c)
        if c == 0:
            continue
        m, s = np.asarray(m, f32), np.asarray(s, f32)
        v = f32(1) / s
        v = (v * v - eps) * c
        factor = f32(1) / (n + c)
        d = avg - m
        var_n = var_n + (v + d * d * n * c * factor)
        avg = n * factor * avg + c * factor * m
        n = n + c
    invstd = f32(1) / np.sqrt(var_n / n + eps)
    keep = f32(1) - mom
    rm = rv = None
    if running_mean is not None:
        rm = keep * np.asarray(running_mean, f32) + mom * avg
    if running_var is not None:
        rv = keep * np.asarray(running_var, f32) + mom * (var_n / (n - f32(1)))
    return avg, invstd, np.asarray([int(c) for c in counts], np.int32), rm, rv


def sum_rows(rows):
    """Rank-ordered fp32 sum of the W backward rows (K17); None stands for a zero row."""
    C = next(len(r) for r in rows if r is not None)
    acc = None
    for r in rows:
        r = np.zeros(C, f32) if r is None else np.asarray(r, f32)
        acc = r.copy() if acc is None else acc + r
    return acc


def local_stats(x, eps):
    """What torch.batch_norm_stats gives one rank (mean, 1/sqrt(biased var + eps)) over dim 1 as channels, computed
    in float64 and rounded to float32 once."""
    x = np.asarray(x, np.float64)
    xc = np.moveaxis(x, 1, 0).reshape(x.shape[1], -1)
    mean = xc.mean(1)
    var = xc.var(1)
    return mean.astype(f32), (1.0 / np.sqrt(var + eps)).astype(f32), xc.shape[1]
