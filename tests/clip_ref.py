"""NumPy restatement of the global-norm kernels (csrc/b2d_clip.cuh): K18's fixed summation order and K19's arithmetic.

Every float64 add here is one IEEE operation (what __dadd_rn does), the square of a float32 is exact in float64, and
the float32 steps of the coefficient are single numpy.float32 operations, so a kernel that follows the same order
matches these functions bit for bit."""
import numpy as np

TILE = 4096          # elements per tile
THREADS = 256        # threads per block; also the width of every tree
G_MAX = 256          # the library's block cap (kClipGMax)


def _tree(vals):
    """Fixed shared-memory tree over THREADS float64 values (zero-padded), strides 128 .. 1."""
    s = np.zeros(THREADS, np.float64)
    s[:len(vals)] = vals
    stride = THREADS // 2
    while stride:
        s[:stride] = s[:stride] + s[stride:2 * stride]
        stride //= 2
    return s[0]


def grid(n, gmax=G_MAX):
    ntiles = -(-n // TILE)
    return 1 if ntiles == 0 else min(gmax, ntiles)


def tile_sums(x):
    """Sum of squares of every tile: thread t adds vectors t, t+256, t+512, t+768 in order (x, y, z, w within each),
    then the tree over the 256 thread sums."""
    x = np.asarray(x, np.float32)
    n = len(x)
    ntiles = -(-n // TILE)
    pad = np.zeros(ntiles * TILE, np.float64)
    pad[:n] = x
    sq = (pad * pad).reshape(ntiles, 4, THREADS, 4)        # [tile, j, thread, lane]
    acc = np.zeros((ntiles, THREADS), np.float64)
    for j in range(4):
        for k in range(4):
            acc = acc + sq[:, j, :, k]
    return [_tree(acc[t]) for t in range(ntiles)]


def partial(x, gmax=G_MAX):
    """K18: one rank's float64 sum of squares of its n elements."""
    ts = tile_sums(x)
    g = grid(len(ts) * TILE, gmax)
    block = []
    for b in range(g):
        s = np.float64(0.0)
        for t in range(b, len(ts), g):
            s = s + ts[t]
        block.append(s)
    return _tree(np.array(block, np.float64))


def norm_coef(partials, max_norm):
    """K19: rank-ordered float64 total, float32 norm, torch's coefficient (max_norm / (norm + 1e-6), clamped to 1)."""
    total = np.float64(partials[0])
    for p in partials[1:]:
        total = total + np.float64(p)
    norm = np.float32(np.sqrt(total))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        coef = (np.float32(1.0) / (norm + np.float32(1e-6))) * np.float32(max_norm)
    coef = np.float32(1.0) if coef > np.float32(1.0) else np.float32(coef)   # NaN stays NaN
    return norm, coef
