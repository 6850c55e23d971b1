"""csrc/gen.cu restated in numpy, operation by operation: the power-law CSR of als_csr_generate and the factor fill of
als_factors_fill_uniform, bit for bit, for tests/test_gpu_generate.py.

Every hash is computed on uint64 arrays, whose arithmetic wraps like the kernels'; the per-stream constants are Python
ints reduced mod 2^64.  u01 is exact in float64.  The power-law draw is evaluated in float64 in the kernel's order, but
the device's pow is only accurate to 2 ulp and nvcc may fuse the affine step into an FMA: a draw whose x lies within
FLAG_ULPS ulp of an integer may floor to the other side on the device, so it is flagged, and a bitwise comparison holds
only for inputs that flag no draw.  The thinning threshold is computed in x86 80-bit long double, as the host side of
gen.cu computes it (keep_threshold refuses other long doubles)."""
import numpy as np

M64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15
FLAG_ULPS = 64  # the outer exponent 1 / (1 - 0.8) = 5 multiplies a relative error of the inner pow fivefold

_U64 = np.uint64


def mix64_int(x):
    """splitmix64's finaliser on one Python int."""
    x = (x + GOLDEN) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def mix64(x):
    """splitmix64's finaliser on a uint64 array (wrapping arithmetic)."""
    x = np.asarray(x, dtype=_U64) + _U64(GOLDEN)
    x = (x ^ (x >> _U64(30))) * _U64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> _U64(27))) * _U64(0x94D049BB133111EB)
    return x ^ (x >> _U64(31))


def hash3(seed, stream, i):
    """hash3(seed, stream, i) of gen.cu for a uint64 array i (or anything np.asarray makes one of)."""
    inner = mix64_int((seed * 0x2545F4914F6CDD1D + stream) & M64)
    i = np.atleast_1d(np.asarray(i, dtype=_U64))
    return mix64(_U64(inner) ^ (i * _U64(GOLDEN)))


def u01(h):
    """(h >> 11) * 2^-53: a 53-bit integer times a power of two, exact in float64."""
    return (h >> _U64(11)).astype(np.float64) * 2.0 ** -53


def plaw(r, N, a):
    """(draws, flagged): the truncated power law of gen.cu's plaw for the uniforms r, and which draws lie within
    FLAG_ULPS ulp of an integer k before the floor, where the two floors k - 1 and k give different clamped draws."""
    x = np.power((float(N) ** (1.0 - a) - 1.0) * r + 1.0, 1.0 / (1.0 - a))
    k = np.rint(x).astype(np.int64)
    flagged = (np.abs(x - k) <= FLAG_ULPS * np.spacing(x)) & (np.clip(k - 2, 0, N - 1) != np.clip(k - 1, 0, N - 1))
    return np.clip(np.floor(x).astype(np.int64) - 1, 0, N - 1), flagged


def permutation(n, seed, stream):
    """random_permutation: the indices 0 .. n-1 sorted by hash3(seed, stream, i); CUB's radix sort is stable."""
    return np.argsort(hash3(seed, stream, np.arange(n, dtype=_U64)), kind="stable").astype(np.int32)


def draws(users, items, seed, t, pu, pi):
    """(keys, flagged) of the draws t (a uint64 array of draw indices) of draw_keys_kernel, from the permutations."""
    u, fu = plaw(u01(hash3(seed, 11, t)), users, 0.5)
    i, fi = plaw(u01(hash3(seed, 12, t)), items, 0.8)
    return pu[u].astype(_U64) * _U64(items) + pi[i].astype(_U64), fu | fi


def keep_threshold(nnz_target, n_unique):
    """uint64(nnz_target / n_unique * (2^64 - 1)) in x86 80-bit long double, as csr_generate_power_law computes it."""
    if np.finfo(np.longdouble).nmant != 63:
        raise NotImplementedError("needs x86 80-bit long double")
    p = np.longdouble(nnz_target) / np.longdouble(n_unique)
    return int(np.array(p * np.longdouble(M64)).astype(_U64))


def kept(seed, keys, threshold):
    """KeepKey: a key survives the thinning when hash3(seed, 13, key) < threshold."""
    return hash3(seed, 13, keys) < _U64(threshold)


def values(seed, keys):
    """split_keys_kernel's values 1 + 4 (float)u01: 4 x is exact, so an FMA cannot change the sum's rounding."""
    return np.float32(1) + np.float32(4) * u01(hash3(seed, 14, keys)).astype(np.float32)


class Restated:
    """The CSR of als_csr_generate(users, items, nnz_target, seed), with what its stream did on the way."""

    def __init__(self, users, items, nnz_target, seed):
        m = nnz_target + nnz_target // 4
        pu, pi = permutation(users, seed, 1), permutation(items, seed, 2)
        keys, flagged = draws(users, items, seed, np.arange(m, dtype=_U64), pu, pi)
        self.draws, self.flagged = m, int(flagged.sum())
        keys = np.unique(keys)
        self.n_unique = len(keys)
        self.threshold = None
        if self.n_unique > nnz_target:
            self.threshold = keep_threshold(nnz_target, self.n_unique)
            keys = keys[kept(seed, keys, self.threshold)]
        self.shape = (users, items)
        self.nnz = len(keys)
        self.indices = (keys % _U64(items)).astype(np.int32)
        self.data = values(seed, keys)
        self.indptr = np.searchsorted(keys, np.arange(users + 1, dtype=_U64) * _U64(items)).astype(np.int32)


def fill_uniform(f, seed, scale, row0, nrows):
    """Rows row0 .. row0 + nrows - 1 of fill_uniform_kernel's (rows, f) matrix: element (r, j) is
    float32(scale) * float32(u01(hash3(seed, 21, r f + j))); the padding columns past f are zero."""
    e = np.arange(row0, row0 + nrows, dtype=_U64)[:, None] * _U64(f) + np.arange(f, dtype=_U64)[None, :]
    return np.float32(scale) * u01(hash3(seed, 21, e.ravel())).astype(np.float32).reshape(nrows, f)
