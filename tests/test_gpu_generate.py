"""The device generators of csrc/gen.cu against their numpy restatement (tests/_gen_restate.py): als_csr_generate bit
for bit from one draw to the C2 shape, its refusals, the whole C4 input (10M x 1M, 500M nonzeros) by its invariants, a
sample of its draws and its digest on a second run and a second device, its statistics against the host generator
(implicit_b200/synthetic.py) at the C2 shape, and als_factors_fill_uniform bit for bit at every padded width class and
past 2^31 elements.  C4's benchmark inputs and every rank's copy of them come from these two kernels."""
import hashlib

import numpy as np
import pytest

import _gen_restate as gr
import helpers

torch = pytest.importorskip("torch")

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs PyTorch with CUDA to read the padding")]


@pytest.fixture(scope="module")
def lib():
    from implicit_b200 import _lib

    return _lib


@pytest.fixture(scope="module")
def ctx(lib):
    c = lib.Context(0)
    yield c
    c.close()


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def generated(lib, ctx, users, items, nnz, seed):
    """(shape3, indptr, indices, data) of als_csr_generate, downloaded; the device CSR is closed."""
    C = lib.DeviceCSR.generate(ctx, users, items, nnz, seed)
    try:
        m = C.download()
        return C.shape3, m.indptr, m.indices, m.data
    finally:
        C.close()


def restated(users, items, nnz, seed):
    try:
        return gr.Restated(users, items, nnz, seed)
    except NotImplementedError as e:  # the thinning threshold is an x86 80-bit long double computation
        pytest.skip(str(e))


def digest(indptr, indices, data):
    h = hashlib.blake2b()
    for a in (indptr, indices, data):
        h.update(np.ascontiguousarray(a).data)
    return h.hexdigest()


C2 = (360_000, 300_000, 17_000_000, 2)


@pytest.fixture(scope="module")
def c2_device(lib, ctx):
    return generated(lib, ctx, *C2)


# (users, items, nnz_target, seed), whether the unique keys outnumber the target (the thinning runs)
BITWISE = [
    pytest.param((1, 1, 1, 7), False, id="one-draw"),                 # every draw gives the same key
    pytest.param((1, 5000, 800, 7), False, id="one-user"),
    pytest.param((1, 1_000_000, 5000, 7), True, id="one-user-thinned"),
    pytest.param((2000, 1, 1000, 7), False, id="one-item"),
    pytest.param((5000, 1, 800, 7), True, id="one-item-thinned"),
    pytest.param((8, 8, 1000, 7), False, id="fewer-keys-than-target"),
    pytest.param((500, 400, 8000, 22), True, id="alloc-failure-shape"),
    pytest.param((5, (1 << 24) + 3, 300_000, 7), True, id="items-2^24+3"),  # columns past float32's integers
]


@pytest.mark.parametrize("case,thins", BITWISE)
def test_generate_is_restated(lib, ctx, case, thins):
    R = restated(*case)
    assert R.flagged == 0, "a draw of this seed may floor differently on the device: pick another seed"
    assert (R.threshold is not None) == thins
    shape3, indptr, indices, data = generated(lib, ctx, *case)
    assert shape3 == (case[0], case[1], R.nnz)
    np.testing.assert_array_equal(indptr, R.indptr)
    np.testing.assert_array_equal(indices, R.indices)
    np.testing.assert_array_equal(bits(data), bits(R.data))


def test_generate_c2_is_restated(c2_device):
    R = restated(*C2)
    assert R.flagged == 0 and R.threshold is not None
    shape3, indptr, indices, data = c2_device
    assert shape3 == (C2[0], C2[1], R.nnz)
    np.testing.assert_array_equal(indptr, R.indptr)
    np.testing.assert_array_equal(indices, R.indices)
    np.testing.assert_array_equal(bits(data), bits(R.data))


INT32_MAX = 2**31 - 1
M_AT_INT32_MAX = 1_717_986_918  # the least target whose draws, nnz + nnz / 4, reach INT32_MAX


@pytest.mark.parametrize("shape,code,match", [
    ((1000, 1000, M_AT_INT32_MAX), "UNSUPPORTED", rf"csr_generate: sizes beyond int32 \(m = {INT32_MAX}\)"),
    ((INT32_MAX, 1000, 1000), "UNSUPPORTED", "csr_generate: sizes beyond int32"),
    ((1000, INT32_MAX, 1000), "UNSUPPORTED", "csr_generate: sizes beyond int32"),
    ((0, 1000, 1000), "INVALID", "als_csr_generate: empty shape"),
    ((1000, 0, 1000), "INVALID", "als_csr_generate: empty shape"),
    ((1000, 1000, 0), "INVALID", "als_csr_generate: empty shape"),
    ((-1, 1000, 1000), "INVALID", "als_csr_generate: empty shape"),
])
def test_generate_refusals(lib, ctx, shape, code, match):
    assert M_AT_INT32_MAX + M_AT_INT32_MAX // 4 == INT32_MAX
    assert (M_AT_INT32_MAX - 1) + (M_AT_INT32_MAX - 1) // 4 < INT32_MAX
    used = ctx.mem_peak()[0]
    with pytest.raises(lib.AlsError, match=match) as e:
        lib.DeviceCSR.generate(ctx, *shape, 1)
    assert e.value.code == getattr(lib, "ALS_E_" + code)
    assert ctx.mem_peak()[0] == used


def ks(a, b):
    """The two-sample Kolmogorov-Smirnov distance sup |F_a - F_b| (ties included: the CDFs are taken right-closed)."""
    a, b = np.sort(a), np.sort(b)
    v = np.concatenate([a, b])
    return float(np.max(np.abs(np.searchsorted(a, v, "right") / len(a) - np.searchsorted(b, v, "right") / len(b))))


def test_c2_statistics_match_the_host_generator(c2_device):
    """The device recipe hashes where the host one draws from PCG64, and thins by a Bernoulli draw per key where the host
    samples exactly nnz keys: the row degrees, column degrees and values must be as close to the host generator's at
    seed 2 as the host generator's at seed 3 are, up to a factor of 2 (Kolmogorov-Smirnov distances)."""
    from implicit_b200 import synthetic

    users, items, nnz, seed = C2
    _, indptr, indices, data = c2_device
    h2 = synthetic.power_law_csr(users, items, nnz, seed)
    h3 = synthetic.power_law_csr(users, items, nnz, seed + 1)

    def stats(indptr, indices, data):
        return {"row degrees": np.diff(indptr), "column degrees": np.bincount(indices, minlength=items), "values": data}

    dev, a, b = stats(indptr, indices, data), stats(h2.indptr, h2.indices, h2.data), stats(h3.indptr, h3.indices, h3.data)
    for name in dev:
        d, s = ks(dev[name], a[name]), ks(a[name], b[name])
        print(f"C2 {name}: KS(device, host seed 2) {d:.2e}, KS(host seed 2, host seed 3) {s:.2e}")
        assert d <= 2 * s, name


# ------------------------------------------------------------------------------------------------ the C4 shape
C4 = (10_000_000, 1_000_000, 500_000_000, 4)


@pytest.fixture(scope="module")
def c4(lib, ctx):
    """The C4 input, generated once and downloaded: (indptr, indices, data, digest)."""
    if ctx.mem_info()[0] < (20 << 30):
        pytest.skip("needs ~20 GB of free device memory")
    ctx.mem_peak()  # restarts the peak mark
    C = lib.DeviceCSR.generate(ctx, *C4)
    try:
        peak = ctx.mem_peak()[1]
        print(f"C4 generation: pool peak {peak / 2**30:.2f} GiB (the key arrays and CUB temporaries are cudaMalloc "
              f"blocks outside the pool)")
        m = C.download()
        assert C.shape3 == (C4[0], C4[1], m.nnz)
    finally:
        C.close()
    return m.indptr, m.indices, m.data, digest(m.indptr, m.indices, m.data)


def test_c4_invariants(c4):
    users, items, target, _ = C4
    indptr, indices, data, _ = c4
    nnz = len(indices)
    assert len(indptr) == users + 1 and indptr[0] == 0 and indptr[-1] == nnz
    assert (np.diff(indptr) >= 0).all()
    assert indices.min() >= 0 and indices.max() < items
    starts = np.zeros(nnz, dtype=bool)  # entries that open a row: no predecessor in the row to compare with
    starts[indptr[:-1][indptr[:-1] < nnz]] = True
    for a in range(1, nnz, 1 << 26):
        b = min(nnz, a + (1 << 26))
        assert ((indices[a:b] > indices[a - 1:b - 1]) | starts[a:b]).all(), "columns must strictly increase in a row"
    assert data.min() >= 1 and data.max() <= 5
    print(f"C4: nnz {nnz}, {int((data == 5).sum())} values of 5.0 (3 keys in 2^25 expected: {nnz * 3 / 2**25:.1f})")
    assert abs(nnz - target) <= 6 * np.sqrt(target), "the thinning keeps a binomial share of the unique keys"


def find(indptr, indices, keys, items):
    """Position of every key (row * items + column) in the CSR, or -1: a binary search within each key's row."""
    rows, cols = (keys // np.uint64(items)).astype(np.int64), (keys % np.uint64(items)).astype(np.int32)
    lo, end = indptr[rows].astype(np.int64), indptr[rows + 1].astype(np.int64)
    hi = end.copy()
    last = len(indices) - 1
    while (lo < hi).any():
        mid = (lo + hi) // 2
        right = (lo < hi) & (indices[np.minimum(mid, last)] < cols)
        hi = np.where((lo < hi) & ~right, mid, hi)
        lo = np.where(right, mid + 1, lo)
    hit = (lo < end) & (indices[np.minimum(lo, last)] == cols)
    return np.where(hit, lo, -1)


def test_c4_sampled_draws(c4):
    """200k draws restated: the keys they make are in the output exactly when their thinning hash lies below one
    threshold, the share kept agrees with that threshold, and every kept key holds its restated value."""
    users, items, target, seed = C4
    indptr, indices, data, _ = c4
    m = target + target // 4
    t = np.unique(np.random.default_rng(0).integers(0, m, 200_000)).astype(np.uint64)
    keys, flagged = gr.draws(users, items, seed, t, gr.permutation(users, seed, 1), gr.permutation(items, seed, 2))
    assert flagged.sum() <= 2, "the flagging bound should leave nearly every draw unambiguous"
    keys = np.unique(keys[~flagged])
    pos = find(indptr, indices, keys, items)
    present = pos >= 0
    h = gr.hash3(seed, 13, keys)
    assert present.any() and not present.all(), "C4 draws more unique keys than its target: the thinning runs"
    below, above = int(h[present].max()), int(h[~present].min())
    assert below < above, "kept and dropped keys must be separated by one threshold on hash3(seed, 13, key)"
    p = (below + above) / 2 / 2.0**64
    n = len(keys)
    share = present.mean()
    print(f"C4 sample: {n} distinct keys, {share:.5f} kept, threshold / 2^64 = {p:.5f}, {int(flagged.sum())} flagged")
    assert abs(share - p) <= 6 * np.sqrt(p * (1 - p) / n)
    np.testing.assert_array_equal(bits(data[pos[present]]), bits(gr.values(seed, keys[present])))


def test_c4_is_the_same_on_a_second_run(lib, ctx, c4):
    _, ip, ix, d = generated(lib, ctx, *C4)
    assert digest(ip, ix, d) == c4[3]


def test_c4_is_the_same_on_a_second_device(lib, c4):
    if lib.device_count() < 2:
        pytest.skip("needs a second GPU")
    other = lib.Context(1)
    try:
        if other.mem_info()[0] < (20 << 30):
            pytest.skip("needs ~20 GB of free device memory on device 1")
        _, ip, ix, d = generated(lib, other, *C4)
        assert digest(ip, ix, d) == c4[3]
    finally:
        other.close()


# ------------------------------------------------------------------------------------------------ fill_uniform
FILL_WIDTHS = [1, 15, 16, 17, 63, 64, 100, 128, 129, 200, 1024]  # every ld class: 16, 32, 64, 112, 128, 256, 1024


@pytest.mark.parametrize("scale", [0.01, 1.0])
@pytest.mark.parametrize("f", FILL_WIDTHS)
def test_fill_uniform_is_restated(lib, ctx, f, scale):
    seed = (gr.GOLDEN * f) & gr.M64  # seeds across the whole 64-bit range
    for rows in (0, 1, 3, 2053):
        d = lib.DeviceFactors(ctx, rows, f)
        try:
            if rows:
                helpers.padded_view(d).fill_(float("nan"))  # the padding must be written, not left as it was
                torch.cuda.synchronize()
            d.fill_uniform(seed, scale)
            if rows:
                full = helpers.padded(d)
                np.testing.assert_array_equal(bits(full[:, :f]), bits(gr.fill_uniform(f, seed, scale, 0, rows)))
                assert (bits(full[:, f:]) == 0).all(), "padding columns must be +0.0"
        finally:
            d.close()


def test_fill_uniform_past_2_31_elements(lib, ctx):
    """2^25 + 4099 rows of 64 factors: element and hash indices past 2^31."""
    f, seed, scale = 64, 5, 0.01
    rows = (1 << 25) + 4099
    if ctx.mem_info()[0] < rows * f * 4 + (2 << 30):
        pytest.skip("needs ~11 GB of free device memory")
    d = lib.DeviceFactors(ctx, rows, f)
    try:
        d.fill_uniform(seed, scale)
        cross = (1 << 31) // f  # the first row at element 2^31
        for r0, n in ((0, 3), (cross - 2, 4), (rows - 4099, 4099)):
            np.testing.assert_array_equal(bits(d.download(r0, n)), bits(gr.fill_uniform(f, seed, scale, r0, n)))
    finally:
        d.close()
