"""fit() draws its initial factors on the device, bit for bit numpy's default_rng draw: DeviceFactors.fill_pcg64 against
Generator.random((rows, f), dtype=np.float32) * np.float32(0.01) at every width class, with and without a buffered half,
past 2^32 values of the stream; fit(iterations=0) for every random_state kind, the generator's state afterwards, whole
fits against the same fit from pre-set numpy factors, failing fits and allocation failures against the host draw (a
PCG64 subclass keeps fit on the host path, on the same stream).  PyTorch plays the producer of the CUDA inputs."""
import copy
import gc

import numpy as np
import pytest
import scipy.sparse as sp

import helpers

torch = pytest.importorskip("torch")

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs PyTorch with CUDA as the producer")]

WIDTHS = [1, 2, 15, 16, 17, 63, 64, 65, 127, 128, 129, 200, 256, 1000, 1024]
SCALE = np.float32(0.01)


class HostPCG64(np.random.PCG64):
    """PCG64's stream, but not of type PCG64: fit() draws it on the host, as the parent code did for every generator."""


@pytest.fixture(scope="module")
def ctx():
    from implicit_b200 import _lib

    c = _lib.Context(0)
    yield c
    c.close()


def buffered(seed):
    g = np.random.default_rng(seed)
    g.random(1, dtype=np.float32)
    return g


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize("has", [0, 1])
@pytest.mark.parametrize("f", WIDTHS)
def test_fill_is_numpys_draw(ctx, f, has):
    from implicit_b200 import _lib, pcg64

    for rows in (0, 1, 2, 3, 100003):
        g = buffered(f) if has else np.random.default_rng(f)
        st = pcg64.get_state(g)
        d = _lib.DeviceFactors(ctx, rows, f)
        try:
            d.fill_pcg64(st, SCALE)
            want = g.random((rows, f), dtype=np.float32) * SCALE
            if rows:
                full = helpers.padded(d)
                assert np.array_equal(bits(full[:, :f]), bits(want)), (rows, f, has)
                assert not full[:, f:].any(), "padding columns must stay zero"
                assert np.array_equal(bits(d.download()), bits(want))
            assert pcg64.get_state(g) == pcg64.after_float32_draws(st, rows * f)
        finally:
            d.close()


def test_fill_past_2_32_values(ctx):
    """2^26 rows x 65 factors: 4.4e9 values, so stream positions and jumps need 64 bits."""
    from implicit_b200 import _lib, pcg64

    rows, f = 1 << 26, 65
    free = ctx.mem_info()[0]
    if free < rows * 80 * 4 + (2 << 30):
        pytest.skip("needs ~22 GB of free device memory")
    g = buffered(77)
    st = pcg64.get_state(g)
    d = _lib.DeviceFactors(ctx, rows, f)
    try:
        d.fill_pcg64(st, SCALE)
        cross = (1 << 32) // f  # the row holding value 2^32
        sample = sorted({0, 1, rows - 1, rows - 2, cross - 1, cross, cross + 1, (1 << 31) // f, ((1 << 33) // 2) // f}
                        | set(np.random.default_rng(0).integers(0, rows, 24).tolist()))
        for r in sample:
            at = pcg64.generator_at(pcg64.after_float32_draws(st, r * f))
            want = at.random(f, dtype=np.float32) * SCALE
            assert np.array_equal(bits(d.download(r, 1)[0]), bits(want)), r
    finally:
        d.close()


def csr(users, items, nnz, seed):
    rng = np.random.default_rng(seed)
    m = sp.random(users, items, density=nnz / (users * items), format="csr", random_state=rng, dtype=np.float32)
    m.data = (1.0 + 4.0 * m.data).astype(np.float32)
    m.sort_indices()
    return m


def torch_csr(m):
    return torch.sparse_csr_tensor(torch.from_numpy(m.indptr.astype(np.int64)), torch.from_numpy(m.indices.astype(np.int64)),
                                   torch.from_numpy(m.data), size=m.shape).cuda()


KINDS = ["int", "seedsequence", "randomstate", "generator", "buffered", "bitgen", "philox"]


def random_state(kind):
    return {"int": 42, "seedsequence": np.random.SeedSequence(42), "randomstate": np.random.RandomState(42),
            "generator": np.random.default_rng(42), "buffered": buffered(42), "bitgen": np.random.PCG64(42),
            "philox": np.random.Generator(np.random.Philox(42))}[kind]


def host_draws(rs, users, items, f, user_preset=False):
    """What the parent code drew: (user, item, the generator afterwards) from a copy of rs."""
    from implicit_b200.utils import check_random_state

    g = check_random_state(copy.deepcopy(rs))
    X = None if user_preset else g.random((users, f), dtype=np.float32) * SCALE
    Y = g.random((items, f), dtype=np.float32) * SCALE
    return X, Y, g


@pytest.mark.parametrize("source", ["scipy", "torch"])
@pytest.mark.parametrize("kind", KINDS)
def test_fit_zero_iterations_is_numpys_draw(kind, source):
    from implicit_b200 import AlternatingLeastSquares

    users, items, f = 301, 257, 33
    C = csr(users, items, 3000, 1)
    rs = random_state(kind)
    X, Y, g = host_draws(rs, users, items, f)
    m = AlternatingLeastSquares(factors=f, iterations=0, random_state=rs)
    m.fit(torch_csr(C) if source == "torch" else C, show_progress=False)
    if kind != "philox":
        assert m._user_factors is None and m._item_factors is None, "the device draw keeps no host copy"
    assert np.array_equal(bits(m.user_factors), bits(X))
    assert np.array_equal(bits(m.item_factors), bits(Y))
    if isinstance(rs, np.random.Generator):
        np.testing.assert_equal(rs.bit_generator.state, g.bit_generator.state)  # Philox's state holds arrays
    if isinstance(rs, np.random.PCG64):
        assert rs.state == g.bit_generator.state
    if isinstance(rs, np.random.RandomState):
        fresh = np.random.RandomState(42)
        fresh.randint(2**31)  # the seed check_random_state took
        assert rs.randint(2**31) == fresh.randint(2**31)


@pytest.mark.parametrize("kind", ["generator", "buffered"])
def test_fit_with_user_side_preset(kind):
    from implicit_b200 import AlternatingLeastSquares

    users, items, f = 120, 90, 16
    C = csr(users, items, 900, 2)
    rs = random_state(kind)
    _, Y, g = host_draws(rs, users, items, f, user_preset=True)
    X0 = np.random.default_rng(5).standard_normal((users, f)).astype(np.float32)
    m = AlternatingLeastSquares(factors=f, iterations=0, random_state=rs)
    m.user_factors = X0
    m.fit(C, show_progress=False)
    assert np.array_equal(bits(m.user_factors), bits(X0))
    assert np.array_equal(bits(m.item_factors), bits(Y))
    assert rs.bit_generator.state == g.bit_generator.state


@pytest.mark.parametrize("f,use_cg", [(64, False), (64, True), (200, True)])
def test_whole_fit_matches_preset_numpy_factors(f, use_cg):
    from implicit_b200 import AlternatingLeastSquares

    users, items = 1500, 1100
    C = csr(users, items, 30000, 3)
    X, Y, _ = host_draws(7, users, items, f)
    a = AlternatingLeastSquares(factors=f, iterations=3, use_cg=use_cg, regularization=0.05, random_state=7)
    a.fit(torch_csr(C), show_progress=False)
    b = AlternatingLeastSquares(factors=f, iterations=3, use_cg=use_cg, regularization=0.05)
    b.user_factors, b.item_factors = X, Y
    b.fit(torch_csr(C), show_progress=False)
    assert np.array_equal(bits(a.user_factors), bits(b.user_factors))
    assert np.array_equal(bits(a.item_factors), bits(b.item_factors))


@pytest.mark.parametrize("bitgen", [np.random.PCG64, HostPCG64])
def test_failing_fit_leaves_the_initial_draw(bitgen):
    """A row that is not positive definite stops the fit; the getters return the initial draw and the generator is where
    the draws left it, on the device path as on the host path."""
    from implicit_b200 import AlternatingLeastSquares

    f = 16
    C = helpers.bad_row_csr(f, {7})
    users, items = C.shape
    g = np.random.Generator(bitgen(3))
    want = np.random.default_rng(3)
    X = want.random((users, f), dtype=np.float32) * SCALE
    Y = want.random((items, f), dtype=np.float32) * SCALE
    m = AlternatingLeastSquares(factors=f, iterations=2, use_cg=False, regularization=0.0, random_state=g)
    with pytest.raises(ValueError, match="cholesky failed"):
        m.fit(C, show_progress=False)
    assert np.array_equal(bits(m.user_factors), bits(X))
    assert np.array_equal(bits(m.item_factors), bits(Y))
    assert g.bit_generator.state["state"] == want.bit_generator.state["state"]
    assert (g.bit_generator.state["has_uint32"], g.bit_generator.state["uinteger"]) == \
        (want.bit_generator.state["has_uint32"], want.bit_generator.state["uinteger"])


def test_allocation_failures_match_the_host_path(ctx):
    """Every allocation of a fit with unset factors fails in turn: nothing leaks, and the model and its generator end
    as the host draw leaves them for the same failure."""
    from implicit_b200 import AlternatingLeastSquares, _lib

    C = csr(400, 300, 6000, 4)
    f = 32

    def used():
        gc.collect()
        torch.cuda.synchronize()
        ctx.sync()
        return ctx.mem_peak()[0]

    def run(bitgen, n):
        g = np.random.Generator(bitgen(9))
        m = AlternatingLeastSquares(factors=f, iterations=1, regularization=0.1, random_state=g)
        m._ctx = ctx
        ctx.set_knob("alloc_fail_at", n)
        err = None
        try:
            m.fit(C, show_progress=False)
        except (_lib.AlsError, ValueError, RuntimeError, MemoryError) as e:
            err = type(e)
        ctx.set_knob("alloc_fail_at", 0)
        out = [m._factors_shape(s) and m._get_host(s) for s in ("user", "item")]
        state = g.bit_generator.state
        del m
        return err, out, {k: v for k, v in state.items() if k != "bit_generator"}

    base = used()
    n = 1
    while True:
        err, out, state = run(np.random.PCG64, n)
        assert used() == base, f"allocation {n} failed and left {used() - base} bytes of the pool in use"
        herr, hout, hstate = run(HostPCG64, n)
        assert err == herr and state == hstate, n
        for a, b in zip(out, hout):
            assert (a is None) == (b is None) and (a is None or np.array_equal(bits(a), bits(b))), n
        if err is None:
            break
        n += 1
    assert n > 2


def test_other_bit_generators_draw_on_the_host():
    from implicit_b200 import AlternatingLeastSquares

    users, items, f = 50, 40, 8
    C = csr(users, items, 400, 5)
    g = np.random.Generator(np.random.Philox(11))
    want = np.random.Generator(np.random.Philox(11))
    X = want.random((users, f), dtype=np.float32) * SCALE
    Y = want.random((items, f), dtype=np.float32) * SCALE
    m = AlternatingLeastSquares(factors=f, iterations=0, random_state=g)
    m.fit(C, show_progress=False)
    assert np.array_equal(bits(m.user_factors), bits(X)) and np.array_equal(bits(m.item_factors), bits(Y))
    np.testing.assert_equal(g.bit_generator.state, want.bit_generator.state)
