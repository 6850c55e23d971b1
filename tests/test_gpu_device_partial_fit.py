"""partial_fit_users / partial_fit_items with their ids in CUDA memory: the rows are refitted, and the factor matrix
grown, in place on the device, with bitwise the factors of the same call with numpy ids.  PyTorch plays the producer;
the package itself never imports it.

The numpy call stores into the read-only view the factor getters hand out, so today it only succeeds when it grows the
matrix.  For a call without new ids the stand-in is the numpy call's own lines on a writable copy: recalculate_* with
the same ids, then factors[ids] = rows.
"""
import os

import numpy as np
import pytest
import scipy.sparse as sp

from helpers import KNOB_DEFAULTS

torch = pytest.importorskip("torch")

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs PyTorch with CUDA as the producer")]


@pytest.fixture(scope="module")
def ctx():
    names = [f"ALS_B200_{k.upper()}" for k in list(KNOB_DEFAULTS) + ["segment_nnz", "host_csr"]]
    set_in_env = sorted(n for n in names if n in os.environ)
    if set_in_env:
        pytest.fail(f"knob environment variables are set: {', '.join(set_in_env)}; unset them to run these tests")
    from implicit_b200 import _lib

    c = _lib.Context(0)
    yield c
    c.close()


USERS, ITEMS = 700, 600


def pair(ctx, f, seed=0):
    """(host, dev): two models of the same factors, the first assigned from numpy, the second from CUDA tensors."""
    from implicit_b200 import AlternatingLeastSquares

    rng = np.random.default_rng(seed + f)
    X = rng.standard_normal((USERS, f), dtype=np.float32)
    Y = rng.standard_normal((ITEMS, f), dtype=np.float32)
    models = []
    for factors in ((X, Y), (torch.from_numpy(X).cuda(), torch.from_numpy(Y).cuda())):
        m = AlternatingLeastSquares(factors=f, iterations=1, regularization=0.1, random_state=1)
        m._ctx = ctx
        m.user_factors, m.item_factors = factors
        models.append(m)
    return models


def interactions(n, cols, seed):
    """n rows of distinct sorted columns and positive confidences; every fifth row is empty."""
    rng = np.random.default_rng(seed)
    counts = rng.integers(1, 25, n)
    counts[::5] = 0
    indices = np.concatenate([np.sort(rng.choice(cols, c, replace=False)) for c in counts]).astype(np.int32)
    indptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    data = rng.uniform(0.5, 4.0, len(indices)).astype(np.float32)
    return sp.csr_matrix((data, indices, indptr), shape=(n, cols))


def device_csr(M, index_dtype=np.int64):
    ip, ix, v = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in
                 (M.indptr.astype(index_dtype), M.indices.astype(index_dtype), M.data))
    return torch.sparse_csr_tensor(ip, ix, v, size=M.shape)


def cu(a, dtype=np.int64):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=dtype))).cuda()


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def factors_of(m, side):
    return m.user_factors if side == "user" else m.item_factors


def partial_fit(m, side, ids, rows):
    (m.partial_fit_users if side == "user" else m.partial_fit_items)(ids, rows)


def host_partial_fit(m, side, ids, rows):
    """The numpy call; without new ids its lines on a writable copy (see the module docstring)."""
    if ids.max() >= factors_of(m, side).shape[0]:
        return partial_fit(m, side, ids, rows)
    want = np.array(factors_of(m, side))
    want[ids] = (m.recalculate_user if side == "user" else m.recalculate_item)(ids, rows)
    if side == "user":
        m.user_factors = want
    else:
        m.item_factors = want


def id_cases(n, rng):
    """(name, ids): growth by 0 rows, by 1 row and far past the end (a gap of new ids no call names), each with
    repeated ids"""
    old = rng.choice(n, 40, replace=False)
    return [("grow 0", np.concatenate([old, old[:5], old[7:9]])),
            ("grow 1", np.concatenate([old[:30], [n], old[2:6], [n]])),
            ("grow far", np.concatenate([old[:20], [n + 50, n + 7, n + 50], old[:4], [n + 7]]))]


# ---- bitwise against the numpy call -------------------------------------------------------------------------------
@pytest.mark.parametrize("side", ["user", "item"])
@pytest.mark.parametrize("f", [16, 64, 128, 192, 1024])
def test_partial_fit_matches_host(ctx, f, side):
    """Every solver family, int32 and int64 ids, a scipy and a CUDA CSR, growth by 0, 1 and far, repeats in both
    orders: after every call the factors are bitwise the numpy call's.  Then the serving calls with CUDA ids read the
    refitted factors, norms and Gramians: bitwise the host model's."""
    ref, dev = pair(ctx, f)
    rng = np.random.default_rng(f + (side == "item"))
    # fill every cache the refit must drop: device norms of both sides and both Gramians
    dev.similar_items(cu(np.arange(5)), N=3)
    dev.similar_users(cu(np.arange(5)), N=3)
    assert dev.XtX is not None and dev.YtY is not None
    step = 0
    for dtype in (np.int32, np.int64):
        for kind in ("scipy", "cuda"):
            for order in (1, -1):
                for name, ids in id_cases(factors_of(ref, side).shape[0], rng):
                    ids = ids[::order]
                    rows = interactions(len(ids), factors_of(ref, "item" if side == "user" else "user").shape[0],
                                        seed=step)
                    step += 1
                    host_partial_fit(ref, side, ids.astype(dtype), rows)
                    partial_fit(dev, side, cu(ids, dtype), rows if kind == "scipy" else device_csr(rows))
                    assert not dev._host_fresh[side]
                    want, got = factors_of(ref, side), factors_of(dev, side)
                    assert got.shape == want.shape, (name, order, dtype, kind)
                    assert np.array_equal(bits(got), bits(want)), (name, order, dtype, kind)
    # the last call grew n rows to n + 51 and named n + 7 and n + 50 (n itself came from "grow 1"): the rest is zero
    N = factors_of(dev, side).shape[0]
    gap = np.setdiff1d(np.arange(N - 50, N - 1), [N - 51 + 7])
    assert len(gap) == 48 and not factors_of(dev, side)[gap].any()

    users = np.arange(0, dev.user_factors.shape[0], 7)
    items = np.arange(0, dev.item_factors.shape[0], 5)
    L = interactions(len(users), dev.item_factors.shape[0], seed=99)
    M = interactions(len(items), dev.user_factors.shape[0], seed=98)
    same(dev.recommend(cu(users), L, N=10), ref.recommend(users, L, N=10))
    same(dev.recommend(cu(users), L, N=10, recalculate_user=True), ref.recommend(users, L, N=10, recalculate_user=True))
    same(dev.similar_items(cu(items), N=10), ref.similar_items(items, N=10))
    same(dev.similar_users(cu(users), N=10), ref.similar_users(users, N=10))
    same(dev.similar_items(cu(items), N=10, recalculate_item=True, item_users=M),
         ref.similar_items(items, N=10, recalculate_item=True, item_users=M))


def host(x):
    return torch.as_tensor(x, device="cuda").cpu().numpy()


def same(got, want):
    gi, gs = host(got[0]), host(got[1])
    assert np.array_equal(gi, want[0]) and np.array_equal(bits(gs), bits(want[1]))


def test_last_occurrence_wins(ctx):
    """A repeated id takes the row of its last occurrence, in either order; rows no id names keep their bits, and the
    rows the growth adds are zero."""
    _, dev = pair(ctx, 64)
    ids = np.array([9, 4, 9, 9, 4, USERS + 60, 4, USERS + 60], dtype=np.int64)
    rows = interactions(len(ids), ITEMS, seed=3)
    for order in (1, -1):
        solved = dev.recalculate_user(ids[::order], rows[::order])
        before = np.array(dev.user_factors)
        dev.partial_fit_users(cu(ids[::order]), rows[::order])
        got = dev.user_factors
        assert got.shape == (USERS + 61, 64)
        for i, u in enumerate(ids[::order]):
            if u not in ids[::order][i + 1:]:
                assert np.array_equal(bits(got[u]), bits(solved[i]))
        untouched = np.setdiff1d(np.arange(before.shape[0]), ids)
        assert np.array_equal(bits(got[untouched]), bits(before[untouched]))
        assert not got[USERS:USERS + 60].any()


# ---- nothing crosses PCIe ---------------------------------------------------------------------------------------
def test_no_factor_matrix_crosses_pcie(ctx, monkeypatch):
    from implicit_b200 import _lib

    ref, dev = pair(ctx, 64, seed=4)
    moved = []
    real_down, real_up = _lib.DeviceFactors.download, _lib.DeviceFactors.upload

    def download(self, row0=0, nrows=None, pinned=False):
        moved.append(("download", self.rows - row0 if nrows is None else nrows))
        return real_down(self, row0, nrows, pinned)

    def upload(self, a, row0=0):
        moved.append(("upload", np.asarray(a).shape[0]))
        return real_up(self, a, row0)

    monkeypatch.setattr(_lib.DeviceFactors, "download", download)
    monkeypatch.setattr(_lib.DeviceFactors, "upload", upload)
    uids = np.concatenate([np.arange(100, 190), np.arange(USERS, USERS + 10)])
    iids = np.concatenate([np.arange(0, 45), np.arange(ITEMS + 3, ITEMS + 8)])
    R, S = interactions(len(uids), ITEMS, seed=5), interactions(len(iids), USERS + 10, seed=6)
    dev.partial_fit_users(cu(uids), R)
    dev.partial_fit_items(cu(iids), device_csr(S))
    got = [dev.recommend(cu(uids), None, N=10, filter_already_liked_items=False), dev.similar_items(cu(iids), N=10)]
    assert moved == [] and not dev._host_fresh["user"] and not dev._host_fresh["item"]
    monkeypatch.undo()
    ref.partial_fit_users(uids, R)
    ref.partial_fit_items(iids, S)
    assert np.array_equal(bits(dev.user_factors), bits(ref.user_factors))
    assert np.array_equal(bits(dev.item_factors), bits(ref.item_factors))
    same(got[0], ref.recommend(uids, None, N=10, filter_already_liked_items=False))
    same(got[1], ref.similar_items(iids, N=10))


# ---- refusals and the empty call ----------------------------------------------------------------------------------
@pytest.mark.parametrize("side", ["user", "item"])
def test_refusals_leave_the_factors_unchanged(ctx, side):
    ref, dev = pair(ctx, 64, seed=7)
    what = f"{side}ids"
    cols = ITEMS if side == "user" else USERS
    rows = interactions(3, cols, seed=7)
    before = bits(host(dev.user_factors_device if side == "user" else dev.item_factors_device))
    norms = dev._device_norms(side)
    cases = [
        # max ids whose rows could never be allocated, among them byte counts that overflow int64 (2^57 - 1 rows of
        # 256 bytes wrap to 0), refused after the solve and before anything is written
        (cu([3, 2**57 - 1, 5]), rows, "als_factors_grow: .* more than the device's"),
        (cu([2**40, 3, 5]), rows, "als_factors_grow: .* more than the device's"),
        (cu([2**31 - 1, 3, 5], np.int32), rows, "als_factors_grow: .* more than the device's"),
        (cu([3, 2**63 - 1, 5]), device_csr(rows), "als_factors_grow: .* more than the device's"),
        (cu([3, -1, 5]), rows, f"{what} holds a negative id"),
        (cu([USERS + ITEMS, -2, 1]), rows, f"{what} holds a negative id"),
        (cu([3, 4, 5], np.int16), rows, f"{what}: typestr '<i2'"),
        (torch.tensor([3.0, 4.0, 5.0], device="cuda"), rows, f"{what}: typestr '<f4'"),
        (cu([[3, 4, 5]]), rows[:1], f"{what}: shape \\(1, 3\\) is not a 1-D shape"),
        (cu([3, 4]), rows, "must contain 1 row for every user in"),
        (cu([3, 4, 5, 6]), device_csr(rows), "must contain 1 row for every user in"),
    ]
    for ids, m, message in cases:
        with pytest.raises(ValueError, match=message):
            partial_fit(dev, side, ids, m)
        after = host(dev.user_factors_device if side == "user" else dev.item_factors_device)
        assert np.array_equal(bits(after), before), message
    assert dev._dev_norms[side] is norms  # no refusal marked the side updated
    # a host copy that is current stays current
    host_before = bits(np.array(factors_of(ref, side)))
    with pytest.raises(ValueError, match="als_factors_grow"):
        partial_fit(ref, side, cu([3, 2**57 - 1, 5]), rows)
    assert ref._host_fresh[side] and np.array_equal(bits(factors_of(ref, side)), host_before)


def outcome(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001 -- the type is what is compared
        return type(e)
    return None


@pytest.mark.parametrize("side", ["user", "item"])
def test_empty_ids_do_what_the_numpy_call_does(ctx, side):
    ref, dev = pair(ctx, 32, seed=8)
    cols = ITEMS if side == "user" else USERS
    empty = sp.csr_matrix((0, cols), dtype=np.float32)
    before = [bits(np.array(factors_of(m, side))) for m in (ref, dev)]
    for rows in (empty, device_csr(empty)):
        want = outcome(lambda: partial_fit(ref, side, np.array([], dtype=np.int64), rows))
        for dtype in (np.int32, np.int64):
            assert outcome(lambda: partial_fit(dev, side, cu([], dtype), rows)) is want
    if want is not None:  # then nothing was written on either path
        for m, b in zip((ref, dev), before):
            assert np.array_equal(bits(factors_of(m, side)), b)
    else:
        assert np.array_equal(bits(factors_of(dev, side)), bits(factors_of(ref, side)))
