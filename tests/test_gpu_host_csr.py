"""Host-resident CSRs (indices / values in page-locked host memory, streamed through the device per segment): every
call must give bitwise what the device-resident CSR of the same segment cap gives.

Small cases force the cap with the segment_nnz knob on mixed_csr data (duplicates, empty rows, giant rows, negative
confidences, stored zeros), like test_gpu_csr64.py, and compare each host-resident call with the device-resident one.
"""
import ctypes
import os

import numpy as np
import pytest
import scipy.sparse as sp

from helpers import KNOB_DEFAULTS, check_bad_row_in_second_segment, factors_of, mixed_csr

pytestmark = pytest.mark.gpu
REG = 0.05
KNOBS = dict(KNOB_DEFAULTS, segment_nnz=0, host_csr=0)


@pytest.fixture(scope="module")
def lib():
    set_in_env = sorted(n for n in (f"ALS_B200_{k.upper()}" for k in KNOBS) if n in os.environ)
    if set_in_env:  # the device-resident runs would silently be host-resident or segmented too
        pytest.fail(f"knob environment variables are set: {', '.join(set_in_env)}; unset them to run these tests")
    from implicit_b200 import _lib

    return _lib


@pytest.fixture(scope="module")
def ctx(lib):
    c = lib.Context(0)
    yield c
    c.close()


@pytest.fixture(autouse=True)
def knobs(ctx):
    for k, v in KNOBS.items():
        ctx.set_knob(k, v)
    yield
    for k, v in KNOBS.items():
        ctx.set_knob(k, v)


@pytest.fixture(scope="module")
def C():
    return mixed_csr(600, 500, 7, duplicates=True)


def caps_of(C):
    """The forced caps of test_gpu_csr64.py, and 0: the default cap (one segment here, for either residency)."""
    lens = np.diff(C.indptr)
    return {"default": 0, "below_longest": int(lens.max()) - 100, "giant_length": int(lens[50]),
            "after_giant": int(C.indptr[51]), "thirds": C.nnz // 3 + 1}


CAPS = ["default", "below_longest", "giant_length", "after_giant", "thirds"]


def upload(lib, ctx, C, cap, host):
    ctx.set_knob("segment_nnz", cap)
    d = lib.DeviceCSR.upload(ctx, C, host=host)
    assert d.host_resident == host
    assert (d.segment_count > 1) == (cap > 0)
    return d


def both(fn):
    """fn(host) for the device-resident and the host-resident CSR."""
    return fn(False), fn(True)


def close(*hs):
    for h in hs:
        h.close()


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("index_dtype", [np.int32, np.int64])
def test_upload_download(lib, ctx, C, cap, index_dtype):
    Ci = sp.csr_matrix((C.data, C.indices.astype(index_dtype), C.indptr.astype(np.int64)), shape=C.shape)
    d = upload(lib, ctx, Ci, caps_of(C)[cap], True)
    back = d.download()
    assert np.array_equal(back.indptr, C.indptr) and np.array_equal(back.indices, C.indices)
    assert np.array_equal(back.data, C.data)
    d.close()


def test_upload_refusals_match_device(lib, ctx, C):
    def up(fn, indptr, indices, nnz):
        h = ctypes.c_void_p()
        rc = fn(ctx.h, C.shape[0], C.shape[1], nnz, lib.ptr(indptr), lib.ptr(indices), indices.dtype.itemsize,
                lib.ptr(C.data), 0, ctypes.byref(h))
        msg = ctx.lib.als_last_error().decode()
        if rc == 0:
            lib.DeviceCSR(ctx, h).close()
        return rc, msg

    indptr, indices = C.indptr.astype(np.int64), C.indices.astype(np.int64)
    cases = []
    for pos, v in ((17, -1), (C.nnz - 1, C.shape[1])):
        bad = indices.copy()
        bad[pos] = v
        cases.append((indptr, bad, C.nnz))
    nm = indptr.copy()
    nm[100] = nm[101] + 1
    cases += [(nm, indices, C.nnz), (indptr, indices, C.nnz - 1)]
    for ip, ix, n in cases:
        rc_dev, msg_dev = up(ctx.lib.als_csr_upload64, ip, ix, n)
        rc_host, msg_host = up(ctx.lib.als_csr_upload_host64, ip, ix, n)
        assert rc_dev == rc_host == lib.ALS_E_INVALID
        assert msg_host == msg_dev.replace("als_csr_upload64", "als_csr_upload_host64")


@pytest.mark.parametrize("cap", ["one_window", "windows"])
def test_transpose_equals_scipy(lib, ctx, C, cap):
    """A column window holds at most 16 segment caps of output nonzeros (csr.cu kWindowSegments): a cap of nnz / 64
    gives at least 4 windows (no column of C holds more than a window); the default cap gives one."""
    want = C.T.tocsr()
    c = 0 if cap == "one_window" else C.nnz // 64
    assert np.diff(want.indptr).max() <= 16 * c or c == 0
    ts = []
    for host in (False, True):
        d = upload(lib, ctx, C, c, host)
        t = d.transpose()
        assert t.host_resident == host
        got = t.download()
        assert np.array_equal(got.indptr, want.indptr)
        assert np.array_equal(got.indices, want.indices)
        assert np.array_equal(got.data, want.data)
        ts.append(t.segment_count)
        close(t, d)
    assert ts[0] == ts[1]


def cholesky_half(lib, ctx, C, Y, cap, host, YtY=None):
    d = upload(lib, ctx, C, cap, host)
    Yd = lib.DeviceFactors.from_host(ctx, Y)
    X = lib.DeviceFactors(ctx, C.shape[0], Y.shape[1])
    if YtY is None:
        lib.least_squares(ctx, d, X, Yd, REG)
    else:
        lib.least_squares_with_gramian(ctx, YtY, d, X, Yd, REG)
    t = d.transpose()  # the item half over the transpose, host-resident like its input
    assert t.host_resident == host
    Y2 = lib.DeviceFactors(ctx, C.shape[1], Y.shape[1])
    lib.least_squares(ctx, t, Y2, X, REG)
    out = X.download(), Y2.download()
    close(t, d, Yd, X, Y2)
    return out


@pytest.mark.parametrize("f", [16, 48, 64, 100, 200])
@pytest.mark.parametrize("kind", ["cold", "mixed"])
def test_cholesky_half_bitwise(lib, ctx, C, f, kind):
    Y = factors_of(kind, C.shape[1], f, 11)
    for cap in CAPS:
        dev, host = both(lambda h: cholesky_half(lib, ctx, C, Y, caps_of(C)[cap], h))
        assert np.array_equal(host[0], dev[0]), (cap, "user half")
        assert np.array_equal(host[1], dev[1]), (cap, "item half")
    YtY = (Y.astype(np.float64).T @ Y).astype(np.float32)
    dev, host = both(lambda h: cholesky_half(lib, ctx, C, Y, caps_of(C)["thirds"], h, YtY))
    assert np.array_equal(host[0], dev[0]) and np.array_equal(host[1], dev[1])


@pytest.mark.parametrize("variant", ["long_tc", "short_max0"])
def test_cholesky_variants_bitwise(lib, ctx, C, variant):
    """The wgmma long-row kernel (64 padded factors, no weight below zero: positive confidences of at least 1) and
    the full-size kernel alone (no short-row path)."""
    Cv = C
    if variant == "long_tc":
        ctx.set_knob("long_tc", 1)
        Cv = abs(C)
        Cv.data += np.float32(1)
    else:
        ctx.set_knob("short_max", 0)
    Y = factors_of("mixed", C.shape[1], 64, 12)
    for cap in CAPS:
        dev, host = both(lambda h: cholesky_half(lib, ctx, Cv, Y, caps_of(C)[cap], h))
        assert np.array_equal(host[0], dev[0]) and np.array_equal(host[1], dev[1]), cap


@pytest.mark.parametrize("f", [64, 200])
def test_cg_half_bitwise(lib, ctx, C, f):
    Y = factors_of("mixed", C.shape[1], f, 3)
    X0 = factors_of("mixed", C.shape[0], f, 4)

    def run(cap, host):
        d = upload(lib, ctx, C, cap, host)
        Yd, X = lib.DeviceFactors.from_host(ctx, Y), lib.DeviceFactors.from_host(ctx, X0)
        lib.least_squares_cg(ctx, d, X, Yd, REG, 3)
        out = X.download()
        close(d, Yd, X)
        return out

    for cap in CAPS:
        dev, host = both(lambda h: run(caps_of(C)[cap], h))
        assert np.array_equal(host, dev), cap


def test_loss_and_scale(lib, ctx, C):
    Y = factors_of("mixed", C.shape[1], 64, 5)
    X = factors_of("mixed", C.shape[0], 64, 6)
    Yd, Xd = lib.DeviceFactors.from_host(ctx, Y), lib.DeviceFactors.from_host(ctx, X)
    for cap in CAPS:
        c = caps_of(C)[cap]
        # the loss sums per-segment terms in fp64 atomics: equal up to their order
        dev, host = both(lambda h: lib.loss_terms(ctx, upload(lib, ctx, C, c, h), Xd, Yd, REG))
        assert np.allclose(host, dev, rtol=1e-12, atol=0), (cap, host, dev)

        def scaled(h):
            d = upload(lib, ctx, C, c, h)
            d.scale(3.5)
            back = d.download()
            X2 = lib.DeviceFactors(ctx, C.shape[0], 64)
            lib.least_squares(ctx, d, X2, Yd, REG)
            out = back.data, X2.download()
            close(d, X2)
            return out

        dev, host = both(scaled)
        assert np.array_equal(host[0], C.data * np.float32(3.5)) and np.array_equal(host[0], dev[0])
        assert np.array_equal(host[1], dev[1]), cap
    close(Yd, Xd)


def test_bad_row_in_second_segment(lib, ctx):
    check_bad_row_in_second_segment(lib, ctx, host=True)


def test_refusals(lib, ctx, C):
    d = upload(lib, ctx, C, caps_of(C)["thirds"], True)
    with pytest.raises(lib.AlsError, match="host-resident") as e:
        d.slice_rows(0, 10)
    assert e.value.code == lib.ALS_E_UNSUPPORTED
    items = lib.DeviceFactors.from_host(ctx, factors_of("mixed", C.shape[1], 32, 1))
    q = lib.DeviceFactors.from_host(ctx, factors_of("mixed", C.shape[0], 32, 2))
    with pytest.raises(lib.AlsError, match="host-resident") as e:
        lib.topk(ctx, items, q, 10, liked=d)
    assert e.value.code == lib.ALS_E_UNSUPPORTED
    close(d, items, q)


def _fit(lib, ctx, C, use_cg):
    from implicit_b200 import AlternatingLeastSquares

    m = AlternatingLeastSquares(factors=32, iterations=3, use_cg=use_cg, regularization=REG, random_state=1,
                                calculate_training_loss=True)
    m._ctx = ctx
    losses = []
    m.fit(C, show_progress=False, callback=lambda it, t, loss: losses.append(loss))
    rec = m.recalculate_user(np.arange(0, 300), C[:300])
    m.partial_fit_items(np.arange(400, 650), C.T.tocsr()[:250])  # 150 new items
    return m.user_factors.copy(), m.item_factors.copy(), rec, np.array(losses)


def _positive(C):
    Cp = abs(C)  # the public class takes what a user passes: positive confidences
    Cp.data += np.float32(1)
    return Cp


@pytest.mark.parametrize("use_cg", [False, True])
def test_public_fit_bitwise(lib, ctx, C, use_cg, monkeypatch):
    Cp = _positive(C)
    cap = caps_of(C)["thirds"]
    uploads = []
    real = lib.DeviceCSR.upload.__func__
    monkeypatch.setattr(lib.DeviceCSR, "upload", classmethod(lambda cls, *a, **k: uploads.append(k.get("host", False))
                                                             or real(cls, *a, **k)))
    out = []
    for host in (False, True):
        uploads.clear()
        ctx.set_knob("segment_nnz", cap)
        ctx.set_knob("host_csr", int(host))
        out.append(_fit(lib, ctx, Cp, use_cg))
        assert uploads[0] == host  # the fit's Cui; recalculate_user / partial_fit upload their own rows
    for a, b in zip(out[0][:3], out[1][:3]):
        assert np.array_equal(a, b)
    assert np.allclose(out[0][3], out[1][3], rtol=1e-12, atol=0)


def test_fit_picks_host_when_device_is_full(lib, ctx, C, monkeypatch):
    """With device memory taken by a ballast tensor, fit() stores Cui / Ciu in host memory by itself and reproduces the
    unballasted segmented fit bit for bit."""
    import torch

    Cp = _positive(C)
    cap = caps_of(C)["thirds"]
    ctx.set_knob("segment_nnz", cap)
    want = _fit(lib, ctx, Cp, False)
    users, items = Cp.shape
    free_ctx = ctx.mem_info()[0]
    assert lib.csr_residency(users, items, Cp.nnz, 32, free_ctx) == "device"
    drv_free = torch.cuda.mem_get_info()[0]
    leave = 256 << 20
    ballast = torch.empty(max(drv_free - leave, 0), dtype=torch.uint8, device="cuda")
    try:
        free_now = ctx.mem_info()[0]
        if lib.csr_residency(users, items, Cp.nnz, 32, free_now) != "host":
            pytest.skip(f"the memory pool keeps {(free_now - leave) / 2**20:.0f} MiB cached: the ballast cannot fill the device")
        uploads = []
        real = lib.DeviceCSR.upload.__func__
        monkeypatch.setattr(lib.DeviceCSR, "upload", classmethod(
            lambda cls, *a, **k: uploads.append(k.get("host", False)) or real(cls, *a, **k)))
        got = _fit(lib, ctx, Cp, False)
        assert uploads[0] is True
    finally:
        del ballast
        torch.cuda.empty_cache()
    for a, b in zip(want[:3], got[:3]):
        assert np.array_equal(a, b)
    assert np.allclose(want[3], got[3], rtol=1e-12, atol=0)
