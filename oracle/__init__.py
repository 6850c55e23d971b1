"""CPU oracle for the ALS hot path -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this package.  The product (implicit_b200/) never does.

Two implementations of the same interface (the reference's native operator interface,
implicit/cpu/_als.pyx:67,145,251 and implicit/cpu/topk.pyx:15):

  * ``port``  -- the plain-C restatement in oracle/als_oracle.c (always available; gcc only)
  * ``ref``   -- the reference's own Cython/OpenMP modules compiled unchanged from /root/reference
                 into oracle/_ref/ by oracle/build_ref.py (available wherever that build was run;
                 the built .so files travel to the GPU box with the gpurun snapshot)

``get(kind)`` returns a namespace with least_squares / least_squares_cg / calculate_loss / topk.
``fit(...)`` restates the reference fit loop (implicit/cpu/als.py:98-202) over either of them.
"""
import ctypes
import glob
import importlib.util
import os
import subprocess
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
_PORT_SO = os.path.join(HERE, "libals_oracle.so")
_REF_DIR = os.path.join(HERE, "_ref")


# ----------------------------------------------------------------------------- build
def build_port(force=False):
    src = os.path.join(HERE, "als_oracle.c")
    if force or not os.path.exists(_PORT_SO) or os.path.getmtime(_PORT_SO) < os.path.getmtime(src):
        subprocess.run(
            ["/usr/bin/gcc", "-O2", "-fopenmp", "-fPIC", "-shared", "-std=c11", "-ffp-contract=off",
             "-fvisibility=hidden", src, "-o", _PORT_SO, "-lm"],
            check=True,
        )
    return _PORT_SO


def build_ref(force=False):
    import importlib

    # not `from . import build_ref`: that name is this function once the package is initialised
    return importlib.import_module(__name__ + ".build_ref").build(force=force)


def have_ref():
    return bool(glob.glob(os.path.join(_REF_DIR, "_als*.so"))) and bool(
        glob.glob(os.path.join(_REF_DIR, "topk*.so"))
    )


# ----------------------------------------------------------------------------- port (ctypes)
_lib = None


def _port_lib():
    global _lib
    if _lib is None:
        build_port()
        lib = ctypes.CDLL(_PORT_SO)
        f32p = ctypes.POINTER(ctypes.c_float)
        i32p = ctypes.POINTER(ctypes.c_int32)
        lib.oracle_gramian.argtypes = [f32p, ctypes.c_int64, ctypes.c_int, f32p]
        lib.oracle_gramian.restype = None
        lib.oracle_least_squares.argtypes = [f32p, i32p, i32p, f32p, f32p, f32p, ctypes.c_int64,
                                             ctypes.c_int, ctypes.c_double, ctypes.c_int]
        lib.oracle_least_squares.restype = ctypes.c_int64
        lib.oracle_least_squares_cg.argtypes = [f32p, i32p, i32p, f32p, f32p, f32p, ctypes.c_int64,
                                                ctypes.c_int, ctypes.c_int, ctypes.c_int]
        lib.oracle_least_squares_cg.restype = None
        lib.oracle_calculate_loss.argtypes = [f32p, i32p, i32p, f32p, f32p, f32p, ctypes.c_int64,
                                              ctypes.c_int64, ctypes.c_int, ctypes.c_float, ctypes.c_int]
        lib.oracle_calculate_loss.restype = ctypes.c_double
        lib.oracle_select.argtypes = [f32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, i32p, f32p]
        lib.oracle_select.restype = None
        lib.oracle_topk.argtypes = [f32p, ctypes.c_int64, f32p, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
                                    f32p, i32p, i32p, i32p, ctypes.c_int64, i32p, f32p, ctypes.c_int]
        lib.oracle_topk.restype = None
        _lib = lib
    return _lib


def _f32(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float)) if a is not None else None


def _i32(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)) if a is not None else None


def _csr_parts(Cui):
    indptr = np.ascontiguousarray(Cui.indptr, dtype=np.int32)
    indices = np.ascontiguousarray(Cui.indices, dtype=np.int32)
    data = np.ascontiguousarray(Cui.data, dtype=np.float32)
    return indptr, indices, data


def _check(X):
    if X.dtype != np.float32 or not X.flags.c_contiguous:
        raise ValueError("oracle port handles C-contiguous float32 factors only")


def _port_gramian(Y):
    _check(Y)
    G = np.zeros((Y.shape[1], Y.shape[1]), dtype=np.float32)
    _port_lib().oracle_gramian(_f32(Y), Y.shape[0], Y.shape[1], _f32(G))
    return G


def _port_least_squares(Cui, X, Y, regularization, num_threads=0):
    """implicit/cpu/_als.pyx:67-72"""
    _check(X), _check(Y)
    YtY = _port_gramian(Y)
    return _port__least_squares(YtY, Cui.indptr, Cui.indices, Cui.data.astype("float32"), X, Y,
                                regularization, num_threads)


def _port__least_squares(YtY, indptr, indices, data, X, Y, regularization, num_threads=0):
    """implicit/cpu/_als.pyx:76"""
    _check(X), _check(Y)
    indptr = np.ascontiguousarray(indptr, dtype=np.int32)
    indices = np.ascontiguousarray(indices, dtype=np.int32)
    data = np.ascontiguousarray(data, dtype=np.float32)
    YtY = np.ascontiguousarray(YtY, dtype=np.float32)
    bad = _port_lib().oracle_least_squares(_f32(YtY), _i32(indptr), _i32(indices), _f32(data), _f32(X),
                                           _f32(Y), X.shape[0], X.shape[1], float(regularization),
                                           int(num_threads))
    if bad >= 0:
        raise ValueError("cython_lapack.posv failed (err=%i) on row %i. Try "
                         "increasing the regularization parameter." % (1, bad))


def _port_least_squares_cg(Cui, X, Y, regularization, num_threads=0, cg_steps=3):
    """implicit/cpu/_als.pyx:145-149, :154"""
    _check(X), _check(Y)
    N = X.shape[1]
    YtY = _port_gramian(Y) + np.float32(regularization) * np.eye(N, dtype=np.float32)
    YtY = np.ascontiguousarray(YtY, dtype=np.float32)
    indptr, indices, data = _csr_parts(Cui)
    _port_lib().oracle_least_squares_cg(_f32(YtY), _i32(indptr), _i32(indices), _f32(data), _f32(X), _f32(Y),
                                        X.shape[0], N, int(cg_steps), int(num_threads))


def _port_least_squares_cg_with_gramian(YtY, Cui, X, Y, regularization, num_threads=0, cg_steps=3):
    """_port_least_squares_cg with the caller's fp32 Gramian in place of Y^T Y (a shard's Gramian, as
    als_least_squares_cg_pregram takes it): YtY + reg I is formed in fp32 like :164."""
    _check(X), _check(Y)
    N = X.shape[1]
    YtY = np.ascontiguousarray(np.asarray(YtY, dtype=np.float32) + np.float32(regularization) * np.eye(N, dtype=np.float32))
    indptr, indices, data = _csr_parts(Cui)
    _port_lib().oracle_least_squares_cg(_f32(YtY), _i32(indptr), _i32(indices), _f32(data), _f32(X), _f32(Y),
                                        X.shape[0], N, int(cg_steps), int(num_threads))


def _port_calculate_loss(Cui, X, Y, regularization, num_threads=0):
    """implicit/cpu/_als.pyx:251-308"""
    _check(X), _check(Y)
    YtY = _port_gramian(Y)
    indptr, indices, data = _csr_parts(Cui)
    return _port_lib().oracle_calculate_loss(_f32(YtY), _i32(indptr), _i32(indices), _f32(data), _f32(X),
                                             _f32(Y), X.shape[0], Y.shape[0], X.shape[1],
                                             float(regularization), int(num_threads))


def _port_topk(items, query, k, item_norms=None, filter_query_items=None, filter_items=None, num_threads=0):
    """implicit/cpu/topk.pyx:15"""
    if query.ndim == 1:
        query = query.reshape((1, len(query)))
    items = np.ascontiguousarray(items, dtype=np.float32)
    query = np.ascontiguousarray(query, dtype=np.float32)
    rows = query.shape[0]
    indices = np.zeros((rows, k), dtype="int32")
    distances = np.zeros((rows, k), dtype=np.float32)
    fp = fi = None
    if filter_query_items is not None:
        fp = np.ascontiguousarray(filter_query_items.indptr, dtype=np.int32)
        fi = np.ascontiguousarray(filter_query_items.indices, dtype=np.int32)
    fl = None
    if filter_items is not None:
        fl = np.ascontiguousarray(np.asarray(filter_items).ravel(), dtype=np.int32)
    norms = None if item_norms is None else np.ascontiguousarray(item_norms, dtype=np.float32)
    _port_lib().oracle_topk(_f32(items), items.shape[0], _f32(query), rows, items.shape[1], int(k),
                            _f32(norms), _i32(fp), _i32(fi), _i32(fl), 0 if fl is None else len(fl),
                            _i32(indices), _f32(distances), int(num_threads))
    return indices, distances


def _port_select(scores, k):
    """select<float>(batch, k, ids, distances) on precomputed scores (implicit/cpu/select.h:12-39): (ids, scores) of
    shape [rows, k], zero past the row's item count like topk.pyx:20-21."""
    scores = np.ascontiguousarray(np.atleast_2d(scores), dtype=np.float32)
    rows, cols = scores.shape
    ids = np.zeros((rows, k), dtype=np.int32)
    distances = np.zeros((rows, k), dtype=np.float32)
    _port_lib().oracle_select(_f32(scores), rows, cols, int(k), _i32(ids), _f32(distances))
    return ids, distances


port = types.SimpleNamespace(
    name="port", least_squares=_port_least_squares, _least_squares=_port__least_squares,
    least_squares_cg=_port_least_squares_cg, least_squares_cg_with_gramian=_port_least_squares_cg_with_gramian,
    calculate_loss=_port_calculate_loss, topk=_port_topk, gramian=_port_gramian, select=_port_select,
)


# ----------------------------------------------------------------------------- ref (compiled reference)
_ref = None


def _load_ext(name):
    path = glob.glob(os.path.join(_REF_DIR, name + "*.so"))[0]
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _ref_ns():
    global _ref
    if _ref is None:
        if not have_ref():
            raise RuntimeError("oracle/_ref is not built (run `python oracle/build_ref.py` where "
                               "/root/reference exists)")
        als = _load_ext("_als")
        tk = _load_ext("topk")
        _ref = types.SimpleNamespace(
            name="ref", least_squares=als.least_squares, _least_squares=als._least_squares,
            least_squares_cg=als.least_squares_cg, calculate_loss=als.calculate_loss, topk=tk.topk,
            gramian=lambda Y: np.dot(np.transpose(Y), Y),
        )
    return _ref


def have_ref_evaluation():
    return bool(glob.glob(os.path.join(_REF_DIR, "evaluation*.so")))


_ref_eval = None


def ref_evaluation():
    """The reference's compiled implicit/evaluation.pyx.  It does `from .utils import check_random_state`,
    so it is loaded as a member of a synthetic package whose `utils` holds that one function."""
    global _ref_eval
    if _ref_eval is None:
        import sys

        if not have_ref_evaluation():
            raise RuntimeError("oracle/_ref/evaluation*.so is not built (python oracle/build_ref.py --force)")
        pkg = types.ModuleType("_als_b200_refpkg")
        pkg.__path__ = [_REF_DIR]
        utils = types.ModuleType("_als_b200_refpkg.utils")

        def check_random_state(random_state):  # implicit/utils.py:65-83
            if isinstance(random_state, np.random.RandomState):
                return np.random.default_rng(random_state.randint(2**31))
            return np.random.default_rng(random_state)

        utils.check_random_state = check_random_state
        sys.modules["_als_b200_refpkg"] = pkg
        sys.modules["_als_b200_refpkg.utils"] = utils
        path = glob.glob(os.path.join(_REF_DIR, "evaluation*.so"))[0]
        spec = importlib.util.spec_from_file_location("_als_b200_refpkg.evaluation", path)
        mod = importlib.util.module_from_spec(spec)
        sys.modules["_als_b200_refpkg.evaluation"] = mod
        spec.loader.exec_module(mod)
        _ref_eval = mod
    return _ref_eval


def get(kind="auto"):
    """kind: 'port', 'ref', or 'auto' (ref when built, else port)."""
    if kind == "port":
        return port
    if kind == "ref":
        return _ref_ns()
    return _ref_ns() if have_ref() else port


# ----------------------------------------------------------------------------- R5: the fit loop
def fit(Cui, user_factors, item_factors, regularization=0.01, iterations=15, use_cg=True, cg_steps=3,
        alpha=1.0, num_threads=0, kind="auto", callback=None):
    """Restates implicit/cpu/als.py:126-177 on pre-set factors (updated in place, like :144-147 keeps them).

    Cui: scipy CSR (users x items).  Returns (user_factors, item_factors).
    """
    impl = get(kind)
    if Cui.dtype != np.float32:
        Cui = Cui.astype(np.float32)  # :129-130
    if alpha != 1.0:
        Cui = alpha * Cui  # :133-134
    Ciu = Cui.T.tocsr()  # :137
    for it in range(iterations):  # :162
        if use_cg:
            impl.least_squares_cg(Cui, user_factors, item_factors, regularization, num_threads=num_threads,
                                  cg_steps=cg_steps)
            impl.least_squares_cg(Ciu, item_factors, user_factors, regularization, num_threads=num_threads,
                                  cg_steps=cg_steps)
        else:
            impl.least_squares(Cui, user_factors, item_factors, regularization, num_threads=num_threads)
            impl.least_squares(Ciu, item_factors, user_factors, regularization, num_threads=num_threads)
        if callback:
            callback(it)
    return user_factors, item_factors


def row_rel_err(A, B):
    """Per-row ||A-B||_2 / ||B||_2 (rows with ||B|| == 0 compare absolutely).  SURVEY.md section 8(c)."""
    A = np.asarray(A, dtype=np.float64)
    B = np.asarray(B, dtype=np.float64)
    num = np.linalg.norm(A - B, axis=1)
    den = np.linalg.norm(B, axis=1)
    return np.where(den > 0, num / np.where(den > 0, den, 1), num)
