"""CPU-only: the package reads CUDA arrays by duck typing, without importing PyTorch or CuPy, and its
__cuda_array_interface__ parser refuses what it cannot take before any pointer is used (the pointers below point
nowhere)."""
import ast
import os

import pytest

from implicit_b200.utils import CudaArray, is_device_csr, parse_cai

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOWHERE = 0xDEAD0000


def test_product_imports_neither_torch_nor_cupy():
    pkg = os.path.join(ROOT, "implicit_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if not f.endswith(".py"):
                continue
            tree = ast.parse(open(os.path.join(dirpath, f)).read())
            for node in ast.walk(tree):
                names = []
                if isinstance(node, ast.Import):
                    names = [a.name for a in node.names]
                elif isinstance(node, ast.ImportFrom) and node.module:
                    names = [node.module]
                elif isinstance(node, ast.Call) and getattr(node.func, "id", None) == "__import__":
                    names = [a.value for a in node.args if isinstance(a, ast.Constant)]
                for n in names:
                    assert n.split(".")[0] not in ("torch", "cupy", "cupyx"), f"{f} imports {n}"


def cai(**kw):
    d = dict(shape=(10,), typestr="<i4", data=(NOWHERE, False), version=3)
    d.update(kw)
    return d


def test_parser_takes_versions_2_and_3_and_their_streams():
    a = parse_cai(cai(), "indices", ("<i4", "<i8"), 1)
    assert isinstance(a, CudaArray) and (a.ptr, a.shape, a.itemsize, a.stream) == (NOWHERE, (10,), 4, 0)
    assert parse_cai(cai(stream=None), "x", ("<i4",), 1).stream == 0
    assert parse_cai(cai(stream=0x1234), "x", ("<i4",), 1).stream == 0x1234
    assert parse_cai(cai(version=2), "x", ("<i4",), 1).stream == 1  # version 2: the legacy default stream
    assert parse_cai(cai(strides=(4,)), "x", ("<i4",), 1).ld == 1
    f = parse_cai(cai(shape=(5, 3), typestr="<f4", strides=(4 * 7, 4)), "f", ("<f4",), 2)
    assert (f.shape, f.ld) == ((5, 3), 7)
    assert parse_cai(cai(shape=(5, 3), typestr="<f4", strides=None), "f", ("<f4",), 2).ld == 3
    assert parse_cai(cai(shape=(0,), data=(0, False)), "x", ("<i4",), 1).shape == (0,)


@pytest.mark.parametrize("bad,match", [
    (dict(version=1), "version"),
    (dict(version=4), "version"),
    (dict(version=None), "version"),
    (dict(mask=cai()), "mask"),
    (dict(typestr="<f4"), "typestr"),
    (dict(typestr=">i4"), "typestr"),
    (dict(typestr="|b1"), "typestr"),
    (dict(shape=(10, 1)), "shape"),
    (dict(shape=10), "shape"),
    (dict(shape=(-1,)), "shape"),
    (dict(strides=(8,)), "not contiguous"),
    (dict(strides=(-4,)), "not contiguous"),
    (dict(strides=(4, 4)), "strides"),
    (dict(data=NOWHERE), "pointer"),
    (dict(data=(0, False)), "NULL"),
    (dict(stream=0), "stream"),
    (dict(stream="s"), "stream"),
])
def test_parser_refuses_1d(bad, match):
    with pytest.raises(ValueError, match=match):
        parse_cai(cai(**bad), "indices", ("<i4", "<i8"), 1)


@pytest.mark.parametrize("bad,match", [
    (dict(strides=(12, 8)), "column stride"),
    (dict(strides=(8, 4)), "row stride"),
    (dict(strides=(14, 4)), "row stride"),
    (dict(shape=(5,)), "shape"),
    (dict(typestr="<f8"), "typestr"),
])
def test_parser_refuses_2d(bad, match):
    d = cai(shape=(5, 3), typestr="<f4")
    d.update(bad)
    with pytest.raises(ValueError, match=match):
        parse_cai(d, "user_factors", ("<f4",), 2)


def test_parser_refuses_what_is_not_a_dict():
    with pytest.raises(ValueError, match="not a dict"):
        parse_cai([("shape", (10,))], "x", ("<i4",), 1)


def test_device_csr_detection():
    import numpy as np
    import scipy.sparse as sp

    class Arr:
        def __init__(self):
            self.__cuda_array_interface__ = cai()

    class Dev:
        shape = (3, 4)
        indptr, indices, data = Arr(), Arr(), Arr()

    class TorchLike:
        layout = "torch.sparse_csr"

        def crow_indices(self):
            return None

    assert is_device_csr(Dev()) and is_device_csr(TorchLike())
    assert not is_device_csr(sp.csr_matrix(np.eye(3, dtype=np.float32)))
    assert not is_device_csr(np.eye(3))
