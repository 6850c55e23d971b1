"""CPU: the reader of ids given in CUDA memory (utils.cuda_ids) refuses what a device serving call cannot take, before
any pointer is used, and the device branch is taken for CUDA arrays only."""
import types

import numpy as np
import pytest

from implicit_b200.utils import cuda_ids, is_cuda_array


def ids(**over):
    d = dict(shape=(5,), typestr="<i8", strides=None, data=(0x7000_0000, False), version=3, stream=None)
    d.update(over)
    return types.SimpleNamespace(__cuda_array_interface__=d)


def test_accepts_int32_and_int64():
    a = cuda_ids(ids(), "userid")
    assert (a.ptr, len(a), a.itemsize, a.stream) == (0x7000_0000, 5, 8, 0)
    assert cuda_ids(ids(typestr="<i4", version=2), "userid").itemsize == 4
    assert cuda_ids(ids(typestr="<i4", version=2), "userid").stream == 1
    assert len(cuda_ids(ids(shape=(0,), data=(0, False)), "userid")) == 0


@pytest.mark.parametrize("bad,words", [
    (dict(typestr="<f4"), "typestr"), (dict(typestr="<f8"), "typestr"), (dict(typestr="<u4"), "typestr"),
    (dict(shape=(2, 3)), "1-D"), (dict(shape=()), "1-D"), (dict(strides=(16,)), "not contiguous"),
    (dict(version=1), "version"), (dict(stream=0), "stream"), (dict(data=(0, False)), "NULL"),
])
def test_refusals(bad, words):
    with pytest.raises(ValueError, match=words) as e:
        cuda_ids(ids(**bad), "itemid")
    assert str(e.value).startswith("itemid: ")


def test_device_branch_only_for_cuda_arrays():
    assert is_cuda_array(ids())
    assert not is_cuda_array(np.arange(3)) and not is_cuda_array([1, 2]) and not is_cuda_array(3)
