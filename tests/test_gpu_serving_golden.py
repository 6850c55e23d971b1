"""recommend, rank_items and similar_* against tests/golden/serving.npz, what they returned or raised for host ids
before the host ids were served through the device path (tests/golden/make_golden_serving.py).  Host ids must give the
recorded outputs bitwise, with their dtypes and shapes, or the recorded exception and message; where the case allows it,
the same ids as an int32 or int64 CUDA array must give the same values."""
import os

import numpy as np
import pytest

import _serving_cases as sc

torch = pytest.importorskip("torch")

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs PyTorch with CUDA")]

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "serving.npz"))
CASES = {c[0]: c for c in sc.cases()}


@pytest.fixture(scope="module")
def models():
    from implicit_b200 import _lib

    ctx = _lib.Context(0)
    yield {f: sc.model(ctx, f) for f in sc.WIDTHS}
    ctx.close()


def test_every_case_is_recorded():
    recorded = {k.rsplit("__", 1)[0] for k in GOLD.files}
    assert recorded == set(CASES)


def same_bits(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape, (got.dtype, want.dtype, got.shape, want.shape)
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8))


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_and_cuda_ids_match_golden(models, name, monkeypatch):
    from implicit_b200 import als

    _, f, method, kw, cuda, liked_max = CASES[name]
    if liked_max is not None:
        monkeypatch.setattr(als, "_LIKED_NNZ_MAX", liked_max)
    m = models[f]
    if f"{name}__exc" in GOLD.files:
        with pytest.raises(Exception) as e:
            sc.call(m, method, kw)
        assert (type(e.value).__name__, str(e.value)) == (str(GOLD[f"{name}__exc"]), str(GOLD[f"{name}__msg"]))
        return
    want_ids, want_scores = GOLD[f"{name}__ids"], GOLD[f"{name}__scores"]
    ids, scores = sc.call(m, method, kw)
    assert isinstance(ids, np.ndarray) and isinstance(scores, np.ndarray)
    same_bits(ids, want_ids)
    same_bits(scores, want_scores)
    if not cuda:
        return
    key = "userid" if "userid" in kw else "itemid"
    for dtype in (np.int32, np.int64):
        dev = dict(kw)
        dev[key] = torch.from_numpy(np.atleast_1d(np.asarray(kw[key])).astype(dtype)).cuda()
        ids, scores = (torch.as_tensor(x, device="cuda").cpu().numpy() for x in sc.call(m, method, dev))
        same_bits(ids, np.atleast_2d(want_ids))
        same_bits(scores, np.atleast_2d(want_scores))
