"""CPU: partial_fit_users / partial_fit_items with CUDA ids refit on one GPU.  On every rank of a two-rank gloo process
group the call is refused with ValueError before any device work -- the ids' pointer is never read and no context is
made -- and the factors are left as they were."""
import multiprocessing as mp
import os

import numpy as np
import pytest
import scipy.sparse as sp


class FakeCudaIds:
    """Looks like a 1-D int64 CUDA array to the package; its address is never dereferenced."""

    def __init__(self, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (0x7F0000000000, False),
                                         "strides": None, "version": 3, "stream": None}


def _worker(port, rank, world, out_dir):
    import torch.distributed as dist

    from implicit_b200 import AlternatingLeastSquares
    from implicit_b200.distributed import ProcessGroup

    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    rng = np.random.default_rng(rank)
    X = rng.standard_normal((30, 8), dtype=np.float32)
    Y = rng.standard_normal((20, 8), dtype=np.float32)
    m = AlternatingLeastSquares(factors=8, process_group=ProcessGroup(dist.get_rank(), dist.get_world_size(), None))
    m.user_factors, m.item_factors = X, Y
    messages = []
    for fit, cols in ((m.partial_fit_users, 20), (m.partial_fit_items, 30)):
        try:
            fit(FakeCudaIds(3), sp.csr_matrix(np.ones((3, cols), dtype=np.float32)))
            messages.append("")
        except ValueError as e:
            messages.append(str(e))
    unchanged = np.array_equal(m.user_factors, X) and np.array_equal(m.item_factors, Y) and m._ctx is None
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), messages=np.array(messages), unchanged=unchanged)
    dist.barrier()
    dist.destroy_process_group()


def test_cuda_ids_refused_on_a_two_rank_group(tmp_path):
    pytest.importorskip("torch")
    ctx = mp.get_context("spawn")
    port = 33000 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(port, r, 2, str(tmp_path))) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    for r in range(2):
        z = np.load(tmp_path / f"rank{r}.npz")
        assert bool(z["unchanged"])
        users, items = (str(s) for s in z["messages"])
        assert "userids in CUDA memory" in users and "several ranks" in users
        assert "itemids in CUDA memory" in items and "several ranks" in items
