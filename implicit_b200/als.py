"""Implicit Alternating Least Squares on H100 -- the host-side mirror of the reference model classes.

Same surface as ``implicit.als.AlternatingLeastSquares`` (factory, implicit/als.py:7-80) /
``implicit.cpu.als.AlternatingLeastSquares`` (implicit/cpu/als.py:20-477) for the ALS hot path:
``fit``, ``recommend``, ``recalculate_user`` / ``recalculate_item``, ``partial_fit_users`` /
``partial_fit_items``, ``similar_items`` / ``similar_users``, ``save`` / ``load`` and the attributes the
reference exposes.  All arithmetic runs in libals_b200.so (hand-written sm_90a CUDA) through ctypes;
this file only orders the calls the way the reference does and keeps its error behaviour.
"""
import logging
import os
import time

import numpy as np
from scipy.sparse import csr_matrix

from . import _lib, pcg64
from .distributed import RowBlock
from .utils import CudaArray
from .utils import (BLOCK_FIELDS, ModelFitError, block_cuts, check_block_table, check_csr, check_random_state,
                    column_splits, cuda_ids, is_cuda_array, is_device_csr, nnz_balanced_splits, splits_from_cuts)

log = logging.getLogger("implicit")

#: nonzeros of the filter CSR ("already liked") that one top-k call takes: its kernels walk int32 positions
_LIKED_NNZ_MAX = _lib.INT32_CSR_MAX_NNZ


def liked_batches(indptr, limit):
    """Consecutive query ranges [(start, end), ...] covering every row of a CSR with this `indptr`, each holding at
    most `limit` nonzeros (recommend splits its top-k call along them)."""
    indptr = np.asarray(indptr, dtype=np.int64)
    n = len(indptr) - 1
    out = []
    start = 0
    while start < n:
        end = min(int(np.searchsorted(indptr, indptr[start] + limit, side="right")) - 1, n)
        if end <= start:
            raise ValueError(f"row {start} of user_items holds {int(indptr[start + 1] - indptr[start])} nonzeros, "
                             f"more than one top-k call takes ({limit})")
        out.append((start, end))
        start = end
    return out


class _Ingest:
    """The failure protocol of a multi-GPU ingest: every rank raises if any rank's step fails, before the next
    collective; the failing rank its own error, the others an AlsError.  held: every device CSR this rank has built so
    far, closed when any rank fails."""

    def __init__(self, ctx, what="ingest of user_items"):
        self.ctx, self.held, self.what = ctx, [], what

    @staticmethod
    def run(fn):
        try:
            return fn(), None
        except Exception as e:  # noqa: BLE001 -- whatever it is, the other ranks must learn of it
            return None, e

    def fail(self, err, failed):
        if not failed:
            return
        for c in self.held:
            c.close()
        if err is not None:
            raise err
        raise _lib.AlsError(_lib.ALS_E_INVALID, f"another rank's {self.what} failed (see its error message)")

    def agreed(self, fn):
        """fn() on every rank, then one all-reduce of a failure flag before anyone goes on"""
        out, err = self.run(fn)
        self.fail(err, self.ctx.allreduce([1.0 if err is not None else 0.0], "max")[0] > 0)
        return out

    def keep(self, csrs):
        self.held.extend(csrs)
        return csrs


def block_pieces(ctx, block, first_row, usplit):
    """The rows of a row block (scipy CSR, rows [first_row, first_row + block.shape[0]) of user_items) cut along the
    user split: one device CSR per rank q, its rows in [usplit[q], usplit[q + 1]) (mostly none), each uploaded straight
    out of the block's arrays.  A bad index or indptr raises ValueError naming its row of user_items."""
    cut = np.clip(np.asarray(usplit, dtype=np.int64) - int(first_row), 0, block.shape[0])
    pieces = []
    try:
        for q in range(len(cut) - 1):
            pieces.append(_lib.DeviceCSR.upload_rows(ctx, block, cut[q], cut[q + 1]))
    except BaseException as e:
        for c in pieces:
            c.close()
        where = _first_bad_row(block, first_row) if isinstance(e, ValueError) else None
        if where is not None:
            raise ValueError(where) from e
        raise
    return pieces


def _first_bad_row(block, first_row):
    """What als_csr_upload64 refuses in a row block, named by its row of user_items (None if nothing is found)."""
    ip = np.asarray(block.indptr, dtype=np.int64)
    down = np.flatnonzero(np.diff(ip) < 0)
    if down.size:
        return f"user_items: indptr is not monotone at row {first_row + int(down[0])}"
    idx = block.indices[ip[0]:ip[-1]]
    bad = np.flatnonzero((idx < 0) | (idx >= block.shape[1]))
    if not bad.size:
        return None
    row = int(np.searchsorted(ip, ip[0] + bad[0], side="right")) - 1
    return (f"user_items: row {first_row + row} holds column index {int(idx[bad[0]])}, which is outside "
            f"[0, {block.shape[1]})")


class AlternatingLeastSquares:
    """Alternating Least Squares (Hu, Koren & Volinsky 2008; CG variant Takacs et al. 2011) on one or more H100s.

    Parameters mirror implicit/als.py:7-19.  ``use_gpu`` must stay True and ``dtype`` float32: this
    package has no CPU path and computes in fp32.  New: ``device`` (CUDA ordinal) and
    ``process_group`` (implicit_b200.distributed.ProcessGroup) for row-sharded multi-GPU fits.

    Inputs in CUDA memory: ``fit``, ``recommend`` (its liked filter and ``recalculate_user``), ``recalculate_*`` and
    ``partial_fit_*`` also take a CSR whose arrays live on the model's device -- a CUDA ``torch.sparse_csr_tensor``, or any
    object with ``shape`` and ``indptr`` / ``indices`` / ``data`` exposing ``__cuda_array_interface__`` (versions 2 and 3,
    e.g. ``cupyx.scipy.sparse.csr_matrix``).  It is copied on the device into arrays the library owns (never aliased),
    with int32 / int64 indices and float32 / float64 values, and gives bitwise the results of the same scipy CSR of
    float32 values, entry for entry.  (A scipy CSR of other values is cast with ``astype``, which also merges its
    duplicates and sorts its rows; a device CSR keeps its entries as they are.  In ``recalculate_*`` a device CSR is
    scaled by ``alpha`` after the cast, a scipy one before it.)  ``user_factors`` /
    ``item_factors`` take CUDA float32 2-D arrays too (rows may be strided), copied device to device; the numpy getters
    download them lazily.  ``user_factors_device`` / ``item_factors_device`` hand out device snapshots of the factors.
    Serving: ``recommend`` / ``rank_items``, ``similar_items`` and ``similar_users`` run on the device whatever their
    ids, and no factor matrix is downloaded (norms and subsets are computed on the device).  When the ids argument
    (``userid`` / ``itemid``) is a 1-D int32 / int64 CUDA array, ``(ids, scores)`` come back as CUDA arrays
    (``__cuda_array_interface__`` v3, shape (n, N), complete when returned, outliving the model), and ``filter_items``,
    ``items`` and the ``similar_*`` subsets may be host or CUDA arrays.  Host ids (scalars, lists, numpy arrays) are
    checked and converted as numpy does, in the same order and with the same errors, uploaded, and the results come
    back as numpy arrays (1-D for a scalar id), bitwise those of the CUDA-id call for the same values.  A host-id
    ``similar_*`` call therefore neither downloads device-resident factors nor fills the ``user_norms`` /
    ``item_norms`` caches.
    Refitting on the device: when ``userids`` / ``itemids`` of ``partial_fit_users`` / ``partial_fit_items`` is a 1-D
    int32 / int64 CUDA array, the rows are solved, the factor matrix grown (new rows zero) and the rows stored on the
    device, the last occurrence of a repeated id winning as in numpy; no factor matrix crosses PCIe and the host copy is
    downloaded only when a getter asks for it.  The factors are bitwise those of the numpy call where it succeeds: with
    numpy ids, a call that adds no new rows raises ("assignment destination is read-only", the getters hand out
    read-only views), where the CUDA-id call stores the rows.  A max id whose rows would not fit in the device's memory
    is refused with ValueError (the numpy call raises MemoryError).
    Not covered, and refused with ValueError: device CSRs on a process group of several ranks (RowBlocks of device
    arrays included), CUDA ids in ``partial_fit_*`` there too, a negative CUDA id in ``partial_fit_*``, a device liked
    filter of 2^31 - 1 or more nonzeros, and ``evaluation`` with device CSRs; DLPack is not read.
    """

    def __init__(
        self,
        factors=100,
        regularization=0.01,
        alpha=1.0,
        dtype=np.float32,
        use_native=True,
        use_cg=True,
        use_gpu=True,
        iterations=15,
        calculate_training_loss=False,
        num_threads=0,
        random_state=None,
        device=None,
        process_group=None,
    ):
        if not use_gpu:
            raise ValueError("implicit_b200 has no CPU implementation: use_gpu must be True")
        if np.dtype(dtype) != np.float32:
            raise ValueError("implicit_b200 computes in float32: dtype must be np.float32")
        if factors > 1024:
            raise ValueError("implicit_b200 supports factors <= 1024 (like the reference's CUDA solver, implicit/gpu/als.cu:177-178)")
        if factors > 128 and not use_cg:
            raise ValueError("factors > 128 need use_cg=True: the Cholesky solver covers factors <= 128 "
                             "(the reference's GPU path is CG-only as well, implicit/gpu/als.py:126-165)")
        self.factors = factors
        self.regularization = regularization
        self.alpha = alpha
        self.dtype = np.dtype(dtype)
        self.use_native = use_native
        self.use_cg = use_cg
        self.iterations = iterations
        self.calculate_training_loss = calculate_training_loss
        self.num_threads = num_threads  # accepted for signature parity; the GPU schedules itself
        self.fit_callback = None
        self.cg_steps = 3  # attribute, not a kwarg: implicit/cpu/als.py:88
        self.random_state = random_state
        self.process_group = process_group
        self._device = device
        self._ctx = None
        self._p2p = False

        # host copies (authoritative between calls) and device replicas
        self._user_factors = None
        self._item_factors = None
        self._dev = {"user": None, "item": None}       # DeviceFactors
        self._dev_fresh = {"user": False, "item": False}   # device replica matches the host copy
        self._host_fresh = {"user": True, "item": True}    # host copy matches the device replica
        self._user_norms = self._item_norms = None
        self._dev_norms = {"user": None, "item": None}  # DeviceSnapshots of the norms the device serving path reads
        self._YtY = self._XtX = None

    # ------------------------------------------------------------------ device plumbing
    @property
    def ctx(self):
        if self._ctx is None:
            if self.process_group is not None:
                self._ctx = self.process_group.ctx
            else:
                self._ctx = _lib.Context(0 if self._device is None else self._device)
        return self._ctx

    def _get_host(self, side):
        host = self._user_factors if side == "user" else self._item_factors
        if not self._host_fresh[side] and self._dev[side] is not None:
            host = self._dev[side].download(pinned=True)  # page-locked: the D2H copy runs at PCIe speed
            if side == "user":
                self._user_factors = host
            else:
                self._item_factors = host
            self._host_fresh[side] = True
        if host is not None and host.flags.writeable:
            # the device replica is refreshed only by assignment (model.item_factors = new): an in-place edit of the
            # returned array would silently leave recommend / similar_items on the old factors, so it fails loudly
            host = host.view()
            host.setflags(write=False)
        return host

    def _set_host(self, side, value):
        if value is not None and not isinstance(value, np.ndarray) and hasattr(value, "__cuda_array_interface__"):
            self._set_device(side, value)
            return
        if value is not None:
            value = np.ascontiguousarray(value, dtype=np.float32)
        if side == "user":
            self._user_factors, self._user_norms, self._XtX = value, None, None
        else:
            self._item_factors, self._item_norms, self._YtY = value, None, None
        self._dev_norms[side] = None
        self._host_fresh[side] = True
        self._dev_fresh[side] = False

    def _set_device(self, side, value):
        """Assignment of a CUDA float32 2-D array: the device replica is filled device to device and the host copy is
        stale until a getter downloads it."""
        self._adopt_device(side, _lib.DeviceFactors.from_cuda(self.ctx, value, f"{side}_factors"))

    def _adopt_device(self, side, d):
        """d (a DeviceFactors the model now owns) becomes the device replica; the host copy is dropped."""
        if self._dev[side] is not None:
            self._dev[side].close()
        self._dev[side] = d
        if side == "user":
            self._user_factors, self._user_norms, self._XtX = None, None, None
        else:
            self._item_factors, self._item_norms, self._YtY = None, None, None
        self._dev_norms[side] = None
        self._dev_fresh[side] = True
        self._host_fresh[side] = False

    def _factors_shape(self, side):
        """The shape of one side's factors, from whichever copy is current (None: not set); downloads nothing."""
        if not self._host_fresh[side] and self._dev[side] is not None:
            return self._dev[side].rows, self._dev[side].factors
        host = self._user_factors if side == "user" else self._item_factors
        return None if host is None else host.shape

    user_factors = property(lambda self: self._get_host("user"), lambda self, v: self._set_host("user", v))
    item_factors = property(lambda self: self._get_host("item"), lambda self, v: self._set_host("item", v))

    @property
    def user_factors_device(self):
        """A snapshot of the user factors in device memory of its own, exposing __cuda_array_interface__ version 3:
        shape (users, factors), byte strides (4 ld, 4) with ld the padded width, '<f4'.  torch.as_tensor(...,
        device="cuda") or cupy.asarray(...) keep it alive; a later fit or assignment does not change it."""
        return self._device_factors("user").snapshot()

    @property
    def item_factors_device(self):
        """The item factors' snapshot, like user_factors_device."""
        return self._device_factors("item").snapshot()

    def _device_factors(self, side):
        """Device replica of one side, uploaded if the host copy is newer."""
        if not self._dev_fresh[side]:
            host = self._user_factors if side == "user" else self._item_factors
            if host is None:
                raise ValueError(f"{side}_factors are not set: fit the model first")
            d = self._dev[side]
            if d is None or d.rows != host.shape[0] or d.factors != host.shape[1]:
                if d is not None:
                    d.close()
                d = _lib.DeviceFactors(self.ctx, host.shape[0], host.shape[1])
                self._dev[side] = d
            d.upload(host)
            self._dev_fresh[side] = True
        return self._dev[side]

    def _mark_device_updated(self, side):
        self._dev_fresh[side] = True
        self._host_fresh[side] = False
        self._dev_norms[side] = None
        if side == "user":
            self._user_norms = self._XtX = None
        else:
            self._item_norms = self._YtY = None

    # ------------------------------------------------------------------ fit (implicit/cpu/als.py:98-202)
    def fit(self, user_items, show_progress=True, callback=None):
        """Factorizes the user_items matrix (CSR, users x items, values = confidence; scipy, or in CUDA memory on one
        GPU).  On a process group of several ranks, each rank may instead pass only its own rows, as a
        distributed.RowBlock."""
        random_state = check_random_state(self.random_state)
        pg = self.process_group
        from_blocks = isinstance(user_items, RowBlock) and pg is not None and pg.world > 1
        from_device = not isinstance(user_items, RowBlock) and is_device_csr(user_items)
        if from_device and pg is not None and pg.world > 1:
            raise ValueError("a CSR in CUDA memory is fitted on one GPU; on a process group of several ranks pass a "
                             "scipy CSR or RowBlocks of scipy CSRs")
        if from_blocks or from_device:
            Cui_host = None
        elif isinstance(user_items, RowBlock):
            Cui_host = user_items.whole()  # one rank: the block must be the whole matrix
        else:
            Cui_host = check_csr(user_items)  # ParameterWarning on non-CSR input (utils.py:159-169)
            if Cui_host.dtype != np.float32:
                Cui_host = Cui_host.astype(np.float32)  # cpu/als.py:129-130
        ctx = self.ctx

        Cui_s = Ciu_s = None
        drawn = {}  # side -> (generator state its device draw starts from, rows)
        try:
            s = time.time()
            # shards balanced by estimated cost: a row costs its nonzeros plus a fixed factorisation /
            # CG-recurrence term worth ~60 (Cholesky) or ~20 (CG) nonzeros
            row_cost = 20 if self.use_cg else 60
            if from_blocks:
                Cui_s, Ciu_s, usplit, isplit, (users, items, nnz) = self._ingest_row_blocks(user_items, row_cost)
            elif pg is not None and pg.world > 1:
                users, items, nnz = *Cui_host.shape, Cui_host.nnz
                Cui_s, Ciu_s, usplit, isplit = self._ingest_shards(Cui_host, row_cost)
            elif from_device:
                # copied on the device into the library's arrays and always device-resident (the host_csr rule is for
                # host arrays); the same layout, so bitwise the factors of the same scipy CSR
                Cui_s = _lib.DeviceCSR.from_device(ctx, user_items)
                users, items, nnz = Cui_s.shape3
                if self.alpha != 1.0:
                    Cui_s.scale(self.alpha)  # cpu/als.py:133-134, on device
                Ciu_s = Cui_s.transpose()
                usplit = isplit = None
            else:
                users, items, nnz = *Cui_host.shape, Cui_host.nnz
                # Cui / Ciu stay in page-locked host memory, streamed through the device segment by segment, when a
                # single-GPU fit would not fit in device memory (or the host_csr knob asks for it); the factors are bitwise
                # the same
                host = False
                if self.process_group is None:
                    host = bool(ctx.get_knob("host_csr")) or \
                        _lib.csr_residency(users, items, Cui_host.nnz, self.factors, ctx.mem_info()[0]) == "host"
                Cui_s = _lib.DeviceCSR.upload(ctx, Cui_host, host=host)
                if self.alpha != 1.0:
                    Cui_s.scale(self.alpha)  # cpu/als.py:133-134, on device
                Ciu_s = Cui_s.transpose()    # cpu/als.py:137, on device
                usplit = isplit = None
            log.debug("Uploaded and transposed in %.3fs", time.time() - s)

            # cpu/als.py:144-147: pre-set factors are kept, otherwise rng.random(...) * 0.01
            if self.process_group is not None and self.process_group.world > 1 and \
                    (self._factors_shape("user") is None or self._factors_shape("item") is None):
                # every rank must start from the same replicas: rank 0 draws a seed, everyone initialises from it
                seed = int(random_state.integers(1, 2**31 - 1)) if self.process_group.rank == 0 else 0
                seed = int(ctx.allreduce([float(seed)], "max")[0])
                random_state = np.random.default_rng(seed)
            if pcg64.device_drawable(random_state):
                # numpy's PCG64 draw is computed on the device: the generator is moved to the state the host draws
                # would leave before anything is allocated, and no host copy is made
                state = pcg64.get_state(random_state)
                for side, rows in (("user", users), ("item", items)):
                    if self._factors_shape(side) is None:
                        drawn[side] = (state, rows)
                        state = pcg64.after_float32_draws(state, rows * self.factors)
                pcg64.set_state(random_state, state)
            else:
                if self._factors_shape("user") is None:
                    self._set_host("user", random_state.random((users, self.factors), dtype=np.float32) * np.float32(0.01))
                if self._factors_shape("item") is None:
                    self._set_host("item", random_state.random((items, self.factors), dtype=np.float32) * np.float32(0.01))
            if any(self._factors_shape(side) not in (None, (rows, self.factors)) for side, rows in (("user", users),
                                                                                                   ("item", items))):
                raise ValueError("pre-set factors do not match the shape of user_items / the factors parameter")
            for side, (state, rows) in drawn.items():
                d = _lib.DeviceFactors(ctx, rows, self.factors)
                try:
                    d.fill_pcg64(state, np.float32(0.01))
                except BaseException:
                    d.close()
                    raise
                self._adopt_device(side, d)
            X = self._device_factors("user")
            Y = self._device_factors("item")
            self._user_norms = self._item_norms = self._YtY = self._XtX = None  # cpu/als.py:152-154
            self._dev_norms = {"user": None, "item": None}

            self._p2p = False
            if usplit is not None and os.environ.get("ALS_B200_NO_P2P") != "1":
                # fused exchange: solved rows are stored straight into the peers' replicas over NVLink
                ctx.attach_peers(X)
                ctx.attach_peers(Y)
                self._p2p = True
                # Gramian of the item factors for the first user half (each rank sums its own rows)
                _lib.gramian_shard(ctx, Y, isplit[pg.rank], isplit[pg.rank + 1] - isplit[pg.rank])

            loss = None
            progress = None
            if show_progress:
                try:
                    from tqdm.auto import tqdm

                    progress = tqdm(total=self.iterations)
                except ImportError:
                    progress = None
            try:
                for iteration in range(self.iterations):  # cpu/als.py:162-177
                    s = time.time()
                    self._half(Cui_s, X, Y, usplit)
                    self._half(Ciu_s, Y, X, isplit)
                    if self._p2p and not self.use_cg:
                        _lib.solver_status(ctx)  # raises on every rank in the same iteration if any rank's half failed
                    if progress is not None:
                        progress.update(1)
                    if self.calculate_training_loss:
                        loss = self._loss(Cui_s, X, Y, users, items, nnz)
                        if self._p2p:  # the loss pass reuses the Gramian buffers: restore Y^T Y for the next half
                            _lib.gramian_shard(ctx, Y, isplit[pg.rank], isplit[pg.rank + 1] - isplit[pg.rank])
                        if progress is not None:
                            progress.set_postfix({"loss": loss})
                        elif not show_progress:
                            log.info("loss %.4f", loss)
                    if not callback:
                        callback = self.fit_callback  # backward compatibility, cpu/als.py:193-195
                    if callback:
                        ctx.sync()
                        callback(iteration, time.time() - s, loss)
                ctx.sync()
            except BaseException:
                if self._p2p:  # failures are raised on every rank in the same half (_raise_together): unmap and leave
                    ctx.detach_peers(X)
                    ctx.detach_peers(Y)
                    self._p2p = False
                raise
            finally:
                if progress is not None:
                    progress.close()
            if self.calculate_training_loss and loss is not None:
                log.info("Final training loss %.4f", loss)
            if self._p2p:
                ctx.barrier()
                ctx.detach_peers(X)
                ctx.detach_peers(Y)
            self._mark_device_updated("user")
            self._mark_device_updated("item")
        except BaseException:
            # the getters of a failed fit return its initial factors, as when they were drawn on the host: numpy draws
            # them again from the saved states (the device replica, if filled, stays the current one, as after an upload)
            for side, (state, rows) in drawn.items():
                fresh = self._dev_fresh[side]
                self._set_host(side, pcg64.generator_at(state).random((rows, self.factors), dtype=np.float32) *
                               np.float32(0.01))
                self._dev_fresh[side] = fresh
            raise
        finally:  # on every exit: a traceback would otherwise keep both CSRs alive through this frame
            if Ciu_s is not None:
                Ciu_s.close()
            if Cui_s is not None:
                Cui_s.close()
        self._check_fit_errors()  # cpu/als.py:202

    def _ingest_shards(self, Cui_host, row_cost):
        """Multi-GPU: (Cui_s, Ciu_s, usplit, isplit), this rank's rows of user_items and of its transpose and the user and
        item splits, built without either whole matrix on any device.  The rank uploads its own user rows; the ranks sum
        their column counts, which plan the item split; each cuts the transpose of its rows into one piece per rank; the
        pieces are exchanged and every rank concatenates the ones it received in rank order (scipy's Cui.T.tocsr() order,
        since rank p's users precede rank p + 1's).  Every rank raises if any rank's part fails, before the next
        collective: the failing rank its own error, the others an AlsError."""
        pg, ctx = self.process_group, self.ctx
        users, items = Cui_host.shape
        usplit = nnz_balanced_splits(Cui_host.indptr, pg.world, row_cost)
        ing = _Ingest(ctx)
        # the first collective of the fit is the column-count all-reduce, which carries the upload's failure flag
        Cui_s, Ciu_s, isplit = self._transpose_shards(
            ing, lambda: _lib.DeviceCSR.upload_rows(ctx, Cui_host, usplit[pg.rank], usplit[pg.rank + 1]),
            users, items, row_cost)
        return Cui_s, Ciu_s, usplit, isplit

    def _ingest_row_blocks(self, block, row_cost):
        """Multi-GPU from row blocks: (Cui_s, Ciu_s, usplit, isplit, (users, items, nnz)) like _ingest_shards, when this
        rank holds only its own distributed.RowBlock of user_items.  The ranks all-gather their blocks' extents, plan
        the user split _ingest_shards would plan from the whole indptr (each searches only its own indptr), upload
        their rows in one piece per rank of that split and exchange the pieces; every rank stacks the pieces it
        received into its user shard, and the transpose follows as in _ingest_shards.  Failures are agreed on the same
        way; a bad index or indptr names its row of the whole matrix."""
        pg, ctx = self.process_group, self.ctx
        rank, W = pg.rank, pg.world
        ing = _Ingest(ctx)

        def read():
            m = block.csr()
            return m, (block.first_row, m.shape[0], block.users, m.shape[1], int(m.indptr[-1]) - int(m.indptr[0]), 0)

        out, err = ing.run(read)
        mine = out[1] if err is None else (0, 0, 0, 0, 0, 1)
        # the first collective of the fit: every rank's block extent and whether it could read its block (48 bytes)
        table = np.frombuffer(ctx.allgather_bytes(np.array(mine, dtype=np.int64).tobytes()), dtype=np.int64)
        table = table.reshape(W, len(BLOCK_FIELDS))
        ing.fail(err, table[:, -1].any())
        m = out[0]
        users, items, nnz = check_block_table(table)  # the same table on every rank: the same error on every rank
        cuts, err = ing.run(lambda: block_cuts(table, m.indptr, rank, row_cost))
        if err is not None:
            cuts = np.zeros(W - 1, dtype=np.int64)
        total = ctx.allreduce_i64(np.append(cuts, 1 if err is not None else 0))
        ing.fail(err, total[-1] > 0)
        usplit = splits_from_cuts(total[:-1], users)
        pieces = ing.agreed(lambda: ing.keep(block_pieces(ctx, m, block.first_row, usplit)))
        received = ing.agreed(lambda: ing.keep(ctx.exchange_csr(pieces)))
        for c in pieces:
            c.close()

        def stack():
            s = _lib.DeviceCSR.concat_rows(ctx, received, items, usplit[rank])
            for c in received:
                c.close()
            return s

        # the stack's failure flag rides along with the column counts
        Cui_s, Ciu_s, isplit = self._transpose_shards(ing, stack, users, items, row_cost)
        return Cui_s, Ciu_s, usplit, isplit, (users, items, nnz)

    def _transpose_shards(self, ing, build, users, items, row_cost):
        """(Cui_s, Ciu_s, isplit): this rank's user shard from build(), scaled by alpha; the ranks sum their column
        counts, which plan the item split; each cuts the transpose of its rows into one piece per rank; the pieces are
        exchanged and every rank concatenates the ones it received in rank order (scipy's Cui.T.tocsr() order, since
        rank p's users precede rank p + 1's)."""
        pg, ctx = self.process_group, self.ctx

        def shard():
            s = ing.keep([build()])[0]
            if self.alpha != 1.0:
                s.scale(self.alpha)  # cpu/als.py:133-134, on device
            return s, s.column_counts()

        out, err = ing.run(shard)
        counts = out[1] if err is None else np.zeros(items, dtype=np.int64)
        # the failure flag rides along with the column counts
        total = ctx.allreduce_i64(np.append(counts, 1 if err is not None else 0))
        ing.fail(err, total[-1] > 0)
        Cui_s = out[0]
        isplit = column_splits(total[:-1], pg.world, row_cost)
        pieces = ing.agreed(lambda: ing.keep(Cui_s.transpose_pieces(isplit)))
        # the exchange agrees inside on its own preparation and allocations; this flag covers what follows its last round
        received = ing.agreed(lambda: ing.keep(ctx.exchange_csr(pieces)))
        for c in pieces:
            c.close()
        Ciu_s = ing.agreed(lambda: ing.keep([_lib.DeviceCSR.merge_rows(ctx, received, users, isplit[pg.rank])])[0])
        for c in received:
            c.close()
        return Cui_s, Ciu_s, isplit

    def _half(self, C, X, Y, splits, ysplits=None):
        """One half-iteration: solve the rows of (this rank's shard of) C, then exchange them.

        Multi-GPU (peer replicas attached): the Gramian of Y was accumulated shard-wise and all-reduced by the
        previous half (`gramian_shard`), the solve kernel stores its rows into every replica, and the
        all-reduce of the NEXT Gramian -- over the rows this rank just solved -- doubles as the barrier that
        orders the next half after every peer's stores.  Nothing blocks the host."""
        ctx = self.ctx
        err = None
        if splits is not None and self._p2p:
            rank = self.process_group.rank
            # queued, not awaited: a row that is not positive definite is remembered on the device and flagged to every
            # rank through the Gramian all-reduce; fit() asks for the status once per iteration, on all ranks alike
            _lib.half_pregram_async(ctx, C, X, Y, self.regularization, self.use_cg, self.cg_steps)
            _lib.gramian_shard(ctx, X, splits[rank], splits[rank + 1] - splits[rank])
            return
        try:
            if self.use_cg:
                _lib.least_squares_cg(ctx, C, X, Y, self.regularization, self.cg_steps)
            else:
                _lib.least_squares(ctx, C, X, Y, self.regularization)
        except (ValueError, _lib.AlsError) as e:
            if splits is None:
                raise
            err = e
        if splits is not None:
            ctx.allgather_rows(X, splits)
            self._raise_together(err)

    def _raise_together(self, err):
        """Multi-GPU: all ranks agree on failure (max-reduce of a flag) and raise in the same half-iteration."""
        failed = self.ctx.allreduce([1.0 if err is not None else 0.0], "max")[0] > 0
        if err is not None:
            raise err
        if failed:
            raise _lib.AlsError(_lib.ALS_E_NOT_POSDEF, "another rank failed in this half-iteration (see its error message)")

    def _loss(self, C, X, Y, users, items, nnz):
        ctx = self.ctx
        t = _lib.loss_terms(ctx, C, X, Y, self.regularization)
        if self.process_group is not None and self.process_group.world > 1:
            tot = ctx.allreduce(t[:2], "sum")
            t = np.array([tot[0], tot[1], t[2]])
        return float((t[0] + t[2]) / (t[1] + float(users) * float(items) - float(nnz)))

    def _check_fit_errors(self):
        """implicit/recommender_base.py:218-223 (the NaN scan runs on the device replicas)"""
        is_nan = self._device_factors("user").has_nan() or self._device_factors("item").has_nan()
        if is_nan:
            raise ModelFitError("NaN encountered in factors")

    # ------------------------------------------------------------------ recalculate / partial fit
    def _recalculate(self, ids, matrix, other_side, gram):
        """implicit/cpu/als.py:204-265: Cholesky on purpose, with the cached Gramian of the other side.  A device CSR is
        scaled by alpha on the device, after its values are cast to float32."""
        out = self._recalculate_device(1 if np.isscalar(ids) else len(ids), matrix, other_side, gram)
        try:
            res = out.download()
        finally:
            out.close()
        return res[0] if np.isscalar(ids) else res

    def _recalculate_device(self, n, matrix, other_side, gram):
        """The n rows _recalculate returns, left on the device: a DeviceFactors the caller closes."""
        device = is_device_csr(matrix)
        if not device:
            matrix = check_csr(matrix)
        if matrix.shape[0] != n:
            raise ValueError("user_items should have one row for every item in user")
        if self.alpha != 1.0 and not device:
            matrix = self.alpha * matrix
        ctx = self.ctx
        Y = self._device_factors(other_side)
        if device:
            C = _lib.DeviceCSR.from_device(ctx, matrix)
            if self.alpha != 1.0:
                C.scale(self.alpha)
        else:
            C = _lib.DeviceCSR.upload(ctx, matrix.astype(np.float32))
        out = _lib.DeviceFactors(ctx, n, self.factors)
        try:
            _lib.least_squares_with_gramian(ctx, gram, C, out, Y, self.regularization)
        except BaseException:
            out.close()
            raise
        finally:
            C.close()
        return out

    def recalculate_user(self, userid, user_items):
        return self._recalculate(userid, user_items, "item", self.YtY)

    def recalculate_item(self, itemid, item_users):
        return self._recalculate(itemid, item_users, "user", self.XtX)

    def partial_fit_users(self, userids, user_items):
        """implicit/cpu/als.py:267-307.  With userids a 1-D int32 / int64 CUDA array the rows are refitted in place on
        the device (_partial_fit_device)."""
        self._partial_fit("user", userids, user_items, "user_items must contain 1 row for every user in userids")

    def partial_fit_items(self, itemids, item_users):
        """implicit/cpu/als.py:309-349.  With itemids a 1-D int32 / int64 CUDA array, as partial_fit_users."""
        self._partial_fit("item", itemids, item_users, "item_users must contain 1 row for every user in itemids")

    def _partial_fit(self, side, ids, matrix, count_message):
        """partial_fit_* of one side: host ids with numpy's semantics (negative ids index from the end, the factors grow
        to max(ids) + 1 rows), CUDA ids on the device."""
        if is_cuda_array(ids):
            return self._partial_fit_device(side, ids, matrix, count_message)
        if len(ids) != matrix.shape[0]:
            raise ValueError(count_message)
        rows = getattr(self, f"recalculate_{side}")(ids, matrix)
        host = self._get_host(side)
        n, factors = host.shape
        max_id = max(ids)
        if max_id >= n:
            host = np.concatenate([host, np.zeros((max_id - n + 1, factors), dtype=self.dtype)])
        host[ids] = rows
        self._set_host(side, host)

    def _partial_fit_device(self, side, ids_in, matrix, count_message):
        """partial_fit_* for ids in CUDA memory: the rows are recalculated on the device (the same solve, with the same
        cached Gramian, as the host path), the device replica grows to max(ids) + 1 rows if it must (new rows zero) and
        takes the rows at their ids, the last occurrence of a repeated id winning, as numpy's host[ids] = rows does.  No
        factor matrix crosses PCIe: one pass over the ids reads back their min and max, and the host copy is downloaded
        only if a getter asks for it.  ValueError, before anything is written: a process group of several ranks, ids
        that are not 1-D int32 / int64, a row count other than len(ids), a negative id; and, after the solve, no ids at
        all (like the host path's max() of no ids) and a max id whose rows would not fit in the device's memory."""
        what = f"{side}ids"
        pg = self.process_group
        if pg is not None and pg.world > 1:
            raise ValueError(f"{what} in CUDA memory refit {side}s on one GPU; on a process group of several ranks pass "
                             f"{what} as a host array")
        ids = cuda_ids(ids_in, what)
        if len(ids) != matrix.shape[0]:
            raise ValueError(count_message)
        ctx = self.ctx
        lo, hi = _lib.ids_range(ctx, ids)
        if lo < 0:
            raise ValueError(f"{what} holds a negative id ({lo})")
        other = "item" if side == "user" else "user"
        rows = self._recalculate_device(len(ids), matrix, other, self.YtY if side == "user" else self.XtX)
        grown = False
        try:
            if not len(ids):
                raise ValueError(f"{what} is empty: no rows to refit")
            F = self._device_factors(side)
            if hi >= F.rows:
                F.grow(hi + 1)  # ValueError, F unchanged, past the device's memory
                grown = True
            F.scatter_rows(ids, rows)
        except BaseException:
            if grown:  # the replica has rows the host copy lacks: it is the current copy from here on
                self._mark_device_updated(side)
            raise
        finally:
            rows.close()
        self._mark_device_updated(side)

    @property
    def YtY(self):
        """implicit/cpu/als.py:425-430 (without lambda)"""
        if self._YtY is None:
            self._YtY = _lib.gramian(self.ctx, self._device_factors("item"))
        return self._YtY

    @property
    def XtX(self):
        if self._XtX is None:
            self._XtX = _lib.gramian(self.ctx, self._device_factors("user"))
        return self._XtX

    # ------------------------------------------------------------------ recommend (cpu/matrix_factorization_base.py:35-96)
    def recommend(self, userid, user_items, N=10, filter_already_liked_items=True, filter_items=None,
                  recalculate_user=False, items=None):
        """cpu/matrix_factorization_base.py:35-96.  With userid a 1-D int32 / int64 CUDA array, (ids, scores) come back
        in CUDA memory (see _recommend).  Host ids are checked here as numpy checks them and in the same order, uploaded
        as int64, and the results downloaded: numpy arrays, 1-D for a scalar id, the ids in the dtype of np.array(items)
        with `items`."""
        if is_cuda_array(userid):
            return self._recommend(userid, user_items, N, filter_already_liked_items, filter_items, recalculate_user,
                                   items)
        self._check_user_items(user_items, 1 if np.isscalar(userid) else len(userid), filter_already_liked_items,
                               recalculate_user)
        rows = np.atleast_1d(np.asarray(userid)).astype(np.int64)
        if not recalculate_user and rows.size and (rows.min() < 0 or rows.max() >= self._device_factors("user").rows):
            raise IndexError("userid out of range")
        subset = None
        if items is not None:
            if filter_items:  # numpy's own ValueError for an array of several ids
                raise ValueError("Can't set both items and filter_items in recommend call")
            subset = _host_subset(items, self._device_factors("item").rows,
                                  "Some itemids in the items parameter in are not in the model")
            if filter_already_liked_items and is_device_csr(user_items):
                raise ValueError("recommend(..., items=...) filters liked items of a scipy CSR only, not of a CSR in "
                                 "CUDA memory")
        n_items = self._device_factors("item").rows if subset is None else len(subset)
        if filter_items is not None:
            filter_items = np.asarray(filter_items).ravel()
            if filter_items.size and (filter_items.min() < 0 or filter_items.max() >= n_items):
                raise IndexError("filter_items contains ids that are not in the model")
            filter_items = filter_items.astype(np.int64)
        if N < 0:  # numpy's, from the output allocation of the host top-k
            raise ValueError("negative dimensions are not allowed")
        if filter_already_liked_items and subset is None and user_items.shape[1] != n_items:
            raise _lib.AlsError(_lib.ALS_E_INVALID, f"als_topk: liked has {user_items.shape[1]} columns for {n_items} items")
        out = self._recommend(rows, user_items, N, filter_already_liked_items, filter_items, recalculate_user,
                              None if subset is None else subset.astype(np.int64), host=True)
        return _to_host(self.ctx, out, np.isscalar(userid), None if subset is None else subset.dtype)

    @staticmethod
    def _check_user_items(user_items, n_query, filter_already_liked_items, recalculate_user):
        if filter_already_liked_items or recalculate_user:
            if not isinstance(user_items, csr_matrix) and not is_device_csr(user_items):
                raise ValueError("user_items needs to be a CSR sparse matrix")
            if user_items.shape[0] != n_query:
                raise ValueError("user_items must contain 1 row for every user in userids")

    def _recommend(self, userid, user_items, N, filter_already_liked_items, filter_items, recalculate_user, items,
                   host=False):
        """recommend() on the device: the ids, the subset, the liked remap and the outputs stay there, and no factor
        matrix is downloaded.  userid, filter_items and items are host or CUDA arrays (_device_ids); user_items a scipy or
        device CSR.  Returns (ids, scores), DeviceSnapshots of shape (len(userid), N): int32 ids (the subset's dtype with
        `items`), float32 scores.  `host`: called by the host adapter, which has made numpy's checks of items and
        filter_items (a filter numpy finds false may come with items) and downloads and frees the outputs at once (they
        are pooled)."""
        ctx = self.ctx
        tmp = []
        try:
            uid = self._device_ids(userid, "userid", tmp)
            n_query = len(uid)
            device = is_device_csr(user_items)
            self._check_user_items(user_items, n_query, filter_already_liked_items, recalculate_user)
            query_rows = None
            if recalculate_user:
                queries = self._recalculate_device(n_query, user_items, "item", self.YtY)
                tmp.append(queries)
            else:
                queries, query_rows = self._device_factors("user"), uid
            item_handle = self._device_factors("item")
            subset = None
            if items is not None:
                N = min(N, _ids_len(items, "items"))
                if not host and filter_items is not None and _ids_len(filter_items, "filter_items"):
                    raise ValueError("Can't set both items and filter_items in recommend call")
                if _ids_len(items, "items") == 0:
                    raise ValueError("zero-size array to reduction operation maximum which has no identity")
                subset = self._device_ids(items, "items", tmp, sort=True)
                item_handle = _lib.DeviceFactors.gather_rows(ctx, item_handle, subset)
                if item_handle is None:
                    raise IndexError("Some itemids in the items parameter in are not in the model")
                tmp.append(item_handle)

            fq = None
            batches = [(0, n_query)]
            if filter_already_liked_items and device:
                fq = _lib.DeviceCSR.from_device(ctx, user_items)  # unsorted rows are sorted on the device
                tmp.append(fq)
                if fq.shape3[2] > _LIKED_NNZ_MAX:
                    raise ValueError(f"a liked filter in CUDA memory holds at most {_LIKED_NNZ_MAX} nonzeros")
                if subset is not None:
                    fq = fq.restrict_columns(subset)
                    tmp.append(fq)
            elif filter_already_liked_items:
                fq = user_items
                if subset is not None:  # liked ids remapped to positions in the subset; only its ids come to the host
                    fq = _filter_items_from_sparse_matrix(_lib.ids_download(ctx, subset), fq)
                if not fq.has_sorted_indices:
                    fq = fq.sorted_indices()
                if fq.nnz > _LIKED_NNZ_MAX:
                    batches = liked_batches(fq.indptr, _LIKED_NNZ_MAX)

            fl = None
            if filter_items is not None:
                fl = self._device_ids(filter_items, "filter_items", tmp)
            stream = self._one_stream(uid, fl, subset)
            N = int(N)
            ids = _lib.DeviceSnapshot(ctx, (n_query, N), f"<i{4 if subset is None else subset.itemsize}", pooled=host)
            scores = _lib.DeviceSnapshot(ctx, (n_query, N), "<f4", pooled=host)
            for b0, b1 in batches:
                liked = None
                if device and fq is not None:
                    liked = fq
                elif fq is not None:
                    liked = _lib.DeviceCSR.upload(ctx, fq if len(batches) == 1 else fq[b0:b1])
                    tmp.append(liked)
                qr = None if query_rows is None else _slice(query_rows, b0, b1)
                bad = _lib.topk_into(ctx, item_handle, queries, N, b1 - b0, ids.cuda(b0), scores.cuda(b0),
                                     query_rows=qr, query_row0=b0 if qr is None and len(batches) > 1 else 0,
                                     liked=liked, filter_items=fl, id_map=subset, stream=stream)
                if bad & 1:
                    raise IndexError("userid out of range")
                if bad:
                    raise IndexError("filter_items contains ids that are not in the model")
                if liked is not None and not device:
                    liked.close()
        finally:
            for t in tmp:
                t.close()
        return ids, scores

    def _ranking_sums(self, userids, user_items, test_items, K, gain, gain_sum):
        """The six sums of evaluation.ranking_metrics_at_k (hits, sum min(K, L), AP, nDCG, AUC, users) for the users
        `userids`: the ids of recommend(userids, user_items, N=K) scored against the same rows of test_items (scipy
        CSRs, one row per user) without leaving the device.  Refuses what recommend refuses, the same way."""
        queries = self._device_factors("user")
        query_rows = np.asarray(userids, dtype=np.int64)
        if query_rows.size and (query_rows.min() < 0 or query_rows.max() >= queries.rows):
            raise IndexError("userid out of range")
        items, ctx = self._device_factors("item"), self.ctx
        batches = [(0, len(query_rows))]
        if user_items.nnz > _LIKED_NNZ_MAX:
            batches = liked_batches(user_items.indptr, _LIKED_NNZ_MAX)
        sums = np.zeros(6)
        for b0, b1 in batches:
            held = []
            try:
                liked = _lib.DeviceCSR.upload_rows(ctx, user_items, b0, b1)
                held.append(liked)
                test = _lib.DeviceCSR.upload_rows(ctx, test_items, b0, b1)
                held.append(test)
                sums += _lib.ranking_metrics(ctx, items, queries, K, query_rows[b0:b1], test, gain, gain_sum, liked)
            finally:
                for c in held:
                    c.close()
        return sums

    def rank_items(self, userid, user_items, selected_items, recalculate_user=False):
        """implicit/recommender_base.py:204-216 (deprecated alias)"""
        return self.recommend(userid, user_items, recalculate_user=recalculate_user, items=selected_items,
                              filter_already_liked_items=False)

    # ------------------------------------------------------------------ similar_* (cpu/matrix_factorization_base.py:149-231)
    @property
    def user_norms(self):
        if self._user_norms is None:
            n = np.linalg.norm(self.user_factors, axis=-1)
            n[n == 0] = 1e-10
            self._user_norms = n
        return self._user_norms

    @property
    def item_norms(self):
        if self._item_norms is None:
            n = np.linalg.norm(self.item_factors, axis=-1)
            n[n == 0] = 1e-10
            self._item_norms = n
        return self._item_norms

    # ------------------------------------------------------------------ serving on the device
    def _device_norms(self, side):
        """The row norms of one side on the device (a DeviceSnapshot, bitwise the user_norms / item_norms properties),
        cached until the factors change; never downloads the factors."""
        if self._dev_norms[side] is None:
            self._dev_norms[side] = self._device_factors(side).row_norms()
        return self._dev_norms[side]

    def _device_ids(self, ids, what, tmp, sort=False):
        """The utils.CudaArray of an ids argument of a device call: a 1-D int32 / int64 CUDA array as it is (sorted into a
        copy when `sort`), or host ids (list, numpy) uploaded, sorted first when `sort`.  Uploads and sorted copies are
        pooled temporaries, appended to `tmp`.  Host ids keep numpy's dtype (np.array of a list of ints is int64); other
        than int32 / int64 they are refused with ValueError."""
        if is_cuda_array(ids):
            a = cuda_ids(ids, what)
            if not sort:
                return a
            s = _lib.ids_sort(self.ctx, a)
            tmp.append(s)
            return s.cuda()
        a = np.array(ids).ravel()
        if a.size == 0 and a.dtype == np.float64:
            a = a.astype(np.int64)  # np.array([]) of an empty list
        if a.dtype not in (np.int32, np.int64):
            raise ValueError(f"{what}: ids of dtype {a.dtype} (a call with ids in CUDA memory takes int32 or int64)")
        if sort:
            a.sort()
        s = _lib.DeviceSnapshot.from_host(self.ctx, a, pooled=True)
        tmp.append(s)
        return s.cuda()

    @staticmethod
    def _one_stream(*arrays):
        """The producer stream the CUDA arrays of one call name (0: none); ValueError when they name different ones."""
        streams = {a.stream for a in arrays if a is not None and a.stream}
        if len(streams) > 1:
            raise ValueError("the CUDA arrays of one call name different producer streams")
        return streams.pop() if streams else 0

    def _similar_host(self, side, ids_in, N, recalculate, filter_ids, subset):
        """_similar for host ids, checked as numpy checks them and in the same order, uploaded as int64, the results
        downloaded (numpy arrays, 1-D for a scalar id, the ids in the dtype of np.array(subset)).  Without a recalculation
        an id past the rows raises numpy's IndexError and a negative one AlsError (when anything is ranked); filter ids
        outside the rows ranked are ignored."""
        rows = self._device_factors(side).rows
        if recalculate is None:
            _index_check(rows, ids_in)
        if subset is not None:
            if filter_ids:  # numpy's own ValueError for an array of several ids
                raise ValueError("Can't set both a subset and a filter in a similar_* call")
            subset = _host_subset(subset, rows, "Some ids in the subset parameter are not in the model")
        if N < 0:  # numpy's, from the output allocation of the host top-k
            raise ValueError("negative dimensions are not allowed")
        query_rows = np.atleast_1d(np.asarray(ids_in)).astype(np.int64)
        negative = query_rows < 0
        if recalculate is None and negative.any() and N > 0:
            raise _lib.AlsError(_lib.ALS_E_INVALID, f"topk: query row {query_rows[negative][0]} out of range")
        query_rows[negative] += rows  # N == 0: nothing is ranked, and numpy indexed the norms from the end
        if filter_ids is not None:
            targets = rows if subset is None else len(subset)
            filter_ids = np.asarray(filter_ids).ravel().astype(np.int32)
            filter_ids = filter_ids[(filter_ids >= 0) & (filter_ids < targets)]
        out = self._similar(side, query_rows, N, recalculate, filter_ids,
                            None if subset is None else subset.astype(np.int64), scalar=np.isscalar(ids_in), host=True)
        return _to_host(self.ctx, out, np.isscalar(ids_in), None if subset is None else subset.dtype)

    def _similar(self, side, ids_in, N, recalculate, filter_ids, subset, scalar=False, host=False):
        """similar_* on the device: the norms computed there (bitwise the user_norms / item_norms properties), a subset
        gathered there (kept unsorted, duplicates included, and N not clamped) and the query norms divided out in the
        top-k's epilogue.  ids_in, filter_ids and subset are host or CUDA arrays (_device_ids); recalculate is
        (item_users,) for similar_items(recalculate_item=True), else None, and `scalar` a recalculation of one host id,
        whose norm numpy takes as a dot product.  Returns DeviceSnapshots (ids, scores) of shape (len(ids_in), N); `host`
        as for _recommend.  An id of filter_ids outside the model raises IndexError."""
        ctx = self.ctx
        what = f"{side}id"
        tmp = []
        try:
            qa = self._device_ids(ids_in, what, tmp)
            handle = self._device_factors(side)
            if recalculate is not None:
                queries = self._recalculate_device(len(qa), recalculate[0], "user", self.XtX)
                tmp.append(queries)
                if scalar:
                    norm = np.linalg.norm(queries.download()[0])
                    qnorms = _lib.DeviceSnapshot.from_host(ctx, np.array([norm if norm != 0 else 1e-10], np.float32),
                                                           pooled=True)
                else:
                    qnorms = queries.row_norms()
                tmp.append(qnorms)
                query_rows = None
            else:
                queries, query_rows, qnorms = handle, qa, self._device_norms(side)
            target, tnorms, sub = handle, self._device_norms(side), None
            if subset is not None:
                if not host and filter_ids is not None and _ids_len(filter_ids, f"filter_{side}s"):
                    raise ValueError("Can't set both a subset and a filter in a similar_* call")
                if _ids_len(subset, "items" if side == "item" else "users") == 0:
                    raise ValueError("zero-size array to reduction operation maximum which has no identity")
                sub = self._device_ids(subset, "items" if side == "item" else "users", tmp)
                target = _lib.DeviceFactors.gather_rows(ctx, handle, sub)
                if target is None:
                    raise IndexError("Some ids in the subset parameter are not in the model")
                tmp.append(target)
                tnorms = target.row_norms()  # bitwise the norms of those rows
                tmp.append(tnorms)
            fl = None
            if filter_ids is not None:
                fl = self._device_ids(filter_ids, f"filter_{side}s", tmp)
            stream = self._one_stream(qa, fl, sub)
            N = int(N)
            ids = _lib.DeviceSnapshot(ctx, (len(qa), N), f"<i{4 if sub is None else sub.itemsize}", pooled=host)
            scores = _lib.DeviceSnapshot(ctx, (len(qa), N), "<f4", pooled=host)
            bad = _lib.topk_into(ctx, target, queries, N, len(qa), ids.cuda(), scores.cuda(), query_rows=query_rows,
                                 item_norms=tnorms, query_norms=qnorms, filter_items=fl, id_map=sub, stream=stream)
            if bad & 1:
                raise IndexError(f"{what} out of range")
            if bad:
                raise IndexError(f"filter_{side}s contains ids that are not in the model")
        finally:
            for t in tmp:
                t.close()
        return ids, scores

    def similar_items(self, itemid, N=10, recalculate_item=False, item_users=None, filter_items=None, items=None):
        serve = self._similar if is_cuda_array(itemid) else self._similar_host
        return serve("item", itemid, N, (item_users,) if recalculate_item else None, filter_items, items)

    def similar_users(self, userid, N=10, filter_users=None, users=None):
        serve = self._similar if is_cuda_array(userid) else self._similar_host
        return serve("user", userid, N, None, filter_users, users)

    # ------------------------------------------------------------------ persistence (cpu/als.py:458-477, recommender_base.py:173-202)
    def save(self, fileobj_or_path):
        args = {
            "user_factors": self.user_factors,
            "item_factors": self.item_factors,
            "regularization": self.regularization,
            "factors": self.factors,
            "num_threads": self.num_threads,
            "iterations": self.iterations,
            "use_native": self.use_native,
            "use_cg": self.use_cg,
            "cg_steps": self.cg_steps,
            "calculate_training_loss": self.calculate_training_loss,
            "dtype": self.dtype.name,
            "random_state": self.random_state,
            "alpha": self.alpha,
        }
        args = {k: v for k, v in args.items() if v is not None}
        np.savez(fileobj_or_path, **args)

    @classmethod
    def load(cls, fileobj_or_path):
        if isinstance(fileobj_or_path, str) and not fileobj_or_path.endswith(".npz"):
            fileobj_or_path = fileobj_or_path + ".npz"
        with np.load(fileobj_or_path, allow_pickle=False) as data:
            ret = cls()
            for k, v in data.items():
                if k == "dtype":
                    v = np.dtype(str(v))
                elif v.shape == ():
                    v = v.item()
                setattr(ret, k, v)
            return ret

    def __getstate__(self):
        state = dict(self.__dict__)
        state["_user_factors"] = self.user_factors
        state["_item_factors"] = self.item_factors
        state.update(_ctx=None, process_group=None, _dev={"user": None, "item": None}, _dev_norms={"user": None, "item": None},
                     _dev_fresh={"user": False, "item": False}, _host_fresh={"user": True, "item": True})
        return state

    def __setstate__(self, state):
        self.__dict__.update(state)
        self.__dict__.setdefault("_dev_norms", {"user": None, "item": None})


def _filter_items_from_sparse_matrix(items, query_items):
    """implicit/cpu/matrix_factorization_base.py:253-264: remap liked ids to positions in the sorted subset."""
    coo = query_items.tocoo()
    positions = np.searchsorted(items, coo.col)
    positions = np.clip(positions, 0, len(items) - 1)
    coo.data[items[positions] != coo.col] = 0
    coo.col = positions
    coo.eliminate_zeros()
    out = coo.tocsr()
    # the reference keeps the original column count; positions index the subset, so shrink to it
    return csr_matrix((out.data, out.indices, out.indptr), shape=(out.shape[0], len(items)))


def _slice(a, b0, b1):
    """Entries [b0, b1) of a 1-D utils.CudaArray."""
    return CudaArray(a.ptr + b0 * a.itemsize, (b1 - b0,), a.itemsize, 1, a.stream)


def _ids_len(ids, what):
    """The number of ids of a host or CUDA ids argument."""
    return len(cuda_ids(ids, what)) if is_cuda_array(ids) else int(np.asarray(ids).size)


def _index_check(rows, ids):
    """Raises the IndexError numpy raises when `ids` index an array of `rows` rows, if any: ids past the rows, float
    ids."""
    np.broadcast_to(np.int8(0), (rows,))[ids]


def _host_subset(ids, rows, message):
    """np.array(ids) of a host subset, checked in numpy's order: ValueError when it is empty (its max), IndexError(message)
    for ids outside [0, rows), then numpy's IndexError for ids that cannot index (_index_check)."""
    a = np.array(ids)
    if a.max() >= rows or a.min() < 0:
        raise IndexError(message)
    _index_check(rows, a)
    return a


def _to_host(ctx, out, scalar, ids_dtype=None):
    """The (ids, scores) DeviceSnapshots of a serving call as numpy arrays, the snapshots freed: 1-D for a scalar id, the
    ids cast to `ids_dtype` (a host subset's own dtype, which holds every id of the subset)."""
    ids, scores = (_lib.ids_download(ctx, CudaArray(s.ptr.value, (s.shape[0] * s.shape[1],), s.itemsize, 1, 0))
                   .reshape(s.shape) for s in out)
    for s in out:
        s.close()
    scores = scores.view(np.float32)
    if ids_dtype is not None:
        ids = ids.astype(ids_dtype, copy=False)
    return (ids[0], scores[0]) if scalar else (ids, scores)
