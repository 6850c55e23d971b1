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

from . import _lib
from .utils import ModelFitError, check_csr, check_random_state, nnz_balanced_splits

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


class AlternatingLeastSquares:
    """Alternating Least Squares (Hu, Koren & Volinsky 2008; CG variant Takacs et al. 2011) on one or more H100s.

    Parameters mirror implicit/als.py:7-19.  ``use_gpu`` must stay True and ``dtype`` float32: this
    package has no CPU path and computes in fp32.  New: ``device`` (CUDA ordinal) and
    ``process_group`` (implicit_b200.distributed.ProcessGroup) for row-sharded multi-GPU fits.
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
        if value is not None:
            value = np.ascontiguousarray(value, dtype=np.float32)
        if side == "user":
            self._user_factors, self._user_norms, self._XtX = value, None, None
        else:
            self._item_factors, self._item_norms, self._YtY = value, None, None
        self._host_fresh[side] = True
        self._dev_fresh[side] = False

    user_factors = property(lambda self: self._get_host("user"), lambda self, v: self._set_host("user", v))
    item_factors = property(lambda self: self._get_host("item"), lambda self, v: self._set_host("item", v))

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
        if side == "user":
            self._user_norms = self._XtX = None
        else:
            self._item_norms = self._YtY = None

    # ------------------------------------------------------------------ fit (implicit/cpu/als.py:98-202)
    def fit(self, user_items, show_progress=True, callback=None):
        """Factorizes the user_items matrix (CSR, users x items, values = confidence)."""
        random_state = check_random_state(self.random_state)
        Cui_host = check_csr(user_items)  # ParameterWarning on non-CSR input (utils.py:159-169)
        if Cui_host.dtype != np.float32:
            Cui_host = Cui_host.astype(np.float32)  # cpu/als.py:129-130
        users, items = Cui_host.shape
        ctx = self.ctx

        s = time.time()
        # Cui / Ciu stay in page-locked host memory, streamed through the device segment by segment, when a single-GPU
        # fit would not fit in device memory (or the host_csr knob asks for it); the factors are bitwise the same
        host = False
        if self.process_group is None:
            host = bool(ctx.get_knob("host_csr")) or \
                _lib.csr_residency(users, items, Cui_host.nnz, self.factors, ctx.mem_info()[0]) == "host"
        Cui = _lib.DeviceCSR.upload(ctx, Cui_host, host=host)
        if self.alpha != 1.0:
            Cui.scale(self.alpha)  # cpu/als.py:133-134, on device
        Ciu = Cui.transpose()      # cpu/als.py:137, on device
        log.debug("Uploaded and transposed in %.3fs", time.time() - s)

        # cpu/als.py:144-147: pre-set factors are kept, otherwise rng.random(...) * 0.01
        if self.process_group is not None and self.process_group.world > 1 and \
                (self._get_host("user") is None or self._get_host("item") is None):
            # every rank must start from the same replicas: rank 0 draws a seed, everyone initialises from it
            seed = int(random_state.integers(1, 2**31 - 1)) if self.process_group.rank == 0 else 0
            seed = int(ctx.allreduce([float(seed)], "max")[0])
            random_state = np.random.default_rng(seed)
        if self._get_host("user") is None:
            self._set_host("user", random_state.random((users, self.factors), dtype=np.float32) * np.float32(0.01))
        if self._get_host("item") is None:
            self._set_host("item", random_state.random((items, self.factors), dtype=np.float32) * np.float32(0.01))
        if self._user_factors.shape != (users, self.factors) or self._item_factors.shape != (items, self.factors):
            raise ValueError("pre-set factors do not match the shape of user_items / the factors parameter")
        X = self._device_factors("user")
        Y = self._device_factors("item")
        self._user_norms = self._item_norms = self._YtY = self._XtX = None  # cpu/als.py:152-154

        # row shards for the multi-GPU fit (whole matrix on one GPU)
        pg = self.process_group
        Cui_s, Ciu_s, usplit, isplit = Cui, Ciu, None, None
        self._p2p = False
        if pg is not None and pg.world > 1:
            # shards balanced by estimated cost: a row costs its nonzeros plus a fixed factorisation /
            # CG-recurrence term worth ~60 (Cholesky) or ~20 (CG) nonzeros
            row_cost = 20 if self.use_cg else 60
            usplit = nnz_balanced_splits(Cui_host.indptr, pg.world, row_cost)
            isplit = nnz_balanced_splits(Ciu.indptr_host(), pg.world, row_cost)
            if os.environ.get("ALS_B200_NO_P2P") != "1":
                # fused exchange: solved rows are stored straight into the peers' replicas over NVLink
                ctx.attach_peers(X)
                ctx.attach_peers(Y)
                self._p2p = True
                # Gramian of the item factors for the first user half (each rank sums its own rows)
                _lib.gramian_shard(ctx, Y, isplit[pg.rank], isplit[pg.rank + 1] - isplit[pg.rank])
            Cui_s = Cui.slice_rows(usplit[pg.rank], usplit[pg.rank + 1])
            Ciu_s = Ciu.slice_rows(isplit[pg.rank], isplit[pg.rank + 1])

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
                    loss = self._loss(Cui_s, X, Y, users, items, Cui_host.nnz)
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
        for c in (Cui_s, Ciu_s):
            if c is not Cui and c is not Ciu:
                c.close()
        Ciu.close()
        Cui.close()
        self._check_fit_errors()  # cpu/als.py:202

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
        """implicit/cpu/als.py:204-265: Cholesky on purpose, with the cached Gramian of the other side."""
        matrix = check_csr(matrix)
        n = 1 if np.isscalar(ids) else len(ids)
        if matrix.shape[0] != n:
            raise ValueError("user_items should have one row for every item in user")
        if self.alpha != 1.0:
            matrix = self.alpha * matrix
        ctx = self.ctx
        Y = self._device_factors(other_side)
        C = _lib.DeviceCSR.upload(ctx, matrix.astype(np.float32))
        out = _lib.DeviceFactors(ctx, n, self.factors)
        try:
            _lib.least_squares_with_gramian(ctx, gram, C, out, Y, self.regularization)
            res = out.download()
        finally:
            C.close()
            out.close()
        return res[0] if np.isscalar(ids) else res

    def recalculate_user(self, userid, user_items):
        return self._recalculate(userid, user_items, "item", self.YtY)

    def recalculate_item(self, itemid, item_users):
        return self._recalculate(itemid, item_users, "user", self.XtX)

    def partial_fit_users(self, userids, user_items):
        """implicit/cpu/als.py:267-307"""
        if len(userids) != user_items.shape[0]:
            raise ValueError("user_items must contain 1 row for every user in userids")
        user_factors = self.recalculate_user(userids, user_items)
        host = self.user_factors
        users, factors = host.shape
        max_userid = max(userids)
        if max_userid >= users:
            host = np.concatenate([host, np.zeros((max_userid - users + 1, factors), dtype=self.dtype)])
        host[userids] = user_factors
        self.user_factors = host

    def partial_fit_items(self, itemids, item_users):
        """implicit/cpu/als.py:309-349"""
        if len(itemids) != item_users.shape[0]:
            raise ValueError("item_users must contain 1 row for every user in itemids")
        item_factors = self.recalculate_item(itemids, item_users)
        host = self.item_factors
        items, factors = host.shape
        max_itemid = max(itemids)
        if max_itemid >= items:
            host = np.concatenate([host, np.zeros((max_itemid - items + 1, factors), dtype=self.dtype)])
        host[itemids] = item_factors
        self.item_factors = host

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
        if filter_already_liked_items or recalculate_user:
            if not isinstance(user_items, csr_matrix):
                raise ValueError("user_items needs to be a CSR sparse matrix")
            user_count = 1 if np.isscalar(userid) else len(userid)
            if user_items.shape[0] != user_count:
                raise ValueError("user_items must contain 1 row for every user in userids")

        ctx = self.ctx
        tmp = []
        try:
            if recalculate_user:
                q = np.atleast_2d(self.recalculate_user(userid, user_items))
                queries = _lib.DeviceFactors.from_host(ctx, q)
                tmp.append(queries)
                query_rows, n_query = None, q.shape[0]
            else:
                queries = self._device_factors("user")
                query_rows = np.atleast_1d(np.asarray(userid)).astype(np.int64)
                if query_rows.size and (query_rows.min() < 0 or query_rows.max() >= queries.rows):
                    raise IndexError("userid out of range")
                n_query = len(query_rows)

            item_handle = self._device_factors("item")
            n_items_model = item_handle.rows
            if items is not None:
                N = min(N, len(items))
                if filter_items:
                    raise ValueError("Can't set both items and filter_items in recommend call")
                items = np.array(items)
                items.sort()
                if items.max() >= n_items_model or items.min() < 0:
                    raise IndexError("Some itemids in the items parameter in are not in the model")
                item_handle = _lib.DeviceFactors.from_host(ctx, self.item_factors[items])
                tmp.append(item_handle)

            fq = None
            batches = [(0, n_query)]
            if filter_already_liked_items:
                fq = user_items
                if items is not None:
                    fq = _filter_items_from_sparse_matrix(items, fq)
                if not fq.has_sorted_indices:
                    fq = fq.sorted_indices()
                if fq.nnz > _LIKED_NNZ_MAX:
                    batches = liked_batches(fq.indptr, _LIKED_NNZ_MAX)

            fl = None
            if filter_items is not None:
                fl = np.asarray(filter_items).ravel()
                if fl.size and (fl.min() < 0 or fl.max() >= item_handle.rows):
                    raise IndexError("filter_items contains ids that are not in the model")

            parts = []
            for b0, b1 in batches:
                qr = query_rows
                if len(batches) > 1:
                    qr = query_rows[b0:b1] if query_rows is not None else np.arange(b0, b1)
                liked = None
                if fq is not None:
                    liked = _lib.DeviceCSR.upload(ctx, fq if len(batches) == 1 else fq[b0:b1])
                    tmp.append(liked)
                parts.append(_lib.topk(ctx, item_handle, queries, int(N), query_rows=qr, n_query=b1 - b0,
                                       liked=liked, filter_items=fl))
                if liked is not None:
                    liked.close()
            ids, scores = parts[0] if len(parts) == 1 else (np.concatenate([p[0] for p in parts]),
                                                             np.concatenate([p[1] for p in parts]))
        finally:
            for t in tmp:
                t.close()

        if np.isscalar(userid):
            ids, scores = ids[0], scores[0]
        if items is not None:
            ids = items[ids]
        return ids, scores

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

    def _similar(self, side, ids_in, N, recalculated, filter_ids, subset):
        ctx = self.ctx
        handle = self._device_factors(side)
        norms = self.user_norms if side == "user" else self.item_norms
        host = self.user_factors if side == "user" else self.item_factors
        tmp = []
        try:
            if recalculated is not None:
                factor = recalculated
                if np.isscalar(ids_in):
                    norm = np.linalg.norm(factor)
                    norm = norm if norm != 0 else 1e-10
                else:
                    norm = np.linalg.norm(factor, axis=1)
                    norm[norm == 0] = 1e-10
                queries = _lib.DeviceFactors.from_host(ctx, np.atleast_2d(factor))
                tmp.append(queries)
                query_rows, n_query = None, queries.rows
            else:
                norm = norms[ids_in]
                queries = handle
                query_rows = np.atleast_1d(np.asarray(ids_in)).astype(np.int64)
                n_query = len(query_rows)
            target, tnorms = handle, norms
            if subset is not None:
                if filter_ids:
                    raise ValueError("Can't set both a subset and a filter in a similar_* call")
                subset = np.array(subset)
                if subset.max() >= host.shape[0] or subset.min() < 0:
                    raise IndexError("Some ids in the subset parameter are not in the model")
                target = _lib.DeviceFactors.from_host(ctx, host[subset])
                tmp.append(target)
                tnorms = norms[subset]
            ids, scores = _lib.topk(ctx, target, queries, int(N), query_rows=query_rows, n_query=n_query,
                                    item_norms=tnorms, filter_items=filter_ids)
        finally:
            for t in tmp:
                t.close()
        if np.isscalar(ids_in):
            ids, scores = ids[0], scores[0]
            scores = scores / np.float32(norm)
        else:
            scores = scores / np.asarray(norm, dtype=np.float32)[:, None]
        if subset is not None:
            ids = subset[ids]
        return ids, scores

    def similar_items(self, itemid, N=10, recalculate_item=False, item_users=None, filter_items=None, items=None):
        rec = self.recalculate_item(itemid, item_users) if recalculate_item else None
        return self._similar("item", itemid, N, rec, filter_items, items)

    def similar_users(self, userid, N=10, filter_users=None, users=None):
        return self._similar("user", userid, N, None, filter_users, users)

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
        state.update(_ctx=None, process_group=None, _dev={"user": None, "item": None},
                     _dev_fresh={"user": False, "item": False}, _host_fresh={"user": True, "item": True})
        return state

    def __setstate__(self, state):
        self.__dict__.update(state)


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
