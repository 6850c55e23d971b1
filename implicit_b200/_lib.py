"""ctypes binding of libals_b200.so (include/als_b200.h) -- the only way Python reaches the GPU here.

There is deliberately no fallback: if the shared library is missing it is built with nvcc; if that
fails, or there is no H100 to run on, the caller gets an exception.
"""
import ctypes
import os

import numpy as np

from . import _build, utils

ALS_OK = 0
ALS_E_INVALID = -1
ALS_E_CUDA = -2
ALS_E_NCCL = -3
ALS_E_UNSUPPORTED = -4
ALS_E_NOT_POSDEF = -5
COMM_ID_BYTES = 128

c_void_p = ctypes.c_void_p
c_int = ctypes.c_int
c_i64 = ctypes.c_int64
c_f32 = ctypes.c_float
c_f64 = ctypes.c_double
P = ctypes.POINTER

#: every symbol include/als_b200.h declares: name -> (restype, argtypes)
SIGNATURES = {
    "als_abi_version": (c_int, []),
    "als_last_error": (ctypes.c_char_p, []),
    "als_device_count": (c_int, []),
    "als_ctx_create": (c_int, [c_int, P(c_void_p)]),
    "als_ctx_destroy": (c_int, [c_void_p]),
    "als_sync": (c_int, [c_void_p]),
    "als_device_info": (c_int, [c_void_p, ctypes.c_char_p, P(c_int), P(c_i64), P(c_i64)]),
    "als_launch_count": (c_i64, [c_void_p]),
    "als_timer_start": (c_int, [c_void_p]),
    "als_timer_stop": (c_int, [c_void_p, P(c_f32)]),
    "als_flush_l2": (c_int, [c_void_p, c_i64]),
    "als_profile_enable": (c_int, [c_void_p, c_int]),
    "als_profile_read": (c_int, [c_void_p, c_int, P(c_f64), P(c_i64)]),
    "als_host_alloc": (c_int, [P(c_void_p), c_i64]),
    "als_host_free": (c_int, [c_void_p]),
    "als_csr_upload": (c_int, [c_void_p, c_i64, c_i64, c_i64, c_void_p, c_void_p, c_void_p, c_i64, P(c_void_p)]),
    "als_csr_upload64": (c_int, [c_void_p, c_i64, c_i64, c_i64, c_void_p, c_void_p, c_int, c_void_p, c_i64, P(c_void_p)]),
    "als_csr_upload_host64": (c_int, [c_void_p, c_i64, c_i64, c_i64, c_void_p, c_void_p, c_int, c_void_p, c_i64,
                                      P(c_void_p)]),
    "als_csr_is_host": (c_int, [c_void_p, P(c_int)]),
    "als_mem_info": (c_int, [c_void_p, P(c_i64), P(c_i64)]),
    "als_ctx_get_knob": (c_int, [c_void_p, ctypes.c_char_p, P(c_int)]),
    "als_csr_segment_count": (c_int, [c_void_p, P(c_i64)]),
    "als_csr_download64": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "als_csr_transpose": (c_int, [c_void_p, c_void_p, P(c_void_p)]),
    "als_csr_generate": (c_int, [c_void_p, c_i64, c_i64, c_i64, ctypes.c_uint64, P(c_void_p)]),
    "als_factors_fill_uniform": (c_int, [c_void_p, c_void_p, ctypes.c_uint64, ctypes.c_float]),
    "als_csr_slice_rows": (c_int, [c_void_p, c_void_p, c_i64, c_i64, P(c_void_p)]),
    "als_csr_scale": (c_int, [c_void_p, c_void_p, c_f32]),
    "als_csr_shape": (c_int, [c_void_p, P(c_i64), P(c_i64), P(c_i64)]),
    "als_csr_download": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "als_csr_destroy": (c_int, [c_void_p]),
    "als_factors_create": (c_int, [c_void_p, c_i64, c_int, P(c_void_p)]),
    "als_factors_upload": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_i64]),
    "als_factors_download": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_i64]),
    "als_factors_shape": (c_int, [c_void_p, P(c_i64), P(c_int), P(c_int)]),
    "als_factors_has_nan": (c_int, [c_void_p, c_void_p, P(c_int)]),
    "als_factors_destroy": (c_int, [c_void_p]),
    "als_ctx_set_knob": (c_int, [c_void_p, ctypes.c_char_p, c_int]),
    "als_gramian": (c_int, [c_void_p, c_void_p, c_void_p]),
    "als_least_squares": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_f64, P(c_i64)]),
    "als_least_squares_with_gramian": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_f64, P(c_i64)]),
    "als_gramian_shard": (c_int, [c_void_p, c_void_p, c_i64, c_i64]),
    "als_gramian_read": (c_int, [c_void_p, c_void_p, c_void_p]),
    "als_least_squares_pregram_async": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_f64]),
    "als_solver_status": (c_int, [c_void_p, P(c_i64), P(c_int)]),
    "als_whitened_factors": (c_int, [c_void_p, c_void_p, c_f64, c_void_p, c_void_p]),
    "als_least_squares_pregram": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_f64, P(c_i64)]),
    "als_least_squares_cg_pregram": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_f32, c_int]),
    "als_least_squares_cg": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_f32, c_int]),
    "als_calculate_loss": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_f32, P(c_f64)]),
    "als_topk": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_int, c_void_p, c_void_p, c_void_p, c_i64,
                         c_void_p, c_void_p]),
    "als_ranking_metrics": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_int, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p]),
    "als_comm_unique_id": (c_int, [c_void_p]),
    "als_comm_init": (c_int, [c_void_p, c_int, c_int, c_void_p]),
    "als_comm_destroy": (c_int, [c_void_p]),
    "als_comm_allgather_rows": (c_int, [c_void_p, c_void_p, c_void_p]),
    "als_factors_ipc_export": (c_int, [c_void_p, c_void_p, c_void_p]),
    "als_factors_ipc_attach": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "als_factors_ipc_detach": (c_int, [c_void_p, c_void_p]),
    "als_comm_allgather_bytes": (c_int, [c_void_p, c_void_p, c_void_p, c_int]),
    "als_comm_allreduce_f64": (c_int, [c_void_p, P(c_f64), c_int, c_int]),
    "als_comm_barrier": (c_int, [c_void_p]),
    "als_mem_peak": (c_int, [c_void_p, P(c_i64), P(c_i64)]),
    "als_csr_column_counts": (c_int, [c_void_p, c_void_p, c_void_p]),
    "als_csr_transpose_pieces": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "als_csr_merge_rows": (c_int, [c_void_p, c_int, c_void_p, c_i64, c_i64, P(c_void_p)]),
    "als_csr_concat_rows": (c_int, [c_void_p, c_int, c_void_p, c_i64, c_i64, P(c_void_p)]),
    "als_comm_allreduce_i64": (c_int, [c_void_p, c_void_p, c_i64]),
    "als_comm_exchange_csr": (c_int, [c_void_p, c_void_p, c_void_p]),
    "als_csr_upload_device": (c_int, [c_void_p, c_i64, c_i64, c_i64, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int,
                                      c_i64, ctypes.c_uint64, P(c_void_p)]),
    "als_factors_import_device": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, ctypes.c_uint64]),
    "als_factors_export_device": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64]),
    "als_device_alloc": (c_int, [c_void_p, c_i64, P(c_void_p)]),
    "als_device_free": (c_int, [c_void_p, c_void_p]),
    "als_pool_alloc": (c_int, [c_void_p, c_i64, P(c_void_p)]),
    "als_pool_free": (c_int, [c_void_p, c_void_p]),
    "als_topk_into": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_i64, c_i64, c_int, c_void_p, c_void_p,
                              c_void_p, c_void_p, c_int, c_i64, c_void_p, c_int, ctypes.c_uint64, c_void_p, c_void_p,
                              P(c_int)]),
    "als_factors_gather_rows": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_i64, ctypes.c_uint64, P(c_void_p),
                                        P(c_int)]),
    "als_device_upload": (c_int, [c_void_p, c_void_p, c_void_p, c_i64]),
    "als_device_download": (c_int, [c_void_p, c_void_p, c_void_p, c_i64]),
    "als_factors_row_norms": (c_int, [c_void_p, c_void_p, c_f32, c_void_p]),
    "als_ids_sort": (c_int, [c_void_p, c_void_p, c_int, c_i64, ctypes.c_uint64, c_void_p]),
    "als_csr_restrict_columns": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_i64, ctypes.c_uint64, P(c_void_p)]),
    "als_ids_range": (c_int, [c_void_p, c_void_p, c_int, c_i64, ctypes.c_uint64, P(c_i64), P(c_i64)]),
    "als_factors_grow": (c_int, [c_void_p, c_void_p, c_i64]),
    "als_factors_scatter_rows": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_i64, ctypes.c_uint64, c_void_p]),
}


class AlsError(RuntimeError):
    """A failing libals_b200 call; .code is the ALS_E_* value."""

    def __init__(self, code, message):
        super().__init__(message)
        self.code = code


_lib = None


def load(build=True):
    """Returns the ctypes library, building it first if needed.  Never falls back to anything else."""
    global _lib
    if _lib is None:
        path = _build.LIB
        override = os.environ.get("ALS_B200_LIB")  # A/B timing of kernel variants (tools/ablate.py)
        if override:
            path = override
        elif build and os.environ.get("ALS_B200_NO_BUILD") != "1":
            path = _build.build()
        if not os.path.exists(path):
            raise ImportError(f"{path} is missing: run `python -m implicit_b200._build` (needs nvcc)")
        lib = ctypes.CDLL(path, mode=ctypes.RTLD_GLOBAL)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError here == header/library mismatch: fail loudly
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = lib
    return _lib


def check(rc):
    if rc != ALS_OK:
        msg = load().als_last_error().decode("utf-8", "replace")
        raise AlsError(rc, msg or f"libals_b200 call failed with code {rc}")


def check_half(rc, bad):
    """check() for a Cholesky half: a row that is not positive definite (its index in `bad`) raises ValueError like
    _als.pyx:136-138."""
    if rc == ALS_E_NOT_POSDEF:
        raise ValueError("cholesky failed on row %i. Try increasing the regularization parameter." % bad.value)
    check(rc)


def ptr(a):
    """Raw data pointer of a C-contiguous numpy array (None -> NULL)."""
    if a is None:
        return None
    assert a.flags.c_contiguous
    return a.ctypes.data_as(c_void_p)


def device_count():
    return load().als_device_count()


class Context:
    """One device context (als_ctx): owns the streams, the Gramian buffers and the communicator."""

    def __init__(self, device=0):
        lib = load()
        n = lib.als_device_count()
        if n <= 0:
            raise AlsError(ALS_E_CUDA, "no CUDA device is visible: implicit_b200 has no CPU path")
        h = c_void_p()
        check(lib.als_ctx_create(int(device), ctypes.byref(h)))
        self.h = h
        self.lib = lib
        self.device = int(device)
        self.rank, self.world = 0, 1

    def close(self):
        if getattr(self, "h", None):
            self.lib.als_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # interpreter shutdown
            pass

    def sync(self):
        check(self.lib.als_sync(self.h))

    def set_knob(self, name, value):
        """Measurement knobs (short_max, short_serial, whiten_fma, gramian_fma, topk_legacy, cg_nv, segment_nnz,
        host_csr); see include/als_b200.h."""
        check(self.lib.als_ctx_set_knob(self.h, name.encode(), int(value)))

    def get_knob(self, name):
        v = c_int()
        check(self.lib.als_ctx_get_knob(self.h, name.encode(), ctypes.byref(v)))
        return v.value

    def mem_info(self):
        """(free, total) device bytes; blocks the context's memory pool keeps for reuse count as free."""
        free, total = c_i64(), c_i64()
        check(self.lib.als_mem_info(self.h, ctypes.byref(free), ctypes.byref(total)))
        return free.value, total.value

    def mem_peak(self):
        """(in use, peak since the previous call) bytes of the device memory pool the library allocates from; the peak
        mark then restarts at the current use."""
        used, peak = c_i64(), c_i64()
        check(self.lib.als_mem_peak(self.h, ctypes.byref(used), ctypes.byref(peak)))
        return used.value, peak.value

    def info(self):
        name = ctypes.create_string_buffer(256)
        sm, l2, mem = c_int(), c_i64(), c_i64()
        check(self.lib.als_device_info(self.h, name, ctypes.byref(sm), ctypes.byref(l2), ctypes.byref(mem)))
        return dict(name=name.value.decode(), sm_count=sm.value, l2_bytes=l2.value, mem_bytes=mem.value)

    def launch_count(self):
        return int(self.lib.als_launch_count(self.h))

    def timer_start(self):
        check(self.lib.als_timer_start(self.h))

    def timer_stop(self):
        ms = c_f32()
        check(self.lib.als_timer_stop(self.h, ctypes.byref(ms)))
        return float(ms.value)

    def flush_l2(self, nbytes=256 << 20):
        check(self.lib.als_flush_l2(self.h, int(nbytes)))

    PROFILE_KINDS = ("gramian", "cholesky", "cholesky_finish", "cg", "cg_giant", "topk", "loss")

    def profile(self, on=True):
        check(self.lib.als_profile_enable(self.h, 1 if on else 0))

    def profile_read(self):
        """{kernel: (total_ms, launches)} since the last read; synchronises the stream."""
        out = {}
        for i, name in enumerate(self.PROFILE_KINDS):
            ms, n = c_f64(), c_i64()
            check(self.lib.als_profile_read(self.h, i, ctypes.byref(ms), ctypes.byref(n)))
            out[name] = (ms.value, n.value)
        return out

    # -- communicator
    def comm_init(self, rank, world, uid):
        check(self.lib.als_comm_init(self.h, int(rank), int(world), ptr(np.frombuffer(uid, dtype=np.uint8))))
        self.rank, self.world = int(rank), int(world)

    def allgather_rows(self, factors, row_splits):
        splits = np.ascontiguousarray(row_splits, dtype=np.int64)
        check(self.lib.als_comm_allgather_rows(self.h, factors.h, ptr(splits)))

    def allgather_bytes(self, payload):
        """Every rank contributes len(payload) <= 256 bytes; returns the concatenation in rank order."""
        send = np.frombuffer(bytes(payload), dtype=np.uint8).copy()
        recv = np.zeros(len(send) * self.world, dtype=np.uint8)
        check(self.lib.als_comm_allgather_bytes(self.h, ptr(send), ptr(recv), len(send)))
        return recv.tobytes()

    def attach_peers(self, factors):
        """Map the other ranks' replicas of `factors` (CUDA IPC over NVLink): from now on every solve that
        writes it mirrors its rows into them, which replaces the all-gather after a half-iteration."""
        h = np.zeros(64, dtype=np.uint8)
        check(self.lib.als_factors_ipc_export(self.h, factors.h, ptr(h)))
        allh = np.frombuffer(self.allgather_bytes(h.tobytes()), dtype=np.uint8).copy()
        check(self.lib.als_factors_ipc_attach(self.h, factors.h, self.rank, self.world, ptr(allh)))

    def detach_peers(self, factors):
        check(self.lib.als_factors_ipc_detach(self.h, factors.h))

    def allreduce(self, values, op="sum"):
        v = np.ascontiguousarray(values, dtype=np.float64).copy()
        check(self.lib.als_comm_allreduce_f64(self.h, v.ctypes.data_as(P(c_f64)), len(v), 1 if op == "max" else 0))
        return v

    def allreduce_i64(self, values):
        """Exact sum of an int64 array of any length over ranks."""
        v = np.ascontiguousarray(values, dtype=np.int64).copy()
        check(self.lib.als_comm_allreduce_i64(self.h, ptr(v), len(v)))
        return v

    def exchange_csr(self, pieces):
        """pieces[q] (one DeviceCSR per rank) goes to rank q; returns the pieces every rank sent here, in rank order."""
        send = (c_void_p * self.world)(*[p.h for p in pieces])
        recv = (c_void_p * self.world)()
        check(self.lib.als_comm_exchange_csr(self.h, send, recv))
        return [DeviceCSR(self, c_void_p(h)) for h in recv]

    def barrier(self):
        check(self.lib.als_comm_barrier(self.h))


# Page-locking memory is slow (cudaMallocHost costs ~0.3 ms per MB), so freed pinned buffers are kept
# in a small pool keyed by size and handed out again: a second fit() downloads its factors into the
# buffers the first one used.
_PINNED_POOL = {}
_PINNED_POOL_BYTES = [0]
_PINNED_POOL_LIMIT = 4 << 30


class _PinnedOwner:
    def __init__(self, ptr, nbytes):
        self.ptr, self.nbytes = ptr, nbytes

    def __del__(self):
        try:
            if _PINNED_POOL_BYTES[0] + self.nbytes <= _PINNED_POOL_LIMIT:
                _PINNED_POOL.setdefault(self.nbytes, []).append(self.ptr)
                _PINNED_POOL_BYTES[0] += self.nbytes
            else:
                load().als_host_free(self.ptr)
        except Exception:  # interpreter shutdown
            pass


def pinned_empty(shape, dtype):
    """numpy array backed by page-locked host memory (cudaMallocHost): H2D / D2H copies of it run at
    full PCIe speed.  The memory returns to a pool when the last view of the array dies."""
    dtype = np.dtype(dtype)
    count = int(np.prod(shape))
    n = max(count * dtype.itemsize, 1)
    free = _PINNED_POOL.get(n)
    if free:
        p = free.pop()
        _PINNED_POOL_BYTES[0] -= n
    else:
        p = c_void_p()
        check(load().als_host_alloc(ctypes.byref(p), n))
    buf = (ctypes.c_char * n).from_address(p.value)
    buf._owner = _PinnedOwner(p, n)  # numpy keeps `buf` alive as the base of every view
    return np.frombuffer(buf, dtype=dtype, count=count).reshape(shape)


def comm_unique_id():
    buf = np.zeros(COMM_ID_BYTES, dtype=np.uint8)
    check(load().als_comm_unique_id(ptr(buf)))
    return buf.tobytes()


#: the largest nnz als_csr_upload takes (int32 positions); above it, als_csr_upload64 stores the CSR as row-block segments
INT32_CSR_MAX_NNZ = 2**31 - 2


def csr_upload_route(nnz):
    """Which upload a CSR of `nnz` nonzeros takes: "int32" (als_csr_upload, int32 host arrays) or "int64"
    (als_csr_upload64: the scipy arrays as they are, int32 or int64, narrowed while they are staged)."""
    return "int32" if nnz <= INT32_CSR_MAX_NNZ else "int64"


#: the segment cap of a host-resident CSR (the default of als_csr_upload_host64): its two-slot device ring takes 4 GB
HOST_SEGMENT_NNZ = 2**28


def _padded_factors(factors):
    return -(-factors // 16) * 16 if factors <= 128 else -(-factors // 128) * 128


def csr_residency(users, items, nnz, factors, free_bytes):
    """Where fit() keeps the pair Cui / Ciu: "device" when everything a device-resident fit allocates fits in
    `free_bytes` of device memory, else "host" (page-locked host memory, streamed through the device per segment).

    Counted: both orientations (int32 index + fp32 value per nonzero, each), the transpose's temporaries (three int32
    arrays and the radix sort's two alternate buffers over the whole matrix, or over one 2^28-nonzero piece when it is
    segmented), the indptrs and launch schedules of both (20 bytes per row, 16 per column count), the factor matrices
    X and Y and the solver's two whitened copies of the larger one, plus 1 GiB for scratch and the pool's
    fragmentation."""
    users, items, nnz, factors = int(users), int(items), int(nnz), int(factors)
    ld = _padded_factors(factors)
    both = 2 * 8 * nnz
    piece = nnz if nnz <= INT32_CSR_MAX_NNZ else min(nnz, HOST_SEGMENT_NNZ)
    transpose = 20 * piece + 16 * (items + 1) * 2
    rows = 20 * (users + items)
    dense = 4 * ld * (users + items) + 2 * 4 * ld * max(users, items)
    need = both + transpose + rows + dense + (1 << 30)
    return "device" if need <= int(free_bytes) else "host"


class DeviceCSR:
    """als_csr: a CSR (or a row shard of one) resident on the device with its launch schedule.  A CSR with more
    nonzeros than the segment cap is held as row-block segments of int32 positions; every call takes it as it is.
    A host-resident CSR (upload(..., host=True)) keeps its indices / values in page-locked host memory and streams
    them through the device segment by segment, with bitwise the results of the device layout of the same cap."""

    def __init__(self, ctx, handle, parent=None):
        self.ctx, self.h, self._parent = ctx, handle, parent

    @classmethod
    def upload(cls, ctx, m, row_offset=0, host=False):
        """m: scipy.sparse.csr_matrix (any float dtype; values are cast to float32).  host: keep it host-resident
        (als_csr_upload_host64)."""
        data = np.ascontiguousarray(m.data, dtype=np.float32)
        h = c_void_p()
        if host or csr_upload_route(m.nnz) == "int64":
            indptr = np.ascontiguousarray(m.indptr, dtype=np.int64)
            indices = m.indices
            if indices.dtype not in (np.int32, np.int64) or not indices.flags.c_contiguous:
                indices = np.ascontiguousarray(indices, dtype=np.int64)
            upload = ctx.lib.als_csr_upload_host64 if host else ctx.lib.als_csr_upload64
            check(upload(ctx.h, m.shape[0], m.shape[1], m.nnz, ptr(indptr), ptr(indices), indices.dtype.itemsize,
                         ptr(data), int(row_offset), ctypes.byref(h)))
            return cls(ctx, h)
        indptr = m.indptr
        if indptr.dtype != np.int32:
            indptr = indptr.astype(np.int32)
        indices = np.ascontiguousarray(m.indices, dtype=np.int32)
        indptr = np.ascontiguousarray(indptr)
        check(ctx.lib.als_csr_upload(ctx.h, m.shape[0], m.shape[1], m.nnz, ptr(indptr), ptr(indices), ptr(data),
                                     int(row_offset), ctypes.byref(h)))
        return cls(ctx, h)

    @classmethod
    def upload_rows(cls, ctx, m, r0, r1):
        """Rows [r0, r1) of the scipy CSR m as a device-resident shard (row_offset = r0), copied straight out of m's
        arrays: no host copy of the rows.  Refuses with ValueError what als_csr_upload64 refuses for these rows (an
        index outside [0, cols), a non-monotone indptr) and an indptr that points past the arrays."""
        r0, r1 = int(r0), int(r1)
        if not 0 <= r0 <= r1 <= m.shape[0]:
            raise ValueError(f"rows [{r0}, {r1}) are not rows of a {m.shape[0]}-row matrix")
        indptr = np.ascontiguousarray(m.indptr[r0:r1 + 1], dtype=np.int64)
        indices = m.indices
        if indices.dtype not in (np.int32, np.int64) or not indices.flags.c_contiguous:
            indices = np.ascontiguousarray(indices, dtype=np.int64)
        data = np.ascontiguousarray(m.data, dtype=np.float32)
        if indptr[0] < 0 or indptr[-1] > min(len(indices), len(data)):
            raise ValueError(f"indptr[{r0}:{r1 + 1}] points outside the {min(len(indices), len(data))} stored entries")
        h = c_void_p()
        rc = ctx.lib.als_csr_upload64(ctx.h, r1 - r0, m.shape[1], int(indptr[-1] - indptr[0]), ptr(indptr), ptr(indices),
                                      indices.dtype.itemsize, ptr(data), r0, ctypes.byref(h))
        if rc == ALS_E_INVALID:
            raise ValueError(ctx.lib.als_last_error().decode("utf-8", "replace"))
        check(rc)
        return cls(ctx, h)

    @classmethod
    def from_device(cls, ctx, m):
        """m: a CSR in CUDA memory (utils.is_device_csr: a CUDA torch.sparse_csr_tensor, or an object with shape and
        indptr / indices / data exposing __cuda_array_interface__, like cupyx.scipy.sparse.csr_matrix), copied into a
        device-resident CSR of the library (als_csr_upload_device) after the work its producer queued on the stream it
        names.  Int32 / int64 indices and fp32 / fp64 values are narrowed on the device.  What als_csr_upload64 refuses,
        and memory that is not on the context's device, raises ValueError."""
        rows, cols, indptr, indices, data, owners = utils.device_csr_arrays(m)
        stream = next(iter({a.stream for a in (indptr, indices, data) if a.stream}), 0)
        h = c_void_p()
        rc = ctx.lib.als_csr_upload_device(ctx.h, rows, cols, len(indices), indptr.ptr, indptr.itemsize, indices.ptr or None,
                                           indices.itemsize, data.ptr or None, data.itemsize, 0, stream, ctypes.byref(h))
        del owners  # the call has read the arrays
        if rc == ALS_E_INVALID:
            raise ValueError(ctx.lib.als_last_error().decode("utf-8", "replace"))
        check(rc)
        return cls(ctx, h)

    def restrict_columns(self, subset):
        """The liked CSR remapped onto the positions of `subset` (a utils.CudaArray sorted ascending), the device
        counterpart of als._filter_items_from_sparse_matrix (als_csr_restrict_columns)."""
        h = c_void_p()
        _check_input(self.ctx, self.ctx.lib.als_csr_restrict_columns(self.ctx.h, self.h, subset.ptr or None,
                                                                     subset.itemsize, len(subset), subset.stream,
                                                                     ctypes.byref(h)))
        return DeviceCSR(self.ctx, h)

    def column_counts(self):
        """int64 entries per column."""
        counts = np.zeros(self.shape3[1], dtype=np.int64)
        check(self.ctx.lib.als_csr_column_counts(self.ctx.h, self.h, ptr(counts)))
        return counts

    def transpose_pieces(self, col_bounds):
        """The transpose of this (device-resident) shard cut at col_bounds[0 = b_0 <= ... <= b_n = cols]: n CSRs, the
        q-th of rows [b_q, b_q+1) of the transpose, with global row ids as column indices."""
        bounds = np.ascontiguousarray(col_bounds, dtype=np.int64)
        n = len(bounds) - 1
        out = (c_void_p * n)()
        check(self.ctx.lib.als_csr_transpose_pieces(self.ctx.h, self.h, n, ptr(bounds), out))
        return [DeviceCSR(self.ctx, c_void_p(h)) for h in out]

    @classmethod
    def merge_rows(cls, ctx, pieces, cols, row_offset):
        """The pieces (equal row counts) concatenated row by row, in list order, as a shard of `cols` columns."""
        arr = (c_void_p * len(pieces))(*[p.h for p in pieces])
        h = c_void_p()
        check(ctx.lib.als_csr_merge_rows(ctx.h, len(pieces), arr, int(cols), int(row_offset), ctypes.byref(h)))
        return cls(ctx, h)

    @classmethod
    def concat_rows(cls, ctx, pieces, cols, row_offset):
        """The pieces (any row counts) stacked in list order, piece 0's rows first, as a shard of `cols` columns."""
        arr = (c_void_p * len(pieces))(*[p.h for p in pieces])
        h = c_void_p()
        check(ctx.lib.als_csr_concat_rows(ctx.h, len(pieces), arr, int(cols), int(row_offset), ctypes.byref(h)))
        return cls(ctx, h)

    @property
    def segment_count(self):
        """Row-block segments of the device layout (1 unless nnz exceeds the segment cap)."""
        n = c_i64()
        check(self.ctx.lib.als_csr_segment_count(self.h, ctypes.byref(n)))
        return n.value

    @property
    def host_resident(self):
        """True when indices / values live in page-locked host memory (als_csr_upload_host64 or its transpose)."""
        v = c_int()
        check(self.ctx.lib.als_csr_is_host(self.h, ctypes.byref(v)))
        return bool(v.value)

    def transpose(self):
        h = c_void_p()
        check(self.ctx.lib.als_csr_transpose(self.ctx.h, self.h, ctypes.byref(h)))
        return DeviceCSR(self.ctx, h)

    @classmethod
    def generate(cls, ctx, rows, cols, nnz, seed):
        """Power-law CSR built on the device (csrc/gen.cu): for configurations too large for the host generator."""
        h = c_void_p()
        check(ctx.lib.als_csr_generate(ctx.h, int(rows), int(cols), int(nnz), int(seed), ctypes.byref(h)))
        return cls(ctx, h)

    def slice_rows(self, r0, r1):
        h = c_void_p()
        check(self.ctx.lib.als_csr_slice_rows(self.ctx.h, self.h, int(r0), int(r1), ctypes.byref(h)))
        return DeviceCSR(self.ctx, h, parent=self)

    def scale(self, alpha):
        check(self.ctx.lib.als_csr_scale(self.ctx.h, self.h, float(alpha)))

    @property
    def shape3(self):
        r, c, n = c_i64(), c_i64(), c_i64()
        check(self.ctx.lib.als_csr_shape(self.h, ctypes.byref(r), ctypes.byref(c), ctypes.byref(n)))
        return r.value, c.value, n.value

    def download(self):
        import scipy.sparse as sp

        rows, cols, nnz = self.shape3
        indptr = self.indptr_host()
        indices = np.zeros(nnz, dtype=np.int32)
        data = np.zeros(nnz, dtype=np.float32)
        check(self.ctx.lib.als_csr_download64(self.ctx.h, self.h, None, ptr(indices), ptr(data)))
        return sp.csr_matrix((data, indices, indptr), shape=(rows, cols))

    def indptr_host(self):
        """int32, or int64 when nnz >= 2^31 (like scipy)."""
        rows, _, nnz = self.shape3
        if nnz >= 2**31:
            indptr = np.zeros(rows + 1, dtype=np.int64)
            check(self.ctx.lib.als_csr_download64(self.ctx.h, self.h, ptr(indptr), None, None))
            return indptr
        indptr = np.zeros(rows + 1, dtype=np.int32)
        check(self.ctx.lib.als_csr_download(self.ctx.h, self.h, ptr(indptr), None, None))
        return indptr

    def close(self):
        if getattr(self, "h", None) and getattr(self.ctx, "h", None):
            self.ctx.lib.als_csr_destroy(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DeviceFactors:
    """als_factors: a dense float32 [rows, factors] matrix on the device."""

    def __init__(self, ctx, rows, factors):
        h = c_void_p()
        check(ctx.lib.als_factors_create(ctx.h, int(rows), int(factors), ctypes.byref(h)))
        self.ctx, self.h, self.rows, self.factors = ctx, h, int(rows), int(factors)

    @classmethod
    def from_host(cls, ctx, a):
        a = np.ascontiguousarray(a, dtype=np.float32)
        f = cls(ctx, a.shape[0], a.shape[1])
        f.upload(a)
        return f

    def upload(self, a, row0=0):
        a = np.ascontiguousarray(a, dtype=np.float32)
        assert a.ndim == 2 and a.shape[1] == self.factors
        check(self.ctx.lib.als_factors_upload(self.ctx.h, self.h, ptr(a), int(row0), a.shape[0]))

    @classmethod
    def from_cuda(cls, ctx, obj, what="factors"):
        """A new matrix filled device to device from a CUDA float32 2-D array (__cuda_array_interface__; rows may be
        strided, like t[:, :f] of a wider tensor), after the work its producer queued on the stream it names.  ValueError
        for what utils.parse_cai refuses and for memory that is not on the context's device."""
        a = utils.cuda_array(obj, what, ("<f4",), 2)
        f = cls(ctx, a.shape[0], a.shape[1])
        try:
            rc = ctx.lib.als_factors_import_device(ctx.h, f.h, a.ptr or None, a.ld, 0, a.shape[0], a.stream)
            if rc == ALS_E_INVALID:
                raise ValueError(ctx.lib.als_last_error().decode("utf-8", "replace"))
            check(rc)
        except BaseException:
            f.close()
            raise
        return f

    def snapshot(self):
        """A DeviceSnapshot: a copy of this matrix in device memory of its own."""
        return DeviceSnapshot.of_factors(self)

    @classmethod
    def gather_rows(cls, ctx, src, rows):
        """A new matrix of the rows src[rows] (rows: a utils.CudaArray of int32 / int64 ids), after the work its producer
        queued on the stream it names.  None when some id is outside [0, src.rows) (nothing is created); ValueError for
        memory that is not on the context's device."""
        h, bad = c_void_p(), c_int(0)
        rc = ctx.lib.als_factors_gather_rows(ctx.h, src.h, rows.ptr or None, rows.itemsize, len(rows), rows.stream,
                                             ctypes.byref(h), ctypes.byref(bad))
        if bad.value:
            return None
        _check_input(ctx, rc)
        f = cls.__new__(cls)
        f.ctx, f.h, f.rows, f.factors = ctx, h, len(rows), src.factors
        return f

    def grow(self, rows):
        """Grows the matrix to `rows` rows on the device (als_factors_grow): the old rows are kept, the new ones are zero.
        ValueError, the matrix unchanged, for more rows than the device's memory holds."""
        rows = min(int(rows), 2**63 - 1)  # max id + 1 of int64 ids: past any device, and still an int64
        _check_input(self.ctx, self.ctx.lib.als_factors_grow(self.ctx.h, self.h, rows))
        self.rows = int(rows)

    def scatter_rows(self, ids, src):
        """self[ids] = src on the device (als_factors_scatter_rows): ids a utils.CudaArray of src.rows int32 / int64
        ids inside the matrix, read after the work its producer queued on the stream it names; of a repeated id the last
        occurrence wins, as in numpy."""
        _check_input(self.ctx, self.ctx.lib.als_factors_scatter_rows(self.ctx.h, self.h, ids.ptr or None, ids.itemsize,
                                                                     len(ids), ids.stream, src.h))

    def row_norms(self, zero_value=1e-10):
        """A DeviceSnapshot [rows] '<f4' of the row norms, bitwise np.linalg.norm(F, axis=-1) with zeros written as
        float32(zero_value) (the `n[n == 0] = 1e-10` of the user_norms / item_norms properties)."""
        out = DeviceSnapshot(self.ctx, (self.rows,), "<f4")
        check(self.ctx.lib.als_factors_row_norms(self.ctx.h, self.h, float(zero_value), out.ptr))
        return out

    def fill_uniform(self, seed, scale):
        """factors = scale * U[0,1) generated on the device (the distribution of implicit/cpu/als.py:144-147)."""
        check(self.ctx.lib.als_factors_fill_uniform(self.ctx.h, self.h, int(seed), float(scale)))

    def has_nan(self):
        flag = c_int(0)
        check(self.ctx.lib.als_factors_has_nan(self.ctx.h, self.h, ctypes.byref(flag)))
        return bool(flag.value)

    def download(self, row0=0, nrows=None, pinned=False):
        nrows = self.rows - row0 if nrows is None else nrows
        out = (pinned_empty if pinned else np.empty)((nrows, self.factors), dtype=np.float32)
        check(self.ctx.lib.als_factors_download(self.ctx.h, self.h, ptr(out), int(row0), int(nrows)))
        return out

    def close(self):
        if getattr(self, "h", None) and getattr(self.ctx, "h", None):
            self.ctx.lib.als_factors_destroy(self.h)
        self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DeviceSnapshot:
    """A 1-D or 2-D array in device memory the library allocated for it alone (als_device_alloc), complete when it is
    handed out, exposed through __cuda_array_interface__ version 3: `shape`, `typestr`, rows `ld` elements apart (2-D),
    no stream to wait for.  The factor snapshots (of_factors) are '<f4' rows of the padded width; the outputs of the
    device serving calls are contiguous ids and scores.  torch.as_tensor(s, device="cuda") and cupy.asarray(s) keep the
    object, and so its memory, alive; the memory is freed (cudaFree, after every stream's work) when the last reference
    dies, and outlives the model and the context object that made it.  `pooled`: a temporary of the library's own calls
    (als_pool_alloc), read only on the context's stream and closed by the caller; no wait for the device to free it."""

    def __init__(self, ctx, shape, typestr, ld=None, pooled=False):
        self.ctx, self.shape, self.typestr, self.pooled = ctx, tuple(int(n) for n in shape), typestr, pooled
        self.itemsize = int(typestr[2:])
        self.ld = self.shape[-1] if ld is None else int(ld)
        count = self.shape[0] * (self.ld if len(self.shape) == 2 else 1)
        self.ptr = c_void_p()
        alloc = ctx.lib.als_pool_alloc if pooled else ctx.lib.als_device_alloc
        check(alloc(ctx.h, self.itemsize * count, ctypes.byref(self.ptr)))

    @classmethod
    def of_factors(cls, factors):
        """A copy of a DeviceFactors matrix: shape (rows, factors), row stride the padded width."""
        ctx = factors.ctx
        rows, f, ld = c_i64(), c_int(), c_int()
        check(ctx.lib.als_factors_shape(factors.h, ctypes.byref(rows), ctypes.byref(f), ctypes.byref(ld)))
        s = cls(ctx, (rows.value, f.value), "<f4", ld.value)
        try:
            check(ctx.lib.als_factors_export_device(ctx.h, factors.h, s.ptr, s.ld, 0, rows.value))
        except BaseException:
            s.close()
            raise
        return s

    @classmethod
    def from_host(cls, ctx, a, pooled=False):
        """A 1-D copy of the contiguous numpy array a ('<i4', '<i8' or '<f4')."""
        a = np.ascontiguousarray(a)
        s = cls(ctx, a.shape, a.dtype.str, pooled=pooled)
        try:
            check(ctx.lib.als_device_upload(ctx.h, s.ptr, ptr(a) if a.size else None, a.nbytes))
        except BaseException:
            s.close()
            raise
        return s

    def cuda(self, row0=0):
        """This array from row `row0` on as a utils.CudaArray (no stream to wait for)."""
        step = self.itemsize * (self.ld if len(self.shape) == 2 else 1)
        return utils.CudaArray(self.ptr.value + step * row0, (self.shape[0] - row0,) + self.shape[1:], self.itemsize,
                               self.ld, 0)

    @property
    def __cuda_array_interface__(self):
        strides = (self.itemsize * self.ld, self.itemsize) if len(self.shape) == 2 else None
        return {"shape": self.shape, "strides": strides, "typestr": self.typestr, "data": (self.ptr.value, False),
                "version": 3, "stream": None}

    def close(self):
        if getattr(self, "ptr", None) and getattr(self.ctx, "h", None):
            (self.ctx.lib.als_pool_free if self.pooled else self.ctx.lib.als_device_free)(self.ctx.h, self.ptr)
        self.ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # interpreter shutdown
            pass


def _check_input(ctx, rc):
    """check(), with ALS_E_INVALID (a refused argument) raised as ValueError."""
    if rc == ALS_E_INVALID:
        raise ValueError(ctx.lib.als_last_error().decode("utf-8", "replace"))
    check(rc)


def ids_download(ctx, ids):
    """The utils.CudaArray ids as a numpy array of their width (int32 / int64)."""
    out = np.empty(len(ids), dtype=np.int32 if ids.itemsize == 4 else np.int64)
    _check_input(ctx, ctx.lib.als_device_download(ctx.h, ptr(out) if out.size else None, ids.ptr or None, out.nbytes))
    return out


def ids_sort(ctx, ids):
    """A pooled DeviceSnapshot of the utils.CudaArray ids sorted ascending on the device, of the same width."""
    out = DeviceSnapshot(ctx, ids.shape, f"<i{ids.itemsize}", pooled=True)
    try:
        _check_input(ctx, ctx.lib.als_ids_sort(ctx.h, ids.ptr or None, ids.itemsize, len(ids), ids.stream, out.ptr))
    except BaseException:
        out.close()
        raise
    return out


def ids_range(ctx, ids):
    """(min, max) of the utils.CudaArray ids, read after the work its producer queued on the stream it names: one pass and
    one 16-byte read-back (als_ids_range).  (0, -1) for no ids."""
    lo, hi = c_i64(), c_i64()
    _check_input(ctx, ctx.lib.als_ids_range(ctx.h, ids.ptr or None, ids.itemsize, len(ids), ids.stream, ctypes.byref(lo),
                                            ctypes.byref(hi)))
    return lo.value, hi.value


# ---- the native operator interface, named like the reference's (implicit/cpu/_als.pyx, topk.pyx) ----
def gramian(ctx, Y):
    G = np.empty((Y.factors, Y.factors), dtype=np.float32)
    check(ctx.lib.als_gramian(ctx.h, Y.h, ptr(G)))
    return G


def least_squares(ctx, Cui, X, Y, regularization):
    """_als.least_squares(Cui, X, Y, regularization): raises ValueError like _als.pyx:136-138."""
    bad = c_i64(-1)
    rc = ctx.lib.als_least_squares(ctx.h, Cui.h, X.h, Y.h, float(regularization), ctypes.byref(bad))
    check_half(rc, bad)


def whitened_factors(ctx, Y, regularization):
    """(W, Z) of the short-row path: W = Y P (P = R^-1, Y^T Y + reg I = R^T R) and Z = Y (Y^T Y + reg I)^-1."""
    W = np.empty((Y.rows, Y.factors), dtype=np.float32)
    Z = np.empty((Y.rows, Y.factors), dtype=np.float32)
    check(ctx.lib.als_whitened_factors(ctx.h, Y.h, float(regularization), ptr(W), ptr(Z)))
    return W, Z


def gramian_shard(ctx, Y, row0, nrows):
    """Gramian over this rank's rows of Y, summed across ranks, left on the device for the *_pregram solves."""
    check(ctx.lib.als_gramian_shard(ctx.h, Y.h, int(row0), int(nrows)))


def gramian_read(ctx, Y):
    """The Gramian the context holds from the last gramian / gramian_shard on Y, downloaded."""
    G = np.empty((Y.factors, Y.factors), dtype=np.float32)
    check(ctx.lib.als_gramian_read(ctx.h, Y.h, ptr(G)))
    return G


def half_pregram_async(ctx, Cui, X, Y, regularization, use_cg, cg_steps=3):
    """half_pregram without the host round trip: failures surface in solver_status()."""
    if use_cg:
        check(ctx.lib.als_least_squares_cg_pregram(ctx.h, Cui.h, X.h, Y.h, float(regularization), int(cg_steps)))
    else:
        check(ctx.lib.als_least_squares_pregram_async(ctx.h, Cui.h, X.h, Y.h, float(regularization)))


def solver_status(ctx):
    """Synchronises; raises ValueError for a bad row of this rank, AlsError when another rank failed."""
    bad, anyf = c_i64(-1), c_int(0)
    rc = ctx.lib.als_solver_status(ctx.h, ctypes.byref(bad), ctypes.byref(anyf))
    check_half(rc, bad)
    if anyf.value:
        raise AlsError(ALS_E_NOT_POSDEF, "another rank failed in this iteration (see its error message)")


def half_pregram(ctx, Cui, X, Y, regularization, use_cg, cg_steps=3):
    """One half-iteration with the device-resident (already all-reduced) Gramian."""
    if use_cg:
        check(ctx.lib.als_least_squares_cg_pregram(ctx.h, Cui.h, X.h, Y.h, float(regularization), int(cg_steps)))
        return
    bad = c_i64(-1)
    rc = ctx.lib.als_least_squares_pregram(ctx.h, Cui.h, X.h, Y.h, float(regularization), ctypes.byref(bad))
    check_half(rc, bad)


def least_squares_with_gramian(ctx, YtY, Cui, X, Y, regularization):
    """_als._least_squares(YtY, indptr, indices, data, X, Y, regularization)"""
    YtY = np.ascontiguousarray(YtY, dtype=np.float32)
    bad = c_i64(-1)
    rc = ctx.lib.als_least_squares_with_gramian(ctx.h, ptr(YtY), Cui.h, X.h, Y.h, float(regularization),
                                                ctypes.byref(bad))
    check_half(rc, bad)


def least_squares_cg(ctx, Cui, X, Y, regularization, cg_steps=3):
    check(ctx.lib.als_least_squares_cg(ctx.h, Cui.h, X.h, Y.h, float(regularization), int(cg_steps)))


def loss_terms(ctx, Cui, X, Y, regularization):
    t = (c_f64 * 3)()
    check(ctx.lib.als_calculate_loss(ctx.h, Cui.h, X.h, Y.h, float(regularization), t))
    return np.array([t[0], t[1], t[2]], dtype=np.float64)


def calculate_loss(ctx, Cui, X, Y, regularization):
    """_als.calculate_loss for an unsharded Cui."""
    rows, cols, nnz = Cui.shape3
    t = loss_terms(ctx, Cui, X, Y, regularization)
    return float((t[0] + t[2]) / (t[1] + float(rows) * float(cols) - float(nnz)))


def topk(ctx, items, queries, k, query_rows=None, n_query=None, item_norms=None, liked=None, filter_items=None):
    """topk.topk(items, query, k, item_norms, filter_query_items, filter_items) on device handles."""
    if query_rows is not None:
        query_rows = np.ascontiguousarray(query_rows, dtype=np.int32)
        n_query = len(query_rows)
    elif n_query is None:
        n_query = queries.rows
    ids = np.zeros((n_query, k), dtype=np.int32)
    scores = np.zeros((n_query, k), dtype=np.float32)
    norms = None if item_norms is None else np.ascontiguousarray(item_norms, dtype=np.float32)
    fl = None
    if filter_items is not None:
        fl = np.ascontiguousarray(np.asarray(filter_items).ravel(), dtype=np.int32)
    check(ctx.lib.als_topk(ctx.h, items.h, queries.h, ptr(query_rows), int(n_query), int(k), ptr(norms),
                           liked.h if liked is not None else None, ptr(fl), 0 if fl is None else len(fl),
                           ptr(ids), ptr(scores)))
    return ids, scores


def topk_into(ctx, items, queries, k, n_query, ids, scores, query_rows=None, query_row0=0, item_norms=None,
              query_norms=None, liked=None, filter_items=None, id_map=None, stream=0):
    """als_topk_into: the top-k of topk() written to the device arrays ids / scores (utils.CudaArrays of n_query rows of
    k), every other id or norm array a utils.CudaArray too (query_rows None: rows [query_row0, query_row0 + n_query) of
    queries).  Returns 0, or the bits of the device ids that were out of range (1: query_rows, 2: filter_items), in
    which case nothing was written."""
    def arr(a):
        return (a.ptr or None, a.itemsize) if a is not None else (None, 4)

    qr, qb = arr(query_rows)
    fl, fb = arr(filter_items)
    mp, mb = arr(id_map)
    bad = c_int(0)
    rc = ctx.lib.als_topk_into(ctx.h, items.h, queries.h, qr, qb, int(query_row0), int(n_query), int(k),
                               item_norms.ptr if item_norms is not None else None,
                               query_norms.ptr if query_norms is not None else None,
                               liked.h if liked is not None else None, fl, fb,
                               0 if filter_items is None else len(filter_items), mp, mb, int(stream), ids.ptr or None,
                               scores.ptr or None, ctypes.byref(bad))
    if bad.value:
        return bad.value
    _check_input(ctx, rc)
    return 0


def ranking_metrics(ctx, items, queries, k, query_rows, test, gain, gain_sum, liked=None):
    """The six fp64 sums of ranking_metrics_at_k (hits, sum min(K, L), AP, nDCG, AUC, users) over the queries
    `query_rows` of `queries`, scored against `test` (a DeviceCSR over those rows) on the device."""
    query_rows = np.ascontiguousarray(query_rows, dtype=np.int32)
    gain = np.ascontiguousarray(gain, dtype=np.float64)
    gain_sum = np.ascontiguousarray(gain_sum, dtype=np.float64)
    sums = np.zeros(6, dtype=np.float64)
    check(ctx.lib.als_ranking_metrics(ctx.h, items.h, queries.h, ptr(query_rows), len(query_rows), int(k),
                                      liked.h if liked is not None else None, test.h, ptr(gain), ptr(gain_sum), ptr(sums)))
    return sums
