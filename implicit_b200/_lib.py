"""ctypes binding of libals_b200.so (include/als_b200.h) -- the only way Python reaches the GPU here.

There is deliberately no fallback: if the shared library is missing it is built with nvcc; if that
fails, or there is no H100 to run on, the caller gets an exception.
"""
import ctypes
import os

import numpy as np

from . import _build

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
    "als_least_squares_pregram_async": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_f64]),
    "als_solver_status": (c_int, [c_void_p, P(c_i64), P(c_int)]),
    "als_whitened_factors": (c_int, [c_void_p, c_void_p, c_f64, c_void_p, c_void_p]),
    "als_least_squares_pregram": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_f64, P(c_i64)]),
    "als_least_squares_cg_pregram": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_f32, c_int]),
    "als_least_squares_cg": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_f32, c_int]),
    "als_calculate_loss": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_f32, P(c_f64)]),
    "als_topk": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_int, c_void_p, c_void_p, c_void_p, c_i64,
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
    def upload(cls, ctx, m, row_offset=0, rows=None, host=False):
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
        download = self.ctx.lib.als_csr_download64 if indptr.dtype == np.int64 else self.ctx.lib.als_csr_download
        check(download(self.ctx.h, self.h, None, ptr(indices), ptr(data)))
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


# ---- the native operator interface, named like the reference's (implicit/cpu/_als.pyx, topk.pyx) ----
def gramian(ctx, Y):
    G = np.empty((Y.factors, Y.factors), dtype=np.float32)
    check(ctx.lib.als_gramian(ctx.h, Y.h, ptr(G)))
    return G


def least_squares(ctx, Cui, X, Y, regularization):
    """_als.least_squares(Cui, X, Y, regularization): raises ValueError like _als.pyx:136-138."""
    bad = c_i64(-1)
    rc = ctx.lib.als_least_squares(ctx.h, Cui.h, X.h, Y.h, float(regularization), ctypes.byref(bad))
    if rc == ALS_E_NOT_POSDEF:
        raise ValueError("cholesky failed on row %i. Try increasing the regularization parameter." % bad.value)
    check(rc)


def whitened_factors(ctx, Y, regularization):
    """(W, Z) of the short-row path: W = Y P (P = R^-1, Y^T Y + reg I = R^T R) and Z = Y (Y^T Y + reg I)^-1."""
    W = np.empty((Y.rows, Y.factors), dtype=np.float32)
    Z = np.empty((Y.rows, Y.factors), dtype=np.float32)
    check(ctx.lib.als_whitened_factors(ctx.h, Y.h, float(regularization), ptr(W), ptr(Z)))
    return W, Z


def gramian_shard(ctx, Y, row0, nrows):
    """Gramian over this rank's rows of Y, summed across ranks, left on the device for the *_pregram solves."""
    check(ctx.lib.als_gramian_shard(ctx.h, Y.h, int(row0), int(nrows)))


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
    if rc == ALS_E_NOT_POSDEF:
        raise ValueError("cholesky failed on row %i. Try increasing the regularization parameter." % bad.value)
    check(rc)
    if anyf.value:
        raise AlsError(ALS_E_NOT_POSDEF, "another rank failed in this iteration (see its error message)")


def half_pregram(ctx, Cui, X, Y, regularization, use_cg, cg_steps=3):
    """One half-iteration with the device-resident (already all-reduced) Gramian."""
    if use_cg:
        check(ctx.lib.als_least_squares_cg_pregram(ctx.h, Cui.h, X.h, Y.h, float(regularization), int(cg_steps)))
        return
    bad = c_i64(-1)
    rc = ctx.lib.als_least_squares_pregram(ctx.h, Cui.h, X.h, Y.h, float(regularization), ctypes.byref(bad))
    if rc == ALS_E_NOT_POSDEF:
        raise ValueError("cholesky failed on row %i. Try increasing the regularization parameter." % bad.value)
    check(rc)


def least_squares_with_gramian(ctx, YtY, Cui, X, Y, regularization):
    """_als._least_squares(YtY, indptr, indices, data, X, Y, regularization)"""
    YtY = np.ascontiguousarray(YtY, dtype=np.float32)
    bad = c_i64(-1)
    rc = ctx.lib.als_least_squares_with_gramian(ctx.h, ptr(YtY), Cui.h, X.h, Y.h, float(regularization),
                                                ctypes.byref(bad))
    if rc == ALS_E_NOT_POSDEF:
        raise ValueError("cholesky failed on row %i. Try increasing the regularization parameter." % bad.value)
    check(rc)


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
