"""Input-handling helpers with the reference's semantics (implicit/utils.py:65-83, :155-169;
implicit/recommender_base.py:9)."""
import time
import warnings

import numpy as np
import scipy.sparse


class ParameterWarning(Warning):
    """implicit/utils.py:155"""


class ModelFitError(Exception):
    """implicit/recommender_base.py:9"""


def check_csr(user_items):
    """implicit/utils.py:159-169: non-CSR input is converted with a ParameterWarning."""
    if not isinstance(user_items, scipy.sparse.csr_matrix):
        class_name = user_items.__class__.__name__
        start = time.time()
        user_items = user_items.tocsr()
        warnings.warn(
            f"Method expects CSR input, and was passed {class_name} instead. "
            f"Converting to CSR took {time.time() - start} seconds",
            ParameterWarning,
        )
    return user_items


class CudaArray:
    """One array of device memory, read from its __cuda_array_interface__ (parse_cai): the address, the shape, the item
    size, the row stride in elements (2-D) and the stream its producer queued it on (0: no ordering needed)."""

    def __init__(self, ptr, shape, itemsize, ld, stream):
        self.ptr, self.shape, self.itemsize, self.ld, self.stream = ptr, shape, itemsize, ld, stream

    def __len__(self):
        return self.shape[0]


def parse_cai(cai, what, typestrs, ndim):
    """The CudaArray a __cuda_array_interface__ dict (version 2 or 3) describes, or ValueError, before its pointer is used:
    a version other than 2 or 3, a mask, a typestr outside `typestrs`, a shape of other than `ndim` dimensions, strides
    other than contiguous (1-D) or row-strided with unit column stride (2-D), or a stream entry of 0, which the interface
    forbids.  Version 3's stream (1: the legacy default stream, 2: the per-thread one, else a cudaStream_t) is the stream
    to order after; an absent or None stream needs no ordering.  Version 2 cannot name a stream: its arrays are ordered
    after the legacy default stream, where PyTorch and CuPy queue their work unless told otherwise."""
    if not isinstance(cai, dict):
        raise ValueError(f"{what}: __cuda_array_interface__ is not a dict")
    version = cai.get("version")
    if version not in (2, 3):
        raise ValueError(f"{what}: __cuda_array_interface__ version {version!r} is not supported (2 or 3)")
    if cai.get("mask") is not None:
        raise ValueError(f"{what}: masked arrays are not supported")
    typestr = cai.get("typestr")
    if typestr not in typestrs:
        raise ValueError(f"{what}: typestr {typestr!r} is not one of {', '.join(typestrs)}")
    itemsize = int(typestr[2:])
    shape = cai.get("shape")
    if not isinstance(shape, tuple) or len(shape) != ndim or not all(isinstance(n, int) and n >= 0 for n in shape):
        raise ValueError(f"{what}: shape {shape!r} is not a {ndim}-D shape")
    strides = cai.get("strides")
    ld = shape[-1] if ndim == 2 else 1
    if strides is not None:
        if not isinstance(strides, tuple) or len(strides) != ndim or not all(isinstance(s, int) for s in strides):
            raise ValueError(f"{what}: strides {strides!r} do not match the shape {shape!r}")
        if ndim == 1 and shape[0] > 1 and strides[0] != itemsize:
            raise ValueError(f"{what}: a 1-D array of stride {strides[0]} bytes is not contiguous")
        if ndim == 2:
            if shape[1] > 1 and strides[1] != itemsize:
                raise ValueError(f"{what}: column stride {strides[1]} bytes: the rows must be contiguous")
            if shape[0] > 1 and (strides[0] % itemsize or strides[0] < shape[1] * itemsize):
                raise ValueError(f"{what}: row stride {strides[0]} bytes is not a whole number of elements at least a row "
                                 f"of {shape[1]} long")
            if shape[0] > 1:
                ld = strides[0] // itemsize
    data = cai.get("data")
    if not isinstance(data, tuple) or len(data) != 2 or not isinstance(data[0], int):
        raise ValueError(f"{what}: data {data!r} is not a (pointer, read-only) pair")
    if data[0] == 0 and all(shape):
        raise ValueError(f"{what}: NULL pointer for a non-empty array")
    if version == 2:
        stream = 1
    else:
        stream = cai.get("stream")
        if stream is None:
            stream = 0
        elif not isinstance(stream, int) or stream == 0:
            raise ValueError(f"{what}: stream {stream!r} is not a stream (0 is forbidden; None means no ordering)")
    return CudaArray(int(data[0]), shape, itemsize, ld, int(stream))


def cuda_array(obj, what, typestrs, ndim):
    """parse_cai of obj.__cuda_array_interface__; ValueError when obj has none (host memory)."""
    cai = getattr(obj, "__cuda_array_interface__", None)
    if cai is None:
        raise ValueError(f"{what}: {type(obj).__name__} does not expose __cuda_array_interface__ (not CUDA memory)")
    return parse_cai(cai, what, typestrs, ndim)


def is_cuda_array(obj):
    """True when obj exposes __cuda_array_interface__ (a CUDA torch tensor, a CuPy array, ...): recommend, rank_items
    and similar_* take their device path for ids given this way."""
    return not isinstance(obj, np.ndarray) and hasattr(obj, "__cuda_array_interface__")


ID_TYPESTRS = ("<i4", "<i8")


def cuda_ids(obj, what):
    """The CudaArray of a 1-D int32 / int64 array of ids in CUDA memory; ValueError, naming `what`, for another typestr
    (float ids), another number of dimensions and whatever parse_cai refuses."""
    return cuda_array(obj, what, ID_TYPESTRS, 1)


def _is_torch_sparse_csr(m):
    return str(getattr(m, "layout", "")) == "torch.sparse_csr" and callable(getattr(m, "crow_indices", None))


def is_device_csr(m):
    """A CSR whose arrays are in CUDA memory: a torch.sparse_csr_tensor (by its layout name), or any object with `shape`
    and indptr / indices / data attributes that expose __cuda_array_interface__ (cupyx.scipy.sparse.csr_matrix)."""
    if _is_torch_sparse_csr(m):
        return True
    return hasattr(m, "shape") and all(hasattr(getattr(m, a, None), "__cuda_array_interface__")
                                       for a in ("indptr", "indices", "data"))


INDEX_TYPESTRS = ("<i4", "<i8")
VALUE_TYPESTRS = ("<f4", "<f8")


def device_csr_arrays(m):
    """(rows, cols, indptr, indices, data, owners) of a device CSR (is_device_csr): the three CudaArrays and the objects
    that own their memory, to be held until the upload returns.  ValueError for what parse_cai refuses, for arrays whose
    lengths do not fit the shape and for arrays that name different streams."""
    if _is_torch_sparse_csr(m):
        owners = (m.crow_indices(), m.col_indices(), m.values())
    else:
        owners = (m.indptr, m.indices, m.data)
    shape = tuple(int(n) for n in m.shape)
    if len(shape) != 2:
        raise ValueError(f"a device CSR must be 2-D, got shape {shape}")
    rows, cols = shape
    indptr = cuda_array(owners[0], "indptr", INDEX_TYPESTRS, 1)
    indices = cuda_array(owners[1], "indices", INDEX_TYPESTRS, 1)
    data = cuda_array(owners[2], "data", VALUE_TYPESTRS, 1)
    if len(indptr) != rows + 1:
        raise ValueError(f"indptr has {len(indptr)} entries, the {rows} rows need {rows + 1}")
    if len(indices) != len(data):
        raise ValueError(f"indices has {len(indices)} entries and data {len(data)}")
    streams = {a.stream for a in (indptr, indices, data) if a.stream}
    if len(streams) > 1:
        raise ValueError("the arrays of a device CSR name different streams")
    return rows, cols, indptr, indices, data, owners


def check_random_state(random_state):
    """implicit/utils.py:65-83: int / None / RandomState / Generator -> np.random.Generator."""
    if isinstance(random_state, np.random.RandomState):
        return np.random.default_rng(random_state.randint(2**31))
    return np.random.default_rng(random_state)


def nnz_balanced_splits(indptr, parts, row_cost=0):
    """Row boundaries [0 = s_0 <= ... <= s_parts = rows] giving every part the same share of
    nnz + row_cost * rows (SURVEY.md section 8(e): nnz-balanced, not row-balanced, shards; row_cost adds the
    per-row fixed work -- the factorisation -- in units of nonzeros)."""
    indptr = np.asarray(indptr, dtype=np.int64)
    rows = len(indptr) - 1
    if row_cost:
        indptr = indptr + row_cost * np.arange(rows + 1, dtype=np.int64)
    nnz = int(indptr[-1] - indptr[0])
    targets = indptr[0] + (nnz * np.arange(1, parts, dtype=np.int64)) // max(parts, 1)
    cuts = np.searchsorted(indptr, targets, side="left")
    splits = np.concatenate([[0], np.clip(cuts, 0, rows), [rows]]).astype(np.int64)
    return np.maximum.accumulate(splits)


#: the fields of one rank's row of the block table a multi-GPU fit from row blocks all-gathers first (int64 each)
BLOCK_FIELDS = ("first_row", "rows", "users", "items", "nnz", "failed")


def check_block_table(table):
    """(users, items, nnz) of the matrix the ranks' blocks tile, from the block table (one row of BLOCK_FIELDS per rank,
    in rank order), or the same ValueError, naming the offending rank, on every rank that checks the same table."""
    t = np.asarray(table, dtype=np.int64).reshape(-1, len(BLOCK_FIELDS))
    users, items = int(t[0, 2]), int(t[0, 3])
    end = 0
    for p, (first, rows, u, i, nnz, _) in enumerate(t.tolist()):
        if u != users:
            raise ValueError(f"rank {p}'s row block is of a {u}-row matrix, rank 0's of a {users}-row one")
        if i != items:
            raise ValueError(f"rank {p}'s row block has {i} columns, rank 0's {items}")
        if first < 0 or rows < 0 or nnz < 0:
            raise ValueError(f"rank {p}'s row block has first_row {first}, {rows} rows and {nnz} nonzeros")
        if first + rows > users:
            raise ValueError(f"rank {p}'s row block, rows [{first}, {first + rows}), runs past the {users} rows of the "
                             "matrix")
        if first != end:
            raise ValueError(f"rank {p}'s row block starts at row {first}, but the blocks of the ranks before it end at "
                             f"row {end}: the blocks must tile the rows in rank order, without gaps or overlaps")
        end = first + rows
    if end != users:
        raise ValueError(f"rank {len(t) - 1}'s row block ends at row {end}: the blocks must tile all {users} rows")
    return users, items, int(t[:, 4].sum())


def block_cuts(table, local_indptr, rank, row_cost=0):
    """This rank's part of the user split of a fit from row blocks: the W - 1 inner cuts of
    nnz_balanced_splits(whole.indptr, W, row_cost) that fall in its block, zeros elsewhere.  Summed over the ranks and
    passed to splits_from_cuts, they are that split exactly, although no rank holds the whole indptr.

    Every rank knows from the (checked) table the value of g = indptr + row_cost * row at every block boundary, so which
    block holds the first row whose g reaches each target; only that block's owner searches its own indptr."""
    t = np.asarray(table, dtype=np.int64).reshape(-1, len(BLOCK_FIELDS))
    W = len(t)
    first, rows, users, nnz = t[:, 0], t[:, 1], int(t[0, 2]), t[:, 4]
    before = np.concatenate([[0], np.cumsum(nnz)])  # nonzeros of the rows before each block
    total = int(before[-1]) + row_cost * users
    targets = (total * np.arange(1, W, dtype=np.int64)) // max(W, 1)
    cuts = np.zeros(max(W - 1, 0), dtype=np.int64)
    lo = before[rank] + row_cost * first[rank]                     # g at the block's first row
    hi = before[rank + 1] + row_cost * (first[rank] + rows[rank])  # ... and one past its last
    mine = np.flatnonzero((targets > lo) & (targets <= hi)) if rows[rank] > 0 else []
    if len(mine):
        ip = np.asarray(local_indptr, dtype=np.int64)
        g = lo + (ip - ip[0]) + row_cost * np.arange(len(ip), dtype=np.int64)
        cuts[mine] = first[rank] + np.searchsorted(g, targets[mine], side="left")
    return cuts


def splits_from_cuts(cuts, users):
    """The user split from the summed block_cuts: the clip and running maximum of nnz_balanced_splits."""
    splits = np.concatenate([[0], np.clip(np.asarray(cuts, dtype=np.int64), 0, users), [users]]).astype(np.int64)
    return np.maximum.accumulate(splits)


def simulate_block_splits(table, local_indptrs, row_cost=0):
    """The user split the W ranks of a fit from row blocks agree on (their block_cuts summed), computed in one process."""
    users, _, _ = check_block_table(table)
    cuts = sum(block_cuts(table, ip, p, row_cost) for p, ip in enumerate(local_indptrs))
    return splits_from_cuts(cuts, users)


def column_splits(col_counts, parts, row_cost=0):
    """nnz_balanced_splits of the transpose, planned from the entries per column of the matrix: the transpose's indptr
    is their running sum."""
    counts = np.asarray(col_counts, dtype=np.int64)
    return nnz_balanced_splits(np.concatenate([[0], np.cumsum(counts)]), parts, row_cost)
