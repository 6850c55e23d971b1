"""One process per GPU: rendezvous + NCCL communicator for the row-sharded ALS fit.

The reference is single-process / single-GPU (``// TODO: multi-gpu support``, implicit/gpu/als.cu:169);
this module is new.  Launch with the usual environment (``torchrun``-compatible):

    RANK, LOCAL_RANK, WORLD_SIZE, MASTER_ADDR, MASTER_PORT

Only the 128-byte NCCL unique id crosses between the processes on the host side: rank 0 creates it
(als_comm_unique_id) and serves it over a loopback/TCP socket next to MASTER_PORT; every rank then
calls als_comm_init.  No PyTorch is involved; all collectives are NCCL calls inside libals_b200.so.
"""
import numbers
import os
import socket
import struct
import time

import numpy as np

from . import _lib
from .utils import check_csr, is_device_csr

_MAGIC = b"ALSB200\x01"
_PORT_OFFSETS = (1, 2, 3, 5, 8, 13, 21, 34)


def _candidate_ports():
    base = int(os.environ.get("ALS_B200_RDZV_PORT", 0))
    if base:
        return [base]
    master = int(os.environ.get("MASTER_PORT", "29500"))
    return [master + o for o in _PORT_OFFSETS]


def _run_token():
    # distinguishes concurrent jobs that share a host: same for every rank of one launch
    return (os.environ.get("TORCHELASTIC_RUN_ID", "") + ":" + os.environ.get("MASTER_PORT", "")).encode()[:64]


def exchange_bytes(rank, world, payload, timeout=300.0):
    """Rank 0 hands `payload` (bytes) to every other rank; returns it on all ranks."""
    if world == 1:
        return payload
    addr = os.environ.get("MASTER_ADDR", "127.0.0.1")
    token = _run_token()
    deadline = time.time() + timeout
    if rank == 0:
        srv = None
        for port in _candidate_ports():
            try:
                srv = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
                srv.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
                srv.bind(("", port))
                break
            except OSError:
                srv.close()
                srv = None
        if srv is None:
            raise RuntimeError("implicit_b200.distributed: no free rendezvous port near MASTER_PORT")
        srv.listen(world)
        srv.settimeout(1.0)
        served = 0
        while served < world - 1:
            if time.time() > deadline:
                raise TimeoutError("implicit_b200.distributed: rendezvous timed out on rank 0")
            try:
                conn, _ = srv.accept()
            except socket.timeout:
                continue
            with conn:
                conn.settimeout(10.0)
                try:
                    hello = _recv_exact(conn, len(_MAGIC) + 64)
                except (OSError, ConnectionError):
                    continue
                if hello[: len(_MAGIC)] != _MAGIC or hello[len(_MAGIC):].rstrip(b"\0") != token:
                    continue  # not one of ours
                conn.sendall(struct.pack("<I", len(payload)) + payload)
                served += 1
        srv.close()
        return payload
    ports = _candidate_ports()
    while True:
        for port in ports:
            try:
                with socket.create_connection((addr, port), timeout=2.0) as c:
                    c.settimeout(10.0)
                    c.sendall(_MAGIC + token.ljust(64, b"\0"))
                    (n,) = struct.unpack("<I", _recv_exact(c, 4))
                    return _recv_exact(c, n)
            except (OSError, ConnectionError, struct.error):
                continue
        if time.time() > deadline:
            raise TimeoutError(f"implicit_b200.distributed: rank {rank} could not reach rank 0")
        time.sleep(0.2)


def _recv_exact(conn, n):
    buf = b""
    while len(buf) < n:
        chunk = conn.recv(n - len(buf))
        if not chunk:
            raise ConnectionError("peer closed")
        buf += chunk
    return buf


def row_block(users, rank, world):
    """(first_row, end_row): rank's even share of `users` rows, for a loader that reads only its own rows from disk and
    passes them to fit as RowBlock(rows, first_row, users).  The blocks of ranks 0 .. world - 1 tile [0, users)."""
    users, rank, world = int(users), int(rank), int(world)
    if world < 1 or not 0 <= rank < world or users < 0:
        raise ValueError(f"row_block: no rank {rank} of {world} for {users} rows")
    return users * rank // world, users * (rank + 1) // world


class RowBlock:
    """This rank's rows [first_row, first_row + user_items.shape[0]) of a `users` x user_items.shape[1] interaction
    matrix, for AlternatingLeastSquares.fit.  On a process group of several ranks each rank passes only its own block;
    the blocks, of any sizes (none at all included), must tile [0, users) in rank order.  Without a process group, or on
    one rank, the block must hold every row, and the fit is the fit of the plain matrix.

    Conversion to CSR (with the usual ParameterWarning) and the cast of the values to float32 happen in fit, where a
    failure on one rank is reported to every rank instead of leaving the others waiting for it."""

    def __init__(self, user_items, first_row, users):
        self.user_items, self.first_row, self.users = user_items, first_row, users

    def csr(self):
        """The block as a float32 scipy CSR, after checking its own shape.  A block of device arrays is refused
        (ValueError): RowBlocks take scipy CSRs."""
        if is_device_csr(self.user_items):
            raise ValueError("a RowBlock takes a scipy CSR: a CSR in CUDA memory is fitted on one GPU only")
        m = check_csr(self.user_items)
        if m.dtype != np.float32:
            m = m.astype(np.float32)  # cpu/als.py:129-130
        first, users = self.first_row, self.users
        if not (isinstance(first, numbers.Integral) and isinstance(users, numbers.Integral)) or first < 0 or users < 0:
            raise ValueError(f"RowBlock: first_row ({first!r}) and users ({users!r}) must be integers >= 0")
        return m

    def whole(self):
        """The block as the whole matrix, for a fit without a process group or on one rank: it must hold every row."""
        m = self.csr()
        if self.first_row != 0 or m.shape[0] != self.users:
            raise ValueError(f"a RowBlock of rows [{self.first_row}, {self.first_row + m.shape[0]}) of a {self.users}-row "
                             "matrix is fitted only on a process group of several ranks; on one it must hold every row")
        return m


class ProcessGroup:
    """rank / world + the device context whose communicator spans all ranks."""

    def __init__(self, rank, world, ctx):
        self.rank, self.world, self.ctx = rank, world, ctx

    def barrier(self):
        self.ctx.barrier()

    def allreduce_max(self, value):
        return float(self.ctx.allreduce([value], "max")[0])

    def allreduce_sum(self, value):
        return float(self.ctx.allreduce([value], "sum")[0])


def init_process_group(device=None):
    """Reads RANK / LOCAL_RANK / WORLD_SIZE, creates this rank's device context and joins the NCCL clique."""
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    ctx = _lib.Context(local if device is None else device)
    if world > 1:
        uid = _lib.comm_unique_id() if rank == 0 else b""
        uid = exchange_bytes(rank, world, uid)
        ctx.comm_init(rank, world, uid)
    return ProcessGroup(rank, world, ctx)
