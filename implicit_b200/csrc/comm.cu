// Multi-GPU exchange steps of the ALS fit loop: one process per GPU, NCCL over NVLink 5 / NVSwitch.
// The reference has no multi-GPU path at all (`// TODO: multi-gpu support`, implicit/gpu/als.cu:169);
// the sharding is described in DESIGN.md: every rank holds full replicas of both factor matrices and
// a contiguous, nnz-balanced row shard of Cui and of Ciu; after each half the freshly solved rows are
// all-gathered into every replica.
//
// NCCL is bound lazily with dlopen so that the single-GPU product has no link-time dependency on it
// (and picks up whichever libnccl.so.2 the process already has mapped).
#include <dlfcn.h>
#include <nccl.h>
#include <string.h>

#include <algorithm>

#include "common.h"

namespace als {
namespace {

struct NcclApi {
  void *handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void *, void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char *(*GetErrorString)(ncclResult_t) = nullptr;
};

NcclApi g_nccl;

int load_nccl() {
  if (g_nccl.handle) return ALS_OK;
  const char *names[] = {"libnccl.so.2", "libnccl.so"};
  void *h = nullptr;
  for (const char *n : names) {
    h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (h) break;
  }
  if (!h) {
    set_error("NCCL is not loadable: %s", dlerror());
    return ALS_E_NCCL;
  }
#define ALS_SYM(field, name)                                           \
  *(void **)(&g_nccl.field) = dlsym(h, name);                          \
  if (!g_nccl.field) {                                                 \
    set_error("NCCL symbol %s not found", name);                       \
    return ALS_E_NCCL;                                                 \
  }
  ALS_SYM(GetUniqueId, "ncclGetUniqueId")
  ALS_SYM(CommInitRank, "ncclCommInitRank")
  ALS_SYM(CommDestroy, "ncclCommDestroy")
  ALS_SYM(AllReduce, "ncclAllReduce")
  ALS_SYM(Broadcast, "ncclBroadcast")
  ALS_SYM(AllGather, "ncclAllGather")
  ALS_SYM(Send, "ncclSend")
  ALS_SYM(Recv, "ncclRecv")
  ALS_SYM(GroupStart, "ncclGroupStart")
  ALS_SYM(GroupEnd, "ncclGroupEnd")
  ALS_SYM(GetErrorString, "ncclGetErrorString")
#undef ALS_SYM
  g_nccl.handle = h;
  return ALS_OK;
}

int nccl_fail(ncclResult_t r, const char *what) {
  set_error("NCCL error %d (%s) in %s", (int)r, g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?", what);
  return ALS_E_NCCL;
}

#define ALS_NCCL(expr)                                   \
  do {                                                   \
    ncclResult_t r__ = (expr);                           \
    if (r__ != ncclSuccess) return nccl_fail(r__, #expr); \
  } while (0)

}  // namespace

int comm_allreduce_gramian(als_ctx *ctx, int n_floats) {
  if (ctx->world == 1 || !ctx->comm) return ALS_OK;
  // + 1: the failure flag written by gramian_reduce_kernel (see als_solver_status)
  ALS_NCCL(g_nccl.AllReduce(ctx->G, ctx->G, (size_t)n_floats + 1, ncclFloat, ncclSum, (ncclComm_t)ctx->comm, ctx->stream));
  return ALS_OK;
}

}  // namespace als

using namespace als;

static_assert(sizeof(ncclUniqueId) == ALS_COMM_ID_BYTES, "ncclUniqueId size");

ALS_API int als_comm_unique_id(void *id) {
  ALS_REQUIRE(id, "als_comm_unique_id: NULL");
  int rc = load_nccl();
  if (rc != ALS_OK) return rc;
  ncclUniqueId uid;
  ALS_NCCL(g_nccl.GetUniqueId(&uid));
  memcpy(id, &uid, sizeof(uid));
  return ALS_OK;
}

ALS_API int als_comm_init(als_ctx *ctx, int rank, int world, const void *id) {
  ALS_REQUIRE(ctx && id, "als_comm_init: NULL argument");
  ALS_REQUIRE(world >= 1 && rank >= 0 && rank < world, "als_comm_init: bad rank %d / world %d", rank, world);
  int rc = load_nccl();
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaSetDevice(ctx->device));
  ncclUniqueId uid;
  memcpy(&uid, id, sizeof(uid));
  ncclComm_t comm;
  ALS_NCCL(g_nccl.CommInitRank(&comm, world, uid, rank));
  ctx->comm = comm;
  ctx->rank = rank;
  ctx->world = world;
  return ALS_OK;
}

ALS_API int als_comm_destroy(als_ctx *ctx) {
  if (!ctx || !ctx->comm) return ALS_OK;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  g_nccl.CommDestroy((ncclComm_t)ctx->comm);
  ctx->comm = nullptr;
  ctx->rank = 0;
  ctx->world = 1;
  return ALS_OK;
}

ALS_API int als_comm_allgather_rows(als_ctx *ctx, als_factors *f, const int64_t *row_splits) {
  ALS_REQUIRE(ctx && f && row_splits, "als_comm_allgather_rows: NULL argument");
  if (ctx->world == 1) return ALS_OK;
  ALS_REQUIRE(ctx->comm, "als_comm_allgather_rows: communicator not initialised");
  ALS_REQUIRE(row_splits[0] == 0 && row_splits[ctx->world] == f->rows,
              "als_comm_allgather_rows: row_splits must run from 0 to %lld", (long long)f->rows);
  ALS_CUDA(cudaSetDevice(ctx->device));
  // variable shard sizes: one in-place broadcast per owner, fused into a single NCCL group
  ALS_NCCL(g_nccl.GroupStart());
  for (int r = 0; r < ctx->world; ++r) {
    const int64_t n = row_splits[r + 1] - row_splits[r];
    if (n <= 0) continue;
    float *p = f->d + row_splits[r] * (int64_t)f->ld;
    ALS_NCCL(g_nccl.Broadcast(p, p, (size_t)(n * f->ld), ncclFloat, r, (ncclComm_t)ctx->comm, ctx->stream));
  }
  ALS_NCCL(g_nccl.GroupEnd());
  return ALS_OK;
}

ALS_API int als_comm_allreduce_f64(als_ctx *ctx, double *values, int n, int op_max) {
  ALS_REQUIRE(ctx && values && n >= 0 && n <= 8, "als_comm_allreduce_f64: bad argument (n must be <= 8)");
  if (ctx->world == 1 || n == 0) return ALS_OK;
  ALS_REQUIRE(ctx->comm, "als_comm_allreduce_f64: communicator not initialised");
  ALS_CUDA(cudaSetDevice(ctx->device));
  ALS_CUDA(cudaMemcpyAsync(ctx->dscalars, values, sizeof(double) * n, cudaMemcpyHostToDevice, ctx->stream));
  ALS_NCCL(g_nccl.AllReduce(ctx->dscalars, ctx->dscalars, n, ncclDouble, op_max ? ncclMax : ncclSum,
                            (ncclComm_t)ctx->comm, ctx->stream));
  ALS_CUDA(cudaMemcpyAsync(values, ctx->dscalars, sizeof(double) * n, cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return ALS_OK;
}

namespace {

// Every rank passes its own rc; returns it, or a failure on every rank when any rank failed.  One all-reduce of a flag
// in ctx->dscalars, which needs no allocation: no rank goes on into a collective that another rank has left.
int agree(als_ctx *ctx, int rc, const char *who, const char *what) {
  double flag = rc != ALS_OK ? 1.0 : 0.0;
  ALS_CUDA(cudaMemcpyAsync(ctx->dscalars, &flag, sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  ALS_NCCL(g_nccl.AllReduce(ctx->dscalars, ctx->dscalars, 1, ncclDouble, ncclMax, (ncclComm_t)ctx->comm, ctx->stream));
  ALS_CUDA(cudaMemcpyAsync(&flag, ctx->dscalars, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  if (rc != ALS_OK) return rc;
  if (flag > 0) {
    set_error("%s: another rank failed %s (see its error message)", who, what);
    return ALS_E_NCCL;
  }
  return ALS_OK;
}

// Two grouped rounds of ncclSend / ncclRecv on the compute stream: the shapes (rows, cols, nnz of each piece), then
// every piece's indptr (64-bit positions from its first nonzero), indices and values straight into the receiving CSR.
// NCCL matches the operations between one pair of ranks in the order they are issued.  The ranks agree before each
// round that every one of them is ready for it (its pieces checked and staged, then its incoming pieces allocated): the
// two immediately invoked lambdas collect a rank's failure for that agreement.  recv is set on success only.
int exchange_csr(als_ctx *ctx, als_csr *const *send, als_csr **recv) {
  static const char *who = "als_comm_exchange_csr";
  const int W = ctx->world;
  ncclComm_t comm = (ncclComm_t)ctx->comm;
  std::vector<std::vector<int64_t>> sip(W);
  std::vector<int64_t> head(6 * (size_t)W, 0), base(W), rip_off(W + 1, 0);
  Dev<int64_t> buf;  // the shapes out and in (6 W), then the outgoing indptrs
  Dev<int64_t> rip;  // the incoming indptrs
  std::vector<CsrHolder> got(W);
  int rc = [&]() -> int {
    for (int q = 0; q < W; ++q) {
      ALS_REQUIRE(send[q], "%s: piece %d is NULL", who, q);
      if (send[q]->host) {
        set_error("%s: piece %d is host-resident", who, q);
        return ALS_E_UNSUPPORTED;
      }
    }
    int64_t sip_total = 0;
    for (int q = 0; q < W; ++q) {
      const int r = csr_indptr64(ctx, send[q], sip[q]);
      if (r != ALS_OK) return r;
      head[3 * q] = send[q]->rows;
      head[3 * q + 1] = send[q]->cols;
      head[3 * q + 2] = send[q]->nnz;
      sip_total += send[q]->rows + 1;
    }
    std::vector<int64_t> out(6 * (size_t)W + sip_total);
    std::copy(head.begin(), head.begin() + 3 * W, out.begin());
    for (int q = 0, at = 6 * W; q < W; at += (int)sip[q].size(), ++q) {
      base[q] = sip[q][0];
      for (size_t r = 0; r < sip[q].size(); ++r) out[at + r] = sip[q][r] - base[q];
    }
    const int r = buf.alloc(ctx, sizeof(int64_t) * out.size());
    if (r != ALS_OK) return r;
    ALS_CUDA(cudaMemcpyAsync(buf, out.data(), sizeof(int64_t) * out.size(), cudaMemcpyHostToDevice, ctx->stream));
    ALS_CUDA(cudaStreamSynchronize(ctx->stream));  // `out` dies here
    return ALS_OK;
  }();
  if ((rc = agree(ctx, rc, who, "to stage its pieces")) != ALS_OK) return rc;
  ALS_NCCL(g_nccl.GroupStart());
  for (int q = 0; q < W; ++q) {
    ALS_NCCL(g_nccl.Send(buf + 3 * q, 3, ncclInt64, q, comm, ctx->stream));
    ALS_NCCL(g_nccl.Recv(buf + 3 * W + 3 * q, 3, ncclInt64, q, comm, ctx->stream));
  }
  ALS_NCCL(g_nccl.GroupEnd());
  ALS_CUDA(cudaMemcpyAsync(head.data() + 3 * W, buf + 3 * W, sizeof(int64_t) * 3 * W, cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  rc = [&]() -> int {
    for (int p = 0; p < W; ++p) {
      got[p] = new_csr(ctx);
      als_csr *c = got[p].get();
      c->rows = head[3 * W + 3 * p];
      c->cols = head[3 * W + 3 * p + 1];
      c->nnz = head[3 * W + 3 * p + 2];
      const int r = csr_alloc(ctx, c);
      if (r != ALS_OK) return r;
      rip_off[p + 1] = rip_off[p] + c->rows + 1;
    }
    return rip.alloc(ctx, sizeof(int64_t) * rip_off[W]);
  }();
  if ((rc = agree(ctx, rc, who, "to allocate the pieces it receives")) != ALS_OK) return rc;
  ALS_NCCL(g_nccl.GroupStart());
  for (int q = 0, at = 6 * W; q < W; at += (int)sip[q].size(), ++q) {
    const als_csr *s = send[q];
    ALS_NCCL(g_nccl.Send(buf + at, sip[q].size(), ncclInt64, q, comm, ctx->stream));
    if (s->nnz) {
      ALS_NCCL(g_nccl.Send(s->indices + base[q], (size_t)s->nnz, ncclInt32, q, comm, ctx->stream));
      ALS_NCCL(g_nccl.Send(s->data + base[q], (size_t)s->nnz, ncclFloat, q, comm, ctx->stream));
    }
  }
  for (int p = 0; p < W; ++p) {
    als_csr *c = got[p].get();
    ALS_NCCL(g_nccl.Recv(rip + rip_off[p], (size_t)(c->rows + 1), ncclInt64, p, comm, ctx->stream));
    if (c->nnz) {
      ALS_NCCL(g_nccl.Recv(c->indices, (size_t)c->nnz, ncclInt32, p, comm, ctx->stream));
      ALS_NCCL(g_nccl.Recv(c->data, (size_t)c->nnz, ncclFloat, p, comm, ctx->stream));
    }
  }
  ALS_NCCL(g_nccl.GroupEnd());
  std::vector<int64_t> ip(rip_off[W]);
  ALS_CUDA(cudaMemcpyAsync(ip.data(), rip, sizeof(int64_t) * ip.size(), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  // the received pieces are only copied by the merge: their schedules wait for a solve that may never come
  for (int p = 0; p < W; ++p)
    if ((rc = csr_layout(ctx, got[p].get(), ip.data() + rip_off[p], /*schedule=*/false)) != ALS_OK) return rc;
  for (int p = 0; p < W; ++p) recv[p] = got[p].release();
  return ALS_OK;
}

int allreduce_i64(als_ctx *ctx, int64_t *buf, int64_t *values, int64_t n) {
  ALS_CUDA(cudaMemcpyAsync(buf, values, sizeof(int64_t) * n, cudaMemcpyHostToDevice, ctx->stream));
  ALS_NCCL(g_nccl.AllReduce(buf, buf, (size_t)n, ncclInt64, ncclSum, (ncclComm_t)ctx->comm, ctx->stream));
  ALS_CUDA(cudaMemcpyAsync(values, buf, sizeof(int64_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return ALS_OK;
}

}  // namespace

ALS_API int als_comm_allreduce_i64(als_ctx *ctx, int64_t *values, int64_t n) {
  ALS_REQUIRE(ctx && n >= 0 && (values || n == 0), "als_comm_allreduce_i64: bad argument");
  if (n == 0 || (ctx->world == 1 && !ctx->comm)) return ALS_OK;
  ALS_REQUIRE(ctx->comm, "als_comm_allreduce_i64: communicator not initialised");
  ALS_CUDA(cudaSetDevice(ctx->device));
  Dev<int64_t> buf;
  const int rc = agree(ctx, buf.alloc(ctx, sizeof(int64_t) * n), "als_comm_allreduce_i64", "to allocate its buffer");
  return rc != ALS_OK ? rc : allreduce_i64(ctx, buf, values, n);
}

ALS_API int als_comm_exchange_csr(als_ctx *ctx, als_csr *const *send, als_csr **recv) {
  ALS_REQUIRE(ctx && send && recv, "als_comm_exchange_csr: NULL argument");
  ALS_REQUIRE(ctx->comm, "als_comm_exchange_csr: communicator not initialised");
  for (int p = 0; p < ctx->world; ++p) recv[p] = nullptr;
  ALS_CUDA(cudaSetDevice(ctx->device));
  return exchange_csr(ctx, send, recv);
}

ALS_API int als_comm_allgather_bytes(als_ctx *ctx, const void *send, void *recv, int nbytes) {
  ALS_REQUIRE(ctx && send && recv && nbytes > 0 && nbytes <= 256, "als_comm_allgather_bytes: bad argument");
  if (ctx->world == 1) {
    memcpy(recv, send, nbytes);
    return ALS_OK;
  }
  ALS_REQUIRE(ctx->comm, "als_comm_allgather_bytes: communicator not initialised");
  ALS_CUDA(cudaSetDevice(ctx->device));
  int rc = ensure_scratch(ctx, (int64_t)(ctx->world + 1) * 256);
  if (rc != ALS_OK) return rc;
  char *base = (char *)ctx->scratch;
  ALS_CUDA(cudaMemcpyAsync(base, send, nbytes, cudaMemcpyHostToDevice, ctx->stream));
  ALS_NCCL(g_nccl.AllGather(base, base + 256, nbytes, ncclChar, (ncclComm_t)ctx->comm, ctx->stream));
  ALS_CUDA(cudaMemcpyAsync(recv, base + 256, (size_t)nbytes * ctx->world, cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return ALS_OK;
}

ALS_API int als_comm_barrier(als_ctx *ctx) {
  double one = 1.0;
  return als_comm_allreduce_f64(ctx, &one, 1, 0);
}
