// C-ABI entry points, device containers and the launch schedule (host side of libals_b200.so).
#include <cuda_fp16.h>
#include <limits.h>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <functional>
#include <thread>

#include "common.h"

namespace als {

static thread_local char g_err[1024] = {0};

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char *what, const char *file, int line) {
  set_error("CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
  cudaGetLastError();  // clear the sticky-less error state
  return ALS_E_CUDA;
}

// the alloc_fail_at knob: ALS_E_CUDA for the n-th allocation since it was set
static int injected_failure(als_ctx *ctx) {
  if (ctx->knobs.alloc_fail_at <= 0 || --ctx->knobs.alloc_fail_at > 0) return ALS_OK;
  set_error("injected allocation failure");
  return ALS_E_CUDA;
}

int dev_alloc(als_ctx *ctx, void **ptr, int64_t bytes, cudaStream_t stream) {
  const int rc = injected_failure(ctx);
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaMallocAsync(ptr, (size_t)std::max<int64_t>(bytes, 16), stream ? stream : ctx->stream));
  return ALS_OK;
}

void dev_free(als_ctx *ctx, void *ptr) {
  if (ptr) cudaFreeAsync(ptr, ctx->stream);
}

DeviceBlock &DeviceBlock::operator=(DeviceBlock &&o) noexcept {
  if (this != &o) {
    reset();
    ctx_ = o.ctx_;
    p_ = o.take();
    pooled_ = o.pooled_;
  }
  return *this;
}

int DeviceBlock::alloc(als_ctx *ctx, int64_t bytes, cudaStream_t stream) {
  reset();
  ctx_ = ctx;
  pooled_ = true;
  return dev_alloc(ctx, &p_, bytes, stream);
}

int DeviceBlock::alloc_cuda(als_ctx *ctx, int64_t bytes) {
  reset();
  ctx_ = ctx;
  pooled_ = false;
  int rc = injected_failure(ctx);
  if (rc == ALS_OK) {
    const cudaError_t e = cudaMalloc(&p_, (size_t)std::max<int64_t>(bytes, 16));
    if (e != cudaSuccess) {
      p_ = nullptr;
      rc = cuda_fail(e, "cudaMalloc", __FILE__, __LINE__);
    }
  }
  return rc;
}

void DeviceBlock::reset() {
  void *p = take();
  if (!p) return;
  if (pooled_)
    dev_free(ctx_, p);
  else
    cudaFree(p);
}

void CsrDestroy::operator()(als_csr *c) const {
  if (c->ctx) cudaStreamSynchronize(c->ctx->stream);  // a copy may still be landing in its arrays
  als_csr_destroy(c);
}

CsrHolder new_csr(als_ctx *ctx) {
  CsrHolder c(new als_csr());
  c->ctx = ctx;
  return c;
}

// Builds the schedules of a CSR laid out without them (csr_layout's schedule = false) from its device indptrs.
int ensure_schedule(als_ctx *ctx, als_csr *csr) {
  if (!csr->sched_lazy) return ALS_OK;
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  std::vector<int32_t> ip;
  csr->max_row_nnz = 0;
  for (const als_csr *S : segments_of(csr)) {
    ip.resize((size_t)S->rows + 1);
    ALS_CUDA(cudaMemcpy(ip.data(), S->indptr, sizeof(int32_t) * ip.size(), cudaMemcpyDeviceToHost));
    int rc = build_schedule(ctx, const_cast<als_csr *>(S), ip.data());
    if (rc != ALS_OK) return rc;
    csr->max_row_nnz = std::max(csr->max_row_nnz, S->max_row_nnz);
  }
  csr->sched_lazy = false;
  return ALS_OK;
}

int ensure_scratch(als_ctx *ctx, int64_t bytes) {
  if (bytes <= ctx->scratch_bytes) return ALS_OK;
  if (ctx->scratch) {
    ALS_CUDA(cudaStreamSynchronize(ctx->stream));
    ALS_CUDA(cudaFree(ctx->scratch));
    ctx->scratch = nullptr;
    ctx->scratch_bytes = 0;
  }
  int64_t cap = std::max<int64_t>(bytes, 1 << 20);
  ALS_CUDA(cudaMalloc(&ctx->scratch, cap));
  ctx->scratch_bytes = cap;
  return ALS_OK;
}

int ensure_device_buffer(als_ctx *ctx, void **buf, int64_t *cap, int64_t bytes) {
  if (bytes <= *cap) return ALS_OK;
  if (*buf) {
    ALS_CUDA(cudaStreamSynchronize(ctx->stream));
    ALS_CUDA(cudaFree(*buf));
    *buf = nullptr;
    *cap = 0;
  }
  ALS_CUDA(cudaMalloc(buf, bytes));
  *cap = bytes;
  return ALS_OK;
}

// ---- host -> device copies of ordinary (pageable) memory ---------------------------------------------------------
// cudaMemcpyAsync from pageable memory is staged by the driver through one thread at ~12 GB/s; a user of the
// reference hands fit() ordinary numpy / scipy arrays, so for large buffers four host threads copy 4 MB chunks into
// page-locked staging buffers of their own and push them over PCIe on their own streams (memcpy and DMA overlap).
// Page-locked sources take the plain asynchronous copy.
static constexpr int kStageThreads = 4;
static constexpr size_t kStageChunk = 4u << 20;

// fill(stage, off, len): writes the `len` bytes that go to dst + off into the staging buffer; false stops the copy
// (the caller's input is bad, ALS_E_INVALID)
using StageFill = std::function<bool(char *stage, size_t off, size_t len)>;

static int staged_h2d(als_ctx *ctx, void *dst, size_t bytes, const StageFill &fill) {
  if (!ctx->stage_buf) {
    ALS_CUDA(cudaMallocHost(&ctx->stage_buf, kStageThreads * 2 * kStageChunk));
    for (int t = 0; t < kStageThreads; ++t) {
      ALS_CUDA(cudaStreamCreateWithFlags(&ctx->stage_stream[t], cudaStreamNonBlocking));
      for (int b = 0; b < 2; ++b) ALS_CUDA(cudaEventCreateWithFlags(&ctx->stage_ev[t][b], cudaEventDisableTiming));
    }
    ALS_CUDA(cudaEventCreateWithFlags(&ctx->stage_ready, cudaEventDisableTiming));
  }
  // the destination was allocated (stream-ordered) on the compute stream: the staging streams start after it
  ALS_CUDA(cudaEventRecord(ctx->stage_ready, ctx->stream));
  for (int t = 0; t < kStageThreads; ++t) ALS_CUDA(cudaStreamWaitEvent(ctx->stage_stream[t], ctx->stage_ready, 0));
  const size_t nchunks = (bytes + kStageChunk - 1) / kStageChunk;
  std::vector<int> status(kStageThreads, (int)cudaSuccess);
  std::atomic<bool> refused{false};
  std::vector<std::thread> pool;
  for (int t = 0; t < kStageThreads; ++t) {
    pool.emplace_back([=, &status, &refused, &fill]() {
      cudaSetDevice(ctx->device);
      // the staging buffers are shared by consecutive calls: a previous call's last DMAs may still be reading them
      cudaError_t e = cudaStreamSynchronize(ctx->stage_stream[t]);
      int use = 0;
      for (size_t c = t; c < nchunks && e == cudaSuccess; c += kStageThreads, ++use) {
        const int b = use & 1;
        char *stage = (char *)ctx->stage_buf + ((size_t)t * 2 + b) * kStageChunk;
        if (use >= 2) e = cudaEventSynchronize(ctx->stage_ev[t][b]);  // the DMA out of this buffer has finished
        const size_t off = c * kStageChunk, len = std::min(kStageChunk, bytes - off);
        if (!fill(stage, off, len)) {
          refused = true;
          break;
        }
        if (e == cudaSuccess) e = cudaMemcpyAsync((char *)dst + off, stage, len, cudaMemcpyHostToDevice, ctx->stage_stream[t]);
        if (e == cudaSuccess) e = cudaEventRecord(ctx->stage_ev[t][b], ctx->stage_stream[t]);
      }
      status[t] = (int)e;
    });
  }
  for (auto &th : pool) th.join();
  for (int t = 0; t < kStageThreads; ++t) {
    if (status[t] != (int)cudaSuccess) return cuda_fail((cudaError_t)status[t], "staged host-to-device copy", __FILE__, __LINE__);
    // the compute stream continues after the last chunk of every staging stream
    ALS_CUDA(cudaEventRecord(ctx->stage_ev[t][0], ctx->stage_stream[t]));
    ALS_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->stage_ev[t][0], 0));
  }
  return refused ? ALS_E_INVALID : ALS_OK;
}

static int h2d_copy(als_ctx *ctx, void *dst, const void *src, size_t bytes) {
  if (bytes == 0) return ALS_OK;
  cudaPointerAttributes at;
  const bool pinned = cudaPointerGetAttributes(&at, src) == cudaSuccess && at.type == cudaMemoryTypeHost;
  cudaGetLastError();  // an unregistered host pointer may leave an error behind on older drivers
  if (pinned || bytes < 2 * kStageChunk * kStageThreads) {
    ALS_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return ALS_OK;
  }
  return staged_h2d(ctx, dst, bytes, [src](char *stage, size_t off, size_t len) {
    memcpy(stage, (const char *)src + off, len);
    return true;
  });
}

// The staging threads of staged_h2d writing straight into a page-locked host array instead (a host-resident CSR): the
// same chunks, the same fill, no DMA.
static int staged_fill_host(void *dst, size_t bytes, const StageFill &fill) {
  const size_t nchunks = (bytes + kStageChunk - 1) / kStageChunk;
  std::atomic<bool> refused{false};
  std::vector<std::thread> pool;
  for (int t = 0; t < kStageThreads; ++t) {
    pool.emplace_back([=, &refused, &fill]() {
      for (size_t c = t; c < nchunks && !refused; c += kStageThreads) {
        const size_t off = c * kStageChunk, len = std::min(kStageChunk, bytes - off);
        if (!fill((char *)dst + off, off, len)) refused = true;
      }
    });
  }
  for (auto &th : pool) th.join();
  return refused ? ALS_E_INVALID : ALS_OK;
}

// n column indices (int32 or int64 on the host) -> int32 on the device, narrowed chunk by chunk in the staging threads
// (no host-side int32 copy of the whole array, half the PCIe bytes of int64).  Every index must lie in [0, cols): the
// first one that does not is reported in *bad_at (else -1) and the call returns ALS_E_INVALID.  host: dst is a
// page-locked host array (a host-resident CSR), written by the same threads.
static int h2d_indices(als_ctx *ctx, int32_t *dst, const void *src, int index_bytes, int64_t n, int64_t cols, int64_t *bad_at,
                       bool host = false) {
  *bad_at = -1;
  if (n == 0) return ALS_OK;
  std::atomic<int64_t> bad{INT64_MAX};
  auto narrow = [&](char *stage, size_t off, size_t len) -> bool {
    int32_t *o = reinterpret_cast<int32_t *>(stage);
    const int64_t i0 = (int64_t)(off / 4), m = (int64_t)(len / 4);
    int64_t first = -1;
    if (index_bytes == 8) {
      const int64_t *in = static_cast<const int64_t *>(src) + i0;
      for (int64_t k = 0; k < m; ++k) {
        const int64_t v = in[k];
        if ((uint64_t)v >= (uint64_t)cols && first < 0) first = k;
        o[k] = (int32_t)v;
      }
    } else {
      const int32_t *in = static_cast<const int32_t *>(src) + i0;
      for (int64_t k = 0; k < m; ++k) {
        const int32_t v = in[k];
        if ((uint64_t)(int64_t)v >= (uint64_t)cols && first < 0) first = k;
        o[k] = v;
      }
    }
    if (first < 0) return true;
    int64_t cur = bad.load();
    while (i0 + first < cur && !bad.compare_exchange_weak(cur, i0 + first)) {
    }
    return false;
  };
  const int rc = host ? staged_fill_host(dst, (size_t)n * sizeof(int32_t), narrow)
                      : staged_h2d(ctx, dst, (size_t)n * sizeof(int32_t), narrow);
  if (rc == ALS_E_INVALID) *bad_at = bad.load();
  return rc;
}

// Writes the n values of a host-resident CSR at dst in the staging threads, chunk by chunk (fill(v, i0, m) writes values
// i0 .. i0 + m - 1 to v), and folds the weight range of csr_wmax_kernel over what they wrote into c->wmax_dev.
static int fill_host_values(als_ctx *ctx, als_csr *c, float *dst, int64_t n,
                            const std::function<void(float *v, int64_t i0, int64_t m)> &fill) {
  std::atomic<unsigned> m{0};
  std::atomic<bool> ng{false};
  staged_fill_host(dst, sizeof(float) * (size_t)n, [&](char *out, size_t off, size_t len) {
    float *v = reinterpret_cast<float *>(out);
    fill(v, (int64_t)(off / 4), (int64_t)(len / 4));
    unsigned cm;
    bool cn;
    host_wmax(v, (int64_t)(len / 4), &cm, &cn);
    unsigned cur = m.load();
    while (cm > cur && !m.compare_exchange_weak(cur, cm)) {
    }
    if (cn) ng = true;
    return true;
  });
  return set_host_wmax(ctx, c, m.load(), ng.load());
}

// Longest-first schedule.  Rows with more than kSplitNnz nonzeros are cut into chunks of kChunkNnz
// so that one power-law giant (SURVEY.md section 7.2: 139k nnz in C2) cannot serialise the tail.
int build_schedule(als_ctx *ctx, als_csr *csr, const int32_t *indptr) {
  std::vector<WorkItem> items;
  std::vector<WorkItem> fin;
  std::vector<WorkItem> chunks;
  std::vector<int32_t> owner;
  items.reserve((size_t)csr->rows + 64);
  int64_t slots = 0;
  csr->max_row_nnz = 0;
  for (int64_t r = 0; r < csr->rows; ++r) {
    const int32_t b = indptr[r], e = indptr[r + 1];
    const int32_t n = e - b;
    csr->max_row_nnz = std::max<int64_t>(csr->max_row_nnz, n);
    if (n > kSplitNnz) {
      const int32_t nchunks = (int32_t)ceil_div(n, kChunkNnz);
      fin.push_back(WorkItem{(int32_t)r, (int32_t)slots, nchunks, -2});
      for (int32_t c = 0; c < nchunks; ++c) {
        const int32_t k0 = b + c * kChunkNnz;
        const int32_t k1 = std::min(e, k0 + kChunkNnz);
        items.push_back(WorkItem{(int32_t)r, k0, k1, (int32_t)slots});
        chunks.push_back(items.back());
        owner.push_back((int32_t)fin.size() - 1);
        ++slots;
      }
    } else {
      items.push_back(WorkItem{(int32_t)r, b, e, -1});
    }
  }
  // counting sort, descending by length (lengths <= kSplitNnz)
  {
    std::vector<int64_t> count(kSplitNnz + 2, 0);
    for (const WorkItem &w : items) ++count[kSplitNnz - (w.k1 - w.k0)];
    int64_t acc = 0;
    for (size_t i = 0; i < count.size(); ++i) {
      int64_t c = count[i];
      count[i] = acc;
      acc += c;
    }
    std::vector<WorkItem> sorted(items.size());
    for (const WorkItem &w : items) sorted[count[kSplitNnz - (w.k1 - w.k0)]++] = w;
    items.swap(sorted);
  }
  csr->n_work = (int64_t)items.size();
  for (int c = 0; c < kNumShortThresholds; ++c) {
    int64_t lo = 0, hi = csr->n_work;  // first item of length <= kShortThresholds[c]
    while (lo < hi) {
      const int64_t mid = (lo + hi) / 2;
      if (items[mid].k1 - items[mid].k0 <= kShortThresholds[c]) hi = mid;
      else lo = mid + 1;
    }
    csr->le_begin[c] = lo;
  }
  csr->n_finish = (int64_t)fin.size();
  csr->n_slots = slots;
  // The lists are allocated and uploaded on the copy stream: when the schedule of a transposed matrix is built, its
  // sort is still running on the compute stream and must not delay them (nor they it).
  cudaStream_t up = ctx->copy;
  int rc;
  if (csr->n_work) {
    if ((rc = dev_alloc(ctx, (void **)&csr->work, sizeof(WorkItem) * items.size(), up)) != ALS_OK) return rc;
    ALS_CUDA(cudaMemcpyAsync(csr->work, items.data(), sizeof(WorkItem) * items.size(), cudaMemcpyHostToDevice, up));
  }
  if (csr->n_finish) {
    if ((rc = dev_alloc(ctx, (void **)&csr->finish, sizeof(WorkItem) * fin.size(), up)) != ALS_OK) return rc;
    ALS_CUDA(cudaMemcpyAsync(csr->finish, fin.data(), sizeof(WorkItem) * fin.size(), cudaMemcpyHostToDevice, up));
  }
  if (!chunks.empty()) {
    if ((rc = dev_alloc(ctx, (void **)&csr->chunks, sizeof(WorkItem) * chunks.size(), up)) != ALS_OK) return rc;
    if ((rc = dev_alloc(ctx, (void **)&csr->chunk_owner, sizeof(int32_t) * owner.size(), up)) != ALS_OK) return rc;
    ALS_CUDA(cudaMemcpyAsync(csr->chunks, chunks.data(), sizeof(WorkItem) * chunks.size(), cudaMemcpyHostToDevice, up));
    ALS_CUDA(cudaMemcpyAsync(csr->chunk_owner, owner.data(), sizeof(int32_t) * owner.size(), cudaMemcpyHostToDevice, up));
  }
  ALS_CUDA(cudaEventRecord(ctx->ev_join, up));
  ALS_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));  // later kernels see the lists
  ALS_CUDA(cudaStreamSynchronize(up));                          // the host vectors die here
  return ALS_OK;
}

ProfScope::ProfScope(als_ctx *c, int w) : ctx(c), which(w) {
  if (!ctx->profiling) return;
  cudaEvent_t e;
  if (cudaEventCreate(&e) == cudaSuccess) {
    cudaEventRecord(e, ctx->stream);
    ctx->prof_events[which].push_back(e);
  }
}
ProfScope::~ProfScope() {
  if (!ctx->profiling || (ctx->prof_events[which].size() & 1) == 0) return;
  cudaEvent_t e;
  if (cudaEventCreate(&e) == cudaSuccess) {
    cudaEventRecord(e, ctx->stream);
    ctx->prof_events[which].push_back(e);
  } else {
    cudaEventDestroy(ctx->prof_events[which].back());
    ctx->prof_events[which].pop_back();
  }
}

__global__ void has_nan_kernel(const float *data, int64_t n, int *flag) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  bool bad = false;
  for (; i < n; i += stride) bad |= isnan(data[i]);
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(flag, 1);
}

__global__ void scale_kernel(float *data, int64_t n, float alpha) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) data[i] *= alpha;
}

__global__ void fill_kernel(float *data, int64_t n, float v) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) data[i] = v;
}

}  // namespace als

using namespace als;

// ---- context -----------------------------------------------------------------------------------
ALS_API int als_abi_version(void) { return ALS_B200_ABI_VERSION; }
ALS_API const char *als_last_error(void) { return g_err; }

ALS_API int als_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

ALS_API int als_ctx_create(int device, als_ctx **out) {
  ALS_REQUIRE(out != nullptr, "als_ctx_create: out is NULL");
  *out = nullptr;
  int n = 0;
  ALS_CUDA(cudaGetDeviceCount(&n));
  ALS_REQUIRE(device >= 0 && device < n, "als_ctx_create: device %d out of range (%d visible)", device, n);
  ALS_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  ALS_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("als_ctx_create: device %d is sm_%d%d; libals_b200 is built for sm_90a only", device, prop.major,
              prop.minor);
    return ALS_E_UNSUPPORTED;
  }
  // torn down with whatever it holds on any failure below
  std::unique_ptr<als_ctx, int (*)(als_ctx *)> ctx(new als_ctx(), als_ctx_destroy);
  ctx->device = device;
  {
    struct { const char *env; const char *name; } table[] = {
        {"ALS_B200_SHORT_MAX", "short_max"}, {"ALS_B200_SHORT_SERIAL", "short_serial"}, {"ALS_B200_WHITEN_FMA", "whiten_fma"},
        {"ALS_B200_GRAMIAN_FMA", "gramian_fma"}, {"ALS_B200_TOPK_LEGACY", "topk_legacy"}, {"ALS_B200_LONG_TC", "long_tc"}, {"ALS_B200_CG_NV", "cg_nv"},
        {"ALS_B200_SEGMENT_NNZ", "segment_nnz"}, {"ALS_B200_HOST_CSR", "host_csr"}};
    for (const auto &t : table) {
      const char *e = getenv(t.env);
      if (!e) continue;
      const int v = *e ? atoi(e) : 1;
      if (als_ctx_set_knob(ctx.get(), t.name, v) != ALS_OK) return ALS_E_INVALID;
      fprintf(stderr, "libals_b200: %s=%s is set (knob %s = %d)\n", t.env, e, t.name, v);
    }
  }
  ctx->sm_count = prop.multiProcessorCount;
  ctx->l2_bytes = prop.l2CacheSize;
  ctx->mem_bytes = (int64_t)prop.totalGlobalMem;
  strncpy(ctx->name, prop.name, sizeof(ctx->name) - 1);
  ALS_CUDA(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
  ALS_CUDA(cudaStreamCreateWithFlags(&ctx->copy, cudaStreamNonBlocking));
  ALS_CUDA(cudaStreamCreateWithFlags(&ctx->aux, cudaStreamNonBlocking));
  for (int i = 0; i < 5; ++i) {
    ALS_CUDA(cudaStreamCreateWithFlags(&ctx->class_stream[i], cudaStreamNonBlocking));
    ALS_CUDA(cudaEventCreateWithFlags(&ctx->class_join[i], cudaEventDisableTiming));
  }
  ALS_CUDA(cudaEventCreateWithFlags(&ctx->class_fork, cudaEventDisableTiming));
  ALS_CUDA(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
  ALS_CUDA(cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming));
  for (int k = 0; k < 2; ++k) {
    ALS_CUDA(cudaEventCreateWithFlags(&ctx->ring_loaded[k], cudaEventDisableTiming));
    ALS_CUDA(cudaEventCreateWithFlags(&ctx->ring_free[k], cudaEventDisableTiming));
  }
  {
    cudaMemPool_t pool;
    ALS_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
    uint64_t keep = UINT64_MAX;  // never hand freed blocks back to the driver while the context lives
    ALS_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
  }
  ALS_CUDA(cudaEventCreate(&ctx->ev0));
  ALS_CUDA(cudaEventCreate(&ctx->ev1));
  ALS_CUDA(cudaMalloc(&ctx->G, sizeof(float) * (1024 * 1024 + 64)));     // up to 1024 padded factors + the failure flag slot
  ALS_CUDA(cudaMalloc(&ctx->Greg, sizeof(float) * (1024 * 1024 + 64)));
  ALS_CUDA(cudaMalloc(&ctx->Pinv, sizeof(float) * 64 * 64));
  ALS_CUDA(cudaMalloc(&ctx->Ginv, sizeof(float) * 64 * 64));
  ALS_CUDA(cudaMalloc(&ctx->counters, sizeof(int32_t) * 16));
  ALS_CUDA(cudaMalloc(&ctx->bad_row, sizeof(long long) * 2));
  {
    const long long init[2] = {LLONG_MAX, LLONG_MAX};
    ALS_CUDA(cudaMemcpy(ctx->bad_row, init, sizeof(init), cudaMemcpyHostToDevice));
  }
  ALS_CUDA(cudaMalloc(&ctx->status, sizeof(int32_t) * 4));
  ALS_CUDA(cudaMemset(ctx->status, 0, sizeof(int32_t) * 4));
  ALS_CUDA(cudaMemset(ctx->G, 0, sizeof(float) * (1024 * 1024 + 64)));
  ALS_CUDA(cudaMalloc(&ctx->dscalars, sizeof(double) * 8));
  *out = ctx.release();
  return ALS_OK;
}

ALS_API int als_ctx_set_knob(als_ctx *ctx, const char *name, int value) {
  ALS_REQUIRE(ctx && name, "als_ctx_set_knob: NULL argument");
  als_knobs &k = ctx->knobs;
  if (!strcmp(name, "short_max")) k.short_max = value >= 48 ? 48 : value <= 0 ? 0 : value / 8 * 8;
  else if (!strcmp(name, "short_serial")) k.short_serial = value != 0;
  else if (!strcmp(name, "whiten_fma")) k.whiten_fma = value != 0;
  else if (!strcmp(name, "gramian_fma")) k.gramian_fma = value != 0;
  else if (!strcmp(name, "topk_legacy")) k.topk_legacy = value != 0;
  else if (!strcmp(name, "long_tc")) k.long_tc = value != 0;
  else if (!strcmp(name, "cg_nv")) {
    ALS_REQUIRE(value == 1 || value == 2 || value == 4, "als_ctx_set_knob: cg_nv must be 1, 2 or 4");
    k.cg_nv = value;
  } else if (!strcmp(name, "segment_nnz")) {
    ALS_REQUIRE(value >= 0 && value < INT32_MAX, "als_ctx_set_knob: segment_nnz must be in [0, 2^31 - 1)");
    k.segment_nnz = value;
  } else if (!strcmp(name, "host_csr")) k.host_csr = value != 0;
  else if (!strcmp(name, "alloc_fail_at")) k.alloc_fail_at = std::max(value, 0);
  else {
    set_error("als_ctx_set_knob: unknown knob '%s'", name);
    return ALS_E_INVALID;
  }
  return ALS_OK;
}

ALS_API int als_ctx_get_knob(als_ctx *ctx, const char *name, int *value) {
  ALS_REQUIRE(ctx && name && value, "als_ctx_get_knob: NULL argument");
  const als_knobs &k = ctx->knobs;
  if (!strcmp(name, "short_max")) *value = k.short_max;
  else if (!strcmp(name, "short_serial")) *value = k.short_serial;
  else if (!strcmp(name, "whiten_fma")) *value = k.whiten_fma;
  else if (!strcmp(name, "gramian_fma")) *value = k.gramian_fma;
  else if (!strcmp(name, "topk_legacy")) *value = k.topk_legacy;
  else if (!strcmp(name, "long_tc")) *value = k.long_tc;
  else if (!strcmp(name, "cg_nv")) *value = k.cg_nv;
  else if (!strcmp(name, "segment_nnz")) *value = (int)k.segment_nnz;
  else if (!strcmp(name, "host_csr")) *value = k.host_csr;
  else if (!strcmp(name, "alloc_fail_at")) *value = k.alloc_fail_at;
  else {
    set_error("als_ctx_get_knob: unknown knob '%s'", name);
    return ALS_E_INVALID;
  }
  return ALS_OK;
}

ALS_API int als_ctx_destroy(als_ctx *ctx) {
  if (!ctx) return ALS_OK;
  // also the teardown of a failed als_ctx_create: members it never created are null and skipped
  auto stream_destroy = [](cudaStream_t s) {
    if (s) cudaStreamDestroy(s);
  };
  auto event_destroy = [](cudaEvent_t e) {
    if (e) cudaEventDestroy(e);
  };
  cudaSetDevice(ctx->device);
  for (cudaStream_t s : {ctx->stream, ctx->copy, ctx->aux})
    if (s) cudaStreamSynchronize(s);
  als_comm_destroy(ctx);
  cudaFree(ctx->G);
  cudaFree(ctx->Greg);
  cudaFree(ctx->gram_partials);
  cudaFree(ctx->Pinv);
  cudaFree(ctx->Ginv);
  cudaFree(ctx->whitened);
  cudaFree(ctx->zfactors);
  cudaFree(ctx->dense_bt);
  cudaFree(ctx->deferred);
  cudaFree(ctx->counters);
  cudaFree(ctx->bad_row);
  cudaFree(ctx->status);
  cudaFree(ctx->dscalars);
  cudaFree(ctx->scratch);
  if (ctx->stage_buf) {
    cudaFreeHost(ctx->stage_buf);
    for (int t = 0; t < 4; ++t) {
      stream_destroy(ctx->stage_stream[t]);
      for (int b = 0; b < 2; ++b) event_destroy(ctx->stage_ev[t][b]);
    }
    event_destroy(ctx->stage_ready);
  }
  for (int k = 0; k < 2; ++k) {
    event_destroy(ctx->ring_loaded[k]);
    event_destroy(ctx->ring_free[k]);
  }
  for (int i = 0; i < 5; ++i) {
    stream_destroy(ctx->class_stream[i]);
    event_destroy(ctx->class_join[i]);
  }
  event_destroy(ctx->class_fork);
  {
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, ctx->device) == cudaSuccess) cudaMemPoolTrimTo(pool, 0);
  }
  event_destroy(ctx->ev0);
  event_destroy(ctx->ev1);
  stream_destroy(ctx->stream);
  stream_destroy(ctx->copy);
  stream_destroy(ctx->aux);
  event_destroy(ctx->ev_fork);
  event_destroy(ctx->ev_join);
  delete ctx;
  return ALS_OK;
}

ALS_API int als_sync(als_ctx *ctx) {
  ALS_REQUIRE(ctx, "als_sync: ctx is NULL");
  ALS_CUDA(cudaSetDevice(ctx->device));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->copy));
  return ALS_OK;
}

ALS_API int als_device_info(als_ctx *ctx, char *name, int *sm_count, int64_t *l2_bytes, int64_t *mem_bytes) {
  ALS_REQUIRE(ctx, "als_device_info: ctx is NULL");
  if (name) strncpy(name, ctx->name, 256);
  if (sm_count) *sm_count = ctx->sm_count;
  if (l2_bytes) *l2_bytes = ctx->l2_bytes;
  if (mem_bytes) *mem_bytes = ctx->mem_bytes;
  return ALS_OK;
}

int als::mem_info(als_ctx *ctx, int64_t *free_bytes, int64_t *total_bytes) {
  ALS_CUDA(cudaSetDevice(ctx->device));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));  // stream-ordered frees land in the pool
  size_t fr = 0, tot = 0;
  ALS_CUDA(cudaMemGetInfo(&fr, &tot));
  cudaMemPool_t pool;
  ALS_CUDA(cudaDeviceGetDefaultMemPool(&pool, ctx->device));
  uint64_t reserved = 0, used = 0;
  ALS_CUDA(cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReservedMemCurrent, &reserved));
  ALS_CUDA(cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemCurrent, &used));
  *free_bytes = (int64_t)fr + (int64_t)(reserved > used ? reserved - used : 0);
  *total_bytes = (int64_t)tot;
  return ALS_OK;
}

ALS_API int als_mem_info(als_ctx *ctx, int64_t *free_bytes, int64_t *total_bytes) {
  ALS_REQUIRE(ctx && free_bytes && total_bytes, "als_mem_info: NULL argument");
  return als::mem_info(ctx, free_bytes, total_bytes);
}

ALS_API int64_t als_launch_count(als_ctx *ctx) { return ctx ? ctx->launches : 0; }

ALS_API int als_timer_start(als_ctx *ctx) {
  ALS_REQUIRE(ctx, "als_timer_start: ctx is NULL");
  ALS_CUDA(cudaEventRecord(ctx->ev0, ctx->stream));
  return ALS_OK;
}

ALS_API int als_timer_stop(als_ctx *ctx, float *ms) {
  ALS_REQUIRE(ctx && ms, "als_timer_stop: NULL argument");
  ALS_CUDA(cudaEventRecord(ctx->ev1, ctx->stream));
  ALS_CUDA(cudaEventSynchronize(ctx->ev1));
  ALS_CUDA(cudaEventElapsedTime(ms, ctx->ev0, ctx->ev1));
  return ALS_OK;
}

ALS_API int als_flush_l2(als_ctx *ctx, int64_t bytes) {
  ALS_REQUIRE(ctx && bytes > 0, "als_flush_l2: bad argument");
  static float *flush = nullptr;  // separate from scratch: scratch holds live solver state
  static int64_t flush_bytes = 0;
  if (bytes > flush_bytes) {
    if (flush) ALS_CUDA(cudaFree(flush));
    ALS_CUDA(cudaMalloc(&flush, bytes));
    flush_bytes = bytes;
  }
  fill_kernel<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(flush, bytes / 4, 1.0f);
  ALS_CUDA(cudaGetLastError());
  return ALS_OK;
}

ALS_API int als_profile_enable(als_ctx *ctx, int on) {
  ALS_REQUIRE(ctx, "als_profile_enable: ctx is NULL");
  ctx->profiling = on != 0;
  return ALS_OK;
}

ALS_API int als_profile_read(als_ctx *ctx, int which, double *ms_total, int64_t *launches) {
  ALS_REQUIRE(ctx && which >= 0 && which < 8 && ms_total && launches, "als_profile_read: bad argument");
  ALS_CUDA(cudaSetDevice(ctx->device));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  std::vector<cudaEvent_t> &ev = ctx->prof_events[which];
  double total = 0.0;
  int64_t n = 0;
  for (size_t i = 0; i + 1 < ev.size(); i += 2) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, ev[i], ev[i + 1]) == cudaSuccess) {
      total += ms;
      ++n;
    }
  }
  for (cudaEvent_t e : ev) cudaEventDestroy(e);
  ev.clear();
  *ms_total = total;
  *launches = n;
  return ALS_OK;
}

ALS_API int als_host_alloc(void **ptr, int64_t bytes) {
  ALS_REQUIRE(ptr && bytes >= 0, "als_host_alloc: bad argument");
  ALS_CUDA(cudaMallocHost(ptr, (size_t)std::max<int64_t>(bytes, 1)));
  return ALS_OK;
}

ALS_API int als_host_free(void *ptr) {
  if (ptr) ALS_CUDA(cudaFreeHost(ptr));
  return ALS_OK;
}

// ---- device memory of the caller ------------------------------------------------------------------
// ALS_E_INVALID unless p is device memory of ctx's device, or managed memory
static int require_device_memory(als_ctx *ctx, const char *who, const char *what, const void *p) {
  cudaPointerAttributes at;
  const cudaError_t e = cudaPointerGetAttributes(&at, p);
  cudaGetLastError();  // an unregistered host pointer may leave an error behind on older drivers
  if (e == cudaSuccess && at.type == cudaMemoryTypeManaged) return ALS_OK;
  if (e == cudaSuccess && at.type == cudaMemoryTypeDevice && at.device == ctx->device) return ALS_OK;
  if (e == cudaSuccess && at.type == cudaMemoryTypeDevice)
    set_error("%s: %s is memory of device %d, not of the context's device %d", who, what, at.device, ctx->device);
  else
    set_error("%s: %s is not device memory (a host pointer, or no CUDA allocation)", who, what);
  return ALS_E_INVALID;
}

// ctx->stream continues after the work queued so far on the caller's stream (0: none)
static int wait_for_producer(als_ctx *ctx, uint64_t producer_stream) {
  if (!producer_stream) return ALS_OK;
  cudaEvent_t ev;
  ALS_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  cudaError_t e = cudaEventRecord(ev, (cudaStream_t)(uintptr_t)producer_stream);
  if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->stream, ev, 0);
  cudaEventDestroy(ev);  // released once the wait has been satisfied
  return e == cudaSuccess ? ALS_OK : cuda_fail(e, "ordering after the producer stream", __FILE__, __LINE__);
}

// ---- CSR ---------------------------------------------------------------------------------------
// Where the arrays of an upload are: host memory (indptr of 4 bytes per entry for als_csr_upload, 8 for the 64-bit
// entries; fp32 values) or, for als_csr_upload_device, device memory of any of the widths it takes.
struct CsrArrays {
  const void *indptr;
  int indptr_bytes;
  const void *indices;
  int index_bytes;
  const void *data;
  int data_bytes;
  bool device;
};

// The one builder behind the four uploads: the checks, the rebase of a row shard (indptr[0] != 0), the arrays of the
// residency, the copies and the layout.  A host int32 indptr is als_csr_upload's: int32 limits on nnz too, and its int32
// indices are copied as they are; the 64-bit entries narrow the indices while they are staged and refuse any outside
// [0, cols).  Device arrays are read by device kernels instead of the staging threads: the indptr comes to the host
// (8 bytes per row, for the layout), the indices and values never do; the checks and their messages are the same.
static int csr_build(const char *who, bool host, als_ctx *ctx, int64_t rows, int64_t cols, int64_t nnz,
                     const CsrArrays &a, int64_t row_offset, als_csr **out) {
  const bool int32_entry = !a.device && a.indptr_bytes == 4;
  ALS_REQUIRE(ctx && out && a.indptr, "%s: NULL argument", who);
  ALS_REQUIRE(a.index_bytes == 4 || a.index_bytes == 8, "%s: index_bytes must be 4 or 8, got %d", who, a.index_bytes);
  ALS_REQUIRE(a.indptr_bytes == 4 || a.indptr_bytes == 8, "%s: indptr_bytes must be 4 or 8, got %d", who, a.indptr_bytes);
  ALS_REQUIRE(a.data_bytes == 4 || a.data_bytes == 8, "%s: data_bytes must be 4 or 8, got %d", who, a.data_bytes);
  ALS_REQUIRE(rows >= 0 && cols >= 0 && nnz >= 0, "%s: negative shape", who);
  if (int32_entry)
    ALS_REQUIRE(nnz < (int64_t)INT32_MAX && rows < (int64_t)INT32_MAX && cols < (int64_t)INT32_MAX,
                "%s: int32 CSR only (rows, cols, nnz < 2^31), like implicit/gpu/matrix.h:93-100", who);
  else
    ALS_REQUIRE(rows < (int64_t)INT32_MAX && cols < (int64_t)INT32_MAX, "%s: rows and cols must be < 2^31 - 1", who);
  std::vector<int64_t> ip;
  int64_t base = 0, bad_row = -1;
  if (a.device) {
    ALS_CUDA(cudaSetDevice(ctx->device));
    int rc = require_device_memory(ctx, who, "indptr", a.indptr);
    if (rc == ALS_OK && nnz > 0 && a.indices) rc = require_device_memory(ctx, who, "indices", a.indices);
    if (rc == ALS_OK && nnz > 0 && a.data) rc = require_device_memory(ctx, who, "data", a.data);
    if (rc == ALS_OK) rc = device_indptr(ctx, a.indptr, a.indptr_bytes, rows, ip, &base, &bad_row);
    if (rc != ALS_OK) return rc;
  } else {
    auto at = [&](int64_t r) -> int64_t {
      return a.indptr_bytes == 8 ? ((const int64_t *)a.indptr)[r] : ((const int32_t *)a.indptr)[r];
    };
    base = at(0);
    ip.resize((size_t)rows + 1);
    for (int64_t r = 0; r <= rows; ++r) ip[r] = at(r) - base;
    for (int64_t r = 0; r < rows && bad_row < 0; ++r)
      if (ip[r + 1] < ip[r]) bad_row = r;
  }
  ALS_REQUIRE(base >= 0 && ip[rows] == nnz, "%s: indptr[rows] - indptr[0] = %lld != nnz = %lld", who, (long long)ip[rows],
              (long long)nnz);
  // device arrays are taken whole: nnz is their length, so a positive indptr[0] would read past their end
  ALS_REQUIRE(!a.device || base == 0, "%s: indptr[0] = %lld, not 0: device arrays hold the matrix from its first entry",
              who, (long long)base);
  ALS_REQUIRE(nnz == 0 || (a.indices && a.data), "%s: indices/data NULL with nnz > 0", who);
  ALS_REQUIRE(bad_row < 0, "%s: indptr is not monotone at row %lld", who, (long long)bad_row);
  *out = nullptr;
  ALS_CUDA(cudaSetDevice(ctx->device));
  CsrHolder c = new_csr(ctx);
  c->rows = rows;
  c->cols = cols;
  c->nnz = nnz;
  c->row_offset = row_offset;
  c->host = host;
  const char *ix = (const char *)a.indices + base * a.index_bytes;
  const char *dv = (const char *)a.data + base * a.data_bytes;
  int64_t bad = -1;
  int rc = csr_alloc(ctx, c.get());
  if (rc == ALS_OK && a.device) {
    rc = device_entries(ctx, c.get(), ix, a.index_bytes, dv, a.data_bytes, &bad);
  } else if (rc == ALS_OK) {
    const float *data = (const float *)dv;
    rc = int32_entry ? h2d_copy(ctx, c->indices, ix, sizeof(int32_t) * nnz)
                     : h2d_indices(ctx, c->indices, ix, a.index_bytes, nnz, cols, &bad, host);
    if (rc == ALS_OK)
      rc = host ? fill_host_values(ctx, c.get(), c->data, nnz,
                                   [&](float *v, int64_t i0, int64_t m) { memcpy(v, data + i0, sizeof(float) * m); })
                : h2d_copy(ctx, c->data, data, sizeof(float) * nnz);
  }
  if (rc == ALS_OK) rc = csr_layout(ctx, c.get(), ip.data());
  if (rc != ALS_OK) {
    if (bad >= 0) {
      int64_t v = 0;
      if (a.device) {
        if (cudaMemcpy(&v, ix + bad * a.index_bytes, a.index_bytes, cudaMemcpyDeviceToHost) != cudaSuccess) cudaGetLastError();
        if (a.index_bytes == 4) v = (int32_t)v;  // little-endian: the low half
      } else {
        v = a.index_bytes == 8 ? ((const int64_t *)ix)[bad] : ((const int32_t *)ix)[bad];
      }
      set_error("%s: indices[%lld] = %lld is outside [0, %lld)", who, (long long)(base + bad), (long long)v, (long long)cols);
    }
    return rc;
  }
  *out = c.release();
  return ALS_OK;
}

ALS_API int als_csr_upload(als_ctx *ctx, int64_t rows, int64_t cols, int64_t nnz, const int32_t *indptr,
                           const int32_t *indices, const float *data, int64_t row_offset, als_csr **out) {
  return csr_build("als_csr_upload", false, ctx, rows, cols, nnz, CsrArrays{indptr, 4, indices, 4, data, 4, false},
                   row_offset, out);
}

// als_csr_upload_host64 keeps indices / data in page-locked host memory (always segmented) instead of uploading them
ALS_API int als_csr_upload64(als_ctx *ctx, int64_t rows, int64_t cols, int64_t nnz, const int64_t *indptr,
                             const void *indices, int index_bytes, const float *data, int64_t row_offset, als_csr **out) {
  return csr_build("als_csr_upload64", false, ctx, rows, cols, nnz,
                   CsrArrays{indptr, 8, indices, index_bytes, data, 4, false}, row_offset, out);
}

ALS_API int als_csr_upload_host64(als_ctx *ctx, int64_t rows, int64_t cols, int64_t nnz, const int64_t *indptr,
                                  const void *indices, int index_bytes, const float *data, int64_t row_offset, als_csr **out) {
  return csr_build("als_csr_upload_host64", true, ctx, rows, cols, nnz,
                   CsrArrays{indptr, 8, indices, index_bytes, data, 4, false}, row_offset, out);
}

ALS_API int als_csr_upload_device(als_ctx *ctx, int64_t rows, int64_t cols, int64_t nnz, const void *indptr,
                                  int indptr_bytes, const void *indices, int index_bytes, const void *data, int data_bytes,
                                  int64_t row_offset, uint64_t producer_stream, als_csr **out) {
  ALS_REQUIRE(ctx && out, "als_csr_upload_device: NULL argument");
  ALS_CUDA(cudaSetDevice(ctx->device));
  const int rc = wait_for_producer(ctx, producer_stream);
  if (rc != ALS_OK) return rc;
  return csr_build("als_csr_upload_device", false, ctx, rows, cols, nnz,
                   CsrArrays{indptr, indptr_bytes, indices, index_bytes, data, data_bytes, true}, row_offset, out);
}

ALS_API int als_csr_is_host(const als_csr *csr, int *host) {
  ALS_REQUIRE(csr && host, "als_csr_is_host: NULL argument");
  *host = csr->host ? 1 : 0;
  return ALS_OK;
}

ALS_API int als_csr_segment_count(const als_csr *csr, int64_t *n) {
  ALS_REQUIRE(csr && n, "als_csr_segment_count: NULL argument");
  *n = csr->segs.empty() ? 1 : (int64_t)csr->segs.size();
  return ALS_OK;
}

ALS_API int als_csr_generate(als_ctx *ctx, int64_t rows, int64_t cols, int64_t nnz_target, uint64_t seed, als_csr **out) {
  ALS_REQUIRE(ctx && out, "als_csr_generate: NULL argument");
  ALS_REQUIRE(rows > 0 && cols > 0 && nnz_target > 0, "als_csr_generate: empty shape");
  *out = nullptr;
  ALS_CUDA(cudaSetDevice(ctx->device));
  return als::csr_generate_power_law(ctx, rows, cols, nnz_target, seed, out);
}

ALS_API int als_factors_fill_uniform(als_ctx *ctx, als_factors *f, uint64_t seed, float scale) {
  ALS_REQUIRE(ctx && f, "als_factors_fill_uniform: NULL argument");
  ALS_CUDA(cudaSetDevice(ctx->device));
  return als::factors_fill_uniform(ctx, f, seed, scale);
}

ALS_API int als_factors_fill_pcg64(als_ctx *ctx, als_factors *f, uint64_t state_hi, uint64_t state_lo, uint64_t inc_hi,
                                   uint64_t inc_lo, int has_uint32, uint32_t uinteger, float scale) {
  ALS_REQUIRE(ctx && f, "als_factors_fill_pcg64: NULL argument");
  ALS_REQUIRE(has_uint32 == 0 || has_uint32 == 1, "als_factors_fill_pcg64: has_uint32=%d is not 0 or 1", has_uint32);
  ALS_CUDA(cudaSetDevice(ctx->device));
  return als::factors_fill_pcg64(ctx, f, state_hi, state_lo, inc_hi, inc_lo, has_uint32, uinteger, scale);
}

ALS_API int als_csr_transpose(als_ctx *ctx, const als_csr *in, als_csr **out) {
  ALS_REQUIRE(ctx && in && out, "als_csr_transpose: NULL argument");
  return als::csr_transpose(ctx, in, out);
}

ALS_API int als_csr_column_counts(als_ctx *ctx, const als_csr *csr, int64_t *counts) {
  ALS_REQUIRE(ctx && csr && (counts || csr->cols == 0), "als_csr_column_counts: NULL argument");
  return als::csr_column_counts(ctx, csr, counts);
}

ALS_API int als_csr_transpose_pieces(als_ctx *ctx, const als_csr *shard, int n, const int64_t *col_bounds,
                                     als_csr **pieces) {
  ALS_REQUIRE(ctx && shard && col_bounds && pieces && n >= 1, "als_csr_transpose_pieces: NULL argument or n < 1");
  ALS_REQUIRE(col_bounds[0] == 0 && col_bounds[n] == shard->cols,
              "als_csr_transpose_pieces: col_bounds must run from 0 to %lld", (long long)shard->cols);
  for (int q = 0; q < n; ++q)
    ALS_REQUIRE(col_bounds[q] <= col_bounds[q + 1], "als_csr_transpose_pieces: col_bounds decrease at %d", q);
  if (shard->host) {
    set_error("als_csr_transpose_pieces: a host-resident CSR cannot be cut into pieces");
    return ALS_E_UNSUPPORTED;
  }
  return als::csr_transpose_pieces(ctx, shard, n, col_bounds, pieces);
}

ALS_API int als_csr_merge_rows(als_ctx *ctx, int n, const als_csr *const *pieces, int64_t cols, int64_t row_offset,
                               als_csr **out) {
  ALS_REQUIRE(ctx && pieces && out && n >= 1, "als_csr_merge_rows: NULL argument or n < 1");
  for (int p = 0; p < n; ++p) {
    ALS_REQUIRE(pieces[p], "als_csr_merge_rows: piece %d is NULL", p);
    ALS_REQUIRE(pieces[p]->rows == pieces[0]->rows, "als_csr_merge_rows: piece %d has %lld rows, piece 0 has %lld", p,
                (long long)pieces[p]->rows, (long long)pieces[0]->rows);
    if (pieces[p]->host) {
      set_error("als_csr_merge_rows: piece %d is host-resident", p);
      return ALS_E_UNSUPPORTED;
    }
  }
  ALS_REQUIRE(cols >= 0 && cols < (int64_t)INT32_MAX && row_offset >= 0, "als_csr_merge_rows: bad cols or row_offset");
  return als::csr_merge_rows(ctx, n, pieces, cols, row_offset, out);
}

ALS_API int als_csr_concat_rows(als_ctx *ctx, int n, const als_csr *const *pieces, int64_t cols, int64_t row_offset,
                                als_csr **out) {
  ALS_REQUIRE(ctx && pieces && out && n >= 1, "als_csr_concat_rows: NULL argument or n < 1");
  ALS_REQUIRE(cols >= 0 && cols < (int64_t)INT32_MAX && row_offset >= 0, "als_csr_concat_rows: bad cols or row_offset");
  *out = nullptr;
  int64_t rows = 0;
  for (int p = 0; p < n; ++p) {
    ALS_REQUIRE(pieces[p], "als_csr_concat_rows: piece %d is NULL", p);
    ALS_REQUIRE(pieces[p]->cols <= cols, "als_csr_concat_rows: piece %d has %lld columns, more than %lld", p,
                (long long)pieces[p]->cols, (long long)cols);
    if (pieces[p]->host) {
      set_error("als_csr_concat_rows: piece %d is host-resident", p);
      return ALS_E_UNSUPPORTED;
    }
    rows += pieces[p]->rows;
  }
  ALS_REQUIRE(rows < (int64_t)INT32_MAX, "als_csr_concat_rows: %lld rows in all, more than 2^31 - 2", (long long)rows);
  return als::csr_concat_rows(ctx, n, pieces, cols, row_offset, out);
}

ALS_API int als_mem_peak(als_ctx *ctx, int64_t *used_bytes, int64_t *peak_bytes) {
  ALS_REQUIRE(ctx && used_bytes && peak_bytes, "als_mem_peak: NULL argument");
  ALS_CUDA(cudaSetDevice(ctx->device));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  cudaMemPool_t pool;
  ALS_CUDA(cudaDeviceGetDefaultMemPool(&pool, ctx->device));
  uint64_t used = 0, high = 0, zero = 0;
  ALS_CUDA(cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemCurrent, &used));
  ALS_CUDA(cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemHigh, &high));
  ALS_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrUsedMemHigh, &zero));  // restarts the mark at `used`
  *used_bytes = (int64_t)used;
  *peak_bytes = (int64_t)high;
  return ALS_OK;
}

ALS_API int als_csr_slice_rows(als_ctx *ctx, const als_csr *in, int64_t r0, int64_t r1, als_csr **out) {
  ALS_REQUIRE(ctx && in && out, "als_csr_slice_rows: NULL argument");
  ALS_REQUIRE(0 <= r0 && r0 <= r1 && r1 <= in->rows, "als_csr_slice_rows: bad row range [%lld, %lld)", (long long)r0,
              (long long)r1);
  ALS_REQUIRE(in->row_offset == 0, "als_csr_slice_rows: cannot slice a shard");
  *out = nullptr;
  if (in->host) {
    set_error("als_csr_slice_rows: a host-resident CSR cannot be sliced into shards; upload it with als_csr_upload64 for a "
              "multi-GPU fit");
    return ALS_E_UNSUPPORTED;
  }
  ALS_CUDA(cudaSetDevice(ctx->device));
  std::vector<int64_t> ip64;
  int rc = csr_indptr64(ctx, in, ip64);
  if (rc != ALS_OK) return rc;
  CsrHolder c = new_csr(ctx);
  c->rows = r1 - r0;
  c->cols = in->cols;
  c->nnz = ip64[r1] - ip64[r0];
  c->row_offset = r0;
  c->owns = false;
  c->indices = in->indices;
  c->data = in->data;
  if (!in->segs.empty()) {  // a shard of a segmented CSR can itself exceed 2^31 nonzeros: a segmented view
    rc = make_segments(ctx, c.get(), ip64.data() + r0);
  } else {  // a view into the parent's indptr: absolute positions into its indices / data
    c->indptr = in->indptr + r0;
    const std::vector<int32_t> ip(ip64.begin() + r0, ip64.begin() + r1 + 1);
    rc = build_schedule(ctx, c.get(), ip.data());
  }
  if (rc != ALS_OK) return rc;
  *out = c.release();
  return ALS_OK;
}

ALS_API int als_csr_scale(als_ctx *ctx, als_csr *csr, float alpha) {
  ALS_REQUIRE(ctx && csr, "als_csr_scale: NULL argument");
  if (csr->nnz == 0) return ALS_OK;
  ALS_CUDA(cudaSetDevice(ctx->device));
  // segments are consecutive blocks of one array: the first one starts the CSR's values
  float *data = csr->segs.empty() ? csr->data : csr->segs[0]->data;
  if (csr->host) {
    // the same single fp32 rounding as scale_kernel, in the page-locked array, once no queued copy reads it any more;
    // the weight range is folded on the way
    ALS_CUDA(cudaStreamSynchronize(ctx->stream));
    ALS_CUDA(cudaStreamSynchronize(ctx->copy));
    return fill_host_values(ctx, csr, data, csr->nnz, [alpha](float *v, int64_t, int64_t m) {
      for (int64_t i = 0; i < m; ++i) v[i] *= alpha;
    });
  }
  csr->wmax_valid = false;
  scale_kernel<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(data, csr->nnz, alpha);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  return ALS_OK;
}

ALS_API int als_csr_shape(const als_csr *csr, int64_t *rows, int64_t *cols, int64_t *nnz) {
  ALS_REQUIRE(csr, "als_csr_shape: NULL");
  if (rows) *rows = csr->rows;
  if (cols) *cols = csr->cols;
  if (nnz) *nnz = csr->nnz;
  return ALS_OK;
}

ALS_API int als_csr_download(als_ctx *ctx, const als_csr *csr, int32_t *indptr, int32_t *indices, float *data) {
  ALS_REQUIRE(ctx && csr, "als_csr_download: NULL argument");
  ALS_REQUIRE(csr->nnz < (int64_t)INT32_MAX, "als_csr_download: %lld nonzeros need a 64-bit indptr: use als_csr_download64",
              (long long)csr->nnz);
  std::vector<int64_t> ip64(indptr ? (size_t)csr->rows + 1 : 0);
  int rc = als_csr_download64(ctx, csr, indptr ? ip64.data() : nullptr, indices, data);
  if (rc == ALS_OK && indptr)
    for (int64_t r = 0; r <= csr->rows; ++r) indptr[r] = (int32_t)ip64[r];
  return rc;
}

ALS_API int als_csr_download64(als_ctx *ctx, const als_csr *csr, int64_t *indptr, int32_t *indices, float *data) {
  ALS_REQUIRE(ctx && csr, "als_csr_download64: NULL argument");
  ALS_CUDA(cudaSetDevice(ctx->device));
  std::vector<int64_t> ip;
  int rc = csr_indptr64(ctx, csr, ip);
  if (rc != ALS_OK) return rc;
  const int64_t base = ip[0];  // a row-slice view keeps absolute positions into its parent's arrays: rebase
  if (indptr)
    for (int64_t r = 0; r <= csr->rows; ++r) indptr[r] = ip[r] - base;
  if (csr->host) {  // the page-locked arrays themselves (csr_indptr64 synchronised the compute stream)
    if (indices && csr->nnz) memcpy(indices, csr->indices + base, sizeof(int32_t) * csr->nnz);
    if (data && csr->nnz) memcpy(data, csr->data + base, sizeof(float) * csr->nnz);
    return ALS_OK;
  }
  if (indices && csr->nnz)
    ALS_CUDA(cudaMemcpy(indices, csr->indices + base, sizeof(int32_t) * csr->nnz, cudaMemcpyDeviceToHost));
  if (data && csr->nnz)
    ALS_CUDA(cudaMemcpy(data, csr->data + base, sizeof(float) * csr->nnz, cudaMemcpyDeviceToHost));
  return ALS_OK;
}

ALS_API int als_csr_destroy(als_csr *csr) {
  if (!csr) return ALS_OK;
  als_ctx *ctx = csr->ctx;
  if (ctx) {
    cudaSetDevice(ctx->device);
    // stream-ordered frees: everything queued so far on the compute stream (which every other stream is joined
    // into before an entry point returns) still sees the arrays
    if (csr->owns && csr->host) {
      // page-locked arrays: every copy out of them is queued on the copy stream and waited for by the compute stream
      cudaStreamSynchronize(ctx->stream);
      cudaStreamSynchronize(ctx->copy);
      cudaFreeHost(csr->indices);
      cudaFreeHost(csr->data);
    } else if (csr->owns) {
      dev_free(ctx, csr->indptr);
      dev_free(ctx, csr->indices);
      dev_free(ctx, csr->data);
    }
    dev_free(ctx, csr->wmax_dev);
    dev_free(ctx, csr->sorted_indptr);
    dev_free(ctx, csr->sorted_indices);
    dev_free(ctx, csr->work);
    dev_free(ctx, csr->finish);
    dev_free(ctx, csr->chunks);
    dev_free(ctx, csr->chunk_owner);
    for (als_csr *seg : csr->segs) als_csr_destroy(seg);
    dev_free(ctx, csr->seg_indptr);
  }
  delete csr;
  return ALS_OK;
}

// ---- factors -----------------------------------------------------------------------------------
ALS_API int als_factors_create(als_ctx *ctx, int64_t rows, int factors, als_factors **out) {
  ALS_REQUIRE(ctx && out, "als_factors_create: NULL argument");
  ALS_REQUIRE(rows >= 0 && factors > 0, "als_factors_create: bad shape (%lld, %d)", (long long)rows, factors);
  ALS_REQUIRE(factors <= 1024, "als_factors_create: factors=%d > 1024 is not supported", factors);
  *out = nullptr;
  ALS_CUDA(cudaSetDevice(ctx->device));
  als_factors *f = new als_factors();
  f->ctx = ctx;
  f->rows = rows;
  f->f = factors;
  f->ld = factors <= 128 ? round_up(factors, 16) : round_up(factors, 128);  // wide models: whole warps per factor row
  const int64_t bytes = sizeof(float) * std::max<int64_t>(rows, 1) * f->ld;
  // with a communicator the matrix will be exported over IPC (multi-GPU fit): take a cudaMalloc block right away
  f->pooled = ctx->world == 1;
  if (f->pooled) {
    int arc = dev_alloc(ctx, (void **)&f->d, bytes);
    if (arc != ALS_OK) {
      delete f;
      return arc;
    }
  } else {
    cudaError_t e = cudaMalloc(&f->d, bytes);
    if (e != cudaSuccess) {
      delete f;
      return cuda_fail(e, "cudaMalloc (factor matrix)", __FILE__, __LINE__);
    }
  }
  ALS_CUDA(cudaMemsetAsync(f->d, 0, bytes, ctx->stream));
  *out = f;
  return ALS_OK;
}

ALS_API int als_factors_upload(als_ctx *ctx, als_factors *f, const float *host, int64_t row0, int64_t nrows) {
  ALS_REQUIRE(ctx && f && host, "als_factors_upload: NULL argument");
  ALS_REQUIRE(row0 >= 0 && nrows >= 0 && row0 + nrows <= f->rows, "als_factors_upload: rows [%lld, %lld) out of range",
              (long long)row0, (long long)(row0 + nrows));
  if (nrows == 0) return ALS_OK;
  ALS_CUDA(cudaSetDevice(ctx->device));
  // ordered after any kernel already queued on the compute stream that reads/writes f
  if (f->f == f->ld) {  // no padding: one contiguous copy (a pitched copy of 256-byte rows is several times slower)
    int hrc = h2d_copy(ctx, f->d + row0 * f->ld, host, sizeof(float) * f->f * nrows);
    if (hrc != ALS_OK) return hrc;
  } else {
    ALS_CUDA(cudaMemcpy2DAsync(f->d + row0 * f->ld, sizeof(float) * f->ld, host, sizeof(float) * f->f,
                               sizeof(float) * f->f, nrows, cudaMemcpyHostToDevice, ctx->stream));
  }
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));  // host buffer may be pageable and reused by the caller
  return ALS_OK;
}

ALS_API int als_factors_download(als_ctx *ctx, const als_factors *f, float *host, int64_t row0, int64_t nrows) {
  ALS_REQUIRE(ctx && f && host, "als_factors_download: NULL argument");
  ALS_REQUIRE(row0 >= 0 && nrows >= 0 && row0 + nrows <= f->rows,
              "als_factors_download: rows [%lld, %lld) out of range", (long long)row0, (long long)(row0 + nrows));
  if (nrows == 0) return ALS_OK;
  ALS_CUDA(cudaSetDevice(ctx->device));
  if (f->f == f->ld) {
    ALS_CUDA(cudaMemcpyAsync(host, f->d + row0 * f->ld, sizeof(float) * f->f * nrows, cudaMemcpyDeviceToHost, ctx->stream));
  } else {
    ALS_CUDA(cudaMemcpy2DAsync(host, sizeof(float) * f->f, f->d + row0 * f->ld, sizeof(float) * f->ld,
                               sizeof(float) * f->f, nrows, cudaMemcpyDeviceToHost, ctx->stream));
  }
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return ALS_OK;
}

ALS_API int als_factors_import_device(als_ctx *ctx, als_factors *f, const float *src, int64_t ld, int64_t row0,
                                      int64_t nrows, uint64_t producer_stream) {
  const char *who = "als_factors_import_device";
  ALS_REQUIRE(ctx && f && (src || nrows == 0), "%s: NULL argument", who);
  ALS_REQUIRE(row0 >= 0 && nrows >= 0 && row0 + nrows <= f->rows, "%s: rows [%lld, %lld) out of range", who,
              (long long)row0, (long long)(row0 + nrows));
  ALS_REQUIRE(ld >= f->f, "%s: a row stride of %lld elements is shorter than a row of %d factors", who, (long long)ld, f->f);
  if (nrows == 0) return ALS_OK;
  ALS_CUDA(cudaSetDevice(ctx->device));
  int rc = require_device_memory(ctx, who, "src", src);
  if (rc == ALS_OK) rc = wait_for_producer(ctx, producer_stream);
  if (rc != ALS_OK) return rc;
  float *dst = f->d + row0 * f->ld;
  ALS_CUDA(cudaMemcpy2DAsync(dst, sizeof(float) * f->ld, src, sizeof(float) * ld, sizeof(float) * f->f, nrows,
                             cudaMemcpyDeviceToDevice, ctx->stream));
  if (f->ld > f->f)  // the padding columns read as zeros, as after als_factors_upload
    ALS_CUDA(cudaMemset2DAsync(dst + f->f, sizeof(float) * f->ld, 0, sizeof(float) * (f->ld - f->f), nrows, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));  // the caller may free or refill src once this returns
  return ALS_OK;
}

ALS_API int als_factors_export_device(als_ctx *ctx, const als_factors *f, float *dst, int64_t ld, int64_t row0,
                                      int64_t nrows) {
  const char *who = "als_factors_export_device";
  ALS_REQUIRE(ctx && f && (dst || nrows == 0), "%s: NULL argument", who);
  ALS_REQUIRE(row0 >= 0 && nrows >= 0 && row0 + nrows <= f->rows, "%s: rows [%lld, %lld) out of range", who,
              (long long)row0, (long long)(row0 + nrows));
  ALS_REQUIRE(ld >= f->f, "%s: a row stride of %lld elements is shorter than a row of %d factors", who, (long long)ld, f->f);
  if (nrows == 0) return ALS_OK;
  ALS_CUDA(cudaSetDevice(ctx->device));
  const int rc = require_device_memory(ctx, who, "dst", dst);
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaMemcpy2DAsync(dst, sizeof(float) * ld, f->d + row0 * f->ld, sizeof(float) * f->ld, sizeof(float) * f->f,
                             nrows, cudaMemcpyDeviceToDevice, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));  // complete when this returns: any stream may read dst
  return ALS_OK;
}

ALS_API int als_device_alloc(als_ctx *ctx, int64_t bytes, void **ptr) {
  ALS_REQUIRE(ctx && ptr && bytes >= 0, "als_device_alloc: bad argument");
  ALS_CUDA(cudaSetDevice(ctx->device));
  ALS_CUDA(cudaMalloc(ptr, (size_t)std::max<int64_t>(bytes, 16)));
  return ALS_OK;
}

ALS_API int als_device_free(als_ctx *ctx, void *ptr) {
  ALS_REQUIRE(ctx, "als_device_free: ctx is NULL");
  if (!ptr) return ALS_OK;
  ALS_CUDA(cudaSetDevice(ctx->device));
  ALS_CUDA(cudaFree(ptr));
  return ALS_OK;
}

ALS_API int als_pool_alloc(als_ctx *ctx, int64_t bytes, void **ptr) {
  ALS_REQUIRE(ctx && ptr && bytes >= 0, "als_pool_alloc: bad argument");
  ALS_CUDA(cudaSetDevice(ctx->device));
  return dev_alloc(ctx, ptr, bytes);
}

ALS_API int als_pool_free(als_ctx *ctx, void *ptr) {
  ALS_REQUIRE(ctx, "als_pool_free: ctx is NULL");
  if (!ptr) return ALS_OK;
  ALS_CUDA(cudaSetDevice(ctx->device));
  dev_free(ctx, ptr);
  return ALS_OK;
}

ALS_API int als_factors_has_nan(als_ctx *ctx, const als_factors *f, int *has_nan) {
  ALS_REQUIRE(ctx && f && has_nan, "als_factors_has_nan: NULL argument");
  ALS_CUDA(cudaSetDevice(ctx->device));
  int *flag = reinterpret_cast<int *>(ctx->counters + kCtrHasNan);
  ALS_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), ctx->stream));
  has_nan_kernel<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(f->d, f->rows * (int64_t)f->ld, flag);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  ALS_CUDA(cudaMemcpyAsync(has_nan, flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return ALS_OK;
}

ALS_API int als_factors_shape(const als_factors *f, int64_t *rows, int *factors, int *stride) {
  ALS_REQUIRE(f, "als_factors_shape: NULL");
  if (rows) *rows = f->rows;
  if (factors) *factors = f->f;
  if (stride) *stride = f->ld;
  return ALS_OK;
}

ALS_API int als_factors_ipc_export(als_ctx *ctx, const als_factors *cf, void *handle) {
  ALS_REQUIRE(ctx && cf && handle, "als_factors_ipc_export: NULL argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == ALS_IPC_HANDLE_BYTES, "IPC handle size");
  ALS_CUDA(cudaSetDevice(ctx->device));
  als_factors *f = const_cast<als_factors *>(cf);
  if (f->pooled) {
    // blocks of the stream-ordered pool cannot be exported with cudaIpcGetMemHandle: move the matrix (once)
    const int64_t bytes = sizeof(float) * std::max<int64_t>(f->rows, 1) * f->ld;
    Dev<float> moved;
    const int rc = moved.alloc_cuda(ctx, bytes);
    if (rc != ALS_OK) return rc;
    ALS_CUDA(cudaMemcpyAsync(moved, f->d, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    ALS_CUDA(cudaStreamSynchronize(ctx->stream));
    dev_free(ctx, f->d);
    f->d = moved.release();
    f->pooled = false;
  }
  cudaIpcMemHandle_t h;
  ALS_CUDA(cudaIpcGetMemHandle(&h, f->d));
  memcpy(handle, &h, sizeof(h));
  return ALS_OK;
}

ALS_API int als_factors_ipc_detach(als_ctx *ctx, als_factors *f) {
  ALS_REQUIRE(ctx && f, "als_factors_ipc_detach: NULL argument");
  ALS_CUDA(cudaSetDevice(ctx->device));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  for (void *m : f->peer_maps) cudaIpcCloseMemHandle(m);
  f->peer_maps.clear();
  if (f->peers_dev) cudaFree(f->peers_dev);
  f->peers_dev = nullptr;
  f->n_peers = 0;
  return ALS_OK;
}

ALS_API int als_factors_ipc_attach(als_ctx *ctx, als_factors *f, int rank, int world, const void *handles) {
  ALS_REQUIRE(ctx && f && handles, "als_factors_ipc_attach: NULL argument");
  ALS_REQUIRE(world >= 1 && rank >= 0 && rank < world, "als_factors_ipc_attach: bad rank %d / world %d", rank, world);
  int rc = als_factors_ipc_detach(ctx, f);
  if (rc != ALS_OK) return rc;
  if (world == 1) return ALS_OK;
  std::vector<float *> ptrs;
  for (int r = 0; r < world; ++r) {
    if (r == rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, (const char *)handles + (size_t)r * ALS_IPC_HANDLE_BYTES, sizeof(h));
    void *m = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&m, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      als_factors_ipc_detach(ctx, f);
      return cuda_fail(e, "cudaIpcOpenMemHandle (peer replica)", __FILE__, __LINE__);
    }
    f->peer_maps.push_back(m);
    ptrs.push_back((float *)m);
  }
  ALS_CUDA(cudaMalloc(&f->peers_dev, sizeof(float *) * ptrs.size()));
  ALS_CUDA(cudaMemcpy(f->peers_dev, ptrs.data(), sizeof(float *) * ptrs.size(), cudaMemcpyHostToDevice));
  f->n_peers = (int)ptrs.size();
  return ALS_OK;
}

ALS_API int als_factors_destroy(als_factors *f) {
  if (!f) return ALS_OK;
  if (f->ctx && (f->n_peers || !f->peer_maps.empty())) als_factors_ipc_detach(f->ctx, f);
  if (f->ctx) {
    cudaSetDevice(f->ctx->device);
    if (f->pooled) {
      dev_free(f->ctx, f->d);
    } else {
      cudaStreamSynchronize(f->ctx->stream);
      cudaFree(f->d);
    }
  }
  delete f;
  return ALS_OK;
}

// ---- hot path ----------------------------------------------------------------------------------
static int check_half(const char *who, als_ctx *ctx, const als_csr *C, const als_factors *X, const als_factors *Y) {
  ALS_REQUIRE(ctx && C && X && Y, "%s: NULL argument", who);
  ALS_REQUIRE(C->ctx == ctx && X->ctx == ctx && Y->ctx == ctx, "%s: objects belong to different contexts", who);
  ALS_REQUIRE(X->f == Y->f, "%s: X has %d factors, Y has %d", who, X->f, Y->f);
  ALS_REQUIRE(C->cols == Y->rows, "%s: C has %lld columns but Y has %lld rows", who, (long long)C->cols,
              (long long)Y->rows);
  ALS_REQUIRE(C->row_offset + C->rows <= X->rows, "%s: C rows [%lld, %lld) exceed X's %lld rows", who,
              (long long)C->row_offset, (long long)(C->row_offset + C->rows), (long long)X->rows);
  return ensure_schedule(ctx, const_cast<als_csr *>(C));
}

ALS_API int als_gramian_read(als_ctx *ctx, const als_factors *Y, float *G_host) {
  ALS_REQUIRE(ctx && Y && G_host, "als_gramian_read: NULL argument");
  ALS_CUDA(cudaSetDevice(ctx->device));
  std::vector<float> tmp((size_t)Y->ld * Y->ld);
  ALS_CUDA(cudaMemcpyAsync(tmp.data(), ctx->G, sizeof(float) * tmp.size(), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < Y->f; ++i) memcpy(G_host + (size_t)i * Y->f, tmp.data() + (size_t)i * Y->ld, sizeof(float) * Y->f);
  return ALS_OK;
}

ALS_API int als_gramian(als_ctx *ctx, const als_factors *Y, float *G_host) {
  ALS_REQUIRE(ctx && Y, "als_gramian: NULL argument");
  ALS_CUDA(cudaSetDevice(ctx->device));
  int rc = launch_gramian(ctx, Y);
  if (rc != ALS_OK) return rc;
  return G_host ? als_gramian_read(ctx, Y, G_host) : ALS_OK;
}

// Reads the first row whose normal equations were not positive definite from bad_row[0, n) (n = 1: the half just run;
// 2: also the halves since the last als_solver_status) into *row, -1 for none (synchronises).  A row found is reported
// here and now: both slots are cleared, so nothing is left for a later call to find.
static int take_bad_row(als_ctx *ctx, int n, int64_t *row) {
  long long bad[2] = {LLONG_MAX, LLONG_MAX};
  ALS_CUDA(cudaMemcpyAsync(bad, ctx->bad_row, n * sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  const long long first = std::min(bad[0], bad[1]);
  if (row) *row = first == LLONG_MAX ? -1 : (int64_t)first;
  if (first == LLONG_MAX) return ALS_OK;
  const long long init[2] = {LLONG_MAX, LLONG_MAX};
  ALS_CUDA(cudaMemcpyAsync(ctx->bad_row, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  set_error("cholesky failed on row %lld: normal equations not positive definite. Try increasing the "
            "regularization parameter.", first);
  return ALS_E_NOT_POSDEF;
}

enum class Gram { kCompute, kHost, kPresent };  // the Gramian of a half: Y^T Y from Y, the caller's YtY_host, or ctx->G
enum class Solver { kCholesky, kCg };

// One half-iteration: the checks, the Gramian, G + reg I and the solver.  With sync_bad_row a Cholesky half reads its
// bad row back and fails with ALS_E_NOT_POSDEF; without, the row waits in bad_row for als_solver_status.
static int solve_half(const char *who, als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y, Gram gram,
                      const float *YtY_host, double reg, Solver solver, int cg_steps, bool sync_bad_row, int64_t *bad_row) {
  int rc = check_half(who, ctx, C, X, Y);
  if (rc != ALS_OK) return rc;
  ALS_REQUIRE(solver != Solver::kCg || cg_steps >= 0, "%s: cg_steps < 0", who);
  ALS_REQUIRE(gram != Gram::kHost || YtY_host, "%s: YtY is NULL", who);
  ALS_CUDA(cudaSetDevice(ctx->device));
  if (gram == Gram::kCompute) {
    rc = launch_gramian(ctx, Y);
    if (rc != ALS_OK) return rc;
  } else if (gram == Gram::kHost) {
    std::vector<float> tmp((size_t)Y->ld * Y->ld, 0.f);
    for (int i = 0; i < Y->f; ++i) memcpy(tmp.data() + (size_t)i * Y->ld, YtY_host + (size_t)i * Y->f, sizeof(float) * Y->f);
    ALS_CUDA(cudaMemcpyAsync(ctx->G, tmp.data(), sizeof(float) * tmp.size(), cudaMemcpyHostToDevice, ctx->stream));
    ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  rc = launch_regularize(ctx, Y->f, Y->ld, (float)reg);
  if (rc != ALS_OK) return rc;
  if (solver == Solver::kCg) return launch_cg(ctx, C, X, Y, cg_steps);
  rc = launch_cholesky(ctx, C, X, Y);
  if (rc != ALS_OK || !sync_bad_row) return rc;
  return take_bad_row(ctx, 1, bad_row);
}

ALS_API int als_least_squares(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y,
                              double regularization, int64_t *bad_row) {
  return solve_half("als_least_squares", ctx, C, X, Y, Gram::kCompute, nullptr, regularization, Solver::kCholesky, 0,
                    true, bad_row);
}

// W = Y (2^14 P) / 2^14 and Z = Y G^-1 of the short-row path, downloaded (tests and tools: the wgmma apply of
// dense.cu against an fp64 product).  Leaves the Gramian of Y in the context like als_gramian.
ALS_API int als_whitened_factors(als_ctx *ctx, const als_factors *Y, double regularization, float *W_host, float *Z_host) {
  ALS_REQUIRE(ctx && Y && W_host && Z_host, "als_whitened_factors: NULL argument");
  ALS_REQUIRE(Y->ld >= 32 && Y->ld <= 64, "als_whitened_factors: the short-row path covers 32..64 padded factors, got %d", Y->ld);
  ALS_CUDA(cudaSetDevice(ctx->device));
  int rc = launch_gramian(ctx, Y);
  if (rc != ALS_OK) return rc;
  rc = launch_regularize(ctx, Y->f, Y->ld, (float)regularization);
  if (rc != ALS_OK) return rc;
  rc = short_rows_prepare(ctx, Y, ctx->stream);
  if (rc != ALS_OK) return rc;
  int32_t ok = 0;
  ALS_CUDA(cudaMemcpyAsync(&ok, ctx->counters + kCtrWhitenOk, sizeof(ok), cudaMemcpyDeviceToHost, ctx->stream));
  std::vector<float> tmp((size_t)Y->rows * Y->ld);
  for (int which = 0; which < 2; ++which) {
    ALS_CUDA(cudaMemcpyAsync(tmp.data(), which ? ctx->zfactors : ctx->whitened, sizeof(float) * tmp.size(),
                             cudaMemcpyDeviceToHost, ctx->stream));
    ALS_CUDA(cudaStreamSynchronize(ctx->stream));
    if (which) {
      for (int64_t r = 0; r < Y->rows; ++r)
        for (int j = 0; j < Y->f; ++j) Z_host[r * Y->f + j] = tmp[(size_t)r * Y->ld + j];
    } else {
      // W is stored split and scaled: per 16 dimensions 8 words of fp16 pairs "hi", then 8 words "lo", of 2^14 W
      for (int64_t r = 0; r < Y->rows; ++r) {
        const uint32_t *row = reinterpret_cast<const uint32_t *>(tmp.data() + (size_t)r * Y->ld);
        for (int j = 0; j < Y->f; ++j) {
          const uint32_t hi = row[(j / 16) * 16 + (j % 16) / 2], lo = row[(j / 16) * 16 + 8 + (j % 16) / 2];
          const int sh = (j & 1) ? 16 : 0;
          const __half_raw hr{(unsigned short)(hi >> sh)}, lr{(unsigned short)(lo >> sh)};
          W_host[r * Y->f + j] = (__half2float(__half(hr)) + __half2float(__half(lr))) * (1.f / 16384.f);
        }
      }
    }
  }
  if (!ok) {
    set_error("als_whitened_factors: Y^T Y + reg I is not positive definite");
    return ALS_E_NOT_POSDEF;
  }
  return ALS_OK;
}

ALS_API int als_gramian_shard(als_ctx *ctx, const als_factors *Y, int64_t row0, int64_t nrows) {
  ALS_REQUIRE(ctx && Y, "als_gramian_shard: NULL argument");
  ALS_REQUIRE(row0 >= 0 && nrows >= 0 && row0 + nrows <= Y->rows, "als_gramian_shard: rows [%lld, %lld) out of range",
              (long long)row0, (long long)(row0 + nrows));
  ALS_CUDA(cudaSetDevice(ctx->device));
  als_factors view = *Y;  // shallow: a window on Y's rows (no ownership, no peers)
  view.d = Y->d + row0 * (int64_t)Y->ld;
  view.rows = nrows;
  view.peers_dev = nullptr;
  view.n_peers = 0;
  view.peer_maps.clear();
  int rc = launch_gramian(ctx, &view);
  if (rc != ALS_OK) return rc;
  return comm_allreduce_gramian(ctx, Y->ld * Y->ld);
}

ALS_API int als_least_squares_pregram(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y,
                                      double regularization, int64_t *bad_row) {
  return solve_half("als_least_squares_pregram", ctx, C, X, Y, Gram::kPresent, nullptr, regularization,
                    Solver::kCholesky, 0, true, bad_row);
}

// The multi-GPU fit loop: the same half as als_least_squares_pregram without the host round trip for bad_row, so
// the next half (and its collectives) are queued while this one runs; failures are collected by als_solver_status.
ALS_API int als_least_squares_pregram_async(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y,
                                            double regularization) {
  return solve_half("als_least_squares_pregram_async", ctx, C, X, Y, Gram::kPresent, nullptr, regularization,
                    Solver::kCholesky, 0, false, nullptr);
}

ALS_API int als_solver_status(als_ctx *ctx, int64_t *bad_row, int *any_rank_failed) {
  ALS_REQUIRE(ctx, "als_solver_status: NULL context");
  ALS_CUDA(cudaSetDevice(ctx->device));
  int32_t st = 0;
  float flag = 0.f;
  ALS_CUDA(cudaMemcpyAsync(&st, ctx->status, sizeof(st), cudaMemcpyDeviceToHost, ctx->stream));
  if (ctx->gram_ld)
    ALS_CUDA(cudaMemcpyAsync(&flag, ctx->G + ctx->gram_ld * ctx->gram_ld, sizeof(flag), cudaMemcpyDeviceToHost, ctx->stream));
  int64_t first = -1;
  const int rc = take_bad_row(ctx, 2, &first);  // synchronises: st and flag have landed too
  if (rc != ALS_OK && rc != ALS_E_NOT_POSDEF) return rc;
  if (bad_row) *bad_row = first;
  if (any_rank_failed) *any_rank_failed = (st != 0 || flag > 0.f || first >= 0) ? 1 : 0;
  // start a new collection period
  ALS_CUDA(cudaMemsetAsync(ctx->status, 0, sizeof(int32_t), ctx->stream));
  if (ctx->gram_ld) ALS_CUDA(cudaMemsetAsync(ctx->G + ctx->gram_ld * ctx->gram_ld, 0, sizeof(float), ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return rc;
}

ALS_API int als_least_squares_cg_pregram(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y,
                                         float regularization, int cg_steps) {
  return solve_half("als_least_squares_cg_pregram", ctx, C, X, Y, Gram::kPresent, nullptr, regularization, Solver::kCg,
                    cg_steps, false, nullptr);
}

ALS_API int als_least_squares_with_gramian(als_ctx *ctx, const float *YtY_host, const als_csr *C, als_factors *X,
                                           const als_factors *Y, double regularization, int64_t *bad_row) {
  return solve_half("als_least_squares_with_gramian", ctx, C, X, Y, Gram::kHost, YtY_host, regularization,
                    Solver::kCholesky, 0, true, bad_row);
}

ALS_API int als_least_squares_cg(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y,
                                 float regularization, int cg_steps) {
  return solve_half("als_least_squares_cg", ctx, C, X, Y, Gram::kCompute, nullptr, regularization, Solver::kCg, cg_steps,
                    false, nullptr);
}

ALS_API int als_calculate_loss(als_ctx *ctx, const als_csr *C, const als_factors *X, const als_factors *Y,
                               float regularization, double *loss) {
  ALS_REQUIRE(loss, "als_calculate_loss: loss is NULL");
  int rc = check_half("als_calculate_loss", ctx, C, const_cast<als_factors *>(X), Y);
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaSetDevice(ctx->device));
  // per segment (launch_loss leaves X^T X of the segment's rows in the Gramian buffer): the terms are shard sums
  double sum[3] = {0.0, 0.0, 0.0};
  rc = for_each_segment(ctx, C, [&](size_t, const als_csr *S) -> int {
    double t[3];
    int lrc;
    if ((lrc = launch_gramian(ctx, Y)) != ALS_OK || (lrc = launch_loss(ctx, S, X, Y, regularization, t)) != ALS_OK) return lrc;
    sum[0] += t[0];
    sum[1] += t[1];
    sum[2] = t[2];  // reg ||Y||^2: once
    return ALS_OK;
  });
  if (rc != ALS_OK) return rc;
  for (int i = 0; i < 3; ++i) loss[i] = sum[i];
  return ALS_OK;
}

// what als_topk and als_ranking_metrics refuse in their common arguments
static int check_topk(const char *who, const als_factors *items, const als_factors *queries, int64_t n_query, int k,
                      const als_csr *liked) {
  ALS_REQUIRE(items->f == queries->f, "%s: items have %d factors, queries %d", who, items->f, queries->f);
  ALS_REQUIRE(k >= 0 && n_query >= 0, "%s: negative k or n_query", who);
  ALS_REQUIRE(!liked || liked->rows == n_query, "%s: liked has %lld rows for %lld queries", who,
              liked ? (long long)liked->rows : 0LL, (long long)n_query);
  ALS_REQUIRE(!liked || liked->host || liked->segs.empty(), "%s: the liked CSR (%lld nonzeros) is held as segments; split the queries "
              "into calls whose liked rows hold fewer than 2^31 - 1 nonzeros", who, liked ? (long long)liked->nnz : 0LL);
  if (liked && liked->host) {
    set_error("%s: the liked CSR is host-resident; upload the filter with als_csr_upload or als_csr_upload64", who);
    return ALS_E_UNSUPPORTED;
  }
  ALS_REQUIRE(!liked || liked->cols == items->rows, "%s: liked has %lld columns for %lld items", who,
              liked ? (long long)liked->cols : 0LL, (long long)items->rows);
  return ALS_OK;
}

ALS_API int als_topk(als_ctx *ctx, const als_factors *items, const als_factors *queries, const int32_t *query_rows,
                     int64_t n_query, int k, const float *item_norms_host, const als_csr *liked,
                     const int32_t *filter_items, int64_t n_filter, int32_t *ids_host, float *scores_host) {
  ALS_REQUIRE(ctx && items && queries && ids_host && scores_host, "als_topk: NULL argument");
  int rc = check_topk("als_topk", items, queries, n_query, k, liked);
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaSetDevice(ctx->device));
  return launch_topk(ctx, items, queries, query_rows, n_query, k, item_norms_host, liked, filter_items, n_filter,
                     ids_host, scores_host);
}

ALS_API int als_ranking_metrics(als_ctx *ctx, const als_factors *items, const als_factors *queries, const int32_t *query_rows,
                                int64_t n_query, int k, const als_csr *liked, const als_csr *test, const double *gain_host,
                                const double *gain_sum_host, double *sums) {
  ALS_REQUIRE(ctx && items && queries && test && sums, "als_ranking_metrics: NULL argument");
  int rc = check_topk("als_ranking_metrics", items, queries, n_query, k, liked);
  if (rc != ALS_OK) return rc;
  ALS_REQUIRE(k >= 1, "als_ranking_metrics: k = %d ranks nothing", k);
  ALS_REQUIRE(gain_host && gain_sum_host, "als_ranking_metrics: NULL gain table");
  ALS_REQUIRE(test->rows == n_query, "als_ranking_metrics: test has %lld rows for %lld queries", (long long)test->rows,
              (long long)n_query);
  ALS_REQUIRE(test->cols == items->rows, "als_ranking_metrics: test has %lld columns for %lld items", (long long)test->cols,
              (long long)items->rows);
  if (test->host || !test->segs.empty()) {
    set_error("als_ranking_metrics: the test CSR is %s; upload it as one device-resident CSR of fewer than 2^31 - 1 "
              "nonzeros (split the queries)", test->host ? "host-resident" : "held as segments");
    return ALS_E_UNSUPPORTED;
  }
  ALS_CUDA(cudaSetDevice(ctx->device));
  return launch_ranking_metrics(ctx, items, queries, query_rows, n_query, k, liked, test, gain_host, gain_sum_host, sums);
}

// ---- serving from device ids (serve.cu) ------------------------------------------------------------------------
// ORs `bit` into the flag of ids outside [0, limit) and reads it back: 0 when every id is in range
static int device_ids_out_of_range(als_ctx *ctx, const void *ids, int bytes, int64_t n, int64_t limit, int *bad) {
  *bad = 0;
  if (n == 0) return ALS_OK;
  int *flag = reinterpret_cast<int *>(ctx->counters + kCtrIdsBad);
  ALS_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), ctx->stream));
  const int rc = stage_ids(ctx, ids, bytes, n, limit, nullptr, flag, 1);
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaMemcpyAsync(bad, flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return ALS_OK;
}

ALS_API int als_device_upload(als_ctx *ctx, void *dst, const void *src, int64_t bytes) {
  const char *who = "als_device_upload";
  ALS_REQUIRE(ctx && ((dst && src) || bytes == 0) && bytes >= 0, "%s: bad argument", who);
  if (bytes == 0) return ALS_OK;
  ALS_CUDA(cudaSetDevice(ctx->device));
  const int rc = require_device_memory(ctx, who, "dst", dst);
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyHostToDevice, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return ALS_OK;
}

ALS_API int als_device_download(als_ctx *ctx, void *dst, const void *src, int64_t bytes) {
  const char *who = "als_device_download";
  ALS_REQUIRE(ctx && ((dst && src) || bytes == 0) && bytes >= 0, "%s: bad argument", who);
  if (bytes == 0) return ALS_OK;
  ALS_CUDA(cudaSetDevice(ctx->device));
  const int rc = require_device_memory(ctx, who, "src", src);
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return ALS_OK;
}

ALS_API int als_ids_sort(als_ctx *ctx, const void *ids, int id_bytes, int64_t n, uint64_t producer_stream, void *sorted) {
  const char *who = "als_ids_sort";
  ALS_REQUIRE(ctx && ((ids && sorted) || n == 0), "%s: NULL argument", who);
  ALS_REQUIRE(id_bytes == 4 || id_bytes == 8, "%s: id_bytes must be 4 or 8, got %d", who, id_bytes);
  ALS_REQUIRE(n >= 0, "%s: negative length", who);
  if (n == 0) return ALS_OK;
  ALS_CUDA(cudaSetDevice(ctx->device));
  int rc = require_device_memory(ctx, who, "ids", ids);
  if (rc == ALS_OK) rc = require_device_memory(ctx, who, "sorted", sorted);
  if (rc == ALS_OK) rc = wait_for_producer(ctx, producer_stream);
  if (rc == ALS_OK) rc = sort_ids(ctx, ids, id_bytes, n, sorted);
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return ALS_OK;
}

ALS_API int als_factors_gather_rows(als_ctx *ctx, const als_factors *src, const void *rows, int row_bytes, int64_t n,
                                    uint64_t producer_stream, als_factors **out, int *bad) {
  const char *who = "als_factors_gather_rows";
  ALS_REQUIRE(ctx && src && out && bad && (rows || n == 0), "%s: NULL argument", who);
  ALS_REQUIRE(row_bytes == 4 || row_bytes == 8, "%s: row_bytes must be 4 or 8, got %d", who, row_bytes);
  ALS_REQUIRE(n >= 0, "%s: negative length", who);
  *out = nullptr;
  *bad = 0;
  ALS_CUDA(cudaSetDevice(ctx->device));
  int rc = n ? require_device_memory(ctx, who, "rows", rows) : ALS_OK;
  if (rc == ALS_OK) rc = wait_for_producer(ctx, producer_stream);
  if (rc == ALS_OK) rc = device_ids_out_of_range(ctx, rows, row_bytes, n, src->rows, bad);
  if (rc != ALS_OK) return rc;
  ALS_REQUIRE(!*bad, "%s: rows holds ids outside [0, %lld)", who, (long long)src->rows);
  als_factors *f = nullptr;
  if ((rc = als_factors_create(ctx, n, src->f, &f)) != ALS_OK) return rc;
  rc = launch_gather_rows(ctx, src, rows, row_bytes, n, f);
  if (rc == ALS_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess)
    rc = cuda_fail(cudaGetLastError(), "als_factors_gather_rows", __FILE__, __LINE__);
  if (rc != ALS_OK) {
    als_factors_destroy(f);
    return rc;
  }
  *out = f;
  return ALS_OK;
}

ALS_API int als_factors_row_norms(als_ctx *ctx, const als_factors *f, float zero_value, float *norms) {
  const char *who = "als_factors_row_norms";
  ALS_REQUIRE(ctx && f && (norms || f->rows == 0), "%s: NULL argument", who);
  if (f->rows == 0) return ALS_OK;
  ALS_CUDA(cudaSetDevice(ctx->device));
  int rc = require_device_memory(ctx, who, "norms", norms);
  if (rc == ALS_OK) rc = launch_row_norms(ctx, f, zero_value, norms);
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return ALS_OK;
}

ALS_API int als_csr_restrict_columns(als_ctx *ctx, const als_csr *liked, const void *subset, int subset_bytes, int64_t m,
                                     uint64_t producer_stream, als_csr **out) {
  const char *who = "als_csr_restrict_columns";
  ALS_REQUIRE(ctx && liked && out && (subset || m == 0), "%s: NULL argument", who);
  ALS_REQUIRE(subset_bytes == 4 || subset_bytes == 8, "%s: subset_bytes must be 4 or 8, got %d", who, subset_bytes);
  ALS_REQUIRE(m >= 0 && m < (int64_t)INT32_MAX, "%s: a subset of %lld ids", who, (long long)m);
  ALS_REQUIRE(!liked->host && liked->segs.empty(),
              "%s: the liked CSR must be one device-resident CSR of fewer than 2^31 - 1 nonzeros", who);
  *out = nullptr;
  ALS_CUDA(cudaSetDevice(ctx->device));
  int rc = m ? require_device_memory(ctx, who, "subset", subset) : ALS_OK;
  if (rc == ALS_OK) rc = wait_for_producer(ctx, producer_stream);
  if (rc != ALS_OK) return rc;
  Dev<int64_t> indptr;
  Dev<int32_t> indices;
  Dev<float> data;
  int64_t nnz = 0;
  if ((rc = csr_restrict_columns(ctx, liked, subset, subset_bytes, m, indptr, indices, data, &nnz)) != ALS_OK) return rc;
  // the remapped entries go through the one upload path, like every other CSR
  return csr_build(who, false, ctx, liked->rows, m, nnz, CsrArrays{indptr, 8, indices, 4, data, 4, true}, 0, out);
}

ALS_API int als_topk_into(als_ctx *ctx, const als_factors *items, const als_factors *queries, const void *query_rows,
                          int query_row_bytes, int64_t query_row0, int64_t n_query, int k, const float *item_norms,
                          const float *query_norms, const als_csr *liked, const void *filter_items, int filter_bytes,
                          int64_t n_filter, const void *id_map, int map_bytes, uint64_t producer_stream, void *ids,
                          float *scores, int *bad) {
  const char *who = "als_topk_into";
  ALS_REQUIRE(ctx && items && queries && bad, "%s: NULL argument", who);
  *bad = 0;
  const bool outputs = n_query > 0 && k > 0;
  ALS_REQUIRE((ids && scores) || !outputs, "%s: NULL outputs", who);
  ALS_REQUIRE(filter_items || n_filter == 0, "%s: NULL filter_items", who);
  ALS_REQUIRE(query_row_bytes == 4 || query_row_bytes == 8, "%s: query_row_bytes must be 4 or 8, got %d", who, query_row_bytes);
  ALS_REQUIRE(filter_bytes == 4 || filter_bytes == 8, "%s: filter_bytes must be 4 or 8, got %d", who, filter_bytes);
  ALS_REQUIRE(map_bytes == 4 || map_bytes == 8, "%s: map_bytes must be 4 or 8, got %d", who, map_bytes);
  ALS_REQUIRE(n_filter >= 0 && query_row0 >= 0, "%s: negative n_filter or query_row0", who);
  ALS_REQUIRE(!query_rows || query_row0 == 0, "%s: query_row0 = %lld with query_rows", who, (long long)query_row0);
  int rc = check_topk(who, items, queries, n_query, k, liked);
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaSetDevice(ctx->device));
  const struct {
    const void *p;
    const char *name;
    bool read;
  } mem[] = {{query_rows, "query_rows", query_rows && n_query > 0},  {item_norms, "item_norms", item_norms && items->rows > 0},
             {query_norms, "query_norms", query_norms && outputs}, {filter_items, "filter_items", n_filter > 0},
             {id_map, "id_map", id_map && outputs},                 {ids, "ids", outputs},
             {scores, "scores", outputs}};
  for (const auto &a : mem)
    if (a.read && (rc = require_device_memory(ctx, who, a.name, a.p)) != ALS_OK) return rc;
  if ((rc = wait_for_producer(ctx, producer_stream)) != ALS_OK) return rc;
  const TopkIds rows{query_rows, query_rows ? n_query : 0, query_row_bytes, true, query_row0};
  const TopkIds filter{filter_items, n_filter, filter_bytes, true, 0};
  TopkDevice t;
  rc = topk_device(ctx, items, queries, rows, n_query, k, item_norms, true, liked, filter, &t);
  *bad = t.bad;
  if (rc == ALS_OK && outputs) rc = launch_topk_epilogue(ctx, t, n_query, k, id_map, map_bytes, query_norms, ids, scores);
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));  // complete when this returns: any stream may read ids / scores
  return ALS_OK;
}

// ---- refitting rows in place from device ids (refit.cu) ----------------------------------------------------------
ALS_API int als_ids_range(als_ctx *ctx, const void *ids, int id_bytes, int64_t n, uint64_t producer_stream,
                          int64_t *min_id, int64_t *max_id) {
  const char *who = "als_ids_range";
  ALS_REQUIRE(ctx && min_id && max_id && (ids || n == 0), "%s: NULL argument", who);
  ALS_REQUIRE(id_bytes == 4 || id_bytes == 8, "%s: id_bytes must be 4 or 8, got %d", who, id_bytes);
  ALS_REQUIRE(n >= 0, "%s: negative length", who);
  *min_id = 0;
  *max_id = -1;
  if (n == 0) return ALS_OK;
  ALS_CUDA(cudaSetDevice(ctx->device));
  int rc = require_device_memory(ctx, who, "ids", ids);
  if (rc == ALS_OK) rc = wait_for_producer(ctx, producer_stream);
  if (rc == ALS_OK) rc = ids_range(ctx, ids, id_bytes, n, min_id, max_id);
  return rc;
}

ALS_API int als_factors_grow(als_ctx *ctx, als_factors *f, int64_t rows) {
  const char *who = "als_factors_grow";
  ALS_REQUIRE(ctx && f, "%s: NULL argument", who);
  ALS_REQUIRE(rows >= f->rows, "%s: %lld rows would shrink a matrix of %lld", who, (long long)rows, (long long)f->rows);
  ALS_REQUIRE(f->pooled && f->n_peers == 0, "%s: the matrix is shared with other ranks", who);
  if (rows == f->rows) return ALS_OK;
  const int64_t row_bytes = sizeof(float) * (int64_t)f->ld;
  // checked before the product is formed: a row count whose bytes overflow int64 or exceed the device's memory (a
  // hashed 64-bit id, say) is refused, never allocated short
  ALS_REQUIRE(rows <= ctx->mem_bytes / row_bytes, "%s: %lld rows of %lld bytes are more than the device's %lld bytes", who,
              (long long)rows, (long long)row_bytes, (long long)ctx->mem_bytes);
  ALS_CUDA(cudaSetDevice(ctx->device));
  Dev<float> d;
  const int rc = d.alloc(ctx, row_bytes * rows);
  if (rc != ALS_OK) return rc;
  if (f->rows) ALS_CUDA(cudaMemcpyAsync(d, f->d, row_bytes * f->rows, cudaMemcpyDeviceToDevice, ctx->stream));
  // the new rows, padding included, are zero: np.concatenate([host, np.zeros(...)]) uploaded
  ALS_CUDA(cudaMemsetAsync(d + f->rows * f->ld, 0, row_bytes * (rows - f->rows), ctx->stream));
  dev_free(ctx, f->d);  // stream-ordered: after the copy has read it
  f->d = d.release();
  f->rows = rows;
  return ALS_OK;
}

ALS_API int als_factors_scatter_rows(als_ctx *ctx, als_factors *dst, const void *ids, int id_bytes, int64_t n,
                                     uint64_t producer_stream, const als_factors *src) {
  const char *who = "als_factors_scatter_rows";
  ALS_REQUIRE(ctx && dst && src && (ids || n == 0), "%s: NULL argument", who);
  ALS_REQUIRE(id_bytes == 4 || id_bytes == 8, "%s: id_bytes must be 4 or 8, got %d", who, id_bytes);
  ALS_REQUIRE(n == src->rows, "%s: %lld ids for %lld rows", who, (long long)n, (long long)src->rows);
  ALS_REQUIRE(src->f == dst->f, "%s: rows of %d factors into a matrix of %d", who, src->f, dst->f);
  ALS_REQUIRE(dst->n_peers == 0, "%s: the matrix is shared with other ranks", who);
  if (n == 0) return ALS_OK;
  ALS_CUDA(cudaSetDevice(ctx->device));
  int rc = require_device_memory(ctx, who, "ids", ids);
  if (rc == ALS_OK) rc = wait_for_producer(ctx, producer_stream);
  if (rc == ALS_OK) rc = scatter_rows(ctx, dst, ids, id_bytes, n, src);
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));  // the ids have been read: the caller may free or refill them
  return ALS_OK;
}

// ---- BM25 / TF-IDF weighting and normalisation of raw arrays (weight.cu) ---------------------------------------------
static int weight_arrays(als_ctx *ctx, const char *who, int64_t rows, int64_t nnz, const void *indptr, int indptr_bytes,
                         const void *row, int row_bytes, const void *indices, int index_bytes, const void *data,
                         int value_kind, uint64_t producer_stream) {
  ALS_REQUIRE(ctx, "%s: ctx is NULL", who);
  ALS_REQUIRE(rows >= 0 && nnz >= 0, "%s: negative shape", who);
  ALS_REQUIRE(!indptr != !row, "%s: exactly one of indptr (CSR) and row (COO) is given", who);
  ALS_REQUIRE(!indptr || indptr_bytes == 4 || indptr_bytes == 8, "%s: indptr_bytes must be 4 or 8, got %d", who,
              indptr_bytes);
  ALS_REQUIRE(!row || row_bytes == 4 || row_bytes == 8, "%s: row_bytes must be 4 or 8, got %d", who, row_bytes);
  ALS_REQUIRE(!indices || index_bytes == 4 || index_bytes == 8, "%s: index_bytes must be 4 or 8, got %d", who,
              index_bytes);
  ALS_REQUIRE(value_kind >= ALS_VALUE_F32 && value_kind <= ALS_VALUE_I64, "%s: value_kind %d is not an ALS_VALUE_*", who,
              value_kind);
  ALS_REQUIRE(nnz == 0 || (data && (indices || !index_bytes)), "%s: NULL array with nnz > 0", who);
  ALS_CUDA(cudaSetDevice(ctx->device));
  int rc = indptr ? require_device_memory(ctx, who, "indptr", indptr) : ALS_OK;
  if (rc == ALS_OK && nnz > 0 && row) rc = require_device_memory(ctx, who, "row", row);
  if (rc == ALS_OK && nnz > 0 && indices) rc = require_device_memory(ctx, who, "indices", indices);
  if (rc == ALS_OK && nnz > 0 && data) rc = require_device_memory(ctx, who, "data", data);
  if (rc == ALS_OK) rc = wait_for_producer(ctx, producer_stream);
  return rc;
}

ALS_API int als_weight_column_counts(als_ctx *ctx, const void *indices, int index_bytes, int64_t nnz, int64_t cols,
                                     uint64_t producer_stream, int64_t *counts) {
  const char *who = "als_weight_column_counts";
  ALS_REQUIRE(ctx && (counts || cols == 0) && (indices || nnz == 0), "%s: NULL argument", who);
  ALS_REQUIRE(index_bytes == 4 || index_bytes == 8, "%s: index_bytes must be 4 or 8, got %d", who, index_bytes);
  ALS_REQUIRE(nnz >= 0 && cols >= 0, "%s: negative shape", who);
  ALS_CUDA(cudaSetDevice(ctx->device));
  int rc = nnz > 0 ? require_device_memory(ctx, who, "indices", indices) : ALS_OK;
  if (rc == ALS_OK) rc = wait_for_producer(ctx, producer_stream);
  if (rc == ALS_OK) rc = weight_column_counts(ctx, indices, index_bytes, nnz, cols, counts);
  return rc;
}

ALS_API int als_weight_row_sums(als_ctx *ctx, int64_t rows, int64_t nnz, const void *indptr, int indptr_bytes,
                                const void *row, int row_bytes, const void *data, int value_kind, int squares,
                                uint64_t producer_stream, void *sums) {
  const char *who = "als_weight_row_sums";
  ALS_REQUIRE(sums || rows == 0, "%s: sums is NULL", who);
  int rc = weight_arrays(ctx, who, rows, nnz, indptr, indptr_bytes, row, row_bytes, nullptr, 0, data, value_kind,
                         producer_stream);
  if (rc == ALS_OK) rc = weight_row_sums(ctx, rows, nnz, indptr, indptr_bytes, row, row_bytes, data, value_kind, squares != 0,
                                         sums);
  return rc;
}

ALS_API int als_weight_entries(als_ctx *ctx, int kind, int64_t rows, int64_t cols, int64_t nnz, const void *indptr,
                               int indptr_bytes, const void *row, int row_bytes, const void *indices, int index_bytes,
                               const void *data, int value_kind, const void *row_values, const double *idf, double k1p1,
                               double k1, int flags, uint64_t producer_stream, double *out) {
  const char *who = "als_weight_entries";
  ALS_REQUIRE(kind == ALS_WEIGHT_BM25 || kind == ALS_WEIGHT_TFIDF || kind == ALS_WEIGHT_NORMALIZE,
              "%s: kind %d is not an ALS_WEIGHT_*", who, kind);
  ALS_REQUIRE(cols >= 0, "%s: negative shape", who);
  ALS_REQUIRE(nnz == 0 || out, "%s: out is NULL", who);
  ALS_REQUIRE(kind == ALS_WEIGHT_TFIDF || row_values || rows == 0, "%s: row_values is NULL", who);
  ALS_REQUIRE(kind == ALS_WEIGHT_NORMALIZE || idf || cols == 0, "%s: idf is NULL", who);
  int rc = weight_arrays(ctx, who, rows, nnz, indptr, indptr_bytes, row, row_bytes, indices, index_bytes, data, value_kind,
                         producer_stream);
  if (rc == ALS_OK && nnz > 0) rc = require_device_memory(ctx, who, "out", out);
  if (rc == ALS_OK && indptr) rc = weight_check_indptr(ctx, indptr, indptr_bytes, rows, nnz, who);
  if (rc == ALS_OK) rc = weight_entries(ctx, kind, rows, cols, nnz, indptr, indptr_bytes, row, row_bytes, indices,
                                        index_bytes, data, value_kind, row_values, idf, k1p1, k1, flags, out);
  return rc;
}

ALS_API int als_device_copy(als_ctx *ctx, void *dst, const void *src, int64_t bytes, uint64_t producer_stream) {
  const char *who = "als_device_copy";
  ALS_REQUIRE(ctx && ((dst && src) || bytes == 0) && bytes >= 0, "%s: bad argument", who);
  if (bytes == 0) return ALS_OK;
  ALS_CUDA(cudaSetDevice(ctx->device));
  int rc = require_device_memory(ctx, who, "dst", dst);
  if (rc == ALS_OK) rc = require_device_memory(ctx, who, "src", src);
  if (rc == ALS_OK) rc = wait_for_producer(ctx, producer_stream);
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDeviceToDevice, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return ALS_OK;
}
