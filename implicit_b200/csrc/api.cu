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

int dev_alloc(als_ctx *ctx, void **ptr, int64_t bytes, cudaStream_t stream) {
  ALS_CUDA(cudaMallocAsync(ptr, (size_t)std::max<int64_t>(bytes, 16), stream ? stream : ctx->stream));
  return ALS_OK;
}

void dev_free(als_ctx *ctx, void *ptr) {
  if (ptr) cudaFreeAsync(ptr, ctx->stream);
}

// Builds the schedule of a device-transposed CSR from the indptr copy that csr_transpose left in flight.
int ensure_schedule(als_ctx *ctx, als_csr *csr) {
  if (!csr->sched_pending) return ALS_OK;
  ALS_CUDA(cudaEventSynchronize(ctx->sched_ev));
  csr->sched_pending = false;
  ctx->sched_owner = nullptr;
  return build_schedule(ctx, csr, ctx->sched_pinned);
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

int ensure_pinned(als_ctx *ctx, int64_t bytes) {
  if (bytes <= ctx->pinned_bytes) return ALS_OK;
  if (ctx->pinned) {
    ALS_CUDA(cudaStreamSynchronize(ctx->copy));
    ALS_CUDA(cudaFreeHost(ctx->pinned));
    ctx->pinned = nullptr;
    ctx->pinned_bytes = 0;
  }
  int64_t cap = std::max<int64_t>(bytes, 1 << 20);
  ALS_CUDA(cudaMallocHost(&ctx->pinned, cap));
  ctx->pinned_bytes = cap;
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

// n values -> a page-locked host array in the staging threads, folding the weight range of csr_wmax_kernel on the way
static int fill_host_values(float *dst, const float *src, int64_t n, unsigned *wmax_bits, bool *neg) {
  std::atomic<unsigned> m{0};
  std::atomic<bool> ng{false};
  const int rc = staged_fill_host(dst, (size_t)n * sizeof(float), [&](char *out, size_t off, size_t len) {
    const float *in = src + off / 4;
    memcpy(out, in, len);
    unsigned cm;
    bool cn;
    host_wmax(in, (int64_t)(len / 4), &cm, &cn);
    unsigned cur = m.load();
    while (cm > cur && !m.compare_exchange_weak(cur, cm)) {
    }
    if (cn) ng = true;
    return true;
  });
  *wmax_bits = m.load();
  *neg = ng.load();
  return rc;
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
  // The lists are allocated and uploaded on the copy stream: when the schedule of a transposed matrix is built
  // lazily, a half-iteration is already running on the compute stream and must not delay them (nor they it).
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
  als_ctx *ctx = new als_ctx();
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
      if (als_ctx_set_knob(ctx, t.name, v) != ALS_OK) {
        delete ctx;
        return ALS_E_INVALID;
      }
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
  ALS_CUDA(cudaEventCreateWithFlags(&ctx->sched_ev, cudaEventDisableTiming));
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
  *out = ctx;
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
  else {
    set_error("als_ctx_get_knob: unknown knob '%s'", name);
    return ALS_E_INVALID;
  }
  return ALS_OK;
}

ALS_API int als_ctx_destroy(als_ctx *ctx) {
  if (!ctx) return ALS_OK;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  cudaStreamSynchronize(ctx->copy);
  cudaStreamSynchronize(ctx->aux);
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
  if (ctx->pinned) cudaFreeHost(ctx->pinned);
  if (ctx->stage_buf) {
    cudaFreeHost(ctx->stage_buf);
    for (int t = 0; t < 4; ++t) {
      cudaStreamDestroy(ctx->stage_stream[t]);
      for (int b = 0; b < 2; ++b) cudaEventDestroy(ctx->stage_ev[t][b]);
    }
    cudaEventDestroy(ctx->stage_ready);
  }
  if (ctx->sched_pinned) cudaFreeHost(ctx->sched_pinned);
  cudaEventDestroy(ctx->sched_ev);
  for (int k = 0; k < 2; ++k) {
    cudaEventDestroy(ctx->ring_loaded[k]);
    cudaEventDestroy(ctx->ring_free[k]);
  }
  for (int i = 0; i < 5; ++i) {
    if (ctx->class_stream[i]) cudaStreamDestroy(ctx->class_stream[i]);
    if (ctx->class_join[i]) cudaEventDestroy(ctx->class_join[i]);
  }
  if (ctx->class_fork) cudaEventDestroy(ctx->class_fork);
  {
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, ctx->device) == cudaSuccess) cudaMemPoolTrimTo(pool, 0);
  }
  cudaEventDestroy(ctx->ev0);
  cudaEventDestroy(ctx->ev1);
  cudaStreamDestroy(ctx->stream);
  cudaStreamDestroy(ctx->copy);
  cudaStreamDestroy(ctx->aux);
  cudaEventDestroy(ctx->ev_fork);
  cudaEventDestroy(ctx->ev_join);
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

// ---- CSR ---------------------------------------------------------------------------------------
ALS_API int als_csr_upload(als_ctx *ctx, int64_t rows, int64_t cols, int64_t nnz, const int32_t *indptr,
                           const int32_t *indices, const float *data, int64_t row_offset, als_csr **out) {
  ALS_REQUIRE(ctx && out && indptr, "als_csr_upload: NULL argument");
  ALS_REQUIRE(rows >= 0 && cols >= 0 && nnz >= 0, "als_csr_upload: negative shape");
  ALS_REQUIRE(nnz < (int64_t)INT32_MAX && rows < (int64_t)INT32_MAX && cols < (int64_t)INT32_MAX,
              "als_csr_upload: int32 CSR only (rows, cols, nnz < 2^31), like implicit/gpu/matrix.h:93-100");
  ALS_REQUIRE(indptr[0] >= 0 && (int64_t)indptr[rows] - indptr[0] == nnz,
              "als_csr_upload: indptr[rows] - indptr[0] = %lld != nnz = %lld",
              (long long)indptr[rows] - indptr[0], (long long)nnz);
  ALS_REQUIRE(nnz == 0 || (indices && data), "als_csr_upload: indices/data NULL with nnz > 0");
  *out = nullptr;
  ALS_CUDA(cudaSetDevice(ctx->device));
  als_csr *c = new als_csr();
  c->ctx = ctx;
  c->rows = rows;
  c->cols = cols;
  c->nnz = nnz;
  c->row_offset = row_offset;
  // a row shard arrives with indptr[0] != 0: rebase
  std::vector<int32_t> rebased;
  const int32_t base = indptr[0];
  const int32_t *ip = indptr;
  if (base != 0) {
    rebased.resize(rows + 1);
    for (int64_t r = 0; r <= rows; ++r) rebased[r] = indptr[r] - base;
    ip = rebased.data();
  }
  for (int64_t r = 0; r < rows; ++r) {
    if (ip[r + 1] < ip[r]) {
      delete c;
      set_error("als_csr_upload: indptr is not monotone at row %lld", (long long)r);
      return ALS_E_INVALID;
    }
  }
  int arc;
  if (needs_segments(ctx, nnz)) {  // a cap set by the segment_nnz knob: the same layout as als_csr_upload64's
    std::vector<int64_t> ip64(ip, ip + rows + 1);
    if ((arc = dev_alloc(ctx, (void **)&c->indices, sizeof(int32_t) * nnz)) != ALS_OK ||
        (arc = dev_alloc(ctx, (void **)&c->data, sizeof(float) * nnz)) != ALS_OK ||
        (arc = h2d_copy(ctx, c->indices, indices + base, sizeof(int32_t) * nnz)) != ALS_OK ||
        (arc = h2d_copy(ctx, c->data, data + base, sizeof(float) * nnz)) != ALS_OK ||
        (arc = make_segments(ctx, c, ip64.data())) != ALS_OK) {
      als_csr_destroy(c);
      return arc;
    }
    *out = c;
    return ALS_OK;
  }
  if ((arc = dev_alloc(ctx, (void **)&c->indptr, sizeof(int32_t) * (rows + 1))) != ALS_OK ||
      (arc = dev_alloc(ctx, (void **)&c->indices, sizeof(int32_t) * std::max<int64_t>(nnz, 1))) != ALS_OK ||
      (arc = dev_alloc(ctx, (void **)&c->data, sizeof(float) * std::max<int64_t>(nnz, 1))) != ALS_OK) {
    als_csr_destroy(c);
    return arc;
  }
  ALS_CUDA(cudaMemcpyAsync(c->indptr, ip, sizeof(int32_t) * (rows + 1), cudaMemcpyHostToDevice, ctx->stream));
  if (nnz) {
    int hrc;
    if ((hrc = h2d_copy(ctx, c->indices, indices + base, sizeof(int32_t) * nnz)) != ALS_OK ||
        (hrc = h2d_copy(ctx, c->data, data + base, sizeof(float) * nnz)) != ALS_OK) {
      als_csr_destroy(c);
      return hrc;
    }
  }
  int rc = build_schedule(ctx, c, ip);
  if (rc != ALS_OK) {
    als_csr_destroy(c);
    return rc;
  }
  *out = c;
  return ALS_OK;
}

// als_csr_upload64 and als_csr_upload_host64: the same checks and refusals; host keeps indices / data in page-locked host
// memory (always segmented) instead of uploading them
static int csr_upload64(const char *who, bool host, als_ctx *ctx, int64_t rows, int64_t cols, int64_t nnz, const int64_t *indptr,
                        const void *indices, int index_bytes, const float *data, int64_t row_offset, als_csr **out) {
  ALS_REQUIRE(ctx && out && indptr, "%s: NULL argument", who);
  ALS_REQUIRE(index_bytes == 4 || index_bytes == 8, "%s: index_bytes must be 4 or 8, got %d", who, index_bytes);
  ALS_REQUIRE(rows >= 0 && cols >= 0 && nnz >= 0, "%s: negative shape", who);
  ALS_REQUIRE(rows < (int64_t)INT32_MAX && cols < (int64_t)INT32_MAX, "%s: rows and cols must be < 2^31 - 1", who);
  ALS_REQUIRE(indptr[0] >= 0 && indptr[rows] - indptr[0] == nnz, "%s: indptr[rows] - indptr[0] = %lld != nnz = %lld", who,
              (long long)(indptr[rows] - indptr[0]), (long long)nnz);
  ALS_REQUIRE(nnz == 0 || (indices && data), "%s: indices/data NULL with nnz > 0", who);
  for (int64_t r = 0; r < rows; ++r)
    ALS_REQUIRE(indptr[r + 1] >= indptr[r], "%s: indptr is not monotone at row %lld", who, (long long)r);
  *out = nullptr;
  ALS_CUDA(cudaSetDevice(ctx->device));
  als_csr *c = new als_csr();
  c->ctx = ctx;
  c->rows = rows;
  c->cols = cols;
  c->nnz = nnz;
  c->row_offset = row_offset;
  c->host = host;
  const int64_t base = indptr[0];  // a row shard arrives with indptr[0] != 0
  int rc;
  int64_t bad = -1;
  unsigned wmax_bits = 0;
  bool neg = false;
  if (host) {
    const size_t bytes = sizeof(int32_t) * (size_t)std::max<int64_t>(nnz, 1);
    cudaError_t e = cudaMallocHost((void **)&c->indices, bytes);
    if (e == cudaSuccess) e = cudaMallocHost((void **)&c->data, bytes);
    if (e != cudaSuccess) {
      als_csr_destroy(c);
      return cuda_fail(e, "cudaMallocHost (host-resident CSR)", __FILE__, __LINE__);
    }
    rc = h2d_indices(ctx, c->indices, (const char *)indices + base * index_bytes, index_bytes, nnz, cols, &bad, true);
    if (rc == ALS_OK) rc = fill_host_values(c->data, data + base, nnz, &wmax_bits, &neg);
  } else if ((rc = dev_alloc(ctx, (void **)&c->indices, sizeof(int32_t) * std::max<int64_t>(nnz, 1))) == ALS_OK &&
             (rc = dev_alloc(ctx, (void **)&c->data, sizeof(float) * std::max<int64_t>(nnz, 1))) == ALS_OK &&
             (rc = h2d_indices(ctx, c->indices, (const char *)indices + base * index_bytes, index_bytes, nnz, cols, &bad)) == ALS_OK) {
    rc = h2d_copy(ctx, c->data, data + base, sizeof(float) * nnz);
  }
  if (rc != ALS_OK) {
    if (bad >= 0) {
      const int64_t v = index_bytes == 8 ? ((const int64_t *)indices)[base + bad] : ((const int32_t *)indices)[base + bad];
      set_error("%s: indices[%lld] = %lld is outside [0, %lld)", who, (long long)(base + bad), (long long)v, (long long)cols);
    }
    ALS_CUDA(cudaStreamSynchronize(ctx->stream));
    als_csr_destroy(c);
    return rc;
  }
  std::vector<int64_t> ip((size_t)rows + 1);
  for (int64_t r = 0; r <= rows; ++r) ip[r] = indptr[r] - base;
  if (host) {
    if ((rc = set_host_wmax(ctx, c, wmax_bits, neg)) == ALS_OK) rc = make_segments(ctx, c, ip.data());
  } else if (needs_segments(ctx, nnz)) {
    rc = make_segments(ctx, c, ip.data());
  } else {
    std::vector<int32_t> ip32(ip.begin(), ip.end());
    if ((rc = dev_alloc(ctx, (void **)&c->indptr, sizeof(int32_t) * (rows + 1))) == ALS_OK) {
      ALS_CUDA(cudaMemcpyAsync(c->indptr, ip32.data(), sizeof(int32_t) * (rows + 1), cudaMemcpyHostToDevice, ctx->stream));
      rc = build_schedule(ctx, c, ip32.data());
      ALS_CUDA(cudaStreamSynchronize(ctx->stream));
    }
  }
  if (rc != ALS_OK) {
    als_csr_destroy(c);
    return rc;
  }
  *out = c;
  return ALS_OK;
}

ALS_API int als_csr_upload64(als_ctx *ctx, int64_t rows, int64_t cols, int64_t nnz, const int64_t *indptr,
                             const void *indices, int index_bytes, const float *data, int64_t row_offset, als_csr **out) {
  return csr_upload64("als_csr_upload64", false, ctx, rows, cols, nnz, indptr, indices, index_bytes, data, row_offset, out);
}

ALS_API int als_csr_upload_host64(als_ctx *ctx, int64_t rows, int64_t cols, int64_t nnz, const int64_t *indptr,
                                  const void *indices, int index_bytes, const float *data, int64_t row_offset, als_csr **out) {
  return csr_upload64("als_csr_upload_host64", true, ctx, rows, cols, nnz, indptr, indices, index_bytes, data, row_offset, out);
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

ALS_API int als_csr_transpose(als_ctx *ctx, const als_csr *in, als_csr **out) {
  ALS_REQUIRE(ctx && in && out, "als_csr_transpose: NULL argument");
  return als::csr_transpose(ctx, in, out);
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
  if (!in->segs.empty()) {  // a shard of a segmented CSR can itself exceed 2^31 nonzeros: a segmented view
    std::vector<int64_t> ip64;
    int rc = csr_indptr64(ctx, in, ip64);
    if (rc != ALS_OK) return rc;
    als_csr *c = new als_csr();
    c->ctx = ctx;
    c->rows = r1 - r0;
    c->cols = in->cols;
    c->nnz = ip64[r1] - ip64[r0];
    c->row_offset = r0;
    c->owns = false;
    c->indices = in->indices;
    c->data = in->data;
    if ((rc = make_segments(ctx, c, ip64.data() + r0)) != ALS_OK) {
      als_csr_destroy(c);
      return rc;
    }
    *out = c;
    return ALS_OK;
  }
  const int64_t rows = r1 - r0;
  std::vector<int32_t> ip((size_t)rows + 1);
  ALS_CUDA(cudaMemcpyAsync(ip.data(), in->indptr + r0, sizeof(int32_t) * (rows + 1), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  als_csr *c = new als_csr();
  c->ctx = ctx;
  c->rows = rows;
  c->cols = in->cols;
  c->nnz = (int64_t)ip[rows] - ip[0];
  c->row_offset = r0;
  c->owns = false;
  c->indptr = in->indptr + r0;  // absolute positions into the parent's indices/data
  c->indices = in->indices;
  c->data = in->data;
  int rc = build_schedule(ctx, c, ip.data());
  if (rc != ALS_OK) {
    als_csr_destroy(c);
    return rc;
  }
  *out = c;
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
    std::atomic<unsigned> m{0};
    std::atomic<bool> ng{false};
    staged_fill_host(data, sizeof(float) * (size_t)csr->nnz, [&](char *out, size_t, size_t len) {
      float *v = reinterpret_cast<float *>(out);
      const int64_t n = (int64_t)(len / 4);
      for (int64_t i = 0; i < n; ++i) v[i] *= alpha;
      unsigned cm;
      bool cn;
      host_wmax(v, n, &cm, &cn);
      unsigned cur = m.load();
      while (cm > cur && !m.compare_exchange_weak(cur, cm)) {
      }
      if (cn) ng = true;
      return true;
    });
    return set_host_wmax(ctx, csr, m.load(), ng.load());
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
  ALS_CUDA(cudaSetDevice(ctx->device));
  if (!csr->segs.empty()) {
    std::vector<int64_t> ip64((size_t)csr->rows + 1);
    int rc = als_csr_download64(ctx, csr, indptr ? ip64.data() : nullptr, indices, data);
    if (rc != ALS_OK) return rc;
    if (indptr)
      for (int64_t r = 0; r <= csr->rows; ++r) indptr[r] = (int32_t)ip64[r];
    return ALS_OK;
  }
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  // a row-slice view keeps absolute positions into its parent's arrays: rebase on the way out
  int32_t base = 0;
  if (!csr->owns) ALS_CUDA(cudaMemcpy(&base, csr->indptr, sizeof(int32_t), cudaMemcpyDeviceToHost));
  if (indptr) {
    ALS_CUDA(cudaMemcpy(indptr, csr->indptr, sizeof(int32_t) * (csr->rows + 1), cudaMemcpyDeviceToHost));
    if (base)
      for (int64_t r = 0; r <= csr->rows; ++r) indptr[r] -= base;
  }
  if (indices && csr->nnz)
    ALS_CUDA(cudaMemcpy(indices, csr->indices + base, sizeof(int32_t) * csr->nnz, cudaMemcpyDeviceToHost));
  if (data && csr->nnz)
    ALS_CUDA(cudaMemcpy(data, csr->data + base, sizeof(float) * csr->nnz, cudaMemcpyDeviceToHost));
  return ALS_OK;
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
    if (ctx->sched_owner == csr) {  // its indptr copy may still be in flight into the shared pinned buffer
      cudaEventSynchronize(ctx->sched_ev);
      ctx->sched_owner = nullptr;
    }
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
    float *moved = nullptr;
    ALS_CUDA(cudaMalloc(&moved, bytes));
    ALS_CUDA(cudaMemcpyAsync(moved, f->d, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    dev_free(ctx, f->d);
    ALS_CUDA(cudaStreamSynchronize(ctx->stream));
    f->d = moved;
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
  return ensure_schedule(ctx, const_cast<als_csr *>(C));  // a device-transposed matrix sorts its rows at first use
}

ALS_API int als_gramian(als_ctx *ctx, const als_factors *Y, float *G_host) {
  ALS_REQUIRE(ctx && Y, "als_gramian: NULL argument");
  ALS_CUDA(cudaSetDevice(ctx->device));
  int rc = launch_gramian(ctx, Y);
  if (rc != ALS_OK) return rc;
  if (G_host) {
    std::vector<float> tmp((size_t)Y->ld * Y->ld);
    ALS_CUDA(cudaMemcpyAsync(tmp.data(), ctx->G, sizeof(float) * tmp.size(), cudaMemcpyDeviceToHost, ctx->stream));
    ALS_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < Y->f; ++i) memcpy(G_host + (size_t)i * Y->f, tmp.data() + (size_t)i * Y->ld, sizeof(float) * Y->f);
  }
  return ALS_OK;
}

static int finish_cholesky(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y, double reg,
                           int64_t *bad_row) {
  int rc = launch_regularize(ctx, Y->f, Y->ld, (float)reg);
  if (rc != ALS_OK) return rc;
  rc = launch_cholesky(ctx, C, X, Y);
  if (rc != ALS_OK) return rc;
  long long bad = -1;
  ALS_CUDA(cudaMemcpyAsync(&bad, ctx->bad_row, sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  if (bad_row) *bad_row = (bad == LLONG_MAX) ? -1 : (int64_t)bad;
  if (bad != LLONG_MAX) {
    // reported here and now: nothing is left for a later als_solver_status to find
    const long long init[2] = {LLONG_MAX, LLONG_MAX};
    ALS_CUDA(cudaMemcpyAsync(ctx->bad_row, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
    ALS_CUDA(cudaStreamSynchronize(ctx->stream));
    set_error("cholesky failed on row %lld: normal equations not positive definite. Try increasing the "
              "regularization parameter.", bad);
    return ALS_E_NOT_POSDEF;
  }
  return ALS_OK;
}

ALS_API int als_least_squares(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y,
                              double regularization, int64_t *bad_row) {
  int rc = check_half("als_least_squares", ctx, C, X, Y);
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaSetDevice(ctx->device));
  rc = launch_gramian(ctx, Y);
  if (rc != ALS_OK) return rc;
  return finish_cholesky(ctx, C, X, Y, regularization, bad_row);
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
  int rc = check_half("als_least_squares_pregram", ctx, C, X, Y);
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaSetDevice(ctx->device));
  return finish_cholesky(ctx, C, X, Y, regularization, bad_row);
}

// The multi-GPU fit loop: the same half as als_least_squares_pregram without the host round trip for bad_row, so
// the next half (and its collectives) are queued while this one runs; failures are collected by als_solver_status.
ALS_API int als_least_squares_pregram_async(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y,
                                            double regularization) {
  int rc = check_half("als_least_squares_pregram_async", ctx, C, X, Y);
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaSetDevice(ctx->device));
  rc = launch_regularize(ctx, Y->f, Y->ld, (float)regularization);
  if (rc != ALS_OK) return rc;
  return launch_cholesky(ctx, C, X, Y);
}

ALS_API int als_solver_status(als_ctx *ctx, int64_t *bad_row, int *any_rank_failed) {
  ALS_REQUIRE(ctx, "als_solver_status: NULL context");
  ALS_CUDA(cudaSetDevice(ctx->device));
  long long bad[2] = {LLONG_MAX, LLONG_MAX};
  int32_t st = 0;
  float flag = 0.f;
  ALS_CUDA(cudaMemcpyAsync(bad, ctx->bad_row, sizeof(bad), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaMemcpyAsync(&st, ctx->status, sizeof(st), cudaMemcpyDeviceToHost, ctx->stream));
  if (ctx->gram_ld)
    ALS_CUDA(cudaMemcpyAsync(&flag, ctx->G + ctx->gram_ld * ctx->gram_ld, sizeof(flag), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  const long long first = std::min(bad[0], bad[1]);
  if (bad_row) *bad_row = first == LLONG_MAX ? -1 : (int64_t)first;
  if (any_rank_failed) *any_rank_failed = (st != 0 || flag > 0.f || first != LLONG_MAX) ? 1 : 0;
  const long long init[2] = {LLONG_MAX, LLONG_MAX};  // start a new collection period
  ALS_CUDA(cudaMemcpyAsync(ctx->bad_row, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
  ALS_CUDA(cudaMemsetAsync(ctx->status, 0, sizeof(int32_t), ctx->stream));
  if (ctx->gram_ld) ALS_CUDA(cudaMemsetAsync(ctx->G + ctx->gram_ld * ctx->gram_ld, 0, sizeof(float), ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  if (first != LLONG_MAX) {
    set_error("cholesky failed on row %lld: normal equations not positive definite. Try increasing the "
              "regularization parameter.", first);
    return ALS_E_NOT_POSDEF;
  }
  return ALS_OK;
}

ALS_API int als_least_squares_cg_pregram(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y,
                                         float regularization, int cg_steps) {
  int rc = check_half("als_least_squares_cg_pregram", ctx, C, X, Y);
  if (rc != ALS_OK) return rc;
  ALS_REQUIRE(cg_steps >= 0, "als_least_squares_cg_pregram: cg_steps < 0");
  ALS_CUDA(cudaSetDevice(ctx->device));
  rc = launch_regularize(ctx, Y->f, Y->ld, regularization);
  if (rc != ALS_OK) return rc;
  return launch_cg(ctx, C, X, Y, cg_steps);
}

ALS_API int als_least_squares_with_gramian(als_ctx *ctx, const float *YtY_host, const als_csr *C, als_factors *X,
                                           const als_factors *Y, double regularization, int64_t *bad_row) {
  int rc = check_half("als_least_squares_with_gramian", ctx, C, X, Y);
  if (rc != ALS_OK) return rc;
  ALS_REQUIRE(YtY_host, "als_least_squares_with_gramian: YtY is NULL");
  ALS_CUDA(cudaSetDevice(ctx->device));
  std::vector<float> tmp((size_t)Y->ld * Y->ld, 0.f);
  for (int i = 0; i < Y->f; ++i) memcpy(tmp.data() + (size_t)i * Y->ld, YtY_host + (size_t)i * Y->f, sizeof(float) * Y->f);
  ALS_CUDA(cudaMemcpyAsync(ctx->G, tmp.data(), sizeof(float) * tmp.size(), cudaMemcpyHostToDevice, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return finish_cholesky(ctx, C, X, Y, regularization, bad_row);
}

ALS_API int als_least_squares_cg(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y,
                                 float regularization, int cg_steps) {
  int rc = check_half("als_least_squares_cg", ctx, C, X, Y);
  if (rc != ALS_OK) return rc;
  ALS_REQUIRE(cg_steps >= 0, "als_least_squares_cg: cg_steps < 0");
  ALS_CUDA(cudaSetDevice(ctx->device));
  rc = launch_gramian(ctx, Y);
  if (rc != ALS_OK) return rc;
  rc = launch_regularize(ctx, Y->f, Y->ld, regularization);
  if (rc != ALS_OK) return rc;
  return launch_cg(ctx, C, X, Y, cg_steps);
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

ALS_API int als_topk(als_ctx *ctx, const als_factors *items, const als_factors *queries, const int32_t *query_rows,
                     int64_t n_query, int k, const float *item_norms_host, const als_csr *liked,
                     const int32_t *filter_items, int64_t n_filter, int32_t *ids_host, float *scores_host) {
  ALS_REQUIRE(ctx && items && queries && ids_host && scores_host, "als_topk: NULL argument");
  ALS_REQUIRE(items->f == queries->f, "als_topk: items have %d factors, queries %d", items->f, queries->f);
  ALS_REQUIRE(k >= 0 && n_query >= 0, "als_topk: negative k or n_query");
  ALS_REQUIRE(!liked || liked->rows == n_query, "als_topk: liked has %lld rows for %lld queries",
              liked ? (long long)liked->rows : 0LL, (long long)n_query);
  ALS_REQUIRE(!liked || liked->host || liked->segs.empty(), "als_topk: the liked CSR (%lld nonzeros) is held as segments; split the queries "
              "into calls whose liked rows hold fewer than 2^31 - 1 nonzeros", liked ? (long long)liked->nnz : 0LL);
  if (liked && liked->host) {
    set_error("als_topk: the liked CSR is host-resident; upload the filter with als_csr_upload or als_csr_upload64");
    return ALS_E_UNSUPPORTED;
  }
  ALS_REQUIRE(!liked || liked->cols == items->rows, "als_topk: liked has %lld columns for %lld items",
              liked ? (long long)liked->cols : 0LL, (long long)items->rows);
  ALS_CUDA(cudaSetDevice(ctx->device));
  return launch_topk(ctx, items, queries, query_rows, n_query, k, item_norms_host, liked, filter_items, n_filter,
                     ids_host, scores_host);
}
