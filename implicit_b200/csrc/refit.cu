// Refitting rows in place on the device (partial_fit_users / partial_fit_items with CUDA ids; als_ids_range,
// als_factors_scatter_rows in api.cu):
//   range    min and max of int32 / int64 ids in one pass and one 16-byte read-back: the caller refuses a negative id
//            and grows the factor matrix to max + 1 rows (als_factors_grow);
//   scatter  n solved rows stored at their ids with the semantics of numpy's host[ids] = rows: the (id, position) pairs
//            are radix-sorted (stable, so the positions of one id stay ascending) and only the last pair of each run of
//            equal ids -- the last occurrence -- writes its row.  An id outside the matrix is skipped, never written.
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>

#include "common.h"

namespace als {
namespace {

template <typename T>
__global__ void ids_range_kernel(const T *__restrict__ ids, int64_t n, long long *range) {
  long long lo = LLONG_MAX, hi = LLONG_MIN;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const long long v = (long long)ids[i];
    lo = min(lo, v);
    hi = max(hi, v);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMin(&range[0], lo);
    atomicMax(&range[1], hi);
  }
}

// element e of the n x ld rows: row i of the sorted pairs writes dst[ids[i]] from src[pos[i]] when it is the last pair
// of its id; the padding columns are written as zeros
template <typename T>
__global__ void scatter_last_kernel(const T *__restrict__ ids, const int32_t *__restrict__ pos, int64_t n,
                                    const float *__restrict__ src, float *__restrict__ dst, int64_t rows, int f, int ld) {
  const int64_t total = n * ld;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / ld;
    const int c = (int)(e - i * ld);
    const long long id = (long long)ids[i];
    if (i + 1 < n && (long long)ids[i + 1] == id) continue;         // a later occurrence of the id wins
    if ((unsigned long long)id >= (unsigned long long)rows) continue;  // outside the matrix: never written
    dst[id * ld + c] = c < f ? src[(int64_t)pos[i] * ld + c] : 0.f;
  }
}

}  // namespace

int ids_range(als_ctx *ctx, const void *ids, int bytes, int64_t n, int64_t *min_id, int64_t *max_id) {
  *min_id = 0;
  *max_id = -1;
  if (n <= 0) return ALS_OK;
  long long *range = nullptr;
  int rc = dev_alloc(ctx, (void **)&range, 2 * sizeof(long long));
  if (rc != ALS_OK) return rc;
  const long long init[2] = {LLONG_MAX, LLONG_MIN};
  long long got[2] = {0, -1};
  cudaError_t e = cudaMemcpyAsync(range, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) {
    if (bytes == 8)
      ids_range_kernel<<<grid_for(ctx, n), 256, 0, ctx->stream>>>((const long long *)ids, n, range);
    else
      ids_range_kernel<<<grid_for(ctx, n), 256, 0, ctx->stream>>>((const int32_t *)ids, n, range);
    ctx->launches++;
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(got, range, sizeof(got), cudaMemcpyDeviceToHost, ctx->stream);
  dev_free(ctx, range);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  if (e != cudaSuccess) return cuda_fail(e, "ids range", __FILE__, __LINE__);
  *min_id = got[0];
  *max_id = got[1];
  return ALS_OK;
}

int scatter_rows(als_ctx *ctx, als_factors *dst, const void *ids, int bytes, int64_t n, const als_factors *src) {
  if (n <= 0) return ALS_OK;
  if (n >= (int64_t)INT32_MAX) {
    set_error("als_factors_scatter_rows: %lld ids, more than one sort takes", (long long)n);
    return ALS_E_UNSUPPORTED;
  }
  void *keys = nullptr, *tmp = nullptr;
  int32_t *pos_in = nullptr, *pos = nullptr;
  size_t tmp_bytes = 0;
  auto sort = [&](void *t) -> cudaError_t {
    if (bytes == 8)
      return cub::DeviceRadixSort::SortPairs(t, tmp_bytes, (const long long *)ids, (long long *)keys, pos_in, pos, (int)n,
                                             0, 64, ctx->stream);
    return cub::DeviceRadixSort::SortPairs(t, tmp_bytes, (const int32_t *)ids, (int32_t *)keys, pos_in, pos, (int)n, 0, 32,
                                           ctx->stream);
  };
  auto done = [&](int code) {
    dev_free(ctx, keys);
    dev_free(ctx, pos_in);
    dev_free(ctx, pos);
    dev_free(ctx, tmp);
    return code;
  };
  int rc = dev_alloc(ctx, &keys, (int64_t)bytes * n);
  if (rc == ALS_OK) rc = dev_alloc(ctx, (void **)&pos_in, sizeof(int32_t) * n);
  if (rc == ALS_OK) rc = dev_alloc(ctx, (void **)&pos, sizeof(int32_t) * n);
  if (rc == ALS_OK) rc = stage_iota(ctx, pos_in, n, 0);
  if (rc != ALS_OK) return done(rc);
  cudaError_t e = sort(nullptr);
  if (e != cudaSuccess) return done(cuda_fail(e, "scatter: sort of the ids", __FILE__, __LINE__));
  if ((rc = dev_alloc(ctx, &tmp, (int64_t)tmp_bytes)) != ALS_OK) return done(rc);
  if ((e = sort(tmp)) != cudaSuccess) return done(cuda_fail(e, "scatter: sort of the ids", __FILE__, __LINE__));
  ctx->launches++;
  const int grid = grid_for(ctx, n * dst->ld);
  if (bytes == 8)
    scatter_last_kernel<<<grid, 256, 0, ctx->stream>>>((const long long *)keys, pos, n, src->d, dst->d, dst->rows, dst->f,
                                                       dst->ld);
  else
    scatter_last_kernel<<<grid, 256, 0, ctx->stream>>>((const int32_t *)keys, pos, n, src->d, dst->d, dst->rows, dst->f,
                                                       dst->ld);
  ctx->launches++;
  if ((e = cudaGetLastError()) != cudaSuccess) return done(cuda_fail(e, "scatter kernel", __FILE__, __LINE__));
  return done(ALS_OK);
}

}  // namespace als
