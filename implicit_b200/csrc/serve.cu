// Serving from device ids (als_topk_into and its helpers, api.cu): the pieces a recommend / similar_* call needs around
// the fused top-k when its ids arrive in CUDA memory and its results leave in it.
//   ids       int32 / int64 ids of the caller narrowed into the top-k's int32 staging, with a range check that sets a
//             flag bit instead of faulting;
//   epilogue  topk_device's [n_query, k_eff] scratch -> the caller's [n_query, k]: zero tail, optional id map
//             (out = map[id]) and per-query norms (score /= qnorm[row]), in one pass;
//   norms     row norms of a factor matrix, bitwise np.linalg.norm(F, axis=-1) in fp32;
//   gather    a factor matrix of chosen rows (the item subsets);
//   restrict  a liked CSR remapped onto the positions of a sorted column subset (_filter_items_from_sparse_matrix).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_radix_sort.cuh>

#include <algorithm>

#include "common.h"

namespace als {
namespace {

template <typename T>
__global__ void stage_ids_kernel(const T *__restrict__ in, int64_t n, int64_t limit, int32_t *__restrict__ out, int *flag,
                                 int bit) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const long long v = (long long)in[i];
    if ((unsigned long long)v >= (unsigned long long)limit) atomicOr(flag, bit);
    if (out) out[i] = (int32_t)v;
  }
}

__global__ void iota_kernel(int32_t *out, int64_t n, int64_t first) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = (int32_t)(first + i);
}

template <typename OutT, typename MapT>
__global__ void topk_epilogue_kernel(const int32_t *__restrict__ ids, const float *__restrict__ scores, int k_eff,
                                     int64_t n_query, int k, const MapT *__restrict__ map,
                                     const int32_t *__restrict__ query_rows, const float *__restrict__ qnorm,
                                     OutT *__restrict__ out_ids, float *__restrict__ out_scores) {
  const int64_t n = n_query * k;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t q = e / k;
    const int j = (int)(e - q * k);
    int32_t id = 0;
    float s = 0.f;
    if (j < k_eff) {  // past k_eff: the zero tail of topk.pyx:20-21
      id = ids[q * k_eff + j];
      s = scores[q * k_eff + j];
    }
    if (qnorm) s = __fdiv_rn(s, qnorm[query_rows ? query_rows[q] : q]);  // scores / norm[:, None]
    out_ids[e] = map ? (OutT)map[id] : (OutT)id;                       // subset[ids]
    out_scores[e] = s;
  }
}

// numpy's float32 pairwise summation (add.reduce over a contiguous axis) of x[i]^2, i < n: below 8 terms a plain
// running sum from 0; up to 128 eight strided accumulators, combined ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the rest
// one by one; above that the halves split at n/2 rounded down to a multiple of 8.  Every product and sum is rounded on
// its own (no FMA contraction).
__device__ __forceinline__ float sq(const float *x, int i) {
  const float v = x[i];
  return __fmul_rn(v, v);
}

__device__ __forceinline__ float pairwise_leaf(const float *x, int n) {
  if (n < 8) {
    float res = 0.f;
    for (int i = 0; i < n; ++i) res = __fadd_rn(res, sq(x, i));
    return res;
  }
  float r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = sq(x, j);
  int i = 8;
  for (; i < n - (n % 8); i += 8)
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], sq(x, i + j));
  float res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                        __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
  for (; i < n; ++i) res = __fadd_rn(res, sq(x, i));
  return res;
}

template <int D>
__device__ __forceinline__ float pairwise_sq(const float *x, int n) {
  if (n <= 128) return pairwise_leaf(x, n);
  const int n2 = n / 2 - (n / 2) % 8;
  return __fadd_rn(pairwise_sq<D - 1>(x, n2), pairwise_sq<D - 1>(x + n2, n - n2));
}
template <>
__device__ __forceinline__ float pairwise_sq<0>(const float *x, int n) {
  return pairwise_leaf(x, n);
}

// one thread per row; four levels of halving cover up to 2048 terms, past the 1024 factors a model may have
__global__ void __launch_bounds__(128) row_norms_kernel(const float *__restrict__ F, int64_t rows, int f, int ld,
                                                        float zero_value, float *__restrict__ out) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x) {
    const float n = __fsqrt_rn(pairwise_sq<4>(F + r * ld, f));
    out[r] = n == 0.f ? zero_value : n;
  }
}

template <typename T>
__global__ void gather_rows_kernel(const float *__restrict__ src, int64_t src_rows, int f, int ld,
                                   const T *__restrict__ rows, int64_t n, float *__restrict__ dst) {
  const int64_t total = n * ld;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / ld;
    const int c = (int)(e - i * ld);
    const long long r = (long long)rows[i];
    // the padding columns stay zero: the wgmma top-k reads all ld of them
    dst[e] = (c < f && (unsigned long long)r < (unsigned long long)src_rows) ? src[r * ld + c] : 0.f;
  }
}

// ---- restrict: one warp per row of the liked CSR ----------------------------------------------------------------
template <typename T>
__device__ __forceinline__ int64_t lower_bound(const T *a, int64_t m, long long v) {
  int64_t lo = 0, hi = m;
  while (lo < hi) {
    const int64_t mid = (lo + hi) / 2;
    if ((long long)a[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// pos[p]: the subset position of entry p, or -1 when its column is not in the subset or its value is 0 (the
// searchsorted / eliminate_zeros of _filter_items_from_sparse_matrix); counts[r]: the entries row r keeps
template <typename T>
__global__ void restrict_count_kernel(const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                                      const float *__restrict__ data, int64_t rows, const T *__restrict__ subset, int64_t m,
                                      int32_t *__restrict__ pos, int64_t *__restrict__ counts) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; r < rows;
       r += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    int64_t kept = 0;
    for (int p = indptr[r] + lane; p < indptr[r + 1]; p += 32) {
      const int c = indices[p];
      const int64_t at = lower_bound(subset, m, c);
      const bool keep = at < m && (long long)subset[at] == c && data[p] != 0.f;
      pos[p] = keep ? (int32_t)at : -1;
      kept += keep;
    }
    kept = __reduce_add_sync(0xffffffffu, (unsigned)kept);
    if (lane == 0) counts[r] = kept;
  }
}

// the kept positions of row r, in entry order, to out[off[r] ...)
__global__ void restrict_scatter_kernel(const int32_t *__restrict__ indptr, int64_t rows, const int32_t *__restrict__ pos,
                                        const int64_t *__restrict__ off, int32_t *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; r < rows;
       r += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    int64_t o = off[r];
    const int end = indptr[r + 1];
    for (int p0 = indptr[r]; p0 < end; p0 += 32) {
      const int p = p0 + lane;
      const int v = p < end ? pos[p] : -1;
      const unsigned b = __ballot_sync(0xffffffffu, v >= 0);
      if (v >= 0) out[o + __popc(b & ((1u << lane) - 1))] = v;
      o += __popc(b);
    }
  }
}

// distinct values of each sorted row [off[r], off[r + 1]): counted (out == NULL) or written to out[off2[r] ...), with
// value 1 (the liked filter reads positions only)
__global__ void restrict_unique_kernel(const int64_t *__restrict__ off, int64_t rows, const int32_t *__restrict__ sorted,
                                       int64_t *__restrict__ counts, const int64_t *__restrict__ off2,
                                       int32_t *__restrict__ out, float *__restrict__ out_data) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; r < rows;
       r += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const int64_t b = off[r], end = off[r + 1];
    int64_t o = out ? off2[r] : 0;
    for (int64_t p0 = b; p0 < end; p0 += 32) {
      const int64_t p = p0 + lane;
      const bool first = p < end && (p == b || sorted[p] != sorted[p - 1]);
      const unsigned m = __ballot_sync(0xffffffffu, first);
      if (out && first) {
        out[o + __popc(m & ((1u << lane) - 1))] = sorted[p];
        out_data[o + __popc(m & ((1u << lane) - 1))] = 1.f;
      }
      o += __popc(m);
    }
    if (!out && lane == 0) counts[r] = o;
  }
}

// exclusive scan of counts[0, rows) into off[0, rows]; counts[rows] must be 0
int scan_counts(als_ctx *ctx, int64_t *counts, int64_t rows, int64_t *off) {
  size_t tmp_bytes = 0;
  ALS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, counts, off, rows + 1, ctx->stream));
  void *tmp = nullptr;
  int rc = dev_alloc(ctx, &tmp, (int64_t)tmp_bytes);
  if (rc != ALS_OK) return rc;
  const cudaError_t e = cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, counts, off, rows + 1, ctx->stream);
  dev_free(ctx, tmp);
  ALS_CUDA(e);
  ctx->launches++;
  return ALS_OK;
}

}  // namespace

int stage_ids(als_ctx *ctx, const void *ids, int bytes, int64_t n, int64_t limit, int32_t *out, int *flag, int bit) {
  if (n <= 0) return ALS_OK;
  if (bytes == 8)
    stage_ids_kernel<<<grid_for(ctx, n), 256, 0, ctx->stream>>>((const long long *)ids, n, limit, out, flag, bit);
  else
    stage_ids_kernel<<<grid_for(ctx, n), 256, 0, ctx->stream>>>((const int32_t *)ids, n, limit, out, flag, bit);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  return ALS_OK;
}

int stage_iota(als_ctx *ctx, int32_t *out, int64_t n, int64_t first) {
  if (n <= 0) return ALS_OK;
  iota_kernel<<<grid_for(ctx, n), 256, 0, ctx->stream>>>(out, n, first);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  return ALS_OK;
}

int launch_topk_epilogue(als_ctx *ctx, const TopkDevice &t, int64_t n_query, int k, const void *map, int map_bytes,
                         const float *qnorm, void *ids, float *scores) {
  const int64_t n = n_query * (int64_t)k;
  if (n == 0) return ALS_OK;
  // with nothing ranked (no items) the outputs are the zero tail alone, and 0 / norm is 0
  if (t.k_eff == 0) qnorm = nullptr;
  const int grid = grid_for(ctx, n);
  auto go = [&](auto *out, auto *mp) {
    topk_epilogue_kernel<<<grid, 256, 0, ctx->stream>>>(t.ids, t.scores, t.k_eff, n_query, k, mp, t.query_rows, qnorm, out,
                                                        scores);
  };
  if (!map) go((int32_t *)ids, (const int32_t *)nullptr);
  else if (map_bytes == 8) go((long long *)ids, (const long long *)map);
  else go((int32_t *)ids, (const int32_t *)map);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  return ALS_OK;
}

int launch_row_norms(als_ctx *ctx, const als_factors *F, float zero_value, float *out) {
  if (F->rows == 0) return ALS_OK;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(F->rows, 128), (int64_t)ctx->sm_count * 32));
  row_norms_kernel<<<grid, 128, 0, ctx->stream>>>(F->d, F->rows, F->f, F->ld, zero_value, out);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  return ALS_OK;
}

int launch_gather_rows(als_ctx *ctx, const als_factors *src, const void *rows, int bytes, int64_t n, als_factors *dst) {
  if (n == 0) return ALS_OK;
  const int grid = grid_for(ctx, n * src->ld);
  if (bytes == 8)
    gather_rows_kernel<<<grid, 256, 0, ctx->stream>>>(src->d, src->rows, src->f, src->ld, (const long long *)rows, n, dst->d);
  else
    gather_rows_kernel<<<grid, 256, 0, ctx->stream>>>(src->d, src->rows, src->f, src->ld, (const int32_t *)rows, n, dst->d);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  return ALS_OK;
}

int sort_ids(als_ctx *ctx, const void *in, int bytes, int64_t n, void *out) {
  if (n == 0) return ALS_OK;
  if (n >= (int64_t)INT32_MAX) {
    set_error("als_ids_sort: %lld ids, more than one sort takes", (long long)n);
    return ALS_E_UNSUPPORTED;
  }
  size_t tmp_bytes = 0;
  auto sort = [&](void *tmp) -> cudaError_t {
    if (bytes == 8)
      return cub::DeviceRadixSort::SortKeys(tmp, tmp_bytes, (const long long *)in, (long long *)out, (int)n, 0, 64,
                                            ctx->stream);
    return cub::DeviceRadixSort::SortKeys(tmp, tmp_bytes, (const int32_t *)in, (int32_t *)out, (int)n, 0, 32, ctx->stream);
  };
  ALS_CUDA(sort(nullptr));
  void *tmp = nullptr;
  int rc = dev_alloc(ctx, &tmp, (int64_t)tmp_bytes);
  if (rc != ALS_OK) return rc;
  const cudaError_t e = sort(tmp);
  dev_free(ctx, tmp);
  ALS_CUDA(e);
  ctx->launches++;
  return ALS_OK;
}

int csr_restrict_columns(als_ctx *ctx, const als_csr *liked, const void *subset, int bytes, int64_t m, int64_t **indptr,
                         int32_t **indices, float **data, int64_t *nnz) {
  const int64_t rows = liked->rows, n = liked->nnz;
  *indptr = nullptr;
  *indices = nullptr;
  *data = nullptr;
  *nnz = 0;
  int32_t *pos = nullptr, *kept = nullptr, *sorted = nullptr;
  int64_t *counts = nullptr, *off = nullptr;
  void *tmp = nullptr;
  int rc = dev_alloc(ctx, (void **)&counts, sizeof(int64_t) * (rows + 1));
  if (rc == ALS_OK) rc = dev_alloc(ctx, (void **)&off, sizeof(int64_t) * (rows + 1));
  if (rc == ALS_OK) rc = dev_alloc(ctx, (void **)indptr, sizeof(int64_t) * (rows + 1));
  if (rc == ALS_OK) rc = dev_alloc(ctx, (void **)&pos, sizeof(int32_t) * n);
  if (rc == ALS_OK) rc = dev_alloc(ctx, (void **)&kept, sizeof(int32_t) * n);
  if (rc == ALS_OK) rc = dev_alloc(ctx, (void **)&sorted, sizeof(int32_t) * n);
  auto done = [&](int code) {
    dev_free(ctx, counts);
    dev_free(ctx, off);
    dev_free(ctx, pos);
    dev_free(ctx, kept);
    dev_free(ctx, sorted);
    dev_free(ctx, tmp);
    if (code != ALS_OK) {
      dev_free(ctx, *indptr);
      dev_free(ctx, *indices);
      dev_free(ctx, *data);
      *indptr = nullptr;
      *indices = nullptr;
      *data = nullptr;
    }
    return code;
  };
  if (rc != ALS_OK) return done(rc);
  const int grid = grid_for(ctx, 32 * rows);
  // count: the subset positions of the kept entries, and how many each row keeps
  if (cudaMemsetAsync(counts + rows, 0, sizeof(int64_t), ctx->stream) != cudaSuccess) return done(cuda_fail(cudaGetLastError(), "memset", __FILE__, __LINE__));
  if (rows > 0) {
    if (bytes == 8)
      restrict_count_kernel<<<grid, 256, 0, ctx->stream>>>(liked->indptr, liked->indices, liked->data, rows,
                                                           (const long long *)subset, m, pos, counts);
    else
      restrict_count_kernel<<<grid, 256, 0, ctx->stream>>>(liked->indptr, liked->indices, liked->data, rows,
                                                           (const int32_t *)subset, m, pos, counts);
    ctx->launches++;
  }
  // scan, scatter in entry order, then each row sorted (CUB segmented radix sort, as rows_in_order)
  if ((rc = scan_counts(ctx, counts, rows, off)) != ALS_OK) return done(rc);
  int64_t total = 0;
  if (cudaMemcpyAsync(&total, off + rows, sizeof(total), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
      cudaStreamSynchronize(ctx->stream) != cudaSuccess)
    return done(cuda_fail(cudaGetLastError(), "restrict: count readback", __FILE__, __LINE__));
  if (total > 0) {
    restrict_scatter_kernel<<<grid, 256, 0, ctx->stream>>>(liked->indptr, rows, pos, off, kept);
    ctx->launches++;
    size_t tmp_bytes = 0;
    if (cub::DeviceSegmentedRadixSort::SortKeys(nullptr, tmp_bytes, kept, sorted, (int)total, (int)rows, off, off + 1, 0, 32,
                                                ctx->stream) != cudaSuccess)
      return done(cuda_fail(cudaGetLastError(), "restrict: segmented sort", __FILE__, __LINE__));
    if ((rc = dev_alloc(ctx, &tmp, (int64_t)tmp_bytes)) != ALS_OK) return done(rc);
    if (cub::DeviceSegmentedRadixSort::SortKeys(tmp, tmp_bytes, kept, sorted, (int)total, (int)rows, off, off + 1, 0, 32,
                                                ctx->stream) != cudaSuccess)
      return done(cuda_fail(cudaGetLastError(), "restrict: segmented sort", __FILE__, __LINE__));
    ctx->launches++;
  }
  // unique per row (scipy's tocsr merges the duplicate positions): count, scan, write
  if (rows > 0) {
    restrict_unique_kernel<<<grid, 256, 0, ctx->stream>>>(off, rows, sorted, counts, nullptr, nullptr, nullptr);
    ctx->launches++;
  }
  if ((rc = scan_counts(ctx, counts, rows, *indptr)) != ALS_OK) return done(rc);
  if (cudaMemcpyAsync(nnz, *indptr + rows, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess ||
      cudaStreamSynchronize(ctx->stream) != cudaSuccess)
    return done(cuda_fail(cudaGetLastError(), "restrict: count readback", __FILE__, __LINE__));
  if ((rc = dev_alloc(ctx, (void **)indices, sizeof(int32_t) * *nnz)) != ALS_OK) return done(rc);
  if ((rc = dev_alloc(ctx, (void **)data, sizeof(float) * *nnz)) != ALS_OK) return done(rc);
  if (*nnz > 0) {
    restrict_unique_kernel<<<grid, 256, 0, ctx->stream>>>(off, rows, sorted, nullptr, *indptr, *indices, *data);
    ctx->launches++;
  }
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return done(cuda_fail(e, "restrict kernels", __FILE__, __LINE__));
  return done(ALS_OK);
}

}  // namespace als
