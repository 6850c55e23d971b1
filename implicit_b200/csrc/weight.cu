// BM25 / TF-IDF weighting and row normalisation of an interaction matrix (implicit_b200/nearest_neighbours.py;
// als_weight_* in api.cu), on raw arrays: int32 / int64 indptr, row and column indices; fp32 / fp64 / int32 / int64
// values; int64 positions throughout.  The results are bitwise those of the reference's numpy code because every
// step follows numpy's order of operations:
//   column counts  exact int64 (atomics; order does not matter);
//   row sums       sequential in entry order per row, as scipy's COO matvec and numpy's bincount(weights) add them:
//                  one warp per row stages chunks of the row in shared memory while lane 0 adds them, so the loads of
//                  the next chunk are in flight while the dependent chain of adds runs;
//   per entry      the formula with every product, sum and quotient rounded in numpy's type (__f*_rn / __d*_rn: no
//                  FMA contraction).
// The host computes the vectors of length rows or cols (idf, the mean, length_norm, sqrt of the sums) with numpy
// from the downloaded counts and sums, so the logs and the pairwise mean are numpy's own bits.
#include <cub/device/device_radix_sort.cuh>

#include <type_traits>

#include "common.h"

namespace als {
namespace {

constexpr int kWarps = 8;      // warps per block of the row-sum kernel
constexpr int kPerLane = 8;    // entries each lane stages per chunk
constexpr int kChunk = 32 * kPerLane;
constexpr int kTile = 1024;    // entries per block tile of the per-entry kernel

template <typename V>
__device__ __forceinline__ V square_wrap(V v) {
  return v * v;
}
template <>
__device__ __forceinline__ int32_t square_wrap<int32_t>(int32_t v) {
  return (int32_t)((uint32_t)v * (uint32_t)v);  // numpy's int32 square wraps modulo 2^32
}
template <>
__device__ __forceinline__ long long square_wrap<long long>(long long v) {
  return (long long)((unsigned long long)v * (unsigned long long)v);
}

// the addend of entry p: the value in the sum type S (scipy's sum dtype), or its square in V cast to double
template <typename V, typename S, bool kSquares>
__device__ __forceinline__ S addend(const V *__restrict__ data, int64_t p) {
  const V v = data[p];
  if (kSquares) {
    if constexpr (sizeof(V) == 4 && V(0.5) != V(0)) return (S)__fmul_rn(v, v);
    else if constexpr (V(0.5) != V(0)) return (S)__dmul_rn(v, v);
    else return (S)square_wrap(v);
  }
  return (S)v;
}

template <typename S>
__device__ __forceinline__ S add_rn(S a, S b) {
  if constexpr (sizeof(S) == 4) return __fadd_rn(a, b);
  else if constexpr (S(0.5) != S(0)) return __dadd_rn(a, b);
  else return (S)((unsigned long long)a + (unsigned long long)b);  // int64 sums wrap like numpy's
}

// sums[r] = 0 + data[p_0] + data[p_1] + ... over the entries p_k of row r in entry order: positions [ip[r], ip[r+1])
// of the CSR order, mapped through perm (a stable sort of COO rows) when perm is not NULL
template <typename V, typename S, bool kSquares, typename IP>
__global__ void __launch_bounds__(kWarps * 32) row_sums_kernel(const IP *__restrict__ ip, const int64_t *__restrict__ perm,
                                                                const V *__restrict__ data, int64_t rows,
                                                                S *__restrict__ sums) {
  __shared__ S buf[kWarps][kChunk];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  S *b = buf[warp];
  for (int64_t r = blockIdx.x * (int64_t)kWarps + warp; r < rows; r += (int64_t)gridDim.x * kWarps) {
    const int64_t begin = (int64_t)ip[r], end = (int64_t)ip[r + 1];
    S acc = S(0);
    S next[kPerLane];
    auto load = [&](int64_t k) {
#pragma unroll
      for (int i = 0; i < kPerLane; ++i) {
        const int64_t j = k + lane + 32 * i;
        next[i] = j < end ? addend<V, S, kSquares>(data, perm ? perm[j] : j) : S(0);
      }
    };
    if (begin < end) load(begin);
    for (int64_t k = begin; k < end; k += kChunk) {
#pragma unroll
      for (int i = 0; i < kPerLane; ++i) b[lane + 32 * i] = next[i];
      __syncwarp();
      if (k + kChunk < end) load(k + kChunk);  // in flight while lane 0 adds this chunk
      if (lane == 0) {
        const int n = end - k < kChunk ? (int)(end - k) : kChunk;
        for (int i = 0; i < n; ++i) acc = add_rn(acc, b[i]);
      }
      __syncwarp();
    }
    if (lane == 0) sums[r] = acc;
  }
}

// flag[0] |= 1 when the CSR indptr is not 0 = ip[0] <= ip[1] <= ... <= ip[rows] = nnz
template <typename IP>
__global__ void check_indptr_kernel(const IP *__restrict__ ip, int64_t rows, int64_t nnz, int *flag) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r <= rows; r += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = (int64_t)ip[r];
    const bool bad = (r == 0 && v != 0) || (r == rows && v != nnz) || (r < rows && (int64_t)ip[r + 1] < v);
    if (bad) atomicOr(flag, 1);
  }
}

// flag[0] |= 1 for an index outside [0, limit); counts (may be NULL) += 1 at every index inside
template <typename I>
__global__ void count_kernel(const I *__restrict__ idx, int64_t n, int64_t limit, unsigned long long *counts, int *flag) {
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    const int64_t c = (int64_t)idx[j];
    if ((uint64_t)c >= (uint64_t)limit) atomicOr(flag, 1);
    else if (counts) atomicAdd(&counts[c], 1ull);
  }
}

// ip[r] = the first position of the sorted rows holding a row >= r (lower bound), r = 0 .. rows
template <typename R>
__global__ void indptr_from_sorted_kernel(const R *__restrict__ sorted, int64_t n, int64_t rows, int64_t *ip) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r <= rows; r += (int64_t)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if ((int64_t)sorted[mid] < r) lo = mid + 1;
      else hi = mid;
    }
    ip[r] = lo;
  }
}

__global__ void iota64_kernel(int64_t *out, int64_t n) {
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) out[j] = j;
}

// the row of CSR position j: the last r in [lo, hi] with ip[r] <= j
template <typename IP>
__device__ __forceinline__ int64_t row_of(const IP *__restrict__ ip, int64_t lo, int64_t hi, int64_t j) {
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if ((int64_t)ip[mid] <= j) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

struct EntryArgs {
  int kind;              // ALS_WEIGHT_BM25 / TFIDF / NORMALIZE
  int64_t rows, cols, nnz;
  const void *row_values;  // bm25: length_norm (fp32 when the denominator is fp32, else fp64); normalize: fp64 norms
  const double *idf;       // bm25, tfidf: [cols]
  double k1p1, k1;
  bool num32, den32;       // bm25: numerator / denominator rounded in fp32 (else fp64)
  int *flag;
};

template <typename V>
__device__ __forceinline__ double entry_value(const EntryArgs &a, V d, int64_t r, int64_t c) {
  constexpr bool kFloat = V(0.5) != V(0);
  if (a.kind == ALS_WEIGHT_TFIDF) {
    if constexpr (sizeof(V) == 4 && kFloat) return __dmul_rn((double)__fsqrt_rn(d), a.idf[c]);
    else return __dmul_rn(__dsqrt_rn((double)d), a.idf[c]);
  }
  if (a.kind == ALS_WEIGHT_NORMALIZE) return __ddiv_rn((double)d, ((const double *)a.row_values)[r]);
  // bm25: d * (K1 + 1) / (K1 * length_norm[r] + d) * idf[c]
  float num32 = 0.f, den32 = 0.f;
  double num64 = 0., den64 = 0.;
  if (a.num32) num32 = __fmul_rn((float)d, (float)a.k1p1);
  else num64 = __dmul_rn((double)d, a.k1p1);
  if (a.den32) den32 = __fadd_rn(__fmul_rn((float)a.k1, ((const float *)a.row_values)[r]), (float)d);
  else den64 = __dadd_rn(__dmul_rn(a.k1, ((const double *)a.row_values)[r]), (double)d);
  const double q = a.num32 && a.den32 ? (double)__fdiv_rn(num32, den32)
                                       : __ddiv_rn(a.num32 ? (double)num32 : num64, a.den32 ? (double)den32 : den64);
  return __dmul_rn(q, a.idf[c]);
}

// out[j] for every entry j: its row from the COO rows (row != NULL) or by a search of the CSR indptr narrowed to the
// rows of the block's tile; an entry whose row or column is outside the matrix sets *flag and writes nothing
template <typename V, typename IP, typename R, typename I>
__global__ void __launch_bounds__(256) entries_kernel(EntryArgs a, const IP *__restrict__ ip, const R *__restrict__ row,
                                                      const I *__restrict__ indices, const V *__restrict__ data,
                                                      double *__restrict__ out) {
  __shared__ int64_t span[2];
  for (int64_t t0 = blockIdx.x * (int64_t)kTile; t0 < a.nnz; t0 += (int64_t)gridDim.x * kTile) {
    const int64_t t1 = (t0 + kTile < a.nnz ? t0 + kTile : a.nnz) - 1;
    if (!row && threadIdx.x < 2) span[threadIdx.x] = row_of(ip, 0, a.rows - 1, threadIdx.x ? t1 : t0);
    __syncthreads();
    for (int64_t j = t0 + threadIdx.x; j <= t1; j += blockDim.x) {
      const int64_t r = row ? (int64_t)row[j] : row_of(ip, span[0], span[1], j);
      const int64_t c = (int64_t)indices[j];
      if ((uint64_t)r >= (uint64_t)a.rows || (uint64_t)c >= (uint64_t)a.cols) {
        atomicOr(a.flag, 1);
        continue;
      }
      out[j] = entry_value(a, data[j], r, c);
    }
    __syncthreads();
  }
}

template <typename F>
int dispatch_value(int kind, F &&f) {
  switch (kind) {
    case ALS_VALUE_F32: return f((const float *)nullptr);
    case ALS_VALUE_F64: return f((const double *)nullptr);
    case ALS_VALUE_I32: return f((const int32_t *)nullptr);
    default: return f((const long long *)nullptr);
  }
}

template <typename F>
int dispatch_index(int bytes, F &&f) {
  return bytes == 8 ? f((const long long *)nullptr) : f((const int32_t *)nullptr);
}

// 0, or ALS_E_INVALID after reading back a flag the kernels raised (synchronises)
int read_flag(als_ctx *ctx, int *flag, const char *what) {
  int bad = 0;
  cudaError_t e = cudaMemcpyAsync(&bad, flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  if (e != cudaSuccess) return cuda_fail(e, what, __FILE__, __LINE__);
  if (bad) {
    set_error("%s", what);
    return ALS_E_INVALID;
  }
  return ALS_OK;
}

int clear_flag(als_ctx *ctx, int **flag) {
  *flag = reinterpret_cast<int *>(ctx->counters + kCtrWeightBad);
  ALS_CUDA(cudaMemsetAsync(*flag, 0, sizeof(int), ctx->stream));
  return ALS_OK;
}

}  // namespace

int weight_check_indptr(als_ctx *ctx, const void *indptr, int indptr_bytes, int64_t rows, int64_t nnz, const char *who) {
  int *flag = nullptr;
  int rc = clear_flag(ctx, &flag);
  if (rc != ALS_OK) return rc;
  dispatch_index(indptr_bytes, [&](auto ip) {
    check_indptr_kernel<<<grid_for(ctx, rows + 1), 256, 0, ctx->stream>>>((decltype(ip))indptr, rows, nnz, flag);
    return 0;
  });
  ctx->launches++;
  ALS_CUDA(cudaGetLastError());
  char what[160];
  snprintf(what, sizeof(what), "%s: indptr is not 0 = indptr[0] <= ... <= indptr[%lld] = nnz = %lld", who, (long long)rows,
           (long long)nnz);
  return read_flag(ctx, flag, what);
}

int weight_column_counts(als_ctx *ctx, const void *indices, int index_bytes, int64_t nnz, int64_t cols, int64_t *counts) {
  Dev<unsigned long long> d;
  int *flag = nullptr;
  int rc;
  if ((rc = d.alloc(ctx, sizeof(int64_t) * std::max<int64_t>(cols, 1))) != ALS_OK || (rc = clear_flag(ctx, &flag)) != ALS_OK)
    return rc;
  ALS_CUDA(cudaMemsetAsync(d, 0, sizeof(int64_t) * cols, ctx->stream));
  if (nnz > 0) {
    dispatch_index(index_bytes, [&](auto ix) {
      count_kernel<<<grid_for(ctx, nnz), 256, 0, ctx->stream>>>((decltype(ix))indices, nnz, cols, d, flag);
      return 0;
    });
    ctx->launches++;
    ALS_CUDA(cudaGetLastError());
  }
  if (cols > 0) ALS_CUDA(cudaMemcpyAsync(counts, d, sizeof(int64_t) * cols, cudaMemcpyDeviceToHost, ctx->stream));
  return read_flag(ctx, flag, "als_weight_column_counts: an index is outside [0, cols)");
}

int weight_row_sums(als_ctx *ctx, int64_t rows, int64_t nnz, const void *indptr, int indptr_bytes, const void *row,
                    int row_bytes, const void *data, int value_kind, bool squares, void *sums_host) {
  const char *who = "als_weight_row_sums";
  Dev<void> keys, tmp, sums;
  Dev<int64_t> perm_in, perm, ip;
  const int sum_bytes = squares || value_kind != ALS_VALUE_F32 ? 8 : 4;
  int rc = sums.alloc(ctx, (int64_t)sum_bytes * std::max<int64_t>(rows, 1));
  if (rc != ALS_OK) return rc;
  if (row) {
    // COO in any order: a stable radix sort of (row, position) gives every row's positions in entry order
    int *flag = nullptr;
    if ((rc = clear_flag(ctx, &flag)) != ALS_OK) return rc;
    if (nnz > 0) {
      dispatch_index(row_bytes, [&](auto rr) {
        count_kernel<<<grid_for(ctx, nnz), 256, 0, ctx->stream>>>((decltype(rr))row, nnz, rows,
                                                                  (unsigned long long *)nullptr, flag);
        return 0;
      });
      ctx->launches++;
      ALS_CUDA(cudaGetLastError());
    }
    char what[96];
    snprintf(what, sizeof(what), "%s: a row index is outside [0, %lld)", who, (long long)rows);
    if ((rc = read_flag(ctx, flag, what)) != ALS_OK) return rc;
    size_t tmp_bytes = 0;
    auto sort = [&](void *t) -> cudaError_t {
      if (row_bytes == 8)
        return cub::DeviceRadixSort::SortPairs(t, tmp_bytes, (const long long *)row, (long long *)keys.get(), perm_in.get(),
                                               perm.get(), nnz, 0, 64, ctx->stream);
      return cub::DeviceRadixSort::SortPairs(t, tmp_bytes, (const int32_t *)row, (int32_t *)keys.get(), perm_in.get(),
                                             perm.get(), nnz, 0, 32, ctx->stream);
    };
    if ((rc = keys.alloc(ctx, (int64_t)row_bytes * std::max<int64_t>(nnz, 1))) != ALS_OK ||
        (rc = perm_in.alloc(ctx, sizeof(int64_t) * std::max<int64_t>(nnz, 1))) != ALS_OK ||
        (rc = perm.alloc(ctx, sizeof(int64_t) * std::max<int64_t>(nnz, 1))) != ALS_OK ||
        (rc = ip.alloc(ctx, sizeof(int64_t) * (rows + 1))) != ALS_OK)
      return rc;
    if (nnz > 0) {
      iota64_kernel<<<grid_for(ctx, nnz), 256, 0, ctx->stream>>>(perm_in, nnz);
      ctx->launches++;
      ALS_CUDA(sort(nullptr));
      if ((rc = tmp.alloc(ctx, (int64_t)tmp_bytes)) != ALS_OK) return rc;
      ALS_CUDA(sort(tmp));
      ctx->launches++;
    }
    dispatch_index(row_bytes, [&](auto rr) {
      indptr_from_sorted_kernel<<<grid_for(ctx, rows + 1), 256, 0, ctx->stream>>>((decltype(rr))keys.get(), nnz, rows, ip);
      return 0;
    });
    ctx->launches++;
    indptr = ip;
    indptr_bytes = 8;
  } else if ((rc = weight_check_indptr(ctx, indptr, indptr_bytes, rows, nnz, who)) != ALS_OK) {
    return rc;
  }
  if (rows > 0) {
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(rows, kWarps), (int64_t)ctx->sm_count * 8));
    dispatch_value(value_kind, [&](auto vt) {
      using V = std::remove_const_t<std::remove_pointer_t<decltype(vt)>>;
      using S = std::conditional_t<sizeof(V) == 4 && V(0.5) != V(0), float,
                                   std::conditional_t<V(0.5) != V(0), double, long long>>;
      return dispatch_index(indptr_bytes, [&](auto ipt) {
        using IP = std::remove_const_t<std::remove_pointer_t<decltype(ipt)>>;
        if (squares)
          row_sums_kernel<V, double, true, IP><<<grid, kWarps * 32, 0, ctx->stream>>>(
              (const IP *)indptr, perm, (const V *)data, rows, (double *)sums.get());
        else
          row_sums_kernel<V, S, false, IP><<<grid, kWarps * 32, 0, ctx->stream>>>((const IP *)indptr, perm, (const V *)data,
                                                                                  rows, (S *)sums.get());
        return 0;
      });
    });
    ctx->launches++;
    ALS_CUDA(cudaGetLastError());
    ALS_CUDA(cudaMemcpyAsync(sums_host, sums, (size_t)sum_bytes * rows, cudaMemcpyDeviceToHost, ctx->stream));
  }
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return ALS_OK;
}

int weight_entries(als_ctx *ctx, int kind, int64_t rows, int64_t cols, int64_t nnz, const void *indptr, int indptr_bytes,
                   const void *row, int row_bytes, const void *indices, int index_bytes, const void *data, int value_kind,
                   const void *row_values_host, const double *idf_host, double k1p1, double k1, int flags, double *out) {
  EntryArgs a{kind, rows, cols, nnz, nullptr, nullptr, k1p1, k1, (flags & ALS_WEIGHT_NUM_F32) != 0,
              (flags & ALS_WEIGHT_DEN_F32) != 0, nullptr};
  Dev<void> rv;
  Dev<double> idf;
  if (nnz == 0) return ALS_OK;
  int rc = clear_flag(ctx, &a.flag);
  if (rc != ALS_OK) return rc;
  if (kind != ALS_WEIGHT_TFIDF) {
    const int64_t bytes = (kind == ALS_WEIGHT_BM25 && a.den32 ? 4 : 8) * rows;
    if ((rc = rv.alloc(ctx, std::max<int64_t>(bytes, 8))) != ALS_OK) return rc;
    ALS_CUDA(cudaMemcpyAsync(rv, row_values_host, (size_t)bytes, cudaMemcpyHostToDevice, ctx->stream));
  }
  if (kind != ALS_WEIGHT_NORMALIZE) {
    if ((rc = idf.alloc(ctx, sizeof(double) * std::max<int64_t>(cols, 1))) != ALS_OK) return rc;
    ALS_CUDA(cudaMemcpyAsync(idf, idf_host, sizeof(double) * cols, cudaMemcpyHostToDevice, ctx->stream));
  }
  a.row_values = rv;
  a.idf = idf;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(nnz, kTile), (int64_t)ctx->sm_count * 8));
  dispatch_value(value_kind, [&](auto vt) {
    using V = std::remove_const_t<std::remove_pointer_t<decltype(vt)>>;
    return dispatch_index(index_bytes, [&](auto ix) {
      using I = std::remove_const_t<std::remove_pointer_t<decltype(ix)>>;
      return dispatch_index(row ? row_bytes : indptr_bytes, [&](auto rt) {
        using X = std::remove_const_t<std::remove_pointer_t<decltype(rt)>>;
        if (row)
          entries_kernel<V, X, X, I><<<grid, 256, 0, ctx->stream>>>(a, nullptr, (const X *)row, (const I *)indices,
                                                                    (const V *)data, out);
        else
          entries_kernel<V, X, X, I><<<grid, 256, 0, ctx->stream>>>(a, (const X *)indptr, nullptr, (const I *)indices,
                                                                    (const V *)data, out);
        return 0;
      });
    });
  });
  ctx->launches++;
  ALS_CUDA(cudaGetLastError());
  return read_flag(ctx, a.flag, "als_weight_entries: a row or column index is outside the matrix");
}

}  // namespace als
