// Ranking metrics at K over the top-k left on the device (reference: ranking_metrics_at_k, implicit/evaluation.pyx:366-475;
// the per-user arithmetic of implicit_b200/evaluation.py).
//
// For each query row: the K ids the top-k produced (ranks past the items are id 0, topk.pyx:20-21) against that row of
// the withheld-items CSR `test`, sorted once by rows_in_order.  L is the number of distinct withheld items (the
// reference's `likes` is a set); rank j hits when its id is in the row (binary search; a repeated id hits each time,
// like the scalar loop).  A warp owns a row and walks its ranks 32 at a time: the running hit count is a ballot prefix,
// the rank terms are summed across the warp in a fixed butterfly order.  Per user, in fp64 and in the host's order of
// operations:
//   hits, min(K, L), AP = sum_hit cum / (j+1) / min(K, L), nDCG = sum_hit gain[j] / gain_sum[min(K, L) - 1],
//   AUC = [sum_miss cum + (hits + L) / 2 (items - L - misses)] / (L (items - L)),
// and users without withheld items count nowhere (evaluation.pyx:421-422).  The gain tables come from the host, so
// they are numpy's values bit for bit.  Sums are deterministic: every CTA owns a fixed block of rows and adds its
// warps' sums in warp order, and one CTA adds the CTA partials in a fixed tree; no atomics.
#include "common.h"

namespace als {
namespace {

constexpr int kWarps = 8;
constexpr int kRowsPerCta = 64;  // fixed, so the partials (and the rounding of the sums) do not depend on the device
constexpr int kSums = 6;         // hits, sum min(K, L), sum AP, sum nDCG, sum AUC, users

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(32 * kWarps) ranking_metrics_kernel(
    const int32_t *__restrict__ ids, int k_eff, int K, int n_query, const int32_t *__restrict__ t_indptr,
    const int32_t *__restrict__ t_indices, const double *__restrict__ gain, const double *__restrict__ gain_sum,
    int64_t n_items, double *__restrict__ partials) {
  __shared__ double part[kWarps][kSums];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double acc[kSums] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  const int q_end = min(n_query, (blockIdx.x + 1) * kRowsPerCta);
  for (int q = blockIdx.x * kRowsPerCta + warp; q < q_end; q += kWarps) {
    const int p0 = t_indptr[q], p1 = t_indptr[q + 1];
    int first_of_value = 0;
    for (int p = p0 + lane; p < p1; p += 32) first_of_value += (p == p0 || t_indices[p] != t_indices[p - 1]);
    const int L = __reduce_add_sync(0xffffffffu, first_of_value);
    if (L == 0) continue;
    int hits = 0;
    double ap = 0.0, dcg = 0.0, auc_miss = 0.0;
    for (int j0 = 0; j0 < K; j0 += 32) {
      const int j = j0 + lane;
      bool hit = false;
      if (j < K) {
        const int id = j < k_eff ? ids[(int64_t)q * k_eff + j] : 0;
        int lo = p0, hi = p1;
        while (lo < hi) {
          const int mid = lo + ((hi - lo) >> 1);
          if (t_indices[mid] < id) lo = mid + 1;
          else hi = mid;
        }
        hit = lo < p1 && t_indices[lo] == id;
      }
      const unsigned m = __ballot_sync(0xffffffffu, hit);
      const int cum = hits + __popc(m & (0xffffffffu >> (31 - lane)));  // hits at ranks <= j
      ap += warp_sum(hit ? (double)cum / (double)(j + 1) : 0.0);
      dcg += warp_sum(hit ? gain[j] : 0.0);
      auc_miss += warp_sum(j < K && !hit ? (double)cum : 0.0);  // integers: exact
      hits += __popc(m);
    }
    if (lane == 0) {
      const double Ld = (double)L, h = (double)hits;
      const double cap = fmin((double)K, Ld);
      const double neg = (double)n_items - Ld, misses = (double)K - h;
      double auc = auc_miss;
      auc += (h + Ld) / 2.0 * (neg - misses);
      acc[0] += h;
      acc[1] += cap;
      acc[2] += ap / cap;
      acc[3] += dcg / gain_sum[(int)cap - 1];
      acc[4] += auc / (Ld * neg);
      acc[5] += 1.0;
    }
  }
  if (lane == 0)
    for (int i = 0; i < kSums; ++i) part[warp][i] = acc[i];
  __syncthreads();
  if (threadIdx.x < kSums) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += part[w][threadIdx.x];
    partials[(int64_t)blockIdx.x * kSums + threadIdx.x] = s;
  }
}

// partials[n][kSums] -> out[kSums]: strided per-thread sums, then a fixed tree
__global__ void __launch_bounds__(256) sum_partials_kernel(const double *__restrict__ partials, int n, double *__restrict__ out) {
  __shared__ double s[256];
  for (int i = 0; i < kSums; ++i) {
    double v = 0.0;
    for (int b = threadIdx.x; b < n; b += 256) v += partials[(int64_t)b * kSums + i];
    s[threadIdx.x] = v;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
      if (threadIdx.x < w) s[threadIdx.x] += s[threadIdx.x + w];
      __syncthreads();
    }
    if (threadIdx.x == 0) out[i] = s[0];
    __syncthreads();
  }
}

}  // namespace

int launch_ranking_metrics(als_ctx *ctx, const als_factors *items, const als_factors *queries, const int32_t *query_rows,
                           int64_t n_query, int k, const als_csr *liked, const als_csr *test, const double *gain_host,
                           const double *gain_sum_host, double *sums) {
  for (int i = 0; i < kSums; ++i) sums[i] = 0.0;
  if (n_query == 0 || test->nnz == 0) return ALS_OK;  // no user has withheld items
  const int32_t *t_indptr = nullptr, *t_indices = nullptr;
  int rc = rows_in_order(ctx, test, &t_indptr, &t_indices);
  if (rc != ALS_OK) return rc;
  TopkIds rows;
  rows.p = query_rows;
  rows.n = query_rows ? n_query : 0;
  TopkDevice t;
  if ((rc = topk_device(ctx, items, queries, rows, n_query, k, nullptr, false, liked, TopkIds(), &t)) != ALS_OK) return rc;
  // the ids stay in ctx->scratch: what this pass needs comes from the pool
  const int grid = (int)ceil_div(n_query, kRowsPerCta);
  Dev<double> buf;
  if ((rc = buf.alloc(ctx, (2 * (int64_t)k + (int64_t)(grid + 1) * kSums) * sizeof(double))) != ALS_OK) return rc;
  double *gain = buf, *gain_sum = buf + k, *partials = buf + 2 * (int64_t)k, *out = partials + (int64_t)grid * kSums;
  ALS_CUDA(cudaMemcpyAsync(gain, gain_host, k * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  ALS_CUDA(cudaMemcpyAsync(gain_sum, gain_sum_host, k * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  ranking_metrics_kernel<<<grid, 32 * kWarps, 0, ctx->stream>>>(t.ids, t.k_eff, k, (int)n_query, t_indptr, t_indices, gain,
                                                               gain_sum, items->rows, partials);
  ALS_CUDA(cudaGetLastError());
  sum_partials_kernel<<<1, 256, 0, ctx->stream>>>(partials, grid, out);
  ALS_CUDA(cudaGetLastError());
  ctx->launches += 2;
  ALS_CUDA(cudaMemcpyAsync(sums, out, kSums * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return ALS_OK;
}

}  // namespace als
