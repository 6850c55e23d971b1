// Synthetic power-law CSR and initial factors generated ON THE DEVICE (SURVEY.md section 8(d), BASELINE.json configs).
//
// The host generator (implicit_b200/synthetic.py) is the bit-exact one for C1..C3 and C5; C4 (10M x 1M, 500M
// nonzeros) needs ~30 GB of transient host memory and minutes of numpy there, and only statistical equivalence is
// required of it (its parity is 8 GPUs against 1 GPU plus an oracle check on a row sample).  Same recipe, counter-based
// hashing instead of numpy's PCG64:  m = 1.25 nnz draws of (user ~ plaw(0.5), item ~ plaw(0.8)) through two random
// permutations, keys = user * items + item sorted and de-duplicated (cub), thinned to ~nnz by an independent
// Bernoulli draw per key, values 1 + 4 U[0,1).  Deterministic for a given seed, independent of the grid.
// (No reference equivalent: the reference loads datasets from disk, implicit/datasets/.)
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>

#include "common.h"

namespace als {

namespace {

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {  // splitmix64 finaliser
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}
__device__ __forceinline__ uint64_t hash3(uint64_t seed, uint64_t stream, uint64_t i) {
  return mix64(mix64(seed * 0x2545f4914f6cdd1dull + stream) ^ (i * 0x9e3779b97f4a7c15ull));
}
__device__ __forceinline__ double u01(uint64_t h) { return (double)(h >> 11) * (1.0 / 9007199254740992.0); }

// truncated power law p(j) ~ (j + 1)^-a on [0, N) by inverse CDF (synthetic.py plaw)
__device__ __forceinline__ int64_t plaw(double r, int64_t N, double a) {
  const double x = pow((pow((double)N, 1.0 - a) - 1.0) * r + 1.0, 1.0 / (1.0 - a));
  int64_t j = (int64_t)floor(x) - 1;
  return j < 0 ? 0 : j >= N ? N - 1 : j;
}

__global__ void perm_keys_kernel(uint64_t *keys, int32_t *vals, int64_t n, uint64_t seed, uint64_t stream) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    keys[i] = hash3(seed, stream, (uint64_t)i);
    vals[i] = (int32_t)i;
  }
}

__global__ void draw_keys_kernel(uint64_t *keys, int64_t m, int64_t users, int64_t items, const int32_t *__restrict__ pu,
                                 const int32_t *__restrict__ pi, uint64_t seed) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < m; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t u = plaw(u01(hash3(seed, 11, (uint64_t)t)), users, 0.5);
    const int64_t i = plaw(u01(hash3(seed, 12, (uint64_t)t)), items, 0.8);
    keys[t] = (uint64_t)pu[u] * (uint64_t)items + (uint64_t)pi[i];
  }
}

struct KeepKey {
  uint64_t seed, threshold;  // keep when the key's hash is below the threshold
  __device__ bool operator()(const uint64_t &k) const { return hash3(seed, 13, k) < threshold; }
};

__global__ void split_keys_kernel(const uint64_t *__restrict__ keys, int64_t n, int64_t items, int32_t *__restrict__ indices,
                                  float *__restrict__ data, uint64_t seed) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    indices[e] = (int32_t)(keys[e] % (uint64_t)items);
    data[e] = 1.f + 4.f * (float)u01(hash3(seed, 14, keys[e]));
  }
}

// indptr[r] = first position whose key is >= r * items (keys sorted)
__global__ void indptr_kernel(const uint64_t *__restrict__ keys, int64_t n, int64_t rows, int64_t items, int32_t *__restrict__ indptr) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r <= rows; r += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t target = (uint64_t)r * (uint64_t)items;
    int64_t lo = 0, hi = n;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (keys[mid] < target) lo = mid + 1;
      else hi = mid;
    }
    indptr[r] = (int32_t)lo;
  }
}

__global__ void fill_uniform_kernel(float *x, int64_t rows, int f, int ld, uint64_t seed, float scale) {
  const int64_t n = rows * ld;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(e % ld);
    x[e] = j < f ? scale * (float)u01(hash3(seed, 21, (uint64_t)((e / ld) * f + j))) : 0.f;
  }
}

int random_permutation(als_ctx *ctx, int64_t n, uint64_t seed, uint64_t stream, Dev<int32_t> &out) {
  Dev<uint64_t> k_in, k_out;
  Dev<int32_t> v_in, v_out;
  Dev<void> tmp;
  size_t tmp_bytes = 0;
  int rc;
  if ((rc = k_in.alloc_cuda(ctx, n * 8)) != ALS_OK || (rc = k_out.alloc_cuda(ctx, n * 8)) != ALS_OK ||
      (rc = v_in.alloc_cuda(ctx, n * 4)) != ALS_OK || (rc = v_out.alloc_cuda(ctx, n * 4)) != ALS_OK)
    return rc;
  perm_keys_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(k_in, v_in, n, seed, stream);
  cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, k_in.get(), k_out.get(), v_in.get(), v_out.get(), (int)n, 0, 64,
                                  ctx->stream);
  if ((rc = tmp.alloc_cuda(ctx, (int64_t)tmp_bytes)) != ALS_OK) return rc;
  cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, k_in.get(), k_out.get(), v_in.get(), v_out.get(), (int)n, 0, 64, ctx->stream);
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  out = std::move(v_out);
  return ALS_OK;
}

}  // namespace

int csr_generate_power_law(als_ctx *ctx, int64_t users, int64_t items, int64_t nnz_target, uint64_t seed, als_csr **out) {
  const int64_t m = nnz_target + nnz_target / 4;
  if (m >= (int64_t)INT32_MAX || users >= (int64_t)INT32_MAX || items >= (int64_t)INT32_MAX) {
    set_error("csr_generate: sizes beyond int32 (m = %lld)", (long long)m);
    return ALS_E_UNSUPPORTED;
  }
  Dev<int32_t> pu, pi;
  int rc;
  if ((rc = random_permutation(ctx, users, seed, 1, pu)) != ALS_OK) return rc;
  if ((rc = random_permutation(ctx, items, seed, 2, pi)) != ALS_OK) return rc;
  Dev<uint64_t> k_a, k_b;
  Dev<int64_t> d_count;
  if ((rc = k_a.alloc_cuda(ctx, m * 8)) != ALS_OK || (rc = k_b.alloc_cuda(ctx, m * 8)) != ALS_OK ||
      (rc = d_count.alloc_cuda(ctx, 8)) != ALS_OK)
    return rc;
  draw_keys_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(k_a, m, users, items, pu, pi, seed);
  Dev<void> tmp;
  size_t t1 = 0, t2 = 0, t3 = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, t1, k_a.get(), k_b.get(), (int)m, 0, 64, ctx->stream);
  cub::DeviceSelect::Unique(nullptr, t2, k_b.get(), k_a.get(), d_count.get(), (int)m, ctx->stream);
  KeepKey keep{seed, 0};
  cub::DeviceSelect::If(nullptr, t3, k_a.get(), k_b.get(), d_count.get(), (int)m, keep, ctx->stream);
  size_t tb = std::max(std::max(t1, t2), std::max<size_t>(t3, 16));
  if ((rc = tmp.alloc_cuda(ctx, (int64_t)tb)) != ALS_OK) return rc;
  cub::DeviceRadixSort::SortKeys(tmp, tb, k_a.get(), k_b.get(), (int)m, 0, 64, ctx->stream);       // k_b sorted
  cub::DeviceSelect::Unique(tmp, tb, k_b.get(), k_a.get(), d_count.get(), (int)m, ctx->stream);    // k_a unique
  int64_t n_unique = 0;
  ALS_CUDA(cudaMemcpyAsync(&n_unique, d_count, 8, cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  const uint64_t *keys = k_a;
  int64_t nnz = n_unique;
  if (n_unique > nnz_target) {  // thin to ~nnz_target: every key kept independently with probability nnz_target / n_unique
    const long double p = (long double)nnz_target / (long double)n_unique;
    keep.threshold = (uint64_t)(p * 18446744073709551615.0L);
    cub::DeviceSelect::If(tmp, tb, k_a.get(), k_b.get(), d_count.get(), (int)n_unique, keep, ctx->stream);
    ALS_CUDA(cudaMemcpyAsync(&nnz, d_count, 8, cudaMemcpyDeviceToHost, ctx->stream));
    ALS_CUDA(cudaStreamSynchronize(ctx->stream));
    keys = k_b;
  }
  tmp.reset();
  pu.reset();
  pi.reset();
  CsrHolder c = new_csr(ctx);
  c->rows = users;
  c->cols = items;
  c->nnz = nnz;
  c->row_offset = 0;
  if ((rc = dev_alloc(ctx, (void **)&c->indptr, sizeof(int32_t) * (users + 1))) != ALS_OK ||
      (rc = dev_alloc(ctx, (void **)&c->indices, sizeof(int32_t) * std::max<int64_t>(nnz, 1))) != ALS_OK ||
      (rc = dev_alloc(ctx, (void **)&c->data, sizeof(float) * std::max<int64_t>(nnz, 1))) != ALS_OK)
    return rc;
  split_keys_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(keys, nnz, items, c->indices, c->data, seed);
  indptr_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(keys, nnz, users, items, c->indptr);
  ALS_CUDA(cudaGetLastError());
  std::vector<int32_t> ip((size_t)users + 1);
  ALS_CUDA(cudaMemcpyAsync(ip.data(), c->indptr, sizeof(int32_t) * (users + 1), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  k_a.reset();
  k_b.reset();
  d_count.reset();
  if ((rc = build_schedule(ctx, c.get(), ip.data())) != ALS_OK) return rc;
  *out = c.release();
  return ALS_OK;
}

int factors_fill_uniform(als_ctx *ctx, als_factors *f, uint64_t seed, float scale) {
  fill_uniform_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(f->d, f->rows, f->f, f->ld, seed, scale);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  return ALS_OK;
}

}  // namespace als
