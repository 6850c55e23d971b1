// Synthetic power-law CSR and initial factors generated ON THE DEVICE (SURVEY.md section 8(d), BASELINE.json configs).
//
// The host generator (implicit_b200/synthetic.py) is the bit-exact one for C1..C3 and C5; C4 (10M x 1M, 500M
// nonzeros) needs ~30 GB of transient host memory and minutes of numpy there, and only statistical equivalence is
// required of it (its parity is 8 GPUs against 1 GPU plus an oracle check on a row sample).  Same recipe, counter-based
// hashing instead of numpy's PCG64:  m = 1.25 nnz draws of (user ~ plaw(0.5), item ~ plaw(0.8)) through two random
// permutations, keys = user * items + item sorted and de-duplicated (cub), thinned to ~nnz by an independent
// Bernoulli draw per key, values 1 + 4 u with u = U[0,1) rounded to float, so in [1, 5]: 5 itself for 3 keys in 2^25,
// where u rounds to 1.0f or to 1 - 2^-24 (whose 1 + 4 u ties to 5).  Deterministic for a given seed, independent of
// the grid; tests/_gen_restate.py restates it in numpy.
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

// ---- numpy's PCG64 float32 stream (implicit_b200/pcg64.py restates it in Python ints) --------------------------------
// A 64-bit draw steps the 128-bit LCG, s = s * MULT + inc (mod 2^128), and outputs rotr64(hi ^ lo, hi >> 58) of the new
// state; random(..., dtype=float32) takes its low 32-bit half, then its high half, each as (u32 >> 8) * 2^-24.
typedef unsigned __int128 u128;

constexpr u128 PCG_MULT = ((u128)0x2360ED051FC65DA4ull << 64) | 0x4385DF649FCCF645ull;
constexpr int PCG_THREADS = 128;
constexpr int PCG_DRAWS = 16;                                // 64-bit draws per thread and tile: 32 consecutive values
constexpr int PCG_TILE = PCG_THREADS * PCG_DRAWS * 2;        // values per tile
constexpr int PCG_BITS = 64;

struct PcgJumps {
  u128 mult[PCG_BITS], plus[PCG_BITS];  // s -> mult[j] s + plus[j] advances 2^j draws
  u128 stride_mult, stride_plus;        // advances gridDim.x tiles
};

__device__ __forceinline__ float pcg_value(uint32_t u, float scale) {
  return __fmul_rn((float)(u >> 8) * 0x1p-24f, scale);  // numpy's float32 product, never contracted into an FMA
}

// Value p of m (p = 0, 1, ...: the low then the high half of draw p / 2 + 1 after s0) goes to element first + p of the
// C-order (rows, f) matrix x of row stride ld; with first = 1, element 0 is the buffered half u0.  Each thread owns the
// 32 values of PCG_DRAWS consecutive draws of a tile: it jumps to its first draw once, then by the grid's stride, and the
// block stages the tile in shared memory so the stores are coalesced.  fdiv = ceil(2^32 / f) for f >= 2:
// __umulhi(c, fdiv) = c / f for every c < 2^19 (the error c (fdiv - 2^32 / f) / 2^32 stays below 1 / f).
__global__ void __launch_bounds__(PCG_THREADS) fill_pcg64_kernel(float *__restrict__ x, int64_t m, int first, uint32_t u0,
                                                                  int f, int ld, uint32_t fdiv, u128 s0, u128 inc,
                                                                  float scale, const __grid_constant__ PcgJumps jumps) {
  __shared__ float tile[PCG_TILE + PCG_TILE / 32];  // one pad word per 32 values: conflict-free both ways
  if (first && blockIdx.x == 0 && threadIdx.x == 0) x[0] = pcg_value(u0, scale);
  const int64_t tiles = (m + PCG_TILE - 1) / PCG_TILE;
  u128 start = s0;  // the state before this thread's first draw of the current tile
  {
    uint64_t k = (uint64_t)blockIdx.x * (PCG_TILE / 2) + threadIdx.x * PCG_DRAWS;
    for (int j = 0; k; ++j, k >>= 1)
      if (k & 1) start = jumps.mult[j] * start + jumps.plus[j];
  }
  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int64_t p0 = t * PCG_TILE;
    if (p0 + threadIdx.x * 2 * PCG_DRAWS < m) {
      u128 s = start;
#pragma unroll
      for (int d = 0; d < PCG_DRAWS; ++d) {
        s = s * PCG_MULT + inc;
        const uint64_t hi = (uint64_t)(s >> 64), v0 = hi ^ (uint64_t)s;
        const unsigned rot = (unsigned)(hi >> 58);
        const uint64_t v = (v0 >> rot) | (v0 << ((64 - rot) & 63));
        const int l = threadIdx.x * 2 * PCG_DRAWS + 2 * d;  // even: l and l + 1 share their 32-value group
        tile[l + l / 32] = pcg_value((uint32_t)v, scale);
        tile[l + 1 + l / 32] = pcg_value((uint32_t)(v >> 32), scale);
      }
    }
    start = jumps.stride_mult * start + jumps.stride_plus;
    __syncthreads();
    const int64_t e0 = p0 + first;
    const int64_t r0 = e0 / f;
    const uint32_t c0 = (uint32_t)(e0 - r0 * f);
    float *const row = x + r0 * ld;  // the tile's rows lie within 2^32 elements of its first row
    const int valid = m - p0 < PCG_TILE ? (int)(m - p0) : PCG_TILE;
    for (int l = threadIdx.x; l < valid; l += PCG_THREADS) {
      const uint32_t c = c0 + l;
      const uint32_t q = f == 1 ? c : __umulhi(c, fdiv);
      row[q * (uint32_t)ld + (c - q * (uint32_t)f)] = tile[l + l / 32];
    }
    __syncthreads();
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
  ALS_CUDA(cudaGetLastError());
  ALS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, k_in.get(), k_out.get(), v_in.get(), v_out.get(), (int)n,
                                           0, 64, ctx->stream));
  if ((rc = tmp.alloc_cuda(ctx, (int64_t)tmp_bytes)) != ALS_OK) return rc;
  ALS_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, k_in.get(), k_out.get(), v_in.get(), v_out.get(), (int)n, 0, 64,
                                           ctx->stream));
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
  ALS_CUDA(cudaGetLastError());
  Dev<void> tmp;
  size_t t1 = 0, t2 = 0, t3 = 0;
  ALS_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, t1, k_a.get(), k_b.get(), (int)m, 0, 64, ctx->stream));
  ALS_CUDA(cub::DeviceSelect::Unique(nullptr, t2, k_b.get(), k_a.get(), d_count.get(), (int)m, ctx->stream));
  KeepKey keep{seed, 0};
  ALS_CUDA(cub::DeviceSelect::If(nullptr, t3, k_a.get(), k_b.get(), d_count.get(), (int)m, keep, ctx->stream));
  size_t tb = std::max(std::max(t1, t2), std::max<size_t>(t3, 16));
  if ((rc = tmp.alloc_cuda(ctx, (int64_t)tb)) != ALS_OK) return rc;
  ALS_CUDA(cub::DeviceRadixSort::SortKeys(tmp, tb, k_a.get(), k_b.get(), (int)m, 0, 64, ctx->stream));     // k_b sorted
  ALS_CUDA(cub::DeviceSelect::Unique(tmp, tb, k_b.get(), k_a.get(), d_count.get(), (int)m, ctx->stream));  // k_a unique
  int64_t n_unique = 0;
  ALS_CUDA(cudaMemcpyAsync(&n_unique, d_count, 8, cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  const uint64_t *keys = k_a;
  int64_t nnz = n_unique;
  if (n_unique > nnz_target) {  // thin to ~nnz_target: every key kept independently with probability nnz_target / n_unique
    const long double p = (long double)nnz_target / (long double)n_unique;
    keep.threshold = (uint64_t)(p * 18446744073709551615.0L);
    ALS_CUDA(cub::DeviceSelect::If(tmp, tb, k_a.get(), k_b.get(), d_count.get(), (int)n_unique, keep, ctx->stream));
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

int factors_fill_pcg64(als_ctx *ctx, als_factors *f, uint64_t state_hi, uint64_t state_lo, uint64_t inc_hi,
                       uint64_t inc_lo, int has_uint32, uint32_t uinteger, float scale) {
  const int64_t n = f->rows * f->f;
  if (n == 0) return ALS_OK;
  const int first = has_uint32 ? 1 : 0;
  const int64_t m = n - first;
  const u128 inc = ((u128)inc_hi << 64) | inc_lo;
  PcgJumps jumps;
  u128 mult = PCG_MULT, plus = inc;  // the map of 2^j draws, j = 0, 1, ...
  for (int j = 0; j < PCG_BITS; ++j) {
    jumps.mult[j] = mult;
    jumps.plus[j] = plus;
    plus = (mult + 1) * plus;
    mult = mult * mult;
  }
  const int64_t tiles = (m + PCG_TILE - 1) / PCG_TILE;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(tiles, (int64_t)ctx->sm_count * 8));
  // the stride of a grid-stride step, grid * PCG_TILE / 2 draws, composed from the maps of its bits
  u128 sm = 1, sp = 0;
  for (uint64_t k = (uint64_t)grid * (PCG_TILE / 2), j = 0; k; ++j, k >>= 1)
    if (k & 1) {
      sm = jumps.mult[j] * sm;
      sp = jumps.mult[j] * sp + jumps.plus[j];
    }
  jumps.stride_mult = sm;
  jumps.stride_plus = sp;
  const uint32_t fdiv = f->f == 1 ? 0 : (uint32_t)(((1ull << 32) + (uint64_t)f->f - 1) / (uint64_t)f->f);
  fill_pcg64_kernel<<<grid, PCG_THREADS, 0, ctx->stream>>>(f->d, m, first, uinteger, f->f, f->ld, fdiv,
                                                            ((u128)state_hi << 64) | state_lo, inc, scale, jumps);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  return ALS_OK;
}

}  // namespace als
