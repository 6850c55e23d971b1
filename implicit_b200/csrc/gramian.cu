// R4: Gramian  G = Y^T Y  (reference: np.dot(Y.T, Y), implicit/cpu/_als.pyx:70,164,268;
// LeastSquaresSolver::calculate_yty, implicit/gpu/als.cu:122-152).
//
// Bandwidth-bound reduction over the rows of Y (f/2 flop per byte): every CTA streams rows through shared
// memory and writes one F x F partial; a second tiny kernel sums the partials in a fixed order in fp64 so the
// result is deterministic and independent of the grid size rounding.
//   64 padded factors: gramian_tc_kernel on wgmma (dense.cu), unless the gramian_fma knob is set;
//   f <= 128: gramian_partial_kernel -- fp32 FMA register tiles (the CG configurations);
//   128 < padded factors <= 1024: gramian_wide_kernel -- fp32 FMA 4 x 4 register tiles per 64 x 64 tile of G.
// No fp32 register accumulator adds more than kFoldRows = 256 rows: each FMA kernel then folds its register tile into
// a second accumulator (fp32 in shared memory at <= 128 factors, fp64 above), and the wgmma kernel adds chains of 64
// rows into fp32 registers.  One fp32 chain over all of a thread's rows (350k rows in the wide kernel at 2^20 rows and
// 1024 factors, 38k in the partial kernel at 10M rows) walks far outside |G - G64| <= 1e-6 |Y|^T|Y| elementwise
// (tests/test_gpu_gramian_widths.py); so did an mma.sync 3xTF32 variant, 8-11x at a million rows on one H100.
#include <limits.h>

#include "cholesky_device.cuh"

namespace als {

namespace {

constexpr int kGramRows = 32;   // rows of Y staged per step (FMA version)
constexpr int kFoldRows = 256;  // rows an fp32 register accumulator adds at most before it is folded

// fp32 FMA version (round-to-nearest accumulation).  Thread (ty, tx) of the 16 x 16 block owns the T x T
// sub-block of G at rows T ty .. T ty + T - 1, columns T tx .. T tx + T - 1 (T = F / 16), so both of its operands
// are contiguous in a staged row and arrive as 16-byte shared-memory loads: T^2 FMAs per 2 T / 4 loads.
// Every kFoldRows / kGramRows steps of the CTA, and after its last step, the register tile is added into the thread's
// fp32 second level in dynamic shared memory, T^2 x 256 floats at word (i T + j) 256 + thread (conflict-free), and the
// partial is written from there: registers have no room for a second level at T = 8 with two CTAs per SM, and adding
// the register tile at the store instead spills at T = 8.  Two fp32 levels suffice, as 2 x SMs CTAs share the rows:
// an fp32 emulation of 10M rows at 128 factors stays within 0.02 of the bar.
template <int T>  // F = 16 * T
__global__ void __launch_bounds__(256) gramian_partial_kernel(const float *__restrict__ Y, int64_t rows, int ld,
                                                              float *__restrict__ partials) {
  constexpr int F = 16 * T;
  __shared__ __align__(16) float tile[kGramRows][F];
  extern __shared__ float folded[];  // [T * T][256]
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[T][T];
#pragma unroll
  for (int a = 0; a < T; ++a)
#pragma unroll
    for (int b = 0; b < T; ++b) {
      acc[a][b] = 0.f;
      folded[(a * T + b) * 256 + threadIdx.x] = 0.f;
    }

  const int64_t steps = (rows + kGramRows - 1) / kGramRows;
  int pending = 0;
  for (int64_t s = blockIdx.x; s < steps; s += gridDim.x) {
    const int64_t r0 = s * kGramRows;
    // coalesced float4 staging (ld == F by construction)
    for (int e = threadIdx.x; e < kGramRows * F / 4; e += 256) {
      const int r = e / (F / 4), c4 = e % (F / 4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r0 + r < rows) v = __ldg(reinterpret_cast<const float4 *>(Y + (r0 + r) * ld) + c4);
      reinterpret_cast<float4 *>(&tile[r][0])[c4] = v;
    }
    __syncthreads();
#pragma unroll 4
    for (int r = 0; r < kGramRows; ++r) {
      float a[T], b[T];
      if constexpr (T % 4 == 0) {
#pragma unroll
        for (int i = 0; i < T; i += 4) {
          const float4 va = *reinterpret_cast<const float4 *>(&tile[r][T * ty + i]);  // 2 addresses per warp
          const float4 vb = *reinterpret_cast<const float4 *>(&tile[r][T * tx + i]);  // contiguous across tx
          a[i] = va.x; a[i + 1] = va.y; a[i + 2] = va.z; a[i + 3] = va.w;
          b[i] = vb.x; b[i + 1] = vb.y; b[i + 2] = vb.z; b[i + 3] = vb.w;
        }
      } else {
#pragma unroll
        for (int i = 0; i < T; ++i) {
          a[i] = tile[r][T * ty + i];
          b[i] = tile[r][T * tx + i];
        }
      }
#pragma unroll
      for (int i = 0; i < T; ++i)
#pragma unroll
        for (int j = 0; j < T; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
    if (++pending == kFoldRows / kGramRows || s + gridDim.x >= steps) {
      pending = 0;
#pragma unroll
      for (int i = 0; i < T; ++i)
#pragma unroll
        for (int j = 0; j < T; ++j) {
          folded[(i * T + j) * 256 + threadIdx.x] += acc[i][j];
          acc[i][j] = 0.f;
        }
    }
  }
  float *out = partials + (size_t)blockIdx.x * F * F;
#pragma unroll
  for (int i = 0; i < T; ++i)
#pragma unroll
    for (int j = 0; j < T; ++j) out[(T * ty + i) * F + T * tx + j] = folded[(i * T + j) * 256 + threadIdx.x];
}

// 128 < padded factors <= 1024: one 64 x 64 tile of G per CTA and row chunk (blockIdx = (tile column, tile row, chunk)),
// fp32 FMA register tiles of 4 x 4 per thread, added every kFoldRows rows into an fp64 tile in shared memory (registers
// would cost a CTA per SM); the chunk partials are summed in fp64 in a fixed order like the others.
__global__ void __launch_bounds__(256) gramian_wide_kernel(const float *__restrict__ Y, int64_t rows, int ld, float *__restrict__ partials,
                                                           int64_t rows_per_part) {
  __shared__ __align__(16) float A[16][64], B[16][64];
  __shared__ double folded[16][256];  // [4 i + j][thread]
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int bj = blockIdx.x, bi = blockIdx.y;
  const int64_t r0 = (int64_t)blockIdx.z * rows_per_part, r1 = min(rows, r0 + rows_per_part);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      acc[i][j] = 0.f;
      folded[4 * i + j][threadIdx.x] = 0.0;
    }
  int pending = 0;
  for (int64_t r = r0; r < r1; r += 16) {
    const int64_t row = r + ty;  // 16 rows x 16 float4 words: one word of each tile per thread
    float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vb = va;
    if (row < r1) {
      va = __ldg(reinterpret_cast<const float4 *>(Y + row * ld + 64 * bi) + tx);
      vb = __ldg(reinterpret_cast<const float4 *>(Y + row * ld + 64 * bj) + tx);
    }
    reinterpret_cast<float4 *>(&A[ty][0])[tx] = va;
    reinterpret_cast<float4 *>(&B[ty][0])[tx] = vb;
    __syncthreads();
#pragma unroll
    for (int rr = 0; rr < 16; ++rr) {
      const float4 a = *reinterpret_cast<const float4 *>(&A[rr][4 * ty]);
      const float4 b = *reinterpret_cast<const float4 *>(&B[rr][4 * tx]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
    if (++pending == kFoldRows / 16) {
      pending = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          folded[4 * i + j][threadIdx.x] += acc[i][j];
          acc[i][j] = 0.f;
        }
    }
  }
  float v[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) v[i][j] = (float)(folded[4 * i + j][threadIdx.x] + acc[i][j]);
  float *out = partials + (size_t)blockIdx.z * ld * ld;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    *reinterpret_cast<float4 *>(out + (size_t)(64 * bi + 4 * ty + i) * ld + 64 * bj + 4 * tx) =
        make_float4(v[i][0], v[i][1], v[i][2], v[i][3]);
}

// 32 consecutive elements x 8 groups of partials per block: group pg sums partials pg, pg + 8, ... in fp64, the 8
// group sums are added in a fixed order -> deterministic, and the loads of a warp are contiguous.
// (Multi-GPU) element n of G carries "a row of this rank's last solve was not positive definite": the all-reduce of
// the Gramian then tells every rank that some rank failed, without any extra collective or host round trip.
__global__ void __launch_bounds__(256) gramian_reduce_kernel(const float *__restrict__ partials, int nparts, int n,
                                                             float *__restrict__ G, const long long *__restrict__ bad_row) {
  if (blockIdx.x == 0 && threadIdx.x == 0) G[n] = (bad_row[0] != LLONG_MAX || bad_row[1] != LLONG_MAX) ? 1.f : 0.f;
  __shared__ double part[8][33];
  const int el = threadIdx.x & 31, pg = threadIdx.x >> 5;
  const int e = blockIdx.x * 32 + el;
  double s = 0.0;
  if (e < n)
    for (int p = pg; p < nparts; p += 8) s += (double)partials[(size_t)p * n + e];
  part[pg][el] = s;
  __syncthreads();
  if (pg == 0 && e < n) {
    double tot = 0.0;
#pragma unroll
    for (int q = 0; q < 8; ++q) tot += part[q][el];
    G[e] = (float)tot;
  }
}

// Greg = G + lambda I on the real dimensions, identity on the zero-padded ones (so that padded
// unknowns solve to exactly 0 even with lambda == 0).  Mirrors `YtY + regularization * np.eye(f)`
// (implicit/cpu/_als.pyx:85, :164): an fp32 add of fp32(lambda).
__global__ void regularize_kernel(const float *__restrict__ G, float *__restrict__ Greg, int f, int ld, float lambda,
                                  int32_t *__restrict__ status) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e == 0 && G[ld * ld] > 0.f) status[0] = 1;  // the flag that rode along with the all-reduced Gramian (sticky)
  if (e >= ld * ld) return;
  const int i = e / ld, j = e % ld;
  float v = G[e];
  if (i == j) v = (i < f) ? v + lambda : 1.0f;
  Greg[e] = v;
}

template <int T>
static int run_gramian(als_ctx *ctx, const als_factors *Y, int grid) {
  const int smem = T * T * 256 * (int)sizeof(float);  // the fp32 second level; up to 64 KB at T = 8
  ALS_CUDA(cudaFuncSetAttribute(gramian_partial_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  gramian_partial_kernel<T><<<grid, 256, smem, ctx->stream>>>(Y->d, Y->rows, Y->ld, ctx->gram_partials);
  return ALS_OK;
}

}  // namespace

int launch_gramian(als_ctx *ctx, const als_factors *Y) {
  const int F = Y->ld;
  if (F > 128) {
    if (F % 128 != 0 || F > 1024) {
      set_error("gramian: factors=%d (padded %d): beyond 128 the padded width must be a multiple of 128 up to 1024", Y->f, F);
      return ALS_E_UNSUPPORTED;
    }
    const int T = F / 64;
    const int64_t rows = std::max<int64_t>(Y->rows, 0);
    int64_t np = std::min<int64_t>(ceil_div(std::max<int64_t>(rows, 1), 64), (int64_t)ctx->sm_count * 4 / (T * T) + 1);
    const int nparts = (int)std::max<int64_t>(1, std::min<int64_t>(np, 64));
    const int64_t rows_per_part = ceil_div(ceil_div(std::max<int64_t>(rows, 1), nparts), 16) * 16;
    const int64_t need = (int64_t)nparts * F * F;
    if (need > ctx->gram_partials_cap) {
      if (ctx->gram_partials) {
        ALS_CUDA(cudaStreamSynchronize(ctx->stream));
        ALS_CUDA(cudaFree(ctx->gram_partials));
        ctx->gram_partials = nullptr;
      }
      ALS_CUDA(cudaMalloc(&ctx->gram_partials, sizeof(float) * need));
      ctx->gram_partials_cap = need;
    }
    ProfScope prof(ctx, kProfGramian);
    gramian_wide_kernel<<<dim3(T, T, nparts), 256, 0, ctx->stream>>>(Y->d, rows, F, ctx->gram_partials, rows_per_part);
    ALS_CUDA(cudaGetLastError());
    gramian_reduce_kernel<<<(F * F + 31) / 32, 256, 0, ctx->stream>>>(ctx->gram_partials, nparts, F * F, ctx->G, ctx->bad_row);
    ALS_CUDA(cudaGetLastError());
    ctx->launches += 2;
    return ALS_OK;
  }
  // Other widths: the FMA version (round to nearest).
  if (F == 64 && Y->rows >= 128 && !ctx->knobs.gramian_fma) {  // (a TMA box is 128 rows)
    ProfScope prof(ctx, kProfGramian);
    return launch_gramian_tc(ctx, Y);  // wgmma + TMA (dense.cu)
  }
  const int64_t steps = ceil_div(std::max<int64_t>(Y->rows, 1), kGramRows);
  const int grid = (int)std::min<int64_t>(steps, (int64_t)ctx->sm_count * 2);
  const int64_t need = (int64_t)grid * F * F;
  if (need > ctx->gram_partials_cap) {
    if (ctx->gram_partials) {
      ALS_CUDA(cudaStreamSynchronize(ctx->stream));
      ALS_CUDA(cudaFree(ctx->gram_partials));
      ctx->gram_partials = nullptr;
    }
    const int64_t cap = std::max<int64_t>(need, (int64_t)ctx->sm_count * 2 * 128 * 128);
    ALS_CUDA(cudaMalloc(&ctx->gram_partials, sizeof(float) * cap));
    ctx->gram_partials_cap = cap;
  }
  ProfScope prof(ctx, kProfGramian);
  int rc = ALS_OK;
  switch (F / 16) {
    case 1: rc = run_gramian<1>(ctx, Y, grid); break;
    case 2: rc = run_gramian<2>(ctx, Y, grid); break;
    case 3: rc = run_gramian<3>(ctx, Y, grid); break;
    case 4: rc = run_gramian<4>(ctx, Y, grid); break;
    case 5: rc = run_gramian<5>(ctx, Y, grid); break;
    case 6: rc = run_gramian<6>(ctx, Y, grid); break;
    case 7: rc = run_gramian<7>(ctx, Y, grid); break;
    case 8: rc = run_gramian<8>(ctx, Y, grid); break;
    default: set_error("gramian: bad padded factors %d", F); return ALS_E_UNSUPPORTED;
  }
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaGetLastError());
  gramian_reduce_kernel<<<(F * F + 31) / 32, 256, 0, ctx->stream>>>(ctx->gram_partials, grid, F * F, ctx->G, ctx->bad_row);
  ALS_CUDA(cudaGetLastError());
  ctx->launches += 2;
  return ALS_OK;
}

int launch_gramian_reduce(als_ctx *ctx, int nparts, int n) {
  gramian_reduce_kernel<<<(n + 31) / 32, 256, 0, ctx->stream>>>(ctx->gram_partials, nparts, n, ctx->G, ctx->bad_row);
  ALS_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return ALS_OK;
}

int launch_regularize(als_ctx *ctx, int f, int ld, float lambda) {
  regularize_kernel<<<(ld * ld + 255) / 256, 256, 0, ctx->stream>>>(ctx->G, ctx->Greg, f, ld, lambda, ctx->status);
  ctx->gram_ld = ld;
  ALS_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return ALS_OK;
}

}  // namespace als
