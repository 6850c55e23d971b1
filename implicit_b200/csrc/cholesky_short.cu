// R1, short rows: the same solve as cholesky.cu (reference: _least_squares, implicit/cpu/_als.pyx:76-142) for a
// row with n nonzeros, n well below the factor count F, through the n x n "push-through" system instead of the
// F x F normal equations.
//
// With G = Y^T Y + lambda I = R^T R (shared by every row of the half), P = R^-1, the whitened factors W = Y P and
// the "solved" factors Z = Y G^-1 = W P^T:
//     A_u = G + V^T D V,  b_u = V^T c+          V = the n gathered rows of Y,  D = diag(|c| - 1),  c+ = max(c, 0)
//     x_u = A_u^-1 b_u = G^-1 V^T (I + D K)^-1 c+,   K = V G^-1 V^T = W_u W_u^T
//         = Z_u^T E (I + E K E)^-1 E^-1 c+,          E = sqrt(D)
// so a row costs an n x n Gram matrix of whitened rows (mma.sync, fp16 hi/lo split: three m16n8k16 products give
// fp32-faithful K), an n x n LDL^T solve of M = I + E K E (eigenvalues >= 1: always well conditioned) and one
// pass x = sum_i t_i z_i over the gathered rows of Z.  Cost drops from O(n F^2 + F^3) to O(n^2 F + n^3 + n F).
//
// Organisation (round 2): a warp takes a BATCH of 32 / G consecutive work items (the list is sorted by length) and
//   A  forms the systems one row at a time, all 32 lanes on one row (cp.async gathers of W, pipelined across the
//      rows of the batch; tensor-core Gram matrix), leaving M and the right-hand sides in shared memory;
//   B  solves all systems of the batch AT ONCE, G lanes per system, the upper triangle of each M distributed by
//      columns over the G lanes and held in registers: an elimination step costs one shuffle per multiplier for
//      32 / G systems (the round-1 kernel spent a whole warp on one system: ~5x the instructions per row);
//   C  gathers the rows of Z one row at a time and writes x (and its peer replicas) straight from registers.
//
// Not every short item qualifies: a negative weight |c| - 1 < 0 (|c| < 1, or an explicit zero) makes M indefinite,
// chunks of giant rows are not rows, and a G that is not positive definite has no R.  Such items are appended to
// a deferred list that the full-size kernel of cholesky.cu processes right after; results never depend on which
// path took a row beyond fp32 rounding.
#include <cuda_fp16.h>

#include <type_traits>

#include "cholesky_device.cuh"

namespace als {

namespace {

// W is stored scaled by 2^14 (|W_ij| <= 1 because W^T W = I - lambda P^T P, so the scaled entries stay inside
// the fp16 range and the hi / lo halves of everything above 2^-17 of the maximum keep 22 bits): the scale is
// folded into P by whiten_factor_kernel and taken out again, exactly, when M and t are formed.
constexpr float kWScale = 16384.f, kWScaleInv = 1.f / 16384.f;

// ---- P = R^-1 and G^-1 = P P^T in fp64 ----------------------------------------------------------
// One CTA of 32 x 32 threads on the augmented matrix [G | I] (F x 2F doubles in shared memory).  Gaussian
// elimination without pivoting (G is SPD) turns it into [D U | L1^-1] with G = U^T D U, U unit upper triangular,
// L1 = U^T; then R = D^1/2 U and P = R^-1 = (D^-1/2 L1^-1)^T.  One barrier per pivot: step k only reads row k.
// Outputs: Ps = 2^14 P (upper triangular) and Ginv = P P^T, both rounded to fp32 once.
__global__ void __launch_bounds__(1024) whiten_factor_kernel(const float *__restrict__ Greg, int F, float *__restrict__ Ps,
                                                             float *__restrict__ Ginv, int32_t *ok) {
  extern __shared__ __align__(16) unsigned char whiten_smem[];
  double *a = reinterpret_cast<double *>(whiten_smem);  // [F][2F + 1]
  const int ld = 2 * F + 1;
  double *Pd = a + F * ld;                              // [F][F + 1]: P in double
  const int ldp = F + 1;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < F; i += 32)
    for (int j = tx; j < 2 * F; j += 32) a[i * ld + j] = j < F ? (double)Greg[i * F + j] : (j - F == i ? 1.0 : 0.0);
  __syncthreads();
  for (int k = 0; k < F; ++k) {
    const double d = a[k * ld + k];
    // same for every thread: G is not positive definite, not finite, or out of the range the fp32 seed covers
    if (!(d > 1e-30) || !(d < 1e30)) {
      if (threadIdx.x == 0) *ok = 0;
      return;
    }
    double rinv = (double)(1.f / (float)d);  // seed + two Newton steps: full double precision
    rinv = rinv * (2.0 - d * rinv);
    rinv = rinv * (2.0 - d * rinv);
    for (int i = k + 1 + ty; i < F; i += 32) {
      const double m = a[k * ld + i] * rinv;  // G is symmetric: the multiplier of row i is (D U)[k][i] / d_k
      for (int j = tx; j < 2 * F; j += 32)
        if ((j >= i && j < F) || (j >= F && j <= F + k)) a[i * ld + j] -= m * a[k * ld + j];
    }
    __syncthreads();  // row k + 1 (the next pivot row) is complete
  }
  for (int j = ty; j < F; j += 32) {  // row j of L1^-1 scaled by d_j^-1/2 is column j of P
    const double d = a[j * ld + j];
    double s = (double)rsqrtf((float)d);
    s = s * (1.5 - 0.5 * d * s * s);
    s = s * (1.5 - 0.5 * d * s * s);
    for (int i = tx; i < F; i += 32) {
      const double p = i <= j ? a[j * ld + F + i] * s : 0.0;
      Pd[i * ldp + j] = p;
      Ps[i * F + j] = (float)(p * (double)kWScale);
    }
  }
  __syncthreads();
  for (int i = ty; i < F; i += 32)
    for (int j = tx; j < F; j += 32) {
      double acc = 0.0;
      for (int k = (i > j ? i : j); k < F; ++k) acc += Pd[i * ldp + k] * Pd[j * ldp + k];
      Ginv[i * F + j] = (float)acc;
    }
  if (threadIdx.x == 0) *ok = 1;
}

// ---- W = Y P (P upper triangular) and Z = Y G^-1 (full) ------------------------------------------
// 128 rows per CTA pass; thread (ty, tx) owns rows 4 ty .. 4 ty + 3 and, in every 32-column half, columns
// 4 tx .. 4 tx + 3 (so both the P reads and the W writes of a warp are contiguous and conflict free).
template <int NB>
struct WhitenCfg {
  static constexpr int F = 16 * NB, LDY = F + 1, RT = 128;
  static constexpr int NH = (F + 31) / 32;  // 32-column halves
  static constexpr int SMEM_FLOATS = F * F + RT * LDY;
};

template <int NB, bool TRI>
__global__ void __launch_bounds__(256) whiten_rows_kernel(const float *__restrict__ Y, const float *__restrict__ P,
                                                          float *__restrict__ W, int64_t rows) {
  using C = WhitenCfg<NB>;
  constexpr int F = C::F, LDY = C::LDY, RT = C::RT, NH = C::NH;
  extern __shared__ __align__(16) unsigned char whiten_rows_smem[];
  float *Ps = reinterpret_cast<float *>(whiten_rows_smem);
  float *Ys = Ps + F * F;
  const int tid = threadIdx.x, tx = tid & 7, ty = tid >> 3;
  for (int e = tid; e < F * F; e += 256) Ps[e] = P[e];
  for (int64_t r0 = (int64_t)blockIdx.x * RT; r0 < rows; r0 += (int64_t)gridDim.x * RT) {
    __syncthreads();
    for (int e = tid; e < RT * (F / 4); e += 256) {
      const int r = e / (F / 4), c4 = e % (F / 4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r0 + r < rows) v = __ldg(reinterpret_cast<const float4 *>(Y + (r0 + r) * F) + c4);
      float *dst = Ys + r * LDY + 4 * c4;
      dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; dst[3] = v.w;
    }
    __syncthreads();
    float acc[4][NH][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int h = 0; h < NH; ++h) acc[i][h][0] = acc[i][h][1] = acc[i][h][2] = acc[i][h][3] = 0.f;
    // an upper triangular P: row k only reaches the 32-column halves h >= k / 32
#pragma unroll
    for (int kb = 0; kb < NH; ++kb) {
#pragma unroll 4
      for (int k = 32 * kb; k < (32 * kb + 32 < F ? 32 * kb + 32 : F); ++k) {
        float y[4];
        float4 p[NH];
#pragma unroll
        for (int i = 0; i < 4; ++i) y[i] = Ys[(4 * ty + i) * LDY + k];
#pragma unroll
        for (int h = (TRI ? kb : 0); h < NH; ++h) {
          const int c = 32 * h + 4 * tx;
          p[h] = c < F ? *reinterpret_cast<const float4 *>(Ps + k * F + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int h = (TRI ? kb : 0); h < NH; ++h) {
            acc[i][h][0] = fmaf(y[i], p[h].x, acc[i][h][0]);
            acc[i][h][1] = fmaf(y[i], p[h].y, acc[i][h][1]);
            acc[i][h][2] = fmaf(y[i], p[h].z, acc[i][h][2]);
            acc[i][h][3] = fmaf(y[i], p[h].w, acc[i][h][3]);
          }
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int64_t r = r0 + 4 * ty + i;
      if (r < rows) {
#pragma unroll
        for (int h = 0; h < NH; ++h) {
          const int c = 32 * h + 4 * tx;
          if (c < F)
            *reinterpret_cast<float4 *>(W + r * F + c) = make_float4(acc[i][h][0], acc[i][h][1], acc[i][h][2], acc[i][h][3]);
        }
      }
    }
  }
}

// fp32 W rows (the FMA fallback of run_whiten_rows) -> the split format the batch kernel gathers: per 16 factor
// dimensions 8 words of fp16 pairs "hi" followed by 8 words "lo" (hi + lo carries 22 bits; both rounded to nearest)
__device__ __forceinline__ void split_f16x2(float2 x, uint32_t &hi, uint32_t &lo) {
  const __half2 h = __floats2half2_rn(x.x, x.y);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(x.x - hf.x, x.y - hf.y);
  hi = *reinterpret_cast<const uint32_t *>(&h);
  lo = *reinterpret_cast<const uint32_t *>(&l);
}

__global__ void __launch_bounds__(256) w_split_kernel(float *__restrict__ W, int64_t n_blocks16) {
  // one thread per (row, 16-dimension block): reads its 16 floats, writes its 16 words in place
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n_blocks16; e += (int64_t)gridDim.x * blockDim.x) {
    float4 *p = reinterpret_cast<float4 *>(W + e * 16);
    const float4 a = p[0], b = p[1], c = p[2], d = p[3];
    uint32_t hi[8], lo[8];
    split_f16x2(make_float2(a.x, a.y), hi[0], lo[0]);
    split_f16x2(make_float2(a.z, a.w), hi[1], lo[1]);
    split_f16x2(make_float2(b.x, b.y), hi[2], lo[2]);
    split_f16x2(make_float2(b.z, b.w), hi[3], lo[3]);
    split_f16x2(make_float2(c.x, c.y), hi[4], lo[4]);
    split_f16x2(make_float2(c.z, c.w), hi[5], lo[5]);
    split_f16x2(make_float2(d.x, d.y), hi[6], lo[6]);
    split_f16x2(make_float2(d.z, d.w), hi[7], lo[7]);
    uint4 *o = reinterpret_cast<uint4 *>(p);
    o[0] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    o[1] = make_uint4(hi[4], hi[5], hi[6], hi[7]);
    o[2] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    o[3] = make_uint4(lo[4], lo[5], lo[6], lo[7]);
  }
}

template <int NB>
int run_whiten_rows(als_ctx *ctx, const als_factors *Y, cudaStream_t stream) {
  // fp32 FMA tiles (round-to-nearest accumulation): W = Y Ps into ctx->whitened, Z = Y Ginv into ctx->zfactors
  using C = WhitenCfg<NB>;
  const int smem = C::SMEM_FLOATS * (int)sizeof(float);
  const int grid = (int)std::min<int64_t>(ceil_div(std::max<int64_t>(Y->rows, 1), C::RT), (int64_t)ctx->sm_count * 4);
  {
    auto kern = whiten_rows_kernel<NB, true>;
    ALS_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kern<<<grid, 256, smem, stream>>>(Y->d, ctx->Pinv, ctx->whitened, Y->rows);
    ALS_CUDA(cudaGetLastError());
    const int64_t n16 = std::max<int64_t>(Y->rows, 1) * (C::F / 16);
    w_split_kernel<<<(int)std::min<int64_t>(ceil_div(n16, 256), (int64_t)ctx->sm_count * 8), 256, 0, stream>>>(ctx->whitened, n16);
    ALS_CUDA(cudaGetLastError());
    ctx->launches += 2;
  }
  {
    auto kern = whiten_rows_kernel<NB, false>;
    ALS_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kern<<<grid, 256, smem, stream>>>(Y->d, ctx->Ginv, ctx->zfactors, Y->rows);
    ALS_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  return ALS_OK;
}

// ---- the batched short-row solver ----------------------------------------------------------------
constexpr int kBatchWarps = 4;

// lanes per system for a system of NS unknowns: the register footprint of the distributed upper triangle is
// G Q (Q + 1) / 2 with Q = NS / G columns per lane -> 36 / 72 / 84 / 80 / 120 / 96 registers
template <int NS> struct BatchShape;
template <> struct BatchShape<8> { static constexpr int G = 1; };
template <> struct BatchShape<16> { static constexpr int G = 2; };
template <> struct BatchShape<24> { static constexpr int G = 4; };
template <> struct BatchShape<32> { static constexpr int G = 8; };
template <> struct BatchShape<40> { static constexpr int G = 8; };
template <> struct BatchShape<48> { static constexpr int G = 16; };

template <int NB, int NS_>
struct BatchCfg {
  static constexpr int F = 16 * NB;
  static constexpr int NS = NS_;
  static constexpr int G = BatchShape<NS>::G;
  static constexpr int B = 32 / G;           // systems per batch
  static constexpr int Q = NS / G;           // columns per lane
  static constexpr int TOT = G * Q * (Q + 1) / 2;
  static constexpr int NT8 = NS / 8;         // 8-row groups of W_u == 8-column tiles of the Gram matrix
  static constexpr int NM = (NS + 15) / 16;  // 16-row tiles (the last one is half empty when NT8 is odd)
  // upper-triangular tile list: tile (i, j), j >= 2 i
  __host__ __device__ static constexpr int tidx(int i, int j) { return i * NT8 - i * (i - 1) + (j - 2 * i); }
  static constexpr int NTILES = tidx(NM - 1, NT8 - 1) + 1;
  static constexpr int KP = 16;              // factor dimensions staged per phase
  static constexpr int NPH = F / KP;
  static constexpr int LDW = 20;             // words per staged row: 8 hi + 8 lo + 4 (conflict-free fragment reads)
  static constexpr int STAGE = NS * LDW;
  static constexpr int NST = NS <= 40 ? 3 : 2;  // stages of the W_u ring: two phases of gathers in flight where shared memory allows
  static constexpr int TRI = NS * (NS + 1) / 2;
  // the B systems of a batch start G banks apart: phase B reads them conflict free
  static constexpr int SYS = TRI + (((G - TRI % 32) % 32) + 32) % 32;
  // packed upper triangle, row major: element (i, c), c >= i, lives at roff(i) + c
  __host__ __device__ static constexpr int roff(int i) { return i * NS - i * (i + 1) / 2; }
  __host__ __device__ static constexpr int off(int q) { return G * q * (q + 1) / 2; }  // registers of column block q
  static constexpr int META = B * NS;
  static constexpr int WARP_FLOATS = NST * STAGE + B * SYS + 3 * META + 32;
  static constexpr int SMEM_FLOATS = kBatchWarps * WARP_FLOATS;
  static_assert((B * NS) % 32 == 0, "prologue loop must be warp uniform");
  static_assert(WARP_FLOATS % 4 == 0 && STAGE % 2 == 0 && (B * SYS) % 4 == 0 && META % 4 == 0, "alignment");
};

// Phase B: the B systems of the batch, G lanes each.  Lane l of a group owns the columns c = l + G q of
// U' = D U (the upper triangle after elimination), rows 0 .. c, in a[off(q) + i]; entries below the diagonal inside
// the last row block of a column block are storage only (never read as data).  Plain Gaussian elimination on the
// symmetric matrix (LDL^T: no square roots on the critical path), right-hand side carried along, then a
// row-oriented back substitution with a G-lane reduction per unknown.
// compile-time loop: every register index below must be a constant (the loop nests are too large for
// "#pragma unroll" to be honoured, and a dynamically indexed array would live in local memory)
template <int I, int N, class Fn>
__device__ __forceinline__ void static_for(Fn &&f) {
  if constexpr (I < N) {
    f(std::integral_constant<int, I>{});
    static_for<I + 1, N>(f);
  }
}

template <class C>
__device__ __forceinline__ void batch_solve(const float *__restrict__ sy, float (&z)[C::Q], int l, float (&s)[C::Q]) {
  constexpr int NS = C::NS, G = C::G, Q = C::Q;
  constexpr unsigned kFull = 0xffffffffu;
  float a[C::TOT];
  float rinvs[Q];
  static_for<0, Q>([&](auto qc) {
    constexpr int q = decltype(qc)::value;
    const int c = l + G * q;
    static_for<0, G *(q + 1)>([&](auto ic) {
      constexpr int i = decltype(ic)::value;
      a[C::off(q) + i] = (i <= c) ? sy[C::roff(i) + c] : 0.f;
    });
    rinvs[q] = 0.f;
    s[q] = 0.f;
  });
  static_for<0, NS>([&](auto rcn) {
    constexpr int r = decltype(rcn)::value;
    constexpr int qr = r / G, lr = r % G;
    const float d = a[C::off(qr) + r];  // the pivot on lane lr
    const float rc = rcp_approx(d);  // within an ulp or two of 1 / d: as good as the division LAPACK would do here
    const float rinv = G > 1 ? __shfl_sync(kFull, rc, lr, G) : rc;
    rinvs[qr] = (l == lr) ? rinv : rinvs[qr];
    const float zr = G > 1 ? __shfl_sync(kFull, z[qr], lr, G) : z[qr];
    // multipliers of this lane's columns: u[q] = A[r][c] / d_r
    float u[Q];
    static_for<qr, Q>([&](auto qc) {
      constexpr int q = decltype(qc)::value;
      u[q] = a[C::off(q) + r] * rinv;
      const float nz = fmaf(-u[q], zr, z[q]);
      z[q] = (q > qr || l > lr) ? nz : z[q];  // rows after the pivot only
    });
    static_for<r + 1, NS>([&](auto r2c) {
      constexpr int r2 = decltype(r2c)::value;
      constexpr int q2 = r2 / G, l2 = r2 % G;
      const float m = G > 1 ? __shfl_sync(kFull, u[q2], l2, G) : u[q2];
      static_for<q2, Q>([&](auto qc) {
        constexpr int q = decltype(qc)::value;
        a[C::off(q) + r2] = fmaf(-m, a[C::off(q) + r], a[C::off(q) + r2]);
      });
    });
  });
  static_for<0, NS>([&](auto rcn) {
    constexpr int r = NS - 1 - decltype(rcn)::value;
    constexpr int qr = r / G, lr = r % G;
    float part = 0.f;
    static_for<qr, Q>([&](auto qc) {
      constexpr int q = decltype(qc)::value;
      const float term = a[C::off(q) + r] * s[q];
      part += (q > qr || l > lr) ? term : 0.f;  // columns after r only
    });
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) part += __shfl_xor_sync(kFull, part, o, G);
    const float sr = (z[qr] - part) * rinvs[qr];
    s[qr] = (l == lr) ? sr : s[qr];
  });
}

template <int NB, int NS>
__global__ void __launch_bounds__(32 * kBatchWarps, 3)
short_batch_kernel(const int32_t *__restrict__ indices, const float *__restrict__ data, const uint32_t *__restrict__ W,
                   const float *__restrict__ Z, float *__restrict__ X, int64_t row_offset,
                   const WorkItem *__restrict__ work, int n_work, int32_t *counter, WorkItem *deferred,
                   int32_t *n_deferred, const int32_t *whiten_ok, float *const *peers, int n_peers) {
  using C = BatchCfg<NB, NS>;
  constexpr int F = C::F, G = C::G, B = C::B, Q = C::Q, NT8 = C::NT8, NM = C::NM, LDW = C::LDW, NPH = C::NPH;
  constexpr unsigned kFull = 0xffffffffu;
  extern __shared__ __align__(16) unsigned char short_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  float *wsm = reinterpret_cast<float *>(short_smem) + warp * C::WARP_FLOATS;
  uint32_t *stage = reinterpret_cast<uint32_t *>(wsm);   // NST stages of W_u: per row 8 fp16-pair words hi, 8 lo
  float *sys = wsm + C::NST * C::STAGE;                   // B packed upper triangles
  int *idxs = reinterpret_cast<int *>(sys + B * C::SYS);  // [B][NS] column indices (padding repeats a real one)
  float *es = reinterpret_cast<float *>(idxs + C::META);  // [B][NS] sqrt(|c| - 1) / 2^14, 0 on padding
  float *zs = es + C::META;                               // [B][NS] E^-1 c+, then t = E s
  unsigned *badbits = reinterpret_cast<unsigned *>(zs + C::META);
  const bool usable = *whiten_ok != 0;
  const int l = lane % G, sb = lane / G;

  for (;;) {
    int v0 = 0;
    if (lane == 0) v0 = atomicAdd(counter, B);
    v0 = __shfl_sync(kFull, v0, 0);
    if (v0 >= n_work) break;
    const int nb = min(B, n_work - v0);
    // lane b keeps item b of the batch
    WorkItem mine{0, 0, 0, -3};
    if (lane < nb) {
      const int4 raw = __ldg(reinterpret_cast<const int4 *>(work) + v0 + lane);
      mine = WorkItem{raw.x, raw.y, raw.z, raw.w};
    }
    const int my_n = mine.k1 - mine.k0;
    bool my_defer = lane < nb && (mine.slot != -1 || !usable || my_n > NS);
    const int my_len = (lane < nb && !my_defer) ? my_n : 0;  // nonzeros this path will use
    __syncwarp();  // the previous batch is done with the metadata
    if (lane == 0) *badbits = 0u;
    __syncwarp();
    // ---- prologue: the nonzeros of the whole batch -> shared memory (_als.pyx:109-124 semantics)
#pragma unroll
    for (int e = lane; e < C::META; e += 32) {
      const int b = e / NS, i = e % NS;
      const int k0 = __shfl_sync(kFull, mine.k0, b);
      const int len = __shfl_sync(kFull, my_len, b);
      const bool valid = i < len;
      int id = 0;
      float c = 1.f;
      if (valid) {
        id = __ldg(indices + k0 + i);
        c = __ldg(data + k0 + i);
      } else if (len > 0) {
        id = __ldg(indices + k0);  // padding repeats a real row of W; its weight is 0
      }
      const float w = fabsf(c) - 1.f;  // _als.pyx:115-118
      if (valid && !(w >= 0.f)) atomicOr(badbits, 1u << b);  // negative weight or NaN: not for this path
      const float ew = valid ? sqrtf(fmaxf(w, 1e-10f)) : 0.f;
      idxs[e] = id;
      es[e] = ew * kWScaleInv;
      zs[e] = (valid && c > 0.f) ? c / ew : 0.f;  // E^-1 c+   (_als.pyx:119-121: only c > 0 feeds b)
    }
    __syncwarp();
    const unsigned bad = *badbits;
    if (bad) {  // such rows go to the full-size kernel; here they become the identity system
#pragma unroll
      for (int e = lane; e < C::META; e += 32)
        if ((bad >> (e / NS)) & 1u) {
          es[e] = 0.f;
          zs[e] = 0.f;
        }
      if (lane < nb && ((bad >> lane) & 1u)) my_defer = true;
      __syncwarp();
    }

    // ---- phase A: K = W_u W_u^T for every row of the batch, 16 factor dimensions per phase; the gathers of
    //      phase p + 1 (possibly the next row's first) are in flight while phase p is multiplied.  W arrives
    //      already split (dense.cu): per row and phase 8 words of fp16 pairs "hi" and 8 words "lo".
    auto issue = [&](int p) {
      const int b = p / NPH, ph = p % NPH;
      uint32_t *st = stage + (p % C::NST) * C::STAGE;
      const int *ix = idxs + b * NS;
#pragma unroll
      for (int q = 0; q < NT8; ++q) {
        const int ri = ix[8 * q + g];
        cp_async16(reinterpret_cast<float *>(st + (8 * q + g) * LDW + 4 * t),
                   reinterpret_cast<const float *>(W + (int64_t)ri * F + C::KP * ph + 4 * t));
      }
      cp_async_commit();
    };
    float acc[C::NTILES][4];
#pragma unroll
    for (int e = 0; e < C::NTILES; ++e) acc[e][0] = acc[e][1] = acc[e][2] = acc[e][3] = 0.f;
    const int TP = nb * NPH;
    // the ring holds the phase being multiplied and NST - 1 phases of gathers in flight (empty groups past the end keep
    // the cp.async group count uniform)
#pragma unroll
    for (int q = 0; q < C::NST - 1; ++q) {
      if (q < TP) issue(q);
      else cp_async_commit();
    }
    for (int p = 0; p < TP; ++p) {
      if (p + C::NST - 1 < TP) issue(p + C::NST - 1);
      else cp_async_commit();
      cp_async_wait<C::NST - 1>();
      __syncwarp();
      const uint32_t *sg = stage + (p % C::NST) * C::STAGE;
      {
        uint32_t h0[NT8], h1[NT8], l0[NT8], l1[NT8];
#pragma unroll
        for (int c = 0; c < NT8; ++c) {
          const uint32_t *rp = sg + (8 * c + g) * LDW + t;
          h0[c] = rp[0];   // dims 2t, 2t+1 (hi)
          h1[c] = rp[4];   // dims 2t+8, 2t+9 (hi)
          l0[c] = rp[8];   // the same, lo
          l1[c] = rp[12];
        }
#pragma unroll
        for (int term = 0; term < 3; ++term) {  // lo * hi, hi * lo, hi * hi: the chain through a tile is a sweep apart
#pragma unroll
          for (int i = 0; i < NM; ++i) {
            constexpr uint32_t kZero = 0u;
            const bool second = 2 * i + 1 < NT8;  // compile time after unrolling: rows 16 i + 8 .. exist
            const uint32_t a0 = term == 0 ? l0[2 * i] : h0[2 * i];
            const uint32_t a1 = second ? (term == 0 ? l0[2 * i + (second ? 1 : 0)] : h0[2 * i + (second ? 1 : 0)]) : kZero;
            const uint32_t a2 = term == 0 ? l1[2 * i] : h1[2 * i];
            const uint32_t a3 = second ? (term == 0 ? l1[2 * i + (second ? 1 : 0)] : h1[2 * i + (second ? 1 : 0)]) : kZero;
#pragma unroll
            for (int j = 2 * i; j < NT8; ++j) {
              float(&d)[4] = acc[C::tidx(i, j)];
              if (term == 1) mma_f16(d, a0, a1, a2, a3, l0[j], l1[j]);
              else mma_f16(d, a0, a1, a2, a3, h0[j], h1[j]);
            }
          }
        }
      }
      if (p % NPH == NPH - 1) {
        // ---- M = I + E K E (identity on the padding: e = 0 there) -> the packed upper triangle of system b
        const int b = p / NPH;
        float *sy = sys + b * C::SYS;
        const float *eb = es + b * NS;
#pragma unroll
        for (int i = 0; i < NM; ++i) {
          const bool second = 2 * i + 1 < NT8;
          const int r0 = 16 * i + g, r1 = r0 + 8;
          const float er0 = eb[r0], er1 = second ? eb[second ? r1 : r0] : 0.f;
          const int ro0 = r0 * NS - ((r0 * (r0 + 1)) >> 1), ro1 = r1 * NS - ((r1 * (r1 + 1)) >> 1);
#pragma unroll
          for (int j = 2 * i; j < NT8; ++j) {
            const int c0 = 8 * j + 2 * t, c1 = c0 + 1;
            const float2 ec = *reinterpret_cast<const float2 *>(eb + c0);
            float(&d)[4] = acc[C::tidx(i, j)];
            if (c0 >= r0) sy[ro0 + c0] = fmaf(er0 * ec.x, d[0], r0 == c0 ? 1.f : 0.f);
            if (c1 >= r0) sy[ro0 + c1] = fmaf(er0 * ec.y, d[1], r0 == c1 ? 1.f : 0.f);
            if (second && c0 >= r1) sy[ro1 + c0] = fmaf(er1 * ec.x, d[2], r1 == c0 ? 1.f : 0.f);
            if (second && c1 >= r1) sy[ro1 + c1] = fmaf(er1 * ec.y, d[3], r1 == c1 ? 1.f : 0.f);
            d[0] = d[1] = d[2] = d[3] = 0.f;
          }
        }
      }
      __syncwarp();  // the stage is free for phase p + NST
    }

    // ---- phase B: all systems of the batch at once, G lanes per system
    bool fin = true;
    {
      float z[Q], e[Q], s[Q];
#pragma unroll
      for (int q = 0; q < Q; ++q) {
        z[q] = zs[sb * NS + l + G * q];
        e[q] = es[sb * NS + l + G * q];
      }
      batch_solve<C>(sys + sb * C::SYS, z, l, s);
#pragma unroll
      for (int q = 0; q < Q; ++q) {
        const float tq = e[q] * s[q] * kWScale;  // t = E s
        fin = fin && (fabsf(tq) <= 3.0e38f);      // false for inf and NaN
        zs[sb * NS + l + G * q] = tq;
      }
    }
    const unsigned notfin = __ballot_sync(kFull, !fin);
    if (lane < nb && ((notfin >> (lane * G)) & ((1u << G) - 1u)))
      my_defer = true;  // cannot happen for finite inputs (M >= I); let the full-size path decide
    if (lane < nb && my_defer) deferred[atomicAdd(n_deferred, 1)] = mine;
    __syncwarp();

    // ---- phase C: x = Z_u^T t, lane owns columns 2 lane, 2 lane + 1
    const bool owns = 2 * lane < F;
    auto store_x = [&](int row, float x0, float x1) {
      const int64_t xoff = (row_offset + row) * F;
      if (owns) {
        *reinterpret_cast<float2 *>(X + xoff + 2 * lane) = make_float2(x0, x1);
        for (int pi = 0; pi < n_peers; ++pi) *reinterpret_cast<float2 *>(peers[pi] + xoff + 2 * lane) = make_float2(x0, x1);
      }
    };
    if constexpr (NS <= 40) {
      // The rows of Z of system b + 1 are gathered (cp.async) into the shared memory that the W_u ring and the solved
      // systems no longer need while system b is reduced: one exposed gather latency per BATCH instead of per row.
      constexpr int CH = F / 4, RPI = 32 / CH;  // 16-byte chunks per row of Z, rows per warp-wide copy
      static_assert(C::NST * C::STAGE + B * C::SYS >= 2 * NS * F, "phase C double buffer does not fit");
      float *zbuf = wsm;
      auto zissue = [&](int b, int buf) {
        const int n = __shfl_sync(kFull, my_n, b);
        const bool skip = __shfl_sync(kFull, (int)my_defer, b) != 0;
        if (!skip) {
          const int *ix = idxs + b * NS;
          const int r = lane / CH, ch = lane % CH;
          for (int i = 0; i < n; i += RPI)  // the padding up to the class size repeats a valid index
            if (r < RPI && i + r < NS)
              cp_async16(zbuf + (buf * NS + i + r) * F + 4 * ch, Z + (int64_t)ix[i + r] * F + 4 * ch);
        }
        cp_async_commit();
      };
      zissue(0, 0);
      for (int b = 0; b < nb; ++b) {
        if (b + 1 < nb) zissue(b + 1, (b + 1) & 1);
        else cp_async_commit();
        cp_async_wait<1>();
        __syncwarp();
        if (!__shfl_sync(kFull, (int)my_defer, b)) {
          const int row = __shfl_sync(kFull, mine.row, b);
          const int n = __shfl_sync(kFull, my_n, b);
          const float *zb = zbuf + (b & 1) * NS * F + 2 * lane;
          const float *tv = zs + b * NS;
          float x0 = 0.f, x1 = 0.f;  // no observations: the reference zeroes the row (_als.pyx:98-100)
          for (int i = 0; i < n; i += 4) {  // t = 0 on the padding (and its rows were gathered whenever i + r < NS)
            const float4 t4 = *reinterpret_cast<const float4 *>(tv + i);
            const float tt[4] = {t4.x, t4.y, t4.z, t4.w};
#pragma unroll
            for (int u = 0; u < 4; ++u)
              if (i + u < n && owns) {
                const float2 z2 = *reinterpret_cast<const float2 *>(zb + (i + u) * F);
                x0 = fmaf(tt[u], z2.x, x0);
                x1 = fmaf(tt[u], z2.y, x1);
              }
          }
          store_x(row, x0, x1);
        }
        __syncwarp();  // the buffer is free for system b + 2
      }
    } else {
      for (int b = 0; b < nb; ++b) {
        if (__shfl_sync(kFull, (int)my_defer, b)) continue;
        const int row = __shfl_sync(kFull, mine.row, b);
        const int n = __shfl_sync(kFull, my_n, b);
        float x0 = 0.f, x1 = 0.f;
        const int *ix = idxs + b * NS;
        const float *tv = zs + b * NS;
        // all NS slots are gathered, 16 loads in flight at a time: the padding has t = 0 and repeats a valid index
#pragma unroll
        for (int i0 = 0; i0 < NS; i0 += 16) {
          constexpr int kMaxChunk = 16;
          const int cn = NS - i0 < kMaxChunk ? NS - i0 : kMaxChunk;  // 16 or 8 (compile time after unrolling)
          if (i0 >= n) break;                                        // warp uniform
          int id[kMaxChunk];
          float tt[kMaxChunk];
#pragma unroll
          for (int u = 0; u < kMaxChunk; u += 4)
            if (u < cn) {
              const int4 iv = *reinterpret_cast<const int4 *>(ix + i0 + u);
              const float4 tv4 = *reinterpret_cast<const float4 *>(tv + i0 + u);
              id[u] = iv.x; id[u + 1] = iv.y; id[u + 2] = iv.z; id[u + 3] = iv.w;
              tt[u] = tv4.x; tt[u + 1] = tv4.y; tt[u + 2] = tv4.z; tt[u + 3] = tv4.w;
            }
          float2 zz[kMaxChunk];
#pragma unroll
          for (int u = 0; u < kMaxChunk; ++u)
            if (u < cn) zz[u] = owns ? __ldcg(reinterpret_cast<const float2 *>(Z + (int64_t)id[u] * F) + lane) : make_float2(0.f, 0.f);
#pragma unroll
          for (int u = 0; u < kMaxChunk; ++u)
            if (u < cn) {
              x0 = fmaf(tt[u], zz[u].x, x0);
              x1 = fmaf(tt[u], zz[u].y, x1);
            }
        }
        store_x(row, x0, x1);
      }
    }
  }
}

template <int NB, int NS>
int run_short(als_ctx *ctx, const als_csr *Cm, als_factors *X, int64_t begin, int64_t end, int slot, cudaStream_t stream) {
  using C = BatchCfg<NB, NS>;
  const int64_t count = end - begin;
  if (count <= 0) return ALS_OK;
  const int smem = C::SMEM_FLOATS * (int)sizeof(float);
  auto kern = short_batch_kernel<NB, NS>;
  ALS_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int ctas_per_sm = 0;
  ALS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, kern, 32 * kBatchWarps, smem));
  if (ctas_per_sm < 1) {
    set_error("short rows: kernel does not fit on an SM (smem %d bytes)", smem);
    return ALS_E_CUDA;
  }
  const int grid = (int)std::min<int64_t>(ceil_div(count, (int64_t)kBatchWarps * C::B), (int64_t)ctx->sm_count * ctas_per_sm);
  kern<<<grid, 32 * kBatchWarps, smem, stream>>>(Cm->indices, Cm->data, reinterpret_cast<const uint32_t *>(ctx->whitened),
                                                  ctx->zfactors, X->d, Cm->row_offset, Cm->work + begin, (int)count,
                                                  ctx->counters + kCtrShort + slot, ctx->deferred,
                                                  ctx->counters + kCtrDeferredCount, ctx->counters + kCtrWhitenOk,
                                                  X->peers_dev, X->n_peers);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  return ALS_OK;
}

// items [begin, n_work) split into the size classes (40, 48], (32, 40], ... [0, 8] by the schedule's suffix offsets
// (kShortThresholds); a system of NS unknowns needs NS < F, so a narrower factor matrix stops earlier
template <int NB>
int run_short_classes(als_ctx *ctx, const als_csr *Cm, als_factors *X, int64_t begin, int max_len, cudaStream_t stream) {
  int64_t lb[kNumShortThresholds];
  for (int c = 0; c < kNumShortThresholds; ++c) lb[c] = std::max(begin, Cm->le_begin[c]);
  if (begin < lb[0]) {
    set_error("short rows: items longer than 48 nonzeros");
    return ALS_E_INVALID;
  }
  (void)max_len;
  // One stream per size class (forked from `stream`, joined back into it): the classes are persistent kernels of very
  // different lengths, and on one stream each would wait for the previous one's tail -- a cost that does not shrink
  // with the row shard of a multi-GPU run.  Longest class first.
  const bool fan = ctx->class_stream[0] != nullptr && !ctx->knobs.short_serial;
  if (fan) ALS_CUDA(cudaEventRecord(ctx->class_fork, stream));
  int rc = ALS_OK;
  int used = 0;
  auto on = [&](int slot) -> cudaStream_t {
    if (!fan || slot == 0) return stream;
    cudaStreamWaitEvent(ctx->class_stream[slot - 1], ctx->class_fork, 0);
    used |= 1 << slot;
    return ctx->class_stream[slot - 1];
  };
  if constexpr (NB >= 4) {
    if (lb[1] > lb[0] && (rc = run_short<NB, 48>(ctx, Cm, X, lb[0], lb[1], 0, on(0))) != ALS_OK) return rc;
    if (lb[2] > lb[1] && (rc = run_short<NB, 40>(ctx, Cm, X, lb[1], lb[2], 1, on(1))) != ALS_OK) return rc;
  }
  if constexpr (NB >= 3) {
    if (lb[3] > lb[2] && (rc = run_short<NB, 32>(ctx, Cm, X, lb[2], lb[3], 2, on(2))) != ALS_OK) return rc;
    if (lb[4] > lb[3] && (rc = run_short<NB, 24>(ctx, Cm, X, lb[3], lb[4], 3, on(3))) != ALS_OK) return rc;
  }
  if (lb[5] > lb[4] && (rc = run_short<NB, 16>(ctx, Cm, X, lb[4], lb[5], 4, on(4))) != ALS_OK) return rc;
  if (Cm->n_work > lb[5] && (rc = run_short<NB, 8>(ctx, Cm, X, lb[5], Cm->n_work, 5, on(5))) != ALS_OK) return rc;
  for (int slot = 1; slot < 6; ++slot)
    if (used & (1 << slot)) {
      ALS_CUDA(cudaEventRecord(ctx->class_join[slot - 1], ctx->class_stream[slot - 1]));
      ALS_CUDA(cudaStreamWaitEvent(stream, ctx->class_join[slot - 1], 0));
    }
  return ALS_OK;
}

}  // namespace

int short_rows_prepare(als_ctx *ctx, const als_factors *Y, cudaStream_t stream) {
  const int F = Y->ld;
  if (F > 64) {
    set_error("short rows: factors beyond 64 are not supported");
    return ALS_E_UNSUPPORTED;
  }
  int rc = ensure_device_buffer(ctx, (void **)&ctx->whitened, &ctx->whitened_bytes,
                                std::max<int64_t>(Y->rows, 1) * F * (int64_t)sizeof(float));
  if (rc != ALS_OK) return rc;
  rc = ensure_device_buffer(ctx, (void **)&ctx->zfactors, &ctx->zfactors_bytes,
                            std::max<int64_t>(Y->rows, 1) * F * (int64_t)sizeof(float));
  if (rc != ALS_OK) return rc;
  const int smem = (F * (2 * F + 1) + F * (F + 1)) * (int)sizeof(double);
  ALS_CUDA(cudaFuncSetAttribute(whiten_factor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  whiten_factor_kernel<<<1, 1024, smem, stream>>>(ctx->Greg, F, ctx->Pinv, ctx->Ginv, ctx->counters + kCtrWhitenOk);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  // 64 padded factors: one pass on the wgmma tensor cores (dense.cu); the whiten_fma knob keeps the fp32 FMA tiles
  if (F == 64 && Y->rows >= 128 && !ctx->knobs.whiten_fma) return launch_dense_whiten(ctx, Y, stream);  // (a TMA box is 128 rows)
  switch (F / 16) {
    case 2: return run_whiten_rows<2>(ctx, Y, stream);
    case 3: return run_whiten_rows<3>(ctx, Y, stream);
    case 4: return run_whiten_rows<4>(ctx, Y, stream);
    default:
      set_error("short rows: padded factors %d not supported", F);
      return ALS_E_UNSUPPORTED;
  }
}

int short_rows_launch(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y, int64_t begin, int max_len,
                      cudaStream_t stream) {
  const int64_t count = C->n_work - begin;
  if (count <= 0) return ALS_OK;
  int rc = ensure_device_buffer(ctx, (void **)&ctx->deferred, &ctx->deferred_cap, count * (int64_t)sizeof(WorkItem));
  if (rc != ALS_OK) return rc;
  switch (Y->ld / 16) {
    case 2: return run_short_classes<2>(ctx, C, X, begin, max_len, stream);
    case 3: return run_short_classes<3>(ctx, C, X, begin, max_len, stream);
    case 4: return run_short_classes<4>(ctx, C, X, begin, max_len, stream);
    default:
      set_error("short rows: padded factors %d not supported", Y->ld);
      return ALS_E_UNSUPPORTED;
  }
}

}  // namespace als
