// R1 for padded factors 256 ... 1024 (reference: _least_squares, implicit/cpu/_als.pyx:76-142).
//
// Past 128 factors the F x (F + 1) system of a row no longer fits in shared memory (257 KB at F = 256), so it lives
// in global memory: every resident CTA owns a workspace of 64 x 64 tiles holding the upper triangle of A, and the
// factorisation is blocked by 64-column panels.  Only fe = roundup(f, 64) columns are factored (Greg is the
// identity on [f, ld) and Y is zero there, so those unknowns are exactly zero); columns [fe, ld) of x are stored as
// zeros.
//
// One 3xTF32 mma.sync tile routine, C(64 x 64) += sum_k w_k P[k]^T Q[k], serves both large steps:
//   * normal equations: P = Y slice of tile row I, Q = Y slice of tile column J, w = |c| - 1 (its sign included);
//   * trailing update:  A_IJ -= U_KI^T U_KJ with P = U_KI, Q = U_KJ, w = -1.
// The diagonal block is eliminated in shared memory (as cholesky_wide.cu does for the whole matrix), with the forward
// solve of b riding along; the panel row U_KK^T U_KJ = A_KJ and the blocked back substitution are triangular solves
// with U_KK in shared memory.
#include <limits.h>

#include <algorithm>

#include "cholesky_device.cuh"

namespace als {
namespace {

constexpr int kXwThreads = 256;                 // 8 warps: each owns a 16 x 32 part of the 64 x 64 output tile
constexpr int kXwKs = 32;                       // nonzeros staged per step of the normal equations
constexpr int kXwLdp = 72;                      // staged-tile row stride: conflict-free fragment reads
constexpr int kXwTileFloats = 64 * 64;
constexpr int kXwLda = 129;                     // diagonal block: [U_KK | b], odd stride
constexpr int kXwStageFloats = 2 * kXwKs * kXwLdp + 2 * kXwKs;  // P slice, Q slice, w[kXwKs], c+[kXwKs]
constexpr int kXwAdFloats = 64 * kXwLda;
constexpr int kXwOpFloats = 64 * kXwLdp;
// shared memory: b / x [1024] | r [64] | w = -1 [64] | flag | union { 2 stages ; Ad, P, Q }
constexpr int kXwUnionFloats = std::max(2 * kXwStageFloats, kXwAdFloats + 2 * kXwOpFloats);
constexpr int kXwSmemFloats = 1024 + 64 + 64 + 4 + kXwUnionFloats;

__host__ __device__ constexpr int xw_ntiles(int nt) { return nt * (nt + 1) / 2; }
// tile (I, J), J >= I, of the packed upper triangle
__device__ __forceinline__ int xw_tidx(int nt, int I, int J) { return I * nt - I * (I - 1) / 2 + (J - I); }
// a workspace (or giant-row slot): the packed tiles, then b [fe]
__host__ __device__ constexpr int64_t xw_ws_floats(int nt) { return (int64_t)xw_ntiles(nt) * kXwTileFloats + 64 * nt; }

// hi + lo = x with both parts rounded to nearest TF32: the products hi * lo and lo * hi then carry errors of 2^-24 |x|,
// the rounding of an fp32 product (split_tf32 hands lo over raw, and the tensor core truncates it to 2^-23 |x|)
__device__ __forceinline__ void split_tf32_rn(float x, uint32_t &hi, uint32_t &lo) {
  hi = rn_tf32(x);
  lo = rn_tf32(x - __uint_as_float(hi));
}

// acc += sum_{k < 8 ksteps} w[k] P[k][m] Q[k][n] on this warp's rows 16 (warp >> 1) .. +16 and columns
// 32 (warp & 1) .. +32 of a 64 x 64 tile.  P and Q are k-major in shared memory (stride kXwLdp).  3xTF32 with both
// parts rounded to nearest, the lo * hi and hi * lo terms first.  Each k-step's three products go to a fresh accumulator
// that is added to acc in fp32: the tensor core's own accumulation (not round-to-nearest) then never runs over more
// than 8 nonzeros or 8 rows of a panel, however long the row or wide the factorisation.  acc[j] is the m16n8 fragment
// of columns n0 + 8 j.
__device__ __forceinline__ void tile_mma(float (&acc)[4][4], const float *P, const float *Q, const float *w, int ksteps,
                                         int warp, int lane) {
  const int g = lane >> 2, t = lane & 3;
  const int m0 = 16 * (warp >> 1), n0 = 32 * (warp & 1);
#pragma unroll 2
  for (int ks = 0; ks < ksteps; ++ks) {
    const int k = 8 * ks;
    float part[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) part[j][0] = part[j][1] = part[j][2] = part[j][3] = 0.f;
    const float w0 = w[k + t], w1 = w[k + t + 4];
    const float *p0 = P + (k + t) * kXwLdp + m0 + g, *p1 = P + (k + t + 4) * kXwLdp + m0 + g;
    uint32_t ah[4], al[4];
    split_tf32_rn(w0 * p0[0], ah[0], al[0]);
    split_tf32_rn(w0 * p0[8], ah[1], al[1]);
    split_tf32_rn(w1 * p1[0], ah[2], al[2]);
    split_tf32_rn(w1 * p1[8], ah[3], al[3]);
    const float *q0 = Q + (k + t) * kXwLdp + n0 + g, *q1 = Q + (k + t + 4) * kXwLdp + n0 + g;
    uint32_t bh[4][2], bl[4][2];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      split_tf32_rn(q0[8 * j], bh[j][0], bl[j][0]);
      split_tf32_rn(q1[8 * j], bh[j][1], bl[j][1]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) mma_tf32(part[j], al[0], al[1], al[2], al[3], bh[j][0], bh[j][1]);  // lo * hi
#pragma unroll
    for (int j = 0; j < 4; ++j) mma_tf32(part[j], ah[0], ah[1], ah[2], ah[3], bl[j][0], bl[j][1]);  // hi * lo
#pragma unroll
    for (int j = 0; j < 4; ++j) mma_tf32(part[j], ah[0], ah[1], ah[2], ah[3], bh[j][0], bh[j][1]);  // hi * hi
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[j][e] += part[j][e];
  }
}

// the accumulator fragments <-> a row-major 64 x 64 tile with row stride ldt (global or shared memory)
__device__ __forceinline__ void acc_load(float (&acc)[4][4], const float *tile, int ldt, int warp, int lane) {
  const int g = lane >> 2, t = lane & 3, m0 = 16 * (warp >> 1), n0 = 32 * (warp & 1);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 lo = *reinterpret_cast<const float2 *>(tile + (m0 + g) * ldt + n0 + 8 * j + 2 * t);
    const float2 hi = *reinterpret_cast<const float2 *>(tile + (m0 + 8 + g) * ldt + n0 + 8 * j + 2 * t);
    acc[j][0] = lo.x, acc[j][1] = lo.y, acc[j][2] = hi.x, acc[j][3] = hi.y;
  }
}
__device__ __forceinline__ void acc_store(const float (&acc)[4][4], float *tile, int ldt, int warp, int lane) {
  const int g = lane >> 2, t = lane & 3, m0 = 16 * (warp >> 1), n0 = 32 * (warp & 1);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    *reinterpret_cast<float2 *>(tile + (m0 + g) * ldt + n0 + 8 * j + 2 * t) = make_float2(acc[j][0], acc[j][1]);
    *reinterpret_cast<float2 *>(tile + (m0 + 8 + g) * ldt + n0 + 8 * j + 2 * t) = make_float2(acc[j][2], acc[j][3]);
  }
}
__device__ __forceinline__ void acc_zero(float (&acc)[4][4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
}

// a 64 x 64 tile (row-major, contiguous) -> shared memory (stride kXwLdp), one cp.async group
__device__ __forceinline__ void tile_fetch(float *dst, const float *src, int tid) {
#pragma unroll
  for (int q = 0; q < kXwTileFloats / 4 / kXwThreads; ++q) {
    const int e = q * kXwThreads + tid, r = e >> 4, c4 = e & 15;
    cp_async16(dst + r * kXwLdp + 4 * c4, src + r * 64 + 4 * c4);
  }
  cp_async_commit();
}

// stage the Y slices (tile row I, and tile column J when J != I) of nonzeros [k, k + kXwKs) with their weights
__device__ __forceinline__ void stage_fetch(float *st, const int32_t *__restrict__ indices, const float *__restrict__ data,
                                            const float *__restrict__ Y, int ld, int k, int kend, int I, int J, int tid) {
  float *P = st, *Q = st + kXwKs * kXwLdp, *ws = st + 2 * kXwKs * kXwLdp, *cs = ws + kXwKs;
  const int first = __ldg(indices + k);  // rows past the end gather a real row with weight 0
  const int nsl = (J == I) ? 1 : 2;
  for (int e = tid; e < nsl * kXwKs * 16; e += kXwThreads) {
    const int sl = e / (kXwKs * 16), r = (e / 16) % kXwKs, c4 = e & 15;
    const int idx = k + r < kend ? __ldg(indices + k + r) : first;
    const int col = 64 * (sl ? J : I) + 4 * c4;
    cp_async16((sl ? Q : P) + r * kXwLdp + 4 * c4, Y + (int64_t)idx * ld + col);
  }
  cp_async_commit();
  if (tid < kXwKs) {
    const bool valid = k + tid < kend;
    const float c = valid ? __ldg(data + k + tid) : 0.f;
    ws[tid] = valid ? fabsf(c) - 1.f : 0.f;  // _als.pyx:115-124: A += (|c| - 1) y y^T, b += c y for c > 0
    cs[tid] = c > 0.f ? c : 0.f;
  }
}

__global__ void __launch_bounds__(kXwThreads)
cholesky_xwide_kernel(const int32_t *__restrict__ indices, const float *__restrict__ data, const float *__restrict__ Y,
                      float *__restrict__ X, int ld, int nt, int64_t row_offset, const float *__restrict__ Greg,
                      const WorkItem *__restrict__ work, int n_work, float *slots, float *workspaces,
                      long long *bad_row, int pass, float *const *peers, int n_peers) {
  extern __shared__ __align__(16) float smem[];
  float *bs = smem;            // [1024] b, then z, then x
  float *rs = bs + 1024;       // [64] back-substitution residual
  float *wneg = rs + 64;       // [64] -1
  int *flag = reinterpret_cast<int *>(wneg + 64);
  float *un = wneg + 64 + 4;
  float *Ad = un;                        // factorisation: [64][kXwLda]
  float *Ps = Ad + kXwAdFloats;          // [64][kXwLdp]
  float *Qs = Ps + kXwOpFloats;          // [64][kXwLdp]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int fe = 64 * nt, nti = xw_ntiles(nt);
  const int64_t wsf = xw_ws_floats(nt);
  float *const ws = workspaces + (int64_t)blockIdx.x * wsf;  // this CTA's A tiles, then its b
  if (tid < 64) wneg[tid] = -1.f;

  for (int item = blockIdx.x; item < n_work; item += gridDim.x) {
    const WorkItem wi = work[item];
    const bool whole = wi.slot == -1, chunk = wi.slot >= 0;
    const int64_t xrow = (row_offset + wi.row) * (int64_t)ld;
    __syncthreads();
    if (whole && wi.k0 == wi.k1) {  // empty row -> zeros (_als.pyx:98-100)
      for (int m = tid; m < ld; m += kXwThreads) {
        X[xrow + m] = 0.f;
        for (int pi = 0; pi < n_peers; ++pi) peers[pi][xrow + m] = 0.f;
      }
      continue;
    }
    // ---------------- normal equations: A tiles -> ws (or the chunk's slot), b -> bs (or the slot)
    float *dst = chunk ? slots + (int64_t)wi.slot * wsf : ws;
    if (pass == 0) {
      const int nch = (wi.k1 - wi.k0 + kXwKs - 1) / kXwKs;
      const int nsteps = nti * nch;
      int fI = 0, fJ = 0, fc = 0;  // the (tile, chunk) step being fetched; step s is staged at un + (s & 1) stages
      stage_fetch(un, indices, data, Y, ld, wi.k0, wi.k1, 0, 0, tid);
      int I = 0, J = 0, c = 0;     // the step being computed
      float acc[4][4], bacc = 0.f;
      for (int s = 0; s < nsteps; ++s) {
        if (c == 0) {
          if (chunk) acc_zero(acc);
          else acc_load(acc, Greg + (int64_t)(64 * I) * ld + 64 * J, ld, warp, lane);
        }
        if (++fc == nch) {
          fc = 0;
          if (++fJ == nt) fJ = ++fI;
        }
        if (s + 1 < nsteps) {
          stage_fetch(un + ((s + 1) & 1) * kXwStageFloats, indices, data, Y, ld, wi.k0 + kXwKs * fc, wi.k1, fI, fJ, tid);
          cp_async_wait<1>();
        } else {
          cp_async_wait<0>();
        }
        __syncthreads();
        const float *P = un + (s & 1) * kXwStageFloats, *Q = (J == I) ? P : P + kXwKs * kXwLdp;
        const float *wk = P + 2 * kXwKs * kXwLdp, *ck = wk + kXwKs;
        tile_mma(acc, P, Q, wk, kXwKs / 8, warp, lane);
        if (J == I && tid < 64) {
#pragma unroll 8
          for (int r = 0; r < kXwKs; ++r) bacc = fmaf(ck[r], P[r * kXwLdp + tid], bacc);
        }
        __syncthreads();
        if (++c == nch) {
          acc_store(acc, dst + (int64_t)xw_tidx(nt, I, J) * kXwTileFloats, 64, warp, lane);
          if (J == I && tid < 64) {
            if (chunk) dst[(int64_t)nti * kXwTileFloats + 64 * I + tid] = bacc;
            else bs[64 * I + tid] = bacc;
            bacc = 0.f;
          }
          c = 0;
          if (++J == nt) J = ++I;
        }
      }
      if (chunk) continue;
    } else {  // finish: Greg plus the chunk partials in slot order
      for (int64_t e = tid; e < (int64_t)nti * kXwTileFloats; e += kXwThreads) {
        const int tile = (int)(e / kXwTileFloats), r = (int)(e / 64) % 64, cc = (int)(e % 64);
        int I = 0;
        while (xw_tidx(nt, I + 1, I + 1) <= tile && I + 1 < nt) ++I;
        const int J = I + tile - xw_tidx(nt, I, I);
        float v = Greg[(int64_t)(64 * I + r) * ld + 64 * J + cc];
        for (int s = 0; s < wi.k1; ++s) v += slots[(int64_t)(wi.k0 + s) * wsf + e];
        ws[e] = v;
      }
      for (int m = tid; m < fe; m += kXwThreads) {
        float v = 0.f;
        for (int s = 0; s < wi.k1; ++s) v += slots[(int64_t)(wi.k0 + s) * wsf + (int64_t)nti * kXwTileFloats + m];
        bs[m] = v;
      }
    }
    if (tid == 0) *flag = 0;
    __syncthreads();

    // ---------------- blocked right-looking Cholesky, 64-column panels
    const int ty = tid >> 4, tx = tid & 15;
    for (int K = 0; K < nt; ++K) {
      // 1. diagonal block [A_KK | b_K] -> [U_KK (reciprocal diagonal) | z_K]
      const float *akk = ws + (int64_t)xw_tidx(nt, K, K) * kXwTileFloats;
      for (int e = tid; e < 64 * 64; e += kXwThreads) {
        const int r = e >> 6, cc = e & 63;
        Ad[r * kXwLda + cc] = akk[e];
      }
      if (tid < 64) Ad[tid * kXwLda + 128] = bs[64 * K + tid];
      __syncthreads();
      for (int k = 0; k < 64; ++k) {
        const float d = Ad[k * kXwLda + k];
        if (!(d > 0.f)) {
          if (tid == 0) *flag = 1;
          break;  // uniform: every thread reads the same d
        }
        float s = rsqrtf(d);
        s = s * fmaf(-0.5f * d * s, s, 1.5f);
        __syncthreads();
        for (int j = k + 1 + tid; j < 64; j += kXwThreads) Ad[k * kXwLda + j] *= s;
        if (tid == 0) {
          Ad[k * kXwLda + k] = s;
          Ad[k * kXwLda + 128] *= s;
        }
        __syncthreads();
        for (int i = k + 1 + ty; i < 64; i += 16) {
          const float uki = Ad[k * kXwLda + i];
          float *ai = Ad + i * kXwLda;
          const float *ak = Ad + k * kXwLda;
          for (int j = i + ((tx - i) & 15); j < 64; j += 16) ai[j] = fmaf(-uki, ak[j], ai[j]);  // j >= i
          if (tx == 0) ai[128] = fmaf(-uki, ak[128], ai[128]);
        }
        __syncthreads();
      }
      __syncthreads();
      if (*flag) break;
      // 2. U_KK (upper, reciprocal diagonal) -> the diagonal tile, for the back substitution; z_K -> bs
      float *ukk = ws + (int64_t)xw_tidx(nt, K, K) * kXwTileFloats;
      for (int e = tid; e < 64 * 64; e += kXwThreads) ukk[e] = Ad[(e >> 6) * kXwLda + (e & 63)];
      if (tid < 64) bs[64 * K + tid] = Ad[tid * kXwLda + 128];
      __syncthreads();
      // 3. panel row: U_KK^T U_KJ = A_KJ by forward substitution in shared memory (one column per thread, four
      //    threads share the rows), then b_J -= U_KJ^T z_K
      for (int J = K + 1; J < nt; ++J) {
        float *akj = ws + (int64_t)xw_tidx(nt, K, J) * kXwTileFloats;
        tile_fetch(Qs, akj, tid);
        cp_async_wait<0>();
        __syncthreads();
        const int c = tid & 63, r4 = tid >> 6;
        for (int r = 0; r < 64; ++r) {
          if (r4 == 0) Qs[r * kXwLdp + c] *= Ad[r * kXwLda + r];
          __syncthreads();
          const float xr = Qs[r * kXwLdp + c];
          for (int i = r + 1 + r4; i < 64; i += 4) Qs[i * kXwLdp + c] = fmaf(-Ad[r * kXwLda + i], xr, Qs[i * kXwLdp + c]);
          __syncthreads();
        }
        for (int e = tid; e < 64 * 64; e += kXwThreads) akj[e] = Qs[(e >> 6) * kXwLdp + (e & 63)];
        if (tid < 64) {
          float v = bs[64 * J + tid];
#pragma unroll 8
          for (int r = 0; r < 64; ++r) v = fmaf(-Qs[r * kXwLdp + tid], bs[64 * K + r], v);
          bs[64 * J + tid] = v;
        }
        __syncthreads();
      }
      // 4. trailing update: A_IJ -= U_KI^T U_KJ for K < I <= J
      for (int I = K + 1; I < nt; ++I) {
        tile_fetch(Ps, ws + (int64_t)xw_tidx(nt, K, I) * kXwTileFloats, tid);
        for (int J = I; J < nt; ++J) {
          if (J != I) tile_fetch(Qs, ws + (int64_t)xw_tidx(nt, K, J) * kXwTileFloats, tid);
          float *aij = ws + (int64_t)xw_tidx(nt, I, J) * kXwTileFloats;
          float acc[4][4];
          acc_load(acc, aij, 64, warp, lane);
          cp_async_wait<0>();
          __syncthreads();
          tile_mma(acc, Ps, J == I ? Ps : Qs, wneg, 8, warp, lane);
          acc_store(acc, aij, 64, warp, lane);
          __syncthreads();
        }
      }
    }
    __syncthreads();
    if (*flag) {
      if (tid == 0) atomicMin(bad_row, (long long)(row_offset + wi.row));
      continue;
    }
    // ---------------- blocked back substitution: U_KK x_K = z_K - sum_{J > K} U_KJ x_J
    for (int K = nt - 1; K >= 0; --K) {
      for (int m = warp; m < 64; m += kXwThreads / 32) {
        float v = 0.f;
        for (int J = K + 1; J < nt; ++J) {
          const float *ukj = ws + (int64_t)xw_tidx(nt, K, J) * kXwTileFloats + m * 64;
          v = fmaf(ukj[lane], bs[64 * J + lane], v);
          v = fmaf(ukj[lane + 32], bs[64 * J + lane + 32], v);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) rs[m] = bs[64 * K + m] - v;
      }
      const float *ukk = ws + (int64_t)xw_tidx(nt, K, K) * kXwTileFloats;
      for (int e = tid; e < 64 * 64; e += kXwThreads) Ad[(e >> 6) * kXwLda + (e & 63)] = ukk[e];
      __syncthreads();
      // U_KK x_K = r, column oriented (the diagonal holds 1 / u_kk)
      for (int k = 63; k >= 0; --k) {
        if (tid == 0) rs[k] *= Ad[k * kXwLda + k];
        __syncthreads();
        if (tid < k) rs[tid] = fmaf(-Ad[tid * kXwLda + k], rs[k], rs[tid]);
        __syncthreads();
      }
      if (tid < 64) bs[64 * K + tid] = rs[tid];
      __syncthreads();
    }
    for (int m = tid; m < ld; m += kXwThreads) {
      const float v = m < fe ? bs[m] : 0.f;
      X[xrow + m] = v;
      for (int pi = 0; pi < n_peers; ++pi) peers[pi][xrow + m] = v;
    }
  }
}

// as init_solver_scalars (cholesky.cu): [1] keeps the first bad row of every half since the last als_solver_status
__global__ void xwide_init_bad_row(long long *bad_row) {
  if (bad_row[0] < bad_row[1]) bad_row[1] = bad_row[0];
  bad_row[0] = LLONG_MAX;
}

}  // namespace

int launch_cholesky_xwide(als_ctx *ctx, const als_csr *Cw, als_factors *X, const als_factors *Y) {
  if (Y->ld > 1024 || Y->ld % 64) {
    set_error("cholesky: padded factors %d out of range", Y->ld);
    return ALS_E_INVALID;
  }
  const int nt = round_up(Y->f, 64) / 64;
  const int64_t wsf = xw_ws_floats(nt);
  const int smem = kXwSmemFloats * (int)sizeof(float);
  auto kern = cholesky_xwide_kernel;
  ALS_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int per_sm = 0;
  ALS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kXwThreads, smem));
  if (per_sm < 1) {
    set_error("cholesky: wide kernel does not fit on an SM (smem %d bytes)", smem);
    return ALS_E_CUDA;
  }
  const int64_t max_grid = (int64_t)ctx->sm_count * per_sm;
  // row-block segments run one after the other: the scratch covers the largest, bad_row is reset once per half
  const std::vector<const als_csr *> segs = segments_of(Cw);
  int64_t max_slots = 0, n_ws = 0;
  for (const als_csr *S : segs) {
    max_slots = std::max(max_slots, S->n_slots);
    // one scratch block: the giant-row slots, then one workspace per resident CTA
    n_ws = std::max(n_ws, std::min<int64_t>(std::max(S->n_work, S->n_finish), max_grid));
  }
  // (n_slots + n_ws) * wsf floats: 2.2 MB per giant-row chunk and per workspace at 1024 factors
  const int64_t bytes = (max_slots + n_ws) * wsf * (int64_t)sizeof(float);
  int rc = ensure_scratch(ctx, bytes);
  if (rc != ALS_OK) {
    set_error("cholesky: factors=%d needs %.2f GB of device scratch (%lld giant-row chunks and %lld workspaces of %.2f MB "
              "each) and the allocation failed; split the rows into smaller calls or use the CG solver",
              Y->f, bytes / 1e9, (long long)max_slots, (long long)n_ws, wsf * 4 / 1e6);
    return rc;
  }
  float *slots = (float *)ctx->scratch;
  float *workspaces = slots + max_slots * wsf;
  xwide_init_bad_row<<<1, 1, 0, ctx->stream>>>(ctx->bad_row);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  return for_each_segment(ctx, Cw, [&](size_t, const als_csr *Cm) -> int {
    const int grid0 = (int)std::min<int64_t>(Cm->n_work, max_grid);
    const int grid1 = (int)std::min<int64_t>(Cm->n_finish, max_grid);
    if (Cm->n_work) {
      ProfScope prof(ctx, kProfCholesky);
      kern<<<grid0, kXwThreads, smem, ctx->stream>>>(Cm->indices, Cm->data, Y->d, X->d, Y->ld, nt, Cm->row_offset, ctx->Greg,
                                                     Cm->work, (int)Cm->n_work, slots, workspaces, ctx->bad_row, 0,
                                                     X->peers_dev, X->n_peers);
      ALS_CUDA(cudaGetLastError());
      ctx->launches++;
    }
    if (Cm->n_finish) {
      ProfScope prof(ctx, kProfCholFinish);
      kern<<<grid1, kXwThreads, smem, ctx->stream>>>(Cm->indices, Cm->data, Y->d, X->d, Y->ld, nt, Cm->row_offset, ctx->Greg,
                                                     Cm->finish, (int)Cm->n_finish, slots, workspaces, ctx->bad_row, 1,
                                                     X->peers_dev, X->n_peers);
      ALS_CUDA(cudaGetLastError());
      ctx->launches++;
    }
    return ALS_OK;
  });
}

}  // namespace als
