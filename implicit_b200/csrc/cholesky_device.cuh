// Device-side building blocks shared by the per-row Cholesky kernels (cholesky.cu: the full F x F normal
// equations; cholesky_short.cu: the n x n push-through system of short rows): TF32 split + mma.sync wrappers,
// cp.async helpers, the packed-panel layout and the blocked register/shared-memory Cholesky solve.
#pragma once
#include <limits.h>
#include <stdlib.h>

#include <cuda_fp16.h>

#include "common.h"

namespace als {

namespace {

__device__ __forceinline__ void mma_tf32(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                         uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void cp_async16(float *smem_dst, const float *gmem_src) {
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory");
}

constexpr uint32_t kTf32Mask = 0xffffe000u;  // keep sign, exponent and the 10 TF32 mantissa bits
constexpr uint32_t kSignBit = 0x80000000u;

// hi = x rounded to nearest TF32 (add half an ulp of the 10-bit mantissa, then clear the low 13 bits),
// lo = (x - hi) -- exact in fp32 -- rounded the same way.  Rounding (instead of letting the tensor core
// truncate) halves the error of each term and, more importantly, removes its bias: on all-positive
// data (the first ALS half-iteration) truncation errors add up linearly instead of as a random walk.
__device__ __forceinline__ uint32_t rn_tf32(float x) { return (__float_as_uint(x) + 0x1000u) & kTf32Mask; }
// lo is handed over raw: the tensor core drops its low 13 bits, an error of at most 2^-21 |x| that is
// unbiased because, with hi rounded to nearest, lo is symmetric around zero.  (Rounding lo as well
// cost two more integer ops per value -- 17% of the kernel's instructions -- for no measurable gain.)
__device__ __forceinline__ void split_tf32(float x, uint32_t &hi, uint32_t &lo) {
  hi = rn_tf32(x);
  lo = __float_as_uint(x - __uint_as_float(hi));
}

__device__ __forceinline__ float rcp_approx(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float rsqrt_approx(float x) {
  float r;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

template <int NB>
struct Cfg {
  static constexpr int F = 16 * NB;         // padded factors
  static constexpr int NT8 = 2 * NB;        // 8-wide column tiles == 8-row panels
  static constexpr int NTILES = NB * (NB + 1);
  static constexpr int LDS = F + 8;         // staged-row stride: conflict-free fragment reads
  static constexpr int NSTAGE = 3;
  static constexpr int STAGE_FLOATS = 8 * LDS + 16;  // 8 rows + sw[8] + cpos[8]
  // packed U: panel p holds rows 8p..8p+7, columns 8p..F-1; stride == 8 or 24 (mod 32)
  __host__ __device__ static constexpr int pstride(int p) { return F - 8 * p + ((p & 1) ? 0 : 8); }
  __host__ __device__ static constexpr int poff(int p) {
    int o = 0;
    for (int q = 0; q < p; ++q) o += 8 * pstride(q);
    return o;
  }
  static constexpr int U_FLOATS = poff(NT8);
  static constexpr int WARP_FLOATS = NSTAGE * STAGE_FLOATS + U_FLOATS + F /* z */;
  // index of tile (i, j), j >= 2i, in the upper-triangular tile list
  __host__ __device__ static constexpr int tidx(int i, int j) { return i * NT8 - i * (i - 1) + (j - 2 * i); }
  static constexpr int SLOT_FLOATS = 32 * (NTILES * 4 + NT8);
};

constexpr int kWarpsPerCta = 1;  // warps share nothing: one-warp CTAs let shared memory (19.5 KB each), not CTA granularity, set the occupancy

template <int NB>
struct RowState {
  float acc[Cfg<NB>::NTILES][4];
  float bp[Cfg<NB>::NT8];  // b partials: b[8c + g] = sum over the 4 lanes of group g of bp[c]
};

// 32 consecutive nonzeros of a row, one per lane, prefetched into registers well before the k-steps
// that gather them (the index load would otherwise sit on the critical path of every k-step).
struct Blk {
  int idx;   // column index, -1 past the end of the row
  float c;   // raw confidence; decoded only when the k-step is issued, so the load stays in flight
};

__device__ __forceinline__ Blk load_block(const WorkItem &wi, int b, const int32_t *__restrict__ indices,
                                          const float *__restrict__ data, int lane) {
  const int k = wi.k0 + 32 * b + lane;
  const bool valid = k < wi.k1;
  Blk r;
  r.idx = valid ? __ldg(indices + k) : -1;
  r.c = valid ? __ldg(data + k) : 0.f;
  return r;
}

// ---- gather: k-step s (0..3) of block `blk` -> stage -----------------------------------------------
template <int NB>
__device__ __forceinline__ void issue_kstep(float *stage, const Blk &blk, int s, bool active,
                                            const float *__restrict__ Y, int lane) {
  using C = Cfg<NB>;
  if (active) {  // warp uniform
    const int src = 8 * s + (lane & 7);
    const float c = __shfl_sync(0xffffffffu, blk.c, src);
    const int myidx = __shfl_sync(0xffffffffu, blk.idx, src);
    if (lane < 8) {
      // A += w y y^T with w = |c| - 1 = sign(w) (sqrt|w| y)(sqrt|w| y)^T; b += c y for c > 0   (_als.pyx:115-124)
      const float w = (myidx >= 0) ? fabsf(c) - 1.f : 0.f;
      stage[8 * C::LDS + lane] = copysignf(__fsqrt_rn(fabsf(w)), w);
      stage[8 * C::LDS + 8 + lane] = (myidx >= 0 && c > 0.f) ? c : 0.f;
    }
    const int first = __shfl_sync(0xffffffffu, blk.idx, 8 * s);  // the first row of an active k-step exists
    constexpr int CH = C::F / 4;  // 16-byte chunks per factor row
#pragma unroll
    for (int q = 0; q < NB; ++q) {
      const int id = q * 32 + lane;
      const int row = id / CH, ch = id % CH;
      int ridx = __shfl_sync(0xffffffffu, blk.idx, 8 * s + row);
      if (ridx < 0) ridx = first;  // padding rows carry sw = cp = 0
      cp_async16(stage + row * C::LDS + ch * 4, Y + (int64_t)ridx * C::F + ch * 4);
    }
  }
  cp_async_commit();
}

// ---- accumulate one k-step (8 nonzeros) --------------------------------------------------------
template <int NB>
__device__ __forceinline__ void consume_kstep(RowState<NB> &st, const float *stage, int g, int t) {
  using C = Cfg<NB>;
  const float s0 = stage[8 * C::LDS + t], s1 = stage[8 * C::LDS + t + 4];
  const float c0 = stage[8 * C::LDS + 8 + t], c1 = stage[8 * C::LDS + 8 + t + 4];
  const float a0 = fabsf(s0), a1 = fabsf(s1);
  const uint32_t m0 = __float_as_uint(s0) & kSignBit, m1 = __float_as_uint(s1) & kSignBit;
  uint32_t vh0[C::NT8], vl0[C::NT8], vh1[C::NT8], vl1[C::NT8];
#pragma unroll
  for (int c = 0; c < C::NT8; ++c) {
    const float y0 = stage[t * C::LDS + 8 * c + g];
    const float y1 = stage[(t + 4) * C::LDS + 8 * c + g];
    st.bp[c] = fmaf(c0, y0, st.bp[c]);
    st.bp[c] = fmaf(c1, y1, st.bp[c]);
    split_tf32(a0 * y0, vh0[c], vl0[c]);  // v = sqrt|w| y: one split serves both mma operands
    split_tf32(a1 * y1, vh1[c], vl1[c]);
  }
  // Term-major order: the three 3xTF32 terms of one tile chain through its accumulator, so they are
  // issued a full sweep of tiles apart instead of back to back (an HMMA result takes ~35 cycles).
#pragma unroll
  for (int term = 0; term < 3; ++term) {
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      // A fragment: rows 16i + g (a0, a2) and 16i + 8 + g (a1, a3) of sign(w) v; lo part for term 0
      const uint32_t a0 = (term == 0 ? vl0[2 * i] : vh0[2 * i]) ^ m0;
      const uint32_t a1 = (term == 0 ? vl0[2 * i + 1] : vh0[2 * i + 1]) ^ m0;
      const uint32_t a2 = (term == 0 ? vl1[2 * i] : vh1[2 * i]) ^ m1;
      const uint32_t a3 = (term == 0 ? vl1[2 * i + 1] : vh1[2 * i + 1]) ^ m1;
#pragma unroll
      for (int j = 2 * i; j < C::NT8; ++j) {
        float(&d)[4] = st.acc[C::tidx(i, j)];
        if (term == 1) mma_tf32(d, a0, a1, a2, a3, vl0[j], vl1[j]);  // hi * lo
        else mma_tf32(d, a0, a1, a2, a3, vh0[j], vh1[j]);            // lo * hi, then hi * hi
      }
    }
  }
}

// ---- fp16-split accumulation: 16 nonzeros per k-step on mma.sync.m16n8k16 ---------------------------------
// v = sigma sqrt|w| y is split into an fp16 pair hi + lo (both rounded to nearest: 22 bits of every value that is
// not tiny against the largest one), with sigma a power of two chosen per half-iteration from max|w| and max|y| so
// that the largest product stays below 2^14.  A_u is then accumulated as  sigma^2 A_u  (the solve is invariant).
// Three HMMAs per tile and 16 nonzeros instead of three per 8: half the tensor instructions of the 3xTF32 path.
__device__ __forceinline__ void mma_f16(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                        uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void split_f16_pair(float x0, float x1, uint32_t &hi, uint32_t &lo) {
  const __half2 h = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
  hi = *reinterpret_cast<const uint32_t *>(&h);
  lo = *reinterpret_cast<const uint32_t *>(&l);
}

// the power of two sigma that scales a positive maximum p to just below 2^14 (see topk_tc.cu).  Its exponent is clamped
// to [-63, 63] so that sigma^2 and 1 / sigma^2 stay normal fp32 numbers (the kernels multiply by both): sigma is exact
// for p in [2^-50, 2^77); a smaller p leaves the operands below 2^14 (p < 2^-50: factors of order 1e-16), a larger one
// is past any Gramian that fits in fp32.
__device__ __forceinline__ float pow2_scale_below_2_14(float p) {
  const unsigned b = __float_as_uint(p);
  const int E = (int)(b >> 23) & 0xff;
  int se = (b & 0x7fffffffu) ? 267 - E : 127;
  se = se < 127 - 63 ? 127 - 63 : se > 127 + 63 ? 127 + 63 : se;
  return __uint_as_float((unsigned)se << 23);
}

template <int NB>
struct Cfg16 {
  using C = Cfg<NB>;
  static constexpr int F = C::F;
  static constexpr int LDS = F + 4;          // staged-row stride: rows 2t, 2t+1, 2t+8, 2t+9 hit distinct banks
  static constexpr int NSTAGE = 2;
  static constexpr int STAGE_FLOATS = 16 * LDS + 32;  // 16 rows + sw[16] + cpos[16]
  static constexpr int WARP_FLOATS = NSTAGE * STAGE_FLOATS + C::U_FLOATS + F /* z */;
};

// gather: k-step s2 (0..1) of block `blk` (32 nonzeros in registers, one per lane) -> stage
template <int NB>
__device__ __forceinline__ void issue_kstep16(float *stage, const Blk &blk, int s2, bool active, float sigma,
                                              const float *__restrict__ Y, int lane) {
  using C = Cfg16<NB>;
  if (active) {  // warp uniform
    const int src = 16 * s2 + (lane & 15);
    const float c = __shfl_sync(0xffffffffu, blk.c, src);
    const int myidx = __shfl_sync(0xffffffffu, blk.idx, src);
    if (lane < 16) {
      // A += w y y^T with w = |c| - 1 = sign(w) (sqrt|w| y)(sqrt|w| y)^T; b += c y for c > 0   (_als.pyx:115-124)
      const float w = (myidx >= 0) ? fabsf(c) - 1.f : 0.f;
      stage[16 * C::LDS + lane] = copysignf(sigma * __fsqrt_rn(fabsf(w)), w);
      stage[16 * C::LDS + 16 + lane] = (myidx >= 0 && c > 0.f) ? c : 0.f;
    }
    const int first = __shfl_sync(0xffffffffu, blk.idx, 16 * s2);  // the first row of an active k-step exists
    constexpr int CH = C::F / 4;  // 16-byte chunks per factor row
#pragma unroll
    for (int q = 0; q < 2 * NB; ++q) {
      const int id = q * 32 + lane;
      const int row = id / CH, ch = id % CH;
      int ridx = __shfl_sync(0xffffffffu, blk.idx, 16 * s2 + row);
      if (ridx < 0) ridx = first;  // padding rows carry sw = cp = 0
      cp_async16(stage + row * C::LDS + ch * 4, Y + (int64_t)ridx * C::F + ch * 4);
    }
  }
  cp_async_commit();
}

// accumulate one k-step (16 nonzeros)
template <int NB>
__device__ __forceinline__ void consume_kstep16(RowState<NB> &st, const float *stage, int g, int t) {
  using C = Cfg<NB>;
  constexpr int LDS = Cfg16<NB>::LDS;
  const float2 s0 = *reinterpret_cast<const float2 *>(stage + 16 * LDS + 2 * t);       // nonzeros 2t, 2t+1
  const float2 s1 = *reinterpret_cast<const float2 *>(stage + 16 * LDS + 2 * t + 8);   // nonzeros 2t+8, 2t+9
  const float2 c0 = *reinterpret_cast<const float2 *>(stage + 16 * LDS + 16 + 2 * t);
  const float2 c1 = *reinterpret_cast<const float2 *>(stage + 16 * LDS + 16 + 2 * t + 8);
  const float a00 = fabsf(s0.x), a01 = fabsf(s0.y), a10 = fabsf(s1.x), a11 = fabsf(s1.y);
  // sign of w on the A side: flip the halves of the packed pairs
  const uint32_t m0 = ((__float_as_uint(s0.x) >> 16) & 0x8000u) | (__float_as_uint(s0.y) & kSignBit);
  const uint32_t m1 = ((__float_as_uint(s1.x) >> 16) & 0x8000u) | (__float_as_uint(s1.y) & kSignBit);
  uint32_t h0[C::NT8], l0[C::NT8], h1[C::NT8], l1[C::NT8];
  const float *r00 = stage + (2 * t) * LDS + g, *r01 = r00 + LDS, *r10 = r00 + 8 * LDS, *r11 = r10 + LDS;
#pragma unroll
  for (int c = 0; c < C::NT8; ++c) {
    const float y00 = r00[8 * c], y01 = r01[8 * c], y10 = r10[8 * c], y11 = r11[8 * c];
    st.bp[c] = fmaf(c0.x, y00, st.bp[c]);
    st.bp[c] = fmaf(c0.y, y01, st.bp[c]);
    st.bp[c] = fmaf(c1.x, y10, st.bp[c]);
    st.bp[c] = fmaf(c1.y, y11, st.bp[c]);
    split_f16_pair(a00 * y00, a01 * y01, h0[c], l0[c]);  // one split serves both mma operands
    split_f16_pair(a10 * y10, a11 * y11, h1[c], l1[c]);
  }
#pragma unroll
  for (int term = 0; term < 3; ++term) {  // lo * hi, hi * lo, hi * hi: term major (see consume_kstep)
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      const uint32_t a0 = (term == 0 ? l0[2 * i] : h0[2 * i]) ^ m0;
      const uint32_t a1 = (term == 0 ? l0[2 * i + 1] : h0[2 * i + 1]) ^ m0;
      const uint32_t a2 = (term == 0 ? l1[2 * i] : h1[2 * i]) ^ m1;
      const uint32_t a3 = (term == 0 ? l1[2 * i + 1] : h1[2 * i + 1]) ^ m1;
#pragma unroll
      for (int j = 2 * i; j < C::NT8; ++j) {
        float(&d)[4] = st.acc[C::tidx(i, j)];
        if (term == 1) mma_f16(d, a0, a1, a2, a3, l0[j], l1[j]);
        else mma_f16(d, a0, a1, a2, a3, h0[j], h1[j]);
      }
    }
  }
}

// ---- blocked Cholesky + solves -----------------------------------------------------------------
// Right-looking, 8-row panels.  Panel p is spilled from the accumulator tiles to shared memory; one
// lane owns one panel column (plus the rhs slice as an extra column) and the 8 pivots are eliminated
// in order: the pivot lane broadcasts 1/sqrt(d), every lane scales its row-r entry, the lanes of the
// diagonal block broadcast U[r][r'] and every lane updates its later rows.  The trailing matrix is
// then updated in registers with 3xTF32 mma tiles.  A non-positive pivot yields a non-finite
// solution, which is how failure is detected (LAPACK posv info != 0, _als.pyx:131-138).
// On return xx[q] holds x[lane + 32 q]; ok == false when any component is non-finite.
template <int NB>
__device__ __forceinline__ void factor_solve(RowState<NB> &st, float *U, float *zb, int lane, bool &ok, int dbg,
                                             float (&xx)[(Cfg<NB>::F + 31) / 32]) {
  using C = Cfg<NB>;
  constexpr int F = C::F;
  const int g = lane >> 2, t = lane & 3;

#pragma unroll
  for (int p = 0; p < C::NT8; ++p) {
    const int i = p >> 1, h = p & 1;
    float *Up = U + C::poff(p);
    const int sp = C::pstride(p);
    const int Wp = F - 8 * p;
    constexpr int NJmax = (F + 9 + 31) / 32;
    const int NJ = (Wp + 9 + 31) / 32;
    // 1. spill panel rows 8p..8p+7 (columns 8p..F-1) and the matching slice of b
#pragma unroll
    for (int j = p; j < C::NT8; ++j) {
      const float2 v = make_float2(st.acc[C::tidx(i, j)][2 * h], st.acc[C::tidx(i, j)][2 * h + 1]);
      *reinterpret_cast<float2 *>(Up + g * sp + 8 * (j - p) + 2 * t) = v;
    }
    {
      float bq = st.bp[p];
      bq += __shfl_xor_sync(0xffffffffu, bq, 1);
      bq += __shfl_xor_sync(0xffffffffu, bq, 2);
      if (t == 0) zb[8 * p + g] = bq;
    }
    __syncwarp();
    // 2. one panel column per lane.  Local columns [0, Wp) are the matrix (the first 8 = the diagonal block),
    //    Wp is the rhs slice, and Wp+1 .. Wp+8 are the unit vectors e_0..e_7: forward-substituted with the rest
    //    they become the rows of U_d^-1, which lets the back substitution resolve a whole panel at once.
    float v[NJmax][8];
#pragma unroll
    for (int j = 0; j < NJmax; ++j) {
      if (j < NJ) {
        const int c = lane + 32 * j;
        const float *colp = (c < Wp) ? (Up + c) : (zb + 8 * p);
        const int rs = (c < Wp) ? sp : 1;
        const int e = c - Wp - 1;  // unit-vector index for the identity columns
#pragma unroll
        for (int r = 0; r < 8; ++r) v[j][r] = (c <= Wp) ? colp[r * rs] : (e == r ? 1.f : 0.f);
      }
    }
    // 3. eliminate the 8 pivots, LDL^T style: the only serial chain is  1/d_r -> (one shuffle) -> the next
    //    pivot's own update; the scaling by 1/sqrt(d_r) that turns the rows into U is applied afterwards,
    //    for all 8 rows at once.  u = a[r][r2] / d_r comes from the lane that owns diagonal-block column r2.
    if (!(dbg & 2)) {
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const float d = v[0][r];  // meaningful on lane r: the pivot
        float rc = rcp_approx(d);
        rc = rc * fmaf(-d, rc, 2.f);  // Newton step
        const float rinv = __shfl_sync(0xffffffffu, rc, r);
#pragma unroll
        for (int r2 = r + 1; r2 < 8; ++r2) {
          const float u = __shfl_sync(0xffffffffu, v[0][r], r2) * rinv;
#pragma unroll
          for (int j = 0; j < NJmax; ++j)
            if (j < NJ) v[j][r2] = fmaf(-u, v[j][r], v[j][r2]);
        }
      }
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const float d = __shfl_sync(0xffffffffu, v[0][r], r);
        float s = rsqrt_approx(d);
        s = s * fmaf(-0.5f * d * s, s, 1.5f);  // Newton step: full fp32 accuracy
#pragma unroll
        for (int j = 0; j < NJmax; ++j)
          if (j < NJ) v[j][r] *= s;
      }
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < NJmax; ++j) {
      if (j < NJ) {
        const int c = lane + 32 * j;
        if (c >= 8 && c < Wp) {
#pragma unroll
          for (int r = 0; r < 8; ++r) Up[r * sp + c] = v[j][r];
        } else if (c == Wp) {
#pragma unroll
          for (int r = 0; r < 8; ++r) zb[8 * p + r] = v[j][r];
        } else if (c > Wp && c <= Wp + 8) {
          // row (c - Wp - 1) of U_d^-1 replaces that row of the diagonal block (U_d itself is not needed again)
          float *dst = Up + (c - Wp - 1) * sp;
          *reinterpret_cast<float4 *>(dst) = make_float4(v[j][0], v[j][1], v[j][2], v[j][3]);
          *reinterpret_cast<float4 *>(dst + 4) = make_float4(v[j][4], v[j][5], v[j][6], v[j][7]);
        }
      }
    }
    __syncwarp();
    // 4. trailing update in registers: A[m][n] -= sum_r U[r][m] U[r][n]; b[m] -= sum_r U[r][m] z[r]
    if (p + 1 < C::NT8 && !(dbg & 4)) {
      const float z0 = zb[8 * p + t], z1 = zb[8 * p + t + 4];
      uint32_t uh0[C::NT8], ul0[C::NT8], uh1[C::NT8], ul1[C::NT8];
#pragma unroll
      for (int j = p + 1; j < C::NT8; ++j) {
        const float u0 = Up[t * sp + 8 * (j - p) + g];
        const float u1 = Up[(t + 4) * sp + 8 * (j - p) + g];
        st.bp[j] = fmaf(-u0, z0, st.bp[j]);
        st.bp[j] = fmaf(-u1, z1, st.bp[j]);
        split_tf32(u0, uh0[j], ul0[j]);
        split_tf32(u1, uh1[j], ul1[j]);
      }
#pragma unroll
      for (int term = 0; term < 3; ++term) {  // term-major, as in consume_kstep
#pragma unroll
        for (int ib = (p + 1) >> 1; ib < NB; ++ib) {
          // rows 16 ib + g (a0, a2) are still live only if 2 ib > p
          const bool top = (2 * ib > p);
          const int jt = top ? 2 * ib : p + 1;
          const uint32_t a0 = top ? ((term == 0 ? ul0[jt] : uh0[jt]) ^ kSignBit) : 0u;
          const uint32_t a2 = top ? ((term == 0 ? ul1[jt] : uh1[jt]) ^ kSignBit) : 0u;
          const uint32_t a1 = (term == 0 ? ul0[2 * ib + 1] : uh0[2 * ib + 1]) ^ kSignBit;
          const uint32_t a3 = (term == 0 ? ul1[2 * ib + 1] : uh1[2 * ib + 1]) ^ kSignBit;
#pragma unroll
          for (int j = (2 * ib > p + 1 ? 2 * ib : p + 1); j < C::NT8; ++j) {
            float(&d)[4] = st.acc[C::tidx(ib, j)];
            if (term == 1) mma_tf32(d, a0, a1, a2, a3, ul0[j], ul1[j]);
            else mma_tf32(d, a0, a1, a2, a3, uh0[j], uh1[j]);
          }
        }
      }
    }
  }

  // 5. back substitution U x = z, column oriented and blocked by panel: lane m (and m + 32) owns z[m];
  //    each panel's 8 unknowns are resolved in order (one shuffle + one multiply on the critical path),
  //    then every earlier row folds the panel in with two 16-byte loads and 8 FMAs.
  constexpr int Q = (F + 31) / 32;
  float zz[Q];
  int rowoff[Q];
#pragma unroll
  for (int q = 0; q < Q; ++q) {
    const int m = lane + 32 * q;
    const int mm = m < F ? m : 0;
    const int pm = mm >> 3;
    // poff(pm) in closed form: 8 * sum_{s<pm} (F - 8 s + 8 [s even])
    const int po = 8 * (pm * F - 4 * pm * (pm - 1) + 8 * ((pm + 1) >> 1));
    const int ps = F - 8 * pm + ((pm & 1) ? 0 : 8);
    rowoff[q] = po + (mm & 7) * ps - 8 * pm;  // U[m][c] lives at U[rowoff + c] for c >= 8 pm
    zz[q] = zb[mm];
    xx[q] = 0.f;
  }
  if (!(dbg & 1))
#pragma unroll
  for (int p = C::NT8 - 1; p >= 0; --p) {
    const int qp = (8 * p) >> 5;        // register slot of the panel's rows
    const int l0 = (8 * p) & 31;        // their first lane
    // this lane's row of U_d^-1 (meaningful on lanes l0..l0+7 of slot qp)
    const float4 da = *reinterpret_cast<const float4 *>(U + rowoff[qp] + 8 * p);
    const float4 db = *reinterpret_cast<const float4 *>(U + rowoff[qp] + 8 * p + 4);
    float rhs[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) rhs[c] = __shfl_sync(0xffffffffu, zz[qp], l0 + c);
    // x_r = sum_{c >= r} U_d^-1[r][c] rhs[c]  (entries below the diagonal of the stored rows are exactly 0)
    const float xm = fmaf(da.x, rhs[0], fmaf(da.y, rhs[1], fmaf(da.z, rhs[2], da.w * rhs[3]))) +
                     fmaf(db.x, rhs[4], fmaf(db.y, rhs[5], fmaf(db.z, rhs[6], db.w * rhs[7])));
    const bool in_panel = (lane >= l0) && (lane < l0 + 8);
    if (in_panel) xx[qp] = xm;
    float xs[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) xs[c] = __shfl_sync(0xffffffffu, xm, l0 + c);
    // rows before the panel fold it in
#pragma unroll
    for (int q = 0; q < Q; ++q) {
      if (32 * q < 8 * p) {
        const int m = lane + 32 * q;
        if (m < 8 * p) {
          const float4 ua = *reinterpret_cast<const float4 *>(U + rowoff[q] + 8 * p);
          const float4 ub = *reinterpret_cast<const float4 *>(U + rowoff[q] + 8 * p + 4);
          const float s0 = fmaf(ua.x, xs[0], fmaf(ua.y, xs[1], fmaf(ua.z, xs[2], ua.w * xs[3])));
          const float s1 = fmaf(ub.x, xs[4], fmaf(ub.y, xs[5], fmaf(ub.z, xs[6], ub.w * xs[7])));
          zz[q] -= s0 + s1;
        }
      }
    }
  }
  bool fin = true;
#pragma unroll
  for (int q = 0; q < Q; ++q) {
    const int m = lane + 32 * q;
    if (m < F) {
      fin = fin && (fabsf(xx[q]) <= 3.0e38f);  // false for inf and NaN
    }
  }
  ok = __all_sync(0xffffffffu, fin);
}

// x -> this replica and, over NVLink, every peer replica of the factor matrix
template <int F>
__device__ __forceinline__ void store_solution(const float (&xx)[(F + 31) / 32], float *__restrict__ xout, int lane,
                                               float *const *peers, int n_peers, int64_t xoff) {
#pragma unroll
  for (int q = 0; q < (F + 31) / 32; ++q) {
    const int m = lane + 32 * q;
    if (m < F) {
      xout[m] = xx[q];
      for (int pi = 0; pi < n_peers; ++pi) peers[pi][xoff + m] = xx[q];
    }
  }
}

}  // namespace

}  // namespace als
