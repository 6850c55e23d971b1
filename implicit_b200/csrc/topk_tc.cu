// R3 on the Hopper tensor cores: fused scores + filter + top-k for large query batches at 64 padded factors
// (reference: topk.topk / _topk_batch, implicit/cpu/topk.pyx:15-67; select<T>, implicit/cpu/select.h:12-39).
//
// The score matrix  S = Q I^T  is the one large dense contraction of the hot path (C5: 1M x 1M x 64).  Here it runs
// on wgmma with TMA-fed operands; the selection is the epilogue, so a score never leaves the SM:
//   pre-pass   both factor matrices are split ONCE per call into fp16 hi / lo halves (x 2^e, e from each query row's
//              own absolute maximum and from the item matrix's, so the halves carry 22 bits however small a query row
//              is next to the others): scores = (Qh + Ql)(Ih + Il)^T ~ Ql Ih^T + Qh Il^T + Qh Ih^T,
//              fp32-faithful like the 3xTF32 split of topk.cu at half the tensor work and half the operand bytes;
//   CTA        2 x 128 query rows (hi and lo tiles resident in shared memory, K-major, 128B swizzle) sweep ALL items;
//              every landed item tile is multiplied with BOTH query tiles (half the L2 -> SM operand traffic of one
//              query tile per CTA):
//              warp 8        TMA producer: 64-item hi + lo boxes into a 4-stage ring (mbarrier complete_tx);
//              warpgroups    one per query tile: 24 wgmma.m64n64k16.f16 per item tile (two 64-row halves x three
//              0 and 1       terms x four k-steps) into fp32 registers, parked in shared memory, then one THREAD per
//                            query row: a running threshold (the k-th best so far) rejects almost everything with one
//                            max + compare per 32 scores; survivors are checked against the row's liked list (a
//                            cursor: both advance in item order) and the global filter mask, then inserted into a
//                            sorted k-list held in REGISTERS with exactly the reference's admission rule
//                            (`size < k || score > min.score`, evict the lexicographic (score, id) minimum), so ties
//                            resolve like select.h.  One warpgroup selects while the other one multiplies.
// Filtered items are skipped instead of being kept at -FLT_MAX: identical to the reference whenever every row has at
// least k unfiltered items; the caller (topk.cu) checks that bound and uses the mma.sync kernel otherwise.
#include <cuda.h>
#include <cuda_fp16.h>
#include <float.h>
#include <limits.h>

#include "common.h"
#include "sm90.cuh"

namespace als {

namespace {

using namespace sm90;

constexpr int kTkF = 64;
constexpr int kTkQ = 128;                // query rows per warpgroup
constexpr int kTkG = 2;                  // query tiles (warpgroups) per CTA: both are multiplied with every landed item tile
constexpr int kTkI = 64;                 // items per tile
constexpr int kTkStages = 4;
constexpr int kTkThreads = 128 * kTkG + 32;
constexpr int kTkProducerWarp = 4 * kTkG;
constexpr int kQBytes = kTkQ * 128;      // one 128-row x 64-half tile
constexpr int kIBytes = kTkI * 128;      // one 64-row x 64-half tile
constexpr int kScLd = kTkI + 1;          // parked scores: one row per query, padded against bank conflicts
constexpr int kTkOffQ = 0;               // per query tile: Qh | Ql
constexpr int kTkOffI = kTkG * 2 * kQBytes;               // kTkStages x (Ih | Il)
constexpr int kTkOffSc = kTkOffI + kTkStages * 2 * kIBytes;  // per query tile [128][kScLd] floats
constexpr int kTkOffBar = kTkOffSc + kTkG * kTkQ * kScLd * 4;
constexpr int kTkSmem = kTkOffBar + 128 + 1024;
static_assert(kTkSmem <= 227 * 1024, "top-k: more shared memory than a Hopper block may have");
enum { kTQFull = 0, kTFull0, kTEmpty0 = kTFull0 + kTkStages, kTNumBars = kTEmpty0 + kTkStages };

__device__ __forceinline__ float fmax3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }

// ---- pre-pass -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) tk_absmax_kernel(const float *__restrict__ x, int ld, const int32_t *__restrict__ rows,
                                                        int64_t n_rows, unsigned *out) {
  // bits of |x| order like unsigned integers for finite values; NaN / inf are left out (they cannot be scaled)
  unsigned m = 0;
  const int64_t n = n_rows * (ld / 4);
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = e / (ld / 4);
    const int64_t s = rows ? rows[r] : r;
    const float4 v = __ldg(reinterpret_cast<const float4 *>(x + s * ld) + e % (ld / 4));
    const unsigned b[4] = {__float_as_uint(v.x) & 0x7fffffffu, __float_as_uint(v.y) & 0x7fffffffu,
                           __float_as_uint(v.z) & 0x7fffffffu, __float_as_uint(v.w) & 0x7fffffffu};
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (b[j] < 0x7f800000u) m = max(m, b[j]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
}

// exponent of the power-of-two scale that brings the matrix maximum just below 2^14, as the biased exponent field
// of the scale itself; clamped so that both the scale and its inverse are normal numbers
__device__ __forceinline__ int scale_exp_field(unsigned absmax_bits) {
  const int E = (int)(absmax_bits >> 23);  // absmax in [2^(E-127), 2^(E-126))
  int se = absmax_bits ? 267 - E : 127;    // 2^(se - 127) = 2^(14 - (E - 126))
  return se < 1 ? 1 : se > 253 ? 253 : se;
}

// Splits rows of x into fp16 hi / lo halves.  absmax != nullptr: one scale for the whole matrix (the items: a score
// is compared only with the scores of the same query, so the item side may share one exponent).  absmax == nullptr:
// one scale per row, taken from that row's own absolute maximum and written to row_exp (the queries: a row far below
// the matrix maximum would otherwise lose its low bits in fp16 subnormals).
__global__ void __launch_bounds__(256) tk_split_kernel(const float *__restrict__ x, int ld, const int32_t *__restrict__ rows,
                                                       int64_t n_rows, const unsigned *__restrict__ absmax,
                                                       int *__restrict__ row_exp, uint4 *__restrict__ hi,
                                                       uint4 *__restrict__ lo) {
  const float mscale = absmax ? __uint_as_float((unsigned)scale_exp_field(*absmax) << 23) : 1.f;
  const int64_t n = n_rows * (kTkF / 8);  // 8 values -> one 16-byte chunk of halves; 8 consecutive lanes hold a row
  const int64_t n_pad = (n + 31) & ~(int64_t)31;  // whole warps stay in the loop for the per-row shuffles
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n_pad; e += (int64_t)gridDim.x * blockDim.x) {
    const bool in = e < n;
    const int64_t r = e / (kTkF / 8);
    const int c = (int)(e % (kTkF / 8));
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (in) {
      const int64_t s = rows ? rows[r] : r;
      a = __ldg(reinterpret_cast<const float4 *>(x + s * ld) + 2 * c);
      b = __ldg(reinterpret_cast<const float4 *>(x + s * ld) + 2 * c + 1);
    }
    float scale = mscale;
    if (!absmax) {
      const float u[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
      unsigned m = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const unsigned bits = __float_as_uint(u[j]) & 0x7fffffffu;
        if (bits < 0x7f800000u) m = max(m, bits);  // NaN / inf cannot be scaled (as in tk_absmax_kernel)
      }
#pragma unroll
      for (int o = 4; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
      const int se = scale_exp_field(m);
      scale = __uint_as_float((unsigned)se << 23);
      if (in && c == 0) row_exp[r] = se;
    }
    if (!in) continue;
    const float v[8] = {a.x * scale, a.y * scale, a.z * scale, a.w * scale, b.x * scale, b.y * scale, b.z * scale, b.w * scale};
    uint32_t h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __half2 hh = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
      const float2 hf = __half22float2(hh);
      const __half2 ll = __floats2half2_rn(v[2 * j] - hf.x, v[2 * j + 1] - hf.y);
      h[j] = *reinterpret_cast<const uint32_t *>(&hh);
      l[j] = *reinterpret_cast<const uint32_t *>(&ll);
    }
    hi[e] = make_uint4(h[0], h[1], h[2], h[3]);
    lo[e] = make_uint4(l[0], l[1], l[2], l[3]);
  }
}

// ---- the fused kernel -------------------------------------------------------------------------------
__device__ __forceinline__ bool pair_greater(float s, int c, float s2, int c2) { return s > s2 || (s == s2 && c > c2); }

template <int KMAX>
__global__ void __launch_bounds__(kTkThreads, 1)
topk_tc_kernel(const __grid_constant__ CUtensorMap map_qh, const __grid_constant__ CUtensorMap map_ql,
               const __grid_constant__ CUtensorMap map_ih, const __grid_constant__ CUtensorMap map_il, int n_items,
               int n_query, int k, const int *__restrict__ q_exp, const unsigned *__restrict__ absmax_i,
               const uint8_t *__restrict__ item_mask, const int32_t *__restrict__ liked_indptr,
               const int32_t *__restrict__ liked_indices, int32_t *__restrict__ out_ids, float *__restrict__ out_scores) {
  extern __shared__ unsigned char tk_smem_raw[];
  const uint32_t raw = smem_u32(tk_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  unsigned char *gbase = tk_smem_raw + (base - raw);
  const uint32_t bars = base + kTkOffBar;
  auto bar = [&](int i) -> uint32_t { return bars + 8u * (uint32_t)i; };
  const int warp = threadIdx.x >> 5;
  const int n_tiles = (n_items + kTkI - 1) / kTkI;
  const int q0 = (int)blockIdx.x * kTkQ * kTkG;

  if (threadIdx.x == 0) {
    mbar_init(bar(kTQFull), 1);
    for (int s = 0; s < kTkStages; ++s) {
      mbar_init(bar(kTFull0 + s), 1);
      mbar_init(bar(kTEmpty0 + s), kTkG);
    }
    mbar_init_fence();
  }
  __syncthreads();

  if (warp == kTkProducerWarp) {
    if ((threadIdx.x & 31) == 0) {
      mbar_expect_tx(bar(kTQFull), kTkG * 2 * kQBytes);
#pragma unroll
      for (int gq = 0; gq < kTkG; ++gq) {
        tma_load_2d(base + kTkOffQ + gq * 2 * kQBytes, &map_qh, bar(kTQFull), 0, q0 + gq * kTkQ);
        tma_load_2d(base + kTkOffQ + gq * 2 * kQBytes + kQBytes, &map_ql, bar(kTQFull), 0, q0 + gq * kTkQ);
      }
      for (int t = 0; t < n_tiles; ++t) {
        const int s = t % kTkStages;
        if (t >= kTkStages) mbar_wait(bar(kTEmpty0 + s), (uint32_t)((t / kTkStages - 1) & 1));  // both warpgroups have read it
        mbar_expect_tx(bar(kTFull0 + s), 2 * kIBytes);
        tma_load_2d(base + kTkOffI + s * 2 * kIBytes, &map_ih, bar(kTFull0 + s), 0, t * kTkI);
        tma_load_2d(base + kTkOffI + s * 2 * kIBytes + kIBytes, &map_il, bar(kTFull0 + s), 0, t * kTkI);
      }
    }
    return;
  }

  // ===== one warpgroup per query tile: multiply, park the scores, select with one thread per query row =====
  const int gq = warp >> 2;
  const int st = threadIdx.x & 127;
  float *sc = reinterpret_cast<float *>(gbase + kTkOffSc) + gq * kTkQ * kScLd;
  const float *my_row = sc + st * kScLd;
  const int q = q0 + gq * kTkQ + st;
  const bool live = q < n_query;
  float ls[KMAX];
  int lc[KMAX];
#pragma unroll
  for (int j = 0; j < KMAX; ++j) {
    ls[j] = -INFINITY;  // empty slots rank below every real (score, id)
    lc[j] = -1;
  }
  float thr = -INFINITY;  // score of the k-th best so far (raw, scaled domain): admission is score > thr
  int lp = 0, lend = 0, lnext = INT_MAX;
  if (live && liked_indptr) {
    lp = liked_indptr[q];
    lend = liked_indptr[q + 1];
    lnext = lp < lend ? liked_indices[lp] : INT_MAX;
  }
  auto consider = [&](float s, int id) {
    if (id >= n_items) return;
    while (lnext < id) {  // both the candidates and the liked list come in increasing item order (rows_in_order)
      ++lp;
      lnext = lp < lend ? liked_indices[lp] : INT_MAX;
    }
    if (lnext == id) return;                    // topk.pyx:51-54
    if (item_mask && item_mask[id]) return;     // topk.pyx:55-56
    float cs = s;
    int ci = id;
#pragma unroll
    for (int j = 0; j < KMAX; ++j) {  // carry the smaller element down the sorted list
      const bool sw = pair_greater(cs, ci, ls[j], lc[j]);
      const float ts = ls[j];
      const int ti = lc[j];
      ls[j] = sw ? cs : ts;
      lc[j] = sw ? ci : ti;
      cs = sw ? ts : cs;
      ci = sw ? ti : ci;
    }
#pragma unroll
    for (int j = 0; j < KMAX; ++j)
      if (j == k - 1) thr = ls[j];
  };
  // one 32-column chunk of the parked row: skip it unless something beats the k-th best so far
  auto scan = [&](const float *r, int id0) {
    float m[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) m[j] = fmax3(r[4 * j], r[4 * j + 1], r[4 * j + 2]);
#pragma unroll
    for (int j = 0; j < 8; ++j) m[j] = fmaxf(m[j], r[4 * j + 3]);
    const float mm = fmaxf(fmax3(m[0], m[1], m[2]), fmaxf(fmax3(m[3], m[4], m[5]), fmaxf(m[6], m[7])));
    if (live && mm > thr) {
      // rare after the first tiles: walk the chunk in item order with a rolled loop, so the k-list code exists once
      // and its arrays stay in registers
#pragma unroll 1
      for (int j = 0; j < 32; ++j) {
        const float s = r[j];
        if (s > thr) consider(s, id0 + j);
      }
    }
  };
  const uint32_t qh = base + kTkOffQ + gq * 2 * kQBytes, ql = qh + kQBytes;
  mbar_wait(bar(kTQFull), 0);
  for (int t = 0; t < n_tiles; ++t) {
    const int s = t % kTkStages;
    mbar_wait(bar(kTFull0 + s), (uint32_t)((t / kTkStages) & 1));
    const uint32_t ih = base + kTkOffI + s * 2 * kIBytes, il = ih + kIBytes;
    float d[2][32] = {};
    wgmma_fence();
#pragma unroll
    for (int mh = 0; mh < 2; ++mh)
#pragma unroll
      for (int term = 0; term < 3; ++term) {  // lo * hi, hi * lo, hi * hi (small terms first)
        const uint32_t a0 = (term == 0 ? ql : qh) + mh * 64 * 128;
        const uint32_t b0 = term == 1 ? il : ih;
#pragma unroll
        for (int ks = 0; ks < kTkF / 16; ++ks)
          wgmma_f16_m64n64k16(d[mh], wgmma_desc_k_sw128(a0 + ks * 32), wgmma_desc_k_sw128(b0 + ks * 32), term + ks > 0);
      }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operand(d[0]);
    wgmma_fence_operand(d[1]);
    if (st == 0) mbar_arrive(bar(kTEmpty0 + s));
    named_sync(1 + gq, 128);  // every row of the previous tile has been scanned
#pragma unroll
    for (int mh = 0; mh < 2; ++mh)
#pragma unroll
      for (int v = 0; v < 32; ++v) sc[(64 * mh + wgmma_row(st, v)) * kScLd + wgmma_col(st, v)] = d[mh][v];
    named_sync(1 + gq, 128);
    scan(my_row, t * kTkI);
    scan(my_row + 32, t * kTkI + 32);
  }
  if (live) {
    // scores leave the scaled domain: exact multiplications by powers of two (this query row's own, the items')
    const float inv_q = __uint_as_float((unsigned)(254 - q_exp[q]) << 23);
    const float inv_i = __uint_as_float((unsigned)(254 - scale_exp_field(*absmax_i)) << 23);
#pragma unroll
    for (int j = 0; j < KMAX; ++j)
      if (j < k && lc[j] >= 0) {  // the tail stays zero when fewer than k items qualified (topk.pyx:20-21)
        out_ids[(int64_t)q * k + j] = lc[j];
        out_scores[(int64_t)q * k + j] = ls[j] * inv_q * inv_i;
      }
  }
}


// rows x 64 fp16 row-major (128-byte rows), boxes of `box_rows` rows, 128B swizzle, rows past the end read as zero
int make_half_map(CUtensorMap *m, const void *ptr, int64_t rows, int box_rows) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess) {
      set_error("topk: cuTensorMapEncodeTiled is not available from this driver");
      return ALS_E_CUDA;
    }
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  const cuuint64_t dims[2] = {(cuuint64_t)kTkF, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)kTkF * 2};
  const cuuint32_t box[2] = {(cuuint32_t)kTkF, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("topk: cuTensorMapEncodeTiled failed with %d", (int)r);
    return ALS_E_CUDA;
  }
  return ALS_OK;
}

}  // namespace

// bytes of device scratch launch_topk_tc needs for `n_query` queries against `n_items` items
int64_t topk_tc_scratch_bytes(int64_t n_query, int64_t n_items) {
  return 256 + (n_query * 4 + 255) / 256 * 256 + 2 * ((n_query * 128 + 255) / 256 * 256) + 2 * ((n_items * 128 + 255) / 256 * 256);
}

bool topk_tc_eligible(int ld, int64_t n_query, int64_t n_items, int k, bool has_norms) {
  return ld == kTkF && k >= 1 && k <= 16 && !has_norms && n_query >= 1024 && n_items >= 256;
}

// out_ids / out_scores: device [n_query][k], zero-initialised by the caller; query_rows: device indices or nullptr
int launch_topk_tc(als_ctx *ctx, const float *items, int64_t n_items, const float *queries, const int32_t *query_rows,
                   int64_t n_query, int k, const uint8_t *mask, const int32_t *liked_indptr, const int32_t *liked_indices,
                   int32_t *out_ids, float *out_scores, void *scratch) {
  char *p = (char *)scratch;
  unsigned *absmax = (unsigned *)p;  // the items' absolute maximum
  p += 256;
  int *q_exp = (int *)p;             // per query row: the exponent field of its scale
  p += (n_query * 4 + 255) / 256 * 256;
  const int64_t qbytes = (n_query * 128 + 255) / 256 * 256, ibytes = (n_items * 128 + 255) / 256 * 256;
  void *qh = p, *ql = p + qbytes, *ih = p + 2 * qbytes, *il = p + 2 * qbytes + ibytes;
  ALS_CUDA(cudaMemsetAsync(absmax, 0, 4, ctx->stream));
  const int g = ctx->sm_count * 8;
  tk_absmax_kernel<<<g, 256, 0, ctx->stream>>>(items, kTkF, nullptr, n_items, absmax);
  tk_split_kernel<<<g, 256, 0, ctx->stream>>>(queries, kTkF, query_rows, n_query, nullptr, q_exp, (uint4 *)qh, (uint4 *)ql);
  tk_split_kernel<<<g, 256, 0, ctx->stream>>>(items, kTkF, nullptr, n_items, absmax, nullptr, (uint4 *)ih, (uint4 *)il);
  ALS_CUDA(cudaGetLastError());
  ctx->launches += 3;
  CUtensorMap mqh, mql, mih, mil;
  int rc;
  if ((rc = make_half_map(&mqh, qh, n_query, kTkQ)) != ALS_OK) return rc;
  if ((rc = make_half_map(&mql, ql, n_query, kTkQ)) != ALS_OK) return rc;
  if ((rc = make_half_map(&mih, ih, n_items, kTkI)) != ALS_OK) return rc;
  if ((rc = make_half_map(&mil, il, n_items, kTkI)) != ALS_OK) return rc;
  auto kern = topk_tc_kernel<16>;
  ALS_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kTkSmem));
  const int grid = (int)ceil_div(n_query, kTkQ * kTkG);
  {
    ProfScope prof(ctx, kProfTopk);
    kern<<<grid, kTkThreads, kTkSmem, ctx->stream>>>(mqh, mql, mih, mil, (int)n_items, (int)n_query, k, q_exp, absmax, mask,
                                                     liked_indptr, liked_indices, out_ids, out_scores);
  }
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  return ALS_OK;
}

}  // namespace als
