// Dense "apply" on the Hopper tensor cores: OUT[rows x 128] = Y[rows x 64] * B[64 x 128], fp32-faithful.
//
// This is the one true dense contraction on the Cholesky half besides the Gramian: the whitened factors
// W = Y (2^14 P) and the solved factors Z = Y G^-1 of the short-row path (cholesky_short.cu) are two
// rows x 64 x 64 products over the same Y, so B = [2^14 P | G^-1] and one pass over Y produces both.
// (The reference has no counterpart: it solves every row with the F x F normal equations, _als.pyx:96-130; the
// Gramian it precomputes, _als.pyx:70, is what P and G^-1 are derived from.)
//
// Data path, one persistent CTA per SM with two warpgroups, each owning 64 rows of every 128-row tile:
//   thread 0    TMA: cp.async.bulk.tensor (128B-swizzled 128 x 32-float boxes) of the Y tiles into a 2-stage ring
//               (the next tile is in flight while this one is multiplied), mbarrier complete_tx; B (hi and lo parts,
//               K-major) is loaded once per CTA;
//   warpgroup   splits its 64 landed rows in place into their TF32-rounded hi part and the exact remainder lo, then
//               issues wgmma.m64n128k8.tf32: three products per k-step (hi*hi + lo*hi + hi*lo, the 3xTF32 split),
//               24 wgmmas per tile, accumulators in registers; stages them 128B-swizzled in shared memory (W as fp16
//               hi / lo pairs, the operand format of the short-row kernel's mma.sync.m16n8k16; Z as fp32) and hands
//               them to TMA stores, which drain while the next tile is multiplied.
// The kernel is bound by HBM (96 KB per 128 rows).
#include <cuda.h>
#include <cuda_fp16.h>

#include "common.h"
#include "sm90.cuh"

namespace als {

namespace {

using namespace sm90;

constexpr int kDenseF = 64;        // K: padded factors (the short-row path is only used for F = 64 here)
constexpr int kDenseN = 128;       // N: [W | Z]
constexpr int kTileM = 128;
constexpr int kBoxBytes = kTileM * 128;          // one 128-row x 32-float box, 128B swizzle
constexpr int kAStage = 2 * kBoxBytes;           // both K halves of a Y tile
constexpr int kDenseThreads = 256;               // two warpgroups
constexpr int kOutBox = 64 * 128;                // one 64-row x 32-float output box

// shared memory map (bytes from a 1024-aligned base)
constexpr int kOffA = 0;                          // 2 stages x 32 KB: raw tile, split in place into its hi part
constexpr int kOffALo = kOffA + 2 * kAStage;      // 32 KB
constexpr int kOffBHi = kOffALo + kAStage;        // 32 KB
constexpr int kOffBLo = kOffBHi + kAStage;        // 32 KB
constexpr int kOffOut = kOffBLo + kAStage;        // per warpgroup 4 output boxes (W words 0-31, 32-63, Z 0-31, 32-63)
constexpr int kOffBar = kOffOut + 2 * 4 * kOutBox;  // mbarriers
constexpr int kDenseSmem = kOffBar + 128 + 1024;  // + slack for the 1024-byte alignment
static_assert(kDenseSmem <= 227 * 1024, "dense apply: more shared memory than a Hopper block may have");

enum { kBarFull0 = 0, kBarFull1, kBarB, kNumBars };

// hi = x rounded to nearest TF32 (low 13 bits cleared), lo = x - hi exactly (the tensor core drops lo's last bits)
__device__ __forceinline__ void split4(float4 x, float4 &hi, float4 &lo) {
  hi.x = __uint_as_float((__float_as_uint(x.x) + 0x1000u) & 0xffffe000u);
  hi.y = __uint_as_float((__float_as_uint(x.y) + 0x1000u) & 0xffffe000u);
  hi.z = __uint_as_float((__float_as_uint(x.z) + 0x1000u) & 0xffffe000u);
  hi.w = __uint_as_float((__float_as_uint(x.w) + 0x1000u) & 0xffffe000u);
  lo.x = x.x - hi.x;
  lo.y = x.y - hi.y;
  lo.z = x.z - hi.z;
  lo.w = x.w - hi.w;
}

// byte offset of float column c (0..31) of row r in a 128B-swizzled box of 128-byte rows
__device__ __forceinline__ int sw128(int r, int c) { return r * 128 + ((((c >> 2) ^ (r & 7))) << 4) + ((c & 3) << 2); }

__global__ void __launch_bounds__(kDenseThreads, 1)
dense_apply_kernel(const __grid_constant__ CUtensorMap map_y, const __grid_constant__ CUtensorMap map_bhi,
                   const __grid_constant__ CUtensorMap map_blo, const __grid_constant__ CUtensorMap map_w,
                   const __grid_constant__ CUtensorMap map_z, int n_tiles) {
  extern __shared__ unsigned char dense_smem_raw[];
  const uint32_t raw = smem_u32(dense_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  unsigned char *gbase = dense_smem_raw + (base - raw);
  const uint32_t bars = base + kOffBar;
  auto bar = [&](int i) -> uint32_t { return bars + 8u * (uint32_t)i; };
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int my_tiles = (n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;  // tiles blockIdx.x + i gridDim.x
  auto tile_row0 = [&](int i) { return ((int)blockIdx.x + i * (int)gridDim.x) * kTileM; };

  if (threadIdx.x == 0) {
    mbar_init(bar(kBarFull0), 1);
    mbar_init(bar(kBarFull1), 1);
    mbar_init(bar(kBarB), 1);
    mbar_init_fence();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar(kBarB), 2 * kAStage);
    tma_load_2d(base + kOffBHi, &map_bhi, bar(kBarB), 0, 0);
    tma_load_2d(base + kOffBHi + kBoxBytes, &map_bhi, bar(kBarB), 32, 0);
    tma_load_2d(base + kOffBLo, &map_blo, bar(kBarB), 0, 0);
    tma_load_2d(base + kOffBLo + kBoxBytes, &map_blo, bar(kBarB), 32, 0);
    for (int i = 0; i < 2 && i < my_tiles; ++i) {
      mbar_expect_tx(bar(kBarFull0 + i), kAStage);
      tma_load_2d(base + kOffA + i * kAStage, &map_y, bar(kBarFull0 + i), 0, tile_row0(i));
      tma_load_2d(base + kOffA + i * kAStage + kBoxBytes, &map_y, bar(kBarFull0 + i), 32, tile_row0(i));
    }
  }
  mbar_wait(bar(kBarB), 0);
  unsigned char *out = gbase + kOffOut + wg * 4 * kOutBox;
  for (int i = 0; i < my_tiles; ++i) {
    const int s = i & 1;
    mbar_wait(bar(kBarFull0 + s), (uint32_t)((i >> 1) & 1));
    // split this warpgroup's 64 rows (8 KB of each K-half box) in place; the swizzle is the same for both buffers
#pragma unroll 4
    for (int e = t; e < 2 * 64 * 8; e += 128) {
      const int off = (e >> 9) * kBoxBytes + wg * 64 * 128 + (e & 511) * 16;
      float4 *a = reinterpret_cast<float4 *>(gbase + kOffA + s * kAStage + off);
      float4 hi, lo;
      split4(*a, hi, lo);
      *a = hi;
      *reinterpret_cast<float4 *>(gbase + kOffALo + off) = lo;
    }
    fence_proxy_async();
    named_sync(1 + wg, 128);
    float d[64] = {};
    const uint32_t a_hi = base + kOffA + s * kAStage + wg * 64 * 128, a_lo = base + kOffALo + wg * 64 * 128;
    const uint32_t b_hi = base + kOffBHi, b_lo = base + kOffBLo;
    wgmma_fence();
#pragma unroll
    for (int term = 0; term < 3; ++term) {  // lo * hi, hi * lo, hi * hi (small terms first)
      const uint32_t a0 = term == 0 ? a_lo : a_hi;
      const uint32_t b0 = term == 1 ? b_lo : b_hi;
#pragma unroll
      for (int ks = 0; ks < kDenseF / 8; ++ks) {
        const uint32_t off = (uint32_t)((ks >> 2) * kBoxBytes + (ks & 3) * 32);
        wgmma_tf32_m64n128k8(d, wgmma_desc_k_sw128(a0 + off), wgmma_desc_k_sw128(b0 + off), term + ks > 0);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operand(d);
    __syncthreads();  // both warpgroups are done with stage s: refill it with tile i + 2
    if (threadIdx.x == 0 && i + 2 < my_tiles) {
      mbar_expect_tx(bar(kBarFull0 + s), kAStage);
      tma_load_2d(base + kOffA + s * kAStage, &map_y, bar(kBarFull0 + s), 0, tile_row0(i + 2));
      tma_load_2d(base + kOffA + s * kAStage + kBoxBytes, &map_y, bar(kBarFull0 + s), 32, tile_row0(i + 2));
    }
    // epilogue: the staging boxes must have been read by the previous tile's TMA stores
    if (t == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    named_sync(1 + wg, 128);
#pragma unroll
    for (int v = 0; v < 64; v += 2) {
      const int r = wgmma_row(t, v), c = wgmma_col(t, v);  // c even: the pair (c, c + 1)
      if (c < kDenseF) {
        // W leaves in the split format the short-row kernel multiplies with (cholesky_short.cu): per 16 dimensions
        // 8 words of fp16 pairs "hi" and 8 words "lo"
        const __half2 h = __floats2half2_rn(d[v], d[v + 1]);
        const float2 hf = __half22float2(h);
        const __half2 lo = __floats2half2_rn(d[v] - hf.x, d[v + 1] - hf.y);
        const int m = c >> 1, w = 16 * (m >> 3) + (m & 7);
        *reinterpret_cast<__half2 *>(out + (w >> 5) * kOutBox + sw128(r, w & 31)) = h;
        *reinterpret_cast<__half2 *>(out + ((w + 8) >> 5) * kOutBox + sw128(r, (w + 8) & 31)) = lo;
      } else {
        const int z = c - kDenseF;
        *reinterpret_cast<float2 *>(out + (2 + (z >> 5)) * kOutBox + sw128(r, z & 31)) = make_float2(d[v], d[v + 1]);
      }
    }
    fence_proxy_async();
    named_sync(1 + wg, 128);
    if (t == 0) {
      const int row0 = tile_row0(i) + 64 * wg;
      const uint32_t ob = base + kOffOut + wg * 4 * kOutBox;
      tma_store_2d(&map_w, ob, 0, row0);
      tma_store_2d(&map_w, ob + kOutBox, 32, row0);
      tma_store_2d(&map_z, ob + 2 * kOutBox, 0, row0);
      tma_store_2d(&map_z, ob + 3 * kOutBox, 32, row0);
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
  }
  if (t == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// B^T = [2^14 P | G^-1]^T (128 x 64, K-major) split into its TF32-rounded hi part and the remainder
__global__ void dense_prepare_b_kernel(const float *__restrict__ Ps, const float *__restrict__ Ginv, float *__restrict__ bt_hi,
                                       float *__restrict__ bt_lo) {
  for (int e = threadIdx.x + blockIdx.x * blockDim.x; e < kDenseN * kDenseF; e += blockDim.x * gridDim.x) {
    const int n = e / kDenseF, k = e % kDenseF;
    const float x = n < kDenseF ? Ps[k * kDenseF + n] : Ginv[k * kDenseF + (n - kDenseF)];
    const float hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
    bt_hi[e] = hi;
    bt_lo[e] = x - hi;
  }
}

// ---- Gramian G = Y^T Y on the tensor cores (R4; reference: np.dot(Y.T, Y), implicit/cpu/_als.pyx:70,164,268) -------
// The contraction runs over the ROWS of Y, so both operands are the transposed tile.  The first warpgroup, which has
// to touch every element anyway for the TF32 hi / lo split, writes the split halves TRANSPOSED into a K-major,
// 128B-swizzled operand tile T = [hi^T ; lo^T] (128 operand rows = 64 factors hi + 64 factors lo, K = the 128 rows of
// the landed Y tile): A = hi^T (M = 64) and B = T (N = 128) start at the same address, and one wgmma.m64n128k8.tf32
// per 8 rows of Y yields hi^T hi (columns 0..63) and hi^T lo (columns 64..127) at once; lo^T hi is the transpose of
// the second block and is added at the end: G = S1 + S2 + S2^T (the 3xTF32 split at two thirds of the tensor work).
// Per CTA: thread 0 issues the TMA loads (128-row tiles, 2 stages), warpgroup 0 splits and transposes, warpgroup 1
// multiplies (T is double buffered, so tile t + 1 is transposed while tile t is multiplied).  The 64 x 128 sum is
// written once, as this CTA's partial; partials are summed in fp64 in a fixed order.
constexpr int kGramRaw = 2 * kBoxBytes;           // a landed Y tile: cols 0-31 | cols 32-63
constexpr int kGramT = 4 * kBoxBytes;             // [128 operand rows][128 K] as 4 K-chunks of 32
constexpr int kGramOffT = 2 * kGramRaw;           // after the 2 raw stages
constexpr int kGramOffBar = kGramOffT + 2 * kGramT;
constexpr int kGramSmem = kGramOffBar + 128 + 1024;
static_assert(kGramSmem <= 227 * 1024, "Gramian: more shared memory than a Hopper block may have");
enum { kGFull0 = 0, kGFull1, kGReady0, kGReady1, kGTFree0, kGTFree1, kGNumBars };

// A chain is kept to 8 MMAs = 64 rows of Y and each finished chain is added into fp32 registers with ordinary
// round-to-nearest additions, so that a tensor core that truncates while it accumulates (measured on the previous
// generation's tensor cores; not measured on H100's wgmma) cannot bias a long all-positive sum.
__global__ void __launch_bounds__(kDenseThreads, 1)
gramian_tc_kernel(const __grid_constant__ CUtensorMap map_y, int n_tiles, float *__restrict__ partials) {
  extern __shared__ unsigned char dense_smem_raw[];
  const uint32_t raw = smem_u32(dense_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  unsigned char *gbase = dense_smem_raw + (base - raw);
  const uint32_t bars = base + kGramOffBar;
  auto bar = [&](int i) -> uint32_t { return bars + 8u * (uint32_t)i; };
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int my_tiles = (n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  auto tile_row0 = [&](int i) { return ((int)blockIdx.x + i * (int)gridDim.x) * kTileM; };

  if (threadIdx.x == 0) {
    mbar_init(bar(kGFull0), 1);
    mbar_init(bar(kGFull1), 1);
    mbar_init(bar(kGReady0), 128);
    mbar_init(bar(kGReady1), 128);
    mbar_init(bar(kGTFree0), 128);
    mbar_init(bar(kGTFree1), 128);
    mbar_init_fence();
  }
  __syncthreads();

  float racc[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) racc[j] = 0.f;
  if (wg == 0) {
    // ===== split + transpose the landed tile into the operand tile =====
    if (t == 0)
      for (int i = 0; i < 2 && i < my_tiles; ++i) {
        mbar_expect_tx(bar(kGFull0 + i), kGramRaw);
        tma_load_2d(base + i * kGramRaw, &map_y, bar(kGFull0 + i), 0, tile_row0(i));
        tma_load_2d(base + i * kGramRaw + kBoxBytes, &map_y, bar(kGFull0 + i), 32, tile_row0(i));
      }
    const int w4 = t >> 5, lane = t & 31;  // K-chunk of the operand tile = rows 32 w4 .. 32 w4 + 31 of the Y tile
    const int r = t;                       // this thread's row of the Y tile
    for (int i = 0; i < my_tiles; ++i) {
      const int s = i & 1;
      mbar_wait(bar(kGFull0 + s), (uint32_t)((i >> 1) & 1));
      if (i >= 2) mbar_wait(bar(kGTFree0 + s), (uint32_t)(((i >> 1) - 1) & 1));  // the MMAs of tile i - 2 have read T[s]
      const unsigned char *src = gbase + s * kGramRaw;
      unsigned char *dst = gbase + kGramOffT + s * kGramT + w4 * kBoxBytes;
#pragma unroll 4
      for (int c4 = 0; c4 < 16; ++c4) {
        // 4 consecutive columns of row r: the 16-byte chunk (c4 % 8) of box (c4 / 8), swizzled with r % 8
        const float4 x = *reinterpret_cast<const float4 *>(src + (c4 >> 3) * kBoxBytes + r * 128 + (((c4 & 7) ^ (r & 7)) << 4));
        float4 hi, lo;
        split4(x, hi, lo);
        const float h[4] = {hi.x, hi.y, hi.z, hi.w}, l[4] = {lo.x, lo.y, lo.z, lo.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c = 4 * c4 + j;  // operand row c (hi) / 64 + c (lo); K index within the chunk = lane
          const int off = (((lane >> 2) ^ (c & 7)) << 4) + ((lane & 3) << 2);  // (64 + c) % 8 == c % 8
          *reinterpret_cast<float *>(dst + c * 128 + off) = h[j];
          *reinterpret_cast<float *>(dst + (64 + c) * 128 + off) = l[j];
        }
      }
      fence_proxy_async();
      mbar_arrive(bar(kGReady0 + s));
      named_sync(1, 128);  // every thread has read raw stage s: refill it with tile i + 2
      if (t == 0 && i + 2 < my_tiles) {
        mbar_expect_tx(bar(kGFull0 + s), kGramRaw);
        tma_load_2d(base + s * kGramRaw, &map_y, bar(kGFull0 + s), 0, tile_row0(i + 2));
        tma_load_2d(base + s * kGramRaw + kBoxBytes, &map_y, bar(kGFull0 + s), 32, tile_row0(i + 2));
      }
    }
  } else {
    // ===== multiply: two chains of 8 wgmmas per tile, each added into racc =====
    for (int i = 0; i < my_tiles; ++i) {
      const int s = i & 1;
      mbar_wait(bar(kGReady0 + s), (uint32_t)((i >> 1) & 1));
      const uint32_t T = base + kGramOffT + s * kGramT;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float d[64] = {};
        wgmma_fence();
#pragma unroll
        for (int k8 = 0; k8 < 8; ++k8) {
          const int ks = 8 * h + k8;  // 8 rows of Y (the K extent of a tf32 MMA) per instruction
          const uint64_t desc = wgmma_desc_k_sw128(T + (uint32_t)((ks >> 2) * kBoxBytes + (ks & 3) * 32));
          wgmma_tf32_m64n128k8(d, desc, desc, k8);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operand(d);
#pragma unroll
        for (int j = 0; j < 64; ++j) racc[j] += d[j];
      }
      mbar_arrive(bar(kGTFree0 + s));
    }
  }
  __syncthreads();  // every TMA load has landed and been read: raw stage 0 is free
  if (wg == 1) {
    // partial of this CTA, symmetrised: P = S1 + S2 + S2^T (S2^T through shared memory)
    float *s2 = reinterpret_cast<float *>(gbase);  // [64][65]
#pragma unroll
    for (int v = 32; v < 64; ++v) s2[wgmma_row(t, v) * 65 + wgmma_col(t, v) - 64] = racc[v];
    named_sync(2, 128);
    float *out = partials + (size_t)blockIdx.x * 64 * 64;
#pragma unroll
    for (int v = 0; v < 32; ++v) {
      const int r = wgmma_row(t, v), c = wgmma_col(t, v);
      out[r * 64 + c] = racc[v] + (racc[v + 32] + s2[c * 65 + r]);
    }
  }
}

typedef sm90::EncodeTiledFn EncodeTiledFn;

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// rows x 64 fp32 row-major matrix, boxes of `box_rows` rows x 32 floats, 128B swizzle
int make_map(CUtensorMap *m, const float *ptr, int64_t rows, int box_rows = kTileM) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) {
    set_error("dense: cuTensorMapEncodeTiled is not available from this driver");
    return ALS_E_CUDA;
  }
  const cuuint64_t dims[2] = {(cuuint64_t)kDenseF, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)kDenseF * sizeof(float)};
  const cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float *>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("dense: cuTensorMapEncodeTiled failed with %d", (int)r);
    return ALS_E_CUDA;
  }
  return ALS_OK;
}

}  // namespace

// W = Y (2^14 P) and Z = Y G^-1 for a 64-wide Y, from ctx->Pinv / ctx->Ginv into ctx->whitened / ctx->zfactors
int launch_dense_whiten(als_ctx *ctx, const als_factors *Y, cudaStream_t stream) {
  if (Y->ld != kDenseF) {
    set_error("dense: only %d padded factors are supported (got %d)", kDenseF, Y->ld);
    return ALS_E_UNSUPPORTED;
  }
  if (!ctx->dense_bt) ALS_CUDA(cudaMalloc(&ctx->dense_bt, 2 * kDenseN * kDenseF * sizeof(float)));
  float *bt_hi = ctx->dense_bt, *bt_lo = ctx->dense_bt + kDenseN * kDenseF;
  dense_prepare_b_kernel<<<8, 256, 0, stream>>>(ctx->Pinv, ctx->Ginv, bt_hi, bt_lo);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  const int64_t rows = std::max<int64_t>(Y->rows, 1);
  CUtensorMap my, mbh, mbl, mw, mz;
  int rc;
  if ((rc = make_map(&my, Y->d, rows)) != ALS_OK) return rc;
  if ((rc = make_map(&mbh, bt_hi, kDenseN)) != ALS_OK) return rc;
  if ((rc = make_map(&mbl, bt_lo, kDenseN)) != ALS_OK) return rc;
  if ((rc = make_map(&mw, ctx->whitened, rows, 64)) != ALS_OK) return rc;
  if ((rc = make_map(&mz, ctx->zfactors, rows, 64)) != ALS_OK) return rc;
  const int n_tiles = (int)ceil_div(rows, kTileM);
  const int grid = std::min(n_tiles, ctx->sm_count);
  ALS_CUDA(cudaFuncSetAttribute(dense_apply_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kDenseSmem));
  dense_apply_kernel<<<grid, kDenseThreads, kDenseSmem, stream>>>(my, mbh, mbl, mw, mz, n_tiles);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  return ALS_OK;
}

// G = Y^T Y for a 64-wide Y on the tensor cores (wgmma) -> ctx->G (the caller regularises)
int launch_gramian_tc(als_ctx *ctx, const als_factors *Y) {
  const int64_t rows = std::max<int64_t>(Y->rows, 1);
  const int n_tiles = (int)ceil_div(rows, kTileM);
  const int grid = std::min(n_tiles, ctx->sm_count);
  const int64_t need = (int64_t)sizeof(float) * grid * 64 * 64;
  int rc = ALS_OK;
  if (need > ctx->gram_partials_cap &&
      (rc = ensure_device_buffer(ctx, (void **)&ctx->gram_partials, &ctx->gram_partials_cap,
                                 (int64_t)sizeof(float) * ctx->sm_count * 2 * 128 * 128)) != ALS_OK)
    return rc;
  CUtensorMap my;
  if ((rc = make_map(&my, Y->d, rows)) != ALS_OK) return rc;
  ALS_CUDA(cudaFuncSetAttribute(gramian_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kGramSmem));
  gramian_tc_kernel<<<grid, kDenseThreads, kGramSmem, ctx->stream>>>(my, n_tiles, ctx->gram_partials);
  ALS_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return launch_gramian_reduce(ctx, grid, 64 * 64);  // partials summed in fp64 in a fixed order (gramian.cu)
}

}  // namespace als
