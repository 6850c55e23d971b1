// R1, rows of more than 48 nonzeros at 64 padded factors: the normal equations on the Hopper tensor cores (wgmma)
// (reference: _least_squares, implicit/cpu/_als.pyx:76-142; the mma.sync kernel of cholesky.cu stays as the path for
// chunks of giant rows, finish items, CSRs with weights below 1 and the other factor widths).  Opt-in: knob long_tc.
//
//   A_u = (Y^T Y + lambda I) + sum_k w_k y_k y_k^T  with  w_k = |c_k| - 1 >= 0   is   G + Z^T Z,  Z = [sqrt(w_k) y_k]:
//   a GEMM whose operand rows are exactly what the gather produces.  One persistent CTA per SM, warp specialised:
//
//   producers (warpgroup 3)  take 32 nonzeros of the current row per ring stage: 16-byte cp.async copies of the
//                        gathered factor rows into a private landing zone (two halves of 16 rows: the next stage's
//                        gathers are in flight while this one is converted; its indices are fetched a stage ahead),
//                        scale by sigma sqrt(w), split into fp16 hi + lo (both rounded to nearest) and store the two
//                        32 x 64 tiles MN-major with the 128-byte swizzle -- a nonzero is one 128-byte row of the tile.
//                        b_u = sum c_k y_k rides along in fp32 (one partial per producer, summed in a fixed order);
//   MMA (warpgroup 2)    per 16 nonzeros two wgmma.m64nNk16.f16 with both operands MN-major:  hi^T [hi | lo]
//                        (N = 128) and lo^T hi (N = 64, onto the second half) into 64 fp32 registers per thread.  The
//                        large term hi^T hi has its own 64 columns, so the small terms never round into the large
//                        sums.  At the end of a row the warpgroup adds the halves and writes the matrix, with b_u, into
//                        the packed panel layout of the blocked Cholesky of one solver warp;
//   solvers (warpgroups 0, 1)  two groups of four warps, four rows per group and batch: every warp adds
//                        sigma^2 (Y^T Y + lambda I), factors and solves one row in registers (factor_solve of
//                        cholesky_device.cuh, shared with the mma.sync kernel) and stores x, also to the peer replicas.
// Rows are dealt to the CTAs round robin from the length-sorted work list, so all roles of a CTA walk the same
// sequence without talking to each other; the only synchronisation is mbarriers (stage full / free, b partials ready /
// consumed, solver panels full / free).  Deterministic: nothing depends on scheduling.  Registers are rebalanced with
// setmaxnreg: the solvers' warpgroups take 168 each, the MMA warpgroup 96 and the producers 80.
#include "cholesky_device.cuh"
#include "sm90.cuh"

namespace als {

namespace {

using namespace sm90;

constexpr int kTcF = 64;
constexpr int kTcStageNnz = 32;                     // nonzeros per ring stage
constexpr int kTcTile = kTcStageNnz * 128;          // one fp16 tile: 32 rows of 64 halves
constexpr int kTcStageBytes = 2 * kTcTile;          // hi | lo
constexpr int kTcStages = 8;
constexpr int kTcSlots = 4;                         // b partials in flight (rows)
constexpr int kTcSolvers = 8;
constexpr int kTcMmaWarp0 = kTcSolvers;             // warpgroup 2
constexpr int kTcProducerWarp0 = kTcSolvers + 4;    // warpgroup 3
constexpr int kTcProducers = 4;
constexpr int kTcThreads = 32 * (kTcSolvers + 4 + kTcProducers);
static_assert(kTcThreads == 512, "four warpgroups: setmaxnreg below assumes 128 registers per thread at launch");
static_assert(2 * 128 * 168 + 128 * 96 + 128 * 80 <= 65536, "setmaxnreg budget");
constexpr int kTcSolverFloats = Cfg<4>::U_FLOATS + kTcF;  // packed panels + rhs
constexpr int kTcOffRing = 0;
constexpr int kTcOffSolver = kTcStages * kTcStageBytes;
constexpr int kTcRawBytes = 2 * 16 * 256;           // per producer: two halves of 16 gathered fp32 rows (cp.async landing zone)
constexpr int kTcOffRaw = kTcOffSolver + kTcSolvers * kTcSolverFloats * 4;
constexpr int kTcOffBpart = kTcOffRaw + kTcProducers * kTcRawBytes;
constexpr int kTcOffBar = kTcOffBpart + kTcSlots * kTcProducers * kTcF * 4;
constexpr int kTcDone = 2 * kTcSlots;
enum { kTcFull = 0, kTcEmpty = kTcStages, kTcRowDone = 2 * kTcStages, kTcSlotFree = 2 * kTcStages + kTcDone,
       kTcPanelFull = kTcSlotFree + kTcSlots, kTcPanelFree = kTcPanelFull + 2, kTcNumBars = kTcPanelFree + 2 };
constexpr int kTcSmem = kTcOffBar + 8 * kTcNumBars + 16 + 1024;
static_assert(kTcSmem <= 227 * 1024, "shared memory budget");

__global__ void __launch_bounds__(kTcThreads, 1)
cholesky_tc_kernel(const int32_t *__restrict__ indices, const float *__restrict__ data, const float *__restrict__ Y,
                   float *__restrict__ X, int64_t row_offset, const float *__restrict__ Greg,
                   const WorkItem *__restrict__ work, int n_work, long long *bad_row, float *const *peers, int n_peers,
                   const unsigned *__restrict__ wmax_bits, const unsigned *__restrict__ yabsmax_bits) {
  using C = Cfg<4>;
  constexpr int F = kTcF;
  extern __shared__ unsigned char tc_smem_raw[];
  const uint32_t raw = smem_u32(tc_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  unsigned char *gbase = tc_smem_raw + (base - raw);
  const uint32_t bars = base + kTcOffBar;
  auto bar = [&](int i) -> uint32_t { return bars + 8u * (uint32_t)i; };
  float *bpart = reinterpret_cast<float *>(gbase + kTcOffBpart);
  float *panels = reinterpret_cast<float *>(gbase + kTcOffSolver);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 7, 0);  // warpgroup, visibly uniform to the compiler
  // this CTA's rows: work[blockIdx.x + n gridDim.x], n = 0 .. n_mine - 1
  const int n_mine = ((int)blockIdx.x < n_work) ? (n_work - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  auto load_item = [&](int n) -> WorkItem {
    const int4 v = __ldg(reinterpret_cast<const int4 *>(work) + ((int64_t)blockIdx.x + (int64_t)n * gridDim.x));
    return WorkItem{v.x, v.y, v.z, v.w};
  };
  const float sigma = pow2_scale_below_2_14(sqrtf(__uint_as_float(*wmax_bits)) * __uint_as_float(*yabsmax_bits));
  const float sigma2 = sigma * sigma;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kTcStages; ++i) {
      mbar_init(bar(kTcFull + i), 1);
      mbar_init(bar(kTcEmpty + i), 1);
    }
    for (int i = 0; i < kTcDone; ++i) mbar_init(bar(kTcRowDone + i), kTcProducers);
    for (int i = 0; i < kTcSlots; ++i) mbar_init(bar(kTcSlotFree + i), 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(bar(kTcPanelFull + i), 4);   // one arrival per row of a batch (MMA warpgroup)
      mbar_init(bar(kTcPanelFree + i), 4);   // one arrival per solver warp of the group
    }
    mbar_init_fence();
  }
  __syncthreads();

  if (wg == kTcProducerWarp0 / 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 80;");
      // ===== producers ==========================================================================================
      const int pw = warp - kTcProducerWarp0;
      const int hl = lane >> 4, cl = lane & 15;  // the row of a pair, the 16-byte word of the factor row
      unsigned char *rawb = gbase + kTcOffRaw + pw * kTcRawBytes;
      // This warp's stages are the CTA's stages G = pw, pw + P, pw + 2 P, ...  A cursor names one of them: the row n
      // (work item wi, nst stages), the stage s inside the row and G itself.
      struct Cursor {
        int n, s, nst, G;
        WorkItem wi;
      };
      auto stages_of = [&](const WorkItem &w) -> int {
        return (w.slot == -1) ? (w.k1 - w.k0 + kTcStageNnz - 1) / kTcStageNnz : 0;  // chunks of giant rows are not ours
      };
      auto settle = [&](Cursor &c) {  // move on to the row that holds stage c.s (counted from row c.n), or to the end
        while (c.n < n_mine && c.s >= c.nst) {
          c.s -= c.nst;
          ++c.n;
          if (c.n < n_mine) {
            c.wi = load_item(c.n);
            c.nst = stages_of(c.wi);
          }
        }
      };
      // index / confidence of this lane's nonzero of the stage under the cursor
      auto load_meta = [&](const Cursor &c, int &idx, float &cf) {
        const int k = c.wi.k0 + kTcStageNnz * c.s + lane;
        const bool valid = c.n < n_mine && k < c.wi.k1;
        idx = valid ? __ldg(indices + k) : -1;
        cf = valid ? __ldg(data + k) : 0.f;
      };
      // 16-byte cp.async gathers of half h (16 nonzeros) of a stage into this warp's landing zone; always one commit
      auto issue_half = [&](int idx, int h, bool active) {
        if (active) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int ir = __shfl_sync(0xffffffffu, idx, 16 * h + 2 * j + hl);
            if (ir >= 0)
              cp_async16(reinterpret_cast<float *>(rawb + h * 4096 + (2 * j + hl) * 256 + cl * 16), Y + (int64_t)ir * F + 4 * cl);
          }
        }
        cp_async_commit();
      };
      // finish row n for this producer: its share of b_u (zero when it had no stage in the row) and the hand-over
      auto finish_row = [&](int n, float4 bs) {
        const int slot = n % kTcSlots;
        bs.x += __shfl_xor_sync(0xffffffffu, bs.x, 16);
        bs.y += __shfl_xor_sync(0xffffffffu, bs.y, 16);
        bs.z += __shfl_xor_sync(0xffffffffu, bs.z, 16);
        bs.w += __shfl_xor_sync(0xffffffffu, bs.w, 16);
        if (n >= kTcSlots) mbar_wait(bar(kTcSlotFree + slot), (uint32_t)((n / kTcSlots - 1) & 1));
        if (lane < 16) *reinterpret_cast<float4 *>(bpart + (slot * kTcProducers + pw) * F + 4 * cl) = bs;
        __syncwarp();
        if (lane == 0) mbar_arrive(bar(kTcRowDone + n % kTcDone));
      };
      const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);

      Cursor cur;
      cur.n = 0;
      cur.s = pw;
      cur.G = pw;
      cur.nst = 0;
      cur.wi = WorkItem{0, 0, 0, -1};
      if (n_mine > 0) {
        cur.wi = load_item(0);
        cur.nst = stages_of(cur.wi);
      }
      settle(cur);
      int idx;
      float cf;
      load_meta(cur, idx, cf);
      int done_rows = 0;  // rows [0, done_rows) are finished
      for (; done_rows < min(cur.n, n_mine); ++done_rows) finish_row(done_rows, zero4);
      if (cur.n < n_mine) {
        const int nv = min(kTcStageNnz, cur.wi.k1 - (cur.wi.k0 + kTcStageNnz * cur.s));
        issue_half(idx, 0, true);
        issue_half(idx, 1, nv > 16);
      }
      float4 bs = zero4;
      while (cur.n < n_mine) {
        // the stage after this one: its indices are fetched now, its gathers are issued as soon as a half of the landing zone is free
        Cursor nxt = cur;
        nxt.s += kTcProducers;
        nxt.G += kTcProducers;
        settle(nxt);
        int nidx;
        float ncf;
        load_meta(nxt, nidx, ncf);
        const int nnv = (nxt.n < n_mine) ? min(kTcStageNnz, nxt.wi.k1 - (nxt.wi.k0 + kTcStageNnz * nxt.s)) : 0;

        const int rs = cur.G % kTcStages, use = cur.G / kTcStages;
        // A += w y y^T with w = |c| - 1 (>= 0 here: CSRs with smaller weights take the mma.sync kernel);
        // b += c y for c > 0   (_als.pyx:115-124)
        const float sw = (idx >= 0) ? sigma * __fsqrt_rn(fmaxf(fabsf(cf) - 1.f, 0.f)) : 0.f;
        const float cp = (idx >= 0 && cf > 0.f) ? cf : 0.f;
        unsigned char *hi = gbase + kTcOffRing + rs * kTcStageBytes, *lo = hi + kTcTile;
        if (use > 0) mbar_wait(bar(kTcEmpty + rs), (uint32_t)((use - 1) & 1));  // the MMAs of the previous use are done
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          cp_async_wait<1>();  // this half has landed (every lane reads back only what it copied itself)
          {  // an empty second half is written as zeros (invalid nonzeros read as zero): the MMAs always take 32 rows
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int r = 16 * h + 2 * j + hl;
              const int ir = __shfl_sync(0xffffffffu, idx, r);
              const float swr = __shfl_sync(0xffffffffu, sw, r), cpr = __shfl_sync(0xffffffffu, cp, r);
              float4 v = *reinterpret_cast<const float4 *>(rawb + h * 4096 + (2 * j + hl) * 256 + cl * 16);
              if (ir < 0) v = zero4;
              bs.x = fmaf(cpr, v.x, bs.x);
              bs.y = fmaf(cpr, v.y, bs.y);
              bs.z = fmaf(cpr, v.z, bs.z);
              bs.w = fmaf(cpr, v.w, bs.w);
              uint32_t h0, l0, h1, l1;
              split_f16_pair(swr * v.x, swr * v.y, h0, l0);
              split_f16_pair(swr * v.z, swr * v.w, h1, l1);
              const int off = r * 128 + (((cl >> 1) ^ (r & 7)) << 4) + (cl & 1) * 8;
              *reinterpret_cast<uint2 *>(hi + off) = make_uint2(h0, h1);
              *reinterpret_cast<uint2 *>(lo + off) = make_uint2(l0, l1);
            }
          }
          issue_half(nidx, h, nxt.n < n_mine && (h == 0 || nnv > 16));  // the landing zone of this half is free again
        }
        fence_proxy_async();  // generic-proxy stores -> the tensor core's reads
        __syncwarp();
        if (lane == 0) mbar_arrive(bar(kTcFull + rs));
        // rows that end between this stage and the next one of this warp
        if (nxt.n != cur.n) {
          finish_row(done_rows++, bs);
          bs = zero4;
          for (; done_rows < min(nxt.n, n_mine); ++done_rows) finish_row(done_rows, zero4);
        }
        cur = nxt;
        idx = nidx;
        cf = ncf;
      }
      cp_async_wait<0>();
  } else if (wg == kTcMmaWarp0 / 4) {
    // ===== MMA warpgroup: accumulate a row in registers, drain it into a solver panel ===========================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 96;");
    const int t = threadIdx.x - 32 * kTcMmaWarp0;  // 0 .. 127
    int G = 0;
    const int n_batched = (n_mine + 3) & ~3;      // whole batches of four rows: the solver groups count four arrivals
    for (int n = 0; n < n_batched; ++n) {
      const int B = n >> 2, e = B & 1, j = n & 3;
      if (j == 0 && B >= 2) mbar_wait(bar(kTcPanelFree + e), (uint32_t)(((B >> 1) - 1) & 1));  // batch B - 2 is solved
      if (n < n_mine) {
        const WorkItem wi = load_item(n);
        const int nnz = (wi.slot == -1) ? wi.k1 - wi.k0 : 0;
        const int nst = (nnz + kTcStageNnz - 1) / kTcStageNnz;
        const int slot = n % kTcSlots;
        float d[64];
        float(&d_small)[32] = *reinterpret_cast<float(*)[32]>(&d[32]);  // columns 64..127 of the accumulator
#pragma unroll
        for (int v = 0; v < 64; ++v) d[v] = 0.f;
        for (int s = 0; s < nst; ++s, ++G) {
          const int rs = G % kTcStages;
          mbar_wait(bar(kTcFull + rs), (uint32_t)((G / kTcStages) & 1));
          const uint32_t hi = base + kTcOffRing + rs * kTcStageBytes, lo = hi + kTcTile;
          wgmma_fence();
          // [hi^T hi | hi^T lo]: B spans the hi tile and, one LBO (kTcTile bytes) on, the lo tile; then + lo^T hi
          wgmma_f16_mn_m64n128k16(d, wgmma_desc_mn_sw128(hi, kTcTile), wgmma_desc_mn_sw128(hi, kTcTile), s > 0);
          wgmma_f16_mn_m64n64k16(d_small, wgmma_desc_mn_sw128(lo, kTcTile), wgmma_desc_mn_sw128(hi, kTcTile), 1);
          // second 16 nonzeros (zero rows where the stage holds fewer)
          wgmma_f16_mn_m64n128k16(d, wgmma_desc_mn_sw128(hi + 2048, kTcTile), wgmma_desc_mn_sw128(hi + 2048, kTcTile), 1);
          wgmma_f16_mn_m64n64k16(d_small, wgmma_desc_mn_sw128(lo + 2048, kTcTile), wgmma_desc_mn_sw128(hi + 2048, kTcTile), 1);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_operand(d);
          if (t == 0) mbar_arrive(bar(kTcEmpty + rs));  // the stage may be refilled
        }
        mbar_wait(bar(kTcRowDone + n % kTcDone), (uint32_t)((n / kTcDone) & 1));  // every producer's b partial is in
        if (wi.slot == -1 && wi.k1 > wi.k0) {
          float *Uj = panels + (4 * e + j) * kTcSolverFloats;
#pragma unroll
          for (int v = 0; v < 32; v += 2) {
            // accumulator row m -> panel m / 8, columns >= 8 (m / 8): large term + small terms
            const int m = wgmma_row(t, v), col = wgmma_col(t, v);
            const int pm = m >> 3;
            const int po = 8 * (pm * F - 4 * pm * (pm - 1) + 8 * ((pm + 1) >> 1));
            const int ps = F - 8 * pm + ((pm & 1) ? 0 : 8);
            if (col >= 8 * pm)
              *reinterpret_cast<float2 *>(Uj + po + (m & 7) * ps - 8 * pm + col) = make_float2(d[v] + d[v + 32], d[v + 1] + d[v + 33]);
          }
          if (t < F) {  // b_u: the producers' partials in a fixed order
            float b = 0.f;
#pragma unroll
            for (int p = 0; p < kTcProducers; ++p) b += bpart[(slot * kTcProducers + p) * F + t];
            Uj[C::U_FLOATS + t] = b;
          }
        }
        named_sync(3, 128);  // the panel is written and the b partials are read
        if (t == 0) mbar_arrive(bar(kTcSlotFree + slot));
      }
      if (t == 0) mbar_arrive(bar(kTcPanelFull + e));
    }
  } else {
    // ===== solvers ============================================================================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 168;");
    const int e = warp >> 2, q = warp & 3;
    const int g = lane >> 2, t = lane & 3;
    float *Uown = panels + warp * kTcSolverFloats;
    float *zown = Uown + C::U_FLOATS;
    for (int B = e; 4 * B < n_mine; B += 2) {
      mbar_wait(bar(kTcPanelFull + e), (uint32_t)((B >> 1) & 1));  // the group's four matrices are in shared memory
      const int n = 4 * B + q;
      if (n < n_mine) {
        const WorkItem wi = load_item(n);
        const int64_t xoff = (row_offset + wi.row) * F;
        if (wi.slot == -1 && wi.k0 == wi.k1) {
          // no observations: the reference zeroes the row (_als.pyx:98-100)
          for (int m = lane; m < F; m += 32) {
            X[xoff + m] = 0.f;
            for (int pi = 0; pi < n_peers; ++pi) peers[pi][xoff + m] = 0.f;
          }
        } else if (wi.slot == -1) {
          RowState<4> st;
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 2 * i; j < C::NT8; ++j) {
              float(&d)[4] = st.acc[C::tidx(i, j)];
              const float2 gt = __ldg(reinterpret_cast<const float2 *>(Greg + (16 * i + g) * F + 8 * j + 2 * t));
              const float2 gb = __ldg(reinterpret_cast<const float2 *>(Greg + (16 * i + g + 8) * F + 8 * j + 2 * t));
              const float2 at = *reinterpret_cast<const float2 *>(Uown + C::poff(2 * i) + g * C::pstride(2 * i) + 8 * (j - 2 * i) + 2 * t);
              d[0] = fmaf(sigma2, gt.x, at.x);
              d[1] = fmaf(sigma2, gt.y, at.y);
              if (j >= 2 * i + 1) {
                const float2 ab = *reinterpret_cast<const float2 *>(Uown + C::poff(2 * i + 1) + g * C::pstride(2 * i + 1) +
                                                                    8 * (j - 2 * i - 1) + 2 * t);
                d[2] = fmaf(sigma2, gb.x, ab.x);
                d[3] = fmaf(sigma2, gb.y, ab.y);
              } else {
                d[2] = d[3] = 0.f;  // below the diagonal: never read
              }
            }
#pragma unroll
          for (int c = 0; c < C::NT8; ++c) st.bp[c] = (t == 0) ? sigma2 * zown[8 * c + g] : 0.f;  // (sigma^2 A) x = sigma^2 b
          __syncwarp();
          bool ok = true;
          float xx[(F + 31) / 32];
          factor_solve<4>(st, Uown, zown, lane, ok, 0, xx);
          if (ok) store_solution<F>(xx, X + xoff, lane, peers, n_peers, xoff);
          if (!ok && lane == 0) atomicMin(bad_row, (long long)(row_offset + wi.row));
          __syncwarp();
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar(kTcPanelFree + e));  // this warp's panel buffer is free for batch B + 2
    }
  }
}

}  // namespace

bool cholesky_tc_eligible(const als_ctx *ctx, const als_csr *C, int ld) {
  return ld == kTcF && ctx->knobs.long_tc && C->neg_w_known && !C->has_neg_w;
}

// items [0, n_items) of C->work that are whole rows (chunk items of giant rows are skipped: the caller runs the mma.sync
// kernel over C->chunks); needs ctx->Greg, the weight range of the whole matrix (wmax_dev: C is one of its segments) and
// max |y| in counters[kCtrYAbsMax]
int launch_cholesky_tc(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y, int64_t n_items,
                       const unsigned *wmax_dev, cudaStream_t stream) {
  if (n_items <= 0) return ALS_OK;
  static bool attr_done = false;
  if (!attr_done) {
    ALS_CUDA(cudaFuncSetAttribute(cholesky_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTcSmem));
    attr_done = true;
  }
  const int grid = (int)std::min<int64_t>(n_items, ctx->sm_count);
  cholesky_tc_kernel<<<grid, kTcThreads, kTcSmem, stream>>>(
      C->indices, C->data, Y->d, X->d, C->row_offset, ctx->Greg, C->work, (int)n_items, ctx->bad_row, X->peers_dev, X->n_peers,
      wmax_dev, reinterpret_cast<const unsigned *>(ctx->counters + kCtrYAbsMax));
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  return ALS_OK;
}

}  // namespace als
