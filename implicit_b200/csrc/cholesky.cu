// R1: fused Cholesky half-iteration (reference: _least_squares, implicit/cpu/_als.pyx:76-142).
//
// One warp owns one row u of the CSR at a time (persistent warps pull rows, longest first, from an
// atomic work counter):
//   gather   the factor rows Y[i] of the row's nonzeros are staged 16 at a time (one k-step) into shared
//            memory with 16-byte cp.async copies (Cfg16: 2 stages per warp, the next row's first two
//            k-steps issued before this row is factored; indices / confidences are prefetched 32 at a
//            time into registers one block ahead);
//   A, b     A_u = (Y^T Y + lambda I) + sum_k (|c_k| - 1) y_k y_k^T is accumulated in REGISTERS as the
//            upper-triangular set of 16x8 mma.sync.m16n8k16 tiles on the fp16 split of sigma sqrt|w| y
//            (hi*hi + hi*lo + lo*hi, both parts rounded to nearest), i.e. as sigma^2 A_u with sigma a
//            power of two chosen per half (DESIGN 4.1); b_u = sum_{c_k > 0} c_k y_k rides along in fp32
//            FMAs;
//   solve    a right-looking blocked Cholesky with 8-row panels: each panel is spilled to shared
//            memory, one lane owns one panel column (the rhs slice and 8 unit vectors ride along as
//            extra columns), the 8 pivots are eliminated LDL^T-style with warp shuffles and the rows
//            scaled by 1/sqrt(d) afterwards; the trailing matrix is updated IN REGISTERS by 3xTF32
//            m16n8k8 tiles; the back substitution resolves a panel at a time with the inverse of
//            its diagonal block (the forward-substituted unit vectors) on the packed U in shared memory.
// Giant rows are split into chunks whose partial (A, b) go to global scratch and are summed in a
// fixed order by a second "finish" launch, so results do not depend on scheduling.
#include "cholesky_device.cuh"

namespace als {

namespace {

// ---- kernel ------------------------------------------------------------------------------------
// pass 0: whole rows and chunks of giant rows;  pass 1: finish giant rows from their chunk slots.
#ifndef ALS_LONG_MIN_BLOCKS
#define ALS_LONG_MIN_BLOCKS 11  // one-warp CTAs per SM the register allocation aims at (variants: tools/build_variant.sh)
#endif
template <int NB>
__global__ void __launch_bounds__(32 * kWarpsPerCta, ALS_LONG_MIN_BLOCKS)
cholesky_half_kernel(const int32_t *__restrict__ indices, const float *__restrict__ data, const float *__restrict__ Y,
                     float *__restrict__ X, int64_t row_offset, const float *__restrict__ Greg,
                     const WorkItem *__restrict__ work, int n_work, const int32_t *n_work_dev, int32_t *counter,
                     float *slots, long long *bad_row, int pass, int dbg_arg, float *const *peers, int n_peers,
                     const unsigned *__restrict__ wmax_bits, const unsigned *__restrict__ yabsmax_bits) {
#ifdef ALS_B200_ABLATE
  const int dbg = dbg_arg;
#else
  constexpr int dbg = 0;
  (void)dbg_arg;
#endif
  using C = Cfg<NB>;
  using C16 = Cfg16<NB>;
  constexpr int F = C::F;
  if (n_work_dev) n_work = *n_work_dev;  // a list built on the device (items deferred by the short-row kernels)
  extern __shared__ __align__(16) float smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  float *wsm = smem + warp * C16::WARP_FLOATS;
  float *stages = wsm;
  float *U = wsm + C16::NSTAGE * C16::STAGE_FLOATS;
  float *zb = U + C::U_FLOATS;
  // sigma: the power of two that brings the largest sqrt|w| |y| of this half just below 2^14 (fp16 operands)
  const float sigma = pow2_scale_below_2_14(sqrtf(__uint_as_float(*wmax_bits)) * __uint_as_float(*yabsmax_bits));
  const float sigma2 = sigma * sigma, inv_sigma2 = 1.f / sigma2;  // exact: powers of two

  auto fetch = [&]() -> int {
    int v = 0;
    if (lane == 0) v = atomicAdd(counter, 1);
    v = __shfl_sync(0xffffffffu, v, 0);
    return v < n_work ? v : -1;
  };
  auto load_item = [&](int i) -> WorkItem {
    const int4 v = __ldg(reinterpret_cast<const int4 *>(work) + i);
    return WorkItem{v.x, v.y, v.z, v.w};
  };
  auto stage_ptr = [&](int s) -> float * { return stages + (s & 1) * C16::STAGE_FLOATS; };
  const Blk kNoBlk{-1, 0.f};

  // software pipeline over work items: `wi` is being processed, `wn` (+ its first index block) is
  // already in registers, the counter for the one after is fetched a whole row ahead
  int i0 = fetch();
  if (i0 < 0) return;
  WorkItem wi = load_item(i0);
  int i1 = fetch();
  WorkItem wn{0, 0, 0, -1};
  Blk b0 = kNoBlk, nb0 = kNoBlk;
  if (pass == 0) {
    b0 = load_block(wi, 0, indices, data, lane);
    const int nks0 = (wi.k1 - wi.k0 + 15) >> 4;
    issue_kstep16<NB>(stage_ptr(0), b0, 0, 0 < nks0, sigma, Y, lane);
    issue_kstep16<NB>(stage_ptr(1), b0, 1, 1 < nks0, sigma, Y, lane);
  }
  if (i1 >= 0) {
    wn = load_item(i1);
    if (pass == 0) nb0 = load_block(wn, 0, indices, data, lane);
  }

  RowState<NB> st;
  for (;;) {
    const bool whole = (wi.slot == -1), chunk = (wi.slot >= 0), finish = (wi.slot == -2);
    const int i2 = (i1 >= 0) ? fetch() : -1;  // consumed after this row's accumulation
    // ---- initialise the accumulators: sigma^2 (Y^T Y + lambda I) for a row that will be solved here, Y^T Y +
    //      lambda I for a finish item (its chunk partials arrive unscaled), 0 for a chunk
    const float ginit = (pass == 0) ? sigma2 : 1.f;
#pragma unroll
    for (int c = 0; c < C::NT8; ++c) st.bp[c] = 0.f;
#pragma unroll
    for (int i = 0; i < NB; ++i)
#pragma unroll
      for (int j = 2 * i; j < C::NT8; ++j) {
        float(&d)[4] = st.acc[C::tidx(i, j)];
        if (chunk) {
          d[0] = d[1] = d[2] = d[3] = 0.f;
        } else {
          const float2 top = __ldg(reinterpret_cast<const float2 *>(Greg + (16 * i + g) * F + 8 * j + 2 * t));
          const float2 bot = __ldg(reinterpret_cast<const float2 *>(Greg + (16 * i + g + 8) * F + 8 * j + 2 * t));
          d[0] = ginit * top.x; d[1] = ginit * top.y; d[2] = ginit * bot.x; d[3] = ginit * bot.y;
        }
      }

    WorkItem wnn{0, 0, 0, -1};
    Blk nnb0 = kNoBlk;
    if (pass == 0) {
      const int nks = (wi.k1 - wi.k0 + 15) >> 4;  // 16 nonzeros per k-step, two k-steps per 32-nonzero block
      Blk cb = b0;
      Blk nb = (nks > 2) ? load_block(wi, 1, indices, data, lane) : kNoBlk;
      for (int ks = 0; ks < nks; ++ks) {
        cp_async_wait<1>();
        __syncwarp();
        consume_kstep16<NB>(st, stage_ptr(ks), g, t);
        __syncwarp();  // the stage is free again
        const int tks = ks + 2;
        if ((tks & 1) == 0 && tks < nks) {  // the gathers move on to the next 32 nonzeros
          cb = nb;
          if (tks + 2 < nks) nb = load_block(wi, (tks >> 1) + 1, indices, data, lane);
        }
        issue_kstep16<NB>(stage_ptr(ks), cb, tks & 1, tks < nks, sigma, Y, lane);
      }
      // the first two k-steps of the next item land while this row is factored (both stages are free: the two
      // groups committed last were empty)
      if (i1 >= 0) {
        const int nks1 = (wn.k1 - wn.k0 + 15) >> 4;
        issue_kstep16<NB>(stage_ptr(0), nb0, 0, 0 < nks1, sigma, Y, lane);
        issue_kstep16<NB>(stage_ptr(1), nb0, 1, 1 < nks1, sigma, Y, lane);
      }
      if (i2 >= 0) {
        wnn = load_item(i2);
        nnb0 = load_block(wnn, 0, indices, data, lane);
      }
    } else {
      // finish: add the chunk partials in slot order
      for (int s = 0; s < wi.k1; ++s) {
        const float *sl = slots + (int64_t)(wi.k0 + s) * C::SLOT_FLOATS;
#pragma unroll
        for (int e = 0; e < C::NTILES; ++e)
#pragma unroll
          for (int v = 0; v < 4; ++v) st.acc[e][v] += sl[(e * 4 + v) * 32 + lane];
#pragma unroll
        for (int c = 0; c < C::NT8; ++c) st.bp[c] += sl[(C::NTILES * 4 + c) * 32 + lane];
      }
      if (i2 >= 0) wnn = load_item(i2);
    }

    if (chunk) {
      float *sl = slots + (int64_t)wi.slot * C::SLOT_FLOATS;  // partials leave the scaled domain
#pragma unroll
      for (int e = 0; e < C::NTILES; ++e)
#pragma unroll
        for (int v = 0; v < 4; ++v) sl[(e * 4 + v) * 32 + lane] = st.acc[e][v] * inv_sigma2;
#pragma unroll
      for (int c = 0; c < C::NT8; ++c) sl[(C::NTILES * 4 + c) * 32 + lane] = st.bp[c];
    } else {
      float *xout = X + (row_offset + wi.row) * F;
      if (whole && wi.k0 == wi.k1) {
        // no observations: the reference zeroes the row (_als.pyx:98-100)
        for (int m = lane; m < F; m += 32) {
          xout[m] = 0.f;
          for (int pi = 0; pi < n_peers; ++pi) peers[pi][(row_offset + wi.row) * F + m] = 0.f;
        }
      } else if (whole || finish) {
        bool ok = true;
        if (!(dbg & 8)) {
          if (pass == 0) {  // (sigma^2 A) x = sigma^2 b
#pragma unroll
            for (int c = 0; c < C::NT8; ++c) st.bp[c] *= sigma2;
          }
          float xx[(F + 31) / 32];
          factor_solve<NB>(st, U, zb, lane, ok, dbg, xx);
          if (ok) store_solution<F>(xx, xout, lane, peers, n_peers, (row_offset + wi.row) * F);
        }
        if (!ok && lane == 0) atomicMin(bad_row, (long long)(row_offset + wi.row));
        __syncwarp();
      }
    }
    if (i1 < 0) break;
    wi = wn;
    b0 = nb0;
    i1 = i2;
    wn = wnn;
    nb0 = nnb0;
  }
  cp_async_wait<0>();
}

// out[0] = max over [begin, end) of | |c| - 1 | (bits; NaN / inf left out), out[1] = 1 when some weight |c| - 1 is negative
// -- the weight range of a CSR, cached in the handle
__global__ void __launch_bounds__(256) csr_wmax_kernel(const int32_t *__restrict__ indptr, int64_t rows,
                                                       const float *__restrict__ data, unsigned *out) {
  const int64_t begin = indptr[0], end = indptr[rows];
  unsigned m = 0, neg = 0;
  for (int64_t e = begin + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < end; e += (int64_t)gridDim.x * blockDim.x) {
    const float w = fabsf(__ldg(data + e)) - 1.f;
    const unsigned b = __float_as_uint(fabsf(w));
    if (b < 0x7f800000u) m = max(m, b);
    if (w < 0.f) neg = 1;
  }
  if (neg) out[1] = 1;  // benign race: every writer stores the same value
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
}

// max |y| over a factor matrix (bits; NaN / inf left out)
__global__ void __launch_bounds__(256) factors_absmax_kernel(const float4 *__restrict__ y, int64_t n4, unsigned *out) {
  unsigned m = 0;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n4; e += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = __ldg(y + e);
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

// before every half of every width family: the counters are zeroed (only the narrow family reads them)
__global__ void init_solver_scalars(int32_t *counters, long long *bad_row) {
  if (threadIdx.x < 16) counters[threadIdx.x] = 0;
  if (threadIdx.x == 0) {
    // [1] keeps the first bad row of every half since the last als_solver_status (the asynchronous multi-GPU fit)
    if (bad_row[0] < bad_row[1]) bad_row[1] = bad_row[0];
    bad_row[0] = LLONG_MAX;
  }
}

// Timing ablations (tools/ablate.py) exist only in builds with -DALS_B200_ABLATE: ALS_B200_DEBUG bit0 skips the back
// substitution, bit1 the pivot elimination, bit2 the trailing updates, bit3 the whole factorisation (results are
// WRONG when set).  A release build compiles the flag to 0 and the branches away.
static int debug_flags() {
#ifdef ALS_B200_ABLATE
  static int v = -1;
  if (v < 0) {
    const char *e = getenv("ALS_B200_DEBUG");
    v = e ? atoi(e) : 0;
  }
  return v;
#else
  return 0;
#endif
}

// zeroes the per-segment work counters between the segments of one half: the whitening flag and max |y| of the half
// (kCtrWhitenOk, kCtrYAbsMax) stay
__global__ void reset_segment_counters(int32_t *counters) {
  const int t = threadIdx.x;
  if (t < 16 && t != kCtrWhitenOk && t != kCtrHasNan && t != kCtrYAbsMax) counters[t] = 0;
}

// Synchronises the side streams of a Cholesky half (aux and the short-row class streams) unless disarmed: an error
// return from the section forked onto them leaves launches there that may still read a ring slot of the segment.
struct JoinSidesOnError {
  als_ctx *ctx;
  bool armed = true;
  ~JoinSidesOnError() {
    if (!armed) return;
    cudaStreamSynchronize(ctx->aux);
    for (cudaStream_t s : ctx->class_stream)
      if (s) cudaStreamSynchronize(s);
  }
};

// The narrow family (ld <= 64) over C, which may be a list of row-block segments.  Everything that affects rounding is
// decided once for the whole matrix (max |y|, max ||c| - 1|, the long-row kernel, whether short rows take the whitened
// path, the whitening itself); the deferred list and its counters are per segment.
template <int NB>
int run_cholesky(als_ctx *ctx, const als_csr *Cm, als_factors *X, const als_factors *Y) {
  const int dbg = debug_flags();
  const int smem = Cfg16<NB>::WARP_FLOATS * kWarpsPerCta * (int)sizeof(float);
  auto kern = cholesky_half_kernel<NB>;
  ALS_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int ctas_per_sm = 0;
  ALS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, kern, 32 * kWarpsPerCta, smem));
  if (ctas_per_sm < 1) {
    set_error("cholesky: kernel does not fit on an SM (smem %d bytes)", smem);
    return ALS_E_CUDA;
  }
  const std::vector<const als_csr *> segs = segments_of(Cm);
  // the range of the fp16-split operands: max |y| of this half (one pass over Y) and max | |c| - 1 | of the CSR
  // (one pass over its values, cached in the handle until als_csr_scale changes them)
  unsigned *yabsmax = reinterpret_cast<unsigned *>(ctx->counters + kCtrYAbsMax);
  factors_absmax_kernel<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(reinterpret_cast<const float4 *>(Y->d),
                                                                     std::max<int64_t>(Y->rows, 0) * (Y->ld / 4), yabsmax);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  als_csr *Cmut = const_cast<als_csr *>(Cm);
  if (!Cmut->wmax_dev) {
    int arc = dev_alloc(ctx, (void **)&Cmut->wmax_dev, 2 * sizeof(unsigned));  // stream-ordered pool: no cudaMalloc per fit
    if (arc != ALS_OK) return arc;
  }
  if (!Cmut->wmax_valid) {
    if (Cm->host) {  // kept valid on the host from the upload on: the segments' values are not on the device here
      set_error("cholesky: host-resident CSR without its weight range");
      return ALS_E_INVALID;
    }
    ALS_CUDA(cudaMemsetAsync(Cmut->wmax_dev, 0, 2 * sizeof(unsigned), ctx->stream));
    for (const als_csr *S : segs) {
      csr_wmax_kernel<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(S->indptr, S->rows, S->data, Cmut->wmax_dev);
      ALS_CUDA(cudaGetLastError());
      ctx->launches++;
    }
    Cmut->wmax_valid = true;
    Cmut->neg_w_known = false;
  }
  if (NB == 4 && !Cmut->neg_w_known && ctx->knobs.long_tc) {
    // which long-row kernel: one 4-byte read-back per CSR (not per half), cached like the weight range
    unsigned flag = 0;
    ALS_CUDA(cudaMemcpyAsync(&flag, Cmut->wmax_dev + 1, sizeof(unsigned), cudaMemcpyDeviceToHost, ctx->stream));
    ALS_CUDA(cudaStreamSynchronize(ctx->stream));
    Cmut->has_neg_w = flag != 0;
    Cmut->neg_w_known = true;
  }
  const bool long_tc = NB == 4 && cholesky_tc_eligible(ctx, Cm, Y->ld);
  // Items of at most `short_max` nonzeros (a suffix of the length-sorted work list) go through the n x n
  // push-through system of cholesky_short.cu when there are enough of them to pay for whitening Y.
  int short_max = std::min(ctx->knobs.short_max, 16 * (NB - 1));  // a multiple of 8; a system of NS unknowns needs NS < F
  const int short_class = (48 - std::max(short_max, 0)) / 8;      // kShortThresholds: 48, 40, ..., 8
  if (short_max > 0) {
    int64_t n_short = 0;
    for (const als_csr *S : segs) n_short += S->n_work - S->le_begin[short_class];
    // worth it when the short rows outweigh whitening all of Y: one short row saves roughly what whitening 16 rows
    // of Y costs
    if (n_short * 16 < Y->rows) short_max = 0;
  }
  CholFamily fam;
  fam.slot_floats = Cfg<NB>::SLOT_FLOATS;
  fam.items_per_cta = kWarpsPerCta;
  fam.max_grid = (int64_t)ctx->sm_count * ctas_per_sm;
  // items[0, n) of S on `stream`: n_dev, when set, replaces n on the device; counter: the work counter they pull from
  auto kernel = [&](const als_csr *S, const WorkItem *items, int n, const int32_t *n_dev, int counter, int pass, int grid,
                    float *slots, cudaStream_t stream) {
    kern<<<grid, 32 * kWarpsPerCta, smem, stream>>>(S->indices, S->data, Y->d, X->d, S->row_offset, ctx->Greg, items, n,
                                                     n_dev, ctx->counters + counter, slots, ctx->bad_row, pass, dbg,
                                                     X->peers_dev, X->n_peers, Cm->wmax_dev, yabsmax);
  };
  fam.launch = [&](const als_csr *S, const WorkItem *items, int n, int pass, int grid, float *slots, float *) {
    kernel(S, items, n, nullptr, pass ? kCtrFinish : kCtrMain, pass, grid, slots, ctx->stream);
  };
  auto grid_of = [&](int64_t n) { return (int)std::min<int64_t>(ceil_div(n, kWarpsPerCta), fam.max_grid); };
  // every launch below reads S on ctx->stream, or on aux / the class streams joined back into it by ev_join before the
  // segment ends, which is what for_each_segment needs to reuse a ring slot of a host-resident C
  fam.pass0 = [&](size_t s, const als_csr *S, float *slots) -> int {
    if (s > 0) {
      reset_segment_counters<<<1, 32, 0, ctx->stream>>>(ctx->counters);
      ALS_CUDA(cudaGetLastError());
      ctx->launches++;
    }
    const int64_t n_main = short_max > 0 ? S->le_begin[short_class] : S->n_work;
    const bool seg_short = short_max > 0 && S->n_work > n_main;
    if (!S->n_work) return ALS_OK;
    JoinSidesOnError join{ctx};
    ProfScope prof(ctx, kProfCholesky);
    // The short-row side (whitening, the short-row kernels, the second pass of the full-size kernel over what they
    // hand back) runs on the aux stream.  The single-CTA factorisation of G is launched first and hides behind the
    // full-size kernel; the rest moves in as that kernel's persistent CTAs run out of long rows.
    const bool overlap = seg_short && n_main > 0 && !ctx->knobs.short_serial;
    cudaStream_t side = overlap ? ctx->aux : ctx->stream;
    if (short_max > 0) {
      if (overlap) {
        ALS_CUDA(cudaEventRecord(ctx->ev_fork, ctx->stream));
        ALS_CUDA(cudaStreamWaitEvent(ctx->aux, ctx->ev_fork, 0));
      }
      if (s == 0) {  // once per half: the later segments find W and Z in place
        int rc = short_rows_prepare(ctx, Y, side);
        if (rc != ALS_OK) return rc;
      }
    }
    if (n_main && long_tc) {
      // whole rows: normal equations on the wgmma tensor cores; chunks of giant rows: the mma.sync kernel
      int rc = launch_cholesky_tc(ctx, S, X, Y, n_main, Cm->wmax_dev, ctx->stream);
      if (rc != ALS_OK) return rc;
      if (S->n_slots) {
        kernel(S, S->chunks, (int)S->n_slots, nullptr, kCtrChunks, 0, grid_of(S->n_slots), slots, side);
        ALS_CUDA(cudaGetLastError());
        ctx->launches++;
      }
    } else if (n_main) {
      fam.launch(S, S->work, (int)n_main, 0, grid_of(n_main), slots, nullptr);
      ALS_CUDA(cudaGetLastError());
      ctx->launches++;
    }
    if (seg_short) {
      int rc = short_rows_launch(ctx, S, X, Y, n_main, short_max, side);
      if (rc != ALS_OK) return rc;
      // whatever the short-row kernels handed back (negative weights, chunks of giant rows, G not PD)
      kernel(S, ctx->deferred, 0, ctx->counters + kCtrDeferredCount, kCtrDeferredWork, 0, grid_of(S->n_work - n_main),
             slots, side);
      ALS_CUDA(cudaGetLastError());
      ctx->launches++;
      if (overlap) {
        ALS_CUDA(cudaEventRecord(ctx->ev_join, ctx->aux));
        ALS_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
      }
    }
    join.armed = false;
    return ALS_OK;
  };
  return run_cholesky_half(ctx, Cm, Y, fam);
}

}  // namespace

int run_cholesky_half(als_ctx *ctx, const als_csr *C, const als_factors *Y, const CholFamily &fam) {
  // row-block segments run one after the other: one scratch block covers the largest, with the giant-row slots first
  int64_t max_slots = 0, n_ws = 0;
  for (const als_csr *S : segments_of(C)) {
    max_slots = std::max(max_slots, S->n_slots);
    if (fam.ws_floats) n_ws = std::max(n_ws, std::min(std::max(S->n_work, S->n_finish), fam.max_grid));
  }
  const int64_t floats = max_slots * fam.slot_floats + n_ws * fam.ws_floats;
  float *slots = nullptr, *ws = nullptr;
  if (floats) {
    const int64_t bytes = floats * (int64_t)sizeof(float);
    int rc = ensure_scratch(ctx, bytes);
    if (rc != ALS_OK) {
      set_error("cholesky: factors=%d needs %.2f GB of device scratch (%lld giant-row chunks and %lld workspaces of %.2f MB "
                "each) and the allocation failed; split the rows into smaller calls or use the CG solver",
                Y->f, bytes / 1e9, (long long)max_slots, (long long)n_ws, fam.slot_floats * 4 / 1e6);
      return rc;
    }
    slots = (float *)ctx->scratch;
    ws = slots + max_slots * fam.slot_floats;
  }
  auto grid_of = [&](int64_t n) { return (int)std::min<int64_t>(ceil_div(n, fam.items_per_cta), fam.max_grid); };
  return for_each_segment(ctx, C, [&](size_t s, const als_csr *S) -> int {
    if (fam.pass0) {
      int rc = fam.pass0(s, S, slots);
      if (rc != ALS_OK) return rc;
    } else if (S->n_work) {
      ProfScope prof(ctx, kProfCholesky);
      fam.launch(S, S->work, (int)S->n_work, 0, grid_of(S->n_work), slots, ws);
      ALS_CUDA(cudaGetLastError());
      ctx->launches++;
    }
    if (S->n_finish) {
      ProfScope prof(ctx, kProfCholFinish);
      fam.launch(S, S->finish, (int)S->n_finish, 1, grid_of(S->n_finish), slots, ws);
      ALS_CUDA(cudaGetLastError());
      ctx->launches++;
    }
    return ALS_OK;
  });
}

int launch_cholesky(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y) {
  if (X->ld != Y->ld) {
    set_error("cholesky: X and Y strides differ (%d vs %d)", X->ld, Y->ld);
    return ALS_E_INVALID;
  }
  if (Y->ld > 1024 || (Y->ld > 128 && Y->ld % 64)) {
    set_error("cholesky: padded factors %d out of range", Y->ld);
    return ALS_E_INVALID;
  }
  init_solver_scalars<<<1, 32, 0, ctx->stream>>>(ctx->counters, ctx->bad_row);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  switch (Y->ld / 16) {
    case 1: return run_cholesky<1>(ctx, C, X, Y);
    case 2: return run_cholesky<2>(ctx, C, X, Y);
    case 3: return run_cholesky<3>(ctx, C, X, Y);
    case 4: return run_cholesky<4>(ctx, C, X, Y);
    case 5: return launch_cholesky_wide<5>(ctx, C, X, Y);
    case 6: return launch_cholesky_wide<6>(ctx, C, X, Y);
    case 7: return launch_cholesky_wide<7>(ctx, C, X, Y);
    case 8: return launch_cholesky_wide<8>(ctx, C, X, Y);
    default: return launch_cholesky_xwide(ctx, C, X, Y);  // 256 ... 1024
  }
}

}  // namespace als
