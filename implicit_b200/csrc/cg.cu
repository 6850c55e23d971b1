// R2: fused conjugate-gradient half-iteration (reference: _least_squares_cg, implicit/cpu/_als.pyx:154-248;
// the reference's own GPU kernel is least_squares_cg_kernel, implicit/gpu/als.cu:23-111).
//
// Matrix-free CG, (1 + cg_steps) passes over the row's nonzeros.  A warp owns a row; inside the warp
// groups of L = F/16 lanes (padded to a power of two) each take one nonzero at a time.  A lane holds
// 16 floats (four float4, interleaved so that a group's lanes read consecutive 16-byte words) of every
// CG vector -- x, r, p, Ap are replicated per group -- so a factor row costs four coalesced loads per
// lane and a dot product only log2(L) shuffles: at F = 64 eight nonzeros are in flight per warp
// instruction and a dot costs 2 shuffles (the first version, one float4 per lane, spent more issue
// slots on shuffles than on FMAs).
//
// Rows with more than kSplitNnz nonzeros ("giant" rows: the 139k-nnz hub item of C2) are not walked by
// one warp: every pass is split over their 2048-nonzero chunks (one warp each, partial sums to scratch)
// and a one-warp-per-row kernel combines the chunk sums in slot order and advances the CG recurrences,
// i.e. 2 (1 + cg_steps) short launches per half-iteration, deterministic.
#include <stdlib.h>

#include "common.h"

namespace als {

namespace {

constexpr int kCgWarps = 8;  // warps per CTA

template <int F, int NV>
struct CgCfg {
  static constexpr int V = F / 4;                    // float4 words per factor row
  static constexpr int LR = (V + NV - 1) / NV;       // lanes really needed per row
  static constexpr int L = LR <= 1 ? 1 : LR <= 2 ? 2 : LR <= 4 ? 4 : LR <= 8 ? 8 : LR <= 16 ? 16 : 32;  // lanes per group
  static constexpr int NG = 32 / L;                  // groups (nonzeros in flight) per warp
  static_assert(F % 16 == 0 && F <= 1024 && LR <= 32, "CG kernel: F / (4 NV) lanes per group must fit a warp");
};

template <int NV>
struct VecT {  // this lane's 4 NV floats of an F-vector: float4 words sub + L*i, i = 0..NV-1
  float4 v[NV];
};

__device__ __forceinline__ float dot4(const float4 &a, const float4 &b) {
  return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w)));
}
__device__ __forceinline__ void axpy4(float4 &y, float a, const float4 &x) {
  y.x = fmaf(a, x.x, y.x); y.y = fmaf(a, x.y, y.y); y.z = fmaf(a, x.z, y.z); y.w = fmaf(a, x.w, y.w);
}
__device__ __forceinline__ void add4(float4 &a, const float4 &b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
__device__ __forceinline__ float4 shfl_xor4(const float4 &v, int m) {
  return make_float4(__shfl_xor_sync(0xffffffffu, v.x, m), __shfl_xor_sync(0xffffffffu, v.y, m),
                     __shfl_xor_sync(0xffffffffu, v.z, m), __shfl_xor_sync(0xffffffffu, v.w, m));
}

template <int F, int NV>
struct Lane {
  using C = CgCfg<F, NV>;
  using Vec = VecT<NV>;
  int lane, sub, grp;
  float *xs;  // per-warp F floats: broadcast buffer for the symv

  __device__ __forceinline__ bool ok(int i) const { return sub + C::L * i < C::V; }

  __device__ __forceinline__ Vec zero() const {
    Vec r;
#pragma unroll
    for (int i = 0; i < NV; ++i) r.v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    return r;
  }
  __device__ __forceinline__ Vec load(const float *__restrict__ row, bool pred = true) const {
    Vec r;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      r.v[i] = (pred && ok(i)) ? __ldg(reinterpret_cast<const float4 *>(row) + sub + C::L * i)
                               : make_float4(0.f, 0.f, 0.f, 0.f);
    return r;
  }
  __device__ __forceinline__ Vec load_rw(const float *row) const {  // data written by a previous kernel/this one
    Vec r;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      r.v[i] = ok(i) ? reinterpret_cast<const float4 *>(row)[sub + C::L * i] : make_float4(0.f, 0.f, 0.f, 0.f);
    return r;
  }
  __device__ __forceinline__ void store(float *row, const Vec &a) const {  // group 0 writes
    if (grp == 0) {
#pragma unroll
      for (int i = 0; i < NV; ++i)
        if (ok(i)) reinterpret_cast<float4 *>(row)[sub + C::L * i] = a.v[i];
    }
  }
  // a solved factor row: local replica + NVLink stores into the peer replicas (multi-GPU)
  __device__ __forceinline__ void store_x(float *X, int64_t off, const Vec &a, float *const *peers, int n_peers) const {
    store(X + off, a);
    for (int pi = 0; pi < n_peers; ++pi) store(peers[pi] + off, a);
  }
  // sum over the L lanes of a group (every lane of the group gets the same bits)
  __device__ __forceinline__ float gsum(float v) const {
#pragma unroll
    for (int m = 1; m < C::L; m <<= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
    return v;
  }
  __device__ __forceinline__ float dot(const Vec &a, const Vec &b) const {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) s += dot4(a.v[i], b.v[i]);
    return gsum(s);
  }
  // sum a per-group Vec over the NG groups of the warp (identical bits in every group afterwards)
  __device__ __forceinline__ void across_groups(Vec &a) const {
#pragma unroll
    for (int m = C::L; m < 32; m <<= 1)
#pragma unroll
      for (int i = 0; i < NV; ++i) add4(a.v[i], shfl_xor4(a.v[i], m));
  }
  // out = G a  (G symmetric F x F, row-major, L1/L2 resident); a is replicated in every group
  __device__ __forceinline__ Vec symv(const float *__restrict__ G, const Vec &a) const {
    if (grp == 0) {
#pragma unroll
      for (int i = 0; i < NV; ++i)
        if (ok(i)) reinterpret_cast<float4 *>(xs)[sub + C::L * i] = a.v[i];
    }
    __syncwarp();
    Vec acc = zero();
    for (int j = grp; j < F; j += C::NG) {
      const float aj = xs[j];
      const float4 *row = reinterpret_cast<const float4 *>(G + j * F);
#pragma unroll
      for (int i = 0; i < NV; ++i)
        if (ok(i)) axpy4(acc.v[i], aj, __ldg(row + sub + C::L * i));
    }
    across_groups(acc);
    __syncwarp();
    return acc;
  }
  // One pass over the nonzeros [k0, k1):  acc += coef_k y_k,  coef_k = pos_k - sign (|c_k| - 1) (y_k . a)
  // with pos_k = c_k if (FIRST and c_k > 0) else 0                  (_als.pyx:190-201 and :214-222).
  // `gid` of `tg` groups take every tg-th nonzero; the trip count is warp-uniform.
  template <bool FIRST>
  __device__ __forceinline__ Vec nnz_pass(const int32_t *__restrict__ indices, const float *__restrict__ data,
                                          const float *__restrict__ Y, int k0, int k1, const Vec &a, float sign,
                                          int gid, int tg) const {
    Vec acc = zero();
    constexpr int UN = NV >= 4 ? 2 : 4;
    for (int kb = k0; kb < k1; kb += UN * tg) {
      Vec y[UN];
      float c[UN];
#pragma unroll
      for (int u = 0; u < UN; ++u) {
        const int k = kb + u * tg + gid;
        const bool valid = k < k1;
        const int idx = valid ? __ldg(indices + k) : 0;
        c[u] = valid ? __ldg(data + k) : 0.f;
        y[u] = load(Y + (int64_t)idx * F, valid);
      }
#pragma unroll
      for (int u = 0; u < UN; ++u) {
        const float d = dot(y[u], a);
        const float conf = fabsf(c[u]);
        const float pos = (FIRST && c[u] > 0.f) ? c[u] : 0.f;
        const float coef = pos - sign * (conf - 1.f) * d;
#pragma unroll
        for (int i = 0; i < NV; ++i) axpy4(acc.v[i], coef, y[u].v[i]);  // masked nonzeros have y == 0
      }
    }
    return acc;
  }
};

template <int F, int NV>
__device__ __forceinline__ Lane<F, NV> make_lane(float *xs_all) {
  Lane<F, NV> ln;
  ln.lane = threadIdx.x & 31;
  ln.sub = ln.lane % CgCfg<F, NV>::L;
  ln.grp = ln.lane / CgCfg<F, NV>::L;
  ln.xs = xs_all + (threadIdx.x >> 5) * F;
  return ln;
}

// ---- whole rows: one warp per row --------------------------------------------------------------
template <int F, int NV>
__global__ void __launch_bounds__(32 * kCgWarps)
cg_rows_kernel(const int32_t *__restrict__ indices, const float *__restrict__ data, const float *__restrict__ Y,
               float *__restrict__ X, int64_t row_offset, const float *__restrict__ Greg,
               const WorkItem *__restrict__ work, int n_work, int32_t *counter, int cg_steps,
               float *const *peers, int n_peers) {
  using C = CgCfg<F, NV>;
  using Vec = VecT<NV>;
  __shared__ __align__(16) float xs_all[kCgWarps * F];
  const Lane<F, NV> ln = make_lane<F, NV>(xs_all);
  for (;;) {
    int it = 0;
    if (ln.lane == 0) it = atomicAdd(counter, 1);
    it = __shfl_sync(0xffffffffu, it, 0);
    if (it >= n_work) break;
    const int4 w = __ldg(reinterpret_cast<const int4 *>(work) + it);
    if (w.w != -1) continue;  // chunks of giant rows: handled by the chunk / combine kernels
    const int64_t xoff = (row_offset + w.x) * F;
    float *xrow = X + xoff;
    const int k0 = w.y, k1 = w.z;
    if (k0 == k1) {  // no observations: zero the row (_als.pyx:182-184)
      ln.store_x(X, xoff, ln.zero(), peers, n_peers);
      continue;
    }
    Vec x = ln.load_rw(xrow);  // warm start (:179)
    // r = -(YtY + lambda I) x + sum_k (c_k^+ - (|c_k| - 1) y_k.x) y_k      (:187-201)
    Vec r = ln.symv(Greg, x);
    {
      Vec a = ln.template nnz_pass<true>(indices, data, Y, k0, k1, x, 1.f, ln.grp, C::NG);
      ln.across_groups(a);
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        r.v[i].x = a.v[i].x - r.v[i].x; r.v[i].y = a.v[i].y - r.v[i].y;
        r.v[i].z = a.v[i].z - r.v[i].z; r.v[i].w = a.v[i].w - r.v[i].w;
      }
    }
    Vec p = r;
    float rsold = ln.dot(r, r);
    if (rsold < 1e-20f) continue;  // :206-207 (x stays as it is)
    for (int s = 0; s < cg_steps; ++s) {
      // Ap = (YtY + lambda I) p + sum_k (|c_k| - 1) (y_k.p) y_k           (:212-222)
      Vec Ap = ln.symv(Greg, p);
      {
        Vec a = ln.template nnz_pass<false>(indices, data, Y, k0, k1, p, -1.f, ln.grp, C::NG);
        ln.across_groups(a);
#pragma unroll
        for (int i = 0; i < NV; ++i) add4(Ap.v[i], a.v[i]);
      }
      const float alpha = rsold / ln.dot(p, Ap);  // :225
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        axpy4(x.v[i], alpha, p.v[i]);    // :228
        axpy4(r.v[i], -alpha, Ap.v[i]);  // :231-232
      }
      const float rsnew = ln.dot(r, r);  // :234
      if (rsnew < 1e-20f) break;         // :235-236
      const float beta = rsnew / rsold;  // :239-242
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        p.v[i].x = fmaf(beta, p.v[i].x, r.v[i].x); p.v[i].y = fmaf(beta, p.v[i].y, r.v[i].y);
        p.v[i].z = fmaf(beta, p.v[i].z, r.v[i].z); p.v[i].w = fmaf(beta, p.v[i].w, r.v[i].w);
      }
      rsold = rsnew;
    }
    ln.store_x(X, xoff, x, peers, n_peers);
  }
}

// ---- giant rows: chunk pass + per-row combine ------------------------------------------------------
// state per giant row g (index into the finish list): rst[g][F], pst[g][F], scal[g] = {rsold, done}
template <int F, int NV>
__global__ void __launch_bounds__(32 * kCgWarps)
cg_chunk_kernel(const int32_t *__restrict__ indices, const float *__restrict__ data, const float *__restrict__ Y,
                const float *X, int64_t row_offset, const WorkItem *__restrict__ chunks,
                const int32_t *__restrict__ owner, int n_chunks, const float *pst, const float *scal,
                float *partials, int first) {
  using C = CgCfg<F, NV>;
  using Vec = VecT<NV>;
  __shared__ __align__(16) float xs_all[kCgWarps * F];
  const Lane<F, NV> ln = make_lane<F, NV>(xs_all);
  const int warp_global = blockIdx.x * kCgWarps + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * kCgWarps;
  for (int ci = warp_global; ci < n_chunks; ci += nwarps) {
    const WorkItem w = chunks[ci];
    const int g = owner[ci];
    if (!first && scal[2 * g + 1] != 0.f) continue;  // this row's CG already stopped
    const Vec a = first ? ln.load_rw(X + (row_offset + w.row) * F) : ln.load_rw(pst + (int64_t)g * F);
    Vec acc = first ? ln.template nnz_pass<true>(indices, data, Y, w.k0, w.k1, a, 1.f, ln.grp, C::NG)
                    : ln.template nnz_pass<false>(indices, data, Y, w.k0, w.k1, a, -1.f, ln.grp, C::NG);
    ln.across_groups(acc);
    ln.store(partials + (int64_t)w.slot * F, acc);
  }
}

template <int F, int NV>
__global__ void __launch_bounds__(32 * kCgWarps)
cg_combine_kernel(float *X, int64_t row_offset, const float *__restrict__ Greg, const WorkItem *__restrict__ finish,
                  int n_finish, float *rst, float *pst, float *scal, const float *partials, int first,
                  float *const *peers, int n_peers) {
  using Vec = VecT<NV>;
  __shared__ __align__(16) float xs_all[kCgWarps * F];
  const Lane<F, NV> ln = make_lane<F, NV>(xs_all);
  const int g = blockIdx.x * kCgWarps + (threadIdx.x >> 5);
  if (g >= n_finish) return;
  const WorkItem w = finish[g];  // row, first slot, number of slots
  const int64_t xoff = (row_offset + w.row) * F;
  float *xrow = X + xoff;
  if (!first && scal[2 * g + 1] != 0.f) return;
  Vec sum = ln.zero();
  for (int s = 0; s < w.k1; ++s) {  // fixed slot order
    const Vec part = ln.load_rw(partials + (int64_t)(w.k0 + s) * F);
#pragma unroll
    for (int i = 0; i < NV; ++i) add4(sum.v[i], part.v[i]);
  }
  Vec x = ln.load_rw(xrow);
  if (first) {
    Vec r = ln.symv(Greg, x);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      r.v[i].x = sum.v[i].x - r.v[i].x; r.v[i].y = sum.v[i].y - r.v[i].y;
      r.v[i].z = sum.v[i].z - r.v[i].z; r.v[i].w = sum.v[i].w - r.v[i].w;
    }
    const float rsold = ln.dot(r, r);
    ln.store(rst + (int64_t)g * F, r);
    ln.store(pst + (int64_t)g * F, r);
    if (ln.lane == 0) {
      scal[2 * g] = rsold;
      scal[2 * g + 1] = rsold < 1e-20f ? 1.f : 0.f;
    }
    return;
  }
  Vec p = ln.load_rw(pst + (int64_t)g * F);
  Vec r = ln.load_rw(rst + (int64_t)g * F);
  const float rsold = scal[2 * g];
  Vec Ap = ln.symv(Greg, p);
#pragma unroll
  for (int i = 0; i < NV; ++i) add4(Ap.v[i], sum.v[i]);
  const float alpha = rsold / ln.dot(p, Ap);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    axpy4(x.v[i], alpha, p.v[i]);
    axpy4(r.v[i], -alpha, Ap.v[i]);
  }
  const float rsnew = ln.dot(r, r);
  ln.store_x(X, xoff, x, peers, n_peers);
  if (rsnew < 1e-20f) {
    if (ln.lane == 0) scal[2 * g + 1] = 1.f;
    return;
  }
  const float beta = rsnew / rsold;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    p.v[i].x = fmaf(beta, p.v[i].x, r.v[i].x); p.v[i].y = fmaf(beta, p.v[i].y, r.v[i].y);
    p.v[i].z = fmaf(beta, p.v[i].z, r.v[i].z); p.v[i].w = fmaf(beta, p.v[i].w, r.v[i].w);
  }
  ln.store(rst + (int64_t)g * F, r);
  ln.store(pst + (int64_t)g * F, p);
  if (ln.lane == 0) scal[2 * g] = rsnew;
}

__global__ void zero_counters(int32_t *counters) {
  if (threadIdx.x < 16) counters[threadIdx.x] = 0;
}

template <int F, int NV>
int run_cg(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y, int cg_steps) {
  zero_counters<<<1, 32, 0, ctx->stream>>>(ctx->counters);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  if (C->n_work) {
    const int64_t want = ceil_div(C->n_work, kCgWarps);
    const int grid = (int)std::min<int64_t>(want, (int64_t)ctx->sm_count * 6);
    ProfScope prof(ctx, kProfCg);
    cg_rows_kernel<F, NV><<<grid, 32 * kCgWarps, 0, ctx->stream>>>(C->indices, C->data, Y->d, X->d, C->row_offset, ctx->Greg,
                                                              C->work, (int)C->n_work, ctx->counters, cg_steps, X->peers_dev,
                                                              X->n_peers);
    ALS_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  if (C->n_finish) {
    // scratch: partials[n_slots][F] | rst[n_finish][F] | pst[n_finish][F] | scal[n_finish][2]
    const int64_t floats = (C->n_slots + 2 * C->n_finish) * (int64_t)F + 2 * C->n_finish;
    int rc = ensure_scratch(ctx, floats * (int64_t)sizeof(float));
    if (rc != ALS_OK) return rc;
    float *partials = (float *)ctx->scratch;
    float *rst = partials + C->n_slots * (int64_t)F;
    float *pst = rst + C->n_finish * (int64_t)F;
    float *scal = pst + C->n_finish * (int64_t)F;
    const int cgrid = (int)std::min<int64_t>(ceil_div(C->n_slots, kCgWarps), (int64_t)ctx->sm_count * 6);
    const int fgrid = (int)ceil_div(C->n_finish, kCgWarps);
    ProfScope prof(ctx, kProfCgGiant);
    for (int pass = 0; pass <= cg_steps; ++pass) {
      const int first = pass == 0;
      cg_chunk_kernel<F, NV><<<cgrid, 32 * kCgWarps, 0, ctx->stream>>>(C->indices, C->data, Y->d, X->d, C->row_offset,
                                                                   C->chunks, C->chunk_owner, (int)C->n_slots, pst, scal,
                                                                   partials, first);
      ALS_CUDA(cudaGetLastError());
      cg_combine_kernel<F, NV><<<fgrid, 32 * kCgWarps, 0, ctx->stream>>>(X->d, C->row_offset, ctx->Greg, C->finish,
                                                                     (int)C->n_finish, rst, pst, scal, partials, first,
                                                                     X->peers_dev, X->n_peers);
      ALS_CUDA(cudaGetLastError());
      ctx->launches += 2;
    }
  }
  return ALS_OK;
}

int launch_cg_segment(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y, int cg_steps) {
  if (X->ld != Y->ld) {
    set_error("cg: X and Y strides differ (%d vs %d)", X->ld, Y->ld);
    return ALS_E_INVALID;
  }
  // float4 words per lane: knob cg_nv
  if (Y->ld > 128) {
    // wide models (the reference's CUDA path takes up to 1024 factors, implicit/gpu/als.cu:177-178): the padded width is
    // a multiple of 128, a whole warp per nonzero with ld / 128 float4 words per lane
    switch (Y->ld % 128 == 0 ? Y->ld / 128 : 0) {
      case 2: return run_cg<256, 2>(ctx, C, X, Y, cg_steps);
      case 3: return run_cg<384, 3>(ctx, C, X, Y, cg_steps);
      case 4: return run_cg<512, 4>(ctx, C, X, Y, cg_steps);
      case 5: return run_cg<640, 5>(ctx, C, X, Y, cg_steps);
      case 6: return run_cg<768, 6>(ctx, C, X, Y, cg_steps);
      case 7: return run_cg<896, 7>(ctx, C, X, Y, cg_steps);
      case 8: return run_cg<1024, 8>(ctx, C, X, Y, cg_steps);
      default:
        set_error("cg: factors padded to %d: beyond 128 the padded width must be a multiple of 128 up to 1024", Y->ld);
        return ALS_E_UNSUPPORTED;
    }
  }
  const int nv = ctx->knobs.cg_nv;
#define ALS_CG_CASE(FF)                                                   \
  case FF / 16:                                                           \
    if (nv == 4) return run_cg<FF, 4>(ctx, C, X, Y, cg_steps);            \
    if (nv == 2) return run_cg<FF, 2>(ctx, C, X, Y, cg_steps);            \
    return run_cg<FF, 1>(ctx, C, X, Y, cg_steps);
  switch (Y->ld / 16) {
    ALS_CG_CASE(16)
    ALS_CG_CASE(32)
    ALS_CG_CASE(48)
    ALS_CG_CASE(64)
    ALS_CG_CASE(80)
    ALS_CG_CASE(96)
    ALS_CG_CASE(112)
    ALS_CG_CASE(128)
    default:
      set_error("cg: factors padded to %d > 128 are not supported yet", Y->ld);
      return ALS_E_UNSUPPORTED;
  }
#undef ALS_CG_CASE
}

}  // namespace

// rows are independent: a CSR of row-block segments is solved one segment after the other with the same Greg (streamed
// through the device ring when C is host-resident; every CG launch is on ctx->stream)
int launch_cg(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y, int cg_steps) {
  return for_each_segment(ctx, C, [&](size_t, const als_csr *S) { return launch_cg_segment(ctx, S, X, Y, cg_steps); });
}

}  // namespace als
