// R3: fused scores + filter + top-k (reference: topk.topk / _topk_batch, implicit/cpu/topk.pyx:15-67, and
// select<T>, implicit/cpu/select.h:12-39; the reference's GPU path is the unfused
// cublasSgemm -> thrust filters -> raft select_k of implicit/gpu/knn.cu:131-265).
//
// A CTA owns a block of QB query rows for the whole call and streams every item tile past them:
//   scores  query block x item tile on the tensor cores: warp-level mma.sync.m16n8k8 TF32 with the
//           3xTF32 split (operands split into hi / lo once when they are staged in shared memory),
//           fp32 accumulate -- fp32-faithful scores at ~9x the rate of the fp32 FMA pipe;
//   filter  the global filter_items mask and the per-row "liked" CSR columns are overwritten with
//           -FLT_MAX in the staged score tile (topk.pyx:51-56);
//   select  each warp walks its rows of the score tile IN COLUMN ORDER against the row's running
//           threshold and keeps a sorted k-list in shared memory, applying exactly the reference's
//           admission rule (`size < k || score > min.score`, evict the lexicographic (score, col)
//           minimum), so ties resolve bit-for-bit like select.h.  The score matrix is never
//           written to HBM.
#include <float.h>
#include <limits.h>
#include <string.h>

#include <algorithm>
#include <cub/device/device_segmented_radix_sort.cuh>

#include "common.h"

namespace als {
namespace {


template <int F, int TQ>
struct TkCfg {
  static constexpr int QB = 16 * TQ;             // query rows per CTA (64 or 16)
  static constexpr int IT = (F <= 64) ? 128 : 64;  // items per tile
  static constexpr int LDF = F + 4;              // operand row stride: conflict-free mma fragment reads
  static constexpr int SLD = IT + 4;             // score tile stride
  // 16 warps for the common 64-row block: with 144 KB of shared memory only one CTA fits per SM, and 8
  // warps (2 per scheduler) cannot keep the tensor pipe busy
  static constexpr int NW = (TQ >= 4) ? 16 : 8;
  static constexpr int THREADS = 32 * NW;
  static constexpr int ROWS_PER_WARP = QB / NW;
  // warp tiling of the QB x IT score tile: WY x WX warps, each MT m16-tiles x NT n8-tiles
  static constexpr int MT = QB >= 32 ? 2 : 1;
  static constexpr int WY = QB / (16 * MT);
  static constexpr int WX = NW / WY;
  static constexpr int NT = IT / (8 * WX);
  static_assert(WY * WX == NW && NT >= 1 && ROWS_PER_WARP >= 1, "warp tiling");
  // the staged score tile reuses the item buffer the tile's MMAs have just consumed when it fits (F >= 64):
  // 110 KB instead of 144 KB per CTA, so two CTAs share an SM and one's selection overlaps the other's MMAs
  static constexpr bool ALIAS_S = (IT * LDF >= QB * SLD);
  static constexpr int CTAS_PER_SM = (ALIAS_S && F <= 64) ? 2 : 1;
  static int smem_floats(int k) {
    return 2 * QB * LDF + 2 * IT * LDF + (ALIAS_S ? 0 : QB * SLD) + 2 * QB * k + 3 * QB;
  }
};

__device__ __forceinline__ void mma_tf32(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                         uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// 3xTF32 split (see cholesky.cu): hi rounded to nearest TF32, lo = x - hi handed over raw
__device__ __forceinline__ void split4(const float4 &v, uint4 &hi, uint4 &lo) {
  hi.x = (__float_as_uint(v.x) + 0x1000u) & 0xffffe000u; lo.x = __float_as_uint(v.x - __uint_as_float(hi.x));
  hi.y = (__float_as_uint(v.y) + 0x1000u) & 0xffffe000u; lo.y = __float_as_uint(v.y - __uint_as_float(hi.y));
  hi.z = (__float_as_uint(v.z) + 0x1000u) & 0xffffe000u; lo.z = __float_as_uint(v.z - __uint_as_float(hi.z));
  hi.w = (__float_as_uint(v.w) + 0x1000u) & 0xffffe000u; lo.w = __float_as_uint(v.w - __uint_as_float(hi.w));
}

__device__ __forceinline__ bool pair_less(float s, int c, float s2, int c2) { return s < s2 || (s == s2 && c < c2); }

// Warp-cooperative insertion of (s, col) into the ascending list (ls, lc)[0..cnt) with capacity k.
// Precondition (checked by the caller): cnt < k or s > ls[0].
__device__ __forceinline__ void list_insert(float *ls, int *lc, int &cnt, int k, float s, int col, int lane) {
  int pos = 0;
  for (int base = 0; base < cnt; base += 32) {
    const int i = base + lane;
    const bool lt = i < cnt && pair_less(ls[i], lc[i], s, col);
    pos += __popc(__ballot_sync(0xffffffffu, lt));
  }
  if (cnt < k) {
    for (int hi = cnt; hi > pos; hi -= 32) {  // shift [pos, cnt) up by one, top chunk first
      const int i = hi - 1 - lane;
      float ts = 0.f;
      int tc = 0;
      if (i >= pos) { ts = ls[i]; tc = lc[i]; }
      __syncwarp();
      if (i >= pos) { ls[i + 1] = ts; lc[i + 1] = tc; }
      __syncwarp();
    }
    if (lane == 0) { ls[pos] = s; lc[pos] = col; }
    ++cnt;
  } else {
    for (int lo = 1; lo < pos; lo += 32) {  // drop entry 0, shift [1, pos) down by one
      const int i = lo + lane;
      float ts = 0.f;
      int tc = 0;
      if (i < pos) { ts = ls[i]; tc = lc[i]; }
      __syncwarp();
      if (i < pos) { ls[i - 1] = ts; lc[i - 1] = tc; }
      __syncwarp();
    }
    if (lane == 0) { ls[pos - 1] = s; lc[pos - 1] = col; }
  }
  __syncwarp();
}

template <int F, int TQ>
__global__ void __launch_bounds__(TkCfg<F, TQ>::THREADS, TkCfg<F, TQ>::CTAS_PER_SM)
topk_kernel(const float *__restrict__ items, int n_items, const float *__restrict__ queries,
            const int32_t *__restrict__ query_rows, int n_query, int k, const float *__restrict__ item_norms,
            const uint8_t *__restrict__ item_mask, const int32_t *__restrict__ liked_indptr,
            const int32_t *__restrict__ liked_indices, int32_t *__restrict__ out_ids, float *__restrict__ out_scores) {
  using C = TkCfg<F, TQ>;
  constexpr int QB = C::QB, IT = C::IT, SLD = C::SLD, LDF = C::LDF, MT = C::MT, NT = C::NT;
  extern __shared__ __align__(16) float smem[];
  uint32_t *Qh = reinterpret_cast<uint32_t *>(smem);  // [QB][LDF] query block, TF32 hi part
  uint32_t *Ql = Qh + QB * LDF;                        // [QB][LDF] lo part
  float *Ib = reinterpret_cast<float *>(Ql + QB * LDF);  // [2][IT][LDF] raw item tiles (cp.async double buffer)
  float *Ssep = Ib + 2 * IT * LDF;    // [QB][SLD] separate score tile (only when it cannot alias an item buffer)
  float *Ls = Ssep + (C::ALIAS_S ? 0 : QB * SLD);  // [QB][k]
  int *Lc = reinterpret_cast<int *>(Ls + QB * k);  // [QB][k]
  int *Cnt = Lc + QB * k;             // [QB]
  int *Cur = Cnt + QB;                // [QB] liked-list cursors
  int *Nxt = Cur + QB;                // [QB] column of the next liked entry (INT_MAX when exhausted)

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int wy = warp % C::WY, wx = warp / C::WY;  // this warp's block of the score tile
  const float neginf = -FLT_MAX;
  constexpr int NCH = IT / 32;
  const int n_tiles = (n_items + IT - 1) / IT;

  // item tile `tile` -> buffer: 16-byte cp.async, rows past n_items zero-filled (src-size 0)
  auto issue_tile = [&](int tile) {
    float *dst = Ib + (tile & 1) * IT * LDF;
    const int i0 = tile * IT;
    for (int e = tid; e < IT * (F / 4); e += C::THREADS) {
      const int it = e / (F / 4), fc = e % (F / 4);
      const bool in = i0 + it < n_items;
      const float *src = items + (int64_t)(in ? i0 + it : 0) * F + 4 * fc;
      const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst + it * LDF + 4 * fc);
      const int nbytes = in ? 16 : 0;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(d), "l"(src), "r"(nbytes) : "memory");
    }
    asm volatile("cp.async.commit_group;\n" ::: "memory");
  };

  for (int q0 = blockIdx.x * QB; q0 < n_query; q0 += gridDim.x * QB) {
    __syncthreads();
    issue_tile(0);
    // stage the query block, split into TF32 hi / lo once; rows past n_query are zero
    for (int e = tid; e < QB * (F / 4); e += C::THREADS) {
      const int q = e / (F / 4), fc = e % (F / 4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (q0 + q < n_query) {
        const int64_t row = query_rows ? query_rows[q0 + q] : (q0 + q);
        v = __ldg(reinterpret_cast<const float4 *>(queries + row * F) + fc);
      }
      uint4 hi, lo;
      split4(v, hi, lo);
      *reinterpret_cast<uint4 *>(Qh + q * LDF + 4 * fc) = hi;
      *reinterpret_cast<uint4 *>(Ql + q * LDF + 4 * fc) = lo;
    }
    for (int q = tid; q < QB; q += C::THREADS) {
      Cnt[q] = 0;
      int cur = 0, nxt = INT_MAX;
      if (liked_indptr && q0 + q < n_query) {
        cur = liked_indptr[q0 + q];
        if (cur < liked_indptr[q0 + q + 1]) nxt = liked_indices[cur];
      }
      Cur[q] = cur;
      Nxt[q] = nxt;
    }

    for (int tile = 0; tile < n_tiles; ++tile) {
      const int i0 = tile * IT;
      // the buffer the next tile lands in was last read two iterations ago (a barrier has passed since)
      if (tile + 1 < n_tiles) issue_tile(tile + 1);
      else asm volatile("cp.async.commit_group;\n" ::: "memory");
      asm volatile("cp.async.wait_group 1;\n" ::: "memory");
      __syncthreads();
      const float *It = Ib + (tile & 1) * IT * LDF;
      float *Ss = C::ALIAS_S ? (Ib + (tile & 1) * IT * LDF) : Ssep;
      // ---- scores on the tensor cores: 3xTF32 (lo*hi + hi*lo + hi*hi), fp32 accumulate.
      // Warp (wy, wx) owns queries [16 MT wy, +16 MT) x items [8 NT wx, +8 NT) of the tile.
      float acc[MT][NT][4];
#pragma unroll
      for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int n = 0; n < NT; ++n) acc[m][n][0] = acc[m][n][1] = acc[m][n][2] = acc[m][n][3] = 0.f;
      const int qb = 16 * MT * wy, ib = 8 * NT * wx;
#pragma unroll 2
      for (int kk = 0; kk < F / 8; ++kk) {
        uint32_t ah[MT][4], al[MT][4], bh[NT][2], bl[NT][2];
#pragma unroll
        for (int m = 0; m < MT; ++m) {
          const int r0 = (qb + 16 * m + g) * LDF + 8 * kk + t, r1 = r0 + 8 * LDF;
          ah[m][0] = Qh[r0]; ah[m][1] = Qh[r1]; ah[m][2] = Qh[r0 + 4]; ah[m][3] = Qh[r1 + 4];
          al[m][0] = Ql[r0]; al[m][1] = Ql[r1]; al[m][2] = Ql[r0 + 4]; al[m][3] = Ql[r1 + 4];
        }
#pragma unroll
        for (int n = 0; n < NT; ++n) {  // item operand split on the fly (the tile is staged raw by cp.async)
          const int c0 = (ib + 8 * n + g) * LDF + 8 * kk + t;
          const float v0 = It[c0], v1 = It[c0 + 4];
          bh[n][0] = (__float_as_uint(v0) + 0x1000u) & 0xffffe000u;
          bh[n][1] = (__float_as_uint(v1) + 0x1000u) & 0xffffe000u;
          bl[n][0] = __float_as_uint(v0 - __uint_as_float(bh[n][0]));
          bl[n][1] = __float_as_uint(v1 - __uint_as_float(bh[n][1]));
        }
#pragma unroll
        for (int term = 0; term < 3; ++term)  // term-major: a tile's three MMAs chain through its accumulator
#pragma unroll
          for (int m = 0; m < MT; ++m)
#pragma unroll
            for (int n = 0; n < NT; ++n) {
              if (term == 0) mma_tf32(acc[m][n], al[m][0], al[m][1], al[m][2], al[m][3], bh[n][0], bh[n][1]);
              else if (term == 1) mma_tf32(acc[m][n], ah[m][0], ah[m][1], ah[m][2], ah[m][3], bl[n][0], bl[n][1]);
              else mma_tf32(acc[m][n], ah[m][0], ah[m][1], ah[m][2], ah[m][3], bh[n][0], bh[n][1]);
            }
      }
      if (C::ALIAS_S) __syncthreads();  // every warp is done reading the item tile the scores overwrite
      // ---- norms, global mask, stage the tile (accumulator rows g / g+8, columns 2t, 2t+1)
#pragma unroll
      for (int n = 0; n < NT; ++n) {
        const int lc = ib + 8 * n + 2 * t;
        float nrm[2];
        bool masked[2];
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          const int col = i0 + lc + b;
          const bool in = col < n_items;
          nrm[b] = (item_norms && in) ? __ldg(item_norms + col) : 1.f;
          masked[b] = item_mask && in && item_mask[col];
        }
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float s0 = acc[m][n][2 * h], s1 = acc[m][n][2 * h + 1];
            if (item_norms) { s0 = __fdiv_rn(s0, nrm[0]); s1 = __fdiv_rn(s1, nrm[1]); }  // topk.pyx:48-49
            if (masked[0]) s0 = neginf;                                                   // topk.pyx:55-56
            if (masked[1]) s1 = neginf;
            *reinterpret_cast<float2 *>(Ss + (qb + 16 * m + g + 8 * h) * SLD + lc) = make_float2(s0, s1);
          }
      }
      __syncthreads();
      // ---- per-row liked filter + ordered selection; a warp owns ROWS_PER_WARP rows throughout
      for (int rr = 0; rr < C::ROWS_PER_WARP; ++rr) {
        const int row = warp * C::ROWS_PER_WARP + rr;
        if (q0 + row >= n_query) break;
        float *srow = Ss + row * SLD;
        if (liked_indptr && Nxt[row] < i0 + IT) {  // topk.pyx:51-53 (rows in ascending column order: liked_in_order)
          const int end = liked_indptr[q0 + row + 1];
          int cur = Cur[row];
          for (;;) {
            const int p = cur + lane;
            const int idx = p < end ? __ldg(liked_indices + p) : INT_MAX;
            const bool hit = idx < i0 + IT;
            if (hit && idx >= i0) srow[idx - i0] = neginf;
            const int n = __popc(__ballot_sync(0xffffffffu, hit));
            cur += n;
            if (n < 32) break;
          }
          __syncwarp();
          if (lane == 0) {
            Cur[row] = cur;
            Nxt[row] = cur < end ? liked_indices[cur] : INT_MAX;
          }
        }
        float *ls = Ls + row * k;
        int *lc = Lc + row * k;
        int cnt = Cnt[row];
        float thr = (cnt == k) ? ls[0] : neginf;
        // fast path: test the whole row of the tile against the threshold first (hits are rare once
        // the k-list has warmed up); the masks stay valid supersets because the threshold only rises
        float sv[NCH];
        unsigned mk[NCH];
        unsigned any = 0;
#pragma unroll
        for (int c = 0; c < NCH; ++c) sv[c] = srow[32 * c + lane];
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
          mk[c] = __ballot_sync(0xffffffffu, (i0 + 32 * c + lane) < n_items && (cnt < k || sv[c] > thr));
          any |= mk[c];
        }
        if (any) {
#pragma unroll
          for (int c = 0; c < NCH; ++c) {
            unsigned m = mk[c];
            while (m) {  // column order inside the chunk: exact select.h semantics
              const int b = __ffs(m) - 1;
              m &= m - 1;
              const float cs = __shfl_sync(0xffffffffu, sv[c], b);
              if (cnt < k || cs > thr) {  // select.h:23, re-checked against the updated threshold
                list_insert(ls, lc, cnt, k, cs, i0 + 32 * c + b, lane);
                thr = (cnt == k) ? ls[0] : neginf;
              }
            }
          }
          if (lane == 0) Cnt[row] = cnt;
          __syncwarp();
        }
      }
      if (C::ALIAS_S) __syncthreads();  // the score tile's buffer is the cp.async target of the tile after next
    }
    asm volatile("cp.async.wait_group 0;\n" ::: "memory");
    // ---- emit: descending by (score, col) (select.h:33); the tail past cnt stays zero (topk.pyx:20-21)
    __syncthreads();
    for (int rr = 0; rr < C::ROWS_PER_WARP; ++rr) {
      const int row = warp * C::ROWS_PER_WARP + rr;
      if (q0 + row >= n_query) break;
      const int cnt = Cnt[row];
      for (int j = lane; j < cnt; j += 32) {
        out_ids[(int64_t)(q0 + row) * k + j] = Lc[row * k + cnt - 1 - j];
        out_scores[(int64_t)(q0 + row) * k + j] = Ls[row * k + cnt - 1 - j];
      }
    }
  }
}

__global__ void mask_scatter_kernel(uint8_t *mask, const int32_t *idx, int64_t n, int n_items) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const int v = idx[i];
    if (v >= 0 && v < n_items) mask[v] = 1;
  }
}

struct TopkArgs {
  const float *items;
  int n_items;
  const float *queries;
  const int32_t *query_rows;
  int n_query;
  int k;        // effective k (<= n_items)
  int k_out;    // row stride of the outputs is k (same here: we run with k_out and clamp admission)
  const float *norms;
  const uint8_t *mask;
  const int32_t *liked_indptr;
  const int32_t *liked_indices;
  int32_t *ids;
  float *scores;
};

template <int F, int TQ>
int run_topk(als_ctx *ctx, const TopkArgs &a) {
  using C = TkCfg<F, TQ>;
  const int smem = C::smem_floats(a.k) * (int)sizeof(float);
  if (smem > 227 * 1024) {
    set_error("topk: k=%d needs %d bytes of shared memory per CTA (limit 227 KB)", a.k, smem);
    return ALS_E_UNSUPPORTED;
  }
  auto kern = topk_kernel<F, TQ>;
  ALS_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int64_t blocks = ceil_div(a.n_query, C::QB);
  const int grid = (int)std::min<int64_t>(blocks, (int64_t)ctx->sm_count * C::CTAS_PER_SM);
  ProfScope prof(ctx, kProfTopk);
  kern<<<grid, C::THREADS, smem, ctx->stream>>>(a.items, a.n_items, a.queries, a.query_rows, a.n_query, a.k, a.norms,
                                                  a.mask, a.liked_indptr, a.liked_indices, a.ids, a.scores);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  return ALS_OK;
}

// ---- very large k (the k-lists no longer fit in shared memory): scores to HBM, one segmented sort ---------------
// rank_items / recommend with N in the thousands up to "all items" (the reference's select.h takes any k).  One CTA per
// query row writes a 64-bit sort key per item -- the score in its order-preserving integer form above a tie-breaker
// that reproduces the reference's heap on ties -- and cub sorts every row descending:
//   * unfiltered items: tie-breaker ~id, so equal scores come out smaller column first and the boundary of the
//     first k prefers the smaller column (select.h:23 admits only strictly better scores); the host then reverses
//     each run of equal scores (select.h:33 emits larger columns first);
//   * filtered items all tie at -FLT_MAX, and there the heap's history matters: the first k columns fill it, later
//     (better) items evict the smallest column first and later filtered columns never enter, so the survivors are the
//     LARGEST filtered columns below k: tie-breaker id + 1 for id < k, 0 beyond (never selected), already in
//     output order.
__global__ void __launch_bounds__(256) score_rows_kernel(const float *__restrict__ items, int n_items, int ld,
                                                         const float *__restrict__ queries, const int32_t *__restrict__ query_rows,
                                                         int q0, int k, const float *__restrict__ norms,
                                                         const uint8_t *__restrict__ mask, const int32_t *__restrict__ liked_indptr,
                                                         const int32_t *__restrict__ liked_indices,
                                                         unsigned long long *__restrict__ keys, int32_t *__restrict__ ids) {
  extern __shared__ float qrow[];
  const int q = q0 + blockIdx.x;
  const int64_t src = query_rows ? query_rows[q] : q;
  for (int j = threadIdx.x; j < ld; j += blockDim.x) qrow[j] = queries[src * ld + j];
  __syncthreads();
  unsigned long long *out = keys + (int64_t)blockIdx.x * n_items;
  int32_t *oid = ids + (int64_t)blockIdx.x * n_items;
  auto key_of = [&](float sc, int i, bool filtered) -> unsigned long long {
    const unsigned b = __float_as_uint(sc);
    const unsigned ord = (b & 0x80000000u) ? ~b : (b | 0x80000000u);  // monotone map of floats onto unsigned integers
    const unsigned tie = filtered ? (i < k ? (unsigned)i + 1u : 0u) : ~(unsigned)i;
    return ((unsigned long long)ord << 32) | tie;
  };
  for (int i = threadIdx.x; i < n_items; i += blockDim.x) {
    const float4 *it = reinterpret_cast<const float4 *>(items + (int64_t)i * ld);
    float acc = 0.f;
    for (int j = 0; j < ld / 4; ++j) {
      const float4 v = __ldg(it + j);
      acc = fmaf(v.x, qrow[4 * j], fmaf(v.y, qrow[4 * j + 1], fmaf(v.z, qrow[4 * j + 2], fmaf(v.w, qrow[4 * j + 3], acc))));
    }
    if (norms) acc /= norms[i];                 // topk.pyx:48-49
    const bool filtered = mask && mask[i];      // topk.pyx:55-56
    out[i] = key_of(filtered ? -FLT_MAX : acc, i, filtered);
    oid[i] = i;
  }
  __syncthreads();
  if (liked_indptr)                              // topk.pyx:51-54
    for (int p = liked_indptr[q] + threadIdx.x; p < liked_indptr[q + 1]; p += blockDim.x) {
      const int i = liked_indices[p];
      out[i] = key_of(-FLT_MAX, i, true);
    }
}

__global__ void segment_offsets_kernel(int32_t *off, int n_seg, int n_items) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= n_seg) off[i] = i * n_items;
}

int topk_by_sort(als_ctx *ctx, const TopkArgs &a, int ld, int32_t *ids_host, float *scores_host, int k_out) {
  const int64_t I = a.n_items;
  // rows per pass: keys + values, in and out, within ~1.5 GB and 2^31 elements
  const int64_t per_row = I * 24;
  const int rows_per_pass =
      (int)std::max<int64_t>(1, std::min<int64_t>({(int64_t)a.n_query, (3ll << 29) / per_row, (int64_t)INT32_MAX / I}));
  unsigned long long *K_in = nullptr, *K_out = nullptr;
  int32_t *V_in = nullptr, *V_out = nullptr, *off = nullptr;
  void *tmp = nullptr;
  size_t tmp_bytes = 0;
  const int64_t n = (int64_t)rows_per_pass * I;
  cub::DeviceSegmentedRadixSort::SortPairsDescending(nullptr, tmp_bytes, K_in, K_out, V_in, V_out, (int)n, rows_per_pass, off, off + 1, 0,
                                                     64, ctx->stream);
  ALS_CUDA(cudaMalloc(&K_in, n * 8));
  ALS_CUDA(cudaMalloc(&K_out, n * 8));
  ALS_CUDA(cudaMalloc(&V_in, n * 4));
  ALS_CUDA(cudaMalloc(&V_out, n * 4));
  ALS_CUDA(cudaMalloc(&off, (rows_per_pass + 1) * 4));
  ALS_CUDA(cudaMalloc(&tmp, std::max<size_t>(tmp_bytes, 16)));
  segment_offsets_kernel<<<(rows_per_pass + 256) / 256, 256, 0, ctx->stream>>>(off, rows_per_pass, (int)I);
  int rc = ALS_OK;
  std::vector<unsigned long long> hk((size_t)rows_per_pass * a.k);
  std::vector<int32_t> hi((size_t)rows_per_pass * a.k);
  for (int q0 = 0; q0 < a.n_query && rc == ALS_OK; q0 += rows_per_pass) {
    const int nq = std::min(rows_per_pass, a.n_query - q0);
    ProfScope prof(ctx, kProfTopk);
    score_rows_kernel<<<nq, 256, ld * sizeof(float), ctx->stream>>>(a.items, a.n_items, ld, a.queries, a.query_rows, q0, a.k, a.norms,
                                                                     a.mask, a.liked_indptr, a.liked_indices, K_in, V_in);
    cudaError_t e = cub::DeviceSegmentedRadixSort::SortPairsDescending(tmp, tmp_bytes, K_in, K_out, V_in, V_out, (int)((int64_t)nq * I), nq,
                                                                       off, off + 1, 0, 64, ctx->stream);
    if (e != cudaSuccess || cudaGetLastError() != cudaSuccess) {
      set_error("topk: segmented sort failed (%s)", cudaGetErrorString(e));
      rc = ALS_E_CUDA;
      break;
    }
    ctx->launches += 2;
    cudaMemcpy2DAsync(hk.data(), 8 * (size_t)a.k, K_out, 8 * (size_t)I, 8 * (size_t)a.k, nq, cudaMemcpyDeviceToHost, ctx->stream);
    cudaMemcpy2DAsync(hi.data(), sizeof(int32_t) * a.k, V_out, sizeof(int32_t) * I, sizeof(int32_t) * a.k, nq, cudaMemcpyDeviceToHost,
                      ctx->stream);
    if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) {
      set_error("topk: fallback pass failed");
      rc = ALS_E_CUDA;
      break;
    }
    for (int r = 0; r < nq; ++r) {
      const unsigned long long *kr = hk.data() + (size_t)r * a.k;
      int32_t *ir = hi.data() + (size_t)r * a.k;
      float *sr = scores_host + (size_t)(q0 + r) * k_out;
      for (int j = 0; j < a.k; ++j) {
        const unsigned ord = (unsigned)(kr[j] >> 32);
        const unsigned b = (ord & 0x80000000u) ? (ord & 0x7fffffffu) : ~ord;
        memcpy(&sr[j], &b, sizeof(float));
      }
      for (int b = 0; b < a.k;) {  // runs of equal scores come out larger column first (select.h:33)
        int e2 = b + 1;
        while (e2 < a.k && sr[e2] == sr[b]) ++e2;
        if (sr[b] != -FLT_MAX) std::reverse(ir + b, ir + e2);  // the filtered tail is already in output order
        b = e2;
      }
      memcpy(ids_host + (size_t)(q0 + r) * k_out, ir, sizeof(int32_t) * a.k);
    }
  }
  cudaFree(K_in);
  cudaFree(K_out);
  cudaFree(V_in);
  cudaFree(V_out);
  cudaFree(off);
  cudaFree(tmp);
  return rc;
}

// ---- liked lists in column order -------------------------------------------------------------------------------
// Both fused kernels advance a cursor through a row's liked columns as the item tiles go by, so they need every row
// sorted ascending.  The reference (topk.pyx:51-54) does not care about the order, and neither may the ABI: a CSR
// is checked once, and one with an unsorted row gets a sorted copy that is kept with it.
__global__ void __launch_bounds__(256) csr_unsorted_kernel(const int32_t *__restrict__ indptr, int64_t rows,
                                                           const int32_t *__restrict__ indices, int *flag) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x)
    for (int p = indptr[r] + 1; p < indptr[r + 1]; ++p)
      if (indices[p - 1] > indices[p]) {
        *flag = 1;
        break;
      }
}

__global__ void rebase_indptr_kernel(const int32_t *__restrict__ in, int64_t n, int32_t *__restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = in[i] - in[0];
}

// (indptr, indices) of `liked` with every row in ascending column order
int liked_in_order(als_ctx *ctx, const als_csr *liked, const int32_t **indptr, const int32_t **indices) {
  als_csr *c = const_cast<als_csr *>(liked);  // the check and the sorted copy are caches of the handle
  if (!c->order_known && c->rows > 0 && c->nnz > 0) {
    int *flag = nullptr;
    int rc = dev_alloc(ctx, (void **)&flag, sizeof(int));
    if (rc != ALS_OK) return rc;
    ALS_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), ctx->stream));
    csr_unsorted_kernel<<<(unsigned)std::min<int64_t>(ceil_div(c->rows, 256), (int64_t)ctx->sm_count * 8), 256, 0, ctx->stream>>>(
        c->indptr, c->rows, c->indices, flag);
    ALS_CUDA(cudaGetLastError());
    ctx->launches++;
    int unsorted = 0, base = 0;
    ALS_CUDA(cudaMemcpyAsync(&unsorted, flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    ALS_CUDA(cudaMemcpyAsync(&base, c->indptr, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    dev_free(ctx, flag);
    ALS_CUDA(cudaStreamSynchronize(ctx->stream));
    if (unsorted) {
      if ((rc = dev_alloc(ctx, (void **)&c->sorted_indptr, (c->rows + 1) * sizeof(int32_t))) != ALS_OK) return rc;
      if ((rc = dev_alloc(ctx, (void **)&c->sorted_indices, c->nnz * sizeof(int32_t))) != ALS_OK) return rc;
      rebase_indptr_kernel<<<(unsigned)ceil_div(c->rows + 1, 256), 256, 0, ctx->stream>>>(c->indptr, c->rows + 1, c->sorted_indptr);
      ALS_CUDA(cudaGetLastError());
      void *tmp = nullptr;
      size_t tmp_bytes = 0;
      ALS_CUDA(cub::DeviceSegmentedRadixSort::SortKeys(nullptr, tmp_bytes, c->indices + base, c->sorted_indices, (int)c->nnz,
                                                       (int)c->rows, c->sorted_indptr, c->sorted_indptr + 1, 0, 32, ctx->stream));
      if ((rc = dev_alloc(ctx, &tmp, (int64_t)tmp_bytes)) != ALS_OK) return rc;
      ALS_CUDA(cub::DeviceSegmentedRadixSort::SortKeys(tmp, tmp_bytes, c->indices + base, c->sorted_indices, (int)c->nnz,
                                                       (int)c->rows, c->sorted_indptr, c->sorted_indptr + 1, 0, 32, ctx->stream));
      dev_free(ctx, tmp);
      ctx->launches += 2;
    }
    c->order_known = true;
  }
  *indptr = c->sorted_indptr ? c->sorted_indptr : c->indptr;
  *indices = c->sorted_indptr ? c->sorted_indices : c->indices;
  return ALS_OK;
}

template <int F>
int run_topk_f(als_ctx *ctx, const TopkArgs &a) {
  if (a.k <= 64) return run_topk<F, 4>(ctx, a);
  return run_topk<F, 1>(ctx, a);
}

}  // namespace

int launch_topk(als_ctx *ctx, const als_factors *items, const als_factors *queries, const int32_t *query_rows,
                int64_t n_query, int k, const float *item_norms_host, const als_csr *liked,
                const int32_t *filter_items, int64_t n_filter, int32_t *ids_host, float *scores_host) {
  if (items->ld != queries->ld) {
    set_error("topk: items and queries strides differ");
    return ALS_E_INVALID;
  }
  if (n_query == 0 || k == 0) return ALS_OK;
  memset(ids_host, 0, sizeof(int32_t) * n_query * k);      // topk.pyx:20-21
  memset(scores_host, 0, sizeof(float) * n_query * k);
  const int64_t I = items->rows;
  if (I == 0) return ALS_OK;
  if (n_query >= INT32_MAX || I >= INT32_MAX) {
    set_error("topk: too many rows");
    return ALS_E_UNSUPPORTED;
  }
  // The output row stride is k; admission is clamped to the number of items (the k-list can never
  // hold more than I entries), which leaves the tail zero exactly like the reference.
  const int k_eff = (int)std::min<int64_t>(k, I);
  // device staging: [ids | scores | query_rows | norms | mask | filter list]
  const int64_t out_elems = n_query * (int64_t)k_eff;
  int64_t off = 0;
  auto take = [&](int64_t bytes) {
    int64_t o = off;
    off += (bytes + 255) / 256 * 256;
    return o;
  };
  const int64_t o_ids = take(out_elems * 4), o_sc = take(out_elems * 4);
  const int64_t o_qr = take(query_rows ? n_query * 4 : 0);
  const int64_t o_nrm = take(item_norms_host ? I * 4 : 0);
  const int64_t o_mask = take(n_filter ? I : 0);
  const int64_t o_fl = take(n_filter * 4);
  // Large batches at 64 padded factors go to the wgmma kernel (topk_tc.cu).  It skips filtered items instead of
  // keeping them at -FLT_MAX, which is the same thing as long as every row has k unfiltered items left.
  const bool use_tc = !ctx->knobs.topk_legacy && topk_tc_eligible(items->ld, n_query, I, k_eff, item_norms_host != nullptr) &&
                      (!liked || !liked->sched_pending) &&
                      I - n_filter - (liked ? liked->max_row_nnz : 0) >= k_eff;
  const int64_t o_tc = take(use_tc ? topk_tc_scratch_bytes(n_query, I) : 0);
  int rc = ensure_scratch(ctx, off);
  if (rc != ALS_OK) return rc;
  char *base = (char *)ctx->scratch;
  ALS_CUDA(cudaMemsetAsync(base + o_ids, 0, out_elems * 4, ctx->stream));
  ALS_CUDA(cudaMemsetAsync(base + o_sc, 0, out_elems * 4, ctx->stream));
  if (query_rows) {
    for (int64_t q = 0; q < n_query; ++q)
      if (query_rows[q] < 0 || query_rows[q] >= queries->rows) {
        set_error("topk: query row %d out of range", query_rows[q]);
        return ALS_E_INVALID;
      }
    ALS_CUDA(cudaMemcpyAsync(base + o_qr, query_rows, n_query * 4, cudaMemcpyHostToDevice, ctx->stream));
  } else if (n_query > queries->rows) {
    set_error("topk: %lld queries requested from a matrix of %lld rows", (long long)n_query, (long long)queries->rows);
    return ALS_E_INVALID;
  }
  if (item_norms_host)
    ALS_CUDA(cudaMemcpyAsync(base + o_nrm, item_norms_host, I * 4, cudaMemcpyHostToDevice, ctx->stream));
  if (n_filter) {
    ALS_CUDA(cudaMemsetAsync(base + o_mask, 0, I, ctx->stream));
    ALS_CUDA(cudaMemcpyAsync(base + o_fl, filter_items, n_filter * 4, cudaMemcpyHostToDevice, ctx->stream));
    mask_scatter_kernel<<<(unsigned)ceil_div(n_filter, 256), 256, 0, ctx->stream>>>(
        (uint8_t *)(base + o_mask), (const int32_t *)(base + o_fl), n_filter, (int)I);
    ALS_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  TopkArgs a;
  a.items = items->d;
  a.n_items = (int)I;
  a.queries = queries->d;
  a.query_rows = query_rows ? (const int32_t *)(base + o_qr) : nullptr;
  a.n_query = (int)n_query;
  a.k = k_eff;
  a.k_out = k;
  a.norms = item_norms_host ? (const float *)(base + o_nrm) : nullptr;
  a.mask = n_filter ? (const uint8_t *)(base + o_mask) : nullptr;
  a.liked_indptr = nullptr;
  a.liked_indices = nullptr;
  if (liked && (rc = liked_in_order(ctx, liked, &a.liked_indptr, &a.liked_indices)) != ALS_OK) return rc;
  a.ids = (int32_t *)(base + o_ids);
  a.scores = (float *)(base + o_sc);
#define CALL(FF) run_topk_f<FF>(ctx, a)
  // k-lists of 2 * QB * k floats (QB = 16 rows per CTA beyond k = 64) must fit next to the operand tiles
  // (also every model wider than 128 padded factors: its scores come from the generic one-CTA-per-query kernel)
  const bool by_sort = !use_tc && ((k_eff > 64 && (int64_t)k_eff * 16 * 2 * 4 + 96 * 1024 > 227 * 1024) || items->ld > 128);
  if (by_sort) {
    return topk_by_sort(ctx, a, items->ld, ids_host, scores_host, k);
  }
  if (use_tc) {
    rc = launch_topk_tc(ctx, a.items, I, a.queries, a.query_rows, n_query, k_eff, a.mask, a.liked_indptr, a.liked_indices,
                        a.ids, a.scores, base + o_tc);
  } else
  switch (items->ld / 16) {
    case 1: rc = CALL(16); break;
    case 2: rc = CALL(32); break;
    case 3: rc = CALL(48); break;
    case 4: rc = CALL(64); break;
    case 5: rc = CALL(80); break;
    case 6: rc = CALL(96); break;
    case 7: rc = CALL(112); break;
    case 8: rc = CALL(128); break;
    default:
      set_error("topk: factors padded to %d > 128 are not supported yet", items->ld);
      return ALS_E_UNSUPPORTED;
  }
#undef CALL
  if (rc != ALS_OK) return rc;
  // outputs: device [n_query, k_eff] -> host [n_query, k]
  ALS_CUDA(cudaMemcpy2DAsync(ids_host, sizeof(int32_t) * k, base + o_ids, sizeof(int32_t) * k_eff,
                             sizeof(int32_t) * k_eff, n_query, cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaMemcpy2DAsync(scores_host, sizeof(float) * k, base + o_sc, sizeof(float) * k_eff,
                             sizeof(float) * k_eff, n_query, cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return ALS_OK;
}

}  // namespace als
