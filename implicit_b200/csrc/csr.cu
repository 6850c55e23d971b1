// Input preparation on the device: CSR transpose (replaces the host `Ciu = Cui.T.tocsr()`,
// implicit/cpu/als.py:137, which costs seconds at 17M-500M nonzeros and would dominate an
// end-to-end fit once the solve itself takes milliseconds).
//
// Transposing a CSR is a STABLE sort of its entries by column: a stable LSD radix sort of
// (column, entry position) pairs yields, per column, the entries in increasing row order, i.e.
// exactly scipy's canonical result, deterministically.  The radix sort is CUB's (toolkit library
// code; this is one-time input preparation, not the per-iteration hot path).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "common.h"

namespace als {
namespace {

__global__ void iota_kernel(int32_t *v, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) v[i] = (int32_t)i;
}

// For each sorted entry j: the row of the original entry e = perm[j] (binary search in indptr) and its value.
__global__ void gather_transposed_kernel(const int32_t *__restrict__ perm, const int32_t *__restrict__ indptr,
                                         int rows, const float *__restrict__ data, int64_t nnz,
                                         int32_t *__restrict__ out_indices, float *__restrict__ out_data) {
  int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; j < nnz; j += stride) {
    const int32_t e = perm[j];
    int lo = 0, hi = rows;  // largest r with indptr[r] <= e
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (indptr[mid] <= e) lo = mid; else hi = mid;
    }
    out_indices[j] = lo;
    out_data[j] = data[e];
  }
}

// out_indptr[c] = first position j with sorted_cols[j] >= c
__global__ void indptr_from_sorted_kernel(const int32_t *__restrict__ sorted_cols, int64_t nnz, int cols,
                                          int32_t *__restrict__ out_indptr) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c > cols) return;
  int64_t lo = 0, hi = nnz;  // first j in [0, nnz] with key >= c
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (sorted_cols[mid] < c) lo = mid + 1; else hi = mid;
  }
  out_indptr[c] = (int32_t)lo;
}

// ---- the transpose of a CSR held as row-block segments -----------------------------------------------------------
// Peak memory: input + output + O(piece).  Output positions are 64-bit: a column histogram over all segments, scanned
// into the output indptr, gives every column its range; the input is then sorted in row pieces of bounded nnz, in row
// order, each piece stably by column, and every entry goes to out_indptr[c] + (entries of column c in earlier pieces)
// + (its rank within the piece's column c).  Pieces in row order and stable sorts keep scipy's order exactly.
constexpr int64_t kPieceNnz = int64_t(1) << 28;

__global__ void column_histogram_kernel(const int32_t *__restrict__ indices, int64_t n, unsigned long long *count) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) atomicAdd(count + indices[i], 1ull);
}

__device__ __forceinline__ int64_t first_of_key(const int32_t *__restrict__ keys, int64_t n, int32_t c) {
  int64_t lo = 0, hi = n;  // first j with keys[j] >= c
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (keys[mid] < c) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// sorted entry j of a piece (perm[j]: its position after the piece's first nonzero, keys[j]: its column) -> its place
// in the output.  indptr: the piece's rows in the segment's indptr (indptr[0] is the piece's first nonzero).  Only the
// columns [c0, c1) are written, to out + (output position - out_base): a window of the output (transpose_host).
__global__ void scatter_piece_kernel(const int32_t *__restrict__ perm, const int32_t *__restrict__ keys, int64_t n,
                                     const int32_t *__restrict__ indptr, int rows, int64_t row0,
                                     const float *__restrict__ data, const long long *__restrict__ next,
                                     int32_t *__restrict__ out_indices, float *__restrict__ out_data, int32_t c0, int32_t c1,
                                     int64_t out_base) {
  int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int32_t base = indptr[0];
  for (; j < n; j += stride) {
    const int32_t e = perm[j], c = keys[j];
    if (c < c0 || c >= c1) continue;
    int lo = 0, hi = rows;  // largest r with indptr[r] - base <= e
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (indptr[mid] - base <= e) lo = mid; else hi = mid;
    }
    const int64_t dst = next[c] + (j - first_of_key(keys, n, c)) - out_base;
    out_indices[dst] = (int32_t)(row0 + lo);
    out_data[dst] = data[e];
  }
}

// after a piece: next[c] += its entries of column c (the last entry of each run of equal keys adds the run length)
__global__ void advance_columns_kernel(const int32_t *__restrict__ keys, int64_t n, long long *next) {
  int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; j < n; j += stride) {
    const int32_t c = keys[j];
    if (j + 1 < n && keys[j + 1] == c) continue;
    next[c] += j - first_of_key(keys, n, c) + 1;
  }
}

int transpose_segmented(als_ctx *ctx, const als_csr *in, als_csr *t) {
  const int64_t cols = in->cols;
  int end_bit = 1;
  while (end_bit < 32 && (1ll << end_bit) < (long long)cols) ++end_bit;
  long long *count = nullptr, *out_ip = nullptr;
  int rc;
  if ((rc = dev_alloc(ctx, (void **)&count, sizeof(long long) * (cols + 1))) != ALS_OK) return rc;
  if ((rc = dev_alloc(ctx, (void **)&out_ip, sizeof(long long) * (cols + 1))) != ALS_OK) return rc;
  ALS_CUDA(cudaMemsetAsync(count, 0, sizeof(long long) * (cols + 1), ctx->stream));
  const std::vector<const als_csr *> segs = segments_of(in);
  for (const als_csr *S : segs) {
    if (!S->nnz) continue;
    column_histogram_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(S->indices, S->nnz, (unsigned long long *)count);
    ALS_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  {
    void *tmp = nullptr;
    size_t tmp_bytes = 0;
    ALS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, count, out_ip, (int)(cols + 1), ctx->stream));
    if ((rc = dev_alloc(ctx, &tmp, (int64_t)tmp_bytes)) != ALS_OK) return rc;
    ALS_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, count, out_ip, (int)(cols + 1), ctx->stream));
    dev_free(ctx, tmp);
  }
  std::vector<int64_t> ip((size_t)cols + 1);
  ALS_CUDA(cudaMemcpyAsync(ip.data(), out_ip, sizeof(int64_t) * (cols + 1), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaMemcpyAsync(count, out_ip, sizeof(long long) * (cols + 1), cudaMemcpyDeviceToDevice, ctx->stream));  // next[c]
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  dev_free(ctx, out_ip);
  // pieces: whole rows of one segment, at most kPieceNnz nonzeros unless a single row is longer
  struct Piece { const als_csr *S; int64_t r0, r1, b0, n; };
  std::vector<Piece> pieces;
  int64_t max_piece = 0;
  for (const als_csr *S : segs) {
    std::vector<int32_t> sip((size_t)S->rows + 1);
    ALS_CUDA(cudaMemcpy(sip.data(), S->indptr, sizeof(int32_t) * (S->rows + 1), cudaMemcpyDeviceToHost));
    for (int64_t a = 0; a < S->rows;) {
      int64_t b = std::upper_bound(sip.begin() + a + 1, sip.end(), (int64_t)sip[a] + kPieceNnz) - sip.begin() - 1;
      b = std::max(b, a + 1);
      pieces.push_back(Piece{S, a, b, sip[a], (int64_t)sip[b] - sip[a]});
      max_piece = std::max(max_piece, pieces.back().n);
      a = b;
    }
  }
  if (max_piece > 0) {
    int32_t *keys_out = nullptr, *vals_in = nullptr, *vals_out = nullptr;
    void *tmp = nullptr;
    size_t tmp_bytes = 0;
    ALS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, segs[0]->indices, keys_out, vals_in, vals_out, (int)max_piece,
                                             0, end_bit, ctx->stream));
    if ((rc = dev_alloc(ctx, (void **)&keys_out, sizeof(int32_t) * max_piece)) != ALS_OK ||
        (rc = dev_alloc(ctx, (void **)&vals_in, sizeof(int32_t) * max_piece)) != ALS_OK ||
        (rc = dev_alloc(ctx, (void **)&vals_out, sizeof(int32_t) * max_piece)) != ALS_OK ||
        (rc = dev_alloc(ctx, &tmp, (int64_t)tmp_bytes)) != ALS_OK)
      return rc;
    iota_kernel<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(vals_in, max_piece);
    ALS_CUDA(cudaGetLastError());
    ctx->launches++;
    for (const Piece &pc : pieces) {
      const int64_t b0 = pc.b0, n = pc.n;
      if (n == 0) continue;
      ALS_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, pc.S->indices + b0, keys_out, vals_in, vals_out, (int)n, 0,
                                               end_bit, ctx->stream));
      scatter_piece_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(
          vals_out, keys_out, n, pc.S->indptr + pc.r0, (int)(pc.r1 - pc.r0), pc.S->row_offset - in->row_offset + pc.r0,
          pc.S->data + b0, count, t->indices, t->data, 0, INT32_MAX, 0);
      ALS_CUDA(cudaGetLastError());
      advance_columns_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(keys_out, n, count);
      ALS_CUDA(cudaGetLastError());
      ctx->launches += 2;
    }
    dev_free(ctx, keys_out);  // stream ordered: after the kernels above
    dev_free(ctx, vals_in);
    dev_free(ctx, vals_out);
    dev_free(ctx, tmp);
  }
  dev_free(ctx, count);
  // the output's segments and their schedules are built right away (no lazy schedule for a segmented transpose)
  return make_segments(ctx, t, ip.data());
}

// ---- the transpose of a host-resident CSR, into a host-resident CSR --------------------------------------------------
// The same arithmetic as transpose_segmented with each segment as one piece, but the output is built on the device one
// column window at a time: a window is a run of whole columns holding at most `budget` output nonzeros.  For each window
// every input segment is streamed through the ring in row order, sorted stably by column, and only its entries of the
// window's columns are scattered; the finished window goes to its contiguous place in the host output.  The device
// working set is the ring, the sort buffers of one segment and one window, whatever nnz is.  When the whole output fits
// the budget there is one window and the input crosses PCIe twice (the column histogram reads the indices only).
constexpr int64_t kWindowSegments = 16;  // a window holds at most this many segment caps of output

int transpose_host(als_ctx *ctx, const als_csr *in, als_csr *t) {
  const int64_t cols = in->cols;
  int end_bit = 1;
  while (end_bit < 32 && (1ll << end_bit) < (long long)cols) ++end_bit;
  long long *next = nullptr, *out_ip = nullptr;
  int rc;
  if ((rc = dev_alloc(ctx, (void **)&next, sizeof(long long) * (cols + 1))) != ALS_OK) return rc;
  if ((rc = dev_alloc(ctx, (void **)&out_ip, sizeof(long long) * (cols + 1))) != ALS_OK) return rc;
  ALS_CUDA(cudaMemsetAsync(next, 0, sizeof(long long) * (cols + 1), ctx->stream));
  rc = for_each_segment(ctx, in, [&](size_t, const als_csr *S) -> int {
    if (!S->nnz) return ALS_OK;
    column_histogram_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(S->indices, S->nnz, (unsigned long long *)next);
    ALS_CUDA(cudaGetLastError());
    ctx->launches++;
    return ALS_OK;
  }, /*with_data=*/false);
  if (rc != ALS_OK) return rc;
  {
    void *tmp = nullptr;
    size_t tmp_bytes = 0;
    ALS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, next, out_ip, (int)(cols + 1), ctx->stream));
    if ((rc = dev_alloc(ctx, &tmp, (int64_t)tmp_bytes)) != ALS_OK) return rc;
    ALS_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, next, out_ip, (int)(cols + 1), ctx->stream));
    dev_free(ctx, tmp);
  }
  std::vector<int64_t> ip((size_t)cols + 1);
  ALS_CUDA(cudaMemcpyAsync(ip.data(), out_ip, sizeof(int64_t) * (cols + 1), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  int64_t max_seg = 1;
  for (const als_csr *S : segments_of(in)) max_seg = std::max(max_seg, S->nnz);
  int32_t *keys_out = nullptr, *vals_in = nullptr, *vals_out = nullptr, *win_indices = nullptr;
  float *win_data = nullptr;
  void *tmp = nullptr;
  size_t tmp_bytes = 0;
  ALS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys_out, keys_out, vals_in, vals_out, (int)max_seg, 0, end_bit,
                                           ctx->stream));
  if ((rc = dev_alloc(ctx, (void **)&keys_out, sizeof(int32_t) * max_seg)) != ALS_OK ||
      (rc = dev_alloc(ctx, (void **)&vals_in, sizeof(int32_t) * max_seg)) != ALS_OK ||
      (rc = dev_alloc(ctx, (void **)&vals_out, sizeof(int32_t) * max_seg)) != ALS_OK ||
      (rc = dev_alloc(ctx, &tmp, (int64_t)tmp_bytes)) != ALS_OK)
    return rc;
  // the window budget: what is left of free memory once the ring (two segments) is counted, less 1/8 for the pool's
  // fragmentation, and at most kWindowSegments segment caps (so that a small segment_nnz forces several windows)
  int64_t free_bytes = 0, total_bytes = 0;
  if ((rc = mem_info(ctx, &free_bytes, &total_bytes)) != ALS_OK) return rc;
  const int64_t avail = free_bytes - free_bytes / 8 - 2 * 8 * max_seg;
  const int64_t budget = std::max<int64_t>(1, std::min(avail / 8, kWindowSegments * segment_cap(ctx, true)));
  std::vector<std::pair<int64_t, int64_t>> windows;  // column ranges [c0, c1)
  int64_t max_win = 1;
  for (int64_t c0 = 0; c0 < cols;) {
    int64_t c1 = std::upper_bound(ip.begin() + c0 + 1, ip.end(), ip[c0] + budget) - ip.begin() - 1;
    c1 = std::max(c1, c0 + 1);  // a column longer than the budget is a window of its own
    windows.emplace_back(c0, c1);
    max_win = std::max(max_win, ip[c1] - ip[c0]);
    c0 = c1;
  }
  if ((rc = dev_alloc(ctx, (void **)&win_indices, sizeof(int32_t) * max_win)) != ALS_OK ||
      (rc = dev_alloc(ctx, (void **)&win_data, sizeof(float) * max_win)) != ALS_OK) {
    set_error("als_csr_transpose: a column window of %lld nonzeros does not fit in device memory (%lld bytes free)",
              (long long)max_win, (long long)free_bytes);
    return rc;
  }
  iota_kernel<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(vals_in, max_seg);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  for (const auto &w : windows) {
    const int64_t c0 = w.first, c1 = w.second, wn = ip[c1] - ip[c0];
    if (wn == 0) continue;
    ALS_CUDA(cudaMemcpyAsync(next, out_ip, sizeof(long long) * (cols + 1), cudaMemcpyDeviceToDevice, ctx->stream));
    rc = for_each_segment(ctx, in, [&](size_t, const als_csr *S) -> int {
      const int64_t n = S->nnz;
      if (n == 0) return ALS_OK;
      size_t tb = tmp_bytes;
      ALS_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb, S->indices, keys_out, vals_in, vals_out, (int)n, 0, end_bit, ctx->stream));
      scatter_piece_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(
          vals_out, keys_out, n, S->indptr, (int)S->rows, S->row_offset - in->row_offset, S->data, next, win_indices, win_data,
          (int32_t)c0, (int32_t)c1, ip[c0]);
      ALS_CUDA(cudaGetLastError());
      advance_columns_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(keys_out, n, next);
      ALS_CUDA(cudaGetLastError());
      ctx->launches += 2;
      return ALS_OK;
    });
    if (rc != ALS_OK) return rc;
    // stream ordered: the next window's scatter starts after these copies
    ALS_CUDA(cudaMemcpyAsync(t->indices + ip[c0], win_indices, sizeof(int32_t) * wn, cudaMemcpyDeviceToHost, ctx->stream));
    ALS_CUDA(cudaMemcpyAsync(t->data + ip[c0], win_data, sizeof(float) * wn, cudaMemcpyDeviceToHost, ctx->stream));
  }
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  for (void *p : {(void *)next, (void *)out_ip, (void *)keys_out, (void *)vals_in, (void *)vals_out, tmp, (void *)win_indices,
                  (void *)win_data})
    dev_free(ctx, p);
  // the values are the input's: so is their range
  if ((rc = dev_alloc(ctx, (void **)&t->wmax_dev, 2 * sizeof(unsigned))) != ALS_OK) return rc;
  ALS_CUDA(cudaMemcpyAsync(t->wmax_dev, in->wmax_dev, 2 * sizeof(unsigned), cudaMemcpyDeviceToDevice, ctx->stream));
  t->wmax_valid = in->wmax_valid;
  t->neg_w_known = in->neg_w_known;
  t->has_neg_w = in->has_neg_w;
  return make_segments(ctx, t, ip.data());
}

}  // namespace

int for_each_segment(als_ctx *ctx, const als_csr *C, const SegmentLaunch &launch, bool with_data) {
  const std::vector<const als_csr *> segs = segments_of(C);
  if (!C->host) {
    for (size_t s = 0; s < segs.size(); ++s) {
      const int rc = launch(s, segs[s]);
      if (rc != ALS_OK) return rc;
    }
    return ALS_OK;
  }
  int64_t slot = 64;  // nonzeros per slot, a multiple of 64 so that every slot array starts 256-byte aligned
  for (const als_csr *S : segs) slot = std::max(slot, (S->nnz + 63) / 64 * 64);
  const int nslots = segs.size() > 1 ? 2 : 1;
  char *ring = nullptr;
  int rc = dev_alloc(ctx, (void **)&ring, nslots * slot * (int64_t)(with_data ? 8 : 4));
  if (rc != ALS_OK) {
    set_error("streaming a host-resident CSR: the device ring of %d x %lld nonzeros does not fit in device memory; lower "
              "segment_nnz", nslots, (long long)slot);
    return rc;
  }
  // the ring comes from the pool on the compute stream: the copy stream starts after that allocation
  for (int k = 0; k < nslots; ++k) ALS_CUDA(cudaEventRecord(ctx->ring_free[k], ctx->stream));
  auto slot_indices = [&](int k) { return reinterpret_cast<int32_t *>(ring) + (int64_t)k * slot * (with_data ? 2 : 1); };
  auto stage = [&](size_t s) -> int {
    const int k = (int)(s % nslots);
    const als_csr *S = segs[s];
    ALS_CUDA(cudaStreamWaitEvent(ctx->copy, ctx->ring_free[k], 0));
    if (S->nnz) {
      ALS_CUDA(cudaMemcpyAsync(slot_indices(k), S->indices, sizeof(int32_t) * S->nnz, cudaMemcpyHostToDevice, ctx->copy));
      if (with_data)
        ALS_CUDA(cudaMemcpyAsync(slot_indices(k) + slot, S->data, sizeof(float) * S->nnz, cudaMemcpyHostToDevice, ctx->copy));
    }
    ALS_CUDA(cudaEventRecord(ctx->ring_loaded[k], ctx->copy));
    return ALS_OK;
  };
  rc = stage(0);
  for (size_t s = 0; s < segs.size() && rc == ALS_OK; ++s) {
    const int k = (int)(s % nslots);
    if (s + 1 < segs.size() && (rc = stage(s + 1)) != ALS_OK) break;  // overlaps segment s
    ALS_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ring_loaded[k], 0));
    als_csr view = *segs[s];
    view.indices = slot_indices(k);
    view.data = with_data ? reinterpret_cast<float *>(slot_indices(k) + slot) : nullptr;
    if ((rc = launch(s, &view)) != ALS_OK) break;
    ALS_CUDA(cudaEventRecord(ctx->ring_free[k], ctx->stream));
  }
  if (rc != ALS_OK) cudaStreamSynchronize(ctx->copy);  // a staged copy may still be writing into the ring
  dev_free(ctx, ring);  // stream ordered: after the last launch, which waited for the last copy
  return rc;
}

void host_wmax(const float *v, int64_t n, unsigned *wmax_bits, bool *neg) {
  unsigned m = 0;
  bool ng = false;
  for (int64_t e = 0; e < n; ++e) {
    const float w = fabsf(v[e]) - 1.f;  // one fp32 rounding, as in csr_wmax_kernel
    unsigned b;
    const float aw = fabsf(w);
    memcpy(&b, &aw, sizeof(b));
    if (b < 0x7f800000u) m = std::max(m, b);
    if (w < 0.f) ng = true;
  }
  *wmax_bits = m;
  *neg = ng;
}

int set_host_wmax(als_ctx *ctx, als_csr *c, unsigned wmax_bits, bool neg) {
  if (!c->wmax_dev) {
    int rc = dev_alloc(ctx, (void **)&c->wmax_dev, 2 * sizeof(unsigned));
    if (rc != ALS_OK) return rc;
  }
  const unsigned h[2] = {wmax_bits, neg ? 1u : 0u};
  ALS_CUDA(cudaMemcpyAsync(c->wmax_dev, h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));  // `h` dies here
  c->wmax_valid = true;
  c->neg_w_known = true;
  c->has_neg_w = neg;
  return ALS_OK;
}

int make_segments(als_ctx *ctx, als_csr *p, const int64_t *ip) {
  const int64_t cap = segment_cap(ctx, p->host), rows = p->rows;
  std::vector<int64_t> starts;
  for (int64_t a = 0; a < rows || starts.empty();) {
    starts.push_back(a);
    if (a >= rows) break;
    // the most whole rows that fit the cap, and at least one
    int64_t b = std::upper_bound(ip + a + 1, ip + rows + 1, ip[a] + cap) - ip - 1;
    b = std::max(b, a + 1);
    if (ip[b] - ip[a] >= (int64_t)INT32_MAX) {
      set_error("CSR row %lld holds %lld nonzeros: a row is limited to 2^31 - 2", (long long)a, (long long)(ip[b] - ip[a]));
      return ALS_E_INVALID;
    }
    a = b;
  }
  const int64_t nseg = (int64_t)starts.size();
  starts.push_back(rows);
  std::vector<int32_t> cat((size_t)(rows + nseg));
  for (int64_t s = 0; s < nseg; ++s)
    for (int64_t r = starts[s]; r <= starts[s + 1]; ++r) cat[r + s] = (int32_t)(ip[r] - ip[starts[s]]);
  int rc = dev_alloc(ctx, (void **)&p->seg_indptr, sizeof(int32_t) * (rows + nseg));
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaMemcpyAsync(p->seg_indptr, cat.data(), sizeof(int32_t) * cat.size(), cudaMemcpyHostToDevice, ctx->stream));
  p->max_row_nnz = 0;
  for (int64_t s = 0; s < nseg; ++s) {
    const int64_t a = starts[s], b = starts[s + 1];
    als_csr *c = new als_csr();
    c->ctx = ctx;
    c->rows = b - a;
    c->cols = p->cols;
    c->nnz = ip[b] - ip[a];
    c->row_offset = p->row_offset + a;
    c->owns = false;
    c->indptr = p->seg_indptr + a + s;
    c->indices = p->indices + ip[a];
    c->data = p->data + ip[a];
    p->segs.push_back(c);
    if ((rc = build_schedule(ctx, c, cat.data() + a + s)) != ALS_OK) return rc;
    p->max_row_nnz = std::max(p->max_row_nnz, c->max_row_nnz);
  }
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));  // `cat` dies here
  return ALS_OK;
}

int csr_indptr64(als_ctx *ctx, const als_csr *c, std::vector<int64_t> &out) {
  out.assign((size_t)c->rows + 1, 0);
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  std::vector<int32_t> ip;
  for (const als_csr *S : segments_of(c)) {
    ip.resize((size_t)S->rows + 1);
    ALS_CUDA(cudaMemcpy(ip.data(), S->indptr, sizeof(int32_t) * ip.size(), cudaMemcpyDeviceToHost));
    const int64_t r0 = S->row_offset - c->row_offset, base = S->indices - c->indices;
    for (int64_t r = 0; r <= S->rows; ++r) out[r0 + r] = base + ip[r];
  }
  return ALS_OK;
}

int csr_transpose(als_ctx *ctx, const als_csr *in, als_csr **out) {
  *out = nullptr;
  if (in->row_offset != 0) {
    set_error("als_csr_transpose: row shards cannot be transposed");
    return ALS_E_INVALID;
  }
  ALS_CUDA(cudaSetDevice(ctx->device));
  const int64_t nnz = in->nnz;
  const int rows = (int)in->rows, cols = (int)in->cols;
  als_csr *t = new als_csr();
  t->ctx = ctx;
  t->rows = cols;
  t->cols = rows;
  t->nnz = nnz;
  int rc;
  if (in->host) {  // host-resident in, host-resident out, built one column window at a time
    t->host = true;
    const size_t bytes = sizeof(int32_t) * (size_t)std::max<int64_t>(nnz, 1);
    cudaError_t e = cudaMallocHost((void **)&t->indices, bytes);
    if (e == cudaSuccess) e = cudaMallocHost((void **)&t->data, bytes);
    if (e != cudaSuccess) {
      als_csr_destroy(t);
      return cuda_fail(e, "cudaMallocHost (host-resident transpose)", __FILE__, __LINE__);
    }
    if ((rc = transpose_host(ctx, in, t)) != ALS_OK) {
      cudaStreamSynchronize(ctx->stream);  // D2H copies of a window may still be landing in t's arrays
      als_csr_destroy(t);
      return rc;
    }
    *out = t;
    return ALS_OK;
  }
  if (!in->segs.empty() || needs_segments(ctx, nnz)) {
    if ((rc = dev_alloc(ctx, (void **)&t->indices, sizeof(int32_t) * std::max<int64_t>(nnz, 1))) != ALS_OK ||
        (rc = dev_alloc(ctx, (void **)&t->data, sizeof(float) * std::max<int64_t>(nnz, 1))) != ALS_OK ||
        (rc = transpose_segmented(ctx, in, t)) != ALS_OK) {
      als_csr_destroy(t);
      return rc;
    }
    *out = t;
    return ALS_OK;
  }
  if ((rc = dev_alloc(ctx, (void **)&t->indptr, sizeof(int32_t) * ((int64_t)cols + 1))) != ALS_OK ||
      (rc = dev_alloc(ctx, (void **)&t->indices, sizeof(int32_t) * std::max<int64_t>(nnz, 1))) != ALS_OK ||
      (rc = dev_alloc(ctx, (void **)&t->data, sizeof(float) * std::max<int64_t>(nnz, 1))) != ALS_OK) {
    als_csr_destroy(t);
    return rc;
  }
  // one pinned landing buffer per context: a transposed matrix whose schedule is still pending owns it
  if (ctx->sched_owner && (rc = ensure_schedule(ctx, ctx->sched_owner)) != ALS_OK) {
    als_csr_destroy(t);
    return rc;
  }
  const int64_t need = sizeof(int32_t) * ((int64_t)cols + 1);
  if (need > ctx->sched_pinned_cap) {
    if (ctx->sched_pinned) ALS_CUDA(cudaFreeHost(ctx->sched_pinned));
    ctx->sched_pinned = nullptr;
    ctx->sched_pinned_cap = 0;
    ALS_CUDA(cudaMallocHost((void **)&ctx->sched_pinned, (size_t)need));
    ctx->sched_pinned_cap = need;
  }
  if (nnz > 0) {
    int32_t *keys_out = nullptr, *vals_in = nullptr, *vals_out = nullptr;
    void *tmp = nullptr;
    size_t tmp_bytes = 0;
    int end_bit = 1;
    while (end_bit < 32 && (1ll << end_bit) < (long long)cols) ++end_bit;
    ALS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, in->indices, keys_out, vals_in, vals_out, (int)nnz, 0,
                                             end_bit, ctx->stream));
    if ((rc = dev_alloc(ctx, (void **)&keys_out, sizeof(int32_t) * nnz)) != ALS_OK ||
        (rc = dev_alloc(ctx, (void **)&vals_in, sizeof(int32_t) * nnz)) != ALS_OK ||
        (rc = dev_alloc(ctx, (void **)&vals_out, sizeof(int32_t) * nnz)) != ALS_OK ||
        (rc = dev_alloc(ctx, &tmp, (int64_t)tmp_bytes)) != ALS_OK) {
      als_csr_destroy(t);
      return rc;
    }
    iota_kernel<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(vals_in, nnz);
    ALS_CUDA(cudaGetLastError());
    ALS_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, in->indices, keys_out, vals_in, vals_out, (int)nnz, 0,
                                             end_bit, ctx->stream));
    gather_transposed_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(vals_out, in->indptr, rows, in->data, nnz,
                                                                        t->indices, t->data);
    ALS_CUDA(cudaGetLastError());
    indptr_from_sorted_kernel<<<(cols + 1 + 255) / 256, 256, 0, ctx->stream>>>(keys_out, nnz, cols, t->indptr);
    ALS_CUDA(cudaGetLastError());
    ctx->launches += 3;
    dev_free(ctx, keys_out);  // stream ordered: after the kernels above
    dev_free(ctx, vals_in);
    dev_free(ctx, vals_out);
    dev_free(ctx, tmp);
  } else {
    ALS_CUDA(cudaMemsetAsync(t->indptr, 0, sizeof(int32_t) * ((int64_t)cols + 1), ctx->stream));
  }
  // The schedule needs the row lengths on the host.  The copy is left in flight and the schedule is built at the
  // first solve over this matrix (ensure_schedule): in a fit that is the item half, so the host-side sort of the
  // rows overlaps the user half that is already running instead of leaving the GPU idle.
  ALS_CUDA(cudaMemcpyAsync(ctx->sched_pinned, t->indptr, (size_t)need, cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaEventRecord(ctx->sched_ev, ctx->stream));
  t->sched_pending = true;
  ctx->sched_owner = t;
  *out = t;
  return ALS_OK;
}

}  // namespace als
