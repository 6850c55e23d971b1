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

// ---- the transpose of a CSR held as row-block segments, device- or host-resident --------------------------------
// Peak memory of a device-resident transpose: input + output + O(piece).  Output positions are 64-bit: a column histogram over all segments, scanned
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
// columns [c0, c1) are written, to out + (output position - out_base): a window of a host-resident output.
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

// The output is built one column window at a time: a window is a run of whole columns, and for each window every
// input segment is walked in row order (through the ring when it is host-resident) and only its entries of the
// window's columns are scattered.  A device-resident output is one window, scattered straight into its arrays.  A
// host-resident output takes windows of at most `budget` output nonzeros in a device buffer, each copied to its
// contiguous place in the host output: the device working set is then the ring, the sort buffers of one piece and one
// window, whatever nnz is.  When the whole output fits the budget there is one window and the input crosses PCIe twice
// (the column histogram reads the indices only).
constexpr int64_t kWindowSegments = 16;  // a window holds at most this many segment caps of output

// count[c] += entries of column c in `in` (either residency; reads the indices only)
int column_histogram(als_ctx *ctx, const als_csr *in, unsigned long long *count) {
  return for_each_segment(ctx, in, [&](size_t, const als_csr *S) -> int {
    if (!S->nnz) return ALS_OK;
    column_histogram_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(S->indices, S->nnz, count);
    ALS_CUDA(cudaGetLastError());
    ctx->launches++;
    return ALS_OK;
  }, /*with_data=*/false);
}

// Writes the transpose of `in` into t->indices / t->data (t->rows, t->nnz and the arrays set) and its indptr, as
// positions into them, into ip[0 .. cols]; the caller lays t out.  index_base is added to every output index: 0 numbers
// the rows of `in` from its first row, in->row_offset gives the global rows of a shard.
int transpose_segmented(als_ctx *ctx, const als_csr *in, als_csr *t, int64_t index_base, std::vector<int64_t> &ip) {
  const int64_t cols = in->cols;
  int end_bit = 1;
  while (end_bit < 32 && (1ll << end_bit) < (long long)cols) ++end_bit;
  long long *next = nullptr, *out_ip = nullptr;
  int rc;
  if ((rc = dev_alloc(ctx, (void **)&next, sizeof(long long) * (cols + 1))) != ALS_OK) return rc;
  if ((rc = dev_alloc(ctx, (void **)&out_ip, sizeof(long long) * (cols + 1))) != ALS_OK) return rc;
  ALS_CUDA(cudaMemsetAsync(next, 0, sizeof(long long) * (cols + 1), ctx->stream));
  if ((rc = column_histogram(ctx, in, (unsigned long long *)next)) != ALS_OK) return rc;
  {
    void *tmp = nullptr;
    size_t tmp_bytes = 0;
    ALS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, next, out_ip, (int)(cols + 1), ctx->stream));
    if ((rc = dev_alloc(ctx, &tmp, (int64_t)tmp_bytes)) != ALS_OK) return rc;
    ALS_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, next, out_ip, (int)(cols + 1), ctx->stream));
    dev_free(ctx, tmp);
  }
  ip.assign((size_t)cols + 1, 0);
  ALS_CUDA(cudaMemcpyAsync(ip.data(), out_ip, sizeof(int64_t) * (cols + 1), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  dev_free(ctx, out_ip);
  // pieces: whole rows of one segment, at most kPieceNnz nonzeros unless a single row is longer, cut from the segment
  // indptrs (on the device for either residency)
  const std::vector<const als_csr *> segs = segments_of(in);
  struct Piece { int64_t r0, r1, b0, n; };
  std::vector<std::vector<Piece>> pieces(segs.size());
  int64_t max_piece = 1, max_seg = 1;
  for (size_t s = 0; s < segs.size(); ++s) {
    const als_csr *S = segs[s];
    std::vector<int32_t> sip((size_t)S->rows + 1);
    ALS_CUDA(cudaMemcpy(sip.data(), S->indptr, sizeof(int32_t) * (S->rows + 1), cudaMemcpyDeviceToHost));
    for (int64_t a = 0; a < S->rows;) {
      int64_t b = std::upper_bound(sip.begin() + a + 1, sip.end(), (int64_t)sip[a] + kPieceNnz) - sip.begin() - 1;
      b = std::max(b, a + 1);
      pieces[s].push_back(Piece{a, b, sip[a], (int64_t)sip[b] - sip[a]});
      max_piece = std::max(max_piece, pieces[s].back().n);
      a = b;
    }
    max_seg = std::max(max_seg, S->nnz);
  }
  int32_t *keys_out = nullptr, *vals_in = nullptr, *vals_out = nullptr, *win_indices = nullptr;
  float *win_data = nullptr;
  void *tmp = nullptr;
  size_t tmp_bytes = 0;
  ALS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys_out, keys_out, vals_in, vals_out, (int)max_piece, 0,
                                           end_bit, ctx->stream));
  if ((rc = dev_alloc(ctx, (void **)&keys_out, sizeof(int32_t) * max_piece)) != ALS_OK ||
      (rc = dev_alloc(ctx, (void **)&vals_in, sizeof(int32_t) * max_piece)) != ALS_OK ||
      (rc = dev_alloc(ctx, (void **)&vals_out, sizeof(int32_t) * max_piece)) != ALS_OK ||
      (rc = dev_alloc(ctx, &tmp, (int64_t)tmp_bytes)) != ALS_OK)
    return rc;
  std::vector<std::pair<int64_t, int64_t>> windows{{0, cols}};  // column ranges [c0, c1)
  if (t->host) {
    // the window budget: what is left of free memory once the ring (two segments) is counted, less 1/8 for the pool's
    // fragmentation, and at most kWindowSegments segment caps (so that a small segment_nnz forces several windows)
    int64_t free_bytes = 0, total_bytes = 0;
    if ((rc = mem_info(ctx, &free_bytes, &total_bytes)) != ALS_OK) return rc;
    const int64_t avail = free_bytes - free_bytes / 8 - 2 * 8 * max_seg;
    const int64_t budget = std::max<int64_t>(1, std::min(avail / 8, kWindowSegments * segment_cap(ctx, true)));
    windows.clear();
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
  }
  int32_t *out_indices = t->host ? win_indices : t->indices;
  float *out_data = t->host ? win_data : t->data;
  iota_kernel<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(vals_in, max_piece);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  for (const auto &w : windows) {
    const int64_t c0 = w.first, c1 = w.second, wn = ip[c1] - ip[c0];
    if (wn == 0) continue;
    ALS_CUDA(cudaMemcpyAsync(next, ip.data(), sizeof(int64_t) * (cols + 1), cudaMemcpyHostToDevice, ctx->stream));
    rc = for_each_segment(ctx, in, [&](size_t s, const als_csr *S) -> int {
      for (const Piece &pc : pieces[s]) {
        if (pc.n == 0) continue;
        ALS_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, S->indices + pc.b0, keys_out, vals_in, vals_out, (int)pc.n,
                                                 0, end_bit, ctx->stream));
        scatter_piece_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(
            vals_out, keys_out, pc.n, S->indptr + pc.r0, (int)(pc.r1 - pc.r0),
            index_base + S->row_offset - in->row_offset + pc.r0,
            S->data + pc.b0, next, out_indices, out_data, (int32_t)c0, (int32_t)c1, ip[c0]);
        ALS_CUDA(cudaGetLastError());
        advance_columns_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(keys_out, pc.n, next);
        ALS_CUDA(cudaGetLastError());
        ctx->launches += 2;
      }
      return ALS_OK;
    });
    if (rc != ALS_OK) return rc;
    if (t->host) {  // stream ordered: the next window's scatter starts after these copies
      ALS_CUDA(cudaMemcpyAsync(t->indices + ip[c0], win_indices, sizeof(int32_t) * wn, cudaMemcpyDeviceToHost, ctx->stream));
      ALS_CUDA(cudaMemcpyAsync(t->data + ip[c0], win_data, sizeof(float) * wn, cudaMemcpyDeviceToHost, ctx->stream));
    }
  }
  for (void *p : {(void *)next, (void *)keys_out, (void *)vals_in, (void *)vals_out, tmp, (void *)win_indices,
                  (void *)win_data})
    dev_free(ctx, p);  // stream ordered: after the kernels and copies above
  if (t->host) {  // the values are the input's: so is their range
    if ((rc = dev_alloc(ctx, (void **)&t->wmax_dev, 2 * sizeof(unsigned))) != ALS_OK) return rc;
    ALS_CUDA(cudaMemcpyAsync(t->wmax_dev, in->wmax_dev, 2 * sizeof(unsigned), cudaMemcpyDeviceToDevice, ctx->stream));
    t->wmax_valid = in->wmax_valid;
    t->neg_w_known = in->neg_w_known;
    t->has_neg_w = in->has_neg_w;
  }
  return ALS_OK;
}

// out[dst[r] + j - ip[r]] = in[j] for every entry j of a piece: its row r is the largest with ip[r] <= j
__global__ void merge_piece_kernel(const int32_t *__restrict__ in_indices, const float *__restrict__ in_data, int64_t n,
                                   const long long *__restrict__ ip, const long long *__restrict__ dst, int rows,
                                   int32_t *__restrict__ out_indices, float *__restrict__ out_data) {
  int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; j < n; j += stride) {
    int lo = 0, hi = rows;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (ip[mid] <= j) lo = mid; else hi = mid;
    }
    const int64_t o = dst[lo] + (j - ip[lo]);
    out_indices[o] = in_indices[j];
    out_data[o] = in_data[j];
  }
}

// tables: per piece its rebased indptr (rows + 1) then its rows' output starts (rows), uploaded to tables_dev
int merge_pieces(als_ctx *ctx, int n, const als_csr *const *pieces, const std::vector<int64_t> &base,
                 const std::vector<int64_t> &tables, long long *tables_dev, als_csr *c) {
  const int64_t rows = c->rows, stride = 2 * rows + 1;
  ALS_CUDA(cudaMemcpyAsync(tables_dev, tables.data(), sizeof(int64_t) * tables.size(), cudaMemcpyHostToDevice, ctx->stream));
  for (int p = 0; p < n; ++p) {
    const int64_t m = tables[p * stride + rows];
    if (!m) continue;
    const long long *tb = tables_dev + p * stride;
    merge_piece_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(pieces[p]->indices + base[p], pieces[p]->data + base[p],
                                                                  m, tb, tb + rows + 1, (int)rows, c->indices, c->data);
    ALS_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  return ALS_OK;
}

// One segment of a piece of a row stack: its rows + 1 entries of the output indptr, as 64-bit positions from the
// output's first nonzero (out_base is where the segment's first nonzero lands), and the segment's first position in
// its own indptr (a row-slice view's indptr does not start at 0), which tells the host where to copy its entries from.
__global__ void concat_indptr_kernel(const int32_t *__restrict__ ip, int64_t rows, long long out_base,
                                     long long *__restrict__ out, long long *__restrict__ first) {
  const long long f = ip[0];
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r == 0) *first = f;
  for (; r <= rows; r += (int64_t)gridDim.x * blockDim.x) out[r] = out_base + (ip[r] - f);
}

// ---- the device source of the one upload path (api.cu csr_build, als_csr_upload_device) ---------------------------
// flags[0]: indptr[0]; flags[1]: the first row r with indptr[r + 1] < indptr[r]; flags[2]: the first position (from
// indptr[0]) of an index outside [0, cols).  Rows and positions are folded with atomicMin from all ones (none).
template <typename T>
__global__ void indptr_rebase_kernel(const T *__restrict__ indptr, int64_t rows, long long *__restrict__ ip,
                                     unsigned long long *flags) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const long long base = (long long)indptr[0];
  if (r == 0) flags[0] = (unsigned long long)base;
  for (; r <= rows; r += stride) {
    const long long v = (long long)indptr[r];
    ip[r] = v - base;
    if (r < rows && (long long)indptr[r + 1] < v) atomicMin(flags + 1, (unsigned long long)r);
  }
}

// indices of 4 or 8 bytes -> int32, with the range check of the host staging (h2d_indices)
template <typename T>
__global__ void narrow_indices_kernel(const T *__restrict__ in, int64_t n, int64_t cols, int32_t *__restrict__ out,
                                      unsigned long long *flags) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const long long v = (long long)in[i];
    if ((unsigned long long)v >= (unsigned long long)cols) atomicMin(flags + 2, (unsigned long long)i);
    out[i] = (int32_t)v;
  }
}

// fp64 values -> fp32, rounded to nearest like numpy's astype(np.float32)
__global__ void narrow_values_kernel(const double *__restrict__ in, int64_t n, float *__restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) out[i] = (float)in[i];
}

}  // namespace

int device_indptr(als_ctx *ctx, const void *indptr, int indptr_bytes, int64_t rows, std::vector<int64_t> &ip,
                  int64_t *base, int64_t *bad_row) {
  long long *ip_dev = nullptr;
  unsigned long long *flags = nullptr;
  int rc = dev_alloc(ctx, (void **)&ip_dev, sizeof(long long) * (rows + 1));
  if (rc == ALS_OK) rc = dev_alloc(ctx, (void **)&flags, 3 * sizeof(unsigned long long));
  if (rc != ALS_OK) {
    dev_free(ctx, ip_dev);
    return rc;
  }
  ALS_CUDA(cudaMemsetAsync(flags, 0xff, 3 * sizeof(unsigned long long), ctx->stream));
  const int blocks = (int)std::min<int64_t>((rows + 256) / 256, (int64_t)ctx->sm_count * 8);
  if (indptr_bytes == 8)
    indptr_rebase_kernel<<<blocks, 256, 0, ctx->stream>>>((const long long *)indptr, rows, ip_dev, flags);
  else
    indptr_rebase_kernel<<<blocks, 256, 0, ctx->stream>>>((const int32_t *)indptr, rows, ip_dev, flags);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  unsigned long long f[2];
  ip.assign((size_t)rows + 1, 0);
  ALS_CUDA(cudaMemcpyAsync(ip.data(), ip_dev, sizeof(int64_t) * (rows + 1), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaMemcpyAsync(f, flags, sizeof(f), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  dev_free(ctx, ip_dev);
  dev_free(ctx, flags);
  *base = (int64_t)f[0];
  *bad_row = f[1] == ~0ull ? -1 : (int64_t)f[1];
  return ALS_OK;
}

int device_entries(als_ctx *ctx, als_csr *c, const void *indices, int index_bytes, const void *data, int data_bytes,
                   int64_t *bad_at) {
  *bad_at = -1;
  const int64_t n = c->nnz;
  if (n == 0) return ALS_OK;
  unsigned long long *flags = nullptr;
  int rc = dev_alloc(ctx, (void **)&flags, 3 * sizeof(unsigned long long));
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaMemsetAsync(flags, 0xff, 3 * sizeof(unsigned long long), ctx->stream));
  const int blocks = ctx->sm_count * 8;
  if (index_bytes == 8)
    narrow_indices_kernel<<<blocks, 256, 0, ctx->stream>>>((const long long *)indices, n, c->cols, c->indices, flags);
  else
    narrow_indices_kernel<<<blocks, 256, 0, ctx->stream>>>((const int32_t *)indices, n, c->cols, c->indices, flags);
  ALS_CUDA(cudaGetLastError());
  ctx->launches++;
  if (data_bytes == 8) {
    narrow_values_kernel<<<blocks, 256, 0, ctx->stream>>>((const double *)data, n, c->data);
    ALS_CUDA(cudaGetLastError());
    ctx->launches++;
  } else {
    ALS_CUDA(cudaMemcpyAsync(c->data, data, sizeof(float) * n, cudaMemcpyDeviceToDevice, ctx->stream));
  }
  unsigned long long bad = 0;
  ALS_CUDA(cudaMemcpyAsync(&bad, flags + 2, sizeof(bad), cudaMemcpyDeviceToHost, ctx->stream));
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));  // the caller's arrays have been read
  dev_free(ctx, flags);
  if (bad != ~0ull) {
    *bad_at = (int64_t)bad;
    return ALS_E_INVALID;
  }
  return ALS_OK;
}

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

int make_segments(als_ctx *ctx, als_csr *p, const int64_t *ip, bool schedule) {
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
    if (!schedule) continue;
    if ((rc = build_schedule(ctx, c, cat.data() + a + s)) != ALS_OK) return rc;
    p->max_row_nnz = std::max(p->max_row_nnz, c->max_row_nnz);
  }
  p->sched_lazy = !schedule;
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));  // `cat` dies here
  return ALS_OK;
}

int csr_layout(als_ctx *ctx, als_csr *c, const int64_t *ip, bool schedule) {
  if (!schedule) {  // what the schedule would have found, for the callers that read it without solving (als_topk)
    c->max_row_nnz = 0;
    for (int64_t r = 0; r < c->rows; ++r) c->max_row_nnz = std::max(c->max_row_nnz, ip[r + 1] - ip[r]);
  }
  if (c->host || needs_segments(ctx, c->nnz)) {
    const int64_t longest = c->max_row_nnz;
    const int rc = make_segments(ctx, c, ip, schedule);
    if (!schedule) c->max_row_nnz = longest;
    return rc;
  }
  std::vector<int32_t> ip32(ip, ip + c->rows + 1);
  int rc = dev_alloc(ctx, (void **)&c->indptr, sizeof(int32_t) * (c->rows + 1));
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaMemcpyAsync(c->indptr, ip32.data(), sizeof(int32_t) * ip32.size(), cudaMemcpyHostToDevice, ctx->stream));
  c->sched_lazy = !schedule;
  if (schedule) rc = build_schedule(ctx, c, ip32.data());
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));  // `ip32` dies here
  return rc;
}

int csr_alloc(als_ctx *ctx, als_csr *c) {
  const int64_t n = std::max<int64_t>(c->nnz, 1);
  if (!c->host) {
    int rc = dev_alloc(ctx, (void **)&c->indices, sizeof(int32_t) * n);
    return rc != ALS_OK ? rc : dev_alloc(ctx, (void **)&c->data, sizeof(float) * n);
  }
  cudaError_t e = cudaMallocHost((void **)&c->indices, sizeof(int32_t) * n);
  if (e == cudaSuccess) e = cudaMallocHost((void **)&c->data, sizeof(float) * n);
  return e == cudaSuccess ? ALS_OK : cuda_fail(e, "cudaMallocHost (host-resident CSR)", __FILE__, __LINE__);
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
  t->host = in->host;  // the transpose of a host-resident CSR is host-resident, built one column window at a time
  int rc;
  if (in->host || !in->segs.empty() || needs_segments(ctx, nnz)) {
    std::vector<int64_t> ip;
    if ((rc = csr_alloc(ctx, t)) != ALS_OK || (rc = transpose_segmented(ctx, in, t, 0, ip)) != ALS_OK ||
        (rc = csr_layout(ctx, t, ip.data())) != ALS_OK) {
      cudaStreamSynchronize(ctx->stream);  // D2H copies of a window may still be landing in t's arrays
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

int csr_column_counts(als_ctx *ctx, const als_csr *in, int64_t *counts) {
  ALS_CUDA(cudaSetDevice(ctx->device));
  unsigned long long *count = nullptr;
  int rc = dev_alloc(ctx, (void **)&count, sizeof(long long) * std::max<int64_t>(in->cols, 1));
  if (rc != ALS_OK) return rc;
  ALS_CUDA(cudaMemsetAsync(count, 0, sizeof(long long) * in->cols, ctx->stream));
  rc = column_histogram(ctx, in, count);
  if (rc == ALS_OK && in->cols) {
    ALS_CUDA(cudaMemcpyAsync(counts, count, sizeof(long long) * in->cols, cudaMemcpyDeviceToHost, ctx->stream));
  }
  dev_free(ctx, count);
  ALS_CUDA(cudaStreamSynchronize(ctx->stream));
  return rc;
}

// One device transpose of the shard into a scratch CSR, in global row ids; piece q is then copied out of its rows
// [col_bounds[q], col_bounds[q + 1]) and laid out.  The scratch costs one more copy of the shard's transpose, freed
// before this returns; a transpose per window would instead sort the whole shard once per piece.
int csr_transpose_pieces(als_ctx *ctx, const als_csr *in, int n, const int64_t *col_bounds, als_csr **pieces) {
  ALS_CUDA(cudaSetDevice(ctx->device));
  for (int q = 0; q < n; ++q) pieces[q] = nullptr;
  als_csr *t = new als_csr();
  t->ctx = ctx;
  t->rows = in->cols;
  t->cols = in->row_offset + in->rows;
  t->nnz = in->nnz;
  std::vector<int64_t> ip;
  int rc = csr_alloc(ctx, t);
  if (rc == ALS_OK) rc = transpose_segmented(ctx, in, t, in->row_offset, ip);
  for (int q = 0; q < n && rc == ALS_OK; ++q) {
    const int64_t r0 = col_bounds[q], r1 = col_bounds[q + 1];
    als_csr *p = new als_csr();
    pieces[q] = p;
    p->ctx = ctx;
    p->rows = r1 - r0;
    p->cols = t->cols;
    p->nnz = ip[r1] - ip[r0];
    if ((rc = csr_alloc(ctx, p)) != ALS_OK) break;
    if (p->nnz) {
      ALS_CUDA(cudaMemcpyAsync(p->indices, t->indices + ip[r0], sizeof(int32_t) * p->nnz, cudaMemcpyDeviceToDevice,
                               ctx->stream));
      ALS_CUDA(cudaMemcpyAsync(p->data, t->data + ip[r0], sizeof(float) * p->nnz, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    std::vector<int64_t> pip(ip.begin() + r0, ip.begin() + r1 + 1);
    for (int64_t &v : pip) v -= ip[r0];
    rc = csr_layout(ctx, p, pip.data(), /*schedule=*/false);  // copied by the merge, rarely solved
  }
  als_csr_destroy(t);  // stream ordered: after the copies above
  if (rc != ALS_OK) {
    cudaStreamSynchronize(ctx->stream);
    for (int q = 0; q < n; ++q) {
      als_csr_destroy(pieces[q]);
      pieces[q] = nullptr;
    }
  }
  return rc;
}

int csr_merge_rows(als_ctx *ctx, int n, const als_csr *const *pieces, int64_t cols, int64_t row_offset, als_csr **out) {
  *out = nullptr;
  ALS_CUDA(cudaSetDevice(ctx->device));
  const int64_t rows = pieces[0]->rows;
  // ips[p]: piece p's indptr, rebased to its first nonzero; dst[p][r]: where its row r starts in the output
  // (csr_indptr64 positions count from the piece's indices pointer: base[p] is its first nonzero)
  std::vector<std::vector<int64_t>> ips(n);
  std::vector<int64_t> base(n), oip((size_t)rows + 1, 0);
  for (int p = 0; p < n; ++p) {
    int rc = csr_indptr64(ctx, pieces[p], ips[p]);
    if (rc != ALS_OK) return rc;
    base[p] = ips[p][0];
    for (int64_t &v : ips[p]) v -= base[p];
    for (int64_t r = 0; r < rows; ++r) oip[r + 1] += ips[p][r + 1] - ips[p][r];
  }
  for (int64_t r = 0; r < rows; ++r) oip[r + 1] += oip[r];
  std::vector<int64_t> tables((size_t)n * (2 * rows + 1));  // per piece: ip[0 .. rows], then dst[0 .. rows - 1]
  std::vector<int64_t> at(oip.begin(), oip.end() - 1);
  for (int p = 0; p < n; ++p) {
    int64_t *tb = tables.data() + (size_t)p * (2 * rows + 1);
    std::copy(ips[p].begin(), ips[p].end(), tb);
    for (int64_t r = 0; r < rows; ++r) {
      tb[rows + 1 + r] = at[r];
      at[r] += ips[p][r + 1] - ips[p][r];
    }
  }
  als_csr *c = new als_csr();
  c->ctx = ctx;
  c->rows = rows;
  c->cols = cols;
  c->nnz = oip[rows];
  c->row_offset = row_offset;
  long long *tables_dev = nullptr;
  int rc = csr_alloc(ctx, c);
  if (rc == ALS_OK) rc = dev_alloc(ctx, (void **)&tables_dev, sizeof(int64_t) * tables.size());
  if (rc == ALS_OK) rc = merge_pieces(ctx, n, pieces, base, tables, tables_dev, c);
  dev_free(ctx, tables_dev);
  if (rc == ALS_OK) rc = csr_layout(ctx, c, oip.data());
  if (rc != ALS_OK) {
    cudaStreamSynchronize(ctx->stream);
    als_csr_destroy(c);
    return rc;
  }
  *out = c;
  return ALS_OK;
}

// One kernel per segment writes its share of the output indptr; one copy of that indptr (and of every segment's first
// position) to the host; then every segment's entries are one asynchronous device-to-device copy each, and the layout
// cuts the result into segments above the cap and builds its schedule.
int csr_concat_rows(als_ctx *ctx, int n, const als_csr *const *pieces, int64_t cols, int64_t row_offset, als_csr **out) {
  *out = nullptr;
  ALS_CUDA(cudaSetDevice(ctx->device));
  struct Seg {
    const als_csr *S;
    int64_t row, pos;  // its first row and first nonzero in the output
  };
  std::vector<Seg> segs;
  int64_t rows = 0, nnz = 0;
  for (int p = 0; p < n; ++p) {
    int64_t pos = nnz;
    for (const als_csr *S : segments_of(pieces[p])) {
      segs.push_back({S, rows + (S->row_offset - pieces[p]->row_offset), pos});
      pos += S->nnz;
    }
    rows += pieces[p]->rows;
    nnz += pieces[p]->nnz;
  }
  const int64_t ns = (int64_t)segs.size();
  als_csr *c = new als_csr();
  c->ctx = ctx;
  c->rows = rows;
  c->cols = cols;
  c->nnz = nnz;
  c->row_offset = row_offset;
  long long *ip_dev = nullptr;  // the output indptr (rows + 1), then the segments' first positions (ns)
  std::vector<int64_t> ip((size_t)(rows + 1 + ns));
  int rc = csr_alloc(ctx, c);
  if (rc == ALS_OK) rc = dev_alloc(ctx, (void **)&ip_dev, sizeof(int64_t) * ip.size());
  for (int64_t k = 0; k < ns && rc == ALS_OK; ++k) {
    const Seg &g = segs[k];
    const int blocks = (int)std::min<int64_t>((g.S->rows + 256) / 256, (int64_t)ctx->sm_count * 8);
    concat_indptr_kernel<<<blocks, 256, 0, ctx->stream>>>(g.S->indptr, g.S->rows, g.pos, ip_dev + g.row, ip_dev + rows + 1 + k);
    ALS_CUDA(cudaGetLastError());
    ctx->launches++;
  }
  if (rc == ALS_OK) {
    ALS_CUDA(cudaMemcpyAsync(ip.data(), ip_dev, sizeof(int64_t) * ip.size(), cudaMemcpyDeviceToHost, ctx->stream));
    ALS_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int64_t k = 0; k < ns; ++k) {
      const Seg &g = segs[k];
      if (!g.S->nnz) continue;
      const int64_t first = ip[rows + 1 + k];
      ALS_CUDA(cudaMemcpyAsync(c->indices + g.pos, g.S->indices + first, sizeof(int32_t) * g.S->nnz,
                               cudaMemcpyDeviceToDevice, ctx->stream));
      ALS_CUDA(cudaMemcpyAsync(c->data + g.pos, g.S->data + first, sizeof(float) * g.S->nnz, cudaMemcpyDeviceToDevice,
                               ctx->stream));
    }
  }
  dev_free(ctx, ip_dev);
  if (rc == ALS_OK) rc = csr_layout(ctx, c, ip.data());
  if (rc != ALS_OK) {
    cudaStreamSynchronize(ctx->stream);
    als_csr_destroy(c);
    return rc;
  }
  *out = c;
  return ALS_OK;
}

}  // namespace als
