/*
 * als_b200.h -- C-ABI of libals_b200.so: the H100 (sm_90a) ALS fit / recommend hot path.
 *
 * This is the drop-in boundary for benfred/implicit's ALS hot path.  Every entry point names the
 * reference interface it replaces (file:line relative to the reference repository).  The reference
 * crosses into native code through two Cython modules (implicit/cpu/_als.pyx, implicit/cpu/topk.pyx)
 * and, on its own GPU path, through C++ classes wrapped by implicit/gpu/_cuda.pyx
 * (LeastSquaresSolver implicit/gpu/als.h:11-24, KnnQuery implicit/gpu/knn.h:20-23,
 * Matrix/CSRMatrix implicit/gpu/matrix.h:18-113).  This header is the C equivalent of that second,
 * device-resident boundary: opaque device containers + solver entry points.
 *
 * Conventions
 *   - plain C, no exceptions: every function returns 0 on success, a negative ALS_E_* code on
 *     failure; als_last_error() returns a human-readable message for the calling thread's last
 *     failure (replaces CHECK_CUDA / std::runtime_error, implicit/gpu/utils.h:15-61).
 *   - the caller owns every host buffer; the library owns device memory until *_destroy.
 *   - one als_ctx per device per process; a ctx owns one compute stream and one copy stream.
 *     Calls on one ctx must not be issued concurrently from several host threads.
 *   - all solver calls are asynchronous on the ctx stream unless they return data to the host;
 *     als_sync() is the explicit join.
 *   - CSR is (indptr int32[rows+1], indices int32[nnz], data float32[nnz]) for als_csr_upload, and indptr
 *     int64[rows+1] with int32 or int64 indices for als_csr_upload64 (scipy's arrays past 2^31 nonzeros).
 *     rows and cols stay below 2^31 - 1.  On the device a CSR of more nonzeros than the segment cap (2^31 - 1
 *     by default, knob "segment_nnz") is held as row-block segments of int32 positions; every call takes either.
 *   - factor matrices are float32 row-major [rows, factors] on the host; on the device they are
 *     stored with the row stride padded to a multiple of 16 floats (zero filled).
 */
#ifndef ALS_B200_H_
#define ALS_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALS_B200_ABI_VERSION 1

enum {
  ALS_OK = 0,
  ALS_E_INVALID = -1,   /* bad argument */
  ALS_E_CUDA = -2,      /* CUDA runtime / driver error */
  ALS_E_NCCL = -3,      /* NCCL error or NCCL not loadable */
  ALS_E_UNSUPPORTED = -4,
  ALS_E_NOT_POSDEF = -5 /* Cholesky hit a non-positive pivot (reference: posv info != 0, implicit/cpu/_als.pyx:131-138) */
};

typedef struct als_ctx als_ctx;
typedef struct als_csr als_csr;
typedef struct als_factors als_factors;

/* ---- context -------------------------------------------------------------------------------- */
int als_abi_version(void);
/* Message for the calling thread's most recent failing call ("" if none). */
const char *als_last_error(void);
/* Number of visible CUDA devices (0 when there is no GPU / no driver). */
int als_device_count(void);
/* Replaces implicit/gpu/__init__.py HAS_CUDA probe + per-object device selection (matrix.cu:241). */
int als_ctx_create(int device, als_ctx **out);
int als_ctx_destroy(als_ctx *ctx);

/* Measurement knobs ("short_max" 0/16/32/48, "short_serial", "whiten_fma", "gramian_fma", "topk_legacy", "cg_nv" 1/2/4,
 * "segment_nnz": 0 = automatic, else the most nonzeros of one row-block segment of a device CSR; "host_csr": the Python
 * fit() keeps Cui / Ciu host-resident even when they fit in device memory).  The
 * environment variables ALS_B200_<KNOB> are read once, in als_ctx_create, and reported on stderr when set; this
 * call changes a knob afterwards (A/B tools).  Results do not depend on any knob beyond fp32 rounding; segment_nnz and
 * host_csr change no bit.  als_ctx_get_knob reads one back.
 * (No reference equivalent.) */
int als_ctx_set_knob(als_ctx *ctx, const char *name, int value);
int als_ctx_get_knob(als_ctx *ctx, const char *name, int *value);
/* Free and total device memory in bytes.  Blocks the context's stream-ordered pool keeps for reuse count as free
 * (cudaMemGetInfo alone under-reports after a fit has freed its arrays).  Synchronises the compute stream. */
int als_mem_info(als_ctx *ctx, int64_t *free_bytes, int64_t *total_bytes);
/* Bytes of the device's stream-ordered pool (every CSR, scratch array and temporary the library allocates per call) in
 * use now, and the most in use at any moment since the previous call; the mark then restarts at the current use.
 * Synchronises the compute stream.  (Measurement entry; no reference equivalent.) */
int als_mem_peak(als_ctx *ctx, int64_t *used_bytes, int64_t *peak_bytes);

/* Join the ctx streams (replaces the cudaDeviceSynchronize after every call, implicit/gpu/als.cu:147,151,196). */
int als_sync(als_ctx *ctx);
/* name[256]; sm count; L2 bytes; total global memory bytes. */
int als_device_info(als_ctx *ctx, char *name, int *sm_count, int64_t *l2_bytes, int64_t *mem_bytes);
/* Kernels launched on this ctx since creation (bench.py "gpu_launches"). */
int64_t als_launch_count(als_ctx *ctx);
/* CUDA-event timer on the ctx compute stream: start ... stop -> elapsed milliseconds. */
int als_timer_start(als_ctx *ctx);
int als_timer_stop(als_ctx *ctx, float *ms);
/* Write `bytes` of device scratch (L2 flush between timed iterations). */
int als_flush_l2(als_ctx *ctx, int64_t bytes);
/* Per-kernel device timing for bench.py's roofline: when enabled, every launch of a hot-path kernel
 * is bracketed by CUDA events on the ctx stream.  which: 0 gramian, 1 cholesky (rows + chunks),
 * 2 cholesky finish (giant rows), 3 cg (warp per row), 4 cg (giant rows), 5 topk, 6 loss.
 * als_profile_read synchronises, returns the summed milliseconds and launch count, and resets. */
int als_profile_enable(als_ctx *ctx, int on);
int als_profile_read(als_ctx *ctx, int which, double *ms_total, int64_t *launches);
/* Page-locked host memory for inputs that are uploaded inside a timed region. */
int als_host_alloc(void **ptr, int64_t bytes);
int als_host_free(void *ptr);

/* ---- sparse matrix --------------------------------------------------------------------------- */
/* Upload a CSR (or a contiguous row shard of one: `rows` local rows that are global rows
 * [row_offset, row_offset + rows) of the other side's factor matrix) and build its launch
 * schedule (rows sorted longest first, giant rows split).
 * Replaces CSRMatrix::CSRMatrix(rows, cols, nonzeros, indptr, indices, data), implicit/gpu/matrix.cu:222-251. */
int als_csr_upload(als_ctx *ctx, int64_t rows, int64_t cols, int64_t nnz, const int32_t *indptr,
                   const int32_t *indices, const float *data, int64_t row_offset, als_csr **out);
/* The same for any nnz (the reference's loops take int32 and int64 indices, implicit/cpu/_als.pyx:76-77): int64
 * indptr, indices of index_bytes = 4 or 8 bytes, narrowed to int32 while they are staged.  Refuses (ALS_E_INVALID,
 * naming the position) an index outside [0, cols), a non-monotone indptr and indptr[rows] - indptr[0] != nnz.  Above
 * the segment cap the CSR is stored as row-block segments of at most 2^30 nonzeros (or segment_nnz). */
int als_csr_upload64(als_ctx *ctx, int64_t rows, int64_t cols, int64_t nnz, const int64_t *indptr,
                     const void *indices, int index_bytes, const float *data, int64_t row_offset, als_csr **out);
/* The same arguments and refusals, for a CSR larger than device memory: indices / data stay in page-locked host memory
 * (indices narrowed to int32 while they are copied there) and the CSR is always held as row-block segments of at most
 * 2^28 nonzeros (or segment_nnz).  The segment indptrs, schedules and weight range live on the device.  Every solve,
 * the loss and als_csr_transpose stream the segments through a two-slot device ring, the copy of one segment under the
 * compute of the one before it, with bitwise the factors of the device-resident CSR of the same segment cap.
 * als_csr_transpose of it is host-resident too, built in column windows bounded by free device memory.
 * als_csr_slice_rows and als_topk's `liked` refuse it (ALS_E_UNSUPPORTED). */
int als_csr_upload_host64(als_ctx *ctx, int64_t rows, int64_t cols, int64_t nnz, const int64_t *indptr,
                          const void *indices, int index_bytes, const float *data, int64_t row_offset, als_csr **out);
/* The arguments and refusals of als_csr_upload64, with every array in device memory of the context's device (or managed
 * memory): indptr of indptr_bytes = 4 or 8, indices of index_bytes = 4 or 8, values of data_bytes = 4 (fp32) or 8 (fp64,
 * rounded to fp32).  The arrays are taken whole: indices / data hold exactly nnz entries and indptr[0] must be 0 (a row
 * shard is rows of its own arrays, with row_offset its first row).  The copy is ordered after the work queued so far on producer_stream (a cudaStream_t as an integer;
 * 0: none).  Device kernels narrow the indices and values into arrays the library owns, and check every index and the
 * indptr; a refusal names the position als_csr_upload64 names for the same input, in the same words.  Only the indptr
 * comes to the host (8 bytes per row, for the layout and the schedule).  The caller's memory is never aliased: it has been
 * read when the call returns.  The CSR is device-resident and segmented above the segment cap like als_csr_upload64's.
 * Refuses pointers that are not device memory of the context's device (ALS_E_INVALID).  (No reference equivalent; the
 * reference's GPU Matrix wraps __cuda_array_interface__ memory, implicit/gpu/_cuda.pyx:97-103.) */
int als_csr_upload_device(als_ctx *ctx, int64_t rows, int64_t cols, int64_t nnz, const void *indptr, int indptr_bytes,
                          const void *indices, int index_bytes, const void *data, int data_bytes, int64_t row_offset,
                          uint64_t producer_stream, als_csr **out);
/* *host = 1 for a host-resident CSR (als_csr_upload_host64 or its transpose), else 0. */
int als_csr_is_host(const als_csr *csr, int *host);
/* Number of row-block segments of the device layout (1 for a CSR within the segment cap). */
int als_csr_segment_count(const als_csr *csr, int64_t *n);
/* Synthetic inputs generated on the device (BASELINE.json configs too large to build on the host, e.g. C4:
 * 10M x 1M, 500M nonzeros): the power-law CSR recipe of SURVEY.md section 8(d) with counter-based hashing
 * (deterministic per seed, statistically equivalent to implicit_b200/synthetic.py, not bit-identical), and
 * factors = scale * U[0,1) like the reference's initialisation (implicit/cpu/als.py:144-147).
 * (No reference equivalent: it reads datasets from disk, implicit/datasets/.) */
int als_csr_generate(als_ctx *ctx, int64_t rows, int64_t cols, int64_t nnz_target, uint64_t seed, als_csr **out);
int als_factors_fill_uniform(als_ctx *ctx, als_factors *f, uint64_t seed, float scale);

/* Device transpose: out = in^T as CSR (replaces the host `Cui.T.tocsr()`, implicit/cpu/als.py:137).
 * Asynchronous: the launch schedule of `out` is built at the first solve that uses it. */
int als_csr_transpose(als_ctx *ctx, const als_csr *in, als_csr **out);
/* A view of rows [r0, r1) of `in` as a shard (row_offset = r0) with its own schedule; shares the
 * parent's device arrays, so the parent must outlive it.  The view of a segmented CSR is segmented itself; its shape
 * is the shard's.  (No reference equivalent: multi-GPU sharding.) */
int als_csr_slice_rows(als_ctx *ctx, const als_csr *in, int64_t r0, int64_t r1, als_csr **out);
/* The transpose of a row-sharded matrix without the whole matrix on one device (multi-GPU fit; no reference
 * equivalent).  Rank p uploads its user rows as a shard (row_offset = its first row), then:
 *   als_csr_column_counts: counts[c] = entries of column c in the CSR (host int64[cols]); summed over ranks
 *     (als_comm_allreduce_i64) they are the row lengths of the whole transpose, from which the item split is planned.
 *   als_csr_transpose_pieces: the transpose of a device-resident CSR cut by col_bounds[0 = b_0 <= ... <= b_n = cols]
 *     into n CSRs: pieces[q] holds rows [b_q, b_q+1) of the transpose, numbered from 0, with the shard's global row
 *     ids as column indices (cols = row_offset + rows of the shard) and row_offset 0.  Segmented inputs are taken and
 *     a piece above the segment cap is segmented.  A host-resident CSR is refused (ALS_E_UNSUPPORTED).
 *   als_comm_exchange_csr sends piece q to rank q and receives the piece of every rank, then
 *   als_csr_merge_rows: n device-resident pieces of equal row count concatenated row by row, piece 0's row first,
 *     into one CSR of `cols` columns with the given row_offset.  Rank order is user order, so the result is exactly
 *     rows [b_p, b_p+1) of scipy's Cui.T.tocsr(), stored zeros and duplicates included, laid out like any CSR.
 *   als_csr_concat_rows: n device-resident CSRs of any row counts stacked in list order, piece 0's rows first (a vstack,
 *     not the row-by-row interleave of merge_rows), into one CSR of `cols` columns with the given row_offset.  When
 *     every rank holds only its own block of user rows, rank p uploads it in one piece per rank q (the rows of its block
 *     that fall in q's share of the user split, mostly none), the pieces go through als_comm_exchange_csr, and rank q
 *     stacks the W pieces it receives, which cover consecutive rows in rank order, into its user shard.  Flat,
 *     segmented and row-slice pieces are taken; the result is laid out with its launch schedule and segmented above
 *     the cap like any CSR.  A host-resident piece is refused (ALS_E_UNSUPPORTED). */
int als_csr_column_counts(als_ctx *ctx, const als_csr *csr, int64_t *counts);
int als_csr_transpose_pieces(als_ctx *ctx, const als_csr *shard, int n, const int64_t *col_bounds, als_csr **pieces);
int als_csr_merge_rows(als_ctx *ctx, int n, const als_csr *const *pieces, int64_t cols, int64_t row_offset,
                       als_csr **out);
int als_csr_concat_rows(als_ctx *ctx, int n, const als_csr *const *pieces, int64_t cols, int64_t row_offset,
                        als_csr **out);
/* data *= alpha on device (replaces `Cui = alpha * Cui`, implicit/cpu/als.py:133-134). */
int als_csr_scale(als_ctx *ctx, als_csr *csr, float alpha);
int als_csr_shape(const als_csr *csr, int64_t *rows, int64_t *cols, int64_t *nnz);
/* Copy the device CSR back (any pointer may be NULL).  als_csr_download needs nnz < 2^31 - 1 (int32 indptr);
 * als_csr_download64 writes an int64 indptr and takes any CSR. */
int als_csr_download(als_ctx *ctx, const als_csr *csr, int32_t *indptr, int32_t *indices, float *data);
int als_csr_download64(als_ctx *ctx, const als_csr *csr, int64_t *indptr, int32_t *indices, float *data);
int als_csr_destroy(als_csr *csr);

/* ---- dense factor matrices ------------------------------------------------------------------- */
/* Replaces Matrix::Matrix(rows, cols, data), implicit/gpu/matrix.cu:66-104.  1 <= factors <= 1024 (the bound of the
 * reference's CUDA solver, implicit/gpu/als.cu:177-178); the device row stride is the width rounded up to 16 (<= 128) or
 * to 128 (wider).  Both solvers cover every width. */
int als_factors_create(als_ctx *ctx, int64_t rows, int factors, als_factors **out);
/* host[nrows, factors] (row-major, unpadded) <-> device rows [row0, row0 + nrows). */
int als_factors_upload(als_ctx *ctx, als_factors *f, const float *host, int64_t row0, int64_t nrows);
int als_factors_download(als_ctx *ctx, const als_factors *f, float *host, int64_t row0, int64_t nrows);
/* Strided fp32 device memory <-> device rows [row0, row0 + nrows): row r of the caller's matrix starts ld >= factors
 * elements after row r - 1 (so t[:, :factors] of a wider row-major matrix is taken as it is).  Import zeroes the padding
 * columns [factors, stride) like als_factors_upload, after the work queued so far on producer_stream (0: none); export
 * writes the factors columns only.  Both refuse memory that is not device memory of the context's device (managed memory
 * is taken), and both synchronise: src has been read, and dst written, when they return. */
int als_factors_import_device(als_ctx *ctx, als_factors *f, const float *src, int64_t ld, int64_t row0, int64_t nrows,
                              uint64_t producer_stream);
int als_factors_export_device(als_ctx *ctx, const als_factors *f, float *dst, int64_t ld, int64_t row0, int64_t nrows);
/* Device memory of the context's device that the caller owns (the factor snapshots of the Python layer): cudaMalloc /
 * cudaFree.  cudaFree waits for the device, so work of any stream that still reads the block finishes first. */
int als_device_alloc(als_ctx *ctx, int64_t bytes, void **ptr);
int als_device_free(als_ctx *ctx, void *ptr);
/* Device memory from the context's stream-ordered pool (cudaMallocAsync / cudaFreeAsync on its stream), for
 * temporaries that only the library's calls on this context read: the free is ordered after the work queued so far on
 * the context's stream, not after other streams' work, and does not wait for the device. */
int als_pool_alloc(als_ctx *ctx, int64_t bytes, void **ptr);
int als_pool_free(als_ctx *ctx, void *ptr);
int als_factors_shape(const als_factors *f, int64_t *rows, int *factors, int *stride);
/* *has_nan = 1 if any element is NaN (device-side scan).  Replaces the host np.isnan pass of
 * RecommenderBase._check_factors, implicit/recommender_base.py:218-223. */
int als_factors_has_nan(als_ctx *ctx, const als_factors *f, int *has_nan);
int als_factors_destroy(als_factors *f);

/* ---- the hot path ---------------------------------------------------------------------------- */
/* G = Y^T Y (without lambda) into the ctx-resident Gramian buffer; G_host (factors*factors floats,
 * may be NULL) receives a copy.  Replaces np.dot(Y.T, Y) (implicit/cpu/_als.pyx:70,164,268) and
 * LeastSquaresSolver::calculate_yty (implicit/gpu/als.cu:122-152). */
int als_gramian(als_ctx *ctx, const als_factors *Y, float *G_host);
/* Copies the Gramian that the context holds (from the last als_gramian or als_gramian_shard on Y, which
 * must not have been followed by another Gramian) into G_host (factors*factors floats).  Test / tooling entry:
 * als_gramian_shard leaves its result on the device. */
int als_gramian_read(als_ctx *ctx, const als_factors *Y, float *G_host);

/* One Cholesky half-iteration: for every row u of C:  X[row_offset + u] = (Y^T Y + reg I + Y^T (|C_u| - I) Y)^-1 Y^T C_u+ p_u.
 * Computes the Gramian of Y itself.  *bad_row = -1, or the first (global) row whose normal
 * equations were not positive definite (then the call returns ALS_E_NOT_POSDEF).
 * Replaces _als.least_squares(Cui, X, Y, regularization, num_threads), implicit/cpu/_als.pyx:67-142. */
int als_least_squares(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y,
                      double regularization, int64_t *bad_row);
/* Same solve with a caller-supplied Gramian (host, factors*factors floats, WITHOUT lambda).
 * Replaces _als._least_squares(YtY, indptr, indices, data, X, Y, regularization, num_threads),
 * implicit/cpu/_als.pyx:76 (recalculate_user / partial_fit, implicit/cpu/als.py:221-240). */
int als_least_squares_with_gramian(als_ctx *ctx, const float *YtY_host, const als_csr *C, als_factors *X,
                                   const als_factors *Y, double regularization, int64_t *bad_row);

/* The per-half preprocessing of the short-row path, downloaded: W = Y P with Y^T Y + reg I = R^T R, P = R^-1
 * (whitened factors) and Z = Y (Y^T Y + reg I)^-1, both rows x factors floats.  Produced on the wgmma
 * tensor cores for 64 padded factors (csrc/dense.cu).  Test / tooling entry: the reference has no
 * counterpart (it forms every row's F x F normal equations, implicit/cpu/_als.pyx:96-130). */
int als_whitened_factors(als_ctx *ctx, const als_factors *Y, double regularization, float *W_host, float *Z_host);

/* Multi-GPU variants: the Gramian is accumulated over each rank's OWN rows [row0, row0 + nrows) of Y and
 * summed across ranks (ncclAllReduce of f x f floats on the ctx stream, which also orders this rank after
 * every peer's preceding solve); als_least_squares*_pregram then solve with that device-resident Gramian
 * instead of recomputing it from the full replica.  (No reference equivalent.) */
int als_gramian_shard(als_ctx *ctx, const als_factors *Y, int64_t row0, int64_t nrows);
int als_least_squares_pregram(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y,
                              double regularization, int64_t *bad_row);
/* The asynchronous flavour for the multi-GPU fit loop: queues the half and returns; a row that is not positive
 * definite is remembered on the device and its flag rides along with the next als_gramian_shard all-reduce, so
 * every rank learns of any rank's failure.  als_solver_status synchronises, reports (and clears) the first bad row
 * of THIS rank since the last call (-1: none; then returns ALS_E_NOT_POSDEF) and whether any rank failed. */
int als_least_squares_pregram_async(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y,
                                    double regularization);
int als_solver_status(als_ctx *ctx, int64_t *bad_row, int *any_rank_failed);
int als_least_squares_cg_pregram(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y,
                                 float regularization, int cg_steps);

/* One conjugate-gradient half-iteration, warm-started from X, updated in place.
 * Replaces _als.least_squares_cg(Cui, X, Y, regularization, num_threads, cg_steps),
 * implicit/cpu/_als.pyx:145-248, and LeastSquaresSolver::least_squares (implicit/gpu/als.cu:154-197). */
int als_least_squares_cg(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y,
                         float regularization, int cg_steps);

/* Training-loss terms over the rows of C (a whole matrix or a row shard):
 *   terms[0] = sum_u [x_u^T Y^T Y x_u + sum_i ((|c|-1)(y_i.x_u)^2 - 2 c+ (y_i.x_u) + |c|)] + reg * ||X_C||^2
 *   terms[1] = sum |c_ui|          terms[2] = reg * ||Y||^2
 * so that  loss = (sum_shards terms[0] + terms[2]) / (sum_shards terms[1] + users*items - nnz).
 * Replaces _als.calculate_loss(Cui, X, Y, regularization, num_threads), implicit/cpu/_als.pyx:251-308,
 * and LeastSquaresSolver::calculate_loss (implicit/gpu/als.cu:253-281). */
int als_calculate_loss(als_ctx *ctx, const als_csr *C, const als_factors *X, const als_factors *Y,
                       float regularization, double *terms /* [3] */);

/* Fused scores + filter + top-k:  for each query row q: top-k of items . q (optionally / item_norms),
 * with the columns in `liked` row q (CSR over the query rows, may be NULL) and the global list
 * filter_items set to -FLT_MAX first.  Queries are rows `query_rows[0..n_query)` of `queries`
 * (query_rows NULL = rows 0..n_query-1).  Outputs are host arrays [n_query, k], zero-initialised
 * by the callee like topk.pyx:20-21; tie-breaking follows implicit/cpu/select.h:12-39 exactly.
 * `liked` has n_query rows and fewer than 2^31 - 1 nonzeros (a segmented CSR is refused: split the queries); its
 * columns may come in any order within a row and may repeat (like the reference's
 * batch_distances[i, liked.indices] = -max).  The first call with a given `liked` checks the order on the device;
 * if a row is unsorted, a sorted copy is built once and kept with the handle (its nnz int32s) until it is destroyed.
 * Replaces topk.topk(items, query, k, item_norms, filter_query_items, filter_items, num_threads),
 * implicit/cpu/topk.pyx:15-67, and KnnQuery::topk (implicit/gpu/knn.cu:131-265). */
int als_topk(als_ctx *ctx, const als_factors *items, const als_factors *queries, const int32_t *query_rows,
             int64_t n_query, int k, const float *item_norms_host, const als_csr *liked,
             const int32_t *filter_items, int64_t n_filter, int32_t *ids_host, float *scores_host);
/* ---- serving from device ids: CUDA ids in, CUDA ids and scores out ------------------------------------------------
 * Every array below is device memory of the context's device (or managed memory); anything else is refused with
 * ALS_E_INVALID, naming the argument.  Ids are int32 (4 bytes) or int64 (8 bytes).  Each call is ordered after the
 * work queued so far on producer_stream (a cudaStream_t as an integer; 0: none) and has read its inputs and completed
 * its outputs when it returns (it synchronises).
 *
 * als_topk_into: the top-k of als_topk, written to ids / scores [n_query, k] that the caller allocated (als_device_alloc),
 * the tail past the items zero as in als_topk.  query_rows [n_query] (NULL: rows [query_row0, query_row0 + n_query) of
 * queries), item_norms [items rows] (NULL: none) and filter_items [n_filter] are device arrays; the query rows and the
 * filter are range-checked on the device before any top-k launch, and an id outside [0, queries rows) / [0, items rows)
 * returns ALS_E_INVALID with *bad = 1 (query_rows) | 2 (filter_items), nothing written.  One epilogue kernel reads the
 * top-k's scratch output and writes the caller's arrays: with id_map (NULL: none) each id becomes id_map[id], and ids
 * holds map_bytes per entry (else int32); with query_norms (NULL: none) each score becomes score / query_norms[r], r the
 * query's row of queries (fp32 division, as numpy's scores / norm[:, None]).  Shares als_topk's checks and top-k driver,
 * so the same inputs give bitwise als_topk's ids and scores. */
int als_topk_into(als_ctx *ctx, const als_factors *items, const als_factors *queries, const void *query_rows,
                  int query_row_bytes, int64_t query_row0, int64_t n_query, int k, const float *item_norms,
                  const float *query_norms, const als_csr *liked, const void *filter_items, int filter_bytes,
                  int64_t n_filter, const void *id_map, int map_bytes, uint64_t producer_stream, void *ids, float *scores,
                  int *bad);
/* A new factor matrix (*out) of the rows src[rows[i]], i < n, its padding columns zero (the wgmma top-k reads them).
 * rows are range-checked on the device first: an id outside [0, src rows) returns ALS_E_INVALID with *bad = 1 and
 * creates nothing. */
int als_factors_gather_rows(als_ctx *ctx, const als_factors *src, const void *rows, int row_bytes, int64_t n,
                            uint64_t producer_stream, als_factors **out, int *bad);
/* norms[r] = the fp32 norm of row r of f, bitwise numpy's np.linalg.norm(F, axis=-1): sqrt of numpy's pairwise float32
 * sum of the squares of exactly f->f elements (never the padding), every step rounded on its own; a zero norm is
 * written as zero_value (1e-10 for similar_items, implicit/cpu/matrix_factorization_base.py). */
int als_factors_row_norms(als_ctx *ctx, const als_factors *f, float zero_value, float *norms);
/* bytes of host memory copied to dst, device memory of the context's device (the host ids of a call whose other ids
 * are in CUDA memory). */
int als_device_upload(als_ctx *ctx, void *dst, const void *src, int64_t bytes);
/* bytes of device memory src (of the context's device) copied to the host: the sorted subset of a call whose liked
 * filter is a scipy CSR, remapped on the host. */
int als_device_download(als_ctx *ctx, void *dst, const void *src, int64_t bytes);
/* sorted[n] = ids[n] in ascending order (CUB radix sort; equal to numpy's sort of the same integers). */
int als_ids_sort(als_ctx *ctx, const void *ids, int id_bytes, int64_t n, uint64_t producer_stream, void *sorted);
/* The liked CSR remapped onto a column subset, as recommend(..., items=subset) remaps a scipy liked filter
 * (_filter_items_from_sparse_matrix): *out has liked's rows and m columns, and row r holds, sorted and once each, the
 * positions in subset[m] (ascending; searched like numpy's searchsorted(side="left")) of the columns of row r that
 * are in the subset and whose stored value is not 0.  Values are 1 (a liked filter reads positions only).  Built on
 * the device -- count, scan, scatter, a CUB segmented sort and unique per row -- and laid out by the one upload path
 * (the layout and max_row_nnz of the scipy remap uploaded with als_csr_upload).  liked must be one device-resident
 * CSR (not segmented, not host-resident). */
int als_csr_restrict_columns(als_ctx *ctx, const als_csr *liked, const void *subset, int subset_bytes, int64_t m,
                             uint64_t producer_stream, als_csr **out);
/* Ranking metrics at k of the top-k above, without its ids leaving the device: the ids als_topk would return (no item
 * norms, no filter_items; ranks past the items are id 0) are scored against `test`, a CSR over the query rows of the
 * withheld items (any order within a row, repeats and stored zeros allowed; sorted on the device like `liked`).  Per
 * query with L > 0 distinct withheld items and hit_j = "the id at rank j is withheld":
 *   sums[0] += sum_j hit_j                          sums[1] += min(k, L)
 *   sums[2] += sum_j hit_j * (hits at ranks <= j) / (j + 1) / min(k, L)
 *   sums[3] += sum_j hit_j * gain[j] / gain_sum[min(k, L) - 1]
 *   sums[4] += [sum_{miss j} (hits before j) + (hits + L) / 2 * (items - L - misses)] / (L * (items - L))
 *   sums[5] += 1
 * in fp64, with the caller's gain[k] (1 / log2(j + 2)) and gain_sum[k] (its running sum) tables.  Queries without
 * withheld items add nothing.  The sums are deterministic: two identical calls return the same bits.  Refuses what
 * als_topk refuses, k < 1, a `test` of other than n_query rows or other than items' row count of columns, and a
 * host-resident or segmented `test`.  Synchronises.
 * Replaces the per-user loop of ranking_metrics_at_k, implicit/evaluation.pyx:366-475 (precision = sums[0] / sums[1],
 * map, ndcg and auc = sums[2 .. 4] / sums[5]). */
int als_ranking_metrics(als_ctx *ctx, const als_factors *items, const als_factors *queries, const int32_t *query_rows,
                        int64_t n_query, int k, const als_csr *liked, const als_csr *test, const double *gain_host,
                        const double *gain_sum_host, double *sums /* [6] */);

/* ---- refitting rows in place from device ids ----------------------------------------------------------------------
 * The device side of partial_fit_users / partial_fit_items (implicit/cpu/als.py:267-349) for ids in CUDA memory: the
 * factor matrix grows and takes the recalculated rows where it lives, and no factor matrix crosses PCIe.  Ids and
 * producer_stream as in the serving calls above.
 *
 * *min_id / *max_id = the smallest and largest of ids[n] (n = 0: 0 and -1), in one pass and one 16-byte read-back
 * (synchronises): the caller refuses a negative id and grows the matrix to max + 1 rows, the max(userids) of
 * implicit/cpu/als.py:301-302. */
int als_ids_range(als_ctx *ctx, const void *ids, int id_bytes, int64_t n, uint64_t producer_stream, int64_t *min_id,
                  int64_t *max_id);
/* f grows to `rows` rows (not fewer than it has) in a new allocation of the same padded row stride: the old rows are
 * copied device to device and rows [old rows, rows) are zero, padding included -- np.concatenate([factors,
 * np.zeros(...)]) of implicit/cpu/als.py:302-305, uploaded.  The old and the new matrix are both allocated while the
 * copy runs.  Refused with ALS_E_INVALID, f unchanged: a matrix shared with other ranks (exported over CUDA IPC), and a
 * row count whose bytes would exceed the device's memory (so no byte count overflows, whatever id asked for it). */
int als_factors_grow(als_ctx *ctx, als_factors *f, int64_t rows);
/* dst[ids[i]] = src[i] for i < n (src has n rows and dst's width), with the semantics of numpy's factors[ids] = rows
 * (implicit/cpu/als.py:308, 345): of an id that repeats, the last occurrence wins, deterministically.  The (id,
 * position) pairs are radix-sorted (stable) and only the last pair of each id writes its row: the `factors` columns
 * from src, the padding columns as zeros.  Rows no id names keep their bits; an id outside [0, dst rows) is skipped,
 * never written (als_ids_range gives the caller the range to grow to).  Synchronises. */
int als_factors_scatter_rows(als_ctx *ctx, als_factors *dst, const void *ids, int id_bytes, int64_t n,
                             uint64_t producer_stream, const als_factors *src);

/* ---- multi-GPU (one process per GPU; NCCL over NVLink/NVSwitch) -------------------------------- */
/* The reference has no multi-GPU path (`// TODO: multi-gpu support`, implicit/gpu/als.cu:169). */
#define ALS_COMM_ID_BYTES 128
/* rank 0: fill id[128]; the host side ships it to the other ranks (implicit_b200/distributed.py). */
int als_comm_unique_id(void *id);
int als_comm_init(als_ctx *ctx, int rank, int world, const void *id);
int als_comm_destroy(als_ctx *ctx);
/* All-gather the row shards of a replicated factor matrix: rank r owns rows
 * [row_splits[r], row_splits[r+1]) and every rank ends with all rows. */
int als_comm_allgather_rows(als_ctx *ctx, als_factors *f, const int64_t *row_splits);
/* Fused exchange: instead of an all-gather AFTER a half-iteration, the solve kernels store every row they
 * produce straight into the other ranks' replicas over NVLink (peer memory mapped with CUDA IPC), so the
 * transfer rides under the compute.  export: this rank's 64-byte handle for f; attach: map the replicas of
 * all ranks (handles = world * 64 bytes, in rank order); after attach every als_least_squares* call that
 * writes f mirrors its rows.  The host must still join all ranks (als_sync + als_comm_barrier) before the
 * next half reads f. */
#define ALS_IPC_HANDLE_BYTES 64
int als_factors_ipc_export(als_ctx *ctx, const als_factors *f, void *handle);
int als_factors_ipc_attach(als_ctx *ctx, als_factors *f, int rank, int world, const void *handles);
int als_factors_ipc_detach(als_ctx *ctx, als_factors *f);
/* All-gather nbytes (<= 256) of host data per rank into recv[world * nbytes] (rank order). */
int als_comm_allgather_bytes(als_ctx *ctx, const void *send, void *recv, int nbytes);
/* In-place sum / max of n doubles across ranks (host values; used for loss terms and timing). */
int als_comm_allreduce_f64(als_ctx *ctx, double *values, int n, int op_max);
/* In-place exact sum of n int64 host values across ranks (any n; the column counts of a sharded transpose). */
int als_comm_allreduce_i64(als_ctx *ctx, int64_t *values, int64_t n);
/* send[world]: device-resident CSRs, send[q] goes to rank q; recv[world] receives a new device CSR from every rank p
 * (shape, indptr, indices and values, over grouped ncclSend / ncclRecv on the ctx stream).  Every rank must call it. */
int als_comm_exchange_csr(als_ctx *ctx, als_csr *const *send, als_csr **recv);
int als_comm_barrier(als_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif /* ALS_B200_H_ */
