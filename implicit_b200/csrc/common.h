// Internal declarations shared by the translation units of libals_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>
#include <stdio.h>

#include <algorithm>
#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "../../include/als_b200.h"

#define ALS_API extern "C" __attribute__((visibility("default")))

namespace als {

// ---- error plumbing (no exceptions cross the C boundary) ------------------------------------------
void set_error(const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what, const char *file, int line);

#define ALS_CUDA(expr)                                                        \
  do {                                                                        \
    cudaError_t e__ = (expr);                                                 \
    if (e__ != cudaSuccess) return ::als::cuda_fail(e__, #expr, __FILE__, __LINE__); \
  } while (0)

#define ALS_REQUIRE(cond, ...)            \
  do {                                    \
    if (!(cond)) {                        \
      ::als::set_error(__VA_ARGS__);      \
      return ALS_E_INVALID;               \
    }                                     \
  } while (0)

static inline int round_up(int x, int m) { return (x + m - 1) / m * m; }
static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---- work schedule ------------------------------------------------------------------------------
// One unit of work for the per-row solvers.  kind: 0 = whole row (k0..k1 = its nnz range),
// 1 = a chunk of a giant row (partial normal equations go to `slot`), 2 = finish a giant row
// (k0 = first slot, k1 = number of slots).
struct WorkItem {
  int32_t row;
  int32_t k0;
  int32_t k1;
  int32_t slot;  // -1: whole row; >= 0: chunk slot; -2: finish item
};

constexpr int kSplitNnz = 3072;   // rows longer than this are split ...
constexpr int kChunkNnz = 2048;   // ... into chunks of this many nonzeros (multiple of 8)

}  // namespace als

// Measurement knobs.  Read from the environment ONCE, in als_ctx_create (which reports every knob that is set on
// stderr); tools flip them afterwards with als_ctx_set_knob.  None changes results beyond fp32 rounding, except the
// test-only alloc_fail_at.
struct als_knobs {
  int short_max = 48;         // ALS_B200_SHORT_MAX: longest row (nonzeros) of the n x n short-row path: 0, 8, ..., 48
  int short_serial = 0;       // ALS_B200_SHORT_SERIAL: short-row kernels on the compute stream instead of the aux stream
  int whiten_fma = 0;         // ALS_B200_WHITEN_FMA: fp32 FMA tiles for W = Y P, Z = Y G^-1 instead of the wgmma apply
  int topk_legacy = 0;        // ALS_B200_TOPK_LEGACY: mma.sync top-k kernel for every call (no wgmma path)
  int gramian_fma = 0;        // ALS_B200_GRAMIAN_FMA: fp32 FMA Gramian instead of the wgmma one (64 padded factors)
  int long_tc = 0;            // ALS_B200_LONG_TC: experimental wgmma kernel for the long rows of a Cholesky half (cholesky_tc.cu)
  int cg_nv = 2;              // ALS_B200_CG_NV: float4 words per lane of the CG kernel (1 / 2 / 4)
  int64_t segment_nnz = 0;    // ALS_B200_SEGMENT_NNZ: nonzeros per row-block segment of a device CSR; 0: automatic (one
                              // segment below 2^31 - 1 nonzeros, else segments of at most 2^30; 2^28 for a host-resident
                              // CSR).  Changes no bit.
  int host_csr = 0;           // ALS_B200_HOST_CSR: fit() keeps Cui / Ciu in page-locked host memory and streams their
                              // segments through the device even when they fit in device memory.  Changes no bit.
  int alloc_fail_at = 0;      // test only, set with als_ctx_set_knob alone (no environment variable), and it changes
                              // results: n > 0 makes the n-th device allocation through dev_alloc or a DeviceBlock,
                              // counted from the set, return ALS_E_CUDA ("injected allocation failure") without calling
                              // CUDA; the knob is then 0 again.
};

struct als_ctx {
  int device = 0;
  als_knobs knobs;
  int sm_count = 0;
  int64_t l2_bytes = 0;
  int64_t mem_bytes = 0;
  char name[256] = {0};
  cudaStream_t stream = nullptr;   // compute
  cudaStream_t copy = nullptr;     // H2D / D2H staging
  cudaStream_t aux = nullptr;      // short-row kernels of a Cholesky half, concurrent with the full-size kernel
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  cudaStream_t class_stream[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};  // short-row size classes 2..6 (the first stays on aux)
  cudaEvent_t class_fork = nullptr, class_join[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int64_t launches = 0;
  // Gramian state: G (f_pad x f_pad, without lambda) and Greg (G + lambda I, identity on padded dims)
  float *G = nullptr;
  float *Greg = nullptr;
  float *gram_partials = nullptr;
  int64_t gram_partials_cap = 0;  // bytes
  // per-launch scalars, see the kCtr* slots below (16 ints, zeroed before every half)
  int32_t *counters = nullptr;
  long long *bad_row = nullptr;   // [0] first non-PD row of the current half, [1] of the halves since als_solver_status
  int32_t *status = nullptr;      // [0] sticky: some rank reported a failed half (rides on the Gramian all-reduce)
  int gram_ld = 0;                // ld of the last regularised Gramian: G[ld * ld] is the failure flag slot
  double *dscalars = nullptr;  // loss accumulators (8 doubles)
  // short-row path of the Cholesky half (cholesky_short.cu): P = R^-1 with G + lambda I = R^T R, the whitened
  // factors W = Y P, and the list of short items handed back to the full-size kernel
  float *Pinv = nullptr;      // 2^14 P (upper triangular)
  float *Ginv = nullptr;      // G^-1 = P P^T
  float *whitened = nullptr;  // W = Y (2^14 P)
  int64_t whitened_bytes = 0;
  float *zfactors = nullptr;  // Z = Y G^-1
  int64_t zfactors_bytes = 0;
  float *dense_bt = nullptr;  // [2^14 P | G^-1]^T split into TF32 hi / lo parts for the wgmma apply (dense.cu)
  als::WorkItem *deferred = nullptr;
  int64_t deferred_cap = 0;
  // generic scratch (giant-row partial slots, L2 flush, top-k staging)
  void *scratch = nullptr;
  int64_t scratch_bytes = 0;
  // staged uploads of pageable host memory (api.cu h2d_copy): 4 threads x 2 page-locked 4 MB buffers, own streams
  void *stage_buf = nullptr;
  cudaStream_t stage_stream[4] = {nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t stage_ev[4][2] = {{nullptr, nullptr}, {nullptr, nullptr}, {nullptr, nullptr}, {nullptr, nullptr}};
  cudaEvent_t stage_ready = nullptr;
  // the two-slot device ring that streams the segments of a host-resident CSR (csr.cu for_each_segment): a slot is
  // loaded (ring_loaded, on the copy stream) and free again once every launch that read it has finished (ring_free)
  cudaEvent_t ring_loaded[2] = {nullptr, nullptr}, ring_free[2] = {nullptr, nullptr};
  // per-kernel profiling (als_profile_*)
  bool profiling = false;
  std::vector<cudaEvent_t> prof_events[8];  // pairs (start, stop) per category
  // NCCL
  void *comm = nullptr;
  int rank = 0, world = 1;
};

struct als_factors {
  als_ctx *ctx = nullptr;
  int64_t rows = 0;
  int f = 0;   // logical factors
  int ld = 0;  // device row stride (multiple of 16, zero padded)
  float *d = nullptr;
  bool pooled = true;  // d comes from the stream-ordered pool (moved to a cudaMalloc block when exported over IPC)
  // peer replicas of the same matrix on the other ranks (CUDA IPC mappings over NVLink): the solve kernels
  // mirror every row they write into these, which replaces the all-gather after a half-iteration
  float **peers_dev = nullptr;  // device array of n_peers base pointers (self excluded)
  int n_peers = 0;
  std::vector<void *> peer_maps;  // what cudaIpcOpenMemHandle returned, for closing
};

struct als_csr {
  als_ctx *ctx = nullptr;
  int64_t rows = 0, cols = 0, nnz = 0, row_offset = 0;
  int32_t *indptr = nullptr;
  int32_t *indices = nullptr;
  float *data = nullptr;
  bool owns = true;  // false for a row-slice view sharing its parent's arrays
  // schedule
  als::WorkItem *work = nullptr;    // main pass: whole rows + chunks, longest first
  int64_t n_work = 0;
  // work is sorted by length, so the items of at most 48 / 40 / ... / 8 / 0 nonzeros are suffixes: first index of each
  int64_t le_begin[7] = {0, 0, 0, 0, 0, 0, 0};
  int64_t max_row_nnz = 0;     // longest row (known once the schedule is built)
  unsigned *wmax_dev = nullptr;  // device: [0] bits of max | |c| - 1 | over the values, [1] != 0 when some |c| < 1 (cholesky.cu), computed lazily
  bool wmax_valid = false;
  bool neg_w_known = false, has_neg_w = false;  // host copy of wmax_dev[1]: weights |c| - 1 < 0 exist (then no wgmma long-row path)
  // laid out without schedules (the pieces of a sharded transpose, which are only copied): ensure_schedule builds them
  // from the device indptrs at the first solve
  bool sched_lazy = false;
  // as the liked lists of als_topk, whose fused kernels walk each row's columns in ascending order: checked once on
  // the device at first use; a CSR with an unsorted row gets a sorted copy (indptr rebased to 0) kept for later calls
  bool order_known = false;
  int32_t *sorted_indptr = nullptr;
  int32_t *sorted_indices = nullptr;
  als::WorkItem *finish = nullptr;  // finish pass: one per giant row (row, first slot, #slots)
  int64_t n_finish = 0;
  int64_t n_slots = 0;
  als::WorkItem *chunks = nullptr;  // the n_slots chunk items in slot order (CG walks them pass by pass)
  int32_t *chunk_owner = nullptr;   // chunk -> index of its row in `finish`
  // A CSR above the segment cap is a list of row-block segments, each an ordinary int32 CSR of whole rows: its own
  // rebased indptr (in seg_indptr), indices / data offset into this CSR's arrays, its own schedule, row_offset = its
  // first row.  The segments are non-owning children destroyed with this CSR; its own indptr and schedule stay empty,
  // and wmax_dev, has_neg_w and max_row_nnz cover all segments.  Empty: one segment, the CSR itself.
  std::vector<als_csr *> segs;
  int32_t *seg_indptr = nullptr;  // the segments' indptrs, concatenated (rows + segs.size() entries)
  // Host-resident (als_csr_upload_host64, or the transpose of such a CSR): indices / data are page-locked host arrays and
  // always segmented; seg_indptr, the schedules and wmax_dev stay on the device.  Every solve streams the segments through
  // a device ring (for_each_segment); wmax_dev is computed on the host, so it is always valid.
  bool host = false;
};

namespace als {

// RAII bracket: records start/stop events around a kernel launch when profiling is on.
struct ProfScope {
  als_ctx *ctx;
  int which;
  ProfScope(als_ctx *c, int w);
  ~ProfScope();
};
enum { kProfGramian = 0, kProfCholesky = 1, kProfCholFinish = 2, kProfCg = 3, kProfCgGiant = 4, kProfTopk = 5, kProfLoss = 6 };

// slots of als_ctx::counters
enum {
  kCtrMain = 0, kCtrFinish = 1, kCtrDeferredCount = 2, kCtrDeferredWork = 3, kCtrWhitenOk = 4, kCtrHasNan = 5, kCtrYAbsMax = 6,
  kCtrChunks = 7,
  kCtrIdsBad = 14,  // out-of-range bits of the device ids of a top-k (serve.cu stage_ids)
  kCtrWeightBad = 15,  // a refused index of the weighting calls (weight.cu)
  kCtrShort = 8 /* +0..5: one per short-row size class */
};
// size classes of the short-row path: als_csr::le_begin[i] is the first work item of at most kShortThresholds[i] nonzeros
constexpr int kNumShortThresholds = 7;
constexpr int kShortThresholds[kNumShortThresholds] = {48, 40, 32, 24, 16, 8, 0};

// Device memory comes from CUDA's stream-ordered pool on ctx->stream with the release threshold lifted, so the
// arrays of a second fit() are served from what the first one freed (cudaMalloc / cudaFree cost 0.1-1 ms each and
// cudaFree synchronises the device).  Factor matrices exported over CUDA IPC are the exception (api.cu).
int dev_alloc(als_ctx *ctx, void **ptr, int64_t bytes, cudaStream_t stream = nullptr);  // nullptr: ctx->stream
void dev_free(als_ctx *ctx, void *ptr);

// The owner of one temporary device block: a pool block (alloc, through dev_alloc) freed stream-ordered on ctx->stream,
// or a cudaMalloc block (alloc_cuda) freed with cudaFree, when the owner dies or at reset().  release() hands the block
// to a handle, whose destroy function frees it from then on.  Before an owner dies, every stream that touched its block
// has been joined into ctx->stream or synchronised: an error return from a section forked onto other streams joins them
// first.
class DeviceBlock {
 public:
  DeviceBlock() = default;
  DeviceBlock(const DeviceBlock &) = delete;
  DeviceBlock &operator=(const DeviceBlock &) = delete;
  DeviceBlock(DeviceBlock &&o) noexcept : ctx_(o.ctx_), p_(o.p_), pooled_(o.pooled_) { o.p_ = nullptr; }
  DeviceBlock &operator=(DeviceBlock &&o) noexcept;
  ~DeviceBlock() { reset(); }
  int alloc(als_ctx *ctx, int64_t bytes, cudaStream_t stream = nullptr);
  int alloc_cuda(als_ctx *ctx, int64_t bytes);
  void reset();

 protected:
  void *take() {
    void *p = p_;
    p_ = nullptr;
    return p;
  }
  als_ctx *ctx_ = nullptr;
  void *p_ = nullptr;
  bool pooled_ = true;
};

// A DeviceBlock of T elements (the byte count is the caller's).
template <typename T>
class Dev : public DeviceBlock {
 public:
  T *get() const { return static_cast<T *>(p_); }
  operator T *() const { return get(); }
  T *release() { return static_cast<T *>(take()); }
};

// A CSR under construction: destroyed once ctx->stream has finished with it, unless released to the caller.
struct CsrDestroy {
  void operator()(als_csr *c) const;
};
using CsrHolder = std::unique_ptr<als_csr, CsrDestroy>;
// a new empty CSR of ctx
CsrHolder new_csr(als_ctx *ctx);

int ensure_schedule(als_ctx *ctx, als_csr *csr);

int ensure_scratch(als_ctx *ctx, int64_t bytes);
int ensure_device_buffer(als_ctx *ctx, void **buf, int64_t *cap, int64_t bytes);
int build_schedule(als_ctx *ctx, als_csr *csr, const int32_t *indptr_host);
// the segments a solve walks: the CSR itself, or its row-block segments in row order
static inline std::vector<const als_csr *> segments_of(const als_csr *c) {
  if (c->segs.empty()) return {c};
  return std::vector<const als_csr *>(c->segs.begin(), c->segs.end());
}
// the largest segment: the knob, else 2^30 (2x headroom on the kernels' int32 positions); 2^28 for a host-resident CSR,
// whose two-slot device ring then takes 4 GB
static inline int64_t segment_cap(const als_ctx *ctx, bool host = false) {
  return ctx->knobs.segment_nnz > 0 ? ctx->knobs.segment_nnz : (int64_t)1 << (host ? 28 : 30);
}
// Runs launch(s, S) for every segment of C in row order.  For a host-resident C, segment s + 1 is copied into a two-slot
// device ring on ctx->copy while segment s computes, and S is a view of segment s whose indices / data point into its
// slot.  launch must queue its work on ctx->stream, or join every other stream it uses back into ctx->stream before it
// returns: a slot is refilled only after ctx->stream has passed that point.
// with_data = false stages the indices only (launch must not read S->data).
using SegmentLaunch = std::function<int(size_t s, const als_csr *S)>;
int for_each_segment(als_ctx *ctx, const als_csr *C, const SegmentLaunch &launch, bool with_data = true);
// free device memory, counting the blocks the stream-ordered pool keeps for reuse as free (synchronises ctx->stream)
int mem_info(als_ctx *ctx, int64_t *free_bytes, int64_t *total_bytes);
// a CSR of nnz nonzeros is held as segments: above the knob when it is set, else from 2^31 - 1 nonzeros on
static inline bool needs_segments(const als_ctx *ctx, int64_t nnz) {
  return ctx->knobs.segment_nnz > 0 ? nnz > ctx->knobs.segment_nnz : nnz >= (int64_t)INT32_MAX;
}
// Cuts `p` (rows, cols, nnz, row_offset, indices and data set) into segments of at most segment_cap nonzeros.
// ip[0 .. rows]: the host indptr as positions into p->indices / p->data.  Builds every segment's schedule, or leaves
// them to the first solve (schedule = false: p->sched_lazy).
int make_segments(als_ctx *ctx, als_csr *p, const int64_t *ip, bool schedule = true);
// The layout of a CSR whose indices / data are set, from its host indptr ip[0 .. rows] (positions into them): segments
// when it is host-resident or above the segment cap, else one int32 indptr on the device and its schedule.
int csr_layout(als_ctx *ctx, als_csr *c, const int64_t *ip, bool schedule = true);
// indices / data for c->nnz entries: page-locked host arrays for a host-resident CSR, else device arrays from the pool
int csr_alloc(als_ctx *ctx, als_csr *c);
// the indptr of any CSR as 64-bit positions relative to its first nonzero (synchronises)
int csr_indptr64(als_ctx *ctx, const als_csr *c, std::vector<int64_t> &out);
int csr_transpose(als_ctx *ctx, const als_csr *in, als_csr **out);
// The ingest of a row-sharded fit (als_b200.h): entries per column (host counts[cols]); the transpose of a device-resident
// shard cut into n pieces of whole columns, in global row ids; pieces of equal row count concatenated row by row.
int csr_column_counts(als_ctx *ctx, const als_csr *in, int64_t *counts);
int csr_transpose_pieces(als_ctx *ctx, const als_csr *in, int n, const int64_t *col_bounds, als_csr **pieces);
int csr_merge_rows(als_ctx *ctx, int n, const als_csr *const *pieces, int64_t cols, int64_t row_offset, als_csr **out);
// The ingest from row blocks: device-resident pieces (any row counts) stacked in list order, piece 0's rows first.
int csr_concat_rows(als_ctx *ctx, int n, const als_csr *const *pieces, int64_t cols, int64_t row_offset, als_csr **out);
// the weight range of a host-resident CSR, computed on the host (bits of max | |c| - 1 | without NaN / inf, and whether
// some |c| < 1: exactly what csr_wmax_kernel finds) -> c->wmax_dev, marked valid
int set_host_wmax(als_ctx *ctx, als_csr *c, unsigned wmax_bits, bool neg);
// the same range folded over n values on the host
void host_wmax(const float *v, int64_t n, unsigned *wmax_bits, bool *neg);
// The device source of an upload (als_csr_upload_device), on ctx->stream.  device_indptr: the caller's device indptr
// (4 or 8 bytes per entry) rebased to its first entry, copied to ip[0 .. rows] on the host (8 bytes per row), with
// *base = indptr[0] and *bad_row the first row r with indptr[r + 1] < indptr[r] (else -1); synchronises.
// device_entries: c->nnz indices (4 or 8 bytes, from the first nonzero) narrowed to int32 into c->indices and values
// (fp32 or fp64) cast to fp32 into c->data; an index outside [0, c->cols) sets *bad_at to the first such position and
// returns ALS_E_INVALID.  Synchronises: the caller's arrays have been read when it returns.
int device_indptr(als_ctx *ctx, const void *indptr, int indptr_bytes, int64_t rows, std::vector<int64_t> &ip,
                  int64_t *base, int64_t *bad_row);
int device_entries(als_ctx *ctx, als_csr *c, const void *indices, int index_bytes, const void *data, int data_bytes,
                   int64_t *bad_at);
// synthetic inputs generated on the device (gen.cu)
int csr_generate_power_law(als_ctx *ctx, int64_t users, int64_t items, int64_t nnz_target, uint64_t seed, als_csr **out);
int factors_fill_uniform(als_ctx *ctx, als_factors *f, uint64_t seed, float scale);
int factors_fill_pcg64(als_ctx *ctx, als_factors *f, uint64_t state_hi, uint64_t state_lo, uint64_t inc_hi,
                       uint64_t inc_lo, int has_uint32, uint32_t uinteger, float scale);

// kernels' host launchers (each returns an ALS_* code)
int launch_gramian(als_ctx *ctx, const als_factors *Y);                  // -> ctx->G
int comm_allreduce_gramian(als_ctx *ctx, int n_floats);                   // sum ctx->G over ranks (comm.cu)
int launch_regularize(als_ctx *ctx, int f, int ld, float lambda);         // ctx->G -> ctx->Greg
// The Cholesky half: resets bad_row (folding the previous half's into bad_row[1]) and the counters, then hands the
// half to the family of Y->ld: cholesky.cu (ld <= 64), cholesky_wide.cu (<= 128), cholesky_xwide.cu (<= 1024).
int launch_cholesky(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y);
// A width family of the Cholesky half, as the per-half driver run_cholesky_half sees it.
struct CholFamily {
  int64_t slot_floats = 0;  // one giant-row slot: a chunk's partial normal equations
  int64_t ws_floats = 0;    // after the slots: one workspace of this many floats per resident CTA (0: none)
  int items_per_cta = 1;    // work items one CTA takes at a time
  int64_t max_grid = 0;     // the grid bound: CTAs resident on the device
  // the family's kernel over items[0, n) on ctx->stream; pass 0: whole rows and chunks, pass 1: finish items
  std::function<void(const als_csr *S, const WorkItem *items, int n, int pass, int grid, float *slots, float *ws)> launch;
  // pass 0 of segment s in place of launch() over S->work (the narrow family: long rows, short rows, deferred items)
  std::function<int(size_t s, const als_csr *S, float *slots)> pass0;
};
// Sizes the giant-row slots (and workspaces) once over the segments of C, then walks them: pass 0, then the finish
// pass.  Y->f names the width in an allocation failure.
int run_cholesky_half(als_ctx *ctx, const als_csr *C, const als_factors *Y, const CholFamily &fam);
template <int T>
int launch_cholesky_wide(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y);   // ld = 16 T, T = 5 ... 8
int launch_cholesky_xwide(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y);  // 128 < ld <= 1024
// long rows on the wgmma tensor cores (cholesky_tc.cu): 64 padded factors, no weights |c| - 1 < 0
bool cholesky_tc_eligible(const als_ctx *ctx, const als_csr *C, int ld);
int launch_cholesky_tc(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y, int64_t n_items,
                       const unsigned *wmax_dev, cudaStream_t stream);
// short-row path (cholesky_short.cu).  prepare: P and W from ctx->Greg and Y.  launch: items [begin, n_work) of
// C->work, all of at most `max_len` nonzeros; whatever it cannot take lands in ctx->deferred / counters[kCtrDeferredCount].
int short_rows_prepare(als_ctx *ctx, const als_factors *Y, cudaStream_t stream);
// W = Y (2^14 P) and Z = Y G^-1 in one pass on the wgmma tensor cores (dense.cu; 64 padded factors)
int launch_dense_whiten(als_ctx *ctx, const als_factors *Y, cudaStream_t stream);
// G = Y^T Y on the wgmma tensor cores (dense.cu; 64 padded factors, Y of at least one row) -> ctx->G
int launch_gramian_tc(als_ctx *ctx, const als_factors *Y);
int launch_gramian_reduce(als_ctx *ctx, int nparts, int n);  // ctx->gram_partials (nparts x n) -> ctx->G, fixed-order fp64 sums
int short_rows_launch(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y, int64_t begin, int max_len,
                      cudaStream_t stream);
int launch_cg(als_ctx *ctx, const als_csr *C, als_factors *X, const als_factors *Y, int cg_steps);
int launch_loss(als_ctx *ctx, const als_csr *C, const als_factors *X, const als_factors *Y, float reg,
                double *loss);
// wgmma path of the fused top-k (topk_tc.cu): 64 padded factors, k <= 16, large query batches, no item norms
bool topk_tc_eligible(int ld, int64_t n_query, int64_t n_items, int k, bool has_norms);
int64_t topk_tc_scratch_bytes(int64_t n_query, int64_t n_items);
int launch_topk_tc(als_ctx *ctx, const float *items, int64_t n_items, const float *queries, const int32_t *query_rows,
                   int64_t n_query, int k, const uint8_t *mask, const int32_t *liked_indptr, const int32_t *liked_indices,
                   int32_t *out_ids, float *out_scores, void *scratch);
int launch_topk(als_ctx *ctx, const als_factors *items, const als_factors *queries, const int32_t *query_rows,
                int64_t n_query, int k, const float *item_norms_host, const als_csr *liked,
                const int32_t *filter_items, int64_t n_filter, int32_t *ids_host, float *scores_host);
// Ids handed to the top-k: a host int32 array (als_topk, checked by its caller), or a device array of 4- or 8-byte ids
// (als_topk_into), narrowed into the top-k's staging and range-checked on the device.  A NULL `p` with first > 0 stands
// for the rows [first, first + n) (a batch of als_topk_into's queries without query rows).
struct TopkIds {
  const void *p = nullptr;
  int64_t n = 0;
  int bytes = 4;
  bool device = false;
  int64_t first = 0;
};
// The top-k of launch_topk left on the device: ids and scores [n_query, k_eff] in ctx->scratch, valid until the next call
// that uses the scratch.  k_eff = min(k, items); 0 (and NULL arrays) when there is nothing to rank.  query_rows: the int32
// query rows the kernels read (NULL: rows 0, 1, ...).  bad: which device ids were out of range when topk_device refused
// them (kBadQueryRows, kBadFilter), before any top-k launch.
struct TopkDevice {
  int32_t *ids = nullptr;
  float *scores = nullptr;
  int k_eff = 0;
  const int32_t *query_rows = nullptr;
  int bad = 0;
};
enum { kBadQueryRows = 1, kBadFilter = 2 };
// item_norms: [items] fp32, in host memory, or in device memory when norms_on_device
int topk_device(als_ctx *ctx, const als_factors *items, const als_factors *queries, const TopkIds &query_rows,
                int64_t n_query, int k, const float *item_norms, bool norms_on_device, const als_csr *liked,
                const TopkIds &filter, TopkDevice *out);
// the grid of a grid-stride loop of 256-thread blocks over `threads` elements: at most 16 blocks per SM
static inline int grid_for(als_ctx *ctx, int64_t threads) {
  return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(threads, 256), (int64_t)ctx->sm_count * 16));
}
// serve.cu: the device side of als_topk_into and its helpers (als_b200.h).
// stage_ids: n ids of `bytes` each -> int32 out (may be NULL: check only); an id outside [0, limit) ORs `bit` into *flag
int stage_ids(als_ctx *ctx, const void *ids, int bytes, int64_t n, int64_t limit, int32_t *out, int *flag, int bit);
int stage_iota(als_ctx *ctx, int32_t *out, int64_t n, int64_t first);
// t's [n_query, k_eff] -> ids / scores [n_query, k]: zero tail, ids = map[id] (map_bytes wide, else int32), scores /=
// qnorm[query row]
int launch_topk_epilogue(als_ctx *ctx, const TopkDevice &t, int64_t n_query, int k, const void *map, int map_bytes,
                         const float *qnorm, void *ids, float *scores);
int launch_row_norms(als_ctx *ctx, const als_factors *F, float zero_value, float *out);
int launch_gather_rows(als_ctx *ctx, const als_factors *src, const void *rows, int bytes, int64_t n, als_factors *dst);
int sort_ids(als_ctx *ctx, const void *in, int bytes, int64_t n, void *out);
// the liked CSR remapped onto positions of the sorted subset[m]: device indptr (int64, rows + 1), indices and values
// (1) from the pool, *nnz entries
int csr_restrict_columns(als_ctx *ctx, const als_csr *liked, const void *subset, int bytes, int64_t m,
                         Dev<int64_t> &indptr, Dev<int32_t> &indices, Dev<float> &data, int64_t *nnz);
// refit.cu: the device side of partial_fit_* with CUDA ids (als_ids_range, als_factors_scatter_rows).
// ids_range: min and max of n ids of `bytes` each (n = 0: 0 and -1); synchronises
int ids_range(als_ctx *ctx, const void *ids, int bytes, int64_t n, int64_t *min_id, int64_t *max_id);
// dst[ids[i]] = src[i] for i < n (src->rows = n, the same width), the last occurrence of a repeated id winning; ids
// outside [0, dst->rows) are skipped
int scatter_rows(als_ctx *ctx, als_factors *dst, const void *ids, int bytes, int64_t n, const als_factors *src);
// (indptr, indices) of a device CSR with every row in ascending column order: checked once on the device, and a CSR with
// an unsorted row gets a sorted copy (indptr rebased to 0) kept with the handle (topk.cu)
int rows_in_order(als_ctx *ctx, const als_csr *csr, const int32_t **indptr, const int32_t **indices);
// The ranking metrics of the top-k against the withheld items in `test` (metrics.cu; als_ranking_metrics)
int launch_ranking_metrics(als_ctx *ctx, const als_factors *items, const als_factors *queries, const int32_t *query_rows,
                           int64_t n_query, int k, const als_csr *liked, const als_csr *test, const double *gain_host,
                           const double *gain_sum_host, double *sums);
// weight.cu: BM25 / TF-IDF / normalize on raw arrays (als_weight_*).  Each synchronises; ALS_E_INVALID for an index
// outside the matrix or an indptr that is not 0 <= ... <= nnz.
int weight_check_indptr(als_ctx *ctx, const void *indptr, int indptr_bytes, int64_t rows, int64_t nnz, const char *who);
int weight_column_counts(als_ctx *ctx, const void *indices, int index_bytes, int64_t nnz, int64_t cols, int64_t *counts);
int weight_row_sums(als_ctx *ctx, int64_t rows, int64_t nnz, const void *indptr, int indptr_bytes, const void *row,
                    int row_bytes, const void *data, int value_kind, bool squares, void *sums_host);
int weight_entries(als_ctx *ctx, int kind, int64_t rows, int64_t cols, int64_t nnz, const void *indptr, int indptr_bytes,
                   const void *row, int row_bytes, const void *indices, int index_bytes, const void *data, int value_kind,
                   const void *row_values_host, const double *idf_host, double k1p1, double k1, int flags, double *out);

}  // namespace als
