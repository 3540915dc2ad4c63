// C-ABI implementation (include/filo_b200.h): context, chunk-arena loader, query orchestration.
// Host side only orchestrates: every query result is produced by the sm_90a kernels in scan_kernels.cu.
#include "../../include/filo_b200.h"
#include "kernels.h"
#include "host_util.h"
#include "scan_tile_layout.h"
#include "scan_wp_layout.h"
#include <cub/cub.cuh>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

using namespace filo;

struct filo_ctx {
  int device = 0;
  filo_cfg cfg{};
  cudaStream_t stream = nullptr;
  int sm_count = 132;
  size_t max_smem_optin = 0;
  std::mutex err_mu;
  std::string err;
  double fn_args[2] = {0.0, 0.0};      // static arguments of the range function (filo_ctx_set_fn_args)
  // device error words of non-synchronising queries (filo_query_device with stats == NULL): copied into pinned slots on the query's
  // stream and surfaced by the next call on this ctx that finds them complete, or by filo_ctx_check
  struct ErrSlot { int* h = nullptr; cudaEvent_t ev = nullptr; bool pending = false; };
  std::mutex errslot_mu;
  ErrSlot errslots[16];
  int errslot_next = 0;
  // filo_scan_series pipeline slots (pinned staging + device buffers), kept across calls
  struct ScanSlot {
    uint8_t* h_in = nullptr; size_t h_in_cap = 0;        // pinned: records of the batch
    int64_t* h_off = nullptr; size_t h_off_cap = 0;      // pinned: record offsets relative to the batch
    uint8_t* d_in = nullptr; size_t d_in_cap = 0;
    int64_t* d_off = nullptr; size_t d_off_cap = 0;
    double* d_out = nullptr; size_t d_out_cap = 0;
    void* h_sink = nullptr;                              // pinned AsyncSink
    void* h_gch = nullptr; size_t h_gch_cap = 0;         // pinned: gather list of the batch (zero-copy path)
    void* d_gch = nullptr; size_t d_gch_cap = 0;
    void* h_gs = nullptr; size_t h_gs_cap = 0;           // pinned: per-series gather headers
    void* d_gs = nullptr; size_t d_gs_cap = 0;
    uint8_t* d_stage = nullptr; size_t d_stage_cap = 0;  // device copy of the host span that holds a batch's vectors (dense batches: one DMA instead of zero-copy reads)
    cudaStream_t stream = nullptr; cudaEvent_t done = nullptr;
  };
  std::mutex scan_mu;
  static constexpr int MAX_SCAN_SLOTS = 8;
  ScanSlot scan[MAX_SCAN_SLOTS];
  // host memory registered for device access (filo_host_register): chunk vectors inside these ranges are gathered by the GPU
  struct HostRange { uintptr_t base; size_t bytes; };
  std::vector<HostRange> ranges;
};

struct filo_table {
  int64_t n_series = 0, n_chunks = 0, n_samples = 0, arena_bytes = 0, algorithmic_bytes = 0;
  int32_t max_rows = 0, max_chunks = 0, schema_flags = 0;
  uint32_t max_rec_bytes = 0;       // largest record (staging buffer size of the v2 kernels)
  bool any_nonconst_ts = true;      // some timestamp vector is not a const DDV (needs decoded ts slots)
  bool any_drop = true;             // some value vector carries the counter drop flag (needs corrected slots)
  uint8_t* d_arena = nullptr;
  int64_t* d_rec_off = nullptr;     // [n_series + 1]
  // grouping
  int32_t n_groups = 1;
  bool grouped = false;             // false: single group, order == identity
  int32_t* d_order = nullptr;       // [n_series] series ordinals sorted by group (stable)
  int64_t* d_group_start = nullptr; // [n_groups + 1]
  int64_t* d_gis = nullptr;         // [n_groups + 1] first item of each group
  int64_t* d_item_begin = nullptr;  // [n_items + 1]
  int64_t n_items = 0;
  int seg = 1;
  // histogram tables (value column = HistogramVector): one bucket scheme for the whole table
  bool hist = false, hist_exp = false; int hist_nb = 0;     // hist_exp: Base2ExpHistogramBuckets (histogram_quantile interpolates in log space)
  bool hist_simple = false;                                  // some histogram vector is a simple (row) vector: not for the second scan kernel
  std::vector<double> hist_tops; double* d_hist_tops = nullptr;
};

static thread_local std::string tl_err;

static int32_t fail(filo_ctx* ctx, int32_t code, const std::string& msg) {
  tl_err = msg;
  if (ctx) { std::lock_guard<std::mutex> g(ctx->err_mu); ctx->err = msg; }
  return code;
}
#define CUDA_TRY(ctx, expr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) \
  return fail(ctx, _e == cudaErrorMemoryAllocation ? FILO_ERR_OOM : FILO_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); } while (0)

extern "C" {

int32_t filo_last_error(filo_ctx* ctx, char* buf, int32_t len) {
  std::string m;
  if (ctx) { std::lock_guard<std::mutex> g(ctx->err_mu); m = ctx->err; } else m = tl_err;
  if (buf && len > 0) { int n = std::min<int>(len - 1, (int)m.size()); std::memcpy(buf, m.data(), n); buf[n] = 0; }
  return (int32_t)m.size();
}

int32_t filo_ctx_create(int32_t device, const filo_cfg* cfg, filo_ctx** out) {
  if (!out) return fail(nullptr, FILO_ERR_INVALID_ARG, "out is null");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(nullptr, FILO_ERR_CUDA, std::string("no CUDA device (no CPU fallback exists): ") + cudaGetErrorString(e));
  if (device < 0 || device >= ndev) return fail(nullptr, FILO_ERR_INVALID_ARG, "bad device ordinal");
  CUDA_TRY(nullptr, cudaSetDevice(device));
  auto* c = new filo_ctx();
  c->device = device;
  if (cfg) c->cfg = *cfg; else { c->cfg.inclusive_range = 1; c->cfg.group_by_cardinality_limit = 0; c->cfg.min_step_ms = 0; c->cfg.max_data_per_shard_query = 0; }
  cudaDeviceProp p; CUDA_TRY(nullptr, cudaGetDeviceProperties(&p, device));
  c->sm_count = p.multiProcessorCount;
  c->max_smem_optin = p.sharedMemPerBlockOptin;
  CUDA_TRY(nullptr, cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  {
    // per-query temporaries come from the stream-ordered pool: keep freed blocks in the pool instead of returning them to the OS at every
    // synchronisation (the default release threshold of 0 makes the first allocation after a sync a driver call)
    cudaMemPool_t pool = nullptr;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess && pool) {
      uint64_t thr = ~0ull;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
    cudaGetLastError();
  }
  *out = c;
  return FILO_OK;
}

int32_t filo_ctx_set_fn_args(filo_ctx* ctx, double arg0, double arg1) {
  if (!ctx) return fail(nullptr, FILO_ERR_INVALID_ARG, "ctx is null");
  ctx->fn_args[0] = arg0; ctx->fn_args[1] = arg1;
  return FILO_OK;
}

void filo_ctx_destroy(filo_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  for (auto& sl : ctx->errslots) { if (sl.ev) { cudaEventSynchronize(sl.ev); cudaEventDestroy(sl.ev); } if (sl.h) cudaFreeHost(sl.h); }
  for (auto& r : ctx->ranges) cudaHostUnregister((void*)r.base);
  for (auto& sl : ctx->scan) {
    if (sl.stream) cudaStreamSynchronize(sl.stream);
    cudaFreeHost(sl.h_in); cudaFreeHost(sl.h_off); cudaFreeHost(sl.h_sink); cudaFree(sl.d_in); cudaFree(sl.d_off); cudaFree(sl.d_out);
    cudaFreeHost(sl.h_gch); cudaFreeHost(sl.h_gs); cudaFree(sl.d_gch); cudaFree(sl.d_gs); cudaFree(sl.d_stage);
    if (sl.done) cudaEventDestroy(sl.done);
    if (sl.stream) cudaStreamDestroy(sl.stream);
  }
  delete ctx;
}

void filo_table_free(filo_ctx* ctx, filo_table* t) {
  if (!t) return;
  if (ctx) cudaSetDevice(ctx->device);
  cudaFree(t->d_arena); cudaFree(t->d_rec_off); cudaFree(t->d_order); cudaFree(t->d_group_start);
  cudaFree(t->d_gis); cudaFree(t->d_item_begin); cudaFree(t->d_hist_tops);
  delete t;
}

int32_t filo_table_get_info(const filo_table* t, filo_table_info* o) {
  if (!t || !o) return FILO_ERR_INVALID_ARG;
  o->n_series = t->n_series; o->n_chunks = t->n_chunks; o->n_samples = t->n_samples; o->arena_bytes = t->arena_bytes;
  o->algorithmic_bytes = t->algorithmic_bytes; o->max_rows_per_series = t->max_rows; o->max_chunks_per_series = t->max_chunks;
  o->n_groups = t->n_groups; o->schema_flags = t->schema_flags; o->hist_buckets = t->hist ? t->hist_nb : 0; o->reserved = 0;
  return FILO_OK;
}

int32_t filo_num_windows(int64_t start, int64_t step, int64_t end) {
  if (step <= 0) step = 1;
  if (end < start) return 1;
  return (int32_t)((end - start) / step) + 1;
}

} // extern "C"

// The second histogram scan kernel (hist_kernels2.cu) serves the shapes it covers unless FILO_HIST_V2=0 (A/B runs against the first)
static bool hist_v2_enabled() { const char* e = getenv("FILO_HIST_V2"); return !(e && e[0] == '0'); }

// ------------------------------------------------------------------------------------------------------------------
// grouping: stable sort of series by group id on the device, group bounds, work items of <= seg series of one group
// ------------------------------------------------------------------------------------------------------------------
static int32_t build_groups_new(filo_ctx* ctx, filo_table* t, const int32_t* d_group_ids, int32_t n_groups);
// the new grouping replaces the old one only when it has been built completely: a failure leaves the table as it was
static int32_t build_groups(filo_ctx* ctx, filo_table* t, const int32_t* d_group_ids /* device, may be null */, int32_t n_groups) {
  int32_t* o_order = t->d_order; int64_t* o_gs = t->d_group_start; int64_t* o_gis = t->d_gis; int64_t* o_ib = t->d_item_begin;
  const int32_t o_ng = t->n_groups; const bool o_grouped = t->grouped; const int64_t o_items = t->n_items; const int o_seg = t->seg;
  t->d_order = nullptr; t->d_group_start = t->d_gis = t->d_item_begin = nullptr;
  const int32_t rc = build_groups_new(ctx, t, d_group_ids, n_groups);
  if (rc != FILO_OK) {
    cudaFree(t->d_order); cudaFree(t->d_group_start); cudaFree(t->d_gis); cudaFree(t->d_item_begin);
    t->d_order = o_order; t->d_group_start = o_gs; t->d_gis = o_gis; t->d_item_begin = o_ib;
    t->n_groups = o_ng; t->grouped = o_grouped; t->n_items = o_items; t->seg = o_seg;
    return rc;
  }
  cudaFree(o_order); cudaFree(o_gs); cudaFree(o_gis); cudaFree(o_ib);
  return FILO_OK;
}
static int32_t build_groups_new(filo_ctx* ctx, filo_table* t, const int32_t* d_group_ids /* device, may be null */, int32_t n_groups) {
  cudaStream_t s = ctx->stream;
  const int64_t S = t->n_series;
  if (n_groups <= 0) n_groups = 1;
  t->n_groups = n_groups;
  t->grouped = d_group_ids != nullptr;
  // seg: enough items to fill the machine a few times over, capped so partial rows stay small
  int64_t target_items = (int64_t)ctx->sm_count * 64 * 4;
  int64_t seg_cap = 256;
  // histogram tables under the second scan kernel: an item's partial is T * buckets doubles (tens of KB) and one CTA folds an
  // item, so a few items per CTA
  if (t->hist && hist_v2_enabled()) { target_items = (int64_t)ctx->sm_count * 2 * 6; seg_cap = 4096; }
  int64_t seg = S / std::max<int64_t>(target_items, 1);
  t->seg = (int)std::min<int64_t>(std::max<int64_t>(seg, 1), seg_cap);
  CUDA_TRY(ctx, cudaMalloc(&t->d_group_start, (size_t)(n_groups + 1) * 8));
  CUDA_TRY(ctx, cudaMalloc(&t->d_gis, (size_t)(n_groups + 1) * 8));
  if (t->grouped && S > 0) {
    int32_t *keys_out = nullptr, *vals_in = nullptr;
    CUDA_TRY(ctx, cudaMalloc(&t->d_order, (size_t)S * 4));
    CUDA_TRY(ctx, cudaMalloc(&keys_out, (size_t)S * 4));
    CUDA_TRY(ctx, cudaMalloc(&vals_in, (size_t)S * 4));
    CUDA_TRY(ctx, launch_iota(vals_in, S, s));
    size_t tmp_bytes = 0;
    int end_bit = 1; while ((1ll << end_bit) < n_groups && end_bit < 31) ++end_bit;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, d_group_ids, keys_out, vals_in, t->d_order, (int)S, 0, end_bit, s);
    void* tmp = nullptr; CUDA_TRY(ctx, cudaMalloc(&tmp, tmp_bytes + 16));
    CUDA_TRY(ctx, cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, d_group_ids, keys_out, vals_in, t->d_order, (int)S, 0, end_bit, s));
    CUDA_TRY(ctx, launch_group_bounds(keys_out, S, n_groups, t->d_group_start, s));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
    cudaFree(tmp); cudaFree(keys_out); cudaFree(vals_in);
  } else {
    std::vector<int64_t> gs(n_groups + 1, S); gs[0] = 0;
    CUDA_TRY(ctx, cudaMemcpyAsync(t->d_group_start, gs.data(), gs.size() * 8, cudaMemcpyHostToDevice, s));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
  }
  // items
  int64_t* d_cnt = nullptr; CUDA_TRY(ctx, cudaMalloc(&d_cnt, (size_t)(n_groups + 1) * 8));
  CUDA_TRY(ctx, cudaMemsetAsync(d_cnt, 0, (size_t)(n_groups + 1) * 8, s));
  CUDA_TRY(ctx, launch_group_item_count(t->d_group_start, n_groups, t->seg, d_cnt, s));
  size_t tmp_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, d_cnt, t->d_gis, n_groups + 1, s);
  void* tmp = nullptr; CUDA_TRY(ctx, cudaMalloc(&tmp, tmp_bytes + 16));
  CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, d_cnt, t->d_gis, n_groups + 1, s));
  int64_t n_items = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(&n_items, t->d_gis + n_groups, 8, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(ctx, cudaStreamSynchronize(s));
  t->n_items = n_items;
  CUDA_TRY(ctx, cudaMalloc(&t->d_item_begin, (size_t)(n_items + 1) * 8));
  CUDA_TRY(ctx, launch_fill_items(t->d_group_start, t->d_gis, n_groups, t->seg, n_items, S, t->d_item_begin, s));
  CUDA_TRY(ctx, cudaStreamSynchronize(s));
  cudaFree(tmp); cudaFree(d_cnt);
  return FILO_OK;
}

// shared by the loader and the synthetic generator
int32_t filo_internal_finish_table(filo_ctx* ctx, filo_table* t, const int32_t* d_group_ids, int32_t n_groups) {
  return build_groups(ctx, t, d_group_ids, n_groups);
}
filo_table* filo_internal_new_table() { return new filo_table(); }
void filo_internal_set_arena(filo_table* t, uint8_t* d_arena, int64_t* d_rec_off, int64_t n_series, int64_t n_chunks, int64_t n_samples,
                             int64_t arena_bytes, int64_t algorithmic_bytes, int32_t max_rows, int32_t max_chunks, int32_t schema_flags) {
  t->d_arena = d_arena; t->d_rec_off = d_rec_off; t->n_series = n_series; t->n_chunks = n_chunks; t->n_samples = n_samples;
  t->arena_bytes = arena_bytes; t->algorithmic_bytes = algorithmic_bytes; t->max_rows = max_rows; t->max_chunks = max_chunks;
  t->schema_flags = schema_flags;
}
void filo_internal_set_layout(filo_table* t, uint32_t max_rec_bytes, bool any_nonconst_ts, bool any_drop) {
  t->max_rec_bytes = max_rec_bytes; t->any_nonconst_ts = any_nonconst_ts; t->any_drop = any_drop;
}
cudaStream_t filo_internal_stream(filo_ctx* ctx) { return ctx->stream; }
int filo_internal_device(filo_ctx* ctx) { return ctx->device; }
int32_t filo_internal_fail(filo_ctx* ctx, int32_t code, const char* msg) { return fail(ctx, code, msg); }

// ------------------------------------------------------------------------------------------------------------------
// loader: walk ChunkSetInfo blocks -> records -> device arena
// ------------------------------------------------------------------------------------------------------------------
namespace {

struct GatherChunk {            // one chunk with rows, in series order
  uint64_t ts_src, val_src;     // host addresses (UVA) of the vectors to copy
  int64_t start_time, end_time;
  int32_t num_rows, ts_bytes, val_bytes, val_len;
  int32_t drop_patch, pad;      // 0: keep, 1: set, 2: clear the counter drop bit (masked wrappers carry it on the outer vector)
};
struct GatherSeries { uint32_t rec_bytes, n_chunks, n_rows, flags; int64_t first_chunk; };

struct VecInfo { const uint8_t* p; int32_t total; int32_t len; bool drop_patch; bool drop; bool hist = false; };

inline int32_t rd32(const uint8_t* p) { int32_t v; std::memcpy(&v, p, 4); return v; }
inline int64_t rd64(const uint8_t* p) { int64_t v; std::memcpy(&v, p, 8); return v; }

// IntBinaryVector.simple validity (MatchError otherwise), IntBinaryVector.scala:120-137
inline bool inner_ok(const uint8_t* in, int32_t& len, int32_t outer_total) {
  const int32_t inner_bytes = rd32(in);
  if (inner_bytes < 4 || (int64_t)20 + 4 + inner_bytes > outer_total) return false;      // the inner vector lies inside the outer one
  int nbits = in[6] & 0x7f; bool sgn = in[6] & 0x80; int bs = in[7] & 0x3f;
  bool ok = sgn ? (nbits == 32 || nbits == 16 || nbits == 8) : (nbits == 32 || nbits == 16 || nbits == 8 || nbits == 4 || nbits == 2);
  if (!ok) return false;
  len = ((rd32(in) - 4) * 8 + (bs != 0 ? bs - 8 : 0)) / nbits;
  return true;
}

// returns 0 ok, else FILO_ERR_*
int classify_ts(const uint8_t* v, VecInfo& o) {
  int wire = (uint16_t)(v[4] | (v[5] << 8));
  if (wire == WIRE_MASKED) { v = v + rd32(v + 8); wire = (uint16_t)(v[4] | (v[5] << 8)); if (wire == WIRE_MASKED) return FILO_ERR_CORRUPT_VECTOR; }
  o.p = v; o.total = rd32(v) + 4; o.drop_patch = false; o.drop = false;
  if (o.total < 8 || o.total > (1 << 28)) return FILO_ERR_CORRUPT_VECTOR;      // numBytes is a positive Int far below the block size
  if (wire == WIRE_DDV_CONST) { if (o.total != 24) return FILO_ERR_CORRUPT_VECTOR; o.len = rd32(v + 8); }
  else if (wire == WIRE_RAW64) o.len = (rd32(v) - 4) / 8;
  else if (wire == WIRE_DDV) { if (o.total < 28 || !inner_ok(v + 20, o.len, o.total)) return FILO_ERR_CORRUPT_VECTOR; }
  else return FILO_ERR_CORRUPT_VECTOR;
  return (o.total >= 8 && o.len >= 0) ? 0 : FILO_ERR_CORRUPT_VECTOR;
}
int classify_val(const uint8_t* v, VecInfo& o) {
  int wire = (uint16_t)(v[4] | (v[5] << 8));
  const bool outer_drop = (v[7] & 0x80) != 0;
  bool masked = false;
  if (wire == WIRE_MASKED) { masked = true; v = v + rd32(v + 8); wire = (uint16_t)(v[4] | (v[5] << 8)); if (wire == WIRE_MASKED) return FILO_ERR_CORRUPT_VECTOR; }
  o.p = v; o.total = rd32(v) + 4; o.drop_patch = masked; o.drop = outer_drop;
  if (o.total < 8 || o.total > (1 << 28)) return FILO_ERR_CORRUPT_VECTOR;
  if (wire == WIRE_RAW64) o.len = (rd32(v) - 4) / 8;
  else if (wire == WIRE_DDV_CONST) { if (o.total != 24) return FILO_ERR_CORRUPT_VECTOR; o.len = rd32(v + 8); }
  else if (wire == WIRE_DDV) { if (o.total < 28 || !inner_ok(v + 20, o.len, o.total)) return FILO_ERR_CORRUPT_VECTOR; }
  else if (wire == WIRE_XOR) {
    o.len = rd32(v + XOR_OFF_N);
    int ng = (uint16_t)(v[12] | (v[13] << 8)), po = (uint16_t)(v[14] | (v[15] << 8));
    if (o.len <= 0 || ng != (o.len - 1 + 7) / 8 || po < 16 + 2 * ng || (po & 7) || po + 8 > o.total) return FILO_ERR_CORRUPT_VECTOR;
  } else if (wire == WIRE_H_SECTDELTA || wire == WIRE_H_SIMPLE) {          // HistogramVector header, HistogramVector.scala:239-244
    if (masked || o.total < 13) return FILO_ERR_CORRUPT_VECTOR;
    o.len = (uint16_t)(v[6] | (v[7] << 8)); o.drop = false; o.hist = true;
    const int fmt = v[8], defBytes = (uint16_t)(v[9] | (v[10] << 8));
    if (o.len > 0 && (!(fmt == 3 || fmt == 4 || fmt == 5 || fmt == 9) || 11 + defBytes > o.total || (fmt == 9 && defBytes != 16)))
      return (fmt == 8 || fmt == 0x0a || fmt == 0x10 || fmt == 9) ? FILO_ERR_UNSUPPORTED : FILO_ERR_CORRUPT_VECTOR;
  } else if (wire == WIRE_H_EXP_SIMPLE) return FILO_ERR_UNSUPPORTED;        // ExpHistogramVector.scala: row-wise schemes (no counter reader in the reference either)
  else return FILO_ERR_CORRUPT_VECTOR;
  return (o.total >= 8 && o.len >= 0) ? 0 : FILO_ERR_CORRUPT_VECTOR;
}

struct SeriesPlan { uint32_t rec_bytes; uint32_t n_chunks; uint32_t n_rows; uint32_t flags; };

struct LoadIn { int64_t n_series; const int32_t* n_chunks; const uint64_t* addrs; const int64_t* chunk_base /* entry of series i at [i - cb0] */; int32_t ts_col, val_col;
                // filo_scan_series: the one walk over the ChunkSetInfo blocks also leaves the gather entries of the chunks with rows (entry k of
                // series i at gc_out[chunk_base[i] - gc_base + k]) and checks the vectors against the registered host ranges
                GatherChunk* gc_out = nullptr; int64_t gc_base = 0; const std::vector<filo_ctx::HostRange>* ranges = nullptr;
                int64_t cb0 = 0; };
struct PlanTotals { int64_t chunks = 0, samples = 0, alg = 0; int32_t maxrows = 0, maxch = 0; uint32_t max_rec = 0, f_or = 0, f_and = ~0u;
                    const uint8_t* hist_def = nullptr; bool any_scalar = false, hist_mismatch = false; bool all_in_ranges = true; bool hist_simple = false; };
// same bucket scheme: format code, definition length and bytes of two HistogramVector headers (HistogramVector.matchBucketDef, :262-268)
inline bool same_hist_def(const uint8_t* a, const uint8_t* b) {
  const int da = (uint16_t)(a[9] | (a[10] << 8)), db = (uint16_t)(b[9] | (b[10] << 8));
  return a[8] == b[8] && da == db && std::memcmp(a + 11, b + 11, (size_t)da) == 0;
}

// pass 1 of the loader for one series: validate the vectors, size the record.  Returns 0 or FILO_ERR_*.
inline int plan_series(const LoadIn& in, int64_t i, SeriesPlan& out, PlanTotals& tot) {
  uint32_t bytes = sizeof(RecordHeader), rows = 0, nch = 0, flags = REC_ALL_TS_CONST;
  int64_t prev_start = INT64_MIN, prev_end = INT64_MIN;
  for (int32_t j = 0; j < in.n_chunks[i]; ++j) {
    const uint8_t* info = reinterpret_cast<const uint8_t*>((uintptr_t)in.addrs[in.chunk_base[i - in.cb0] + j]);
    const int32_t numRows = rd32(info + 8);
    if (numRows <= 0) continue;                                   // skipped by WindowedChunkIterator (ChunkSetInfo.scala:493)
    const int64_t startT = (int64_t)(((1ull << 63) ^ (uint64_t)rd64(info)) >> 22), endT = rd64(info + 20);
    VecInfo tv, vv;
    int rc = classify_ts(reinterpret_cast<const uint8_t*>((uintptr_t)rd64(info + 28 + 8 * in.ts_col)), tv);
    if (!rc) rc = classify_val(reinterpret_cast<const uint8_t*>((uintptr_t)rd64(info + 28 + 8 * in.val_col)), vv);
    if (!rc && (numRows > tv.len || numRows > vv.len)) rc = FILO_ERR_CORRUPT_VECTOR;
    if (!rc && (startT < prev_start || endT < prev_end)) rc = FILO_ERR_UNSUPPORTED;
    if (rc) return rc;
    prev_start = startT; prev_end = endT;
    bytes += sizeof(ChunkEntry) + align_up((uint32_t)tv.total, 8) + align_up((uint32_t)vv.total, 8);
    rows += (uint32_t)vv.len; ++nch;
    const int twire = (uint16_t)(tv.p[4] | (tv.p[5] << 8)), vwire = (uint16_t)(vv.p[4] | (vv.p[5] << 8));
    if (twire != WIRE_DDV_CONST) flags &= ~REC_ALL_TS_CONST;
    if (vv.drop) flags |= REC_ANY_DROP;
    if (vwire != WIRE_RAW64) flags |= REC_ANY_DECODE;
    if (vv.hist) { flags |= REC_HIST; if (vwire == WIRE_H_SIMPLE) tot.hist_simple = true; if (!tot.hist_def) tot.hist_def = vv.p; else if (vv.len > 0 && !same_hist_def(tot.hist_def, vv.p)) tot.hist_mismatch = true; }
    else tot.any_scalar = true;
    tot.samples += numRows; tot.alg += 28 + 16 + tv.total + vv.total;
    if (in.gc_out) {
      GatherChunk g;
      g.ts_src = (uint64_t)(uintptr_t)tv.p; g.val_src = (uint64_t)(uintptr_t)vv.p; g.start_time = startT; g.end_time = endT;
      g.num_rows = numRows; g.ts_bytes = tv.total; g.val_bytes = vv.total; g.val_len = vv.len;
      g.drop_patch = vv.drop_patch ? (vv.drop ? 1 : 2) : 0; g.pad = 0;
      in.gc_out[in.chunk_base[i - in.cb0] - in.gc_base + (int64_t)nch - 1] = g;
      if (in.ranges && tot.all_in_ranges) {
        auto inr = [&](const uint8_t* p, size_t n) { for (auto& r : *in.ranges) if ((uintptr_t)p >= r.base && (uintptr_t)p + n <= r.base + r.bytes) return true; return false; };
        if (!inr(tv.p, (size_t)tv.total) || !inr(vv.p, (size_t)vv.total)) tot.all_in_ranges = false;
      }
    }
  }
  out = SeriesPlan{align_up(bytes, 16), nch, rows, flags};
  tot.chunks += nch; tot.maxrows = std::max<int32_t>(tot.maxrows, (int32_t)rows); tot.maxch = std::max<int32_t>(tot.maxch, (int32_t)nch);
  tot.max_rec = std::max(tot.max_rec, out.rec_bytes); tot.f_or |= flags; tot.f_and &= flags;
  return 0;
}
inline void merge_totals(PlanTotals& a, const PlanTotals& b) {
  a.chunks += b.chunks; a.samples += b.samples; a.alg += b.alg; a.maxrows = std::max(a.maxrows, b.maxrows); a.maxch = std::max(a.maxch, b.maxch);
  a.max_rec = std::max(a.max_rec, b.max_rec); a.f_or |= b.f_or; a.f_and &= b.f_and;
  if (!a.hist_def) a.hist_def = b.hist_def; else if (b.hist_def && !same_hist_def(a.hist_def, b.hist_def)) a.hist_mismatch = true;
  a.any_scalar |= b.any_scalar; a.hist_mismatch |= b.hist_mismatch; a.hist_simple |= b.hist_simple; a.all_in_ranges = a.all_in_ranges && b.all_in_ranges;
}
// host NibblePack.unpackDoubleXOR (NibblePack.scala:374-447) for the custom bucket tops of a table (a few dozen values)
inline bool host_unpack_double_xor(const uint8_t* buf, int cap, double* out, int n) {
  auto rdl = [&](int idx) { uint64_t w = 0; for (int i = 0; i < 8 && idx + i < cap; ++i) w |= (uint64_t)buf[idx + i] << (8 * i); return w; };
  if (cap < 8 || n <= 0) return false;
  uint64_t last = rdl(0); std::memcpy(&out[0], &last, 8);
  int pos = 8, o = 1;
  while (o < n && pos < cap) {
    const uint32_t mask = buf[pos]; uint64_t d[8] = {0, 0, 0, 0, 0, 0, 0, 0}; int used = 1;
    if (mask) {
      const int hdr = buf[pos + 1], numBits = ((hdr >> 4) + 1) * 4, tz = (hdr & 15) * 4;
      used = 2 + (numBits * __builtin_popcount(mask) + 7) / 8;
      int bit = 0;
      for (int i = 0; i < 8; ++i) if (mask & (1u << i)) {
        uint64_t v = 0;
        for (int k = 0; k < numBits; ++k) { const int bb = bit + k; const int by = pos + 2 + (bb >> 3); if (by < cap && ((buf[by] >> (bb & 7)) & 1)) v |= 1ull << k; }
        d[i] = v << tz; bit += numBits;
      }
    }
    for (int i = 0; i < 8 && o < n; ++i, ++o) { last ^= d[i]; std::memcpy(&out[o], &last, 8); }
    pos += used;
  }
  return o == n;
}
// pass 2 of the loader for one series: header, chunk entries, vectors copied verbatim
inline void fill_record(const LoadIn& in, int64_t i, const SeriesPlan& p, uint8_t* rec) {
  std::memset(rec, 0, sizeof(RecordHeader) + p.n_chunks * sizeof(ChunkEntry));
  RecordHeader h{p.rec_bytes, p.n_chunks, p.n_rows, p.flags};
  std::memcpy(rec, &h, sizeof h);
  uint32_t off = sizeof(RecordHeader) + p.n_chunks * (uint32_t)sizeof(ChunkEntry);
  uint32_t c = 0, row_base = 0;
  for (int32_t j = 0; j < in.n_chunks[i]; ++j) {
    const uint8_t* info = reinterpret_cast<const uint8_t*>((uintptr_t)in.addrs[in.chunk_base[i - in.cb0] + j]);
    const int32_t numRows = rd32(info + 8);
    if (numRows <= 0) continue;
    VecInfo tv, vv;
    classify_ts(reinterpret_cast<const uint8_t*>((uintptr_t)rd64(info + 28 + 8 * in.ts_col)), tv);
    classify_val(reinterpret_cast<const uint8_t*>((uintptr_t)rd64(info + 28 + 8 * in.val_col)), vv);
    ChunkEntry ce;
    ce.start_time = (int64_t)(((1ull << 63) ^ (uint64_t)rd64(info)) >> 22); ce.end_time = rd64(info + 20);
    ce.num_rows = numRows; ce.ts_off = off; std::memcpy(rec + off, tv.p, tv.total);
    { const uint32_t pad = align_up((uint32_t)tv.total, 8) - (uint32_t)tv.total; if (pad) std::memset(rec + off + tv.total, 0, pad); off += (uint32_t)tv.total + pad; }
    ce.val_off = off; std::memcpy(rec + off, vv.p, vv.total);
    if (vv.drop_patch) { if (vv.drop) rec[off + 7] |= 0x80; else rec[off + 7] &= 0x7f; }
    { const uint32_t pad = align_up((uint32_t)vv.total, 8) - (uint32_t)vv.total; if (pad) std::memset(rec + off + vv.total, 0, pad); off += (uint32_t)vv.total + pad; }
    ce.row_base = row_base; row_base += (uint32_t)vv.len;
    std::memcpy(rec + sizeof(RecordHeader) + c * sizeof(ChunkEntry), &ce, sizeof ce); ++c;
  }
  if (off < p.rec_bytes) std::memset(rec + off, 0, p.rec_bytes - off);
}
// pass 1 over the series [s_begin, s_end) (pool); fills plan[] and the totals, returns 0 or the first error with its series
inline int plan_range(const LoadIn& in, int64_t s_begin, int64_t s_end, std::vector<SeriesPlan>& plan, PlanTotals& tot, int64_t& err_series_out, int64_t plan_base = 0) {
  HostPool& pool = host_pool();
  std::vector<PlanTotals> part((size_t)pool.size());
  std::atomic<int> err_code{0}; std::atomic<int64_t> err_series{-1};
  pool.run(s_end - s_begin, [&](int w, int64_t b, int64_t e) {
    for (int64_t i = s_begin + b; i < s_begin + e && !err_code.load(std::memory_order_relaxed); ++i) {
      const int rc = plan_series(in, i, plan[(size_t)(i - plan_base)], part[(size_t)w]);
      if (rc) { int z = 0; if (err_code.compare_exchange_strong(z, rc)) err_series = i; return; }
    }
  });
  for (auto& p : part) merge_totals(tot, p);
  err_series_out = err_series.load();
  return err_code.load();
}
inline int plan_all(const LoadIn& in, std::vector<SeriesPlan>& plan, PlanTotals& tot, int64_t& err_series_out) {
  HostPool& pool = host_pool();
  std::vector<PlanTotals> part((size_t)pool.size());
  std::atomic<int> err_code{0}; std::atomic<int64_t> err_series{-1};
  pool.run(in.n_series, [&](int w, int64_t b, int64_t e) {
    for (int64_t i = b; i < e && !err_code.load(std::memory_order_relaxed); ++i) {
      const int rc = plan_series(in, i, plan[(size_t)i], part[(size_t)w]);
      if (rc) { int z = 0; if (err_code.compare_exchange_strong(z, rc)) err_series = i; return; }
    }
  });
  for (auto& p : part) merge_totals(tot, p);
  err_series_out = err_series.load();
  return err_code.load();
}


} // namespace

// histogram table: one bucket scheme for all series; hd = a HistogramVector header (format code at +8, definition at +9) in host memory
int32_t filo_internal_set_hist(filo_ctx* ctx, filo_table* t, const uint8_t* hd) {
  const int fmt = hd[8], nb = (uint16_t)(hd[11] | (hd[12] << 8));
  t->hist = true; t->hist_nb = nb; t->hist_tops.assign((size_t)std::max(nb, 0), 0.0);
  bool ok = nb > 0 && nb <= 64;
  if (ok && (fmt == 3 || fmt == 4)) {                // GeometricBuckets.bucketTop, Histogram.scala:606
    double first, mult; std::memcpy(&first, hd + 13, 8); std::memcpy(&mult, hd + 21, 8);
    for (int i = 0; i < nb; ++i) t->hist_tops[(size_t)i] = first * std::pow(mult, (double)i) + (fmt == 4 ? -1.0 : 0.0);
  } else if (ok && fmt == 5) {                        // CustomBuckets: u16 n + NibblePack.packDoubles(les), Histogram.scala:878-884
    const int defBytes = (uint16_t)(hd[9] | (hd[10] << 8));
    ok = host_unpack_double_xor(hd + 13, defBytes - 2, t->hist_tops.data(), nb);
  } else if (ok && fmt == 9) {                        // Base2ExpHistogramBuckets (otel exponential), Histogram.scala:729-752: i16 scale, i32 startIndexPositiveBuckets,
    // u16 numPositiveBuckets (+ the unused negative pair); numBuckets = numPositive + 1 (the zero bucket).  Tops as bucketTop computes them (:716-727,
    // base / logBase tables :647-658) with the host's libm, the same calls the oracle makes
    const int scale = (int16_t)(hd[13] | (hd[14] << 8)), numPos = (uint16_t)(hd[19] | (hd[20] << 8));
    int32_t startIdx; std::memcpy(&startIdx, hd + 15, 4);
    ok = scale >= -20 && scale <= 20 && numPos == nb - 1;
    if (ok) {
      const double logBase = std::log(std::pow(2.0, std::pow(2.0, (double)-scale)));
      t->hist_tops[0] = 0.0;
      for (int i = 1; i < nb; ++i) t->hist_tops[(size_t)i] = std::exp((double)(int32_t)((uint32_t)startIdx + (uint32_t)i) * logBase);   // index + 1 in the JVM's wrapping Int arithmetic
      t->hist_exp = true;
    }
  } else ok = false;
  if (!ok) return fail(ctx, FILO_ERR_UNSUPPORTED, "histogram bucket scheme not supported on the device path (1..64 geometric, custom or otel exponential buckets)");
  CUDA_TRY(ctx, cudaMalloc(&t->d_hist_tops, (size_t)nb * 8));
  CUDA_TRY(ctx, cudaMemcpy(t->d_hist_tops, t->hist_tops.data(), (size_t)nb * 8, cudaMemcpyHostToDevice));
  return FILO_OK;
}
static int32_t filo_load_series_impl(filo_ctx* ctx, int64_t n_series, const int32_t* n_chunks, const uint64_t* addrs,
                                    int32_t ts_col, int32_t val_col, const int32_t* group_ids, int32_t n_groups,
                                    int32_t schema_flags, filo_table** out) {
  if (!ctx || !out || n_series < 0 || (n_series > 0 && (!n_chunks || !addrs)) || ts_col < 0 || val_col < 0)
    return fail(ctx, FILO_ERR_INVALID_ARG, "filo_load_series: bad arguments");
  if (group_ids && n_groups <= 0) return fail(ctx, FILO_ERR_INVALID_ARG, "group_ids given but n_groups <= 0");
  if (group_ids && ctx->cfg.group_by_cardinality_limit > 0 && n_groups > ctx->cfg.group_by_cardinality_limit)
    return fail(ctx, FILO_ERR_QUERY_LIMIT, "Query exceeded group-by cardinality limit");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  std::vector<int64_t> chunk_base((size_t)n_series + 1, 0);
  for (int64_t i = 0; i < n_series; ++i) {
    if (n_chunks[i] < 0) return fail(ctx, FILO_ERR_INVALID_ARG, "negative n_chunks");
    chunk_base[i + 1] = chunk_base[i] + n_chunks[i];
  }
  // ---- pass 1: validate + size
  std::vector<SeriesPlan> plan((size_t)n_series);
  const LoadIn in{n_series, n_chunks, addrs, chunk_base.data(), ts_col, val_col};
  PlanTotals tot; int64_t err_series = -1;
  if (const int err_code = plan_all(in, plan, tot, err_series)) {
    const char* what = err_code == FILO_ERR_UNSUPPORTED ? "chunks of a series are not in increasing time order (unsupported on the device path)"
                                                       : "CorruptVector: unknown or inconsistent BinaryVector wire format";
    return fail(ctx, err_code, std::string(what) + " at series " + std::to_string(err_series));
  }
  std::vector<int64_t> rec_off((size_t)n_series + 1, 0);
  for (int64_t i = 0; i < n_series; ++i) rec_off[i + 1] = rec_off[i] + plan[i].rec_bytes;
  const int64_t arena_bytes = rec_off[n_series];
  if (ctx->cfg.max_data_per_shard_query > 0 && tot.alg > ctx->cfg.max_data_per_shard_query)
    return fail(ctx, FILO_ERR_QUERY_LIMIT, "raw data bytes scanned exceeds max-data-per-shard-query");
  if (tot.hist_def && tot.any_scalar) return fail(ctx, FILO_ERR_UNSUPPORTED, "histogram and scalar value vectors in one table");
  if (tot.hist_mismatch) return fail(ctx, FILO_ERR_UNSUPPORTED, "histogram bucket schemes differ inside the table (unsupported on the device path)");
  // ---- pass 2: fill pinned slabs, copy
  // everything allocated below is released on every early return (CUDA_TRY) until the table owns the arena
  struct LoadGuard {
    filo_table* t = nullptr; uint8_t* d_arena = nullptr; int64_t* d_rec_off = nullptr; uint8_t* slab[2] = {nullptr, nullptr}; cudaEvent_t ev[2] = {nullptr, nullptr};
    bool owns_table = true;
    ~LoadGuard() {
      for (int b = 0; b < 2; ++b) { if (ev[b]) { cudaEventSynchronize(ev[b]); cudaEventDestroy(ev[b]); } if (slab[b]) cudaFreeHost(slab[b]); }
      if (owns_table) { cudaFree(d_arena); cudaFree(d_rec_off); delete t; }
    }
  } lg;
  lg.t = new filo_table();
  filo_table*& t = lg.t; uint8_t*& d_arena = lg.d_arena; int64_t*& d_rec_off = lg.d_rec_off;
  CUDA_TRY(ctx, cudaMalloc(&d_arena, (size_t)arena_bytes + 64));
  CUDA_TRY(ctx, cudaMalloc(&d_rec_off, (size_t)(n_series + 1) * 8));
  CUDA_TRY(ctx, cudaMemsetAsync(d_arena + arena_bytes, 0, 64, ctx->stream));
  CUDA_TRY(ctx, cudaMemcpyAsync(d_rec_off, rec_off.data(), (size_t)(n_series + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
  const size_t SLAB = std::min<size_t>((size_t)256 << 20, std::max<size_t>((size_t)arena_bytes, 1 << 16));
  uint8_t** slab = lg.slab; cudaEvent_t* ev = lg.ev;
  for (int b = 0; b < 2; ++b) { CUDA_TRY(ctx, cudaHostAlloc(&slab[b], SLAB + (1 << 20), cudaHostAllocDefault)); CUDA_TRY(ctx, cudaEventCreateWithFlags(&ev[b], cudaEventDisableTiming)); }
  int64_t s0 = 0; int which = 0;
  while (s0 < n_series) {
    int64_t s1 = s0; const int64_t base = rec_off[s0];
    while (s1 < n_series && (size_t)(rec_off[s1 + 1] - base) <= SLAB) ++s1;
    if (s1 == s0) {   // a single record larger than the slab: grow this slab
      const size_t need = (size_t)plan[s0].rec_bytes;
      CUDA_TRY(ctx, cudaEventSynchronize(ev[which]));          // the previous copy out of this slab has finished
      cudaFreeHost(slab[which]); slab[which] = nullptr;
      CUDA_TRY(ctx, cudaHostAlloc(&slab[which], need + (1 << 20), cudaHostAllocDefault)); s1 = s0 + 1;
    }
    CUDA_TRY(ctx, cudaEventSynchronize(ev[which]));
    uint8_t* dst0 = slab[which];
    host_pool().run(s1 - s0, [&](int, int64_t b, int64_t e) {
      for (int64_t ii = b; ii < e; ++ii) { const int64_t i = s0 + ii; fill_record(in, i, plan[(size_t)i], dst0 + (rec_off[i] - base)); }
    });
    CUDA_TRY(ctx, cudaMemcpyAsync(d_arena + base, dst0, (size_t)(rec_off[s1] - base), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(ctx, cudaEventRecord(ev[which], ctx->stream));
    which ^= 1; s0 = s1;
  }
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  lg.owns_table = false;                               // from here on the table owns the arena; later failures go through filo_table_free
  filo_internal_set_arena(t, d_arena, d_rec_off, n_series, tot.chunks, tot.samples, arena_bytes + (n_series + 1) * 8, tot.alg, tot.maxrows, tot.maxch, schema_flags);
  filo_internal_set_layout(t, tot.max_rec, n_series > 0 && !(tot.f_and & REC_ALL_TS_CONST), (tot.f_or & REC_ANY_DROP) != 0);
  if (tot.hist_def) {                                  // histogram table: one bucket scheme, tops kept for histogram_quantile
    const int32_t rch = filo_internal_set_hist(ctx, t, tot.hist_def);
    if (rch != FILO_OK) { filo_table_free(ctx, t); return rch; }
    t->hist_simple = tot.hist_simple;
  }
  // groups
  int32_t* d_gid = nullptr;
  if (group_ids && n_series > 0) {
    for (int64_t i = 0; i < n_series; ++i) if (group_ids[i] < 0 || group_ids[i] >= n_groups) { filo_table_free(ctx, t); return fail(ctx, FILO_ERR_INVALID_ARG, "group id out of range"); }
    CUDA_TRY(ctx, cudaMalloc(&d_gid, (size_t)n_series * 4));
    CUDA_TRY(ctx, cudaMemcpy(d_gid, group_ids, (size_t)n_series * 4, cudaMemcpyHostToDevice));
  }
  int32_t rc = build_groups(ctx, t, d_gid, group_ids ? n_groups : 1);
  cudaFree(d_gid);
  if (rc) { filo_table_free(ctx, t); return rc; }
  *out = t;
  return FILO_OK;
}
extern "C" int32_t filo_load_series(filo_ctx* ctx, int64_t n_series, const int32_t* n_chunks, const uint64_t* addrs,
                                    int32_t ts_col, int32_t val_col, const int32_t* group_ids, int32_t n_groups,
                                    int32_t schema_flags, filo_table** out) {
  try { return filo_load_series_impl(ctx, n_series, n_chunks, addrs, ts_col, val_col, group_ids, n_groups, schema_flags, out); }
  catch (const std::bad_alloc&) { return fail(ctx, FILO_ERR_OOM, "filo_load_series: host allocation failed"); }
  catch (const std::exception& e) { return fail(ctx, FILO_ERR_INVALID_ARG, std::string("filo_load_series: ") + e.what()); }
}

extern "C" int32_t filo_table_set_groups(filo_ctx* ctx, filo_table* t, const int32_t* group_ids, int32_t n_groups) {
  if (!ctx || !t) return fail(ctx, FILO_ERR_INVALID_ARG, "null");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  if (group_ids && ctx->cfg.group_by_cardinality_limit > 0 && n_groups > ctx->cfg.group_by_cardinality_limit)
    return fail(ctx, FILO_ERR_QUERY_LIMIT, "Query exceeded group-by cardinality limit");
  int32_t* d_gid = nullptr;
  if (group_ids && t->n_series > 0) {
    for (int64_t i = 0; i < t->n_series; ++i) if (group_ids[i] < 0 || group_ids[i] >= n_groups) return fail(ctx, FILO_ERR_INVALID_ARG, "group id out of range");
    CUDA_TRY(ctx, cudaMalloc(&d_gid, (size_t)t->n_series * 4));
    CUDA_TRY(ctx, cudaMemcpy(d_gid, group_ids, (size_t)t->n_series * 4, cudaMemcpyHostToDevice));
  }
  int32_t rc = build_groups(ctx, t, d_gid, group_ids ? n_groups : 1);
  cudaFree(d_gid);
  return rc;
}

extern "C" int64_t filo_table_read_record(filo_ctx* ctx, const filo_table* t, int64_t series, uint8_t* out, int64_t cap) {
  if (!ctx || !t || series < 0 || series >= t->n_series) return fail(ctx, FILO_ERR_INVALID_ARG, "bad series");
  cudaSetDevice(ctx->device);
  int64_t off[2];
  if (cudaMemcpy(off, t->d_rec_off + series, 16, cudaMemcpyDeviceToHost) != cudaSuccess) return fail(ctx, FILO_ERR_CUDA, "read rec_off");
  int64_t n = off[1] - off[0];
  if (n > cap) return -n;
  if (cudaMemcpy(out, t->d_arena + off[0], (size_t)n, cudaMemcpyDeviceToHost) != cudaSuccess) return fail(ctx, FILO_ERR_CUDA, "read record");
  return n;
}

// ------------------------------------------------------------------------------------------------------------------
// incremental arena: new chunks of a resident table (TimeSeriesPartition.switchBuffers / encodeOneChunkset hand a shard's freshly
// encoded chunks over, core/src/main/scala/filodb.core/memstore/TimeSeriesPartition.scala:251-288).  Only the new chunks cross PCIe
// (loaded like a table of their own); the records are re-packed on the device: record = header + old entries + new entries + old
// vectors + new vectors, which is byte for byte what filo_load_series writes for all the chunks.
// ------------------------------------------------------------------------------------------------------------------
namespace {
// bytes of a record's vector region that hold vectors (the record itself is padded to 16): end of the last chunk's value vector
__device__ __forceinline__ uint32_t rec_used_vectors(const uint8_t* r) {
  const RecordHeader h = *reinterpret_cast<const RecordHeader*>(r);
  const uint32_t v0 = (uint32_t)sizeof(RecordHeader) + 32u * h.n_chunks;
  if (h.n_chunks == 0) return 0;
  const ChunkEntry& e = reinterpret_cast<const ChunkEntry*>(r + sizeof(RecordHeader))[h.n_chunks - 1];
  const uint32_t vt = *reinterpret_cast<const uint32_t*>(r + e.val_off) + 4u;
  return align_up(e.val_off + vt, 8) - v0;
}
__global__ void append_size_kernel(const uint8_t* __restrict__ ar_o, const int64_t* __restrict__ off_o, const uint8_t* __restrict__ ar_d, const int64_t* __restrict__ off_d,
                                   int64_t n, int64_t* __restrict__ sz) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const uint8_t* ro = ar_o + off_o[i]; const uint8_t* rd = ar_d + off_d[i];
    const uint32_t nn = reinterpret_cast<const RecordHeader*>(ro)->n_chunks + reinterpret_cast<const RecordHeader*>(rd)->n_chunks;
    sz[i] = (int64_t)align_up((uint32_t)sizeof(RecordHeader) + 32u * nn + rec_used_vectors(ro) + rec_used_vectors(rd), 16);
  }
  if (i == n) sz[i] = 0;
}
// warp per series; stats: [0] max record bytes, [1] max rows, [2] max chunks, [3] order violations
__global__ void __launch_bounds__(256) append_merge_kernel(const uint8_t* __restrict__ ar_o, const int64_t* __restrict__ off_o, const uint8_t* __restrict__ ar_d,
                                                           const int64_t* __restrict__ off_d, const int64_t* __restrict__ off_n, int64_t n,
                                                           uint8_t* __restrict__ ar_n, unsigned int* __restrict__ stats) {
  const int lane = threadIdx.x & 31;
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= n) return;
  const uint8_t* ro = ar_o + off_o[i]; const uint8_t* rd = ar_d + off_d[i]; uint8_t* rn = ar_n + off_n[i];
  const RecordHeader ho = *reinterpret_cast<const RecordHeader*>(ro), hd = *reinterpret_cast<const RecordHeader*>(rd);
  const uint32_t no = ho.n_chunks, nd = hd.n_chunks, nn = no + nd;
  const uint32_t vo0 = (uint32_t)sizeof(RecordHeader) + 32u * no, vd0 = (uint32_t)sizeof(RecordHeader) + 32u * nd, vn0 = (uint32_t)sizeof(RecordHeader) + 32u * nn;
  const uint32_t Lo = rec_used_vectors(ro), Ld = rec_used_vectors(rd);          // multiples of 8
  const uint32_t rec_bytes = align_up(vn0 + Lo + Ld, 16);
  if (lane == 0) {
    RecordHeader hn; hn.rec_bytes = rec_bytes; hn.n_chunks = nn; hn.n_rows = ho.n_rows + hd.n_rows;
    hn.flags = ((ho.flags & hd.flags) & REC_ALL_TS_CONST) | ((ho.flags | hd.flags) & ~REC_ALL_TS_CONST);
    *reinterpret_cast<RecordHeader*>(rn) = hn;
    atomicMax(&stats[0], hn.rec_bytes); atomicMax(&stats[1], hn.n_rows); atomicMax(&stats[2], nn);
    if (no && nd) {                                         // chunks stay in time order (the loader's rule, plan_series)
      const ChunkEntry& lo = reinterpret_cast<const ChunkEntry*>(ro + sizeof(RecordHeader))[no - 1];
      const ChunkEntry& fd = reinterpret_cast<const ChunkEntry*>(rd + sizeof(RecordHeader))[0];
      if (fd.start_time < lo.start_time || fd.end_time < lo.end_time) atomicAdd(&stats[3], 1u);
    }
    if ((vn0 + Lo + Ld) & 8u) *reinterpret_cast<uint64_t*>(rn + vn0 + Lo + Ld) = 0ull;      // the record's tail pad
  }
  for (uint32_t c = lane; c < nn; c += 32) {
    ChunkEntry e;
    if (c < no) { e = reinterpret_cast<const ChunkEntry*>(ro + sizeof(RecordHeader))[c]; e.ts_off += 32u * nd; e.val_off += 32u * nd; }
    else { e = reinterpret_cast<const ChunkEntry*>(rd + sizeof(RecordHeader))[c - no]; e.ts_off += 32u * no + Lo; e.val_off += 32u * no + Lo; e.row_base += ho.n_rows; }
    reinterpret_cast<ChunkEntry*>(rn + sizeof(RecordHeader))[c] = e;
  }
  // vector regions: multiples of 8 bytes at 8-byte aligned offsets
  const uint64_t* so = reinterpret_cast<const uint64_t*>(ro + vo0); uint64_t* dn = reinterpret_cast<uint64_t*>(rn + vn0);
  for (uint32_t q = lane; q < Lo / 8; q += 32) dn[q] = so[q];
  const uint64_t* sd = reinterpret_cast<const uint64_t*>(rd + vd0); dn = reinterpret_cast<uint64_t*>(rn + vn0 + Lo);
  for (uint32_t q = lane; q < Ld / 8; q += 32) dn[q] = sd[q];
}
}  // namespace

static int32_t filo_table_append_impl(filo_ctx* ctx, filo_table* t, const int32_t* n_chunks, const uint64_t* chunk_info_addrs, int32_t ts_col, int32_t val_col) {
  if (!ctx || !t || !n_chunks || !chunk_info_addrs) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_table_append: null argument");
  if (t->hist) return fail(ctx, FILO_ERR_UNSUPPORTED, "filo_table_append: histogram tables are rebuilt with filo_load_series");
  const int64_t S = t->n_series;
  filo_table* d = nullptr;
  { const int32_t rc = filo_load_series(ctx, S, n_chunks, chunk_info_addrs, ts_col, val_col, nullptr, 0, t->schema_flags, &d); if (rc != FILO_OK) return rc; }
  struct FreeT { filo_ctx* c; filo_table* t; ~FreeT() { filo_table_free(c, t); } } guard{ctx, d};
  if (d->hist) return fail(ctx, FILO_ERR_UNSUPPORTED, "filo_table_append: histogram vectors");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t s = ctx->stream;
  int64_t *d_sz = nullptr, *d_off = nullptr; unsigned int* d_stats = nullptr; void* tmp = nullptr; uint8_t* d_arena = nullptr;
  struct FreeD { std::vector<void*> p; ~FreeD() { for (void* x : p) cudaFree(x); } } tmps;
  CUDA_TRY(ctx, cudaMalloc(&d_sz, (size_t)(S + 1) * 8)); tmps.p.push_back(d_sz);
  CUDA_TRY(ctx, cudaMalloc(&d_off, (size_t)(S + 1) * 8));
  CUDA_TRY(ctx, cudaMalloc(&d_stats, 16)); tmps.p.push_back(d_stats);
  CUDA_TRY(ctx, cudaMemsetAsync(d_stats, 0, 16, s));
  append_size_kernel<<<(unsigned)((S + 1 + 255) / 256), 256, 0, s>>>(t->d_arena, t->d_rec_off, d->d_arena, d->d_rec_off, S, d_sz);
  size_t tmp_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, d_sz, d_off, (int)(S + 1), s);
  if (cudaMalloc(&tmp, tmp_bytes + 16) != cudaSuccess) { cudaFree(d_off); return fail(ctx, FILO_ERR_OOM, "filo_table_append: scan storage"); }
  tmps.p.push_back(tmp);
  if (cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, d_sz, d_off, (int)(S + 1), s) != cudaSuccess) { cudaFree(d_off); return fail(ctx, FILO_ERR_CUDA, "filo_table_append: scan"); }
  int64_t arena_bytes = 0;
  if (cudaMemcpyAsync(&arena_bytes, d_off + S, 8, cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) { cudaFree(d_off); return fail(ctx, FILO_ERR_CUDA, "filo_table_append: sizes"); }
  if (cudaMalloc(&d_arena, (size_t)arena_bytes + 64) != cudaSuccess) { cudaFree(d_off); return fail(ctx, FILO_ERR_OOM, "filo_table_append: the new arena does not fit beside the old one"); }
  cudaMemsetAsync(d_arena + arena_bytes, 0, 64, s);
  if (S > 0) append_merge_kernel<<<(unsigned)((S * 32 + 255) / 256), 256, 0, s>>>(t->d_arena, t->d_rec_off, d->d_arena, d->d_rec_off, d_off, S, d_arena, d_stats);
  unsigned int st[4] = {0, 0, 0, 0};
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpyAsync(st, d_stats, 16, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) { cudaFree(d_off); cudaFree(d_arena); return fail(ctx, FILO_ERR_CUDA, std::string("filo_table_append: ") + cudaGetErrorString(e)); }
  if (st[3]) { cudaFree(d_off); cudaFree(d_arena); return fail(ctx, FILO_ERR_UNSUPPORTED, "filo_table_append: new chunks must follow the resident ones in time (unsupported on the device path)"); }
  // swap the arena in; the table handle, its grouping and its series ordinals stay
  cudaFree(t->d_arena); cudaFree(t->d_rec_off);
  t->d_arena = d_arena; t->d_rec_off = d_off;
  t->n_chunks += d->n_chunks; t->n_samples += d->n_samples; t->algorithmic_bytes += d->algorithmic_bytes;
  t->arena_bytes = arena_bytes + (S + 1) * 8;
  t->max_rec_bytes = st[0]; t->max_rows = (int32_t)st[1]; t->max_chunks = (int32_t)st[2];
  t->any_nonconst_ts = t->any_nonconst_ts || (d->n_chunks > 0 && d->any_nonconst_ts); t->any_drop = t->any_drop || d->any_drop;
  return FILO_OK;
}
extern "C" int32_t filo_table_append(filo_ctx* ctx, filo_table* t, const int32_t* n_chunks, const uint64_t* chunk_info_addrs, int32_t ts_col, int32_t val_col) {
  try { return filo_table_append_impl(ctx, t, n_chunks, chunk_info_addrs, ts_col, val_col); }
  catch (const std::bad_alloc&) { return fail(ctx, FILO_ERR_OOM, "filo_table_append: host allocation failed"); }
  catch (const std::exception& e) { return fail(ctx, FILO_ERR_INVALID_ARG, std::string("filo_table_append: ") + e.what()); }
}

extern "C" int64_t filo_table_read_arena(filo_ctx* ctx, const filo_table* t, int64_t first, int64_t n, uint8_t* out, int64_t cap,
                                         int64_t* rec_off_out) {
  if (!ctx || !t || first < 0 || n < 0 || first + n > t->n_series || !rec_off_out) return fail(ctx, FILO_ERR_INVALID_ARG, "bad range");
  cudaSetDevice(ctx->device);
  if (cudaMemcpy(rec_off_out, t->d_rec_off + first, (size_t)(n + 1) * 8, cudaMemcpyDeviceToHost) != cudaSuccess)
    return fail(ctx, FILO_ERR_CUDA, "read rec_off");
  const int64_t base = rec_off_out[0], bytes = rec_off_out[n] - base;
  for (int64_t i = 0; i <= n; ++i) rec_off_out[i] -= base;
  if (bytes > cap || !out) return -bytes;
  if (bytes > 0 && cudaMemcpy(out, t->d_arena + base, (size_t)bytes, cudaMemcpyDeviceToHost) != cudaSuccess)
    return fail(ctx, FILO_ERR_CUDA, "read arena");
  return bytes;
}

// ------------------------------------------------------------------------------------------------------------------
// query
// ------------------------------------------------------------------------------------------------------------------
namespace {
struct Temp {   // stream-ordered temporaries, freed on scope exit
  cudaStream_t s; std::vector<void*> ptrs;
  explicit Temp(cudaStream_t st) : s(st) {}
  ~Temp() { for (void* p : ptrs) cudaFreeAsync(p, s); }
  cudaError_t alloc(void** p, size_t bytes) { cudaError_t e = cudaMallocAsync(p, bytes ? bytes : 16, s); if (e == cudaSuccess) ptrs.push_back(*p); return e; }
};
}

namespace {
// device error word + scan counters of one asynchronous query, copied to pinned host memory on the query's stream
struct AsyncSink { int herr[4]; unsigned long long hc[2]; int64_t launches; };
}
static int32_t query_device_impl(filo_ctx* ctx, const filo_table* t, int32_t fn, int64_t start, int64_t step, int64_t end, int64_t window,
                                 int32_t agg, int32_t k, int32_t flags, void* d_out_values, void* d_out_aux, void* cuda_stream,
                                 filo_stats* stats, AsyncSink* sink);
extern "C" int32_t filo_query_device(filo_ctx* ctx, const filo_table* t, int32_t fn, int64_t start, int64_t step, int64_t end, int64_t window,
                                     int32_t agg, int32_t k, int32_t flags, void* d_out_values, void* d_out_aux, void* cuda_stream,
                                     filo_stats* stats) {
  return query_device_impl(ctx, t, fn, start, step, end, window, agg, k, flags, d_out_values, d_out_aux, cuda_stream, stats, nullptr);
}
namespace {
struct EventPair {      // timing events of one query, destroyed on every return path
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  ~EventPair() { if (e0) cudaEventDestroy(e0); if (e1) cudaEventDestroy(e1); }
};
}
static int32_t report_device_error(filo_ctx* ctx, const int herr[4], int64_t series_base);
// completed error words of earlier non-synchronising queries; wait = also wait for the ones still in flight
static int32_t poll_async_errors(filo_ctx* ctx, bool wait) {
  std::lock_guard<std::mutex> g(ctx->errslot_mu);
  int32_t rc = FILO_OK;
  for (auto& sl : ctx->errslots) {
    if (!sl.pending) continue;
    cudaError_t e = wait ? cudaEventSynchronize(sl.ev) : cudaEventQuery(sl.ev);
    if (e == cudaErrorNotReady) { cudaGetLastError(); continue; }
    sl.pending = false;
    if (e != cudaSuccess) { if (rc == FILO_OK) rc = fail(ctx, FILO_ERR_CUDA, std::string("asynchronous query: ") + cudaGetErrorString(e)); continue; }
    if (sl.h[0] && rc == FILO_OK) rc = report_device_error(ctx, sl.h, 0);
  }
  return rc;
}
// non-synchronising call: its error word is copied into the next slot of the ring on its stream, so that it still reaches the caller
// (next call on this ctx, or filo_ctx_check)
static int32_t push_async_error(filo_ctx* ctx, const int* d_err, cudaStream_t s) {
  std::lock_guard<std::mutex> g(ctx->errslot_mu);
  filo_ctx::ErrSlot& sl = ctx->errslots[ctx->errslot_next];
  ctx->errslot_next = (ctx->errslot_next + 1) % 16;
  if (!sl.h) { CUDA_TRY(ctx, cudaMallocHost((void**)&sl.h, 16)); CUDA_TRY(ctx, cudaEventCreateWithFlags(&sl.ev, cudaEventDisableTiming)); }
  if (sl.pending) {           // the ring wrapped: the oldest query must have finished by now
    CUDA_TRY(ctx, cudaEventSynchronize(sl.ev)); sl.pending = false;
    if (sl.h[0]) return report_device_error(ctx, sl.h, 0);
  }
  CUDA_TRY(ctx, cudaMemcpyAsync(sl.h, d_err, 16, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(ctx, cudaEventRecord(sl.ev, s));
  sl.pending = true;
  return FILO_OK;
}
extern "C" int32_t filo_ctx_check(filo_ctx* ctx) {
  if (!ctx) return fail(nullptr, FILO_ERR_INVALID_ARG, "ctx is null");
  return poll_async_errors(ctx, true);
}
static int32_t report_device_error(filo_ctx* ctx, const int herr[4], int64_t series_base) {
  if (herr[0] == 5)           // only the histogram kernels set code 5
    return fail(ctx, FILO_ERR_UNSUPPORTED, "histogram series with more chunks / sections / rows in range than the device path holds, at series " +
                std::to_string(series_base + ((int64_t)herr[1] | ((int64_t)herr[2] << 31))));
  const char* what = herr[0] == 4 ? "series needs more decode scratch than the table statistics promised" : "CorruptVector on device";
  return fail(ctx, FILO_ERR_CORRUPT_VECTOR, std::string(what) + " (code " + std::to_string(herr[0]) + ") at series " +
              std::to_string(series_base + ((int64_t)herr[1] | ((int64_t)herr[2] << 31))));
}
static int32_t query_device_impl(filo_ctx* ctx, const filo_table* t, int32_t fn, int64_t start, int64_t step, int64_t end, int64_t window,
                                 int32_t agg, int32_t k, int32_t flags, void* d_out_values, void* d_out_aux, void* cuda_stream,
                                 filo_stats* stats, AsyncSink* sink) {
  if (!ctx || !t || !d_out_values) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_query: null argument");
  if (fn < FILO_FN_LAST || fn > FILO_FN_PRESENT_OVER_TIME) return fail(ctx, FILO_ERR_INVALID_ARG, "unknown range function");
  if (t->hist) return fail(ctx, FILO_ERR_UNSUPPORTED, "histogram table: use filo_query_hist");
  const bool long_values = (t->schema_flags & FILO_SCHEMA_LONG_VALUES) != 0;
  // RangeFunction.longChunkedFunction (RangeFunction.scala:319-339): the other functions fall back to the iterating (row-wise) path
  if (long_values && !fn_long_column_ok(fn)) return fail(ctx, FILO_ERR_UNSUPPORTED, "no chunked range function for this function on a Long column");
  if (fn == FILO_FN_HOLT_WINTERS) {                        // HoltWintersChunkedFunction.parseParameters, AggrOverTimeFunctions.scala:1374-1384
    if (!(ctx->fn_args[0] >= 0 && ctx->fn_args[0] <= 1)) return fail(ctx, FILO_ERR_INVALID_ARG, "Sf should be in between 0 and 1");
    if (!(ctx->fn_args[1] >= 0 && ctx->fn_args[1] <= 1)) return fail(ctx, FILO_ERR_INVALID_ARG, "tf should be in between 0 and 1");
  }
  if (agg < FILO_AGG_NONE || agg > FILO_AGG_GROUP) return fail(ctx, FILO_ERR_INVALID_ARG, "unknown aggregation operator");
  // PeriodicSamplesMapper.scala:45-49, 67-68
  if (start > end) return fail(ctx, FILO_ERR_INVALID_ARG, "start should be <= end");
  if (!(start == end || step > 0)) return fail(ctx, FILO_ERR_INVALID_ARG, "step should be > 0 for range query");
  if (start < end && step < ctx->cfg.min_step_ms) return fail(ctx, FILO_ERR_BAD_QUERY, "step should be at least min-step");
  const int64_t adjustedStep = step > 0 ? step : step + 1;
  const bool isLast = (fn == FILO_FN_LAST || fn == FILO_FN_TIMESTAMP);
  if (window <= 0) { if (isLast) window = 5 * 60 * 1000 + 1; else return fail(ctx, FILO_ERR_INVALID_ARG, "Need positive window lengths to apply range function"); }
  if ((agg == FILO_AGG_TOPK || agg == FILO_AGG_BOTTOMK) && (k <= 0 || k > FILO_MAX_TOPK)) return fail(ctx, FILO_ERR_INVALID_ARG, "topk/bottomk k must be in [1, 32]");
  if ((agg == FILO_AGG_TOPK || agg == FILO_AGG_BOTTOMK || agg == FILO_AGG_AVG) && !d_out_aux && !(agg == FILO_AGG_AVG && !(flags & FILO_Q_PARTIAL)))
    return fail(ctx, FILO_ERR_INVALID_ARG, "out_aux required");
  if ((flags & FILO_Q_PARTIAL) && agg != FILO_AGG_NONE && agg != FILO_AGG_TOPK && agg != FILO_AGG_BOTTOMK && !d_out_aux)
    return fail(ctx, FILO_ERR_INVALID_ARG, "partial aggregates need out_aux (counts)");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  { const int32_t prc = poll_async_errors(ctx, false); if (prc != FILO_OK) return prc; }      // an earlier stats == NULL query failed on the device
  cudaStream_t s = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
  QueryParams q{};
  q.start = start; q.step = adjustedStep; q.end = end; q.window = window; q.T = filo_num_windows(start, adjustedStep, end);
  q.fn = fn; q.cumulative = (t->schema_flags & FILO_SCHEMA_CUMULATIVE) ? 1 : 0; q.inclusive = ctx->cfg.inclusive_range ? 1 : 0;
  q.long_values = long_values ? 1 : 0; q.p0 = ctx->fn_args[0]; q.p1 = ctx->fn_args[1];
  const bool need_corr = (fn == FILO_FN_RATE || fn == FILO_FN_INCREASE) && q.cumulative;
  const bool fused = (agg != FILO_AGG_NONE && agg != FILO_AGG_TOPK && agg != FILO_AGG_BOTTOMK);
  // stddev / stdvar: the scan kernels fold (Σv, Σv², n) in their SUM mode plus a Σv² row; group folds the count partial.  Only
  // the merge / presentation sees the operator itself.
  const bool moments = agg_moments(agg);
  const int scan_op = moments ? AGG_SUM : agg == FILO_AGG_GROUP ? AGG_COUNT : agg;

  Temp tmp(s);
  int* d_err = nullptr; unsigned long long* d_counters = nullptr;
  CUDA_TRY(ctx, tmp.alloc((void**)&d_err, 16)); CUDA_TRY(ctx, tmp.alloc((void**)&d_counters, 16));
  CUDA_TRY(ctx, cudaMemsetAsync(d_err, 0, 16, s)); CUDA_TRY(ctx, cudaMemsetAsync(d_counters, 0, 16, s));
  EventPair evp;
  if (stats) { CUDA_TRY(ctx, cudaEventCreate(&evp.e0)); CUDA_TRY(ctx, cudaEventCreate(&evp.e1)); }
  cudaEvent_t& e0 = evp.e0; cudaEvent_t& e1 = evp.e1;

  // ---- kernel selection.  v2 (TMA-staged, blocked reductions) needs its whole per-warp working set in shared memory;
  //      v1 (generic, global-memory record reads, optional global scratch) takes everything else.  The v4 kernels and the tile
  //      kernel run in front of v2 where they apply.  FILO_KERNEL=v1 forces v1, v2 forces v2, v3 keeps the SUM class on the tile
  //      kernel (the other classes on v2).
  const uint32_t acc_bytes = fused ? align_up((uint32_t)q.T * (moments ? 20u : 12u), 128) : 0;
  const bool need_corr2 = need_corr && t->any_drop;
  uint32_t scratch2 = align_up((uint32_t)t->max_chunks * (uint32_t)CHUNK_DESC_BYTES, 16) +
                      ((uint32_t)t->max_rows + (uint32_t)t->max_chunks * 8u) * 8u * (1u + (t->any_nonconst_ts ? 1u : 0u) + (need_corr2 ? 1u : 0u));
  scratch2 = align_up(scratch2 + 16, 128);
  const uint32_t rec_cap = align_up(t->max_rec_bytes + 16, 128);
  const size_t per_warp2 = v2_smem_per_warp(rec_cap, scratch2, acc_bytes);
  const char* force_env = std::getenv("FILO_KERNEL");
  const std::string force = force_env ? force_env : "";
  const size_t smem_cap = std::min<size_t>(ctx->max_smem_optin, 227 * 1024);
  const bool use_v2 = force != "v1" && t->max_rec_bytes > 0 && per_warp2 * FAST_WARPS + 1024 <= smem_cap;
  const int64_t work = fused ? t->n_items : t->n_series;
  int64_t launches = 0;
  uint8_t* gscratch = nullptr;
  ScanLaunch L{t->d_arena, t->d_rec_off, t->n_series, q, nullptr, 0, 0, d_counters, d_err, 1, s};
  uint32_t rec_cap_used = 0;
  if (use_v2) {
    const size_t cta_smem = per_warp2 * FAST_WARPS + 1024;
    const int ctas_per_sm = (int)std::max<size_t>(1, std::min<size_t>(64 / FAST_WARPS, (size_t)(228 * 1024) / cta_smem));
    L.grid = (int)std::max<int64_t>(1, std::min<int64_t>((work + FAST_WARPS - 1) / FAST_WARPS, (int64_t)ctx->sm_count * ctas_per_sm));
    L.scratch_bytes = scratch2; L.use_smem = 1; rec_cap_used = rec_cap;
  } else {
    uint32_t scratch = align_up((uint32_t)t->max_chunks * (uint32_t)CHUNK_DESC_BYTES, 16) + (uint32_t)t->max_rows * 8u * (need_corr ? 3u : 2u);
    scratch = align_up(scratch + 16, 16);
    const size_t cta_smem = (size_t)(scratch + acc_bytes) * SCAN_WARPS;
    const int use_smem = cta_smem <= std::min<size_t>(ctx->max_smem_optin, 200 * 1024);
    int ctas_per_sm = 16;
    if (use_smem) ctas_per_sm = (int)std::max<size_t>(1, std::min<size_t>(16, (size_t)(220 * 1024) / std::max<size_t>(cta_smem + 1024, 1)));
    L.grid = (int)std::max<int64_t>(1, std::min<int64_t>((work + SCAN_WARPS - 1) / SCAN_WARPS, (int64_t)ctx->sm_count * ctas_per_sm));
    if (!use_smem) CUDA_TRY(ctx, tmp.alloc((void**)&gscratch, (size_t)L.grid * SCAN_WARPS * (scratch + acc_bytes)));
    L.gscratch = gscratch; L.scratch_bytes = scratch; L.use_smem = use_smem;
  }
  const int fn_cls = fn_class_of(fn, q.cumulative, q.long_values);
  const uint64_t wrows = (uint64_t)(q.window / q.step) + 1;
  // the per-series kernel in front of v2 (scan_path, scan_wp_layout.h): the v4 SUM kernels, the tile kernel or the v4 counter kernel;
  // what it declines goes to the v2 kernel
  ScanPathIn pin{};
  pin.max_rec_bytes = t->max_rec_bytes; pin.max_rows = (uint32_t)t->max_rows; pin.max_chunks = (uint32_t)t->max_chunks; pin.T = (uint32_t)q.T;
  pin.wrows = wrows; pin.fn_cls = fn_cls; pin.fused = fused; pin.moments = moments; pin.irr = t->any_nonconst_ts; pin.v2 = use_v2;
  pin.force = force == "v2" ? 2 : force == "v3" ? 3 : 0; pin.smem_cap = smem_cap; pin.n_series = t->n_series; pin.n_items = t->n_items; pin.sm_count = ctx->sm_count;
  const ScanPath SP = scan_path(pin);
  if (SP.refused) return fail(ctx, FILO_ERR_UNSUPPORTED, "scan_wp_batch_kernel: O on V with plans of more than one pass");
  const TileSmem& TL = SP.TL; const WpSmem& WL = SP.WL; const WpBatchSmem& WB = SP.WB; const WpCtrSmem& WC = SP.WC;
  const bool use_tile = SP.tile, use_wp_ctr = SP.wp_ctr;
  auto run_per_series = [&](double* outp) -> int32_t {
    if (use_tile || use_wp_ctr) {
      int64_t* d_list = nullptr; unsigned long long* d_cnt = nullptr;
      CUDA_TRY(ctx, tmp.alloc((void**)&d_list, (size_t)t->n_series * 8));
      CUDA_TRY(ctx, tmp.alloc((void**)&d_cnt, 16));
      CUDA_TRY(ctx, cudaMemsetAsync(d_cnt, 0, 16, s));
      ScanLaunch LT = L;
      static const bool dbg = std::getenv("FILO_DEBUG_SYNC") != nullptr;
      LT.grid = SP.grid;
      if (SP.kernel == SCAN_PATH_WP_BATCH) {
        CUDA_TRY(ctx, launch_scan_wp_batch(LT, outp, WB, d_list, d_cnt));
      } else if (SP.kernel == SCAN_PATH_WP_SUM) {
        CUDA_TRY(ctx, launch_scan_wp(LT, outp, WL, d_list, d_cnt));
      } else if (SP.kernel == SCAN_PATH_WP_CTR) {
        CUDA_TRY(ctx, launch_scan_wp_ctr(LT, outp, WC, d_list, d_cnt));
      } else {
        if (dbg) { fprintf(stderr, "[filo] tile kernel fn=%d T=%d grid=%d smem=%u pitch=%u\n", fn, q.T, LT.grid, TL.total, TL.vals_pitch); fflush(stderr); }
        CUDA_TRY(ctx, launch_scan_tile(LT, outp, TL, d_list, d_cnt));
      }
      if (dbg) { CUDA_TRY(ctx, cudaStreamSynchronize(s)); fprintf(stderr, "[filo] tile kernel done\n"); fflush(stderr); }
      ScanLaunch LF = L; LF.list = d_list; LF.list_count = d_cnt;
      CUDA_TRY(ctx, launch_scan_series_v2(LF, outp, rec_cap_used));
      if (dbg) { CUDA_TRY(ctx, cudaStreamSynchronize(s)); fprintf(stderr, "[filo] fallback kernel done\n"); fflush(stderr); }
      launches += 2;
    } else {
      CUDA_TRY(ctx, use_v2 ? launch_scan_series_v2(L, outp, rec_cap_used) : launch_scan_series(L, outp));
      launches += 1;
    }
    return FILO_OK;
  };
  if (stats) CUDA_TRY(ctx, cudaEventRecord(e0, s));
  if (agg == FILO_AGG_NONE) {
    { int32_t rc = run_per_series((double*)d_out_values); if (rc) return rc; }
  } else if (!fused) {
    double* per = nullptr;
    CUDA_TRY(ctx, tmp.alloc((void**)&per, (size_t)t->n_series * q.T * 8));
    { int32_t rc = run_per_series(per); if (rc) return rc; }
    CUDA_TRY(ctx, launch_topk(per, t->grouped ? t->d_order : nullptr, t->d_group_start, t->n_groups, q.T, k, agg == FILO_AGG_BOTTOMK,
                              (double*)d_out_values, (int64_t*)d_out_aux, s));
    launches += 1;
  } else {
    double* pval = nullptr; uint32_t* pcnt = nullptr;
    CUDA_TRY(ctx, tmp.alloc((void**)&pval, (size_t)t->n_items * q.T * 8 * (moments ? 2 : 1)));      // moments: [2][n_items][T]
    CUDA_TRY(ctx, tmp.alloc((void**)&pcnt, (size_t)t->n_items * q.T * 4));
    const int32_t* order = t->grouped ? t->d_order : nullptr;
    if (SP.fused_kernel != SCAN_PATH_V2) {
      // the tile / v4 counter kernel folds every item into one partial row; items with a series it declines go through the v2 kernel
      int64_t* d_list = nullptr; unsigned long long* d_cnt = nullptr;
      CUDA_TRY(ctx, tmp.alloc((void**)&d_list, (size_t)t->n_items * 8));
      CUDA_TRY(ctx, tmp.alloc((void**)&d_cnt, 16));
      CUDA_TRY(ctx, cudaMemsetAsync(d_cnt, 0, 16, s));
      ScanLaunch LT = L;
      LT.grid = SP.fused_grid;
      if (SP.fused_kernel == SCAN_PATH_WP_CTR) {
        CUDA_TRY(ctx, launch_scan_wp_ctr_agg(LT, WC, order, t->d_item_begin, t->n_items, scan_op, pval, pcnt, d_list, d_cnt, moments));
      } else {
        CUDA_TRY(ctx, launch_scan_tile_agg(LT, TL, order, t->d_item_begin, t->n_items, scan_op, pval, pcnt, d_list, d_cnt, moments));
      }
      ScanLaunch LF = L; LF.list = d_list; LF.list_count = d_cnt;
      CUDA_TRY(ctx, launch_scan_agg_v2(LF, order, t->d_item_begin, t->n_items, scan_op, pval, pcnt, acc_bytes, rec_cap_used, moments));
      launches += 1;
    } else {
      // (the v1 kernel reads the moments mode from the operator itself)
      CUDA_TRY(ctx, use_v2 ? launch_scan_agg_v2(L, order, t->d_item_begin, t->n_items, scan_op, pval, pcnt, acc_bytes, rec_cap_used, moments)
                           : launch_scan_agg(L, order, t->d_item_begin, t->n_items, moments ? agg : scan_op, pval, pcnt, acc_bytes));
    }
    CUDA_TRY(ctx, launch_merge_partials(pval, pcnt, t->d_gis, t->n_groups, q.T, agg, (flags & FILO_Q_PARTIAL) ? 1 : 0,
                                        (double*)d_out_values, (int64_t*)d_out_aux, s));
    launches += 2;
  }
  if (stats) {
    CUDA_TRY(ctx, cudaEventRecord(e1, s));
    int herr[4]; unsigned long long hc[2];
    CUDA_TRY(ctx, cudaMemcpyAsync(herr, d_err, 16, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(hc, d_counters, 16, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaStreamSynchronize(s));
    float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
    stats->kernel_ns = (int64_t)((double)ms * 1e6); stats->samples_scanned = (int64_t)hc[0]; stats->bytes_scanned = (int64_t)hc[1];
    stats->kernel_launches = launches; stats->h2d_bytes = 0; stats->d2h_bytes = 0;
    if (herr[0]) return report_device_error(ctx, herr, 0);
  }
  if (!stats && !sink) { const int32_t rc = push_async_error(ctx, d_err, s); if (rc != FILO_OK) return rc; }
  if (sink) {           // asynchronous caller: the words land in pinned memory when the stream reaches this point
    sink->launches = launches;
    CUDA_TRY(ctx, cudaMemcpyAsync(sink->herr, d_err, 16, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(ctx, cudaMemcpyAsync(sink->hc, d_counters, 16, cudaMemcpyDeviceToHost, s));
  }
  return FILO_OK;
}

static int32_t filo_query_impl(filo_ctx* ctx, const filo_table* t, int32_t fn, int64_t start, int64_t step, int64_t end, int64_t window,
                              int32_t agg, int32_t k, int32_t flags, double* out_values, int64_t* out_aux, filo_stats* stats) {
  if (!ctx || !t || !out_values) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_query: null argument");
  if (start > end) return fail(ctx, FILO_ERR_INVALID_ARG, "start should be <= end");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  const int64_t adjustedStep = step > 0 ? step : step + 1;
  const int T = filo_num_windows(start, adjustedStep, end);
  size_t nvals, naux = 0;
  if (agg == FILO_AGG_NONE) nvals = (size_t)t->n_series * T;
  else if (agg == FILO_AGG_TOPK || agg == FILO_AGG_BOTTOMK) { if (k <= 0 || k > FILO_MAX_TOPK) return fail(ctx, FILO_ERR_INVALID_ARG, "topk/bottomk k must be in [1, 32]"); nvals = naux = (size_t)t->n_groups * T * k; }
  else { naux = (size_t)t->n_groups * T; nvals = naux * ((flags & FILO_Q_PARTIAL) && agg_moments(agg) ? 2 : 1); }      // partial moments: Σv, Σv² blocks
  cudaStream_t s = ctx->stream;
  double* d_vals = nullptr; int64_t* d_aux = nullptr;
  CUDA_TRY(ctx, cudaMallocAsync((void**)&d_vals, std::max<size_t>(nvals, 1) * 8, s));
  if (naux) CUDA_TRY(ctx, cudaMallocAsync((void**)&d_aux, naux * 8, s));
  filo_stats st{};
  int32_t rc = filo_query_device(ctx, t, fn, start, step, end, window, agg, k, flags, d_vals, d_aux, s, &st);
  if (rc == FILO_OK) {
    cudaError_t e = cudaMemcpyAsync(out_values, d_vals, nvals * 8, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess && naux && out_aux) e = cudaMemcpyAsync(out_aux, d_aux, naux * 8, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) rc = fail(ctx, FILO_ERR_CUDA, std::string("result copy: ") + cudaGetErrorString(e));
    st.d2h_bytes = (int64_t)(nvals * 8 + ((naux && out_aux) ? naux * 8 : 0));
  }
  cudaFreeAsync(d_vals, s); if (d_aux) cudaFreeAsync(d_aux, s);
  if (stats) *stats = st;
  return rc;
}
extern "C" int32_t filo_query(filo_ctx* ctx, const filo_table* t, int32_t fn, int64_t start, int64_t step, int64_t end, int64_t window,
                              int32_t agg, int32_t k, int32_t flags, double* out_values, int64_t* out_aux, filo_stats* stats) {
  try { return filo_query_impl(ctx, t, fn, start, step, end, window, agg, k, flags, out_values, out_aux, stats); }
  catch (const std::bad_alloc&) { return fail(ctx, FILO_ERR_OOM, "filo_query: host allocation failed"); }
  catch (const std::exception& e) { return fail(ctx, FILO_ERR_INVALID_ARG, std::string("filo_query: ") + e.what()); }
}



// AvgWithSumAndCountOverTimeFuncD / FuncL (AggrOverTimeFunctions.scala:820-893): avg_over_time over downsampled data
namespace {
__global__ void ratio_kernel(double* __restrict__ num, const double* __restrict__ den, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) num[i] = num[i] / den[i];   // sumFunc.sum / countFunc.sum (IEEE)
}
}
static int32_t filo_query_avg_sum_count_impl(filo_ctx* ctx, const filo_table* t_sum, const filo_table* t_count, int64_t start, int64_t step, int64_t end,
                                             int64_t window, double* out_values, filo_stats* stats) {
  if (!ctx || !t_sum || !t_count || !out_values) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_query_avg_sum_count: null argument");
  if (start > end) return fail(ctx, FILO_ERR_INVALID_ARG, "start should be <= end");
  if (t_sum->hist || t_count->hist) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_query_avg_sum_count: scalar columns only");
  if (t_sum->n_series != t_count->n_series) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_query_avg_sum_count: the two tables hold different numbers of series");
  if (t_count->schema_flags & FILO_SCHEMA_LONG_VALUES) return fail(ctx, FILO_ERR_UNSUPPORTED, "filo_query_avg_sum_count: the count column is read as a DoubleVector (AggrOverTimeFunctions.scala:851,890)");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  const int64_t adjustedStep = step > 0 ? step : step + 1;
  const int T = filo_num_windows(start, adjustedStep, end);
  const size_t n = (size_t)t_sum->n_series * (size_t)T;
  cudaStream_t s = ctx->stream;
  Temp tmp(s);
  double *d_num = nullptr, *d_den = nullptr;
  CUDA_TRY(ctx, tmp.alloc((void**)&d_num, n * 8));
  CUDA_TRY(ctx, tmp.alloc((void**)&d_den, n * 8));
  // FuncD: both columns through SumOverTimeChunkedFunctionD; FuncL (Long sum column): SumOverTimeChunkedFunctionL over the sum column and
  // CountOverTimeChunkedFunction over the count column -- the row range of a window comes from the shared timestamp column either way
  const bool long_sum = (t_sum->schema_flags & FILO_SCHEMA_LONG_VALUES) != 0;
  filo_stats a{}, b{};
  int32_t rc = filo_query_device(ctx, t_sum, FILO_FN_SUM_OVER_TIME, start, step, end, window, FILO_AGG_NONE, 0, 0, d_num, nullptr, s, &a);
  if (rc == FILO_OK) rc = filo_query_device(ctx, t_count, long_sum ? FILO_FN_COUNT_OVER_TIME : FILO_FN_SUM_OVER_TIME, start, step, end, window, FILO_AGG_NONE, 0, 0, d_den, nullptr, s, &b);
  if (rc != FILO_OK) return rc;
  if (n) {
    ratio_kernel<<<(unsigned)std::min<size_t>((n + 255) / 256, (size_t)ctx->sm_count * 16), 256, 0, s>>>(d_num, d_den, (int64_t)n);
    CUDA_TRY(ctx, cudaGetLastError());
    CUDA_TRY(ctx, cudaMemcpyAsync(out_values, d_num, n * 8, cudaMemcpyDeviceToHost, s));
  }
  CUDA_TRY(ctx, cudaStreamSynchronize(s));
  if (stats) {
    *stats = a;
    stats->bytes_scanned += b.bytes_scanned; stats->samples_scanned += b.samples_scanned; stats->kernel_ns += b.kernel_ns;
    stats->kernel_launches += b.kernel_launches + 1; stats->d2h_bytes = (int64_t)(n * 8);
  }
  return FILO_OK;
}
extern "C" int32_t filo_query_avg_sum_count(filo_ctx* ctx, const filo_table* t_sum, const filo_table* t_count, int64_t start, int64_t step, int64_t end,
                                            int64_t window, double* out_values, filo_stats* stats) {
  try { return filo_query_avg_sum_count_impl(ctx, t_sum, t_count, start, step, end, window, out_values, stats); }
  catch (const std::bad_alloc&) { return fail(ctx, FILO_ERR_OOM, "filo_query_avg_sum_count: host allocation failed"); }
  catch (const std::exception& e) { return fail(ctx, FILO_ERR_INVALID_ARG, std::string("filo_query_avg_sum_count: ") + e.what()); }
}

// ------------------------------------------------------------------------------------------------------------------
// zero-copy gather: the GPU reads chunk vectors straight out of registered (pinned, mapped) host memory
// ------------------------------------------------------------------------------------------------------------------
namespace {

__device__ __forceinline__ void copy_bytes_warp(uint8_t* dst, const uint8_t* src, int n, int lane) {
  // dst is 8-byte aligned; BinaryVectors are allocated word aligned (32-bit loads measured faster than 64-bit ones over PCIe)
  const uintptr_t a = reinterpret_cast<uintptr_t>(src);
  if ((a & 3) == 0) {
    const int nw = n >> 2;
    const uint32_t* s4 = reinterpret_cast<const uint32_t*>(src); uint32_t* d4 = reinterpret_cast<uint32_t*>(dst);
    for (int i = lane; i < nw; i += 32) d4[i] = s4[i];
    for (int i = (nw << 2) + lane; i < n; i += 32) dst[i] = src[i];
  } else {
    for (int i = lane; i < n; i += 32) dst[i] = src[i];
  }
}
// warp per series: record header, chunk entries, vectors verbatim (same bytes fill_record writes on the host)
// rebase: added to every source address (0: read the registered host memory directly; otherwise the span was copied to the device
// and the sources are rebased into that copy)
__global__ void __launch_bounds__(256) gather_records_kernel(const GatherSeries* __restrict__ gs, const GatherChunk* __restrict__ gc,
                                                             const int64_t* __restrict__ rec_off, int64_t n, uint8_t* __restrict__ arena, int64_t rebase) {
  const int lane = threadIdx.x & 31;
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = w; i < n; i += nw) {
    const GatherSeries S = gs[i];
    uint8_t* rec = arena + rec_off[i];
    if (lane == 0) { RecordHeader h{S.rec_bytes, S.n_chunks, S.n_rows, S.flags}; *reinterpret_cast<RecordHeader*>(rec) = h; }
    uint32_t off = sizeof(RecordHeader) + S.n_chunks * (uint32_t)sizeof(ChunkEntry), row_base = 0;
    for (uint32_t c = 0; c < S.n_chunks; ++c) {
      const GatherChunk G = gc[S.first_chunk + c];
      const uint32_t ts_off = off, ts_pad = align_up((uint32_t)G.ts_bytes, 8), val_off = off + ts_pad, val_pad = align_up((uint32_t)G.val_bytes, 8);
      if (lane == 0) {
        ChunkEntry ce; ce.start_time = G.start_time; ce.end_time = G.end_time; ce.num_rows = G.num_rows; ce.ts_off = ts_off; ce.val_off = val_off; ce.row_base = row_base;
        reinterpret_cast<ChunkEntry*>(rec + sizeof(RecordHeader))[c] = ce;
      }
      copy_bytes_warp(rec + ts_off, reinterpret_cast<const uint8_t*>(G.ts_src + (uint64_t)rebase), G.ts_bytes, lane);
      copy_bytes_warp(rec + val_off, reinterpret_cast<const uint8_t*>(G.val_src + (uint64_t)rebase), G.val_bytes, lane);
      if (lane < (int)(ts_pad - G.ts_bytes)) rec[ts_off + G.ts_bytes + lane] = 0;
      if (lane < (int)(val_pad - G.val_bytes)) rec[val_off + G.val_bytes + lane] = 0;
      __syncwarp();
      if (lane == 0 && G.drop_patch) { if (G.drop_patch == 1) rec[val_off + 7] |= 0x80; else rec[val_off + 7] &= 0x7f; }
      off = val_off + val_pad; row_base += (uint32_t)G.val_len;
    }
    for (uint32_t k = off + lane; k < S.rec_bytes; k += 32) rec[k] = 0;
  }
}
}

extern "C" int32_t filo_host_register(filo_ctx* ctx, const void* base, int64_t bytes) {
  if (!ctx || !base || bytes <= 0) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_host_register: bad arguments");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  CUDA_TRY(ctx, cudaHostRegister(const_cast<void*>(base), (size_t)bytes, cudaHostRegisterMapped | cudaHostRegisterPortable));
  std::lock_guard<std::mutex> g(ctx->scan_mu);
  ctx->ranges.push_back({(uintptr_t)base, (size_t)bytes});
  return FILO_OK;
}
extern "C" int32_t filo_host_unregister(filo_ctx* ctx, const void* base) {
  if (!ctx || !base) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_host_unregister: bad arguments");
  std::lock_guard<std::mutex> g(ctx->scan_mu);
  for (size_t i = 0; i < ctx->ranges.size(); ++i) if (ctx->ranges[i].base == (uintptr_t)base) {
    for (auto& sl : ctx->scan) if (sl.stream) cudaStreamSynchronize(sl.stream);
    CUDA_TRY(ctx, cudaHostUnregister(const_cast<void*>(base)));
    ctx->ranges.erase(ctx->ranges.begin() + (long)i);
    return FILO_OK;
  }
  return fail(ctx, FILO_ERR_INVALID_ARG, "filo_host_unregister: range not registered");
}

// ------------------------------------------------------------------------------------------------------------------
// filo_scan_series: ingest + query + result read-back of host-resident chunks in one pipelined call
// ------------------------------------------------------------------------------------------------------------------
namespace {
template <class T> int32_t grow_pinned(filo_ctx* ctx, T*& p, size_t& cap, size_t need) {
  if (need <= cap) return FILO_OK;
  cudaFreeHost(p); p = nullptr; cap = 0;
  CUDA_TRY(ctx, cudaHostAlloc((void**)&p, need, cudaHostAllocDefault));
  cap = need; return FILO_OK;
}
template <class T> int32_t grow_device(filo_ctx* ctx, T*& p, size_t& cap, size_t need) {
  if (need <= cap) return FILO_OK;
  cudaFree(p); p = nullptr; cap = 0;
  CUDA_TRY(ctx, cudaMalloc((void**)&p, need));
  cap = need; return FILO_OK;
}
}

static int32_t filo_scan_series_impl(filo_ctx* ctx, int64_t n_series, const int32_t* n_chunks, const uint64_t* addrs,
                                    int32_t ts_col, int32_t val_col, int32_t schema_flags,
                                    int32_t fn, int64_t start, int64_t step, int64_t end, int64_t window,
                                    double* out_values, filo_stats* stats) {
  if (!ctx || n_series < 0 || (n_series > 0 && (!n_chunks || !addrs || !out_values)) || ts_col < 0 || val_col < 0)
    return fail(ctx, FILO_ERR_INVALID_ARG, "filo_scan_series: bad arguments");
  if (start > end) return fail(ctx, FILO_ERR_INVALID_ARG, "start should be <= end");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  std::lock_guard<std::mutex> one(ctx->scan_mu);          // the slots are shared: one streaming scan per context at a time
  const int64_t adjustedStep = step > 0 ? step : step + 1;
  const int T = filo_num_windows(start, adjustedStep, end);
  static const bool timing = std::getenv("FILO_DEBUG_TIMING") != nullptr;
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto ms_since = [](std::chrono::steady_clock::time_point a) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count(); };
  const auto t_begin = now();
  double t_fill = 0, t_retire = 0, t_enq = 0;
  // The series are planned (validated + sized, same rules as filo_load_series) in chunks of PLAN_CHUNK series right before their batches
  // are enqueued, so that the host walk of chunk k + 1 runs while the GPU still works on the batches of chunk k.
  // (per-call state is sized by the plan chunk, not by n_series: the first batch is on its way after one chunk's walk)
  std::vector<SeriesPlan> plan;
  std::vector<int64_t> chunk_base;                      // ChunkSetInfo list positions of the plan chunk's series (+ one past the end)
  int64_t chunks_before = 0;                            // ... of the series before the chunk
  LoadIn in{n_series, n_chunks, addrs, nullptr, ts_col, val_col};
  auto env_int = [](const char* name, long dflt, long lo, long hi) { const char* e = std::getenv(name); if (!e || !*e) return dflt; const long v = std::atol(e); return v < lo ? lo : v > hi ? hi : v; };
  const int64_t PLAN_CHUNK = env_int("FILO_SCAN_PLAN_CHUNK", 65536, 1024, 1 << 24);
  std::vector<GatherChunk> gc_walk;                     // gather entries of the plan chunk, written by the planning walk
  const size_t SLAB = (size_t)env_int("FILO_SCAN_SLAB_MB", 192, 1, 4096) << 20;
  const int64_t max_rows_out = std::max<int64_t>(1, (int64_t)(((size_t)env_int("FILO_SCAN_OUT_MB", 256, 1, 4096) << 20) / ((size_t)std::max(T, 1) * 8)));
  // FILO_SCAN_TRACE=<file>: device timeline of every batch (ms since the first batch was enqueued): start, inputs on the device, kernels done, result on the host
  const char* trace_path = std::getenv("FILO_SCAN_TRACE");
  struct TraceRow { int64_t nb; size_t bytes; double host_ms; cudaEvent_t ev[4]; };
  std::vector<TraceRow> trace; cudaEvent_t trace_t0 = nullptr;
  struct Batch { int64_t s0, s1; size_t bytes; int64_t chunks; };
  std::vector<filo_ctx::HostRange> ranges = ctx->ranges;
  auto in_ranges = [&](const uint8_t* p, size_t n) { for (auto& r : ranges) if ((uintptr_t)p >= r.base && (uintptr_t)p + n <= r.base + r.bytes) return true; return false; };
  const int NSLOT = (int)env_int("FILO_SCAN_SLOTS", 6, 2, filo_ctx::MAX_SCAN_SLOTS);   // 3 drain while the host walks the next plan chunk
  for (int i = 0; i < NSLOT; ++i) {
    filo_ctx::ScanSlot& sl = ctx->scan[i];
    if (!sl.stream) { CUDA_TRY(ctx, cudaStreamCreateWithFlags(&sl.stream, cudaStreamNonBlocking)); CUDA_TRY(ctx, cudaEventCreateWithFlags(&sl.done, cudaEventDisableTiming)); }
    if (!sl.h_sink) CUDA_TRY(ctx, cudaHostAlloc(&sl.h_sink, sizeof(AsyncSink), cudaHostAllocDefault));
  }
  double t_plan = 0;
  int64_t alg_total = 0; size_t n_batches = 0;
  // ---- pipeline: gather batch b (host pool) while the GPU copies/scans batch b-1 and returns batch b-2
  filo_stats acc{};
  struct InFlight { int64_t s0 = -1; } fl[filo_ctx::MAX_SCAN_SLOTS];
  int32_t rc = FILO_OK;
  auto retire = [&](int i) -> int32_t {             // the slot's previous batch has completed: collect its counters / errors
    filo_ctx::ScanSlot& sl = ctx->scan[i];
    if (fl[i].s0 < 0) return FILO_OK;
    CUDA_TRY(ctx, cudaEventSynchronize(sl.done));
    const AsyncSink* k = reinterpret_cast<const AsyncSink*>(sl.h_sink);
    acc.samples_scanned += (int64_t)k->hc[0]; acc.bytes_scanned += (int64_t)k->hc[1]; acc.kernel_launches += k->launches;
    const int64_t base = fl[i].s0; fl[i].s0 = -1;
    if (k->herr[0]) return report_device_error(ctx, k->herr, base);
    return FILO_OK;
  };
  for (int64_t c0 = 0; c0 < n_series && rc == FILO_OK; c0 += PLAN_CHUNK) {
    const int64_t c1 = std::min<int64_t>(n_series, c0 + PLAN_CHUNK);
    const auto t_p0 = now();
    PlanTotals tot; int64_t err_series = -1;
    plan.resize((size_t)(c1 - c0)); chunk_base.resize((size_t)(c1 - c0) + 1);
    chunk_base[0] = chunks_before;
    for (int64_t i = c0; i < c1; ++i) {
      if (n_chunks[i] < 0) { rc = fail(ctx, FILO_ERR_INVALID_ARG, "negative n_chunks"); break; }
      chunk_base[(size_t)(i - c0) + 1] = chunk_base[(size_t)(i - c0)] + n_chunks[i];
    }
    if (rc != FILO_OK) break;
    chunks_before = chunk_base[(size_t)(c1 - c0)];
    in.chunk_base = chunk_base.data(); in.cb0 = c0;
    if (!ranges.empty()) {                              // one walk: plan + gather entries + range check
      gc_walk.resize((size_t)(chunk_base[(size_t)(c1 - c0)] - chunk_base[0]) + 1);
      in.gc_out = gc_walk.data(); in.gc_base = chunk_base[0]; in.ranges = &ranges;
    }
    if (const int err_code = plan_range(in, c0, c1, plan, tot, err_series, c0)) {
      const char* what = err_code == FILO_ERR_UNSUPPORTED ? "chunks of a series are not in increasing time order (unsupported on the device path)"
                                                         : "CorruptVector: unknown or inconsistent BinaryVector wire format";
      rc = fail(ctx, err_code, std::string(what) + " at series " + std::to_string(err_series)); break;
    }
    alg_total += tot.alg;
    if (ctx->cfg.max_data_per_shard_query > 0 && alg_total > ctx->cfg.max_data_per_shard_query) { rc = fail(ctx, FILO_ERR_QUERY_LIMIT, "raw data bytes scanned exceeds max-data-per-shard-query"); break; }
    if (tot.hist_def) { rc = fail(ctx, FILO_ERR_UNSUPPORTED, "filo_scan_series: histogram columns go through filo_load_series + filo_query_hist"); break; }
    // zero-copy gather when every vector of the chunk lies in memory registered with filo_host_register (checked by the planning walk)
    const bool use_gather = !ranges.empty() && tot.all_in_ranges;
    // batches of the chunk: consecutive series, <= SLAB bytes of records and a bounded result block
    std::vector<Batch> batches;
    size_t chunk_bytes = 0; for (int64_t i = c0; i < c1; ++i) chunk_bytes += plan[(size_t)(i - c0)].rec_bytes;
    const size_t parts = std::max<size_t>((chunk_bytes + SLAB - 1) / SLAB, (size_t)((c1 - c0 + max_rows_out - 1) / max_rows_out));
    const size_t part_bytes = std::min(SLAB, chunk_bytes / std::max<size_t>(parts, 1) + (size_t)tot.max_rec);   // even parts: equal transfers keep both copy engines busy
    for (int64_t s0 = c0; s0 < c1;) {
      int64_t s1 = s0; size_t bytes = 0; int64_t chunks = 0;
      while (s1 < c1 && s1 - s0 < max_rows_out && (s1 == s0 || bytes + plan[(size_t)(s1 - c0)].rec_bytes <= part_bytes)) { bytes += plan[(size_t)(s1 - c0)].rec_bytes; chunks += plan[(size_t)(s1 - c0)].n_chunks; ++s1; }
      batches.push_back(Batch{s0, s1, bytes, chunks});
      s0 = s1;
    }
    t_plan += ms_since(t_p0);
  for (size_t bi = 0; bi < batches.size() && rc == FILO_OK; ++bi, ++n_batches) {
    const Batch& B = batches[bi];
    const int si = (int)(n_batches % NSLOT);
    filo_ctx::ScanSlot& sl = ctx->scan[si];
    { const auto t0 = now(); rc = retire(si); t_retire += ms_since(t0); }
    if (rc != FILO_OK) break;
    const int64_t nb = B.s1 - B.s0;
    {   // the slot is idle: its buffers may grow to this batch's needs
      int32_t rg = FILO_OK;
      if (!use_gather) rg = grow_pinned(ctx, sl.h_in, sl.h_in_cap, B.bytes + 64);
      else {
        rg = grow_pinned(ctx, sl.h_gch, sl.h_gch_cap, (size_t)(B.chunks + 1) * sizeof(GatherChunk));
        if (!rg) rg = grow_device(ctx, sl.d_gch, sl.d_gch_cap, (size_t)(B.chunks + 1) * sizeof(GatherChunk));
        if (!rg) rg = grow_pinned(ctx, sl.h_gs, sl.h_gs_cap, (size_t)(nb + 1) * sizeof(GatherSeries));
        if (!rg) rg = grow_device(ctx, sl.d_gs, sl.d_gs_cap, (size_t)(nb + 1) * sizeof(GatherSeries));
      }
      if (!rg) rg = grow_pinned(ctx, sl.h_off, sl.h_off_cap, (size_t)(nb + 1) * 8);
      if (!rg) rg = grow_device(ctx, sl.d_in, sl.d_in_cap, B.bytes + 64);
      if (!rg) rg = grow_device(ctx, sl.d_off, sl.d_off_cap, (size_t)(nb + 1) * 8);
      if (!rg) rg = grow_device(ctx, sl.d_out, sl.d_out_cap, (size_t)nb * (size_t)std::max(T, 1) * 8);
      if (rg) { rc = rg; break; }
    }
    if (trace_path) {
      TraceRow tr{nb, B.bytes, ms_since(t_begin), {nullptr, nullptr, nullptr, nullptr}};
      for (auto& e : tr.ev) cudaEventCreate(&e);
      if (!trace_t0) { cudaEventCreate(&trace_t0); cudaEventRecord(trace_t0, sl.stream); }
      cudaEventRecord(tr.ev[0], sl.stream);
      trace.push_back(tr);
    }
    const auto t_f0 = now();
    sl.h_off[0] = 0;
    for (int64_t j = 0; j < nb; ++j) sl.h_off[j + 1] = sl.h_off[j] + plan[(size_t)(B.s0 + j - c0)].rec_bytes;
    cudaError_t ce = cudaSuccess;
    if (use_gather) {
      // gather list: per series header + per chunk source addresses; the GPU copies the vectors out of the registered memory
      GatherSeries* gs = reinterpret_cast<GatherSeries*>(sl.h_gs); GatherChunk* gc = reinterpret_cast<GatherChunk*>(sl.h_gch);
      int64_t cb = 0;
      for (int64_t j = 0; j < nb; ++j) { const SeriesPlan& p = plan[(size_t)(B.s0 + j - c0)]; gs[j] = GatherSeries{p.rec_bytes, p.n_chunks, p.n_rows, p.flags, cb}; cb += p.n_chunks; }
      std::atomic<uint64_t> span_lo{~0ull}, span_hi{0};       // host span that holds the batch's vectors
      host_pool().run(nb, [&](int, int64_t b, int64_t e) {     // the walk's entries, compacted into the batch's list
        uint64_t lo = ~0ull, hi = 0;
        for (int64_t j = b; j < e; ++j) {
          const int64_t i = B.s0 + j; GatherChunk* o = gc + gs[j].first_chunk;
          const GatherChunk* src = gc_walk.data() + (chunk_base[(size_t)(i - c0)] - in.gc_base);
          for (uint32_t jj = 0; jj < gs[j].n_chunks; ++jj) {
            const GatherChunk g = src[jj];
            *o++ = g;
            lo = std::min(lo, std::min(g.ts_src, g.val_src));
            hi = std::max(hi, std::max(g.ts_src + (uint64_t)g.ts_bytes, g.val_src + (uint64_t)g.val_bytes));
          }
        }
        uint64_t cur = span_lo.load(); while (lo < cur && !span_lo.compare_exchange_weak(cur, lo)) {}
        cur = span_hi.load(); while (hi > cur && !span_hi.compare_exchange_weak(cur, hi)) {}
      });
      t_fill += ms_since(t_f0);
      // dense batch (the vectors fill most of one host span, e.g. consecutive series of a block): ONE copy-engine transfer of the span
      // at full PCIe rate, the gather then runs device to device; sparse batches keep the zero-copy reads of the registered memory
      int64_t rebase = 0;
      {
        static const bool no_span = [] { const char* e = std::getenv("FILO_SCAN_SPAN"); return e && e[0] == '0'; }();
        const uint64_t lo = span_lo.load() & ~(uint64_t)15, hi = span_hi.load();
        if (!no_span && hi > lo && (hi - lo) <= (uint64_t)B.bytes + (uint64_t)B.bytes / 2 + (1u << 20) && in_ranges(reinterpret_cast<const uint8_t*>((uintptr_t)lo), (size_t)(hi - lo))) {
          if (int32_t rcg = grow_device(ctx, sl.d_stage, sl.d_stage_cap, (size_t)(hi - lo) + 64)) return rcg;
          ce = cudaMemcpyAsync(sl.d_stage, reinterpret_cast<const void*>((uintptr_t)lo), (size_t)(hi - lo), cudaMemcpyHostToDevice, sl.stream);
          rebase = (int64_t)((uint64_t)(uintptr_t)sl.d_stage - lo);
        }
      }
      if (ce == cudaSuccess)
      ce = cudaMemcpyAsync(sl.d_gs, sl.h_gs, (size_t)nb * sizeof(GatherSeries), cudaMemcpyHostToDevice, sl.stream);
      if (ce == cudaSuccess) ce = cudaMemcpyAsync(sl.d_gch, sl.h_gch, (size_t)B.chunks * sizeof(GatherChunk), cudaMemcpyHostToDevice, sl.stream);
      if (ce == cudaSuccess) ce = cudaMemcpyAsync(sl.d_off, sl.h_off, (size_t)(nb + 1) * 8, cudaMemcpyHostToDevice, sl.stream);
      if (ce == cudaSuccess) {
        const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((nb + 7) / 8, (int64_t)ctx->sm_count * 8));
        gather_records_kernel<<<grid, 256, 0, sl.stream>>>(reinterpret_cast<const GatherSeries*>(sl.d_gs), reinterpret_cast<const GatherChunk*>(sl.d_gch),
                                                           sl.d_off, nb, sl.d_in, rebase);
        ce = cudaGetLastError();
      }
      if (ce == cudaSuccess) ce = cudaMemsetAsync(sl.d_in + B.bytes, 0, 64, sl.stream);
    } else {
      host_pool().run(nb, [&](int, int64_t b, int64_t e) {
        for (int64_t j = b; j < e; ++j) fill_record(in, B.s0 + j, plan[(size_t)(B.s0 + j - c0)], sl.h_in + sl.h_off[j]);
      });
      std::memset(sl.h_in + B.bytes, 0, 64);
      t_fill += ms_since(t_f0);
      ce = cudaMemcpyAsync(sl.d_in, sl.h_in, B.bytes + 64, cudaMemcpyHostToDevice, sl.stream);
      if (ce == cudaSuccess) ce = cudaMemcpyAsync(sl.d_off, sl.h_off, (size_t)(nb + 1) * 8, cudaMemcpyHostToDevice, sl.stream);
    }
    const auto t_e0 = now();
    if (ce != cudaSuccess) { rc = fail(ctx, FILO_ERR_CUDA, std::string("scan H2D: ") + cudaGetErrorString(ce)); break; }
    if (trace_path) cudaEventRecord(trace.back().ev[1], sl.stream);
    filo_table view;                                    // a table over the slot's buffers (not owned)
    view.n_series = nb; view.d_arena = sl.d_in; view.d_rec_off = sl.d_off; view.max_rows = tot.maxrows; view.max_chunks = tot.maxch;
    view.max_rec_bytes = tot.max_rec; view.any_nonconst_ts = !(tot.f_and & REC_ALL_TS_CONST); view.any_drop = (tot.f_or & REC_ANY_DROP) != 0;
    view.schema_flags = schema_flags; view.n_groups = 1; view.grouped = false;
    rc = query_device_impl(ctx, &view, fn, start, step, end, window, FILO_AGG_NONE, 0, 0, sl.d_out, nullptr, sl.stream, nullptr,
                           reinterpret_cast<AsyncSink*>(sl.h_sink));
    if (rc != FILO_OK) break;
    if (trace_path) cudaEventRecord(trace.back().ev[2], sl.stream);
    ce = cudaMemcpyAsync(out_values + (size_t)B.s0 * T, sl.d_out, (size_t)nb * T * 8, cudaMemcpyDeviceToHost, sl.stream);
    if (trace_path) cudaEventRecord(trace.back().ev[3], sl.stream);
    if (ce == cudaSuccess) ce = cudaEventRecord(sl.done, sl.stream);
    if (ce != cudaSuccess) { rc = fail(ctx, FILO_ERR_CUDA, std::string("scan D2H: ") + cudaGetErrorString(ce)); break; }
    fl[si].s0 = B.s0;
    t_enq += ms_since(t_e0);
    acc.h2d_bytes += (int64_t)B.bytes + (nb + 1) * 8 + (use_gather ? (int64_t)(nb * sizeof(GatherSeries) + B.chunks * sizeof(GatherChunk)) : 0); acc.d2h_bytes += nb * (int64_t)T * 8;
  }
  }
  for (int i = 0; i < NSLOT; ++i) { const int32_t r2 = retire(i); if (rc == FILO_OK) rc = r2; }
  if (rc != FILO_OK) { for (int i = 0; i < NSLOT; ++i) if (ctx->scan[i].stream) cudaStreamSynchronize(ctx->scan[i].stream); return rc; }
  if (trace_path) {
    if (FILE* f = std::fopen(trace_path, "w")) {
      std::fprintf(f, "batch,series,bytes,host_enqueue_ms,start_ms,h2d_done_ms,kernels_done_ms,d2h_done_ms\n");
      for (size_t i = 0; i < trace.size(); ++i) {
        float t[4] = {0, 0, 0, 0};
        for (int j = 0; j < 4; ++j) cudaEventElapsedTime(&t[j], trace_t0, trace[i].ev[j]);
        std::fprintf(f, "%zu,%lld,%zu,%.3f,%.3f,%.3f,%.3f,%.3f\n", i, (long long)trace[i].nb, trace[i].bytes, trace[i].host_ms, t[0], t[1], t[2], t[3]);
      }
      std::fclose(f);
    }
    for (auto& r : trace) for (auto& e : r.ev) cudaEventDestroy(e);
    if (trace_t0) cudaEventDestroy(trace_t0);
  }
  if (timing) fprintf(stderr, "[filo] scan_series: %lld series, %zu batches, total %.1f ms: plan %.1f, fill %.1f, enqueue %.1f, slot waits %.1f\n",
                      (long long)n_series, n_batches, ms_since(t_begin), t_plan, t_fill, t_enq, t_retire);
  if (stats) *stats = acc;
  return FILO_OK;
}
extern "C" int32_t filo_scan_series(filo_ctx* ctx, int64_t n_series, const int32_t* n_chunks, const uint64_t* addrs,
                                    int32_t ts_col, int32_t val_col, int32_t schema_flags,
                                    int32_t fn, int64_t start, int64_t step, int64_t end, int64_t window,
                                    double* out_values, filo_stats* stats) {
  try { return filo_scan_series_impl(ctx, n_series, n_chunks, addrs, ts_col, val_col, schema_flags, fn, start, step, end, window, out_values, stats); }
  catch (const std::bad_alloc&) { return fail(ctx, FILO_ERR_OOM, "filo_scan_series: host allocation failed"); }
  catch (const std::exception& e) { return fail(ctx, FILO_ERR_INVALID_ARG, std::string("filo_scan_series: ") + e.what()); }
}


// ------------------------------------------------------------------------------------------------------------------
// filo_query_hist: PeriodicSamplesMapper over a histogram column (+ HistSumRowAggregator, + histogram_quantile)
// ------------------------------------------------------------------------------------------------------------------
// One orchestration for both entry points.  filo_query_hist_device (host_out false): out_values / out_quantile are device buffers, the call
// synchronises only when stats != NULL.  filo_query_hist (host_out true): they are host buffers; the results go to device temporaries
// allocated once every argument has been checked, and their copies to the host are enqueued before the one synchronisation.
static int32_t hist_query_impl(filo_ctx* ctx, const filo_table* t, int32_t fn, int64_t start, int64_t step, int64_t end, int64_t window,
                               int32_t agg, double quantile, double* out_values, double* out_quantile, void* cuda_stream, filo_stats* stats, bool host_out) {
  if (!ctx || !t || (!out_values && !out_quantile)) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_query_hist: null argument");
  if (!t->hist) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_query_hist: not a histogram table");
  if (agg != FILO_AGG_NONE && agg != FILO_AGG_SUM) return fail(ctx, FILO_ERR_UNSUPPORTED, "histogram aggregates: sum only");
  if (!(fn == FILO_FN_RATE || fn == FILO_FN_INCREASE || fn == FILO_FN_SUM_OVER_TIME || fn == FILO_FN_LAST))
    return fail(ctx, FILO_ERR_UNSUPPORTED, "histogram range functions on the device path: rate, increase, sum_over_time, last");
  // PeriodicSamplesMapper.scala:45-49, 67-68
  if (start > end) return fail(ctx, FILO_ERR_INVALID_ARG, "start should be <= end");
  if (!(start == end || step > 0)) return fail(ctx, FILO_ERR_INVALID_ARG, "step should be > 0 for range query");
  if (start < end && step < ctx->cfg.min_step_ms) return fail(ctx, FILO_ERR_BAD_QUERY, "step should be at least min-step");
  const bool last = fn == FILO_FN_LAST;
  if (window <= 0) { if (last) window = 5 * 60 * 1000 + 1; else return fail(ctx, FILO_ERR_INVALID_ARG, "Need positive window lengths to apply range function"); }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  { const int32_t prc = poll_async_errors(ctx, false); if (prc != FILO_OK) return prc; }      // an earlier stats == NULL query failed on the device
  cudaStream_t s = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
  const int64_t adjustedStep = step > 0 ? step : step + 1;
  QueryParams q{};
  q.start = start; q.step = adjustedStep; q.end = end; q.window = window; q.T = filo_num_windows(start, adjustedStep, end);
  q.fn = fn; q.cumulative = (t->schema_flags & FILO_SCHEMA_CUMULATIVE) ? 1 : 0; q.inclusive = ctx->cfg.inclusive_range ? 1 : 0;
  const int nb = t->hist_nb, T = q.T;
  const bool fused = agg == FILO_AGG_SUM;
  const bool pq = !fused && out_quantile;                // per-series histogram_quantile
  const size_t smem = hist_smem_bytes(t->max_rows, nb, T, fused || pq, t->max_rec_bytes);
  // second kernel: rate / increase over cumulative histograms and last over SectDelta vectors (its table parser takes no other vector),
  // fused or per series, when its working set leaves room for two CTAs per SM
  const size_t smem2 = hist2_smem_bytes(t->max_rows, nb, t->max_rec_bytes);
  // Per series it takes the quantile and last; rate / increase bucket rows alone stay on the first kernel, whose (window, bucket) threads
  // store [S][T][nb] contiguously (H100: 20.6 ms against 27.7 ms for 100 k series x 481 windows x 20 buckets, DESIGN §7).
  const bool v2 = hist_v2_enabled() && ((q.cumulative && (fn == FILO_FN_RATE || fn == FILO_FN_INCREASE)) || (last && !t->hist_simple)) && T <= 32 * 512 && nb <= 64 &&
                  smem2 + 1024 <= std::min<size_t>(ctx->max_smem_optin, 227 * 1024) && (fused || pq || last);
  // the first kernel's working set (its per-series quantile and the fused sum keep a [T][nb] block in shared memory); a per-series query on
  // the second kernel does not depend on it.  The fused sum keeps its limit whichever kernel runs it.
  if (!(v2 && !fused) && smem + 2048 > std::min<size_t>(ctx->max_smem_optin, 227 * 1024))
    return fail(ctx, FILO_ERR_UNSUPPORTED, "histogram query does not fit the device working set (rows x buckets or windows x buckets too large)");
  Temp tmp(s);
  int* d_err = nullptr; unsigned long long* d_counters = nullptr;
  CUDA_TRY(ctx, tmp.alloc((void**)&d_err, 16)); CUDA_TRY(ctx, tmp.alloc((void**)&d_counters, 16));
  CUDA_TRY(ctx, cudaMemsetAsync(d_err, 0, 16, s)); CUDA_TRY(ctx, cudaMemsetAsync(d_counters, 0, 16, s));
  EventPair evp;
  if (stats) { CUDA_TRY(ctx, cudaEventCreate(&evp.e0)); CUDA_TRY(ctx, cudaEventCreate(&evp.e1)); }
  cudaEvent_t& e0 = evp.e0; cudaEvent_t& e1 = evp.e1;
  const int64_t work = fused ? t->n_items : t->n_series;
  ScanLaunch L{t->d_arena, t->d_rec_off, t->n_series, q, nullptr, 0, 0, d_counters, d_err, 1, s};
  const int ctas_per_sm = (int)std::max<size_t>(1, (size_t)(228 * 1024) / (smem + 2048));
  L.grid = (int)std::max<int64_t>(1, std::min<int64_t>(work, (int64_t)ctx->sm_count * ctas_per_sm));
  const int64_t rows = fused ? t->n_groups : t->n_series;
  double *d_out = out_values, *d_q = out_quantile, *pval = nullptr; uint8_t* pany = nullptr;
  if (host_out) {
    if (out_values) CUDA_TRY(ctx, tmp.alloc((void**)&d_out, (size_t)rows * T * nb * 8));
    if (out_quantile) CUDA_TRY(ctx, tmp.alloc((void**)&d_q, (size_t)rows * T * 8));
  }
  if (stats) CUDA_TRY(ctx, cudaEventRecord(e0, s));
  if (v2 && !fused) {
    const int cps = (int)std::max<size_t>(1, std::min<size_t>(2, (size_t)(228 * 1024) / (smem2 + 1024)));
    L.grid = (int)std::max<int64_t>(1, std::min<int64_t>(hist2_series_items(t->n_series), (int64_t)ctx->sm_count * cps));
    double* scratch = nullptr;                          // quantile only: each CTA's window columns, grid * T * nb doubles
    if (!out_values) CUDA_TRY(ctx, tmp.alloc((void**)&scratch, (size_t)L.grid * T * nb * 8));
    CUDA_TRY(ctx, launch_hist_scan2_series(L, nb, t->max_rows, t->max_rec_bytes, d_out, d_q, scratch, t->d_hist_tops, quantile, t->hist_exp ? 1 : 0));
  } else if (v2) {
    const int cps = (int)std::max<size_t>(1, std::min<size_t>(2, (size_t)(228 * 1024) / (smem2 + 1024)));
    L.grid = (int)std::max<int64_t>(1, std::min<int64_t>(t->n_items, (int64_t)ctx->sm_count * cps));
    CUDA_TRY(ctx, tmp.alloc((void**)&pval, (size_t)t->n_items * T * nb * 8));
    CUDA_TRY(ctx, tmp.alloc((void**)&pany, (size_t)t->n_items * T + 16));
    CUDA_TRY(ctx, launch_hist_scan2(L, nb, t->max_rows, t->max_rec_bytes, t->grouped ? t->d_order : nullptr, t->d_item_begin, t->n_items, pval, pany));
    CUDA_TRY(ctx, launch_hist_merge2(pval, pany, t->d_gis, t->n_groups, T, nb, t->hist_exp ? 1 : 0, t->d_hist_tops, out_quantile ? quantile : std::nan(""), d_out, d_q, s));
  } else if (fused) {
    CUDA_TRY(ctx, tmp.alloc((void**)&pval, (size_t)t->n_items * T * nb * 8));
    CUDA_TRY(ctx, tmp.alloc((void**)&pany, (size_t)t->n_items * T + 16));
    CUDA_TRY(ctx, launch_hist_scan(L, nb, t->max_rows, t->max_rec_bytes, t->grouped ? t->d_order : nullptr, t->d_item_begin, t->n_items, 1, nullptr, pval, pany));
    CUDA_TRY(ctx, launch_hist_merge(pval, pany, t->d_gis, t->n_groups, T, nb, t->hist_exp ? 1 : 0, t->d_hist_tops, out_quantile ? quantile : std::nan(""), d_out, d_q, s));
  } else {
    CUDA_TRY(ctx, launch_hist_scan(L, nb, t->max_rows, t->max_rec_bytes, nullptr, nullptr, 0, 0, d_out, nullptr, nullptr, t->d_hist_tops, quantile, t->hist_exp ? 1 : 0, d_q));
  }
  if (!stats) return push_async_error(ctx, d_err, s);
  CUDA_TRY(ctx, cudaEventRecord(e1, s));
  int herr[4]; unsigned long long hc[2];
  CUDA_TRY(ctx, cudaMemcpyAsync(herr, d_err, 16, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(ctx, cudaMemcpyAsync(hc, d_counters, 16, cudaMemcpyDeviceToHost, s));
  const size_t d2h = host_out ? (out_values ? (size_t)rows * T * nb * 8 : 0) + (out_quantile ? (size_t)rows * T * 8 : 0) : 0;
  if (host_out && out_values) CUDA_TRY(ctx, cudaMemcpyAsync(out_values, d_out, (size_t)rows * T * nb * 8, cudaMemcpyDeviceToHost, s));
  if (host_out && out_quantile) CUDA_TRY(ctx, cudaMemcpyAsync(out_quantile, d_q, (size_t)rows * T * 8, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(ctx, cudaStreamSynchronize(s));
  float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
  stats->kernel_ns = (int64_t)((double)ms * 1e6); stats->samples_scanned = (int64_t)hc[0]; stats->bytes_scanned = (int64_t)hc[1];
  stats->kernel_launches = fused ? 2 : 1; stats->h2d_bytes = 0; stats->d2h_bytes = (int64_t)d2h;
  if (herr[0]) return report_device_error(ctx, herr, 0);
  return FILO_OK;
}
extern "C" int32_t filo_query_hist_device(filo_ctx* ctx, const filo_table* t, int32_t fn, int64_t start, int64_t step, int64_t end, int64_t window,
                                          int32_t agg, double quantile, void* d_out_values, void* d_out_quantile, void* cuda_stream, filo_stats* stats) {
  try { return hist_query_impl(ctx, t, fn, start, step, end, window, agg, quantile, (double*)d_out_values, (double*)d_out_quantile, cuda_stream, stats, false); }
  catch (const std::bad_alloc&) { return fail(ctx, FILO_ERR_OOM, "filo_query_hist: host allocation failed"); }
  catch (const std::exception& e) { return fail(ctx, FILO_ERR_INVALID_ARG, std::string("filo_query_hist: ") + e.what()); }
}
extern "C" int32_t filo_query_hist(filo_ctx* ctx, const filo_table* t, int32_t fn, int64_t start, int64_t step, int64_t end, int64_t window,
                                   int32_t agg, double quantile, double* out_values, double* out_quantile, filo_stats* stats) {
  filo_stats st{};         // the host form always synchronises
  try { const int32_t rc = hist_query_impl(ctx, t, fn, start, step, end, window, agg, quantile, out_values, out_quantile, nullptr, &st, true);
        if (stats) *stats = st;
        return rc; }
  catch (const std::bad_alloc&) { return fail(ctx, FILO_ERR_OOM, "filo_query_hist: host allocation failed"); }
  catch (const std::exception& e) { return fail(ctx, FILO_ERR_INVALID_ARG, std::string("filo_query_hist: ") + e.what()); }
}

extern "C" int32_t filo_merge_hist_partials(filo_ctx* ctx, const filo_table* t, int32_t n_parts, int32_t n_windows, double quantile,
                                            const void* d_parts, void* d_out_values, void* d_out_quantile, void* cuda_stream) {
  if (!ctx || !t || !d_parts) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_merge_hist_partials: null argument");
  if (!t->hist) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_merge_hist_partials: not a histogram table");
  if (n_parts < 1 || n_windows < 1) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_merge_hist_partials: n_parts and n_windows must be >= 1");
  double* d_q = quantile == quantile ? (double*)d_out_quantile : nullptr;              // quantile NaN: the values alone
  if (!d_out_values && !d_q) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_merge_hist_partials: no output (values NULL, and quantile NaN or its output NULL)");
  if (t->hist_nb > 64) return fail(ctx, FILO_ERR_UNSUPPORTED, "filo_merge_hist_partials: more than 64 buckets");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  { const int32_t prc = poll_async_errors(ctx, false); if (prc != FILO_OK) return prc; }      // e.g. the query that produced a part failed
  cudaStream_t s = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
  CUDA_TRY(ctx, launch_hist_merge_parts((const double*)d_parts, n_parts, (int64_t)t->n_groups * n_windows, t->hist_nb, t->hist_exp ? 1 : 0, t->d_hist_tops,
                                        quantile, (double*)d_out_values, d_q, s));
  return FILO_OK;
}

extern "C" int32_t filo_merge_topk_partials(filo_ctx* ctx, int32_t agg, int32_t k, int32_t n_parts, int32_t n_groups, int32_t n_windows,
                                            const void* d_part_values, const void* d_part_ids, void* d_out_values, void* d_out_ids, void* cuda_stream) {
  if (!ctx || !d_part_values || !d_part_ids || !d_out_values || !d_out_ids) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_merge_topk_partials: null argument");
  if (agg != FILO_AGG_TOPK && agg != FILO_AGG_BOTTOMK) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_merge_topk_partials: the operator must be topk or bottomk");
  if (k < 1 || k > FILO_MAX_TOPK) return fail(ctx, FILO_ERR_INVALID_ARG, "topk/bottomk k must be in [1, 32]");
  if (n_parts < 1 || n_groups < 1 || n_windows < 1) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_merge_topk_partials: n_parts, n_groups and n_windows must be >= 1");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  { const int32_t prc = poll_async_errors(ctx, false); if (prc != FILO_OK) return prc; }      // e.g. the query that produced a part failed
  cudaStream_t s = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
  CUDA_TRY(ctx, launch_topk_merge_parts((const double*)d_part_values, (const int64_t*)d_part_ids, n_parts, (int64_t)n_groups * n_windows, k,
                                        agg == FILO_AGG_BOTTOMK ? 1 : 0, (double*)d_out_values, (int64_t*)d_out_ids, s));
  return FILO_OK;
}

extern "C" int32_t filo_present_partials(filo_ctx* ctx, int32_t agg, int64_t n, void* d_values, void* d_counts, void* d_out, void* cuda_stream) {
  if (!ctx || !d_values || !d_counts || !d_out || n < 0) return fail(ctx, FILO_ERR_INVALID_ARG, "filo_present_partials: bad argument");
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t s = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
  if (n > 0) CUDA_TRY(ctx, launch_present(agg, n, (const double*)d_values, (const int64_t*)d_counts, (double*)d_out, s));
  return FILO_OK;
}
