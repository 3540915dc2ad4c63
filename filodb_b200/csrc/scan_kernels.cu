// sm_90a kernels: fused chunk decode + windowed range function (+ across-series aggregate), one warp per series.
// See scan_device.cuh for the per-window semantics and DESIGN.md for the layout / roofline discussion.
#include <cuda_runtime.h>
#include <stdint.h>
#define FILO_DEV_ERR_TS_WIRE 1
#define FILO_DEV_ERR_VAL_WIRE 2
#define FILO_DEV_ERR_EMPTY 3
#define FILO_DEV_ERR_SCRATCH 4
#include "scan_device.cuh"
#include "kernels.h"
#include "scan_fast.cuh"
#include "scan_tile.cuh"
#include "scan_wp.cuh"
#include "scan_wp_ctr.cuh"

namespace filo {

__device__ __forceinline__ void report_error(int* d_err, int code, int64_t series) {
  if (atomicCAS(&d_err[0], 0, code) == 0) { d_err[1] = (int)(series & 0x7fffffff); d_err[2] = (int)(series >> 31); }
}

// Resolve all chunks of one series that intersect [start - window, end] (TimeSeriesPartition.infos(start,end),
// TimeSeriesPartition.scala:365-366 + ChunkSetInfo.intersection :99-108).  Returns number of resolved chunks (D[0..n)).
__device__ __forceinline__ int resolve_series(const uint8_t* rec, const QueryParams& q, uint8_t* scratch, uint32_t scratch_bytes,
                                              bool need_corrected, int lane, int& err, int64_t& rows_scanned, int64_t& bytes_scanned) {
  const RecordHeader* h = reinterpret_cast<const RecordHeader*>(rec);
  const ChunkEntry* E = reinterpret_cast<const ChunkEntry*>(rec + sizeof(RecordHeader));
  const int nch = (int)h->n_chunks;
  const int64_t t1 = q.start - q.window, t2 = q.end;
  // chunks are time ordered: [cLo, cHi) = those with end_time >= t1 and start_time <= t2
  int cLo = 0; while (cLo < nch && E[cLo].end_time < t1) ++cLo;
  int cHi = cLo; while (cHi < nch && E[cHi].start_time <= t2) ++cHi;
  if (t1 > t2) cHi = cLo;
  const int n = cHi - cLo;
  err = 0;
  if (n <= 0) return 0;
  // scratch need: descriptors + decoded rows (host sized scratch_bytes for the worst series; double-check)
  ChunkDesc* D = reinterpret_cast<ChunkDesc*>(scratch);
  ScratchCursor sc; sc.p = scratch + align_up((uint32_t)n * (uint32_t)sizeof(ChunkDesc), 16);
  uint32_t need = (uint32_t)(sc.p - scratch) + (uint32_t)h->n_rows * 8u * (need_corrected ? 3u : 2u);
  if (need > scratch_bytes) { err = FILO_DEV_ERR_SCRATCH; return 0; }
  for (int c = 0; c < n; ++c) {
    int e = resolve_chunk(rec, &E[cLo + c], &D[c], sc, need_corrected, lane, false, q.long_values != 0);
    if (e) { err = e; return 0; }
  }
  // CountingChunkInfoIterator (ChunkSetInfo.scala:336-380): chunks pulled by the window iterator
  if (lane == 0) {
    const int64_t lastEnd = q.start + (int64_t)(q.T - 1) * q.step;
    int f = 0; while (f < n - 1 && D[f].end_time < lastEnd) ++f;
    for (int c = 0; c <= f; ++c) {
      rows_scanned += D[c].num_rows;
      bytes_scanned += (int64_t)ld32(rec + E[cLo + c].ts_off) + 4 + (int64_t)ld32(rec + E[cLo + c].val_off) + 4;
    }
  }
  return n;
}

// ---------------------------------------------------------------------------------------------------------------
// Kernel 1: PeriodicSamplesMapper without aggregate — out[series * T + k]
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SCAN_WARPS * 32)
scan_series_kernel(const uint8_t* __restrict__ arena, const int64_t* __restrict__ rec_off, int64_t n_series,
                   QueryParams q, double* __restrict__ out,
                   uint8_t* gscratch, uint32_t scratch_bytes, int use_smem,
                   unsigned long long* d_counters, int* d_err) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t gw = (int64_t)blockIdx.x * SCAN_WARPS + warp, nw = (int64_t)gridDim.x * SCAN_WARPS;
  uint8_t* scratch = use_smem ? smem + (size_t)warp * scratch_bytes : gscratch + (size_t)gw * scratch_bytes;
  const int fn = q.fn;
  const bool need_corrected = ((fn == FN_RATE || fn == FN_INCREASE) && q.cumulative);
  int64_t rows = 0, bytes = 0;
  for (int64_t i = gw; i < n_series; i += nw) {
    const uint8_t* rec = arena + rec_off[i];
    int err;
    const int n = resolve_series(rec, q, scratch, scratch_bytes, need_corrected, lane, err, rows, bytes);
    if (err) { if (lane == 0) report_error(d_err, err, i); continue; }
    const ChunkDesc* D = reinterpret_cast<const ChunkDesc*>(scratch);
    double* o = out + (size_t)i * q.T;
    for (int k = lane; k < q.T; k += 32) o[k] = eval_window(D, 0, n, q, k);
    __syncwarp();
  }
  if (lane == 0 && (rows | bytes)) { atomicAdd(&d_counters[0], (unsigned long long)rows); atomicAdd(&d_counters[1], (unsigned long long)bytes); }
}

// ---------------------------------------------------------------------------------------------------------------
// Kernel 2: fused PeriodicSamplesMapper + AggregateMapReduce map/reduce phase.
// Work item = run of <= SEG consecutive series (in group-sorted order) of ONE group.  The warp folds the item's series
// into per-window accumulators (shared memory, or global scratch when T is large) and writes one partial row:
//   pval[item*T + k] = Σ non-NaN (SUM/AVG/COUNT) | min | max ;  pcnt[item*T + k] = number of non-NaN inputs
//   STDDEV/STDVAR (moments): pval[item*T + k] = Σv, pval[(n_items + item)*T + k] = Σv² (accumulators [T] Σv, [T] Σv², [T] counts)
// A second kernel folds the partial rows of each group in item order (deterministic, atomics-free).
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SCAN_WARPS * 32)
scan_agg_kernel(const uint8_t* __restrict__ arena, const int64_t* __restrict__ rec_off, const int32_t* __restrict__ order,
                const int64_t* __restrict__ item_begin, int64_t n_items,
                QueryParams q, int agg_op, double* __restrict__ pval, uint32_t* __restrict__ pcnt,
                uint8_t* gscratch, uint32_t scratch_bytes, uint32_t acc_bytes, int use_smem,
                unsigned long long* d_counters, int* d_err) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t gw = (int64_t)blockIdx.x * SCAN_WARPS + warp, nw = (int64_t)gridDim.x * SCAN_WARPS;
  const uint32_t per_warp = scratch_bytes + acc_bytes;
  uint8_t* base = use_smem ? smem + (size_t)warp * per_warp : gscratch + (size_t)gw * per_warp;
  const bool mom = agg_moments(agg_op);
  double* acc = reinterpret_cast<double*>(base);
  double* acc2 = acc + q.T;                                  // moments only
  uint32_t* cnt = reinterpret_cast<uint32_t*>(base + (size_t)q.T * (mom ? 16 : 8));
  uint8_t* scratch = base + acc_bytes;
  const int fn = q.fn;
  const bool need_corrected = ((fn == FN_RATE || fn == FN_INCREASE) && q.cumulative);
  const double ident = agg_op == AGG_MIN ? __longlong_as_double(0x7ff0000000000000LL)
                     : agg_op == AGG_MAX ? __longlong_as_double(0xfff0000000000000LL) : 0.0;
  int64_t rows = 0, bytes = 0;
  for (int64_t it = gw; it < n_items; it += nw) {
    for (int k = lane; k < q.T; k += 32) { acc[k] = ident; cnt[k] = 0; if (mom) acc2[k] = 0.0; }
    const int64_t b = item_begin[it], e = item_begin[it + 1];
    for (int64_t pos = b; pos < e; ++pos) {
      const int64_t i = order ? order[pos] : pos;
      const uint8_t* rec = arena + rec_off[i];
      int err;
      const int n = resolve_series(rec, q, scratch, scratch_bytes, need_corrected, lane, err, rows, bytes);
      if (err) { if (lane == 0) report_error(d_err, err, i); continue; }
      const ChunkDesc* D = reinterpret_cast<const ChunkDesc*>(scratch);
      for (int k = lane; k < q.T; k += 32) {
        const double v = eval_window(D, 0, n, q, k);
        if (v == v) {                                       // RowAggregators skip NaN (SumRowAggregator.scala:22-29 ...)
          double a = acc[k];
          // min/maxIgnoreNaN(acc, v) (QueryUtils.scala:111-123): of two equal values (+0.0 / -0.0) the later one is kept
          if (agg_op == AGG_MIN) a = a < v ? a : v;
          else if (agg_op == AGG_MAX) a = a > v ? a : v;
          else if (agg_op == AGG_COUNT) a = a;             // count only
          else a += v;
          acc[k] = a; cnt[k] += 1;
          if (mom) acc2[k] += v * v;
        }
      }
      __syncwarp();
    }
    double* pv = pval + (size_t)it * q.T; uint32_t* pc = pcnt + (size_t)it * q.T;
    for (int k = lane; k < q.T; k += 32) { pv[k] = acc[k]; pc[k] = cnt[k]; }
    if (mom) { double* pv2 = pval + (size_t)(n_items + it) * q.T; for (int k = lane; k < q.T; k += 32) pv2[k] = acc2[k]; }
    __syncwarp();
  }
  if (lane == 0 && (rows | bytes)) { atomicAdd(&d_counters[0], (unsigned long long)rows); atomicAdd(&d_counters[1], (unsigned long long)bytes); }
}

// Fold the partial rows of each group (items [gis[g], gis[g+1])) in item order.  Block = (32 windows) x (8 item lanes);
// thread (kk, j) folds items j, j+8, ... sequentially, then the 8 lanes are folded in fixed order -> deterministic.
// MIN / MAX fold as min/maxIgnoreNaN(acc, v) (QueryUtils.scala:111-123): of equal values (+0.0 / -0.0) the later one is kept.  That
// rule is associative, so the tree equals one sequential fold over the items in the order 0, 8, 16, ..., 1, 9, 17, ..., 7, 15, ...,
// with each item's series folded in group order by the scan kernel.
// partial_out: values/counts in mergeable form; otherwise presented (NaN when count == 0; Σ/n for AVG; n for COUNT).
// EXT = MERGE_MOMENTS (STDDEV/STDVAR): the Σv² rows follow the Σv rows (pval + n_items * T, n_items = gis[n_groups]) and are folded
// by the same tree; their mergeable form is [2][n_groups][T].  EXT = MERGE_GROUP: the count partial, presented as 1.0 / NaN.
// RowAggregator.present of one merged cell: s = Σ (or min / max), s2 = Σv² (moments), c = non-NaN inputs
__device__ __forceinline__ double present_cell(int agg_op, double s, double s2, int64_t c) {
  const double NaNv = __longlong_as_double(0x7ff8000000000000LL);
  if (c == 0) return NaNv;
  if (agg_op == AGG_AVG) return s / (double)c;
  if (agg_op == AGG_COUNT) return (double)c;
  if (agg_op == AGG_GROUP) return 1.0;                      // GroupRowAggregator.scala:23-29
  if (agg_moments(agg_op)) {
    // sumSquare/count - mean^2 (StdvarRowAggregator.scala:52-72); stddev = Math.pow(stdvar, 0.5) (StddevRowAggregator.scala:51):
    // sqrt for x >= +0, NaN below zero, with pow(-0.0, 0.5) = +0.0 and pow(-Inf, 0.5) = +Inf
    const double m = s / (double)c;
    const double var = s2 / (double)c - m * m;
    if (agg_op == AGG_STDVAR) return var;
    if (var < 0.0) return var == -__longlong_as_double(0x7ff0000000000000LL) ? __longlong_as_double(0x7ff0000000000000LL) : NaNv;
    return var == 0.0 ? 0.0 : sqrt(var);
  }
  return s;
}

enum { MERGE_PLAIN = 0, MERGE_MOMENTS = 1, MERGE_GROUP = 2 };
template <int EXT = MERGE_PLAIN>
__global__ void __launch_bounds__(256)
merge_partials_kernel(const double* __restrict__ pval, const uint32_t* __restrict__ pcnt, const int64_t* __restrict__ gis,
                      int n_groups, int T, int agg_op, int partial_out, double* __restrict__ out_val, int64_t* __restrict__ out_cnt) {
  __shared__ double sv[8][33]; __shared__ unsigned long long sc[8][33];
  const int kk = threadIdx.x & 31, j = threadIdx.x >> 5;
  const int ktiles = (T + 31) / 32;
  const int g = blockIdx.x / ktiles, k = (blockIdx.x % ktiles) * 32 + kk;
  if (g >= n_groups) return;
  const double ident = agg_op == AGG_MIN ? __longlong_as_double(0x7ff0000000000000LL)
                     : agg_op == AGG_MAX ? __longlong_as_double(0xfff0000000000000LL) : 0.0;
  double a = ident; unsigned long long c = 0;
  constexpr bool MOM = EXT == MERGE_MOMENTS;
  MomOnly<MOM, double> a2;
  if constexpr (MOM) a2.v = 0.0;
  if (k < T) {
    for (int64_t it = gis[g] + j; it < gis[g + 1]; it += 8) {
      const double v = pval[(size_t)it * T + k]; const uint32_t n = pcnt[(size_t)it * T + k];
      if (n) {
        if (agg_op == AGG_MIN) a = a < v ? a : v; else if (agg_op == AGG_MAX) a = a > v ? a : v; else a += v;
        if constexpr (MOM) a2.v += pval[(size_t)(gis[n_groups] + it) * T + k];
        c += n;
      }
    }
  }
  sv[j][kk] = a; sc[j][kk] = c;
  if constexpr (MOM) { __shared__ double sv2[8][33]; sv2[j][kk] = a2.v; __syncthreads(); if (j == 0 && k < T) for (int jj = 1; jj < 8; ++jj) if (sc[jj][kk]) a2.v += sv2[jj][kk]; }
  __syncthreads();
  if (j == 0 && k < T) {
    for (int jj = 1; jj < 8; ++jj) {
      const double v = sv[jj][kk]; const unsigned long long n = sc[jj][kk];
      if (n) { if (agg_op == AGG_MIN) a = a < v ? a : v; else if (agg_op == AGG_MAX) a = a > v ? a : v; else a += v; c += n; }
    }
    const size_t o = (size_t)g * T + k;
    if constexpr (EXT != MERGE_PLAIN) {
      double s2 = 0.0;
      if constexpr (MOM) s2 = a2.v;
      if (partial_out) { out_val[o] = a; if constexpr (MOM) out_val[(size_t)n_groups * T + o] = s2; if (out_cnt) out_cnt[o] = (int64_t)c; }
      else { out_val[o] = present_cell(agg_op, a, s2, (int64_t)c); if (out_cnt) out_cnt[o] = (int64_t)c; }
    } else if (partial_out) { out_val[o] = a; if (out_cnt) out_cnt[o] = (int64_t)c; }
    else {
      const double NaNv = __longlong_as_double(0x7ff8000000000000LL);
      double r;
      if (c == 0) r = NaNv;
      else if (agg_op == AGG_AVG) r = a / (double)c;
      else if (agg_op == AGG_COUNT) r = (double)c;
      else r = a;
      out_val[o] = r; if (out_cnt) out_cnt[o] = (int64_t)c;
    }
  }
}

// present after a cross-GPU merge of partials (STDDEV/STDVAR: the Σv² block follows the n cells of Σv)
__global__ void present_kernel(int agg_op, int64_t n, const double* __restrict__ vals, const int64_t* __restrict__ cnts, double* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = present_cell(agg_op, vals[i], agg_moments(agg_op) ? vals[n + i] : 0.0, cnts[i]);
}

// topk / bottomk over per-series results (TopBottomKRowAggregator.scala:84-95): one thread per (group, window) scans the
// group's series in sorted (arrival) order keeping the k best non-NaN values; ties keep the earlier series.
// Output row in the reference's dequeue order: topk ascending, bottomk descending; empty slots = ±Double.MaxValue, id -1.
__global__ void topk_kernel(const double* __restrict__ per_series, const int32_t* __restrict__ order, const int64_t* __restrict__ group_start,
                            int n_groups, int T, int kk, int bottom, double* __restrict__ out_val, int64_t* __restrict__ out_id) {
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= (int64_t)n_groups * T) return;
  const int g = (int)(tid / T), t = (int)(tid % T);
  double bv[FILO_MAX_TOPK]; int64_t bi[FILO_MAX_TOPK]; int n = 0;    // sorted best-first
  for (int64_t pos = group_start[g]; pos < group_start[g + 1]; ++pos) {
    const int64_t s = order ? order[pos] : pos;
    const double v = per_series[(size_t)s * T + t];
    if (v != v) continue;
    // insertion position: after all elements at least as good (ties keep earlier arrival ahead)
    int p = n;
    while (p > 0 && (bottom ? (v < bv[p - 1]) : (v > bv[p - 1]))) --p;
    if (p >= kk) continue;
    const int last = n < kk ? n : kk - 1;
    for (int m = last; m > p; --m) { bv[m] = bv[m - 1]; bi[m] = bi[m - 1]; }
    bv[p] = v; bi[p] = s; if (n < kk) ++n;
  }
  double* ov = out_val + (size_t)tid * kk; int64_t* oi = out_id + (size_t)tid * kk;
  for (int m = 0; m < kk; ++m) {
    if (m < n) { ov[m] = bv[n - 1 - m]; oi[m] = bi[n - 1 - m]; }          // worst of the kept first (dequeue order)
    else { ov[m] = bottom ? 1.7976931348623157e308 : -1.7976931348623157e308; oi[m] = -1; }
  }
}

// topk / bottomk across GPUs (ReduceAggregateExec over TopBottomKRowAggregator rows): n_parts outputs of topk_kernel, ids mapped to
// global series ordinals, [n_parts][n_cells][k] in rank order.  (value, ordinal) is a strict total order: among equal values (==, so
// +0.0 ties -0.0) the smaller ordinal is better.  An empty slot is one whose id is -1 (±DBL_MAX padding is also a real value); a NaN value,
// which topk_kernel never writes with an id, is skipped like one, so that the order stays total.
__device__ __forceinline__ bool topk_better(double a, int64_t ai, double b, int64_t bi, int bottom) {
  if (bi < 0) return ai >= 0;                                         // any candidate beats an empty slot
  if (ai < 0) return false;
  if (a != b) return bottom ? a < b : a > b;
  return ai < bi;
}
// folds slot (v, id) into (cv, cid) when it lies strictly below the bound (tv, tid) (tid < 0: no bound)
__device__ __forceinline__ void topk_fold_below(double v, int64_t id, double tv, int64_t tid, int bottom, double& cv, int64_t& cid) {
  if (id < 0 || v != v) return;
  if (tid >= 0 && !topk_better(tv, tid, v, id, bottom)) return;      // emitted already
  if (topk_better(v, id, cv, cid, bottom)) { cv = v; cid = id; }
}
// warp-wide arg-best: every lane ends with the best (v, id) of the warp, a non-empty one whenever any lane holds one
__device__ __forceinline__ void topk_warp_best(double& v, int64_t& id, int bottom) {
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int64_t oi = __shfl_xor_sync(0xffffffffu, id, o);
    if (topk_better(ov, oi, v, id, bottom)) { v = ov; id = oi; }
  }
}
// One warp per (group, window) cell: a W-way merge.  Lane l holds the best candidate of parts l, l + 32, ... not emitted yet; k rounds
// of a warp-wide arg-best emit the candidates best first.  The elements emitted are exactly those at or above the last winner, so a
// lane's next candidate is the best slot of its parts strictly below the winner: after each round the whole warp reads the winning
// lane's parts (lane j reads slot j) and reduces them.  Nothing depends on the order of the slots inside a part, so the result is the k
// best of all non-empty slots whatever local -> global map produced the ordinals.  Round r's winner stays in lane r, and the cell is
// written the way topk_kernel writes one: worst first, then the padding.  Value bits pass through unchanged.
__global__ void topk_merge_parts_kernel(const double* __restrict__ pv, const int64_t* __restrict__ pid, int n_parts, int64_t n_cells, int kk,
                                        int bottom, double* __restrict__ out_val, int64_t* __restrict__ out_id) {
  const int64_t cell = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (cell >= n_cells) return;                                        // warp-uniform
  const int lane = threadIdx.x & 31;
  double cv = 0.0; int64_t cid = -1;
  for (int p = lane; p < n_parts; p += 32) {
    const size_t base = ((size_t)p * n_cells + cell) * kk;
    for (int s = 0; s < kk; ++s) topk_fold_below(pv[base + s], pid[base + s], 0.0, -1, bottom, cv, cid);
  }
  double rv = 0.0; int64_t rid = -1;
  int m = 0;
  for (; m < kk; ++m) {
    double bv = cv; int64_t bi = cid;
    topk_warp_best(bv, bi, bottom);
    if (bi < 0) break;                                                // every part is exhausted (uniform: see topk_warp_best)
    if (lane == m) { rv = bv; rid = bi; }
    // the lane the winner came from (the winner is some lane's candidate, so the ballot is never empty; the lowest such lane)
    const int wl = __ffs(__ballot_sync(0xffffffffu, cid >= 0 && cid == bi)) - 1;
    double nv = 0.0; int64_t ni = -1;
    for (int p = wl; p < n_parts; p += 32) {
      const size_t i = ((size_t)p * n_cells + cell) * kk + lane;
      if (lane < kk) topk_fold_below(pv[i], pid[i], bv, bi, bottom, nv, ni);
    }
    topk_warp_best(nv, ni, bottom);
    if (lane == wl) { cv = nv; cid = ni; }
  }
  const int src = lane < m ? m - 1 - lane : lane;
  const double wv = __shfl_sync(0xffffffffu, rv, src);
  const int64_t wi = __shfl_sync(0xffffffffu, rid, src);
  if (lane < kk) {
    const size_t o = (size_t)cell * kk + lane;
    if (lane < m) { out_val[o] = wv; out_id[o] = wi; }
    else { out_val[o] = bottom ? 1.7976931348623157e308 : -1.7976931348623157e308; out_id[o] = -1; }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// group bookkeeping (device side, so that synthetic tables never leave the GPU)
// ---------------------------------------------------------------------------------------------------------------
__global__ void iota_kernel(int32_t* a, int64_t n) { int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; if (i < n) a[i] = (int32_t)i; }
// group_start[g] = lower_bound(sorted_keys, g)
__global__ void group_bounds_kernel(const int32_t* __restrict__ sorted_keys, int64_t n, int n_groups, int64_t* __restrict__ group_start) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g > n_groups) return;
  int64_t lo = 0, hi = n;
  while (lo < hi) { int64_t m = (lo + hi) >> 1; if (sorted_keys[m] < g) lo = m + 1; else hi = m; }
  group_start[g] = lo;
}
// items per group -> gis (exclusive scan done by caller with cub); fill item_begin
__global__ void group_item_count_kernel(const int64_t* __restrict__ group_start, int n_groups, int seg, int64_t* __restrict__ cnt) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n_groups) { int64_t n = group_start[g + 1] - group_start[g]; cnt[g] = (n + seg - 1) / seg; }
}
__global__ void fill_items_kernel(const int64_t* __restrict__ group_start, const int64_t* __restrict__ gis, int n_groups, int seg,
                                  int64_t n_items, int64_t n_series, int64_t* __restrict__ item_begin) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n_groups) {
    const int64_t b = group_start[g], e = group_start[g + 1];
    int64_t it = gis[g];
    for (int64_t p = b; p < e; p += seg) item_begin[it++] = p;
  }
  if (g == 0) item_begin[n_items] = n_series;
}

// ---------------------------------------------------------------------------------------------------------------
// v2 kernels (scan_fast.cuh): TMA-staged records + blocked window reductions.  Per-warp shared memory:
//   [mbarrier 16 B][record staging buffer rec_cap][result transpose stage][accumulators (agg only)][decode scratch]
// One staging buffer per warp: the record is dead as soon as its chunks are resolved into scratch, so the bulk copy of the
// NEXT series is issued right after resolve and overlaps the whole window phase of the current one.
// ---------------------------------------------------------------------------------------------------------------
struct WarpStage {
  uint64_t* bar; uint8_t* buf; uint32_t cap; uint32_t parity; bool staged;
  const uint8_t* arena; const int64_t* rec_off;
  __device__ __forceinline__ void issue(int64_t series, int lane) {        // all lanes call; lane 0 issues
    const int64_t o = rec_off[series];
    const uint32_t bytes = (uint32_t)(rec_off[series + 1] - o);
    staged = cap != 0 && bytes <= cap;
    if (staged && lane == 0) { mbar_expect_tx(bar, bytes); tma_load_1d(buf, arena + o, bytes, bar); }
  }
  __device__ __forceinline__ const uint8_t* acquire(int64_t series) {       // record of `series`, previously issued
    if (!staged) return arena + rec_off[series];
    mbar_wait(bar, parity); parity ^= 1;
    return buf;
  }
};

template <int CLS>
__global__ void __launch_bounds__(FAST_WARPS * 32, FAST_MIN_CTAS)
scan_series_kernel_v2(const uint8_t* __restrict__ arena, const int64_t* __restrict__ rec_off, int64_t n_series,
                      QueryParams q, double* __restrict__ out, uint32_t rec_cap, uint32_t scratch_bytes,
                      unsigned long long* d_counters, int* d_err,
                      const int64_t* __restrict__ list, const unsigned long long* __restrict__ list_count) {
  if (list) n_series = (int64_t)*list_count;             // fallback pass of the tile kernel: only the listed series
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t gw = (int64_t)blockIdx.x * FAST_WARPS + warp, nw = (int64_t)gridDim.x * FAST_WARPS;
  const uint32_t per_warp = WARP_HDR_BYTES + rec_cap + STAGE_BYTES + scratch_bytes;
  uint8_t* base = smem + (size_t)warp * per_warp;
  WarpStage st{reinterpret_cast<uint64_t*>(base), base + WARP_HDR_BYTES, rec_cap, 0, false, arena, rec_off};
  double* stage = reinterpret_cast<double*>(base + WARP_HDR_BYTES + rec_cap);
  uint8_t* scratch = base + WARP_HDR_BYTES + rec_cap + STAGE_BYTES;
  if (lane == 0) { mbar_init(st.bar, 1); mbar_fence_init(); }
  __syncwarp();
  int64_t rows = 0, bytes = 0;
  int64_t ii = gw;
  if (ii < n_series) st.issue(list ? list[ii] : ii, lane);
  for (; ii < n_series; ii += nw) {
    const int64_t i = list ? list[ii] : ii;
    const uint8_t* rec = st.acquire(i);
    double* o = out + (size_t)i * q.T;
    int err;
    const int64_t inext_i = ii + nw;
    const bool has_next = inext_i < n_series;
    const int64_t inext = has_next ? (list ? list[inext_i] : inext_i) : 0;
    process_series<CLS>(rec, q, scratch, scratch_bytes, stage, lane, err, rows, bytes,
                   [&](int k, double v, bool valid) { if (valid) o[k] = v; },
                   [&]() { if (has_next) st.issue(inext, lane); });
    if (err) {
      if (lane == 0) report_error(d_err, err, i);
      __syncwarp();
      if (has_next) st.issue(inext, lane);      // process_series returned before its release hook ran
    }
    __syncwarp();
  }
  if (lane == 0 && (rows | bytes)) { atomicAdd(&d_counters[0], (unsigned long long)rows); atomicAdd(&d_counters[1], (unsigned long long)bytes); }
}

// MOM: stddev / stdvar moments (agg_op = AGG_SUM): a [T] Σv² row, written to pval + n_items * T
template <int CLS, bool MOM = false>
__global__ void __launch_bounds__(FAST_WARPS * 32, FAST_MIN_CTAS)
scan_agg_kernel_v2(const uint8_t* __restrict__ arena, const int64_t* __restrict__ rec_off, const int32_t* __restrict__ order,
                   const int64_t* __restrict__ item_begin, int64_t n_items,
                   QueryParams q, int agg_op, double* __restrict__ pval, uint32_t* __restrict__ pcnt,
                   uint32_t rec_cap, uint32_t scratch_bytes, uint32_t acc_bytes,
                   unsigned long long* d_counters, int* d_err,
                   const int64_t* __restrict__ list, const unsigned long long* __restrict__ list_count) {
  MomOnly<MOM, double*> pval2;
  if constexpr (MOM) pval2.v = pval + (size_t)n_items * q.T;            // (all items of the query, before the list narrows them)
  if (list) n_items = (int64_t)*list_count;              // fallback pass of the tile kernel: only the listed items
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t gw = (int64_t)blockIdx.x * FAST_WARPS + warp, nw = (int64_t)gridDim.x * FAST_WARPS;
  const uint32_t per_warp = WARP_HDR_BYTES + rec_cap + STAGE_BYTES + acc_bytes + scratch_bytes;
  uint8_t* base = smem + (size_t)warp * per_warp;
  WarpStage st{reinterpret_cast<uint64_t*>(base), base + WARP_HDR_BYTES, rec_cap, 0, false, arena, rec_off};
  double* stage = reinterpret_cast<double*>(base + WARP_HDR_BYTES + rec_cap);
  double* acc = reinterpret_cast<double*>(base + WARP_HDR_BYTES + rec_cap + STAGE_BYTES);
  MomOnly<MOM, double*> acc2;
  if constexpr (MOM) acc2.v = acc + q.T;                  // [T] Σv² between Σv and the counts
  uint32_t* cnt = reinterpret_cast<uint32_t*>(base + WARP_HDR_BYTES + rec_cap + STAGE_BYTES + (size_t)q.T * (MOM ? 16 : 8));
  uint8_t* scratch = base + WARP_HDR_BYTES + rec_cap + STAGE_BYTES + acc_bytes;
  if (lane == 0) { mbar_init(st.bar, 1); mbar_fence_init(); }
  __syncwarp();
  const double ident = agg_op == AGG_MIN ? __longlong_as_double(0x7ff0000000000000LL)
                     : agg_op == AGG_MAX ? __longlong_as_double(0xfff0000000000000LL) : 0.0;
  int64_t rows = 0, bytes = 0;
  // flattened (item, position) walk so that the next series to prefetch is always known
  int64_t it = gw;
  int64_t pos = 0, pend = 0;
  auto real_item = [&](int64_t x) -> int64_t { return list ? list[x] : x; };
  auto advance_item = [&]() { while (it < n_items) { const int64_t ri = real_item(it); pos = item_begin[ri]; pend = item_begin[ri + 1]; if (pos < pend) return true; it += nw; } return false; };
  bool have = advance_item();
  if (have) st.issue(order ? order[pos] : pos, lane);
  while (have) {
    for (int k = lane; k < q.T; k += 32) { acc[k] = ident; cnt[k] = 0; if constexpr (MOM) acc2.v[k] = 0.0; }
    __syncwarp();
    const int64_t my_item = real_item(it);
    while (true) {
      const int64_t i = order ? order[pos] : pos;
      // next series in walk order
      int64_t npos = pos + 1, nit = it, npend = pend; bool nhave = true;
      if (npos >= pend) { nit = it + nw; nhave = false; while (nit < n_items) { const int64_t ri = real_item(nit); npos = item_begin[ri]; npend = item_begin[ri + 1]; if (npos < npend) { nhave = true; break; } nit += nw; } }
      const int64_t inext = nhave ? (order ? order[npos] : npos) : -1;
      const uint8_t* rec = st.acquire(i);
      int err;
      process_series<CLS>(rec, q, scratch, scratch_bytes, stage, lane, err, rows, bytes,
                     [&](int k, double v, bool valid) {
                       if (valid && v == v) {              // RowAggregators skip NaN (SumRowAggregator.scala:22-29 ...)
                         double a = acc[k];
                         // min/maxIgnoreNaN(acc, v) (QueryUtils.scala:111-123): of two equal values the later one is kept
                         if (agg_op == AGG_MIN) a = a < v ? a : v;
                         else if (agg_op == AGG_MAX) a = a > v ? a : v;
                         else if (agg_op != AGG_COUNT) a += v;
                         acc[k] = a; cnt[k] += 1;
                         if constexpr (MOM) acc2.v[k] += v * v;
                       }
                     },
                     [&]() { if (inext >= 0) st.issue(inext, lane); });
      if (err) {
        if (lane == 0) report_error(d_err, err, i);
        __syncwarp();
        if (inext >= 0) st.issue(inext, lane);
      }
      __syncwarp();
      const bool same_item = nhave && nit == it;
      pos = npos; pend = npend; it = nit; have = nhave;
      if (!same_item) break;
    }
    double* pv = pval + (size_t)my_item * q.T; uint32_t* pc = pcnt + (size_t)my_item * q.T;
    for (int k = lane; k < q.T; k += 32) { pv[k] = acc[k]; pc[k] = cnt[k]; }
    if constexpr (MOM) { double* pv2 = pval2.v + (size_t)my_item * q.T; for (int k = lane; k < q.T; k += 32) pv2[k] = acc2.v[k]; }
    __syncwarp();
  }
  if (lane == 0 && (rows | bytes)) { atomicAdd(&d_counters[0], (unsigned long long)rows); atomicAdd(&d_counters[1], (unsigned long long)bytes); }
}

#ifndef FILO_CUSIM      // the launchers need nvcc; the emulation build (tests/cpp) calls the kernels through cusim::launch
#ifdef FILO_TILE_PROF
extern "C" int filo_debug_tile_prof(unsigned long long* out16, int reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out16, g_tile_prof, sizeof(unsigned long long) * 16);
  if (e == cudaSuccess && reset) { unsigned long long z[16] = {}; e = cudaMemcpyToSymbol(g_tile_prof, z, sizeof z); }
  return (int)e;
}
#endif
#ifdef FILO_WP_PROF
extern "C" int filo_debug_wp_prof(unsigned long long* out32, int reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out32, g_wp_prof, sizeof(unsigned long long) * 32);
  if (e == cudaSuccess && reset) { unsigned long long z[32] = {}; e = cudaMemcpyToSymbol(g_wp_prof, z, sizeof z); }
  return (int)e;
}
#endif
// ---------------------------------------------------------------------------------------------------------------
// host-callable launchers
// ---------------------------------------------------------------------------------------------------------------
template <int CLS>
static cudaError_t launch_series_v2_cls(const ScanLaunch& L, double* out, uint32_t rec_cap, size_t smem) {
  cudaError_t e = cudaFuncSetAttribute(scan_series_kernel_v2<CLS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  scan_series_kernel_v2<CLS><<<L.grid, FAST_WARPS * 32, smem, L.stream>>>(L.arena, L.rec_off, L.n_series, L.q, out, rec_cap, L.scratch_bytes,
                                                                           L.d_counters, L.d_err, L.list, L.list_count);
  return cudaGetLastError();
}
cudaError_t launch_scan_series_v2(const ScanLaunch& L, double* out, uint32_t rec_cap) {
  const size_t smem = (size_t)(WARP_HDR_BYTES + rec_cap + STAGE_BYTES + L.scratch_bytes) * FAST_WARPS;
  switch (fn_class_of(L.q.fn, L.q.cumulative, L.q.long_values)) {
    case CLASS_SUM: return launch_series_v2_cls<CLASS_SUM>(L, out, rec_cap, smem);
    case CLASS_MINMAX: return launch_series_v2_cls<CLASS_MINMAX>(L, out, rec_cap, smem);
    case CLASS_COUNTER: return launch_series_v2_cls<CLASS_COUNTER>(L, out, rec_cap, smem);
    default: return launch_series_v2_cls<CLASS_POINT>(L, out, rec_cap, smem);
  }
}
template <int CLS, bool MOM>
static cudaError_t launch_agg_v2_cls(const ScanLaunch& L, const int32_t* order, const int64_t* item_begin, int64_t n_items, int agg_op,
                                     double* pval, uint32_t* pcnt, uint32_t acc_bytes, uint32_t rec_cap, size_t smem) {
  cudaError_t e = cudaFuncSetAttribute(scan_agg_kernel_v2<CLS, MOM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  scan_agg_kernel_v2<CLS, MOM><<<L.grid, FAST_WARPS * 32, smem, L.stream>>>(L.arena, L.rec_off, order, item_begin, n_items, L.q, agg_op, pval, pcnt,
                                                                             rec_cap, L.scratch_bytes, acc_bytes, L.d_counters, L.d_err, L.list, L.list_count);
  return cudaGetLastError();
}
template <bool MOM>
static cudaError_t launch_agg_v2_any(const ScanLaunch& L, const int32_t* order, const int64_t* item_begin, int64_t n_items, int agg_op,
                                     double* pval, uint32_t* pcnt, uint32_t acc_bytes, uint32_t rec_cap, size_t smem) {
  switch (fn_class_of(L.q.fn, L.q.cumulative, L.q.long_values)) {
    case CLASS_SUM: return launch_agg_v2_cls<CLASS_SUM, MOM>(L, order, item_begin, n_items, agg_op, pval, pcnt, acc_bytes, rec_cap, smem);
    case CLASS_MINMAX: return launch_agg_v2_cls<CLASS_MINMAX, MOM>(L, order, item_begin, n_items, agg_op, pval, pcnt, acc_bytes, rec_cap, smem);
    case CLASS_COUNTER: return launch_agg_v2_cls<CLASS_COUNTER, MOM>(L, order, item_begin, n_items, agg_op, pval, pcnt, acc_bytes, rec_cap, smem);
    default: return launch_agg_v2_cls<CLASS_POINT, MOM>(L, order, item_begin, n_items, agg_op, pval, pcnt, acc_bytes, rec_cap, smem);
  }
}
cudaError_t launch_scan_agg_v2(const ScanLaunch& L, const int32_t* order, const int64_t* item_begin, int64_t n_items, int agg_op,
                               double* pval, uint32_t* pcnt, uint32_t acc_bytes, uint32_t rec_cap, bool moments) {
  const size_t smem = (size_t)(WARP_HDR_BYTES + rec_cap + STAGE_BYTES + acc_bytes + L.scratch_bytes) * FAST_WARPS;
  return moments ? launch_agg_v2_any<true>(L, order, item_begin, n_items, agg_op, pval, pcnt, acc_bytes, rec_cap, smem)
                 : launch_agg_v2_any<false>(L, order, item_begin, n_items, agg_op, pval, pcnt, acc_bytes, rec_cap, smem);
}
struct TileAggArgs { const int32_t* order; const int64_t* item_begin; int64_t n_items; int agg_op; double* pval; uint32_t* pcnt; };
template <int FN, bool AGG, bool MOM>
static cudaError_t launch_tile_fn(const ScanLaunch& L, double* out, const TileSmem& T, int64_t* fallback_list, unsigned long long* fallback_count,
                                  const TileAggArgs& A) {
  cudaError_t e = cudaFuncSetAttribute(scan_tile_kernel<FN, AGG, MOM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T.total);
  if (e != cudaSuccess) return e;
  scan_tile_kernel<FN, AGG, MOM><<<L.grid, TILE_LAUNCH_THREADS, T.total, L.stream>>>(L.arena, L.rec_off, L.n_series, L.q, out, T, fallback_list, fallback_count,
      L.d_counters, L.d_err, A.order, A.item_begin, A.n_items, A.agg_op, A.pval, A.pcnt);
  return cudaGetLastError();
}
template <bool AGG, bool MOM = false>
static cudaError_t launch_tile_any(const ScanLaunch& L, double* out, const TileSmem& T, int64_t* fallback_list, unsigned long long* fallback_count,
                                   const TileAggArgs& A) {
  switch (L.q.fn) {
    case FN_RATE: return launch_tile_fn<FN_RATE, AGG, MOM>(L, out, T, fallback_list, fallback_count, A);
    case FN_AVG: return launch_tile_fn<FN_AVG, AGG, MOM>(L, out, T, fallback_list, fallback_count, A);
    case FN_COUNT: return launch_tile_fn<FN_COUNT, AGG, MOM>(L, out, T, fallback_list, fallback_count, A);
    default: return launch_tile_fn<FN_SUM, AGG, MOM>(L, out, T, fallback_list, fallback_count, A);      // FN_SUM, FN_INCREASE on a delta schema
  }
}
cudaError_t launch_scan_tile(const ScanLaunch& L, double* out, const TileSmem& T, int64_t* fallback_list, unsigned long long* fallback_count) {
  return launch_tile_any<false>(L, out, T, fallback_list, fallback_count, TileAggArgs{nullptr, nullptr, 0, 0, nullptr, nullptr});
}
// fused across-series aggregate: one partial row per item (same contract as launch_scan_agg_v2); items with an irregular series
// are appended to fallback_list
cudaError_t launch_scan_tile_agg(const ScanLaunch& L, const TileSmem& T, const int32_t* order, const int64_t* item_begin, int64_t n_items, int agg_op,
                                 double* pval, uint32_t* pcnt, int64_t* fallback_list, unsigned long long* fallback_count, bool moments) {
  const TileAggArgs A{order, item_begin, n_items, agg_op, pval, pcnt};
  return moments ? launch_tile_any<true, true>(L, nullptr, T, fallback_list, fallback_count, A)
                 : launch_tile_any<true>(L, nullptr, T, fallback_list, fallback_count, A);
}
// v4 warp-pipeline kernel (scan_wp.cuh): one CTA of W.warps warps per SM; declined series go to fallback_list
template <int FN, int NW>
static cudaError_t launch_wp_nw(const ScanLaunch& L, double* out, const WpSmem& W, int64_t* fallback_list, unsigned long long* fallback_count) {
  const size_t smem = (size_t)W.per_warp * W.warps;
  cudaError_t e = cudaFuncSetAttribute(scan_wp_sum_kernel<FN, NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  scan_wp_sum_kernel<FN, NW><<<L.grid, W.warps * 32, smem, L.stream>>>(L.arena, L.rec_off, L.n_series, L.q, out, W, fallback_list, fallback_count, L.d_counters, L.d_err);
  return cudaGetLastError();
}
template <int FN>
static cudaError_t launch_wp_fn(const ScanLaunch& L, double* out, const WpSmem& W, int64_t* fallback_list, unsigned long long* fallback_count) {
  // the register budget follows the warps per CTA: 128 registers up to 16 warps, 96 up to 20
  if (W.warps <= (uint32_t)WP_MAX_WARPS) return launch_wp_nw<FN, WP_MAX_WARPS>(L, out, W, fallback_list, fallback_count);
  return launch_wp_nw<FN, WP_MAX_WARPS_ALIAS>(L, out, W, fallback_list, fallback_count);
}
cudaError_t launch_scan_wp(const ScanLaunch& L, double* out, const WpSmem& W, int64_t* fallback_list, unsigned long long* fallback_count) {
  switch (L.q.fn) {
    case FN_RATE: return launch_wp_fn<FN_RATE>(L, out, W, fallback_list, fallback_count);
    case FN_AVG: return launch_wp_fn<FN_AVG>(L, out, W, fallback_list, fallback_count);
    case FN_COUNT: return launch_wp_fn<FN_COUNT>(L, out, W, fallback_list, fallback_count);
    default: return launch_wp_fn<FN_SUM>(L, out, W, fallback_list, fallback_count);      // FN_SUM, FN_INCREASE on a delta schema
  }
}
// the same with a CTA-wide record stream (scan_wp_batch_kernel): 15 consumer warps + 1 producer warp per SM
template <int FN>
static cudaError_t launch_wp_batch_fn(const ScanLaunch& L, double* out, const WpBatchSmem& W, int64_t* fallback_list, unsigned long long* fallback_count) {
  cudaError_t e = cudaFuncSetAttribute(scan_wp_batch_kernel<FN, WP_BATCH_WARPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)W.total);
  if (e != cudaSuccess) return e;
  scan_wp_batch_kernel<FN, WP_BATCH_WARPS><<<L.grid, WP_BATCH_WARPS * 32, W.total, L.stream>>>(L.arena, L.rec_off, L.n_series, L.q, out, W, fallback_list,
      fallback_count, L.d_counters, L.d_err);
  return cudaGetLastError();
}
cudaError_t launch_scan_wp_batch(const ScanLaunch& L, double* out, const WpBatchSmem& W, int64_t* fallback_list, unsigned long long* fallback_count) {
  switch (L.q.fn) {
    case FN_RATE: return launch_wp_batch_fn<FN_RATE>(L, out, W, fallback_list, fallback_count);
    case FN_AVG: return launch_wp_batch_fn<FN_AVG>(L, out, W, fallback_list, fallback_count);
    case FN_COUNT: return launch_wp_batch_fn<FN_COUNT>(L, out, W, fallback_list, fallback_count);
    default: return launch_wp_batch_fn<FN_SUM>(L, out, W, fallback_list, fallback_count);      // FN_SUM, FN_INCREASE on a delta schema
  }
}
// v4 counter-class kernel (scan_wp_ctr.cuh): per-series rows (order == nullptr, n_items == 0) or one partial row per work item
template <int FN, bool AGG, int NW, bool IRR, bool MOM>
static cudaError_t launch_wp_ctr_nw(const ScanLaunch& L, double* out, const WpCtrSmem& W, int64_t* fallback_list, unsigned long long* fallback_count,
                                    const TileAggArgs& A) {
  const size_t smem = (size_t)W.per_warp * W.warps + sizeof(TileCtrTab) * (TILE_CTR_TABMAX + 1);
  cudaError_t e = cudaFuncSetAttribute(scan_wp_ctr_kernel<FN, AGG, NW, IRR, MOM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  scan_wp_ctr_kernel<FN, AGG, NW, IRR, MOM><<<L.grid, W.warps * 32, smem, L.stream>>>(L.arena, L.rec_off, L.n_series, L.q, out, W, fallback_list, fallback_count,
      L.d_counters, L.d_err, A.order, A.item_begin, A.n_items, A.agg_op, A.pval, A.pcnt);
  return cudaGetLastError();
}
template <int FN, bool AGG, bool MOM>
static cudaError_t launch_wp_ctr_fn(const ScanLaunch& L, double* out, const WpCtrSmem& W, int64_t* fallback_list, unsigned long long* fallback_count, const TileAggArgs& A) {
  if (W.tsr != 0) return launch_wp_ctr_nw<FN, AGG, 16, true, MOM>(L, out, W, fallback_list, fallback_count, A);      // irregular timestamps: the larger shared-memory footprint keeps it at <= 16 warps
  if (W.warps <= 16) return launch_wp_ctr_nw<FN, AGG, 16, false, MOM>(L, out, W, fallback_list, fallback_count, A);
  return launch_wp_ctr_nw<FN, AGG, WP_CTR_MAX_WARPS, false, MOM>(L, out, W, fallback_list, fallback_count, A);
}
template <bool AGG, bool MOM = false>
static cudaError_t launch_wp_ctr_any(const ScanLaunch& L, double* out, const WpCtrSmem& W, int64_t* fallback_list, unsigned long long* fallback_count, const TileAggArgs& A) {
  switch (L.q.fn) {
    case FN_RATE: return launch_wp_ctr_fn<FN_RATE, AGG, MOM>(L, out, W, fallback_list, fallback_count, A);
    case FN_INCREASE: return launch_wp_ctr_fn<FN_INCREASE, AGG, MOM>(L, out, W, fallback_list, fallback_count, A);
    default: return launch_wp_ctr_fn<FN_DELTA, AGG, MOM>(L, out, W, fallback_list, fallback_count, A);
  }
}
cudaError_t launch_scan_wp_ctr(const ScanLaunch& L, double* out, const WpCtrSmem& W, int64_t* fallback_list, unsigned long long* fallback_count) {
  return launch_wp_ctr_any<false>(L, out, W, fallback_list, fallback_count, TileAggArgs{nullptr, nullptr, 0, 0, nullptr, nullptr});
}
cudaError_t launch_scan_wp_ctr_agg(const ScanLaunch& L, const WpCtrSmem& W, const int32_t* order, const int64_t* item_begin, int64_t n_items, int agg_op,
                                   double* pval, uint32_t* pcnt, int64_t* fallback_list, unsigned long long* fallback_count, bool moments) {
  const TileAggArgs A{order, item_begin, n_items, agg_op, pval, pcnt};
  return moments ? launch_wp_ctr_any<true, true>(L, nullptr, W, fallback_list, fallback_count, A)
                 : launch_wp_ctr_any<true>(L, nullptr, W, fallback_list, fallback_count, A);
}
size_t v2_smem_per_warp(uint32_t rec_cap, uint32_t scratch_bytes, uint32_t acc_bytes) { return WARP_HDR_BYTES + (size_t)rec_cap + STAGE_BYTES + acc_bytes + scratch_bytes; }
cudaError_t launch_scan_series(const ScanLaunch& L, double* out) {
  size_t smem = L.use_smem ? (size_t)L.scratch_bytes * SCAN_WARPS : 0;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(scan_series_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  scan_series_kernel<<<L.grid, SCAN_WARPS * 32, smem, L.stream>>>(L.arena, L.rec_off, L.n_series, L.q, out,
      L.gscratch, L.scratch_bytes, L.use_smem, L.d_counters, L.d_err);
  return cudaGetLastError();
}
cudaError_t launch_scan_agg(const ScanLaunch& L, const int32_t* order, const int64_t* item_begin, int64_t n_items, int agg_op,
                            double* pval, uint32_t* pcnt, uint32_t acc_bytes) {
  size_t smem = L.use_smem ? (size_t)(L.scratch_bytes + acc_bytes) * SCAN_WARPS : 0;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(scan_agg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  scan_agg_kernel<<<L.grid, SCAN_WARPS * 32, smem, L.stream>>>(L.arena, L.rec_off, order, item_begin, n_items, L.q, agg_op,
      pval, pcnt, L.gscratch, L.scratch_bytes, acc_bytes, L.use_smem, L.d_counters, L.d_err);
  return cudaGetLastError();
}
cudaError_t launch_merge_partials(const double* pval, const uint32_t* pcnt, const int64_t* gis, int n_groups, int T, int agg_op,
                                  int partial_out, double* out_val, int64_t* out_cnt, cudaStream_t s) {
  const int ktiles = (T + 31) / 32;
  if (agg_moments(agg_op)) merge_partials_kernel<MERGE_MOMENTS><<<n_groups * ktiles, 256, 0, s>>>(pval, pcnt, gis, n_groups, T, agg_op, partial_out, out_val, out_cnt);
  else if (agg_op == AGG_GROUP) merge_partials_kernel<MERGE_GROUP><<<n_groups * ktiles, 256, 0, s>>>(pval, pcnt, gis, n_groups, T, agg_op, partial_out, out_val, out_cnt);
  else merge_partials_kernel<<<n_groups * ktiles, 256, 0, s>>>(pval, pcnt, gis, n_groups, T, agg_op, partial_out, out_val, out_cnt);
  return cudaGetLastError();
}
cudaError_t launch_present(int agg_op, int64_t n, const double* vals, const int64_t* cnts, double* out, cudaStream_t s) {
  present_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(agg_op, n, vals, cnts, out);
  return cudaGetLastError();
}
cudaError_t launch_topk(const double* per_series, const int32_t* order, const int64_t* group_start, int n_groups, int T, int k, int bottom,
                        double* out_val, int64_t* out_id, cudaStream_t s) {
  const int64_t n = (int64_t)n_groups * T;
  topk_kernel<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(per_series, order, group_start, n_groups, T, k, bottom, out_val, out_id);
  return cudaGetLastError();
}
cudaError_t launch_topk_merge_parts(const double* part_val, const int64_t* part_id, int n_parts, int64_t n_cells, int k, int bottom,
                                    double* out_val, int64_t* out_id, cudaStream_t s) {
  topk_merge_parts_kernel<<<(unsigned)((n_cells + 7) / 8), 256, 0, s>>>(part_val, part_id, n_parts, n_cells, k, bottom, out_val, out_id);
  return cudaGetLastError();
}
cudaError_t launch_iota(int32_t* a, int64_t n, cudaStream_t s) {
  iota_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a, n); return cudaGetLastError();
}
cudaError_t launch_group_bounds(const int32_t* sorted_keys, int64_t n, int n_groups, int64_t* group_start, cudaStream_t s) {
  group_bounds_kernel<<<(n_groups + 1 + 127) / 128, 128, 0, s>>>(sorted_keys, n, n_groups, group_start); return cudaGetLastError();
}
cudaError_t launch_group_item_count(const int64_t* group_start, int n_groups, int seg, int64_t* cnt, cudaStream_t s) {
  group_item_count_kernel<<<(n_groups + 127) / 128, 128, 0, s>>>(group_start, n_groups, seg, cnt); return cudaGetLastError();
}
cudaError_t launch_fill_items(const int64_t* group_start, const int64_t* gis, int n_groups, int seg, int64_t n_items, int64_t n_series,
                              int64_t* item_begin, cudaStream_t s) {
  fill_items_kernel<<<(n_groups + 127) / 128, 128, 0, s>>>(group_start, gis, n_groups, seg, n_items, n_series, item_begin);
  return cudaGetLastError();
}

#endif // FILO_CUSIM

} // namespace filo
