// Histogram column scan, second version (hist rate / increase over cumulative SectDelta histograms and hist last over SectDelta
// histograms, fused sum or per series with histogram_quantile): the kernel that
// strings the phases of hist_phases.h together.  filo_query_hist selects it for the shapes it serves (capi.cu; FILO_HIST_V2=0 turns it
// off for A/B runs); the first version (hist_kernels.cu) serves every other shape.
#include "kernels.h"
#include "hist_phases.h"

namespace filo {

// Per-phase cycle counters for profiling builds (-DFILO_HIST_PROF; scratch/hist_prof.py): thread 0 of every CTA reads clock64() after each
// phase barrier.  Compiled out of the product build.
#if defined(FILO_HIST_PROF) && !defined(FILO_CUSIM)
__device__ unsigned long long g_hist2_prof[16];
#define H2PROF_DECL long long hp_t0 = clock64(), hp_acc[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
#define H2PROF(i) { const long long hp_t1 = clock64(); hp_acc[i] += hp_t1 - hp_t0; hp_t0 = hp_t1; }
#define H2PROF_FLUSH if (threadIdx.x == 0) { for (int hp_i = 0; hp_i < 12; ++hp_i) atomicAdd(&g_hist2_prof[hp_i], (unsigned long long)hp_acc[hp_i]); atomicAdd(&g_hist2_prof[15], 1ull); }
#else
#define H2PROF_DECL
#define H2PROF(i)
#define H2PROF_FLUSH
#endif

__device__ __forceinline__ void h2_report(int* d_err, int code, int64_t sid) {
  if (atomicCAS(&d_err[0], 0, code) == 0) { d_err[1] = (int)(sid & 0x7fffffff); d_err[2] = (int)(sid >> 31); }
}

// record bytes global -> shared with 16-byte cp.async (LDGSTS); the caller waits with cp.async.wait_group + a CTA barrier
#ifdef FILO_CUSIM          // host emulation build (tests/cpp/cusim.h)
inline void h2_stage_async(uint8_t* dst, const uint8_t* src, uint32_t bytes, int tid) {
  for (uint32_t i = (uint32_t)tid * 16; i < bytes; i += H2_THREADS * 16) cusim::cp_async(dst + i, src + i, 16);
}
inline void h2_stage_wait() { cusim::cp_async_wait_all(); }
#else
__device__ __forceinline__ void h2_stage_async(uint8_t* dst, const uint8_t* __restrict__ src, uint32_t bytes, int tid) {
  const uint32_t d0 = (uint32_t)__cvta_generic_to_shared(dst);
  for (uint32_t i = (uint32_t)tid * 16; i < bytes; i += H2_THREADS * 16)
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d0 + i), "l"(src + i) : "memory");
  asm volatile("cp.async.commit_group;" ::: "memory");
}
__device__ __forceinline__ void h2_stage_wait() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
#endif

// One CTA folds work items (runs of series of one group, positions index `order`) into the item's partial row
// pval[it][bucket][window] (bucket-major) and pany[it][window].
// SERIES (per-series mode, no aggregate): a work item is the run of series [it * H2_RUN, ...), and the thread that owns a window presents the
// series' own window histogram: its buckets to S.out_v[S][T][nb] and / or its Histogram.quantile to S.out_q[S][T].  Without out_v the buckets
// pass through the CTA's column block S.scratch[cta][nb][T] (bucket-major: the owners of consecutive windows touch consecutive doubles), so
// [S][T][nb] exists nowhere.  LAST: LastSampleChunkedFunctionH (h2_window_last); the counter corrections (P4-P6) do not run.
constexpr int H2_RUN = 64;
struct H2Series { double* out_v; double* out_q; double* scratch; const double* tops; double qtl; int exp_buckets; };
template <bool SERIES = false, bool LAST = false>
__global__ void __launch_bounds__(H2_THREADS, 2)
hist_scan2_kernel(const uint8_t* __restrict__ arena, const int64_t* __restrict__ rec_off, QueryParams q, int nb, int max_rows, uint32_t max_rec,
                  const int32_t* __restrict__ order, const int64_t* __restrict__ item_begin, int64_t n_items,
                  double* __restrict__ pval, uint8_t* __restrict__ pany, unsigned long long* d_counters, int* d_err, H2Series S = H2Series{}, int64_t n_series = 0) {
  extern __shared__ __align__(16) uint8_t smem[];
  H2Ctx X; h2_ctx_init(X, smem, h2_layout(max_rows, nb, max_rec), q, nb);
  const int tid = threadIdx.x;
  int64_t rows_scanned = 0, bytes_scanned = 0;
  H2PROF_DECL
  for (int64_t it = blockIdx.x; it < n_items; it += gridDim.x) {
    int64_t pb, pe;
    double* pv = nullptr; uint8_t* pa = nullptr;
    uint32_t anyb = 0;                                   // bit j: window tid + j * H2_THREADS has a histogram
    if constexpr (SERIES) {
      pb = it * H2_RUN; pe = pb + H2_RUN < n_series ? pb + H2_RUN : n_series;
    } else {
      pb = item_begin[it]; pe = item_begin[it + 1];
      pv = pval + (size_t)it * q.T * nb; pa = pany + (size_t)it * q.T;
      for (int i = tid; i < q.T * nb; i += H2_THREADS) pv[i] = 0.0;
      __syncthreads();                                   // the zero fill is visible to the owners of the windows
    }
    bool prefetched = false;                             // the record of `pos` is already on its way (cp.async issued after the previous decode)
    for (int64_t pos = pb; pos < pe; ++pos) {
      const int64_t sid = order ? (int64_t)order[pos] : pos;
      if (!prefetched) {                                 // stage the record (16-byte aligned, size a multiple of 16)
        const int64_t ro = rec_off[sid];
        h2_stage_async(smem + X.L.rec, arena + ro, (uint32_t)(rec_off[sid + 1] - ro), tid);
      }
      h2_stage_wait();
      __syncthreads();
      H2PROF(0)                                           // record staged (prefetched behind the previous series)
      h2_tables(tid, X, max_rows);
      __syncthreads();
      H2PROF(1)                                           // chunk range + section table (thread 0)
      if (tid == 0) {
        const H2Ctl* C = X.ctl();
        rows_scanned += C->rows_scanned; bytes_scanned += C->bytes_scanned;
        if (C->err) h2_report(d_err, C->err, sid);
      }
      h2_decode_rows(tid, H2_THREADS, X);
      __syncthreads();
      H2PROF(2)                                           // timestamps + rows decoded
      // the staged record is dead from here on: fetch the next series' record behind the remaining phases
      prefetched = pos + 1 < pe;
      if (prefetched) {
        const int64_t nsid = order ? (int64_t)order[pos + 1] : pos + 1;
        const int64_t ro = rec_off[nsid];
        h2_stage_async(smem + X.L.rec, arena + ro, (uint32_t)(rec_off[nsid + 1] - ro), tid);
      }
      if (tid == 0 && X.ctl()->bad) h2_report(d_err, 1, sid);
      h2_add_base(tid, H2_THREADS, X);
      __syncthreads();
      H2PROF(3)                                           // next record issued, SectDelta bases added
      if constexpr (!LAST) {
        h2_chunk_corrections(tid, H2_THREADS, X);
        __syncthreads();
        h2_chunk_less(tid, X);
        __syncthreads();
        h2_carried(tid, H2_THREADS, X);
        __syncthreads();
      }
      H2PROF(4)                                           // corrections inside and across chunks
      if constexpr (SERIES) {
        const double NaNv = h2_nan();
        for (int k = tid; k < q.T; k += H2_THREADS) {
          // the window's buckets: in the output row when one is asked for (re-read below by this thread only), else in the CTA's column block
          double* w = S.out_v ? S.out_v + ((size_t)sid * q.T + k) * nb : S.scratch + (size_t)blockIdx.x * q.T * nb + k;
          const size_t ws = S.out_v ? 1 : (size_t)q.T;
          const bool has = LAST ? h2_window_last<true>(k, X, w, true, ws) : h2_window<true>(k, X, w, true, ws);
          if (!has && S.out_v) for (int b = 0; b < nb; ++b) w[b] = NaNv;                      // Histogram.empty: NaN buckets
          if (S.out_q) S.out_q[(size_t)sid * q.T + k] = (has && S.qtl == S.qtl) ? hist_quantile(w, ws, nb, S.tops, S.qtl, S.exp_buckets != 0) : NaNv;
        }
      } else {
        int j = 0;
        if constexpr (LAST) { for (int k = tid; k < q.T; k += H2_THREADS, ++j) if (h2_window_last(k, X, pv, !((anyb >> j) & 1u))) anyb |= 1u << j; }
        else { for (int k = tid; k < q.T; k += H2_THREADS, ++j) if (h2_window(k, X, pv, !((anyb >> j) & 1u))) anyb |= 1u << j; }
      }
      __syncthreads();                                   // the series' rows and record are dead
      H2PROF(5)                                           // windows: descriptors + rates + partial-row update
    }
    if constexpr (!SERIES) { int j = 0; for (int k = tid; k < q.T; k += H2_THREADS, ++j) pa[k] = (uint8_t)((anyb >> j) & 1u); }
  }
  H2PROF_FLUSH
  if (tid == 0 && (rows_scanned | bytes_scanned)) { atomicAdd(&d_counters[0], (unsigned long long)rows_scanned); atomicAdd(&d_counters[1], (unsigned long long)bytes_scanned); }
}

// Fold the partial rows of each group in item order (deterministic), MutableHistogram.add per item (Histogram.scala:428-449),
// then Histogram.quantile (:65-108, hist_quantile in hist_phases.h).  Thread per (group, window); partial rows are bucket-major.
__global__ void hist_merge2_kernel(const double* __restrict__ pval, const uint8_t* __restrict__ pany, const int64_t* __restrict__ gis,
                                   int n_groups, int T, int nb, int exp_buckets, const double* __restrict__ tops, double qtl,
                                   double* __restrict__ out_values /* [G][T][nb] or null */, double* __restrict__ out_q /* [G][T] or null */) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_groups * T) return;
  const int g = (int)(i / T), k = (int)(i - (int64_t)g * T);
  const double NaNv = __longlong_as_double(0x7ff8000000000000LL);
  double v[64]; bool any = false;
  for (int b = 0; b < nb; ++b) v[b] = 0.0;
  // ReduceAggregateExec over the items' partial aggregates with the same reduceAggregate: the first one is copied, every further one
  // is added and the sum made monotonic (HistSumRowAggregator.scala:25-36, Histogram.scala:428-449)
  for (int64_t it = gis[g]; it < gis[g + 1]; ++it) {
    if (!pany[(size_t)it * T + k]) continue;
    const double* pv = pval + (size_t)it * T * nb + k;
    if (!any) { for (int b = 0; b < nb; ++b) v[b] = pv[(size_t)b * T]; any = true; continue; }
    hist_add_monotonic(v, pv, (size_t)T, nb);
  }
  const double qv = (any && qtl == qtl) ? hist_quantile(v, nb, tops, qtl, exp_buckets != 0) : NaNv;
  if (out_values) for (int b = 0; b < nb; ++b) out_values[(size_t)i * nb + b] = any ? v[b] : NaNv;
  if (out_q) out_q[i] = qv;
}

// The cross-GPU reduce of histogram sums (filo_merge_hist_partials): parts holds n_parts SUM outputs of filo_query_hist_device back to
// back, [n_parts][n_cells][nb] with n_cells = G * T, in rank order.  A part's cell is empty when its bucket 0 is NaN: a SUM output is NaN
// in every bucket where its group had no histogram, and never NaN in bucket 0 otherwise (integer-count inputs give finite window
// histograms, and makeMonotonic replaces a NaN by the running maximum, which starts at 0).  ReduceAggregateExec with
// HistSumRowAggregator.reduceAggregate folds the parts in rank order: the first non-empty one is copied, every further one goes through
// hist_add_monotonic.  Then Histogram.quantile when out_q is given.  Thread per (group, window).
__global__ void hist_merge_parts_kernel(const double* __restrict__ parts, int n_parts, int64_t n_cells, int nb, int exp_buckets,
                                        const double* __restrict__ tops, double qtl,
                                        double* __restrict__ out_values /* [G][T][nb] or null */, double* __restrict__ out_q /* [G][T] or null */) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_cells) return;
  const double NaNv = __longlong_as_double(0x7ff8000000000000LL);
  double v[64]; bool any = false;
  for (int p = 0; p < n_parts; ++p) {
    const double* pv = parts + ((size_t)p * (size_t)n_cells + (size_t)i) * nb;
    if (pv[0] != pv[0]) continue;                                  // Histogram.empty on this rank
    if (!any) { for (int b = 0; b < nb; ++b) v[b] = pv[b]; any = true; continue; }
    hist_add_monotonic(v, pv, 1, nb);
  }
  if (out_values) for (int b = 0; b < nb; ++b) out_values[(size_t)i * nb + b] = any ? v[b] : NaNv;
  if (out_q) out_q[i] = any ? hist_quantile(v, nb, tops, qtl, exp_buckets != 0) : NaNv;
}

#ifndef FILO_CUSIM      // launchers need nvcc
#ifdef FILO_HIST_PROF
extern "C" int filo_debug_hist2_prof(unsigned long long* out16, int reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out16, g_hist2_prof, sizeof(unsigned long long) * 16);
  if (e == cudaSuccess && reset) { unsigned long long z[16] = {}; e = cudaMemcpyToSymbol(g_hist2_prof, z, sizeof z); }
  return (int)e;
}
#endif
size_t hist2_smem_bytes(int max_rows, int nb, uint32_t max_rec) { return h2_layout(max_rows, nb, max_rec).total; }
template <bool SERIES, bool LAST>
static cudaError_t launch_hist_scan2_t(const ScanLaunch& L, int nb, int max_rows, uint32_t max_rec, const int32_t* order, const int64_t* item_begin, int64_t n_items,
                                       double* pval, uint8_t* pany, const H2Series& S) {
  const size_t smem = h2_layout(max_rows, nb, max_rec).total;
  cudaError_t e = cudaFuncSetAttribute(hist_scan2_kernel<SERIES, LAST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  hist_scan2_kernel<SERIES, LAST><<<L.grid, H2_THREADS, smem, L.stream>>>(L.arena, L.rec_off, L.q, nb, max_rows, max_rec, order, item_begin, n_items, pval, pany,
                                                                          L.d_counters, L.d_err, S, L.n_series);
  return cudaGetLastError();
}
cudaError_t launch_hist_scan2(const ScanLaunch& L, int nb, int max_rows, uint32_t max_rec, const int32_t* order, const int64_t* item_begin, int64_t n_items,
                              double* pval, uint8_t* pany) {
  const H2Series S{};
  return L.q.fn == FN_LAST ? launch_hist_scan2_t<false, true>(L, nb, max_rows, max_rec, order, item_begin, n_items, pval, pany, S)
                           : launch_hist_scan2_t<false, false>(L, nb, max_rows, max_rec, order, item_begin, n_items, pval, pany, S);
}
int64_t hist2_series_items(int64_t n_series) { return (n_series + H2_RUN - 1) / H2_RUN; }
cudaError_t launch_hist_scan2_series(const ScanLaunch& L, int nb, int max_rows, uint32_t max_rec, double* out_values, double* out_q, double* scratch,
                                     const double* tops, double qtl, int exp_buckets) {
  const H2Series S{out_values, out_q, scratch, tops, qtl, exp_buckets};
  const int64_t n_items = hist2_series_items(L.n_series);
  return L.q.fn == FN_LAST ? launch_hist_scan2_t<true, true>(L, nb, max_rows, max_rec, nullptr, nullptr, n_items, nullptr, nullptr, S)
                           : launch_hist_scan2_t<true, false>(L, nb, max_rows, max_rec, nullptr, nullptr, n_items, nullptr, nullptr, S);
}
cudaError_t launch_hist_merge2(const double* pval, const uint8_t* pany, const int64_t* gis, int n_groups, int T, int nb, int exp_buckets, const double* tops, double q,
                               double* out_values, double* out_q, cudaStream_t s) {
  const int64_t n = (int64_t)n_groups * T;
  if (n <= 0) return cudaSuccess;
  hist_merge2_kernel<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(pval, pany, gis, n_groups, T, nb, exp_buckets, tops, q, out_values, out_q);
  return cudaGetLastError();
}
cudaError_t launch_hist_merge_parts(const double* parts, int n_parts, int64_t n_cells, int nb, int exp_buckets, const double* tops, double q,
                                    double* out_values, double* out_q, cudaStream_t s) {
  if (n_cells <= 0) return cudaSuccess;
  hist_merge_parts_kernel<<<(unsigned)((n_cells + 127) / 128), 128, 0, s>>>(parts, n_parts, n_cells, nb, exp_buckets, tops, q, out_values, out_q);
  return cudaGetLastError();
}

#endif // FILO_CUSIM

} // namespace filo
