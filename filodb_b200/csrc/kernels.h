// Host-visible declarations of the CUDA launchers (scan_kernels.cu, synth_kernels.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "filo_record.h"

namespace filo {

constexpr int SCAN_WARPS = 4;          // warps (= series in flight) per CTA, v1 kernels
constexpr int FAST_WARPS = 4;          // v2 kernels
constexpr int FAST_MIN_CTAS = 4;       // register budget of the v2 kernels: 4 CTAs x 128 threads per SM (<= 128 regs/thread)
constexpr int CHUNK_DESC_BYTES = 144;  // sizeof(ChunkDesc), scan_device.cuh
constexpr int FILO_MAX_TOPK = 32;
enum { AGG_NONE = 0, AGG_SUM = 1, AGG_AVG = 2, AGG_MIN = 3, AGG_MAX = 4, AGG_COUNT = 5, AGG_TOPK = 6, AGG_BOTTOMK = 7,
       AGG_STDDEV = 8, AGG_STDVAR = 9, AGG_GROUP = 10 };
// stddev / stdvar fold the moments (Σv, Σv², n) of an (item, window): the scan kernels run their SUM mode plus a second partial block
__host__ __device__ inline bool agg_moments(int agg_op) { return agg_op == AGG_STDDEV || agg_op == AGG_STDVAR; }
// a variable of the moments instantiation of a kernel only: the other instantiations declare nothing (their code stays as it was)
template <bool ON, typename T> struct MomOnly { T v; };
template <typename T> struct MomOnly<false, T> {};

struct QueryParams;

} // namespace filo
#include "scan_params.h"
#include "scan_tile_layout.h"
namespace filo {

struct ScanLaunch {
  const uint8_t* arena; const int64_t* rec_off; int64_t n_series;
  QueryParams q;
  uint8_t* gscratch; uint32_t scratch_bytes; int use_smem;
  unsigned long long* d_counters; int* d_err;
  int grid; cudaStream_t stream;
  const int64_t* list = nullptr; const unsigned long long* list_count = nullptr;   // optional: process only these series
};

cudaError_t launch_scan_series(const ScanLaunch& L, double* out);
cudaError_t launch_scan_agg(const ScanLaunch& L, const int32_t* order, const int64_t* item_begin, int64_t n_items, int agg_op,
                            double* pval, uint32_t* pcnt, uint32_t acc_bytes);
cudaError_t launch_scan_series_v2(const ScanLaunch& L, double* out, uint32_t rec_cap);
// moments: pval holds [2][n_items][T] (Σv, then Σv²); agg_op is then AGG_SUM
cudaError_t launch_scan_agg_v2(const ScanLaunch& L, const int32_t* order, const int64_t* item_begin, int64_t n_items, int agg_op,
                               double* pval, uint32_t* pcnt, uint32_t acc_bytes, uint32_t rec_cap, bool moments = false);
size_t v2_smem_per_warp(uint32_t rec_cap, uint32_t scratch_bytes, uint32_t acc_bytes);
cudaError_t launch_scan_tile(const ScanLaunch& L, double* out, const TileSmem& T, int64_t* fallback_list, unsigned long long* fallback_count);
cudaError_t launch_scan_tile_agg(const ScanLaunch& L, const TileSmem& T, const int32_t* order, const int64_t* item_begin, int64_t n_items, int agg_op,
                                 double* pval, uint32_t* pcnt, int64_t* fallback_list, unsigned long long* fallback_count, bool moments = false);
cudaError_t launch_merge_partials(const double* pval, const uint32_t* pcnt, const int64_t* gis, int n_groups, int T, int agg_op,
                                  int partial_out, double* out_val, int64_t* out_cnt, cudaStream_t s);
cudaError_t launch_present(int agg_op, int64_t n, const double* vals, const int64_t* cnts, double* out, cudaStream_t s);
cudaError_t launch_topk(const double* per_series, const int32_t* order, const int64_t* group_start, int n_groups, int T, int k, int bottom,
                        double* out_val, int64_t* out_id, cudaStream_t s);
// merge of n_parts topk_kernel outputs [n_parts][n_cells][k] (ids global series ordinals, -1 = empty) into [n_cells][k]
cudaError_t launch_topk_merge_parts(const double* part_val, const int64_t* part_id, int n_parts, int64_t n_cells, int k, int bottom,
                                    double* out_val, int64_t* out_id, cudaStream_t s);
struct WpSmem;
cudaError_t launch_scan_wp(const ScanLaunch& L, double* out, const WpSmem& W, int64_t* fallback_list, unsigned long long* fallback_count);
struct WpBatchSmem;
cudaError_t launch_scan_wp_batch(const ScanLaunch& L, double* out, const WpBatchSmem& W, int64_t* fallback_list, unsigned long long* fallback_count);
struct WpCtrSmem;
cudaError_t launch_scan_wp_ctr(const ScanLaunch& L, double* out, const WpCtrSmem& W, int64_t* fallback_list, unsigned long long* fallback_count);
cudaError_t launch_scan_wp_ctr_agg(const ScanLaunch& L, const WpCtrSmem& W, const int32_t* order, const int64_t* item_begin, int64_t n_items, int agg_op,
                                   double* pval, uint32_t* pcnt, int64_t* fallback_list, unsigned long long* fallback_count, bool moments = false);
size_t hist_smem_bytes(int max_rows, int nb, int T, bool agg, uint32_t max_rec);
// agg == 0 with out_q: per-series histogram_quantile (tops, qtl, exp_buckets) to out_q [S][T], the rows to out when given
cudaError_t launch_hist_scan(const ScanLaunch& L, int nb, int max_rows, uint32_t max_rec, const int32_t* order, const int64_t* item_begin, int64_t n_items, int agg,
                             double* out, double* pval, uint8_t* pany, const double* tops = nullptr, double qtl = 0.0, int exp_buckets = 0, double* out_q = nullptr);
cudaError_t launch_hist_merge(const double* pval, const uint8_t* pany, const int64_t* gis, int n_groups, int T, int nb, int exp_buckets, const double* tops, double q,
                              double* out_values, double* out_q, cudaStream_t s);
// second version of the histogram scan (hist_kernels2.cu): rate / increase over cumulative SectDelta histograms and last over SectDelta
// histograms, fused sum (launch_hist_scan2) or per series (launch_hist_scan2_series: buckets to out_values [S][T][nb] and / or
// histogram_quantile to out_q [S][T]; without out_values, scratch holds grid * T * nb doubles)
size_t hist2_smem_bytes(int max_rows, int nb, uint32_t max_rec);
cudaError_t launch_hist_scan2(const ScanLaunch& L, int nb, int max_rows, uint32_t max_rec, const int32_t* order, const int64_t* item_begin, int64_t n_items,
                              double* pval, uint8_t* pany);
int64_t hist2_series_items(int64_t n_series);
cudaError_t launch_hist_scan2_series(const ScanLaunch& L, int nb, int max_rows, uint32_t max_rec, double* out_values, double* out_q, double* scratch,
                                     const double* tops, double qtl, int exp_buckets);
cudaError_t launch_hist_merge2(const double* pval, const uint8_t* pany, const int64_t* gis, int n_groups, int T, int nb, int exp_buckets, const double* tops, double q,
                               double* out_values, double* out_q, cudaStream_t s);
// rank-order fold of n_parts histogram SUM outputs [n_parts][n_cells][nb] (empty cell: NaN bucket 0), histogram_quantile when out_q is given
cudaError_t launch_hist_merge_parts(const double* parts, int n_parts, int64_t n_cells, int nb, int exp_buckets, const double* tops, double q,
                                    double* out_values, double* out_q, cudaStream_t s);
cudaError_t launch_iota(int32_t* a, int64_t n, cudaStream_t s);
cudaError_t launch_group_bounds(const int32_t* sorted_keys, int64_t n, int n_groups, int64_t* group_start, cudaStream_t s);
cudaError_t launch_group_item_count(const int64_t* group_start, int n_groups, int seg, int64_t* cnt, cudaStream_t s);
cudaError_t launch_fill_items(const int64_t* group_start, const int64_t* gis, int n_groups, int seg, int64_t n_items, int64_t n_series,
                              int64_t* item_begin, cudaStream_t s);

} // namespace filo
