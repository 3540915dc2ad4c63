// The per-series kernel filo_query runs for one table shape (scan_path, scan_wp_layout.h), with its layout, its grid and how deep
// into a persistent grid the table's series reach: series per warp and the last buffer round every warp gets to.  Test
// infrastructure: built with g++ and run by tests/test_scan_path.py, tests/test_gpu_steady_state.py and tests/test_gpu_fused_steady_state.py.
//   scan_path rec=<max_rec_bytes> rows=<max_rows> chunks=<max_chunks> T=<windows> wrows=<window / step + 1> n=<series>
//             [cls=sum|counter|minmax|point] [fused=0|1 items=<work items>] [moments=0|1] [irr=0|1] [v2=0|1] [smem=<cap bytes>] [sms=<SMs>]
// v2=1 (the default) says the v2 kernel's per-warp working set fits, which filo_query checks before it asks scan_path.
// Prints one key=value per line:
//   kernel      batch | sum | tile | ctr | v2 (batch: scan_wp_batch_kernel, sum: scan_wp_sum_kernel, ctr: scan_wp_ctr_kernel)
//   alias       1 when O sits on V (batch and sum)
//   warps       warps per CTA that take series (batch: consumer warps)
//   rec_bufs    record buffers a warp's series rotate through (batch: batch buffers)
//   B           series per batch (batch)
//   grid, smem  CTAs and dynamic shared memory per CTA
//   series_per_warp  the fewest series any warp takes (tile: the fewest tiles any CTA takes)
//   rounds      the last buffer round u = k / rec_bufs every warp reaches (k: the warp's series index from 0); -1 below one series
// and with fused=1, the fused aggregate path over `items` work items:
//   fused_kernel    ctr | tile | v2 (ctr: scan_wp_ctr_kernel<AGG>, tile: scan_tile_kernel<AGG>, each with scan_agg_kernel_v2 behind it
//                   for the items it declines; v2: the v2 / v1 aggregate kernel alone)
//   fused_grid      CTAs of the ctr / tile kernel (0 for v2)
//   items_per_warp  the fewest items any warp (ctr) or CTA (tile) takes; -1 for v2
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include "scan_wp_layout.h"

using namespace filo;

int main(int argc, char** argv) {
  ScanPathIn in{};
  in.v2 = true; in.smem_cap = 227 * 1024; in.sm_count = 132; in.fn_cls = CLASS_SUM;
  for (int a = 1; a < argc; ++a) {
    const char* eq = std::strchr(argv[a], '=');
    if (!eq) { std::fprintf(stderr, "argument %s: want key=value\n", argv[a]); return 2; }
    const std::string k(argv[a], eq - argv[a]), v(eq + 1);
    const long long x = std::strtoll(v.c_str(), nullptr, 10);
    if (k == "rec") in.max_rec_bytes = (uint32_t)x;
    else if (k == "rows") in.max_rows = (uint32_t)x;
    else if (k == "chunks") in.max_chunks = (uint32_t)x;
    else if (k == "T") in.T = (uint32_t)x;
    else if (k == "wrows") in.wrows = (uint64_t)x;
    else if (k == "n") in.n_series = x;
    else if (k == "items") in.n_items = x;
    else if (k == "cls") {
      if (v == "sum") in.fn_cls = CLASS_SUM; else if (v == "counter") in.fn_cls = CLASS_COUNTER;
      else if (v == "minmax") in.fn_cls = CLASS_MINMAX; else if (v == "point") in.fn_cls = CLASS_POINT;
      else { std::fprintf(stderr, "unknown class %s\n", v.c_str()); return 2; }
    }
    else if (k == "fused") in.fused = x != 0;
    else if (k == "moments") in.moments = x != 0;
    else if (k == "irr") in.irr = x != 0;
    else if (k == "v2") in.v2 = x != 0;
    else if (k == "smem") in.smem_cap = (uint64_t)x;
    else if (k == "sms") in.sm_count = (int)x;
    else { std::fprintf(stderr, "unknown key %s\n", k.c_str()); return 2; }
  }
  if (in.T == 0 || in.wrows == 0) { std::fprintf(stderr, "T and wrows are required\n"); return 2; }
  const ScanPath P = scan_path(in);
  if (P.refused) { std::printf("kernel=refused\n"); return 0; }
  const int64_t n = in.n_series, grid = P.grid;
  const char* name = "v2";
  int64_t warps = 0, bufs = 1, B = 0, smem = 0, alias = 0;
  switch (P.kernel) {
    case SCAN_PATH_WP_BATCH: name = "batch"; warps = P.WB.consumers; bufs = P.WB.nbuf; B = P.WB.B; smem = P.WB.total; alias = P.WB.W.alias; break;
    case SCAN_PATH_WP_SUM: name = "sum"; warps = P.WL.warps; bufs = P.WL.rec2 ? 2 : 1; smem = (int64_t)P.WL.per_warp * P.WL.warps; alias = P.WL.alias; break;
    case SCAN_PATH_WP_CTR: name = "ctr"; warps = P.WC.warps; smem = P.WC.tab + (int64_t)sizeof(TileCtrTab) * (TILE_CTR_TABMAX + 1); break;
    case SCAN_PATH_TILE: name = "tile"; smem = P.TL.total; break;
    default: break;
  }
  // the fewest series a warp takes, and the last buffer round every warp reaches
  int64_t fewest = -1;
  if (P.kernel == SCAN_PATH_WP_BATCH) {
    // CTA c takes batches g = c + i * grid (i = 0, 1, ..) of B consecutive series; its consumer warp w takes positions w, w + warps, ..
    // of the CTA's series in batch order
    for (int64_t c = 0; c < grid; ++c) {
      int64_t cta_series = 0;
      for (int64_t i = 0; (c + i * grid) * B < n; ++i) { const int64_t s0 = (c + i * grid) * B; cta_series += (n - s0 < B ? n - s0 : B); }
      for (int64_t w = 0; w < warps; ++w) {
        const int64_t k = cta_series > w ? (cta_series - w + warps - 1) / warps : 0;
        if (fewest < 0 || k < fewest) fewest = k;
      }
    }
  } else if (P.kernel == SCAN_PATH_WP_SUM || P.kernel == SCAN_PATH_WP_CTR) {
    fewest = n / (grid * warps);                          // warp gw takes series gw + k * (grid * warps)
  } else if (P.kernel == SCAN_PATH_TILE) {
    fewest = ((n + TILE_NS - 1) / TILE_NS) / grid;        // CTA c takes tiles c + k * grid
  }
  // a batch warp's k-th series is in batch i = k * warps / B of its CTA (warps = B), so its round is k / nbuf like the per-warp kernels'
  const int64_t rounds = fewest > 0 ? (fewest - 1) / bufs : -1;
  std::printf("kernel=%s\nalias=%lld\nwarps=%lld\nrec_bufs=%lld\nB=%lld\ngrid=%lld\nsmem=%lld\nseries_per_warp=%lld\nrounds=%lld\n", name,
              (long long)alias, (long long)warps, (long long)bufs, (long long)B, (long long)grid, (long long)smem, (long long)fewest,
              (long long)rounds);
  if (in.fused) {
    // ctr: warp gw takes items gw + k * (grid * warps); tile: CTA c takes items c + k * grid
    const int64_t ni = in.n_items, fg = P.fused_grid;
    const char* fname = P.fused_kernel == SCAN_PATH_WP_CTR ? "ctr" : P.fused_kernel == SCAN_PATH_TILE ? "tile" : "v2";
    const int64_t per = P.fused_kernel == SCAN_PATH_WP_CTR ? ni / (fg * (int64_t)P.WC.warps) : P.fused_kernel == SCAN_PATH_TILE ? ni / fg : -1;
    std::printf("fused_kernel=%s\nfused_grid=%lld\nitems_per_warp=%lld\n", fname, (long long)fg, (long long)per);
  }
  return 0;
}
