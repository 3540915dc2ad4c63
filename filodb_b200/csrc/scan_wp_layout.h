// Shared-memory layout of the v4 warp-pipeline kernel (scan_wp.cuh); plain structs, usable from host code.
#pragma once
#include <stdint.h>
#include "filo_record.h"
#include "scan_params.h"
#include "scan_tile_layout.h"
namespace filo {
constexpr int WP_MAXC = 4;             // chunks in range per series on this path
constexpr int WP_MAXG = 64;            // NibblePack groups per series (two per lane)
constexpr int WP_R = 8;                // windows per block
constexpr int WP_MAX_WARPS = 16;       // warps per CTA (one CTA per SM) when O has its own region
constexpr int WP_MAX_WARPS_ALIAS = 20; // ... when O takes V's place (single-pass plans): 20 warps = 96 registers per thread (22 = 88 registers, spills)

struct WpChunk {                       // per warp, per chunk in range (shared memory)
  uint64_t first;                      // XOR vectors: bits of the first value
  int32_t kT0, kT1;                    // windows whose (unclamped) row range meets the chunk's rows, clipped to [0, T)
  int32_t ownLo, ownHi;                // ... of which only this chunk contributes to [ownLo, ownHi]
  int32_t blk0, nblk;                  // block items of this chunk: [blk0, blk0 + nblk)
  int32_t vidx0;                       // V index of the first row of block 0
  int32_t rowpos;                      // V position (before skewing) of row 0
  int32_t nrows, s0, e0;               // rows; unclamped first / last row of window 0
  int32_t grp_base, ng, wire;          // group slots [grp_base, grp_base + ng)
  uint32_t grp_off, tab_off, val_off;  // byte offsets in R: first group, u16 group table, value vector
  int32_t joff, hs;                    // head share: windows [kT0, ownLo) also take rows from the previous chunk
  int32_t jzb, tb;                     // blocks [0, jzb) (the head share rounded up to whole blocks) leave their raw sums at J[joff ..]; blocks [tb, nblk)
                                       // (from the block that holds ownHi + 1) leave raw sums in O; the blocks in between hold own windows only
  int32_t dropped;                     // counter drop flag of the value vector (PrimitiveVectorReader.dropped, BinaryVector.scala:530-531)
};
static_assert(sizeof(WpChunk) == 96, "WpChunk");

// fixed part of a warp's region: mbarrier, descriptors, J -- compile-time offsets keep the kernel's address arithmetic in immediates
constexpr uint32_t WP_OFF_DESC = 16, WP_OFF_J = WP_OFF_DESC + WP_MAXC * 96, WP_J_DOUBLES = 128, WP_OFF_REC = WP_OFF_J + WP_J_DOUBLES * 8;
struct WpSmem {                        // byte offsets inside a warp's region, all multiples of 16
  uint32_t desc, jbuf, rec, vals, out, per_warp;
  uint32_t rec_cap, vcap /*doubles*/, jcap /*doubles*/, ocap /*doubles*/;
  uint32_t warps;                      // warps per CTA
  uint32_t alias;                      // O lives in V's region: every block of a series is summed (one pass of <= 64 blocks) before the first result is stored
  uint32_t rec2;                       // second record buffer (0: one): the records of the warp's next two series are in flight
};
// wrows = window / step + 1: the most rows a window can span
FILO_HD inline WpSmem wp_layout(uint32_t max_rec_bytes, uint32_t max_rows, uint32_t max_chunks, uint32_t T, uint32_t wrows, bool alias, bool two_rec = false) {
  WpSmem L;
  if (max_chunks > (uint32_t)WP_MAXC) max_chunks = WP_MAXC;
  L.rec_cap = align_up(max_rec_bytes + 16, 16);
  const uint32_t P = max_rows + (max_chunks + 1) * (wrows + 7) + 16;         // positions: rows + zero gaps + slack
  L.vcap = align_up(P + P / 8 + 2, 2);
  L.jcap = WP_J_DOUBLES;               // raw sums of the windows two chunks share (a plan that needs more is declined); also the XOR prefix table of the decode (64 words)
  (void)wrows;
  L.ocap = align_up(T + T / 8 + 4, 2);                                       // skewed like V: one pad slot per 8 windows
  if (alias && L.vcap < L.ocap) L.vcap = L.ocap;
  static_assert(sizeof(WpChunk) == 96, "WP_OFF_J");
  uint32_t o = WP_OFF_REC;
  L.desc = WP_OFF_DESC; L.jbuf = WP_OFF_J;
  L.rec = o; o += L.rec_cap;
  L.rec2 = 0;
  if (two_rec) { L.rec2 = o; o += L.rec_cap; }
  L.vals = o; o += L.vcap * 8;
  if (alias) L.out = L.vals; else { L.out = o; o += L.ocap * 8; }
  L.per_warp = align_up(o, 16);
  L.warps = 0;
  L.alias = alias ? 1u : 0u;
  return L;
}

// SUM-class kernel with a CTA-wide record stream (scan_wp_batch_kernel): 15 consumer warps and 1 producer warp (16 warps x 128 registers).
// The producer fetches batches of WP_BATCH_SERIES consecutive records into WP_BATCH_BUFS batch buffers: 30 records per CTA, the record
// bytes of two buffers per warp at 15 warps.  On C2, 15 x 2 ran 4 % faster than 5 x 6 (DESIGN §4.1).
constexpr int WP_BATCH_WARPS = 16;
constexpr int WP_BATCH_SERIES = 15;
constexpr int WP_BATCH_BUFS = 2;
struct WpEntryChunk {                  // what the producer's header parse found of one chunk in range (zero for chunks c >= n)
  uint64_t first;                      // XOR: bits of the first value; raw f64: the first value
  int64_t init, end_time;              // with nrows and wire: the memo key of the window plan
  uint32_t grp_off, val_off;           // byte offsets in the record: first group (XOR), value vector
  int32_t nrows, grp_base, ng;         // rows, group slots [grp_base, grp_base + ng)
  uint32_t wire;                       // value vector wire | drop flag << 16
};
static_assert(sizeof(WpEntryChunk) == 48, "WpEntryChunk");
struct WpEntry {                       // one series of a batch (shared memory, written by the producer, read by one consumer warp)
  uint32_t rofs;                       // the record's byte offset in the batch buffer
  int32_t n;                           // chunks in range
  int32_t flags;                       // bit 0: regular as far as the header goes (wp_parse), bit 1: a chunk has raw f64 values
  int32_t ngroups, cnt_rows, cnt_bytes;   // NibblePack groups; the series' scan counters
  int32_t pad[2];
  WpEntryChunk c[WP_MAXC];
};
static_assert(sizeof(WpEntry) == 224, "WpEntry");
struct WpBatchSmem {                   // byte offsets inside the CTA's shared memory, all multiples of 16
  WpSmem W;                            // a consumer warp's region: wp_layout without record buffers (V at WP_OFF_REC)
  uint32_t B, nbuf, consumers;         // series per batch, batch buffers, consumer warps (the producer is warp `consumers`)
  uint32_t buf, buf_stride, buf_cap;   // batch buffer b at buf + b * buf_stride; a batch is staged when its records take <= buf_cap bytes
  uint32_t ent;                        // WpEntry[nbuf][B]
  uint32_t bars;                       // mbarriers full[nbuf], parsed[nbuf], empty[nbuf]
  uint32_t total;                      // bytes per CTA
  uint32_t rt, rtcap;                  // raw tail area of a warp's region (byte offset, doubles): the raw sums of every chunk's blocks from tb on,
                                       // behind the dense result row in O (windows [0, T) at O[h .. T - 1 + h], h <= 1)
};
FILO_HD inline WpBatchSmem wp_batch_layout(uint32_t max_rec_bytes, uint32_t max_rows, uint32_t max_chunks, uint32_t T, uint32_t wrows, bool alias,
                                           uint32_t B = WP_BATCH_SERIES, uint32_t nbuf = WP_BATCH_BUFS, uint32_t consumers = WP_BATCH_WARPS - 1) {
  WpBatchSmem S;
  WpSmem L = wp_layout(max_rec_bytes, max_rows, max_chunks, T, wrows, alias);
  const uint32_t shift = L.vals - WP_OFF_REC;                                 // the record buffer leaves the warp's region
  L.vals -= shift; L.out -= shift; L.per_warp -= shift; L.rec = 0;
  // raw tail area: a chunk followed by another leaves raw sums in its blocks [tb, nblk), at most (Wr - 1) / 8 + 2 blocks with
  // Wr <= wrows - 1 (at most Wr windows take rows from both chunks).  O's region grows only where T + 1 + rtcap exceed it; vcap (what
  // the plan checks V against) stays as it is
  const uint32_t mc = max_chunks < (uint32_t)WP_MAXC ? max_chunks : (uint32_t)WP_MAXC;
  S.rtcap = mc > 1 ? (uint32_t)WP_R * (mc - 1) * ((wrows + 14) / 8) : 0;
  S.rt = L.out + 8 * (T + 1);
  { const uint32_t oreg = alias ? L.vcap : L.ocap, need = T + 1 + S.rtcap;
    L.per_warp = align_up(L.out + 8 * (oreg > need ? oreg : need), 16); }
  S.consumers = consumers;
  L.warps = S.consumers;
  S.W = L; S.B = B; S.nbuf = nbuf;
  uint32_t o = L.per_warp * S.consumers;
  S.buf = o;
  S.buf_cap = B * align_up(max_rec_bytes, 16);                                // records are 16-byte aligned and adjacent in the arena
  S.buf_stride = S.buf_cap + 16;                                              // (the group decode reads up to 8 bytes past a record)
  o += nbuf * S.buf_stride;
  S.ent = o; o += nbuf * B * (uint32_t)sizeof(WpEntry);
  S.bars = o; o += 3 * nbuf * 8;
  S.total = align_up(o, 16);
  return S;
}

// an upper bound of the blocks of a series: sum over chunks of ceil(touched windows / 8), with at most wrows - 1 windows shared per junction
FILO_HD inline uint32_t wp_max_items(uint32_t max_chunks, uint32_t T, uint32_t wrows) {
  if (max_chunks > (uint32_t)WP_MAXC) max_chunks = WP_MAXC;
  if (max_chunks == 0) max_chunks = 1;
  return (T + (max_chunks - 1) * (wrows - 1) + 7 * max_chunks) / 8;
}

constexpr int WP_CTR_MAX_WARPS = 20;   // counter kernel: warps per CTA at the lower register budget
// TileCtr: per-chunk constants of the extrapolation for windows whose rows lie inside the chunk and are not clamped
// (RateFunctions.scala:72-111 with every window-invariant subexpression evaluated once).
struct TileCtr {
  double dTS, thr, half, endpart, sI, ratio0, skipC;   // see the plan in scan_wp_ctr.cuh for the definitions
  int32_t dropped, pad;
};
// TileDrops: counter drops of a drop-flagged chunk, found while its rows are decoded
// (CorrectingDoubleVectorReader.corrected, DoubleVector.scala:325-342): row position and the amount added to the correction
constexpr int TILE_MAXDROP = 8;
// per-query table of the extrapolation terms that depend only on (numSamples - 1) = m when the samples are m steps apart
constexpr int TILE_CTR_TABMAX = 64;
struct TileCtrTab { double sI, thr, half, rcpSI; };      // sampledInterval, 1.1 * average interval, average / 2, RN(1 / sI)
struct TileDrops {
  int32_t n, pos[TILE_MAXDROP], pad[3];
  double amt[TILE_MAXDROP];
};
struct WpCtrChunk {                    // per warp, per chunk in range: plan (window intervals, extrapolation constants)
  int64_t init, end_time;
  int32_t nrows, s0, e0, rowpos;
  int32_t kA, kB;                      // unclamped single-chunk windows with at least two samples ([0, -1] if none)
  int32_t kA2, kB2;                    // every single-chunk window of the chunk, clamped ones included
  TileCtr kc;                          // per-series: kc.dropped
};
static_assert(sizeof(WpCtrChunk) == 112, "WpCtrChunk");

struct WpCtrSmem {                     // byte offsets inside a warp's region (multiples of 16); R sits at WP_OFF_REC, xtab at WP_OFF_J, drops behind it
  uint32_t vals, kc, acc, nbad, per_warp, tab /* per CTA, behind the warps' regions */;
  uint32_t rec_cap, vcap /*doubles*/, warps, agg;
  uint32_t tsr;                        // irregular timestamps: int32 row times relative to the chunk's first (0: the table has const-DDV timestamps only)
};
constexpr uint32_t WP_OFF_DROPS = WP_OFF_J + 64 * 8;          // TileDrops[WP_MAXC] behind the 64-word XOR prefix table
static_assert(WP_OFF_DROPS + WP_MAXC * sizeof(TileDrops) <= WP_OFF_REC, "drops fit in front of the record");
FILO_HD inline WpCtrSmem wp_ctr_layout(uint32_t max_rec_bytes, uint32_t max_rows, uint32_t max_chunks, uint32_t T, bool agg, bool irr = false,
                                       bool moments = false) {
  WpCtrSmem L;
  if (max_chunks > (uint32_t)WP_MAXC) max_chunks = WP_MAXC;
  L.rec_cap = align_up(max_rec_bytes + 16, 16);
  const uint32_t P = max_rows + 8 * max_chunks + 8;            // 8 spare rows behind every chunk: the group decode runs up to 7 rows past it
  L.vcap = align_up(P + P / 8 + 2, 2);
  uint32_t o = WP_OFF_REC + L.rec_cap;
  L.vals = o; o += L.vcap * 8;
  L.kc = o; o += (uint32_t)(WP_MAXC * sizeof(WpCtrChunk));
  L.tsr = 0;
  if (irr) { L.tsr = o; o += align_up(P * 4, 16); }
  L.acc = o; L.nbad = o;
  if (agg) { o += T * 8; L.nbad = o; o += align_up(T * 2, 16); }
  if (agg && moments) o += T * 8;      // stddev / stdvar: the [T] Σv² row at nbad + align_up(T * 2, 16)
  L.per_warp = align_up(o, 16);
  L.tab = 0; L.warps = 0; L.agg = agg ? 1u : 0u;
  return L;
}
// The counter kernel takes a table only when eight of its series, staged the way the round-1 tile kernel staged counter tables
// (tile_layout plus per-chunk extrapolation constants, drop lists and the extrapolation table), fit in `cap` bytes: the selection
// this kernel was measured under.  Lifting the bound would move large-record counter tables from the v2 kernel to this one, a
// speed change to be measured on its own.
FILO_HD inline bool wp_ctr_tile_footprint_ok(uint32_t max_rec_bytes, uint32_t max_rows, uint32_t T, uint64_t cap) {
  const uint32_t ctr = 2 * align_up(TILE_NS * TILE_MAXC * (uint32_t)sizeof(TileCtr), 128) + align_up(TILE_NS * TILE_MAXC * (uint32_t)sizeof(TileDrops), 128) +
                       align_up((TILE_CTR_TABMAX + 1) * (uint32_t)sizeof(TileCtrTab), 128);
  return (uint64_t)(tile_layout(max_rec_bytes, max_rows, T, 0).total + ctr) + 1024 <= cap;
}

// ---- the per-series kernel a query runs in front of the v2 kernel (filo_query); the v2 kernel takes what that kernel declines
enum { SCAN_PATH_V2 = 0, SCAN_PATH_TILE = 1, SCAN_PATH_WP_SUM = 2, SCAN_PATH_WP_BATCH = 3, SCAN_PATH_WP_CTR = 4 };
struct ScanPathIn {
  uint32_t max_rec_bytes, max_rows, max_chunks, T;   // the table's largest record, rows and chunks per series; windows
  uint64_t wrows;                      // window / step + 1
  int fn_cls;                          // fn_class_of
  bool fused, moments;                 // an across-series aggregate folded in the scan kernels; stddev / stdvar
  bool irr;                            // the table has series whose timestamps are not const-DDV
  bool v2;                             // the v2 kernel takes the table (its per-warp working set fits)
  int force;                           // FILO_KERNEL: 2 keeps every class on v2, 3 keeps the SUM class on the tile kernel; 0 otherwise
  uint64_t smem_cap;                   // shared memory one CTA may opt into
  int64_t n_series;
  int64_t n_items;                     // work items of the table's grouping (build_groups_new): the fused kernels' work
  int sm_count;
};
struct ScanPath {
  int kernel;                          // SCAN_PATH_*: the per-series kernel
  bool tile, wp, wp_batch, wp_ctr;     // tile: the tile layout fits (it also serves fused SUM-class aggregates); the v4 kernels in front of it
  bool refused;                        // the batch kernel with O on V and plans of more than one pass: the query is refused
  int tile_ctas_per_sm;
  int grid;                            // CTAs of the per-series kernel (persistent: at most one per SM for the v4 kernels)
  int fused_kernel;                    // fused aggregates: SCAN_PATH_WP_CTR or SCAN_PATH_TILE in front of the v2 aggregate kernel, or
                                       // SCAN_PATH_V2 (the v2 / v1 aggregate kernel alone)
  int fused_grid;                      // CTAs of the fused ctr / tile kernel (items are strided over warps / CTAs); 0 for SCAN_PATH_V2
  TileSmem TL; WpSmem WL; WpBatchSmem WB; WpCtrSmem WC;
};
FILO_HD inline ScanPath scan_path(const ScanPathIn& in) {
  ScanPath P{};
  P.kernel = SCAN_PATH_V2;
  const uint32_t T = in.T, wrows = (uint32_t)in.wrows;
  // v3 tile kernel (scan_tile.cuh): SUM-class functions over regular series.  Zero rows around a chunk let clamped windows run without
  // bounds checks: a window spans at most window/step + 1 rows at either end; when that does not leave room for two CTAs per SM the
  // tile kernel falls back to checked loads.
  if (in.v2 && in.force != 2 && in.fn_cls == CLASS_SUM && in.n_series > 0) {
    P.TL = tile_layout(in.max_rec_bytes, in.max_rows, T, (uint32_t)(2 * in.wrows < (1u << 20) ? 2 * in.wrows : (1u << 20)) + 16);
    if (((uint64_t)P.TL.total + 1024) * 2 > (uint64_t)228 * 1024) P.TL = tile_layout(in.max_rec_bytes, in.max_rows, T, 16);
    P.tile = (uint64_t)P.TL.total + 1024 <= in.smem_cap;
  }
  P.tile_ctas_per_sm = ((uint64_t)P.TL.total + 1024) * 2 <= (uint64_t)228 * 1024 ? 2 : 1;
  // v4 SUM kernel (scan_wp.cuh): per-series rows, in front of the tile kernel
  if (P.tile && in.force != 3 && in.wrows <= 4096 && in.max_chunks > 0) {
    // O in V's place (more warps per SM) when every series is summed in one pass of <= 64 blocks
    const bool alias = wp_max_items(in.max_chunks, T, wrows) <= 64;
    P.WL = wp_layout(in.max_rec_bytes, in.max_rows, in.max_chunks, T, wrows, alias);
    { const uint64_t w = in.smem_cap / P.WL.per_warp, wmax = alias ? WP_MAX_WARPS_ALIAS : WP_MAX_WARPS; P.WL.warps = (uint32_t)(w < wmax ? w : wmax); }
    // two record buffers per warp (the records of the next two series in flight) when 16 warps of them fit
    const WpSmem WL2 = wp_layout(in.max_rec_bytes, in.max_rows, in.max_chunks, T, wrows, alias, true);
    if (in.smem_cap / WL2.per_warp >= (uint64_t)WP_MAX_WARPS) {
      P.WL = WL2; P.WL.warps = WP_MAX_WARPS;
      // that layout's record bytes as one CTA-wide stream: batches of consecutive records, a producer warp parses their headers.  Its
      // layout adds the raw tail area behind the result row (no bytes for C2: the row and the area fit in V's region); where that does
      // not fit, the table stays on scan_wp_sum_kernel with two record buffers per warp
      P.WB = wp_batch_layout(in.max_rec_bytes, in.max_rows, in.max_chunks, T, wrows, alias);
      P.wp_batch = P.WB.total <= in.smem_cap;
      // the batch kernel's window blocks write finished windows over O right after the pass's reads of V: with O on V every plan must be
      // one pass of at most 64 blocks
      if (P.wp_batch && P.WB.W.alias && wp_max_items(in.max_chunks, T, wrows) > 64) P.refused = true;
    }
    P.wp = P.WL.warps >= 4;
  }
  // v4 counter-class kernel (scan_wp_ctr.cuh): per-series rows, or fused partial rows of up to TILE_AGG_ACC * TILE_THREADS windows
  if (in.v2 && in.force != 2 && in.force != 3 && in.fn_cls == CLASS_COUNTER && in.n_series > 0 && in.max_chunks > 0 &&
      (!in.fused || T <= (uint32_t)(TILE_AGG_ACC * TILE_THREADS)) && wp_ctr_tile_footprint_ok(in.max_rec_bytes, in.max_rows, T, in.smem_cap)) {
    P.WC = wp_ctr_layout(in.max_rec_bytes, in.max_rows, in.max_chunks, T, in.fused, in.irr, in.moments);
    // the irregular-timestamp instantiation is built for <= 16 warps
    const uint64_t w = (in.smem_cap - sizeof(TileCtrTab) * (TILE_CTR_TABMAX + 1) - 64) / P.WC.per_warp, wmax = P.WC.tsr != 0 ? 16 : WP_CTR_MAX_WARPS;
    P.WC.warps = (uint32_t)(w < wmax ? w : wmax); P.WC.tab = (uint32_t)(P.WC.per_warp * P.WC.warps);
    P.wp_ctr = P.WC.warps >= 4;
  }
  // the per-series kernel and its grid
  const int64_t n = in.n_series, sms = in.sm_count;
  int64_t g = 1;
  if (P.wp_batch)    { P.kernel = SCAN_PATH_WP_BATCH; g = (n + P.WB.B - 1) / P.WB.B; if (g > sms) g = sms; }
  else if (P.wp)     { P.kernel = SCAN_PATH_WP_SUM;   g = (n + P.WL.warps - 1) / P.WL.warps; if (g > sms) g = sms; }
  else if (P.wp_ctr) { P.kernel = SCAN_PATH_WP_CTR;   g = (n + P.WC.warps - 1) / P.WC.warps; if (g > sms) g = sms; }
  else if (P.tile)   { P.kernel = SCAN_PATH_TILE;     g = (n + TILE_NS - 1) / TILE_NS; if (g > sms * P.tile_ctas_per_sm) g = sms * P.tile_ctas_per_sm; }
  P.grid = (int)(g > 1 ? g : 1);
  // the fused kernel and its grid: the counter kernel folds warp gw's items gw, gw + warps * grid, ..; the tile kernel CTA c's items
  // c, c + grid, ..; the tile kernel's accumulators hold TILE_AGG_ACC * TILE_THREADS windows
  const int64_t ni = in.n_items;
  P.fused_kernel = SCAN_PATH_V2; P.fused_grid = 0;
  if (P.wp_ctr) {
    P.fused_kernel = SCAN_PATH_WP_CTR; g = (ni + P.WC.warps - 1) / P.WC.warps; if (g > sms) g = sms; P.fused_grid = (int)(g > 1 ? g : 1);
  } else if (P.tile && T <= (uint32_t)(TILE_AGG_ACC * TILE_THREADS)) {
    P.fused_kernel = SCAN_PATH_TILE; g = ni; if (g > sms * P.tile_ctas_per_sm) g = sms * P.tile_ctas_per_sm; P.fused_grid = (int)(g > 1 ? g : 1);
  }
  return P;
}

} // namespace filo
