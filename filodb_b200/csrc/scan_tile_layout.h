// Shared-memory layout of the v3 tile kernel (scan_tile.cuh); plain structs, usable from host code.
#pragma once
#include <stdint.h>
#include "filo_record.h"
#include "scan_params.h"
namespace filo {
constexpr int TILE_NS = 8;               // series per tile (even: keeps the bulk store 16-byte aligned for odd T)
constexpr int TILE_THREADS = 256;        // consumer threads (decode + windows)
constexpr int TILE_LAUNCH_THREADS = TILE_THREADS + 32;   // + one producer warp (tile load, per-series setup of the next tile)
constexpr int TILE_MAXC = 4;             // chunks in range per series on the fast path
constexpr int TILE_AGG_ACC = 2;           // fused aggregate: per-thread accumulators -> T <= TILE_AGG_ACC * TILE_THREADS windows
constexpr int TILE_MAXG = 64;            // NibblePack groups per series on the fast path (64 * 8 = 512 rows)
// pitches (in 8-byte words) of the cross-warp XOR exchange tables: lane = series + 8 * k stores slot 8 * warp + k of series
// `series`; a pitch of 2 (mod 16) puts the 16 lanes of a half-warp into 16 different bank pairs, 9 does the same for [series][warp]
constexpr int TILE_GX_PITCH = TILE_MAXG + 2, TILE_GW_PITCH = 9;

struct TileChunk {
  int64_t init, end_time;
  uint64_t first;             // XOR vectors: bits of the chunk's first value
  int32_t nrows, row_base;
  int32_t kA, kB, sA, Wr;
  uint32_t val_off; int32_t wire;
  uint32_t grp_off, tab_off;  // XOR vectors: byte offsets (in the staged tile) of the first group / of the u16 group table
  int32_t ngroups, grp_base;
  int32_t blk0, blk_n;
  int32_t s0, e0;             // unclamped first / last row of window k = 0 (rows advance by one per window)
  int32_t lowz, highz;        // zero rows before / after the chunk's rows (clamped windows read them as +0.0)
  // unused: the descriptors keep their size, and with it tile_layout's footprint, which decides what this kernel and the v4 SUM
  // kernel admit (filo_query)
  int32_t spare[8];
};
static_assert(sizeof(TileChunk) == 128, "TileChunk");
struct TileSeries {
  int32_t n, regular, rec_off, nblocks, nrest, ngroups, nrows, any_raw;
  int64_t sid;                // series ordinal in the table
  int32_t cnt_rows, cnt_bytes; // rows / vector bytes of the chunks the window iterator pulls (scan counters)
  int32_t gb[TILE_MAXC];      // grp_base of chunk c (INT_MAX for c >= n): chunk of a group slot = #{c >= 1 : gb[c] <= slot}
  TileChunk c[TILE_MAXC];
};

struct TileMeta {                         // per-tile work-list prefixes and flags
  int32_t pref[TILE_NS + 1];              // blocked work items per series (prefix)
  int32_t rpref[TILE_NS + 1];             // other windows per series (prefix)
  int32_t any_nan, any_raw, all_regular, all_padded;
  int32_t staged, ns; int64_t i0;
};

struct TileSmem {                         // byte offsets inside dynamic shared memory (all multiples of 128)
  uint32_t rec, vals, out, desc, gtot, meta, total;
  uint32_t rec_cap, vals_pitch /*doubles per series*/, out_pitch /*doubles per series = T*/, desc_stride /*bytes between the two descriptor buffers*/;
};
FILO_HD inline TileSmem tile_layout(uint32_t max_rec_bytes, uint32_t max_rows, uint32_t T, uint32_t pad_rows) {
  TileSmem L;
  L.rec_cap = align_up(TILE_NS * max_rec_bytes + 128, 128);
  L.desc_stride = align_up(TILE_NS * (uint32_t)sizeof(TileSeries), 128);
  L.vals_pitch = (max_rows + pad_rows + 2 + 1) | 1;            // odd pitch (doubles); pad_rows: zero rows for clamped windows
  L.out_pitch = T;
  uint32_t o = 128;                                            // mbarrier slot
  L.rec = o; o += L.rec_cap;
  L.vals = o; o += align_up(TILE_NS * L.vals_pitch * 8, 128);
  L.out = o; o += align_up(TILE_NS * T * 8, 128);
  L.desc = o; o += 2 * align_up(TILE_NS * (uint32_t)sizeof(TileSeries), 128);      // double-buffered: setup of tile t+1 overlaps tile t
  L.gtot = o; o += align_up(TILE_NS * TILE_GX_PITCH * 8 + TILE_NS * TILE_GW_PITCH * 8, 128);     // per-slot in-warp prefixes + per-warp totals (padded pitches)
  L.meta = o; o += 2 * 128;
  L.total = o;
  return L;
}

} // namespace filo
