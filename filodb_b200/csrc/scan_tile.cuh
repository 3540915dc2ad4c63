// v3 scan path: CTA-tile kernel for the SUM class (sum / avg / count_over_time, rate / increase on delta schemas) over regular series.
// It serves the fused across-series aggregates (the v4 kernel of scan_wp.cuh has no aggregate mode) and the per-series queries the v4
// SUM kernel turns away (windows over more than 4096 rows, fewer than 4 warps in shared memory).
//
// A CTA processes tiles of TILE_NS consecutive series.  Records of consecutive series are adjacent in the arena, so a tile's
// chunk pages arrive with ONE cp.async.bulk (TMA) into shared memory, and the tile's [TILE_NS x T] results leave with ONE
// cp.async.bulk store.  Between the two, all 256 threads work on uniform work items:
//   setup    warp w resolves series w, lane = (chunk, quantity): chunk range, regularity, single-chunk window intervals
//            (same definition as scan_fast.cuh chunk_interval, three divisions per chunk)
//   decode   item = (series, NibblePack group), two items per thread held in registers: branch-free field extraction +
//            local XOR prefix, group totals combined inside the warp, warp totals exchanged through shared memory, then the
//            finished values are stored once.  Raw f64 vectors are copied.  NaN/Inf presence is recorded.
//   windows  item = (series, block of BLK_R single-chunk windows): register-blocked sequential sums (exact reference order);
//            item = (series, other window): literal per-chunk fold for windows that take rows from two chunks.
// A series is "regular" when every chunk in range has const-DDV timestamps with slope == step and XOR/raw double values,
// with at most TILE_MAXC chunks and TILE_MAXG NibblePack groups; anything else is appended to a fallback list that the
// generic v2 kernel processes afterwards (same output buffer), so the result is always complete and identical.
#pragma once
#include "scan_fast.cuh"
#include "scan_tile_layout.h"

namespace filo {

// bulk store shared -> global (one bulk group): both addresses 16-byte aligned, size a nonzero multiple of 16 (checked on the emulator)
#ifdef FILO_CUSIM
inline void tma_store_1d(void* gdst, const void* ssrc, uint32_t bytes) {
  if ((reinterpret_cast<uintptr_t>(gdst) & 15) || (reinterpret_cast<uintptr_t>(ssrc) & 15) || bytes == 0 || (bytes & 15)) {
    std::fprintf(stderr, "cusim: bulk store of %u bytes from %p to %p: needs 16-byte alignment and a nonzero multiple of 16 bytes\n", bytes, ssrc, gdst);
    std::abort();
  }
  cusim::tma_store(gdst, ssrc, bytes);
}
inline void tma_store_wait_read() { cusim::tma_store_wait_read(); }
inline void tma_store_wait_all() { cusim::tma_store_wait_read(); }
inline void fence_async_smem() {}
#else
__device__ __forceinline__ void tma_store_1d(void* gdst, const void* ssrc, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(ssrc)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
#endif

// Per-phase cycle counters of the consumer side for profiling builds (-DFILO_TILE_PROF; scratch/tile_prof.py): lane 0 of every
// consumer warp reads clock64() at the phase boundaries of a tile, summed over warps and CTAs.  Compiled out of the product build.
#if defined(FILO_TILE_PROF) && !defined(FILO_CUSIM)
__device__ unsigned long long g_tile_prof[16];
#define TPROF_DECL long long tp_t0 = clock64(), tp_acc[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
#define TPROF(i) { const long long tp_t1 = clock64(); tp_acc[i] += tp_t1 - tp_t0; tp_t0 = tp_t1; }
#define TPROF_FLUSH if (lane == 0) { for (int tp_i = 0; tp_i < 10; ++tp_i) atomicAdd(&g_tile_prof[tp_i], (unsigned long long)tp_acc[tp_i]); atomicAdd(&g_tile_prof[15], 1ull); }
#else
#define TPROF_DECL
#define TPROF(i)
#define TPROF_FLUSH
#endif

// compile-time specialised finish of one single-chunk window (SumFinish of scan_fast.cuh with FN known)
template <int FN>
__device__ __forceinline__ double tile_finish(double cs, int nn, double div, double rcp) {
  const double NaNv = __longlong_as_double(0x7ff8000000000000LL);
  if (FN == FN_COUNT) return (double)nn;
  const double sum = nn ? cs : NaNv;
  if (FN == FN_RATE) return __dmul_rn(div_invariant(sum, div, rcp), 1000.0);
  if (FN == FN_AVG) return nn > 0 ? sum / (double)nn : sum;            // AggrOverTimeFunctions.scala:1000
  return sum;                                                          // FN_SUM, FN_INCREASE (delta schema)
}

// literal per-chunk fold for one window of a regular series (TimeRangeFunction family on const-DDV timestamps):
// chunk-set membership ChunkSetInfo.scala:481-510, row range RangeFunction.scala:185-190, fold AggrOverTimeFunctions.scala:560-571.
// Rows advance one per window, so the unclamped row range of window k is [s0 + k, e0 + k] (no search, no division).
template <int FN, bool CHECK_NAN>
__device__ __forceinline__ double tile_eval_window(const TileSeries& S, const double* vals, int64_t wStart, int64_t wEnd, double div, int k) {
  const double NaNv = __longlong_as_double(0x7ff8000000000000LL);
  double sum = NaNv; int cnt = 0; bool anyrows = false;
  for (int c = 0; c < S.n; ++c) {
    const TileChunk& ch = S.c[c];
    bool member = !(ch.end_time < wStart);
    if (c > 0 && !(S.c[c - 1].end_time < wEnd)) member = false;
    int su = ch.s0 + k; if (su < 0) su = 0;
    int eu = ch.e0 + k; if (eu > ch.nrows - 1) eu = ch.nrows - 1;
    if (!member || su > eu) continue;
    const double* v = vals + ch.row_base;
    double cs = 0.0; int nn = 0;
    if (CHECK_NAN) { for (int r = su; r <= eu; ++r) { const double x = v[r]; if (x == x) { cs += x; ++nn; } } }
    else { for (int r = su; r <= eu; ++r) cs += v[r]; nn = eu - su + 1; }
    anyrows = true;
    const double csn = nn ? cs : NaNv;
    if (nn && sum != sum) sum = 0.0;
    sum += csn; cnt += nn;
  }
  if (FN == FN_RATE) return sum / div * 1000.0;
  if (FN == FN_AVG) return cnt > 0 ? sum / (double)cnt : (sum != sum ? sum : 0.0);
  if (FN == FN_COUNT) return anyrows ? (double)cnt : NaNv;
  return sum;
}

__device__ __forceinline__ uint64_t shfl_u64(uint64_t v, int src) { return (uint64_t)__shfl_sync(0xffffffffu, (unsigned long long)v, src); }
__device__ __forceinline__ uint64_t shfl_up_u64(uint64_t v, int d) { return (uint64_t)__shfl_up_sync(0xffffffffu, (unsigned long long)v, d); }

// ---------------------------------------------------------------------------------------------------------------------
// Tile kernel: sum/avg/count_over_time, rate/increase on delta schemas.  AGG: fused across-series aggregate (partial rows).
// MOM (with AGG, agg_op = AGG_SUM): stddev / stdvar moments, a second register accumulator of Σv² per window, its partial rows
// at pval + n_items * T.
// ---------------------------------------------------------------------------------------------------------------------
template <int FN, bool AGG, bool MOM = false>
__global__ void __launch_bounds__(TILE_LAUNCH_THREADS, 2)
scan_tile_kernel(const uint8_t* __restrict__ arena, const int64_t* __restrict__ rec_off, int64_t n_series,
                     QueryParams q, double* __restrict__ out, TileSmem L,
                     int64_t* __restrict__ fallback_list, unsigned long long* __restrict__ fallback_count,
                     unsigned long long* d_counters, int* d_err,
                     const int32_t* __restrict__ order, const int64_t* __restrict__ item_begin, int64_t n_items, int agg_op,
                     double* __restrict__ pval, uint32_t* __restrict__ pcnt) {
  static_assert(TILE_NS == 8 && TILE_THREADS == 256 && TILE_MAXC == 4 && TILE_MAXG == 64, "item mappings below assume this shape");
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const bool producer = warp == TILE_THREADS / 32;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem);
  uint8_t* recbuf = smem + L.rec;
  double* vals = reinterpret_cast<double*>(smem + L.vals);
  double* otile = reinterpret_cast<double*>(smem + L.out);
  uint64_t* gexcl = reinterpret_cast<uint64_t*>(smem + L.gtot);        // [series][slot]: XOR of the warp's earlier group totals
  uint64_t* gwtot = gexcl + TILE_NS * TILE_GX_PITCH;                       // [series][warp]: XOR of the warp's 8 group totals
  // Tile walk.  Work items are strided over the CTAs; an item is a run of consecutive positions processed in tiles of
  // TILE_NS.  Per-series mode: item = one tile of consecutive series.  AGG mode: item = <= seg series of ONE group in
  // group-sorted order (positions index `order`), folded into one partial row per item (pval/pcnt, see scan_agg_kernel).
  const int64_t n_work = AGG ? n_items : (n_series + TILE_NS - 1) / TILE_NS;
  struct Walk { int64_t it, pb, pe; };
  auto item_range = [&](Walk& w) {
    if (AGG) { w.pb = item_begin[w.it]; w.pe = item_begin[w.it + 1]; }
    else { w.pb = w.it * TILE_NS; w.pe = w.pb + TILE_NS < n_series ? w.pb + TILE_NS : n_series; }
  };
  auto walk_seek = [&](Walk& w) -> bool { while (w.it < n_work) { item_range(w); if (w.pb < w.pe) return true; w.it += gridDim.x; } return false; };
  auto walk_start = [&](Walk& w) -> bool { w.it = blockIdx.x; return walk_seek(w); };
  auto walk_next = [&](Walk& w) -> bool { w.pb += TILE_NS; if (w.pb < w.pe) return true; w.it += gridDim.x; return walk_seek(w); };
  uint64_t* ready = bar + 1;            // ready[b]: descriptors of the tile in buffer b are complete (producer -> consumers)
  if (tid == 0) { mbar_init(bar, 1); mbar_init(ready, 1); mbar_init(ready + 1, 1); mbar_fence_init(); }
  __syncthreads();
  int64_t winDur = q.inclusive ? q.window : q.window - 1; if (winDur < 0) winDur = 0;
  const double fdiv = (double)(q.inclusive ? winDur : winDur + 1), frcp = 1.0 / fdiv;     // RateFunctions.scala:436-442
  const int64_t S0 = q.start - winDur, E0 = q.start;
#ifdef FILO_CUSIM
  auto bar_consumers = [] { cusim::bar_sync(1, TILE_THREADS); };
#else
  auto bar_consumers = [] { asm volatile("bar.sync 1, %0;" ::"n"(TILE_THREADS) : "memory"); };
#endif
  // Per tile: A = "descriptors of the tile are ready" (producer -> consumers, an mbarrier), B = "the tile's record bytes are
  // dead" (a CTA-wide barrier: consumers -> producer, the staging buffer may be refilled; decode -> windows among consumers).  The producer warp
  // loads and resolves tile t+1 while the consumers reduce the windows of tile t.

  if (producer) {
    // ================================================================== producer warp: tile load + per-series setup
    StepDiv sd; sd.init(q.step);
    uint32_t parity = 0;
    int b = 0;
    Walk w;
    for (bool more = walk_start(w); more; more = walk_next(w), b ^= 1) {
      TileSeries* SDn = reinterpret_cast<TileSeries*>(smem + L.desc + b * L.desc_stride);
      TileMeta* Mn = reinterpret_cast<TileMeta*>(smem + L.meta + b * 128);
      const int64_t i0 = w.pb;
      const int ns = (int)(w.pe - w.pb < TILE_NS ? w.pe - w.pb : TILE_NS);
      // lanes 0..ns-1: series id, record offset and size; records land back to back in the staging buffer
      int64_t sid_l = -1, src_l = 0; uint32_t sz_l = 0;
      if (lane < ns) { sid_l = (AGG && order) ? (int64_t)order[i0 + lane] : i0 + lane; src_l = rec_off[sid_l]; sz_l = (uint32_t)(rec_off[sid_l + 1] - src_l); }
      uint32_t incl = sz_l;
#pragma unroll
      for (int o = 1; o < TILE_NS; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += y; }
      const uint32_t tile_bytes = __shfl_sync(0xffffffffu, incl, TILE_NS - 1), roff_l = incl - sz_l;
      const bool staged = tile_bytes <= L.rec_cap - 64;
      if (staged) {
        if (lane == 0) mbar_expect_tx(bar, tile_bytes);
        __syncwarp();
        if (AGG) { if (lane < ns) tma_load_1d(recbuf + roff_l, arena + src_l, sz_l, bar); }      // gathered through `order`
        else if (lane == 0) tma_load_1d(recbuf, arena + src_l, tile_bytes, bar);                   // adjacent records: one copy
        mbar_wait(bar, parity); parity ^= 1;
      }
      // ---------------------------------------------------------------- setup: lane = series * 4 + chunk
      const int s = lane >> 2, c = lane & 3, lb = lane & 28;
      TileSeries& S = SDn[s];
      const bool present = s < ns;
      bool regular = false; int n = 0, cLo = 0;
      const uint32_t roff = __shfl_sync(0xffffffffu, roff_l, s);
      const int64_t sid = __shfl_sync(0xffffffffu, sid_l, s);
      const uint8_t* rec = recbuf;
      if (present && staged) {
        rec = recbuf + roff;
        const RecordHeader* h = reinterpret_cast<const RecordHeader*>(rec);
        const ChunkEntry* E = reinterpret_cast<const ChunkEntry*>(rec + sizeof(RecordHeader));
        const int nch = (int)h->n_chunks;
        const int64_t t1 = q.start - q.window, t2 = q.end;
        while (cLo < nch && E[cLo].end_time < t1) ++cLo;
        int cHi = cLo; while (cHi < nch && E[cHi].start_time <= t2) ++cHi;
        if (t1 > t2) cHi = cLo;
        n = cHi - cLo;
        regular = n <= TILE_MAXC && (n == 0 || (h->flags & REC_ALL_TS_CONST));
      }
      const ChunkEntry* E = reinterpret_cast<const ChunkEntry*>(rec + sizeof(RecordHeader)) + cLo;
      bool have = regular && c < n;
      int64_t init = 0, end_time = 0; int tlen = 0, vlen = 0, ng = 0, vwire = 0, nrows = 0, num_rows = 0, vbytes = 0; uint32_t voff = 0, w12 = 0;
      bool okc = true;
      if (have) {
        const ChunkEntry& e = E[c];
        const uint8_t* tv = rec + e.ts_off; const uint8_t* vv = rec + e.val_off;
        vwire = ld32(vv + 4) & 0xffff;
        tlen = (int)ld32(tv + 8); init = (int64_t)ld64_a4(tv + 12); const int slope = (int)ld32(tv + 20);
        end_time = e.end_time; num_rows = e.num_rows; voff = roff + e.val_off;
        vbytes = (int)ld32(tv) + 4 + (int)ld32(vv) + 4;
        if (vwire == WIRE_XOR) { vlen = (int)ld32(vv + XOR_OFF_N); w12 = ld32(vv + XOR_OFF_NGROUPS); ng = (int)(w12 & 0xffff); }
        else if (vwire == WIRE_RAW64) vlen = ((int)ld32(vv) - 4) / 8;
        else okc = false;
        if ((int64_t)slope != q.step || tlen <= 0 || vlen <= 0) okc = false;
        nrows = num_rows < tlen ? num_rows : tlen; if (vlen < nrows) nrows = vlen;
      }
      const unsigned okm = __ballot_sync(0xffffffffu, okc);     // (not inside the &&: every lane must take part)
      regular = regular && ((okm >> lb) & 0xfu) == 0xfu;
      have = have && regular;
      if (!have) { ng = 0; nrows = 0; }
      // exclusive prefix / total over the series' chunks (lanes lb .. lb+3)
      auto xpre = [&](int v, int& total) -> int {
        const int a0 = __shfl_sync(0xffffffffu, v, lb), a1 = __shfl_sync(0xffffffffu, v, lb + 1), a2 = __shfl_sync(0xffffffffu, v, lb + 2), a3 = __shfl_sync(0xffffffffu, v, lb + 3);
        total = a0 + a1 + a2 + a3;
        return (c > 0 ? a0 : 0) + (c > 1 ? a1 : 0) + (c > 2 ? a2 : 0);
      };
      int ngroups = 0;
      const int grp_base = xpre(ng, ngroups);
      // three divisions per chunk: s0, e0 = unclamped first / last row of window 0; v4 = last window whose start is <= endTime.
      // The other bounds of scan_fast.cuh chunk_interval follow from these and the neighbours':
      //   ceil((init - E0)/step) = -e0           floor((lastTs - S0)/step) = nrows - 1 - s0
      //   ceil((max(prevEnd, prevLastTs) + 1 - S0)/step) = max(prev.v4 + 1, prev.tlen - prev.s0)
      //   floor((next.init - 1 - E0)/step) = -(next.e0 + 1)
      int64_t s0 = 0, e0 = 0, v4 = 0;
      if (have) { s0 = sd.ceil_div(S0 - init); e0 = sd.floor_div(E0 - init); v4 = sd.floor_div(end_time - S0); }
      const int64_t s0p = __shfl_up_sync(0xffffffffu, s0, 1), v4p = __shfl_up_sync(0xffffffffu, v4, 1), e0n = __shfl_down_sync(0xffffffffu, e0, 1);
      const int tlenp = __shfl_up_sync(0xffffffffu, tlen, 1);
      const int64_t endp = __shfl_up_sync(0xffffffffu, end_time, 1);
      int64_t kA = -e0;
      if (c > 0) { int64_t x = v4p + 1; const int64_t y = (int64_t)tlenp - s0p; if (y > x) x = y; if (x > kA) kA = x; }
      int64_t kB = (int64_t)(nrows - 1) - s0;
      { const int64_t x = (c + 1 < n) ? -(e0n + 1) : (int64_t)q.T; if (x < kB) kB = x; }
      if (v4 < kB) kB = v4;
      if (kA < 0) kA = 0;
      if (kB > q.T - 1) kB = q.T - 1;
      const int64_t sA = s0 + kA, eA = e0 + kA;
      const bool ok = have && kA <= kB && eA >= sA;
      const int Wr = ok ? (int)(eA - sA) : 0;
      const int nwin = ok ? (int)(kB - kA + 1) : 0;
      // blocked only when the windows are long enough to amortise a block; short windows go through the per-window path
      const bool blocked = ok && Wr >= BLK_R - 1;
      const int nb = blocked ? (nwin + BLK_R - 1) / BLK_R : 0;
      // zero rows around the chunk so that blocked sums read clamped-away rows as +0.0 without a bounds check
      int lowz = 0, highz = 0;
      if (blocked) {
        if (sA < 0) lowz = (int)-sA;
        const int64_t over = sA + (nwin - 1) + Wr - (nrows - 1); if (over > 0) highz = (int)over;
      }
      int need = 0;
      (void)xpre(lowz + nrows + highz, need);
      const bool padded = need + BLK_R <= (int)L.vals_pitch;
      if (!padded) { lowz = 0; highz = 0; }
      int nrows_tot = 0;
      const int row_base = xpre(lowz + nrows + highz, nrows_tot) + lowz;
      if (ngroups > TILE_MAXG || nrows_tot + 2 > (int)L.vals_pitch) { regular = false; have = false; }
      int nblocks = 0, covered = 0;
      const int blk0 = xpre(have ? nb : 0, nblocks); (void)xpre(have && blocked ? nwin : 0, covered);
      int cnt_rows = 0, cnt_bytes = 0;            // this chunk's contribution to the scan counters
      if (have) {
        TileChunk& ch = S.c[c];
        ch.init = init; ch.end_time = end_time; ch.nrows = nrows; ch.row_base = row_base;
        ch.val_off = voff; ch.wire = vwire; ch.ngroups = ng; ch.grp_base = grp_base;
        ch.kA = blocked ? (int)kA : 0; ch.kB = blocked ? (int)kB : -1; ch.sA = (int)sA; ch.Wr = Wr; ch.blk0 = blk0; ch.blk_n = nb;
        ch.s0 = (int)s0; ch.e0 = (int)e0;
        if (vwire == WIRE_XOR) {
          const uint32_t po = w12 >> 16;
          ch.first = ld64(recbuf + voff + po); ch.grp_off = voff + po + 8; ch.tab_off = voff + XOR_OFF_GROUPTAB;
        } else { ch.first = ld64(recbuf + voff + 8); ch.grp_off = 0; ch.tab_off = 0; }
        ch.lowz = lowz; ch.highz = highz;          // zeroed by the consumers before they decode the tile
        // CountingChunkInfoIterator, ChunkSetInfo.scala:336-380: every chunk in range is pulled, except one that starts after
        // the last window end (the window iterator never reaches it)
        const int64_t lastEnd = q.start + (int64_t)(q.T - 1) * q.step;
        if (!(c > 0 && !(endp < lastEnd))) { cnt_rows = num_rows; cnt_bytes = vbytes; }
      }
      { int tr = 0, tb = 0; (void)xpre(cnt_rows, tr); (void)xpre(cnt_bytes, tb); if (c == 0) { S.cnt_rows = tr; S.cnt_bytes = tb; } }
      S.gb[c] = have ? grp_base : 0x7fffffff;
      const unsigned rawm = __ballot_sync(0xffffffffu, have && vwire == WIRE_RAW64);
      const unsigned irrm = __ballot_sync(0xffffffffu, present && !regular);
      if (AGG && irrm != 0) regular = false;      // an item is folded as a whole: one irregular series sends the item to the fallback
      const unsigned unpm = __ballot_sync(0xffffffffu, have && !padded);
      if (c == 0) {
        if (regular) {
          S.sid = sid; S.n = n; S.regular = 1; S.rec_off = (int)roff; S.nblocks = nblocks; S.nrest = q.T - covered; S.ngroups = ngroups; S.nrows = nrows_tot;
          S.any_raw = ((rawm >> lb) & 0xfu) != 0;
        } else {
          S.n = 0; S.regular = present ? 0 : 2; S.nblocks = 0; S.nrest = 0; S.ngroups = 0; S.nrows = 0; S.any_raw = 0;
          if (present && !AGG) {
            const unsigned long long slot = atomicAdd(fallback_count, 1ull);
            fallback_list[slot] = sid;
          }
        }
      }
      // tile work-list prefixes over the series (values sit in the c == 0 lanes)
      int p = (c == 0 && regular) ? nblocks : 0, r = (c == 0 && regular) ? q.T - covered : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int pp = __shfl_up_sync(0xffffffffu, p, o), rr = __shfl_up_sync(0xffffffffu, r, o);
        if (lane >= o) { p += pp; r += rr; }
      }
      if (c == 0) { Mn->pref[s + 1] = p; Mn->rpref[s + 1] = r; }
      if (lane == 0) { Mn->pref[0] = 0; Mn->rpref[0] = 0; Mn->any_nan = 0; Mn->any_raw = rawm != 0; Mn->all_regular = irrm == 0; Mn->all_padded = unpm == 0; Mn->staged = staged; Mn->ns = ns; Mn->i0 = i0; }
      __syncwarp();
      if (lane == 0) mbar_arrive(ready + b);      // A(t): release the descriptors
      __syncthreads();          // B(t)
    }
    return;
  }

  // ==================================================================== consumer warps
  const bool out_aligned = (reinterpret_cast<uintptr_t>(out) & 15) == 0;
  uint32_t parity = 0;
  int b = 0;
  // AGG: this thread's windows tid + j * TILE_THREADS; MOM: their Σv² at aacc[TILE_AGG_ACC + j]
  double aacc[MOM ? 2 * TILE_AGG_ACC : TILE_AGG_ACC]; uint32_t acnt[TILE_AGG_ACC]; bool item_bad = false;
  const double agg_ident = agg_op == AGG_MIN ? __longlong_as_double(0x7ff0000000000000LL)
                         : agg_op == AGG_MAX ? __longlong_as_double(0xfff0000000000000LL) : 0.0;
#pragma unroll
  for (int j = 0; j < TILE_AGG_ACC; ++j) { aacc[j] = agg_ident; acnt[j] = 0; if constexpr (MOM) aacc[TILE_AGG_ACC + j] = 0.0; }
  int64_t rows_scanned = 0, bytes_scanned = 0, pend_rows = 0, pend_bytes = 0;
  uint32_t tj = 0;                      // tiles done by this CTA: buffer tj & 1, phase (tj >> 1) & 1 of its ready barrier
  TPROF_DECL
  Walk w;
  for (bool more = walk_start(w); more; more = walk_next(w), b ^= 1) {
    const TileSeries* SDc = reinterpret_cast<const TileSeries*>(smem + L.desc + b * L.desc_stride);
    TileMeta* Mc = reinterpret_cast<TileMeta*>(smem + L.meta + b * 128);
    TPROF(9)                                                // results of the previous tile (fold / store, loop overhead)
    mbar_wait_parked(ready + b, (tj >> 1) & 1); ++tj;   // A(t): descriptors ready (no consumer-wide barrier: the windows-end barrier of the
                                                 // previous tile already separates the tiles)
    if (Mc->staged) { mbar_wait(bar, parity); parity ^= 1; }    // already complete (the producer saw it); orders the TMA writes
    const int64_t i0 = Mc->i0; const int ns = Mc->ns;
    TPROF(0)                                                // wait: descriptors (+ tile bytes) ready
    // zero rows around the chunks (warp 0, lane = series * 4 + chunk); read by the blocked sums after the next barriers
    if (warp == 0) {
      const TileSeries& S = SDc[lane >> 2];
      const int c = lane & 3;
      if (S.regular == 1 && c < S.n) {
        const TileChunk& ch = S.c[c];
        double* zr = vals + (size_t)(lane >> 2) * L.vals_pitch + ch.row_base;
        for (int i = 1; i <= ch.lowz; ++i) zr[-i] = 0.0;
        for (int i = 0; i < ch.highz; ++i) zr[ch.nrows + i] = 0.0;
      }
    }
    // ------------------------------------------------------------------ decode: two (series, group slot) items per thread
    // Lane -> series lane & 7 (neighbouring lanes store to different series' rows: with the odd row pitch the 8-byte stores
    // of a warp spread over all banks); warp w owns the slots 8w .. 8w+7 of every series: item jj -> slot 8w + 4jj + (lane >> 3).
    {
      const int ds = lane & 7;
      const TileSeries& S = SDc[ds];
      const bool sreg = S.regular == 1;
      uint64_t d[2][8]; uint64_t excl[2]; int cc[2]; bool act[2];
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        const int slot = warp * 8 + jj * 4 + (lane >> 3);
        const bool active = sreg && slot < S.ngroups;
        const int c = (slot >= S.gb[1] ? 1 : 0) + (slot >= S.gb[2] ? 1 : 0) + (slot >= S.gb[3] ? 1 : 0);
        const TileChunk& ch = S.c[c];
        cc[jj] = c; act[jj] = active;
        const uint8_t* gp = recbuf;
        if (active) gp = recbuf + ch.grp_off + reinterpret_cast<const uint16_t*>(recbuf + ch.tab_off)[slot - ch.grp_base];
        const uint32_t mask = active ? gp[0] : 0u;
        const uint32_t hdr = gp[1];
        const uint32_t numBits = ((hdr >> 4) + 1) * 4;
        const uint32_t tz = (hdr & 0x0f) * 4;
        const uint64_t fmask = ~0ull >> (64 - numBits);
        // word-aligned base of the group's fields, derived by pointer arithmetic from the staging buffer so that the loads stay in the
        // shared window (an integer round trip made them generic loads)
        const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(gp + 2) & 3);
        uint32_t bit = mis * 8;
        const uint32_t* base = reinterpret_cast<const uint32_t*>(gp + 2 - mis);
        uint64_t x = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const bool on = (mask >> i) & 1u;
          const uint32_t* wp = base + (bit >> 5);
          const uint32_t w0 = wp[0], w1 = wp[1], w2 = wp[2];
          const uint32_t lo = __funnelshift_r(w0, w1, bit), hi = __funnelshift_r(w1, w2, bit);
          const uint64_t fm = on ? fmask : 0ull;
          x ^= (((uint64_t)hi << 32) | lo) & fm;       // running XOR of the unshifted fields ((a ^ b) << tz == (a << tz) ^ (b << tz))
          bit += on ? numBits : 0u;
          d[jj][i] = x << tz;
        }
      }
      uint64_t pre0, pre1;
      // XOR of the group totals of earlier slots of the same series inside this warp (lanes ds, ds+8, ds+16, ds+24; item 0 first)
      uint64_t i0x = d[0][7], i1x = d[1][7];
      { const uint64_t y0 = shfl_up_u64(i0x, 8), y1 = shfl_up_u64(i1x, 8); if (lane >= 8) { i0x ^= y0; i1x ^= y1; } }
      { const uint64_t y0 = shfl_up_u64(i0x, 16), y1 = shfl_up_u64(i1x, 16); if (lane >= 16) { i0x ^= y0; i1x ^= y1; } }
      const uint64_t tot0 = shfl_u64(i0x, 24 + ds), tot1 = shfl_u64(i1x, 24 + ds);
      excl[0] = i0x ^ d[0][7]; excl[1] = i1x ^ d[1][7] ^ tot0;
      gexcl[ds * TILE_GX_PITCH + warp * 8 + (lane >> 3)] = excl[0];
      gexcl[ds * TILE_GX_PITCH + warp * 8 + 4 + (lane >> 3)] = excl[1];
      if (lane >= 24) gwtot[ds * TILE_GW_PITCH + warp] = tot0 ^ tot1;
      TPROF(1)                                              // decode: field extraction + in-warp prefix
      bar_consumers();
      TPROF(2)                                              // wait: cross-warp exchange barrier
      // value before group g of chunk c = first_c ^ (prefix at the slot) ^ (prefix at the chunk's first slot); the prefix at a
      // slot = XOR of the earlier warps' totals ^ the in-warp part
      {
        const TileChunk& c0 = S.c[cc[0]]; const TileChunk& c1 = S.c[cc[1]];
        const int gb0 = act[0] ? c0.grp_base : 0, gb1 = act[1] ? c1.grp_base : 0;
        pre0 = c0.first ^ excl[0] ^ gexcl[ds * TILE_GX_PITCH + gb0];
        pre1 = c1.first ^ excl[1] ^ gexcl[ds * TILE_GX_PITCH + gb1];
        const int wl0 = gb0 >> 3, wl1 = gb1 >> 3;
        for (int w = 0; w < warp; ++w) {
          const uint64_t tw = gwtot[ds * TILE_GW_PITCH + w];
          if (w >= wl0) pre0 ^= tw;
          if (w >= wl1) pre1 ^= tw;
        }
      }
      uint32_t nz = 0x7ff00000u;
      {
        const TileChunk& c0 = S.c[cc[0]]; const TileChunk& c1 = S.c[cc[1]];
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          const TileChunk& ch = jj ? c1 : c0;
          const uint64_t pre = jj ? pre1 : pre0;
          const int g = act[jj] ? warp * 8 + jj * 4 + (lane >> 3) - ch.grp_base : 0;   // an inactive slot's chunk descriptor is not initialised
          uint64_t* dst = reinterpret_cast<uint64_t*>(vals + (size_t)ds * L.vals_pitch + ch.row_base) + 1 + g * 8;
          const int nleft = act[jj] ? ch.nrows - 1 - g * 8 : 0;     // rows past nrows are never read as data
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const uint64_t b = d[jj][i] ^ pre;
            if (i < nleft) { dst[i] = b; const uint32_t e = ~(uint32_t)(b >> 32) & 0x7ff00000u; nz = e < nz ? e : nz; }
          }
          if (act[jj] && g == 0) { dst[-1] = ch.first; const uint32_t e = ~(uint32_t)(ch.first >> 32) & 0x7ff00000u; nz = e < nz ? e : nz; }
        }
      }
      if (nz == 0) Mc->any_nan = 1;               // an exponent of all ones: NaN or Inf (conservative)
    }
    // raw f64 vectors: plain copy (+ NaN/Inf presence)
    if (Mc->any_raw) {
      for (int s = 0; s < TILE_NS; ++s) {
        const TileSeries& S = SDc[s];
        if (S.regular != 1) continue;
        for (int c = 0; c < S.n; ++c) {
          const TileChunk& ch = S.c[c];
          if (ch.wire != WIRE_RAW64) continue;
          const uint64_t* src = reinterpret_cast<const uint64_t*>(recbuf + ch.val_off + 8);
          uint64_t* dst = reinterpret_cast<uint64_t*>(vals + (size_t)s * L.vals_pitch + ch.row_base);
          bool nan = false;
          for (int r = tid; r < ch.nrows; r += TILE_THREADS) {
            const uint64_t b = src[r]; dst[r] = b; nan |= ((uint32_t)(b >> 32) & 0x7ff00000u) == 0x7ff00000u;
          }
          if (nan) Mc->any_nan = 1;
        }
      }
    }
    TPROF(3)                                                // decode: prefixes applied, rows stored (+ raw copies)
    if (tid == 0) tma_store_wait_read();       // the previous tile's bulk store must have finished reading `otile`
    __syncthreads();            // B(t): the record bytes are dead, the producer refills the staging buffer
    // ------------------------------------------------------------------ windows: blocked single-chunk windows
    {
      const bool any_nan = Mc->any_nan != 0, padded = Mc->all_padded != 0;
      TPROF(4)                                              // wait: barrier B
      const int nitems = Mc->pref[TILE_NS];
      for (int it = tid; it < nitems; it += TILE_THREADS) {
        int s = 0;
#pragma unroll
        for (int j = 1; j < TILE_NS; ++j) if (it >= Mc->pref[j]) s = j;
        const TileSeries& S = SDc[s];
        const int B = it - Mc->pref[s];
        int c = 0; while (c + 1 < S.n && B >= S.c[c].blk0 + S.c[c].blk_n) ++c;
        const TileChunk& ch = S.c[c];
        const int b = B - ch.blk0;
        const int r0 = ch.sA + b * BLK_R;
        const double* slots = vals + (size_t)s * L.vals_pitch + ch.row_base;
        double acc[BLK_R]; int cnt[BLK_R];
        constexpr bool NEED_CNT = FN == FN_AVG || FN == FN_COUNT;
        if (any_nan) blocked_sum<true, true, true>(slots, r0, ch.nrows, ch.Wr, acc, cnt);
        else if (padded) blocked_sum<false, false, NEED_CNT>(slots, r0, ch.nrows, ch.Wr, acc, cnt);
        else blocked_sum<false, true, NEED_CNT>(slots, r0, ch.nrows, ch.Wr, acc, cnt);
        const int k0 = ch.kA + b * BLK_R;
        int nw = ch.kB - k0 + 1; if (nw > BLK_R) nw = BLK_R;
        double* o = otile + (size_t)s * L.out_pitch + k0;
        if (FN == FN_RATE) {
          // sum / window * 1000 for 15 windows: one range test for the whole block (div_invariant's exactness condition),
          // then the two-FMA correction without per-window branches; any unusual quotient (0, NaN, Inf, tiny, huge) sends
          // the block through the per-window version
          double q0[BLK_R]; uint32_t worst = 0;
#pragma unroll
          for (int j = 0; j < BLK_R; ++j) {
            acc[j] = cnt[j] ? acc[j] : __longlong_as_double(0x7ff8000000000000LL);
            q0[j] = __dmul_rn(acc[j], frcp);
            const uint32_t e = ((uint32_t)__double2hiint(q0[j]) & 0x7ff00000u) - (65u << 20);
            worst = e > worst ? e : worst;
          }
          if (worst < (1918u << 20)) {
#pragma unroll
            for (int j = 0; j < BLK_R; ++j) {
              const double r = __fma_rn(-q0[j], fdiv, acc[j]);
              const double v = __dmul_rn(__fma_rn(r, frcp, q0[j]), 1000.0);
              if (j < nw) o[j] = v;
            }
          } else {
#pragma unroll
            for (int j = 0; j < BLK_R; ++j) if (j < nw) o[j] = __dmul_rn(div_invariant(acc[j], fdiv, frcp), 1000.0);
          }
        } else {
#pragma unroll
          for (int j = 0; j < BLK_R; ++j) if (j < nw) o[j] = tile_finish<FN>(acc[j], cnt[j], fdiv, frcp);
        }
      }
      // ---------------------------------------------------------------- windows: everything else (chunk junctions, short windows)
      TPROF(5)                                              // windows: blocked items
      const int nrest = Mc->rpref[TILE_NS];
      for (int it = tid; it < nrest; it += TILE_THREADS) {
        int s = 0;
#pragma unroll
        for (int j = 1; j < TILE_NS; ++j) if (it >= Mc->rpref[j]) s = j;
        const TileSeries& S = SDc[s];
        int u = it - Mc->rpref[s];
        int prev = -1; bool found = false;          // u-th window not covered by a blocked interval
        for (int c = 0; c < S.n && !found; ++c) {
          if (S.c[c].kA > S.c[c].kB) continue;
          const int gap = S.c[c].kA - prev - 1;
          if (u < gap) found = true; else { u -= gap; prev = S.c[c].kB; }
        }
        const int k = prev + 1 + u;
        const int64_t wEnd = q.start + (int64_t)k * q.step, wStart = wEnd - winDur;
        const double* sv = vals + (size_t)s * L.vals_pitch;
        otile[(size_t)s * L.out_pitch + k] = any_nan ? tile_eval_window<FN, true>(S, sv, wStart, wEnd, fdiv, k)
                                                     : tile_eval_window<FN, false>(S, sv, wStart, wEnd, fdiv, k);
      }
    }
    TPROF(6)                                                // windows: literal per-window folds
    fence_async_smem();        // make this thread's writes to the output tile visible to the async proxy (bulk store below)
    bar_consumers();
    TPROF(7)                                                // wait: windows-end barrier
    // tile flags of this tile stay valid until the producer's setup two tiles ahead, which waits for the next B barrier
    const bool all_reg = Mc->all_regular != 0;
    // scan counters (CountingChunkInfoIterator): series this kernel answers; series / items handed to the fallback are counted there
    if (tid < ns && SDc[tid].regular == 1) { pend_rows += SDc[tid].cnt_rows; pend_bytes += SDc[tid].cnt_bytes; }
    if (!AGG) { rows_scanned += pend_rows; bytes_scanned += pend_bytes; pend_rows = 0; pend_bytes = 0; }
    // ------------------------------------------------------------------ results
    if (AGG) {
      // fold the tile's rows into this thread's accumulators (RowAggregators skip NaN: SumRowAggregator.scala:22-29 ...);
      // the item's partial row leaves after its last tile
      item_bad |= !all_reg;
      if (all_reg) {
#pragma unroll
        for (int j = 0; j < TILE_AGG_ACC; ++j) {
          const int k = tid + j * TILE_THREADS;
          if (k < q.T) {
            double a = aacc[j]; uint32_t n = acnt[j];
            for (int s = 0; s < ns; ++s) {
              const double v = otile[(size_t)s * L.out_pitch + k];
              if (v == v) {
                // min/maxIgnoreNaN(acc, v) (QueryUtils.scala:111-123): of two equal values the later one is kept
                if (agg_op == AGG_MIN) a = a < v ? a : v; else if (agg_op == AGG_MAX) a = a > v ? a : v; else if (agg_op != AGG_COUNT) a += v;
                if constexpr (MOM) aacc[TILE_AGG_ACC + j] += v * v;
                ++n;
              }
            }
            aacc[j] = a; acnt[j] = n;
          }
        }
      }
      if (w.pb + TILE_NS >= w.pe) {               // last tile of the item
        if (!item_bad) {
#pragma unroll
          for (int j = 0; j < TILE_AGG_ACC; ++j) {
            const int k = tid + j * TILE_THREADS;
            if (k < q.T) {
              pval[(size_t)w.it * q.T + k] = aacc[j]; pcnt[(size_t)w.it * q.T + k] = acnt[j];
              if constexpr (MOM) pval[(size_t)(n_items + w.it) * q.T + k] = aacc[TILE_AGG_ACC + j];
            }
          }
          rows_scanned += pend_rows; bytes_scanned += pend_bytes;
        } else if (tid == 0) {
          const unsigned long long slot = atomicAdd(fallback_count, 1ull);
          fallback_list[slot] = w.it;
        }
        pend_rows = 0; pend_bytes = 0;
#pragma unroll
        for (int j = 0; j < TILE_AGG_ACC; ++j) { aacc[j] = agg_ident; acnt[j] = 0; if constexpr (MOM) aacc[TILE_AGG_ACC + j] = 0.0; }
        item_bad = false;
      }
    } else {
      // one bulk store for the tile (regular rows only)
      double* gout = out + (size_t)i0 * q.T;
      const uint32_t bytes = (uint32_t)ns * (uint32_t)q.T * 8u;
      if (all_reg && out_aligned && (bytes & 15) == 0 && (((size_t)i0 * q.T * 8) & 15) == 0) {
        if (tid == 0) tma_store_1d(gout, otile, bytes);
      } else {
        for (int s = 0; s < ns; ++s) {
          if (SDc[s].regular != 1) continue;
          for (int k = tid; k < q.T; k += TILE_THREADS) gout[(size_t)s * q.T + k] = otile[(size_t)s * L.out_pitch + k];
        }
        bar_consumers();
      }
    }
  }
  if (tid == 0) tma_store_wait_read();
  TPROF(9)
  TPROF_FLUSH
  if (rows_scanned | bytes_scanned) {
    atomicAdd(&d_counters[0], (unsigned long long)rows_scanned); atomicAdd(&d_counters[1], (unsigned long long)bytes_scanned);
  }
}

} // namespace filo
