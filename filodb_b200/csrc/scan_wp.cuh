// v4 scan path ("wp": warp pipeline).  One warp owns one series end to end; warps never synchronise with each other.
//
// Each warp runs its own three-buffer pipeline in shared memory:
//   R  the series' record (ChunkSetInfo entries + BinaryVectors verbatim), filled by ONE cp.async.bulk (TMA 1-D) per series that is
//      issued as soon as the previous record is no longer read (its fields extracted, raw f64 vectors copied), i.e. it is in flight
//      during the rest of the previous series' decode and its window phase.  With two record buffers (L.rec2) the warp's series
//      alternate between them, and the copy issued there is the record of the series after next: two records are in flight;
//   V  the decoded rows, laid out per chunk with zero rows in between so that clamped windows read +0.0 instead of testing bounds
//      (x + 0.0 == x for every sum of non-zero values and +0.0 rows), skewed by one pad slot per 8 rows: both the 8-byte row stores of the
//      group decode (lane stride 8 rows) and the 8-byte row loads of the window blocks (lane stride 8 windows) then walk the banks with
//      an odd stride of 9 words -- conflict-free;
//   O  the series' window sums, in V's place when the plan allows it: finished values, or raw sums still to be finished.
// Phases of a series (all 32 lanes, only __syncwarp between them):
//   setup    lane c = chunk c: header parse, regularity checks, window plan (touch interval, block list, row positions, and the class
//            of every window a lane stores, see wp_class).  The plan depends on (init, nrows, endTime) of the chunks only, so it is
//            reused while consecutive series share those (memo);
//   decode   lane = NibblePack group (two groups per lane): branch-free field extraction, XOR prefix inside the group, warp-wide
//            XOR scan over the group totals, rows stored once;
//   windows  item = (chunk, block of 8 windows), two items per lane: register-blocked sequential sums in the reference's row order
//            (DoubleVector.scala:243-253, AggrOverTimeFunctions.scala:560-571).  A window that takes rows from two chunks gets one
//            partial sum from each chunk's block list (the earlier chunk's in O, the later one's in J);
//   finish   lane l = windows l + 32 m: one pass loads O (and J), finishes by the window's class (junction sums in chunk order, raw
//            sums, windows without rows) and stores straight to the output: lane-consecutive streaming stores, 256 contiguous bytes
//            per store instruction.  Nothing is written back to O.  scan_wp_batch_kernel instead stages the row densely in O: its window
//            blocks write the finished windows there, a fix-up writes the rest, and one bulk copy stores the row (wp_finish_store<FN, true>).
// Anything outside this fast path (irregular timestamps, DDV-long values, > 4 chunks, NaN / Inf / denormal / zero values, windows
// shorter than 9 rows, windows over three chunks ...) is appended to the fallback list and answered by the v2 kernel into the same
// output buffer, exactly as the tile kernel does.
#pragma once
#include "scan_tile.cuh"
#include "scan_wp_layout.h"

namespace filo {

// shared-memory word loads by byte offset (keeps the field extraction in the shared window: LDS, not generic loads)
#ifdef FILO_CUSIM
__device__ __forceinline__ uint32_t wp_soff(const void* p) { return (uint32_t)(reinterpret_cast<const uint8_t*>(p) - smem); }
__device__ __forceinline__ uint32_t wp_lds32(uint32_t off) { uint32_t v; std::memcpy(&v, smem + off, 4); return v; }
#else
__device__ __forceinline__ uint32_t wp_soff(const void* p) { return smem_u32(p); }
__device__ __forceinline__ uint32_t wp_lds32(uint32_t off) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(off)); return v; }
#endif

// Per-phase cycle counters of the SUM-class kernels for profiling builds (-DFILO_WP_PROF; scratch/wp_prof.py): every lane reads the
// SM clock at the phase boundaries of a series, lane 0 adds its sums to g_wp_prof (slots 0 .. 9: phases, slot 8 the batch kernel's wait
// for the previous result row's bulk store; 10 .. 13: event counts, 15: warps; 16 .. 20: the producer warp of scan_wp_batch_kernel).  32-bit sums
// (a warp's share of one launch is far below 2^32 cycles) keep the register cost low.  Compiled out of the product build.
#if defined(FILO_WP_PROF) && !defined(FILO_CUSIM)
__device__ unsigned long long g_wp_prof[32];
#define WPROF_DECL uint32_t wpp_t0 = (uint32_t)clock(), wpp_acc[14] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
#define WPROF(i) { const uint32_t wpp_t1 = (uint32_t)clock(); wpp_acc[i] += wpp_t1 - wpp_t0; wpp_t0 = wpp_t1; }
#define WPROF_COUNT(i) { ++wpp_acc[i]; }
#define WPROF_FLUSH if (lane == 0) { for (int wpp_i = 0; wpp_i < 14; ++wpp_i) atomicAdd(&g_wp_prof[wpp_i], (unsigned long long)wpp_acc[wpp_i]); atomicAdd(&g_wp_prof[15], 1ull); }
#else
#define WPROF_DECL
#define WPROF(i)
#define WPROF_COUNT(i)
#define WPROF_FLUSH
#endif

__device__ __forceinline__ int wp_vidx(int p) { return p + (p >> 3); }
__device__ __forceinline__ double nan0(double x) { return x != x ? 0.0 : x; }
// results are written once and not read again by the scan: streaming store
#ifdef FILO_CUSIM
__device__ __forceinline__ void wp_store_result(double* g, double v) { *g = v; }
#else
__device__ __forceinline__ void wp_store_result(double* g, double v) { __stcs(g, v); }
#endif

// finish of one window of a SUM-class function from (sum over the rows, number of rows); values are known to be finite, normal and
// of moderate magnitude (the decode checked), so the invariant division needs no range test
template <int FN>
__device__ __forceinline__ double wp_finish(double cs, int nn, double div, double rcp, double scale, int nfull, double rcpn, bool raw) {
  // raw blocks pass div = rcp = scale = 1: the sequence below then returns cs itself, bit for bit
  if (FN == FN_RATE) { const double q0 = __dmul_rn(cs, rcp); const double r = __fma_rn(-q0, div, cs); return __dmul_rn(__fma_rn(r, rcp, q0), scale); }
  if (FN == FN_COUNT) return (double)nn;
  if (FN == FN_AVG) {
    if (raw) return cs;
    if (nn == nfull) { const double q0 = __dmul_rn(cs, rcpn); const double r = __fma_rn(-q0, (double)nfull, cs); return __fma_rn(r, rcpn, q0); }
    return cs / (double)nn;
  }
  return cs;
}

// the last two row groups of a block: rows 8q .. Wr + 7 with Wr = 8q + U.  Row t of group q feeds windows max(0, t - U) .. 7, row t < U of
// group q + 1 feeds windows 8 + t - U .. 7 (window w takes rows w .. w + Wr of the block)
template <int U>
__device__ __forceinline__ void wp_block_tail(const double* __restrict__ pa, const double* __restrict__ pb, double a[WP_R], double b[WP_R]) {
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    const double va = pa[t], vb = pb[t];
#pragma unroll
    for (int w = 0; w < 8; ++w) if (w >= t - U) { a[w] += va; b[w] += vb; }
  }
#pragma unroll
  for (int t = 0; t < U; ++t) {
    const double va = pa[9 + t], vb = pb[9 + t];
#pragma unroll
    for (int w = 0; w < 8; ++w) if (w >= 8 + t - U) { a[w] += va; b[w] += vb; }
  }
}

// two blocks per lane: a[w] / b[w] = sum of rows w .. w + Wr (in row order, starting from +0.0) of the block at pa / pb.  Wr >= 8.
// A window's sum starts at its first row instead of at +0.0 + that row: the same bits, because every row the windows read is either a
// decoded value (finite, normal, non-zero, or the series is declined before its windows) or a +0.0 zero row, and +0.0 + x == x for both.
__device__ __forceinline__ void wp_block_pair(const double* __restrict__ pa, const double* __restrict__ pb, int Wr, double a[WP_R], double b[WP_R]) {
#pragma unroll
  for (int t = 0; t < 8; ++t) {                        // group 0: row t opens window t and feeds windows 0 .. t - 1
    const double va = pa[t], vb = pb[t];
#pragma unroll
    for (int w = 0; w < t; ++w) { a[w] += va; b[w] += vb; }
    a[t] = va; b[t] = vb;
  }
  const int q = Wr >> 3;
  pa += 9; pb += 9;
  for (int m = 1; m < q; ++m, pa += 9, pb += 9) {      // full groups: every window
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const double va = pa[t], vb = pb[t];
#pragma unroll
      for (int w = 0; w < 8; ++w) { a[w] += va; b[w] += vb; }
    }
  }
  switch (Wr & 7) {
    case 0: wp_block_tail<0>(pa, pb, a, b); break;
    case 1: wp_block_tail<1>(pa, pb, a, b); break;
    case 2: wp_block_tail<2>(pa, pb, a, b); break;
    case 3: wp_block_tail<3>(pa, pb, a, b); break;
    case 4: wp_block_tail<4>(pa, pb, a, b); break;
    case 5: wp_block_tail<5>(pa, pb, a, b); break;
    case 6: wp_block_tail<6>(pa, pb, a, b); break;
    default: wp_block_tail<7>(pa, pb, a, b); break;
  }
}

// per-series parse, lane c = chunk c of the chunks in range: what the record says about the chunk, and whether the series qualifies
struct WpParsed {
  bool regular, have, any_raw; bool irr;            // irr: some chunk's timestamps are not on the query's step grid (DDV residuals or slope != step)
  int tslope; uint32_t toff;                         // timestamp vector: slope, byte offset in R
  int n, cLo;
  int64_t init, end_time; int nrows, num_rows, vbytes, ng, vwire, dropped, tlen, grp_base, ngroups; uint32_t voff, w12;
};
// what one chunk's entry and vectors say (the per-lane part of wp_parse; okc: the chunk qualifies on its own)
template <bool STRICT, bool IRR>
__device__ __forceinline__ void wp_chunk_fields(const uint8_t* R, const ChunkEntry& e, const QueryParams& q, int64_t& init, int64_t& end_time, int& nrows,
                                                int& num_rows, int& vbytes, int& ng, int& vwire, int& dropped, int& tlen, uint32_t& voff, uint32_t& w12,
                                                bool& okc, bool& irrc, int& slope, uint32_t& toff) {
  const uint8_t* tv = R + e.ts_off; const uint8_t* vv = R + e.val_off;
  const uint32_t vw4 = ld32(vv + 4);
  vwire = (int)(vw4 & 0xffff); dropped = (int)((vw4 >> 31) & 1);
  toff = e.ts_off;
  const int twire = (int)(ld32(tv + 4) & 0xffff);
  if (!IRR || twire == WIRE_DDV_CONST) { tlen = (int)ld32(tv + 8); init = (int64_t)ld64_a4(tv + 12); slope = (int)ld32(tv + 20); if (IRR && twire != WIRE_DDV_CONST) okc = false; }
  else if (twire == WIRE_DDV) {                          // DeltaDeltaVector.scala:138-156: +8 init, +16 slope, +20 IntBinaryVector of residuals
    init = (int64_t)ld64(tv + 8); slope = (int)ld32(tv + 16); tlen = int_length(tv + 20); irrc = true;
    const int nb = (int)((ld32(tv + 24) >> 16) & 0x7f);
    if (!(nb == 2 || nb == 4 || nb == 8 || nb == 16 || nb == 32)) okc = false;
  } else okc = false;
  if (IRR && (int64_t)slope != q.step) irrc = true;
  end_time = e.end_time; num_rows = e.num_rows; voff = e.val_off;
  vbytes = (int)ld32(tv) + 4 + (int)ld32(vv) + 4;
  int vlen = 0;
  if (vwire == WIRE_XOR) { vlen = (int)ld32(vv + XOR_OFF_N); w12 = ld32(vv + XOR_OFF_NGROUPS); ng = (int)(w12 & 0xffff); if (ng != (vlen + 6) / 8) okc = false; }
  else if (vwire == WIRE_RAW64) vlen = ((int)ld32(vv) - 4) / 8;
  else okc = false;
  if ((!IRR && (int64_t)slope != q.step) || slope <= 0 || tlen <= 0 || vlen <= 0 || num_rows <= 0) okc = false;
  nrows = num_rows < tlen ? num_rows : tlen;
  if (vlen != nrows) okc = false;                       // the decode writes every row of the vector
  if (STRICT && end_time < init + (int64_t)(nrows - 1) * q.step) okc = false;
}

// STRICT (SUM class): endTime covers the chunk's rows and lies before the next chunk's first row, so that "has a row in the window" and
// "is in the window's chunk set" (ChunkSetInfo.scala:481-510) coincide; the counter class evaluates the chunk set itself
template <bool STRICT, bool IRR = false>
__device__ __forceinline__ WpParsed wp_parse(const uint8_t* R, const QueryParams& q, bool staged, int lane) {
  const unsigned FULL = 0xffffffffu;
  WpParsed P;
  bool regular = staged;
  int n = 0, cLo = 0;
  if (staged) {
    const RecordHeader* h = reinterpret_cast<const RecordHeader*>(R);
    const ChunkEntry* Eall = reinterpret_cast<const ChunkEntry*>(R + sizeof(RecordHeader));
    const int nch = (int)h->n_chunks;
    regular = nch <= 32 && (IRR || (h->flags & REC_ALL_TS_CONST) != 0);
    const int64_t t1 = q.start - q.window, t2 = q.end;
    bool below = false, within = false;
    if (regular && lane < nch) { below = Eall[lane].end_time < t1; within = !below && Eall[lane].start_time <= t2; }
    const unsigned mb = __ballot_sync(FULL, below), mw = __ballot_sync(FULL, within);
    cLo = __ffs((int)~mb) - 1; if (cLo < 0) cLo = 32;                         // chunks are time-ordered: `below` is a prefix
    const unsigned rest = cLo < 32 ? (mw >> cLo) : 0u;
    n = __ffs((int)~rest) - 1; if (n < 0) n = 32;
    if (n > WP_MAXC) regular = false;
  }
  const int c = lane;
  bool have = regular && c < n;
  int64_t init = 0, end_time = 0; int nrows = 0, num_rows = 0, vbytes = 0, ng = 0, vwire = 0, dropped = 0, tlen = 0; uint32_t voff = 0, w12 = 0;
  bool okc = true, irrc = false; int slope = 0; uint32_t toff = 0;
  if (have)
    wp_chunk_fields<STRICT, IRR>(R, reinterpret_cast<const ChunkEntry*>(R + sizeof(RecordHeader))[cLo + c], q, init, end_time, nrows, num_rows, vbytes, ng,
                                 vwire, dropped, tlen, voff, w12, okc, irrc, slope, toff);
  {
    const int64_t endp = __shfl_up_sync(FULL, end_time, 1);
    if (STRICT && have && c > 0 && !(endp < init)) okc = false;
    if (!__all_sync(FULL, okc)) regular = false;
  }
  have = have && regular;
  if (!have) { ng = 0; nrows = 0; }
  // group slots: exclusive prefix over the chunks
  int grp_base = ng;
  { const int a0 = __shfl_sync(FULL, ng, 0), a1 = __shfl_sync(FULL, ng, 1), a2 = __shfl_sync(FULL, ng, 2), a3 = __shfl_sync(FULL, ng, 3);
    grp_base = (c > 0 ? a0 : 0) + (c > 1 ? a1 : 0) + (c > 2 ? a2 : 0);
    if (a0 + a1 + a2 + a3 > WP_MAXG) regular = false; }
  P.ngroups = __shfl_sync(FULL, grp_base + ng, WP_MAXC - 1);
  P.any_raw = __any_sync(FULL, have && vwire == WIRE_RAW64);
  P.irr = IRR && __any_sync(FULL, have && irrc); P.tslope = slope; P.toff = toff;
  P.regular = regular; P.have = have && regular; P.n = n; P.cLo = cLo; P.init = init; P.end_time = end_time; P.nrows = nrows; P.num_rows = num_rows;
  P.vbytes = vbytes; P.ng = ng; P.vwire = vwire; P.dropped = dropped; P.tlen = tlen; P.grp_base = grp_base; P.voff = voff; P.w12 = w12;
  return P;
}

// Decode of a series into V: lane = NibblePack group (slots lane and lane + 32, described by dd_dst / dd_inf, see the plan); raw f64
// vectors are copied.  Returns the AND over every value v of hi(v) ^ (hi(v) << 1): bit 30 is set while every value has exponent bits
// 10 and 9 different, i.e. 2^-511 <= |v| < 2^513 (finite, normal, not zero).  DROPS (counter class): counter drops inside drop-flagged
// chunks (DoubleVector.scala:330-340) are recorded as (row, amount) in DR[chunk]; row r drops when (NaN -> 0) of it is below
// (NaN -> 0) of row r - 1, the amount is the value before the drop.
// r_done() is called, by the whole warp, as soon as R is not read any more: right after the field extraction, or after the raw copy when
// a chunk has raw f64 values (any_raw is the same on every lane).
struct WpNoop { __device__ __forceinline__ void operator()() const {} };
template <bool DROPS, typename RDone = WpNoop>
__device__ __forceinline__ uint32_t wp_decode(const uint8_t* R, double* V, const WpChunk* CD, uint64_t* xtab, const int dd_dst[2], const int dd_inf[2],
                                              int n, bool any_raw, int lane, TileDrops* DR, RDone r_done = RDone()) {
  uint32_t okbits = 0xffffffffu;
  uint64_t d[2][8];
#pragma unroll
  for (int jj = 0; jj < 2; ++jj) {
    const bool active = dd_inf[jj] & 1;
    const WpChunk& ch = CD[(dd_inf[jj] >> 1) & 3];
    const uint8_t* gp = R;
    if (active) gp = R + ch.grp_off + reinterpret_cast<const uint16_t*>(R + ch.tab_off)[dd_inf[jj] >> 8];
    const uint32_t mask = active ? gp[0] : 0u;
    const uint32_t hdr = gp[1];
    const uint32_t numBits = ((hdr >> 4) + 1) * 4;
    const uint32_t tz = (hdr & 0x0f) * 4;
    const uint64_t fm = (~0ull >> (64 - numBits)) << tz;       // the field's bits in the value
    // bit address (in shared memory) of the 64-bit window that has field 0 at bit tz
    uint32_t xb = (wp_soff(gp + 2) << 3) - tz;
    uint64_t x = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const bool on = (mask >> i) & 1u;
      const uint32_t wa = (xb >> 3) & ~3u;
      const uint32_t w0 = wp_lds32(wa), w1 = wp_lds32(wa + 4), w2 = wp_lds32(wa + 8);
      const uint32_t lo = __funnelshift_r(w0, w1, xb), hi = __funnelshift_r(w1, w2, xb);
      const uint64_t f = on ? fm : 0ull;
      x ^= (((uint64_t)hi << 32) | lo) & f;                    // running XOR of the fields, already shifted by tz
      xb += on ? numBits : 0u;
      d[jj][i] = x;
    }
  }
  if (!any_raw) r_done();
  // exclusive XOR scan of the group totals over the 64 slots
  uint64_t i0x = d[0][7], i1x = d[1][7];
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint64_t y0 = shfl_up_u64(i0x, o), y1 = shfl_up_u64(i1x, o);
    if (lane >= o) { i0x ^= y0; i1x ^= y1; }
  }
  const uint64_t tot0 = shfl_u64(i0x, 31);
  const uint64_t ex0 = i0x ^ d[0][7], ex1 = i1x ^ d[1][7] ^ tot0;
  xtab[lane] = ex0; xtab[32 + lane] = ex1;
  __syncwarp();
#pragma unroll
  for (int jj = 0; jj < 2; ++jj) {
    const bool active = dd_inf[jj] & 1;
    const int ci = (dd_inf[jj] >> 1) & 3;
    const WpChunk& ch = CD[ci];
    // value before the group = first ^ (prefix at the slot) ^ (prefix at the chunk's first slot)
    const uint64_t pre = ch.first ^ (jj ? ex1 : ex0) ^ xtab[active ? ch.grp_base : 0];
    uint64_t* dst = reinterpret_cast<uint64_t*>(V) + dd_dst[jj];
    const int t = (dd_inf[jj] >> 3) & 7;                       // rows t' with t + t' >= 8 sit one pad slot further
    if (active) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint64_t b = d[jj][i] ^ pre;
        dst[i + ((t + i) >> 3)] = b;
        const uint32_t h = (uint32_t)(b >> 32);
        okbits &= h ^ (h << 1);
      }
      if ((dd_inf[jj] >> 8) == 0) { dst[t == 0 ? -2 : -1] = ch.first; const uint32_t h = (uint32_t)(ch.first >> 32); okbits &= h ^ (h << 1); }
      if (DROPS && ch.dropped) {
        const int g = dd_inf[jj] >> 8;
        const int nleft = ch.nrows - 1 - g * 8;                // rows past the chunk are not data
        double prevv = nan0(__longlong_as_double((long long)pre));
        TileDrops& D = DR[ci];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const double cur = nan0(__longlong_as_double((long long)(d[jj][i] ^ pre)));
          if (i < nleft && cur < prevv) {                      // rare: position and amount (the value before the drop)
            const int at = atomicAdd(&D.n, 1);
            if (at < TILE_MAXDROP) { D.pos[at] = 1 + g * 8 + i; D.amt[at] = prevv; }
          }
          prevv = cur;
        }
      }
    }
  }
  // raw f64 vectors: plain copy
  for (int ci = 0; any_raw && ci < n; ++ci) {
    const WpChunk& ch = CD[ci];
    if (ch.wire != WIRE_RAW64) continue;
    const uint64_t* src = reinterpret_cast<const uint64_t*>(R + ch.val_off + 8);
    const bool drp = DROPS && ch.dropped;
    for (int r = lane; r < ch.nrows; r += 32) {
      const uint64_t b = src[r];
      reinterpret_cast<uint64_t*>(V)[wp_vidx(ch.rowpos + r)] = b;
      const uint32_t h = (uint32_t)(b >> 32);
      okbits &= h ^ (h << 1);
      if (drp && r > 0) {
        const double cur = nan0(__longlong_as_double((long long)b)), prevv = nan0(__longlong_as_double((long long)src[r - 1]));
        if (cur < prevv) { TileDrops& D = DR[ci]; const int at = atomicAdd(&D.n, 1); if (at < TILE_MAXDROP) { D.pos[at] = r; D.amt[at] = prevv; } }
      }
    }
  }
  if (any_raw) r_done();
  return okbits;
}

// Class of window k after the window blocks (chunks 0 .. n-1 of the plan in CD):
//   WP_FINAL   the window block left the finished value in O;
//   WP_RAWFIN  a raw sum in O: an own window of a block from tb on (that block stores raw sums because its later windows are shared);
//   WP_JUNC    a raw sum at J[jslot & 127] (the chunk's blocks [0, jzb)); jslot & 128: the window is in the chunk's head share, and the
//              earlier chunk's raw partial in O is added first (AggrOverTimeFunctions.scala:560-571);
//   WP_GAP     no chunk has rows in the window: NaN (the reference leaves the NaN seed).
constexpr uint32_t WP_FINAL = 0, WP_RAWFIN = 1, WP_JUNC = 2, WP_GAP = 3;
__device__ __forceinline__ int wp_chunk_of(const WpChunk* CD, int n, int k) {      // the last chunk with blocks whose kT0 <= k, or -1
  int ci = -1;
  for (int c = 0; c < n; ++c) if (CD[c].nblk > 0 && k >= CD[c].kT0) ci = c;
  return ci;
}
__device__ __forceinline__ uint32_t wp_class(const WpChunk* CD, int n, int k, uint32_t& jslot) {
  const int ci = wp_chunk_of(CD, n, k);
  jslot = 0;
  if (ci < 0 || k > CD[ci].kT1) return WP_GAP;
  const WpChunk& ch = CD[ci];
  const int i = k - ch.kT0;
  if (i < ch.jzb * WP_R) { jslot = (uint32_t)(ch.joff + i) | (i < ch.hs ? 128u : 0u); return WP_JUNC; }
  return i >= ch.tb * WP_R ? WP_RAWFIN : WP_FINAL;       // (a window past ownHi belongs to the next chunk's head share)
}
__device__ __forceinline__ int wp_rows_in(const WpChunk& x, int k, int Wr) {    // rows of chunk x in window k
  int lo = x.s0 + k; if (lo < 0) lo = 0; int hi = x.s0 + k + Wr; if (hi > x.nrows - 1) hi = x.nrows - 1;
  return hi - lo + 1;
}

// first slot of chunk c's raw tail partials in the raw tail area of scan_wp_batch_kernel: the chunks before it take (nblk - tb) blocks each
__device__ __forceinline__ int wp_tail_base(const WpChunk* CD, int c) {
  int t = 0;
#pragma unroll
  for (int x = 0; x < WP_MAXC - 1; ++x) if (x < c) t += CD[x].nblk - CD[x].tb;
  return WP_R * t;
}

// window block `it` of the plan: V index of its first row, byte offset (inside the warp's region) of its first result slot, and
// inf = (jEnd + 1) | raw << 4 | skew phase of the first slot << 5 | chunk << 8 | first window << 10, where slots 0 .. jEnd are stored.
// STAGE (scan_wp_batch_kernel): every block's slots are contiguous.  An own block's first slot is window k0 of the dense result row
// (O[k0], the row's phase h is added by the window blocks), a raw tail block's is in the raw tail area at byte offset rt.
template <bool STAGE = false>
__device__ __forceinline__ void wp_item(const WpChunk* CD, const WpSmem& L, int it, int items, int psi, int& pp, int& op, int& inf, uint32_t rt = 0) {
  const bool active = it < items;
  int ci = 0;                                             // the last chunk with blocks whose blk0 <= it
  if (CD[1].nblk > 0 && it >= CD[1].blk0) ci = 1;
  if (CD[2].nblk > 0 && it >= CD[2].blk0) ci = 2;
  if (CD[3].nblk > 0 && it >= CD[3].blk0) ci = 3;
  const WpChunk& ch = CD[ci];
  const int b = active ? it - ch.blk0 : 0;
  const int k0 = ch.kT0 + WP_R * b;
  pp = ch.vidx0 + 9 * b;
  const bool tojz = b < ch.jzb;                           // raw sums to J (every slot of the block exists there)
  const bool raw = tojz || b >= ch.tb;
  if (STAGE) op = tojz ? (int)WP_OFF_J + 8 * (ch.joff + WP_R * b) : b >= ch.tb ? (int)rt + 8 * (wp_tail_base(CD, ci) + WP_R * (b - ch.tb)) : (int)L.out + 8 * k0;
  else op = tojz ? (int)WP_OFF_J + 8 * (ch.joff + WP_R * b) : (int)L.out + 8 * (k0 + ((k0 + psi) >> 3));
  int jEnd = !active ? -1 : tojz ? WP_R - 1 : ch.kT1 - k0;
  if (jEnd > WP_R - 1) jEnd = WP_R - 1;
  const int ot = tojz || STAGE ? 0 : (k0 + psi) & 7;      // slots j with ot + j >= 8 sit one pad slot further
  inf = (jEnd + 1) | ((raw ? 1 : 0) << 4) | (ot << 5) | (ci << 8) | (k0 << 10);
}

// ---------------------------------------------------------------------------------------------------------------------
// Phases of a SUM-class series shared by scan_wp_sum_kernel and scan_wp_batch_kernel: the memo check and window plan, the zero rows,
// the window blocks and the finish-and-store pass.  A warp's plan state lives in registers (WpPlan) and in its descriptors CD.
// ---------------------------------------------------------------------------------------------------------------------
struct WpQuery {                       // per-query constants of the SUM-class phases
  double fdiv, frcp;                   // rate: the window length in ms and RN(1 / it) (RateFunctions.scala:436-442)
  int64_t S0, E0, lastEnd;             // window 0 spans [S0, E0]; the last window ends at lastEnd
  StepDiv sd;
  __device__ __forceinline__ void init(const QueryParams& q) {
    int64_t winDur = q.inclusive ? q.window : q.window - 1; if (winDur < 0) winDur = 0;
    fdiv = (double)(q.inclusive ? winDur : winDur + 1); frcp = 1.0 / fdiv;
    S0 = q.start - winDur; E0 = q.start;
    lastEnd = q.start + (int64_t)(q.T - 1) * q.step;
    sd.init(q.step);
  }
};
struct WpPlan {
  // memo of the window plan (lane c holds chunk c's key; the plan itself stays in CD)
  int64_t m_init = 0, m_end = 0; int m_nrows = -1, m_n = -1, m_wire = -1; bool m_ok = false;
  // per-lane work items of the plan: two decode slots and the two window blocks of the first pass (see the plan)
  int dd_dst[2] = {0, 0}, dd_inf[2] = {0, 0}, wi_pp[2] = {0, 0}, wi_op[2] = {0, 0}, wi_inf[2] = {0, 0};
  int gz[3] = {-1, -1, -1}; bool gz_all = true;      // this lane's zero rows (V indices) when the plan has at most 96 of them
  int p_Wr = 0, p_items = 0, p_nfull = 0, p_psi = 0; double p_rcpn = 0.0; bool p_oal = false;
  // classes of this lane's windows lane + 32 m, m < 16 (2 bits each, wp_class), and the J slots of its WP_JUNC windows among them in
  // window order (8 bits each: at most 6, since the J slots of the plan are at most 128 over at most 3 chunks)
  uint32_t p_cls = 0; uint64_t p_jx = 0;
};

// Memo check and, on a miss, the window plan of a regular series (lane c = chunk c, the fields wp_parse gives).  Clears `regular` when the
// plan declines the series.  Returns true on a memo miss.  STAGE: the work items of scan_wp_batch_kernel (wp_item<true>), raw tail area at
// byte offset rt with rtcap doubles.
template <bool STAGE = false>
__device__ __forceinline__ bool wp_plan_series(WpPlan& M, bool& regular, bool have, int n, int64_t init, int64_t end_time, int nrows, int vwire,
                                               int grp_base, int ngroups, const QueryParams& q, const WpSmem& L, const WpQuery& Q, WpChunk* CD, int lane,
                                               uint32_t rt = 0, uint32_t rtcap = 0) {
  const unsigned FULL = 0xffffffffu;
  const int c = lane;
  const bool samec = !(c < n) || (init == M.m_init && nrows == M.m_nrows && end_time == M.m_end && vwire == M.m_wire);
  const bool same_all = __all_sync(FULL, samec);
  const bool same = M.m_ok && n == M.m_n && same_all;
  const bool miss = regular && !same;
  if (miss) {
    M.m_init = init; M.m_end = end_time; M.m_nrows = nrows; M.m_n = n; M.m_wire = vwire; M.m_ok = false;
    int64_t s0 = 0, e0 = 0;
    if (have) { s0 = Q.sd.ceil_div(Q.S0 - init); e0 = Q.sd.floor_div(Q.E0 - init); }
    const int Wr = (int)(e0 - s0);
    int64_t kT0 = -e0; if (kT0 < 0) kT0 = 0;
    int64_t kT1 = (int64_t)(nrows - 1) - s0; if (kT1 > q.T - 1) kT1 = q.T - 1;
    const bool touch = have && kT0 <= kT1;
    if (!touch) { kT0 = 0x3fffffff; kT1 = -1; }
    const int Wr0 = __shfl_sync(FULL, Wr, 0);
    bool okp = !have || Wr == Wr0;
    if (Wr0 < 8 || (uint32_t)Wr0 + 1 > L.jcap) okp = false;
    // touched chunks must be contiguous, and a window may take rows from at most two chunks
    const unsigned tm = __ballot_sync(FULL, touch) & 0xfu;
    if (tm != 0) { const unsigned lowbit = tm & (0u - tm); const unsigned filled = tm + lowbit; if ((filled & (filled - 1)) != 0) okp = false; }
    const int64_t kT1p = __shfl_up_sync(FULL, kT1, 1), kT1pp = __shfl_up_sync(FULL, kT1, 2), kT0n = __shfl_down_sync(FULL, kT0, 1);
    const bool prev_t = c > 0 && ((tm >> (c - 1)) & 1u), next_t = c + 1 < WP_MAXC && ((tm >> (c + 1)) & 1u);
    if (touch && c >= 2 && ((tm >> (c - 2)) & 1u) && !(kT1pp < kT0)) okp = false;
    int64_t ownLo = kT0, ownHi = kT1;
    if (touch && prev_t && kT1p + 1 > ownLo) ownLo = kT1p + 1;
    if (touch && next_t && kT0n - 1 < ownHi) ownHi = kT0n - 1;
    const int hs = touch ? (int)(ownLo - kT0) : 0;
    const int nblk = touch ? (int)((kT1 - kT0 + WP_R) / WP_R) : 0;
    // whole blocks: [0, jzb) raw to J (the head share, rounded up), [tb, nblk) raw to O (from the block of ownHi + 1), own blocks in between
    const int jzb = (hs + WP_R - 1) / WP_R;
    const int tb = (touch && ownHi < kT1) ? (int)((ownHi + 1 - kT0) / WP_R) : nblk;
    if (touch && jzb > tb) okp = false;
    int blk0, items, joff, jtot;
    { const int a0 = __shfl_sync(FULL, nblk, 0), a1 = __shfl_sync(FULL, nblk, 1), a2 = __shfl_sync(FULL, nblk, 2), a3 = __shfl_sync(FULL, nblk, 3);
      blk0 = (c > 0 ? a0 : 0) + (c > 1 ? a1 : 0) + (c > 2 ? a2 : 0); items = a0 + a1 + a2 + a3; }
    { const int z = jzb * WP_R;
      const int a0 = __shfl_sync(FULL, z, 0), a1 = __shfl_sync(FULL, z, 1), a2 = __shfl_sync(FULL, z, 2), a3 = __shfl_sync(FULL, z, 3);
      joff = (c > 0 ? a0 : 0) + (c > 1 ? a1 : 0) + (c > 2 ? a2 : 0); jtot = a0 + a1 + a2 + a3; }
    if ((uint32_t)jtot > L.jcap) okp = false;
    if (STAGE) {                                            // (wp_batch_layout sizes the area for every plan: this never declines)
      const int t = nblk - tb;
      const int a0 = __shfl_sync(FULL, t, 0), a1 = __shfl_sync(FULL, t, 1), a2 = __shfl_sync(FULL, t, 2);
      if ((uint32_t)(WP_R * (a0 + a1 + a2)) > rtcap) okp = false;
    }
    if (L.alias && items > 64) okp = false;                 // O takes V's place: every block is summed before the first result is stored
    // row positions: chunk after chunk, Wr .. Wr + 7 zero rows in between, every chunk's block 0 at a multiple of 8
    const int fr = touch ? (int)(s0 + kT0) : 0;              // first row of block 0 (may be negative: zero rows in front)
    int rowpos = 0;
    {
      int base = 0;                                           // first position this chunk's rows may take
#pragma unroll
      for (int cc = 0; cc < WP_MAXC; ++cc) {
        int x;
        if (cc == 0) { x = fr < 0 ? -fr : ((8 - (fr & 7)) & 7); }
        else { x = base + ((-(base + fr)) & 7); }
        if (c == cc) rowpos = x;
        const int nb = __shfl_sync(FULL, x + nrows + Wr0, cc);   // (lane cc's own x is the valid one)
        base = nb;
      }
    }
    const int pend = __shfl_sync(FULL, rowpos + nrows, n > 0 ? n - 1 : 0) + Wr0 + 8;
    if ((uint32_t)(pend + (pend >> 3) + 2) > L.vcap) okp = false;
    if (!__all_sync(FULL, okp)) regular = false;
    if (regular) {
      if (c < WP_MAXC) {
        WpChunk& d = CD[c];
        d.kT0 = (int)kT0; d.kT1 = (int)kT1; d.ownLo = (int)ownLo; d.ownHi = (int)ownHi; d.blk0 = blk0; d.nblk = nblk;
        d.vidx0 = wp_vidx(rowpos + fr); d.rowpos = rowpos; d.nrows = nrows; d.s0 = (int)s0; d.e0 = (int)e0; d.joff = joff; d.hs = hs; d.jzb = jzb; d.tb = tb;
      }
      // O is skewed like V (one pad slot per 8 windows, block starts of the first touched chunk on the 9-word grid): the 8-byte result
      // stores of a warp (lane stride 8 windows) then spread over the banks.  p_oal: every chunk's blocks start on that grid
      { const int first_t = tm ? __ffs((int)tm) - 1 : 0;
        M.p_psi = (-(int)__shfl_sync(FULL, (int)(touch ? kT0 : 0), first_t)) & 7;
        M.p_oal = __all_sync(FULL, !touch || (((int)kT0 + M.p_psi) & 7) == 0); }
      M.p_Wr = Wr0; M.p_items = items; M.p_nfull = Wr0 + 1; M.p_rcpn = 1.0 / (double)(Wr0 + 1);
      __syncwarp();
      // zero rows: in front of chunk 0, between chunks, behind the last chunk (+ slack the last block's unused windows read).  They are
      // written again for every series (the group decode runs up to 7 rows past a chunk; with O in V's place the results land on them)
      {
        int tot = 0;
        M.gz[0] = M.gz[1] = M.gz[2] = -1;
        for (int g = 0; g <= n; ++g) {
          const int g0 = g == 0 ? 0 : CD[g - 1].rowpos + CD[g - 1].nrows;
          const int g1 = g == n ? pend : CD[g].rowpos;
#pragma unroll
          for (int u = 0; u < 3; ++u) { const int i = u * 32 + lane - tot; if (i >= 0 && i < g1 - g0) M.gz[u] = wp_vidx(g0 + i); }
          tot += g1 - g0;
        }
        M.gz_all = tot <= 96;
      }
      // window classes of the finish pass, for this lane's windows below T (windows from 512 on are classified in the pass itself)
      {
        uint32_t cls = 0; uint64_t jx = 0; int nj = 0;
#pragma unroll 1
        for (int m = 0; m < 16 && lane + 32 * m < q.T; ++m) {
          uint32_t js;
          const uint32_t code = wp_class(CD, n, lane + 32 * m, js);
          cls |= code << (2 * m);
          if (code == WP_JUNC) { jx |= (uint64_t)js << (8 * nj); ++nj; }
        }
        M.p_cls = cls; M.p_jx = jx;
      }
      // this lane's work items (they stay valid with the plan): decode slots lane, lane + 32 and window blocks lane, lane + 32
      {
        const int gb1 = __shfl_sync(FULL, have ? grp_base : 0x7fffffff, 1), gb2 = __shfl_sync(FULL, have ? grp_base : 0x7fffffff, 2),
                  gb3 = __shfl_sync(FULL, have ? grp_base : 0x7fffffff, 3);
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          const int slot = jj * 32 + lane;
          const bool active = slot < ngroups;
          const int ci = active ? (slot >= gb1 ? 1 : 0) + (slot >= gb2 ? 1 : 0) + (slot >= gb3 ? 1 : 0) : 0;
          const int gbc = ci == 0 ? 0 : ci == 1 ? gb1 : ci == 2 ? gb2 : gb3;
          const int g = active ? slot - gbc : 0;
          const int pq = CD[ci].rowpos + 1 + g * 8;
          M.dd_dst[jj] = wp_vidx(pq);
          M.dd_inf[jj] = (active ? 1 : 0) | (ci << 1) | ((pq & 7) << 3) | (g << 8);      // active, chunk, skew phase of the first row, group in chunk
        }
#pragma unroll
        for (int X = 0; X < 2; ++X) wp_item<STAGE>(CD, L, X * 32 + lane, items, M.p_psi, M.wi_pp[X], M.wi_op[X], M.wi_inf[X], rt);
      }
      M.m_ok = true;
    }
  }
  return miss;
}

// zero rows (the last group of an XOR chunk decoded up to 7 rows past the chunk; results of the previous series when O is in V's place)
__device__ __forceinline__ void wp_zero_rows(double* V, const WpChunk* CD, int n, const WpPlan& M, int lane) {
  if (M.gz_all) {
#pragma unroll
    for (int u = 0; u < 3; ++u) if (M.gz[u] >= 0) V[M.gz[u]] = 0.0;
  } else {
    const int pend = CD[n - 1].rowpos + CD[n - 1].nrows + M.p_Wr + 8;
    for (int g = 0; g <= n; ++g) {
      const int g0 = g == 0 ? 0 : CD[g - 1].rowpos + CD[g - 1].nrows;
      const int g1 = g == n ? pend : CD[g].rowpos;
      for (int pz = g0 + lane; pz < g1; pz += 32) V[wp_vidx(pz)] = 0.0;
    }
  }
}

// window blocks of a decoded series: two items per lane, 64 per pass, results (finished or raw) into O and J of the warp's region wb.
// STAGE (scan_wp_batch_kernel): an own block writes its finished windows k straight into the dense result row, O[k + h] (h: the row's
// phase, see wp_finish_store); raw tail blocks write to the raw tail area, head-share blocks to J.  With O on V the single __syncwarp
// between a pass's row loads and its stores separates the last read of V from the first write over it: O sits on V only when every
// plan is one pass of at most 64 items (WpSmem::alias; the plan declines longer ones, the host asserts it).  A block's 8 slots are
// stored in an order rotated by r = 4 ((lane >> 1) & 1): lane l's block starts 8 l windows on, so with the same slot order the lanes of
// one parity would all hit one bank pair (16 wavefronts per 8-byte store).  Rotated, step j stores slot (j + r) & 7 and each parity
// hits two bank pairs: 8 wavefronts per store, 64 per 32 items, for one stage of selects.  (Rotations over 4 and 8 slot orders, 32
// and 16 wavefronts per 32 items for two and three stages of selects, ran C2 slower on an H100: its per-series path is bound by
// issued instructions more than by shared-memory wavefronts.  Without rotation it ran slower than with the finish pass.)
template <int FN, bool STAGE = false>
__device__ __forceinline__ void wp_window_blocks(const double* V, uint8_t* wb, const WpChunk* CD, const WpSmem& L, const WpPlan& M, const WpQuery& Q,
                                                 int lane, int h = 0, uint32_t rt = 0) {
  const int psi = M.p_psi;
  const int Wr = M.p_Wr;
  for (int it0 = 0; it0 < M.p_items; it0 += 64) {
    int ipp[2], iop[2], iinf[2];
#pragma unroll
    for (int X = 0; X < 2; ++X) {
      if (it0 == 0) { ipp[X] = M.wi_pp[X]; iop[X] = M.wi_op[X]; iinf[X] = M.wi_inf[X]; }
      else wp_item<STAGE>(CD, L, it0 + X * 32 + lane, M.p_items, psi, ipp[X], iop[X], iinf[X], rt);
    }
    const double* pp[2]; double* op[2]; int jEnd[2], ot[2]; bool rawm[2];
#pragma unroll
    for (int X = 0; X < 2; ++X) {
      pp[X] = V + ipp[X]; op[X] = reinterpret_cast<double*>(wb + iop[X]);
      jEnd[X] = (iinf[X] & 15) - 1; rawm[X] = (iinf[X] >> 4) & 1; ot[X] = (iinf[X] >> 5) & 7;
      if (STAGE && !rawm[X]) op[X] += h;
    }
    double a[WP_R], bb[WP_R];
    wp_block_pair(pp[0], pp[1], Wr, a, bb);
    __syncwarp();                                       // (O may sit on V: every lane has read its rows)
#pragma unroll
    for (int X = 0; X < 2; ++X) {
      const double dv = rawm[X] ? 1.0 : Q.fdiv, rc = rawm[X] ? 1.0 : Q.frcp, sc = rawm[X] ? 1.0 : 1000.0;
#pragma unroll
      for (int j = 0; j < WP_R; ++j) {
        const double raw = X ? bb[j] : a[j];
        int nn = 1;
        if (FN == FN_AVG || FN == FN_COUNT) {
          const WpChunk& ch = CD[(iinf[X] >> 8) & 3];
          int lo = ch.s0 + (iinf[X] >> 10) + j; const int hi0 = lo + Wr; if (lo < 0) lo = 0;
          const int hi = hi0 > ch.nrows - 1 ? ch.nrows - 1 : hi0;
          nn = hi - lo + 1;
        }
        const double fin = wp_finish<FN>(raw, nn, dv, rc, sc, M.p_nfull, M.p_rcpn, rawm[X]);
        if (X) bb[j] = fin; else a[j] = fin;
      }
    }
    if (STAGE) {
      const int r = 4 * ((lane >> 1) & 1);
#pragma unroll
      for (int X = 0; X < 2; ++X) {
        double (&v)[WP_R] = X ? bb : a;
        double t[WP_R];                                   // v[j] = slot (j + r) & 7, by selects (no dynamic register index)
#pragma unroll
        for (int j = 0; j < WP_R; ++j) t[j] = r ? v[(j + 4) & 7] : v[j];
#pragma unroll
        for (int j = 0; j < WP_R; ++j) v[j] = t[j];
#pragma unroll
        for (int j = 0; j < WP_R; ++j) { const int sj = (j + r) & 7; if (sj <= jEnd[X]) op[X][sj] = v[j]; }
      }
    } else if (M.p_oal) {                               // every block starts on O's 9-word grid: constant store offsets
#pragma unroll
      for (int j = 0; j < WP_R; ++j) { if (j <= jEnd[0]) op[0][j] = a[j]; if (j <= jEnd[1]) op[1][j] = bb[j]; }
    } else {
#pragma unroll
      for (int j = 0; j < WP_R; ++j) {
        if (j <= jEnd[0]) op[0][j + ((ot[0] + j) >> 3)] = a[j];
        if (j <= jEnd[1]) op[1][j + ((ot[1] + j) >> 3)] = bb[j];
      }
    }
  }
  __syncwarp();
}

// finish and store: lane-consecutive windows, 256 contiguous bytes per store instruction; O index of window lane + 32 m = oidx(lane) + 36 m.
// STAGE (scan_wp_batch_kernel): the row is dense in O, window k at O[k + h] (h = 1 when the row starts at 8 mod 16, so that O + 2h and
// the row's window h are both 16-byte aligned).  The window blocks (wp_window_blocks<FN, true>) already wrote every WP_FINAL window there;
// this fix-up writes the others: junction sums (the earlier chunk's raw partial from the raw tail area RT first, then J), raw sums of own
// windows from RT, NaN for windows without rows.  Each window is written by one lane, and nothing the fix-up reads is written here.
// Then the row's span of windows [h, h + ((T - h) & ~1)) leaves as one bulk store issued by lane 0; the window outside the span (0 or
// T - 1, at most one each) is stored directly.  The caller waits for that store to have read O (wp_stage_wait) before anything writes V
// or O again.
template <int FN, bool STAGE = false>
__device__ __forceinline__ void wp_finish_store(double* __restrict__ out, int64_t s, const QueryParams& q, double* O, const double* J,
                                                const WpChunk* CD, int n, const WpPlan& M, const WpQuery& Q, int lane, const double* RT = nullptr,
                                                int h = 0) {
  const double NaNv = __longlong_as_double(0x7ff8000000000000LL);
  const int psi = M.p_psi, Wr = M.p_Wr;
  auto oidx = [&](int k) -> int { return k + ((k + psi) >> 3); };
  double* gp = out + (size_t)s * q.T + lane;
  const double* sp = O + oidx(lane);
  auto fin = [&](double o, uint32_t code, uint32_t js, int k) -> double {
    double v = o;
    if (code == WP_JUNC) { const double jv = J[js & 127u]; v = (js & 128u) ? o + jv : jv; }    // earlier chunk's partial first
    double r;
    if (FN == FN_COUNT) r = v;          // the raw blocks left (double) rows of their chunk: the junction sum is the window's count
    else {
      int nn = 1;
      if (FN == FN_AVG && (code == WP_RAWFIN || code == WP_JUNC)) {
        const int ci = wp_chunk_of(CD, n, k);
        nn = wp_rows_in(CD[ci], k, Wr);
        if (code == WP_JUNC && (js & 128u)) nn += wp_rows_in(CD[ci - 1], k, Wr);
      }
      r = wp_finish<FN>(v, nn, Q.fdiv, Q.frcp, 1000.0, M.p_nfull, M.p_rcpn, false);
    }
    return code == WP_FINAL ? o : code == WP_GAP ? NaNv : r;
  };
  uint32_t cls = M.p_cls; uint64_t jx = M.p_jx;
  auto fin_m = [&](double o, int k) -> double {        // windows lane + 32 m, m < 16: class from the plan, J slot from the cursor
    const uint32_t code = cls & 3u, js = (uint32_t)jx & 0xffu;
    cls >>= 2;
    if (code == WP_JUNC) jx >>= 8;
    return fin(o, code, js, k);
  };
  if (STAGE) {
    const int T = q.T;
    double* row = out + (size_t)s * T;
    // the raw partial of chunk c for window k, from the raw tail area
    auto tail = [&](int c, int k) -> double { return RT[wp_tail_base(CD, c) + k - CD[c].kT0 - WP_R * CD[c].tb]; };
    auto fix = [&](uint32_t code, uint32_t js, int k) {
      double o = 0.0;
      if (code == WP_RAWFIN) o = tail(wp_chunk_of(CD, n, k), k);
      else if (code == WP_JUNC && (js & 128u)) o = tail(wp_chunk_of(CD, n, k) - 1, k);
      O[k + h] = fin(o, code, js, k);
    };
    // windows lane + 32 m, m < 16, that the window blocks left unfinished: class from the plan, J slot from the cursor
    uint32_t nf = (cls | (cls >> 1)) & 0x55555555u;
    while (nf) {
      const int b = __ffs((int)nf) - 1;
      nf &= nf - 1;
      const uint32_t code = (cls >> b) & 3u;
      uint32_t js = 0;
      if (code == WP_JUNC) { js = (uint32_t)jx & 0xffu; jx >>= 8; }
      fix(code, js, lane + 16 * b);
    }
    for (int k = lane + 512; k < T; k += 32) {                  // windows from 512 on (multi-pass plans only)
      uint32_t js;
      const uint32_t code = wp_class(CD, n, k, js);
      if (code != WP_FINAL) fix(code, js, k);
    }
    fence_async_smem();                                         // the row's writes, before the bulk store reads them
    __syncwarp();
    if (lane == 0) {
      const int nb = (T - h) & ~1;
      if (h) wp_store_result(row, O[1]);
      if ((T - h) & 1) wp_store_result(row + T - 1, O[T - 1 + h]);
      if (nb > 0) tma_store_1d(row + h, O + 2 * h, (uint32_t)nb * 8u);
    }
    return;
  }
  int k = lane, iters = (q.T - lane + 31) >> 5;
  int rest = iters > 16 ? iters - 16 : 0;
  if (rest) iters = 16;
  for (; iters >= 4; iters -= 4, gp += 128, sp += 144, k += 128) {
    const double v0 = sp[0], v1 = sp[36], v2 = sp[72], v3 = sp[108];
    const double r0 = fin_m(v0, k), r1 = fin_m(v1, k + 32), r2 = fin_m(v2, k + 64), r3 = fin_m(v3, k + 96);
    wp_store_result(gp, r0); wp_store_result(gp + 32, r1); wp_store_result(gp + 64, r2); wp_store_result(gp + 96, r3);
  }
  for (; iters > 0; --iters, gp += 32, sp += 36, k += 32) wp_store_result(gp, fin_m(*sp, k));
  for (; rest > 0; --rest, gp += 32, sp += 36, k += 32) {      // windows from 512 on (multi-pass plans only)
    uint32_t js;
    const uint32_t code = wp_class(CD, n, k, js);
    wp_store_result(gp, fin(*sp, code, js, k));
  }
}
// the warp's previous result row (wp_finish_store<FN, true>) has been read out of O: V and O may be written again
__device__ __forceinline__ void wp_stage_wait(int lane) {
  if (lane == 0) tma_store_wait_read();
  __syncwarp();
}

// per-series parts of the descriptors (lane c = chunk c): what the decode reads of each chunk
__device__ __forceinline__ void wp_series_desc(WpChunk* CD, int c, bool have, int grp_base, int ng, int vwire, uint32_t voff, int dropped, uint64_t first,
                                               uint32_t grp_off, uint32_t tab_off) {
  if (c < WP_MAXC) {
    WpChunk& d = CD[c];
    d.grp_base = have ? grp_base : 0x7fffffff; d.ng = ng; d.wire = vwire; d.val_off = voff; d.dropped = dropped;
    d.first = first; d.grp_off = grp_off; d.tab_off = tab_off;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// SUM-class kernel: sum / avg / count_over_time, rate / increase on delta-temporality schemas.  No across-series aggregate.
// Every warp streams its own records (one or two record buffers per warp).
// ---------------------------------------------------------------------------------------------------------------------
template <int FN, int NW>
__global__ void __launch_bounds__(NW * 32, 1)
scan_wp_sum_kernel(const uint8_t* __restrict__ arena, const int64_t* __restrict__ rec_off, int64_t n_series, QueryParams q,
                   double* __restrict__ out, WpSmem L, int64_t* __restrict__ fallback_list, unsigned long long* __restrict__ fallback_count,
                   unsigned long long* d_counters, int* d_err) {
  extern __shared__ __align__(128) uint8_t smem[];
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t* wb = smem + (size_t)warp * L.per_warp;
  uint64_t* bar = reinterpret_cast<uint64_t*>(wb);
  WpChunk* CD = reinterpret_cast<WpChunk*>(wb + WP_OFF_DESC);
  uint64_t* xtab = reinterpret_cast<uint64_t*>(wb + WP_OFF_J);     // decode: exclusive XOR prefix per group slot (dead before J is written)
  double* J = reinterpret_cast<double*>(wb + WP_OFF_J);
  // R: this series' record; with two record buffers the warp's series alternate between them (stage = iteration & 1)
  const bool two = L.rec2 != 0;
  uint8_t* R = wb + WP_OFF_REC;
  double* V = reinterpret_cast<double*>(wb + L.vals);
  double* O = reinterpret_cast<double*>(wb + L.out);
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  int64_t s = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  if (lane == 0) { mbar_init(bar, 1); if (two) mbar_init(bar + 1, 1); mbar_fence_init(); }
  __syncwarp();

  WpQuery Q; Q.init(q);
  WpPlan M;
  int64_t rows_scanned = 0, bytes_scanned = 0;
  uint32_t parity = 0;

  auto issue = [&](int64_t off, uint32_t sz) {            // lane 0: fetch a record into R (the buffer of the current stage)
    uint64_t* b = bar + (R == wb + WP_OFF_REC ? 0 : 1);
    mbar_expect_tx(b, sz);
    tma_load_1d(R, arena + off, sz, b);
  };
  // cur_sz: size of the record of series s; with two buffers, nb_sz: of series s + nwarps (already in flight in the other buffer)
  uint32_t cur_sz = 0, nb_sz = 0;
  int64_t cur_off = 0;
  if (s < n_series) { cur_off = rec_off[s]; cur_sz = (uint32_t)(rec_off[s + 1] - cur_off); }
  if (s < n_series && cur_sz <= L.rec_cap && lane == 0) issue(cur_off, cur_sz);
  if (two && s + nwarps < n_series) {
    const int64_t o1 = rec_off[s + nwarps]; nb_sz = (uint32_t)(rec_off[s + nwarps + 1] - o1);
    R = wb + L.rec2;
    if (nb_sz <= L.rec_cap && lane == 0) issue(o1, nb_sz);
    R = wb + WP_OFF_REC;
  }
  uint32_t stage = 0;
  WPROF_DECL

  for (; s < n_series; s += nwarps) {
    // the record this iteration issues: series s + nwarps (one buffer) or s + 2 nwarps (two buffers), into this series' buffer
    const int64_t sn = s + (two ? 2 : 1) * nwarps;
    // its offsets: loaded here, their difference taken after the parse, so that the loads' latency passes behind it
    int64_t nxt_off = 0; uint32_t nxt_end = 0;                 // (the size needs the low word of the end only)
    if (sn < n_series) { nxt_off = rec_off[sn]; nxt_end = (uint32_t)rec_off[sn + 1]; }
    const bool staged = cur_sz <= L.rec_cap;
    WPROF_COUNT(10)
    WPROF(9)                                               // loop head (+ the declined series' exits)
    if (staged) { mbar_wait(bar + stage, (parity >> stage) & 1u); parity ^= 1u << stage; }      // bit b: phase of buffer b's mbarrier
    WPROF(0)                                               // wait: record
    // ------------------------------------------------------------------------------------------------ setup (lane c = chunk c)
    const WpParsed P = wp_parse<true>(R, q, staged, lane);
    const uint32_t nxt_sz = nxt_end - (uint32_t)nxt_off;
    WPROF(1)                                               // parse
    bool regular = P.regular;
    const bool have = P.have; const int n = P.n, c = lane;
    // ---- window plan, reused while the chunk shapes repeat
    if (wp_plan_series(M, regular, have, n, P.init, P.end_time, P.nrows, P.vwire, P.grp_base, P.ngroups, q, L, Q, CD, lane)) { WPROF_COUNT(11) }
    WPROF(2)                                               // memo check (+ window plan on a miss)
    if (!regular) {
      // declined: the v2 kernel answers this series
      WPROF_COUNT(12)
      if (lane == 0) { const unsigned long long slot = atomicAdd(fallback_count, 1ull); fallback_list[slot] = s; }
      __syncwarp();
      if (sn < n_series && nxt_sz <= L.rec_cap && lane == 0) issue(nxt_off, nxt_sz);
      if (two) { cur_sz = nb_sz; nb_sz = nxt_sz; stage ^= 1u; R = wb + (stage ? L.rec2 : WP_OFF_REC); } else cur_sz = nxt_sz;
      continue;
    }
    // per-series parts of the descriptors
    {
      const uint32_t voff = P.voff, po = P.w12 >> 16;
      const bool x = have && P.vwire == WIRE_XOR;
      wp_series_desc(CD, c, have, P.grp_base, P.ng, P.vwire, voff, P.dropped, x ? ld64(R + voff + po) : have ? ld64(R + voff + 8) : 0ull,
                     x ? voff + po + 8 : 0u, x ? voff + XOR_OFF_GROUPTAB : 0u);
    }
    // scan counters (CountingChunkInfoIterator, ChunkSetInfo.scala:336-380): every chunk in range is pulled, except one that starts
    // after the last window end
    int cnt_rows = 0, cnt_bytes = 0;
    { const int64_t endp = __shfl_up_sync(FULL, P.end_time, 1);
      if (have && !(c > 0 && !(endp < Q.lastEnd))) { cnt_rows = P.num_rows; cnt_bytes = P.vbytes; } }
#pragma unroll
    for (int o = 1; o < WP_MAXC; o <<= 1) { cnt_rows += __shfl_xor_sync(FULL, cnt_rows, o); cnt_bytes += __shfl_xor_sync(FULL, cnt_bytes, o); }
    __syncwarp();
    WPROF(3)                                               // per-series descriptors, scan counters
    // ------------------------------------------------------------------------------------------------ decode
    // R is dead once its fields are extracted: the next record's copy starts there and runs behind the rest of the decode and the
    // window phase (every lane has read its fields when the copy is issued)
    auto rec_done = [&]() {
      __syncwarp();
      if (sn < n_series && nxt_sz <= L.rec_cap && lane == 0) issue(nxt_off, nxt_sz);
    };
    const uint32_t okbits = wp_decode<false>(R, V, CD, xtab, M.dd_dst, M.dd_inf, n, P.any_raw, lane, nullptr, rec_done);
    const bool vals_ok = __all_sync(FULL, (okbits >> 30) & 1u);
    __syncwarp();
    if (two) { cur_sz = nb_sz; nb_sz = nxt_sz; stage ^= 1u; R = wb + (stage ? L.rec2 : WP_OFF_REC); } else cur_sz = nxt_sz;
    WPROF(4)                                               // decode (+ the next record's copy issued)
    wp_zero_rows(V, CD, n, M, lane);
    WPROF(5)                                               // zero rows
    if (!vals_ok) {
      // NaN / Inf / zero / denormal / very large or small values: the literal kernel answers (it needs the NaN-aware sums)
      WPROF_COUNT(13)
      if (lane == 0) { const unsigned long long slot = atomicAdd(fallback_count, 1ull); fallback_list[slot] = s; }
      __syncwarp();
      continue;
    }
    if (lane == 0) { rows_scanned += cnt_rows; bytes_scanned += cnt_bytes; }
    __syncwarp();
    // ------------------------------------------------------------------------------------------------ windows
    wp_window_blocks<FN>(V, wb, CD, L, M, Q, lane);
    WPROF(6)                                               // window blocks
    // ------------------------------------------------------------------------------------------------ finish and store
    wp_finish_store<FN>(out, s, q, O, J, CD, n, M, Q, lane);
    __syncwarp();
    WPROF(7)                                               // finish and store (slot 8 stays empty in this kernel)
  }
  WPROF(9)
  WPROF_FLUSH
  if (lane == 0) {
    if (rows_scanned | bytes_scanned) { atomicAdd(&d_counters[0], (unsigned long long)rows_scanned); atomicAdd(&d_counters[1], (unsigned long long)bytes_scanned); }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// SUM-class kernel with a CTA-wide record stream (L.consumers consumer warps + 1 producer warp, see WpBatchSmem).
//   producer  walks the CTA's batches of L.B consecutive series (batch g = blockIdx.x + i * gridDim.x, into buffer i % L.nbuf): loads
//             the batch's record offsets once, fetches its records with ONE cp.async.bulk (they are adjacent in the arena), and parses
//             every series' header with all 32 lanes (lane = series * 4 + chunk, eight series per pass) into one WpEntry per series;
//             the next batch's copy is in flight while it parses;
//   consumer  warp w takes the CTA's series w, w + consumers, ... in batch order, starts at the memo check with the entry's fields, and
//             runs the phases of scan_wp_sum_kernel.  It releases the record (and the entry) on the buffer's `empty` barrier as soon as
//             the decode has read it.
// Per buffer three mbarriers: full (the copy, tx count), parsed (the entries are written, producer -> consumers) and empty (count L.B:
// one arrival per series of the batch).  A partial batch is the last one of its CTA, so its buffer is never waited for again.
// ---------------------------------------------------------------------------------------------------------------------
// Producer-side cycle counters for profiling builds (-DFILO_WP_PROF): slots 16 .. 19 of g_wp_prof: stalled on the empty barrier,
// offsets + copy issue + waiting for the copy, parse and entries, batches; 20: producer warps.
#if defined(FILO_WP_PROF) && !defined(FILO_CUSIM)
#define WPPROD_DECL uint32_t wpq_t0 = (uint32_t)clock(), wpq_acc[4] = {0, 0, 0, 0};
#define WPPROD(i) { const uint32_t wpq_t1 = (uint32_t)clock(); wpq_acc[i] += wpq_t1 - wpq_t0; wpq_t0 = wpq_t1; }
#define WPPROD_COUNT { ++wpq_acc[3]; }
#define WPPROD_FLUSH if (lane == 0) { for (int wpq_i = 0; wpq_i < 4; ++wpq_i) atomicAdd(&g_wp_prof[16 + wpq_i], (unsigned long long)wpq_acc[wpq_i]); atomicAdd(&g_wp_prof[20], 1ull); }
#else
#define WPPROD_DECL
#define WPPROD(i)
#define WPPROD_COUNT
#define WPPROD_FLUSH
#endif

template <int FN, int NW>
__global__ void __launch_bounds__(NW * 32, 1)
scan_wp_batch_kernel(const uint8_t* __restrict__ arena, const int64_t* __restrict__ rec_off, int64_t n_series, QueryParams q,
                     double* __restrict__ out, WpBatchSmem BL, int64_t* __restrict__ fallback_list, unsigned long long* __restrict__ fallback_count,
                     unsigned long long* d_counters, int* d_err) {
  extern __shared__ __align__(128) uint8_t smem[];
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const WpSmem& L = BL.W;
  const int B = (int)BL.B, NB = (int)BL.nbuf, NC = (int)BL.consumers;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + BL.bars);
  uint64_t* parsed = full + NB;
  uint64_t* empty = parsed + NB;
  WpEntry* ENT = reinterpret_cast<WpEntry*>(smem + BL.ent);
  if (threadIdx.x == 0) {
    for (int b = 0; b < NB; ++b) { mbar_init(full + b, 1); mbar_init(parsed + b, 1); mbar_init(empty + b, B); }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == NC) {
    // ================================================================== producer warp: batch copies + header parse
    const int64_t t1 = q.start - q.window, t2 = q.end;
    const int64_t lastEnd = q.start + (int64_t)(q.T - 1) * q.step;
    const int c = lane & 3, lb = lane & 28;
    WPPROD_DECL
    // lanes 0 .. ns: rec_off[b0 + lane] of batch i (loaded one batch ahead of its copy)
    auto batch_start = [&](int i) -> int64_t { return ((int64_t)blockIdx.x + (int64_t)i * gridDim.x) * B; };
    auto load_offs = [&](int i) -> int64_t {
      const int64_t b0 = batch_start(i);
      int64_t o = 0;
      if (b0 < n_series && lane <= B && b0 + lane <= n_series) o = rec_off[b0 + lane];
      return o;
    };
    // issue batch i into its (released) buffer: one copy of its records, or a plain arrival when they do not fit
    auto issue = [&](int i, int64_t offs) {
      const int64_t b0 = batch_start(i);
      const int ns = (int)(n_series - b0 < B ? n_series - b0 : B);
      const int b = i % NB;
      const int64_t o0 = __shfl_sync(FULL, offs, 0), o1 = __shfl_sync(FULL, offs, ns);
      const uint32_t bytes = (uint32_t)(o1 - o0);
      if (lane == 0) {
        if (bytes <= BL.buf_cap) { mbar_expect_tx(full + b, bytes); tma_load_1d(smem + BL.buf + (size_t)b * BL.buf_stride, arena + o0, bytes, full + b); }
        else mbar_arrive(full + b);
      }
    };
    int64_t offs = load_offs(0), offs_n = 0;
    if (batch_start(0) < n_series) { issue(0, offs); offs_n = load_offs(1); }
    WPPROD(1)
    for (int i = 0; batch_start(i) < n_series; ++i) {
      const int64_t b0 = batch_start(i);
      const int ns = (int)(n_series - b0 < B ? n_series - b0 : B);
      const int b = i % NB, u = i / NB;
      const int64_t offs_c = offs;
      // the next batch's copy runs behind this batch's parse
      if (batch_start(i + 1) < n_series) {
        const int bn = (i + 1) % NB, un = (i + 1) / NB;
        if (un > 0) mbar_wait_parked(empty + bn, (un - 1) & 1);
        WPPROD(0)                                              // stalled on the empty barrier
        issue(i + 1, offs_n);
        offs = offs_n; offs_n = load_offs(i + 2);
      }
      const uint8_t* buf = smem + BL.buf + (size_t)b * BL.buf_stride;
      const uint32_t bytes = (uint32_t)(__shfl_sync(FULL, offs_c, ns) - __shfl_sync(FULL, offs_c, 0));
      const bool staged = bytes <= BL.buf_cap;
      mbar_wait(full + b, u & 1);
      WPPROD(1)                                                // offsets, copy issue, copy wait
      WpEntry* E = ENT + (size_t)b * B;
      for (int g = 0; g < ns; g += 8) {
        // ---------------------------------------------------------------- lane = series * 4 + chunk (the fields of wp_parse)
        const int sl = g + (lane >> 2);
        const bool present = sl < ns;
        const uint32_t rofs = (uint32_t)(__shfl_sync(FULL, offs_c, present ? sl : 0) - __shfl_sync(FULL, offs_c, 0));
        const uint8_t* R = buf + rofs;
        bool regular = present && staged;
        int nch = 0;
        if (regular) {
          const RecordHeader* h = reinterpret_cast<const RecordHeader*>(R);
          nch = (int)h->n_chunks;
          regular = nch <= 32 && (h->flags & REC_ALL_TS_CONST) != 0;
        }
        // chunks in range: `below` is a prefix of the time-ordered chunks, the ones `within` follow it; bits of chunks c, c + 4, ...
        uint32_t mb = 0, mw = 0;
        const ChunkEntry* Eall = reinterpret_cast<const ChunkEntry*>(R + sizeof(RecordHeader));
        for (int r = 0; __any_sync(FULL, regular && 4 * r < nch); ++r) {
          const int ci = 4 * r + c;
          bool below = false, within = false;
          if (regular && ci < nch) { below = Eall[ci].end_time < t1; within = !below && Eall[ci].start_time <= t2; }
          const unsigned bb = __ballot_sync(FULL, below), bw = __ballot_sync(FULL, within);
          mb |= ((bb >> lb) & 0xfu) << (4 * r); mw |= ((bw >> lb) & 0xfu) << (4 * r);
        }
        int cLo = __ffs((int)~mb) - 1; if (cLo < 0) cLo = 32;
        const unsigned rest = cLo < 32 ? (mw >> cLo) : 0u;
        int n = __ffs((int)~rest) - 1; if (n < 0) n = 32;
        if (n > WP_MAXC) regular = false;
        bool have = regular && c < n;
        int64_t init = 0, end_time = 0; int nrows = 0, num_rows = 0, vbytes = 0, ng = 0, vwire = 0, dropped = 0, tlen = 0; uint32_t voff = 0, w12 = 0;
        bool okc = true, irrc = false; int slope = 0; uint32_t toff = 0;
        if (have)
          wp_chunk_fields<true, false>(R, Eall[cLo + c], q, init, end_time, nrows, num_rows, vbytes, ng, vwire, dropped, tlen, voff, w12, okc, irrc, slope, toff);
        const int64_t endp = __shfl_up_sync(FULL, end_time, 1);
        if (have && c > 0 && !(endp < init)) okc = false;
        if (((__ballot_sync(FULL, okc) >> lb) & 0xfu) != 0xfu) regular = false;
        have = have && regular;
        if (!have) { ng = 0; nrows = 0; }
        const int a0 = __shfl_sync(FULL, ng, lb), a1 = __shfl_sync(FULL, ng, lb + 1), a2 = __shfl_sync(FULL, ng, lb + 2), a3 = __shfl_sync(FULL, ng, lb + 3);
        const int grp_base = (c > 0 ? a0 : 0) + (c > 1 ? a1 : 0) + (c > 2 ? a2 : 0);
        if (a0 + a1 + a2 + a3 > WP_MAXG) regular = false;
        const bool any_raw = ((__ballot_sync(FULL, have && vwire == WIRE_RAW64) >> lb) & 0xfu) != 0;
        have = have && regular;
        // what the decode reads of the chunk, and the chunk's share of the scan counters
        uint64_t first = 0; uint32_t grp_off = 0;
        if (have && vwire == WIRE_XOR) { const uint32_t po = w12 >> 16; first = ld64(R + voff + po); grp_off = voff + po + 8; }
        else if (have) first = ld64(R + voff + 8);
        int cnt_rows = 0, cnt_bytes = 0;
        if (have && !(c > 0 && !(endp < lastEnd))) { cnt_rows = num_rows; cnt_bytes = vbytes; }
        cnt_rows += __shfl_xor_sync(FULL, cnt_rows, 1); cnt_bytes += __shfl_xor_sync(FULL, cnt_bytes, 1);
        cnt_rows += __shfl_xor_sync(FULL, cnt_rows, 2); cnt_bytes += __shfl_xor_sync(FULL, cnt_bytes, 2);
        if (present) {
          WpEntry& e = E[sl];
          WpEntryChunk& ec = e.c[c];
          ec.first = first; ec.init = init; ec.end_time = end_time; ec.grp_off = grp_off; ec.val_off = voff;
          ec.nrows = nrows; ec.grp_base = grp_base; ec.ng = ng; ec.wire = (uint32_t)vwire | ((uint32_t)dropped << 16);
          if (c == 0) {
            e.rofs = rofs; e.n = n; e.flags = (regular ? 1 : 0) | (any_raw ? 2 : 0); e.ngroups = a0 + a1 + a2 + a3;
            e.cnt_rows = cnt_rows; e.cnt_bytes = cnt_bytes;
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(parsed + b);
      WPPROD(2)                                                // parse, entries
      WPPROD_COUNT
    }
    WPPROD_FLUSH
    return;
  }

  // ==================================================================== consumer warps
  uint8_t* wb = smem + (size_t)warp * L.per_warp;
  WpChunk* CD = reinterpret_cast<WpChunk*>(wb + WP_OFF_DESC);
  uint64_t* xtab = reinterpret_cast<uint64_t*>(wb + WP_OFF_J);     // decode: exclusive XOR prefix per group slot (dead before J is written)
  double* J = reinterpret_cast<double*>(wb + WP_OFF_J);
  double* V = reinterpret_cast<double*>(wb + L.vals);
  double* O = reinterpret_cast<double*>(wb + L.out);
  const int c = lane;
  WpQuery Q; Q.init(q);
  WpPlan M;
  int64_t rows_scanned = 0, bytes_scanned = 0;
  // this warp's series: position p = warp + NC k of the CTA's series, = slot `slot` of the CTA's batch i
  int i = warp / B, slot = warp % B;
  WPROF_DECL
  for (;; slot += NC) {
    while (slot >= B) { slot -= B; ++i; }
    const int64_t s = ((int64_t)blockIdx.x + (int64_t)i * gridDim.x) * B + slot;
    if (s >= n_series) break;
    const int b = i % NB, u = i / NB;
    WPROF_COUNT(10)
    WPROF(9)                                               // loop head (+ the declined series' exits)
    mbar_wait(parsed + b, u & 1);
    mbar_wait(full + b, u & 1);                            // already complete (the producer saw it); orders the copy's writes
    WPROF(0)                                               // wait: entry and record
    const WpEntry& e = ENT[(size_t)b * B + slot];
    const uint8_t* R = smem + BL.buf + (size_t)b * BL.buf_stride + e.rofs;
    const int n = e.n, flags = e.flags;
    bool regular = flags & 1;
    const bool have = regular && c < n;
    int64_t init = 0, end_time = 0; int nrows = 0, grp_base = 0, ng = 0, wire = 0; uint32_t voff = 0, grp_off = 0; uint64_t first = 0;
    if (c < WP_MAXC) {
      const WpEntryChunk& ec = e.c[c];
      init = ec.init; end_time = ec.end_time; nrows = ec.nrows; grp_base = ec.grp_base; ng = ec.ng; wire = (int)ec.wire;
      voff = ec.val_off; grp_off = ec.grp_off; first = ec.first;
    }
    const int vwire = wire & 0xffff;
    WPROF(1)                                               // entry
    if (wp_plan_series<true>(M, regular, have, n, init, end_time, nrows, vwire, grp_base, e.ngroups, q, L, Q, CD, lane, BL.rt, BL.rtcap)) { WPROF_COUNT(11) }
    WPROF(2)                                               // memo check (+ window plan on a miss)
    if (!regular) {
      // declined: the v2 kernel answers this series
      WPROF_COUNT(12)
      __syncwarp();
      if (lane == 0) {
        const unsigned long long fs = atomicAdd(fallback_count, 1ull); fallback_list[fs] = s;
        mbar_arrive(empty + b);
      }
      __syncwarp();
      continue;
    }
    wp_series_desc(CD, c, have, grp_base, ng, vwire, voff, wire >> 16, first, grp_off, have && vwire == WIRE_XOR ? voff + XOR_OFF_GROUPTAB : 0u);
    const int cnt_rows = e.cnt_rows, cnt_bytes = e.cnt_bytes;
    const bool any_raw = (flags & 2) != 0;
    __syncwarp();
    WPROF(3)                                               // per-series descriptors, scan counters
    wp_stage_wait(lane);                                   // the previous row's bulk store has read O (O may sit on V)
    WPROF(8)                                               // wait: previous result row's bulk store
    // ------------------------------------------------------------------------------------------------ decode
    // the record and the entry are dead once the fields are extracted: this series' share of the buffer is released
    auto rec_done = [&]() {
      __syncwarp();
      if (lane == 0) mbar_arrive(empty + b);
    };
    const uint32_t okbits = wp_decode<false>(R, V, CD, xtab, M.dd_dst, M.dd_inf, n, any_raw, lane, nullptr, rec_done);
    const bool vals_ok = __all_sync(FULL, (okbits >> 30) & 1u);
    __syncwarp();
    WPROF(4)                                               // decode (+ the record released)
    wp_zero_rows(V, CD, n, M, lane);
    WPROF(5)                                               // zero rows
    if (!vals_ok) {
      // NaN / Inf / zero / denormal / very large or small values: the literal kernel answers (it needs the NaN-aware sums)
      WPROF_COUNT(13)
      if (lane == 0) { const unsigned long long fs = atomicAdd(fallback_count, 1ull); fallback_list[fs] = s; }
      __syncwarp();
      continue;
    }
    if (lane == 0) { rows_scanned += cnt_rows; bytes_scanned += cnt_bytes; }
    __syncwarp();
    // ------------------------------------------------------------------------------------------------ windows
    // the row's phase: h = 1 when out + s T is 8 mod 16 (filo_query_device writes into a caller's buffer)
    const int h = (int)((reinterpret_cast<uintptr_t>(out + s * q.T) >> 3) & 1);
    wp_window_blocks<FN, true>(V, wb, CD, L, M, Q, lane, h, BL.rt);
    WPROF(6)                                               // window blocks (finished windows into the dense row)
    // ------------------------------------------------------------------------------------------------ fix-up and store
    wp_finish_store<FN, true>(out, s, q, O, J, CD, n, M, Q, lane, reinterpret_cast<const double*>(wb + BL.rt), h);
    __syncwarp();
    WPROF(7)                                               // fix-up and store
  }
  WPROF(9)
  WPROF_FLUSH
  if (lane == 0) {
    tma_store_wait_all();
    if (rows_scanned | bytes_scanned) { atomicAdd(&d_counters[0], (unsigned long long)rows_scanned); atomicAdd(&d_counters[1], (unsigned long long)bytes_scanned); }
  }
}

} // namespace filo
