// v4 scan path, counter class: rate / increase on cumulative schemas (counter correction + Prometheus extrapolation) and delta, on the
// per-warp pipeline of scan_wp.cuh (one warp per series, TMA-staged record, group decode into V, no CTA barriers after start-up).
//
// Window phase, warp <-> series and lanes over windows:
//   * windows whose rows sit unclamped inside one chunk: the sample times move with the window, so durationToStart / End,
//     sampledInterval and numSamples of RateFunctions.extrapolatedRate (RateFunctions.scala:72-111) are per-chunk constants of the plan;
//     a window costs two row loads, the correction lookup, one subtraction, a test that rules out the zero-point clamp without
//     dividing, one multiply and the exact invariant-divisor division;
//   * clamped single-chunk windows: a per-query table indexed by (numSamples - 1);
//   * everything else (chunk junctions, windows before / after the data): the literal CounterChunkedRangeFunction fold
//     (RangeFunction.scala:131-172, RateFunctions.scala:230-285, DoubleVector.scala:177-207, 375-391).
// Counter drops of drop-flagged chunks are found during the decode (wp_decode<true>), sorted and prefix-summed per chunk.
// Results: per-series rows leave lane-consecutive straight from registers (coalesced 8-byte stores, no staging);  with AGG the
// series of one work item (<= seg series of ONE group, positions of `order`) are folded into a per-warp accumulator row in shared memory
// and leave as one mergeable partial row per item (pval / pcnt, same contract as scan_agg_kernel_v2 and the tile kernel).
#pragma once
#include "scan_wp.cuh"

namespace filo {

// correction accumulated up to and including row r.  The list has been sorted by position and its amounts replaced by their
// running sums in position order (start of the window phase) -- the same additions as the reference's running
// `_correction += last` -- so the answer is the entry of the last drop at or before r.
__device__ __forceinline__ double drops_cum(const TileDrops& D, int r) {
  const int n = D.n < TILE_MAXDROP ? D.n : TILE_MAXDROP;
  double cum = 0.0;
#pragma unroll
  for (int j = 0; j < TILE_MAXDROP; ++j) if (j < n && D.pos[j] <= r) cum = D.amt[j];
  return cum;
}

// RateFunctions.extrapolatedRate (RateFunctions.scala:72-111), same operations in the same order; the divisions by the constants
// 1000 and (windowEnd - windowStart) use the exact invariant-divisor sequence, and the zero-point quotient is only formed
// when durationToZero can be below durationToStart: v1 * sI > 2 * dTS * delta  =>  sI * (v1 / delta) >= dTS
template <bool IS_COUNTER, bool IS_RATE>
__device__ __forceinline__ double extrapolated_rate_tile(int64_t windowStart, int64_t windowEnd, int32_t numSamples, int64_t t1, double v1,
                                                         int64_t t2, double v2, double fdiv, double frcp, int64_t step, const TileCtrTab* tab) {
  double durationToStart = div_invariant((double)(t1 - windowStart), 1000.0, 0.001);
  const double durationToEnd = div_invariant((double)(windowEnd - t2), 1000.0, 0.001);
  const int64_t si_ms = t2 - t1;
  const int m = numSamples - 1;
  double sampledInterval, extrapolationThreshold, half, rcpSI;
  if (m <= TILE_CTR_TABMAX && si_ms == (int64_t)m * step) {      // samples m steps apart: the terms depend on m only (see the table)
    const TileCtrTab e = tab[m];
    sampledInterval = e.sI; extrapolationThreshold = e.thr; half = e.half; rcpSI = e.rcpSI;
  } else {
    sampledInterval = div_invariant((double)si_ms, 1000.0, 0.001);
    const double averageDurationBetweenSamples = ddiv_rare(sampledInterval, (double)numSamples - 1.0);
    extrapolationThreshold = averageDurationBetweenSamples * 1.1; half = averageDurationBetweenSamples / 2.0; rcpSI = 0.0;
  }
  const double delta = v2 - v1;
  if (IS_COUNTER && delta > 0 && v1 >= 0) {
    if (!(v1 * sampledInterval > 2.0 * durationToStart * delta)) {
      const double durationToZero = sampledInterval * ddiv_rare(v1, delta);
      if (durationToZero < durationToStart) durationToStart = durationToZero;
    }
  }
  double extrapolateToInterval = sampledInterval;
  extrapolateToInterval += (durationToStart < extrapolationThreshold) ? durationToStart : half;
  extrapolateToInterval += (durationToEnd < extrapolationThreshold) ? durationToEnd : half;
  const double ratio = rcpSI != 0.0 ? div_invariant(extrapolateToInterval, sampledInterval, rcpSI) : ddiv_rare(extrapolateToInterval, sampledInterval);
  const double scaledDelta = delta * ratio;
  return IS_RATE ? __dmul_rn(div_invariant(scaledDelta, fdiv, frcp), 1000.0) : scaledDelta;
}

__device__ __forceinline__ double wp_row(const double* V, const WpCtrChunk& ch, int r) { return V[wp_vidx(ch.rowpos + r)]; }
// value of row r as the counter functions see it: CorrectingDoubleVectorReader.corrected for a drop-flagged chunk, raw otherwise
__device__ __forceinline__ double wp_ctr_value(const double* V, const WpCtrChunk& ch, int r, const TileDrops& D, bool dropped) {
  const double x = wp_row(V, ch, r);
  if (!dropped) return x;
  return nan0(x) + drops_cum(D, r);
}

// literal per-chunk fold of the counter functions for one window of a regular series: CounterChunkedRangeFunction.addChunks
// (RangeFunction.scala:131-172), ChunkedRateFunctionBase (RateFunctions.scala:230-285), correction carry
// (DoubleVector.scala:177-207, 375-391), over the skewed V layout
template <int FN>
__device__ __forceinline__ double wp_eval_counter(int n, const WpCtrChunk* K, const WpChunk* CD, const TileDrops* DR, const double* V, int64_t qstep, int qinclusive,
                                                  int64_t wStart, int64_t wEnd, int k, double fdiv, double frcp, const TileCtrTab* tab) {
  const double NaNv = __longlong_as_double(0x7ff8000000000000LL);
  int32_t numSamples = 0; int64_t loT = INT64_MAX, hiT = 0; double loV = NaNv, hiV = NaNv;
  bool some = false; double corrLast = 0.0, corr = 0.0;                // correctionMeta
  for (int c = 0; c < n; ++c) {
    const WpCtrChunk& ch = K[c];
    if (ch.end_time < wStart) continue;                                // ChunkSetInfo.scala:481-510
    if (c > 0 && !(K[c - 1].end_time < wEnd)) continue;
    int su = ch.s0 + k; if (su < 0) su = 0;
    int eu = ch.e0 + k; if (eu > ch.nrows - 1) eu = ch.nrows - 1;
    const double first = __longlong_as_double((long long)CD[c].first);
    if (FN != FN_DELTA && some) { if (first != first || first < corrLast) corr = corr + corrLast; }
    if (su <= eu) {
      const int64_t tS = ch.init + (int64_t)su * qstep, tE = ch.init + (int64_t)eu * qstep;
      const bool skip = FN != FN_DELTA && su == 0 && eu == 0 && first != first;      // RateFunctions.scala:255-256
      if (!skip && (tS < loT || tE > hiT)) {
        numSamples += eu - su + 1;
        const bool drp = FN != FN_DELTA && ch.kc.dropped;
        if (tS < loT) { loT = tS; const double b = wp_ctr_value(V, ch, su, DR[c], drp); loV = (FN != FN_DELTA && some) ? b + corr : b; }
        if (tE > hiT) { hiT = tE; const double b = wp_ctr_value(V, ch, eu, DR[c], drp); hiV = (FN != FN_DELTA && some) ? b + corr : b; }
      }
    }
    if (FN != FN_DELTA) {
      if (ch.kc.dropped) {                                               // CorrectingDoubleVectorReader.updateCorrection, :375-391
        int idx = ch.nrows - 1; double lastValue = 0.0;
        do { lastValue = wp_row(V, ch, idx); idx -= 1; } while (lastValue != lastValue && idx >= 0);
        corrLast = nan0(lastValue); corr = (some ? corr : 0.0) + drops_cum(DR[c], ch.nrows - 1);
      }
      else { corrLast = wp_row(V, ch, ch.nrows - 1); corr = some ? corr : 0.0; }
    }
    some = true;
  }
  const int64_t cws = qinclusive ? wStart : wStart - 1;                // RateFunctions.scala:270-285
  if (hiT > loT) return extrapolated_rate_tile<FN != FN_DELTA, FN == FN_RATE>(cws, wEnd, numSamples, loT, loV, hiT, hiV, fdiv, frcp, qstep, tab);
  return NaNv;
}

// ---- irregular timestamps (DDV with residuals, or a scrape interval that differs from the query step): row times live in TSR as int32
// offsets from the chunk's first timestamp (TSR[rowpos + r] = ts(r) - init); row ranges by a (float) guess on the chunk's slope + a short walk
// (exact for any data: the walk ends at the first row with ts >= t)
__device__ __forceinline__ int wp_irr_lower(const int32_t* TSR, const WpCtrChunk& ch, int64_t t) {
  const int64_t d64 = t - ch.init;
  if (d64 <= 0) return 0;
  const int32_t* p = TSR + ch.rowpos;
  const int nr = ch.nrows;
  if (d64 > (int64_t)p[nr - 1]) return nr;
  const int32_t d = (int32_t)d64;                          // 0 < d <= last row's offset: 32-bit from here on
  int g = (int)((float)d * __int_as_float(ch.kc.pad));     // kc.pad holds the bits of (float)(1 / slope) for an irregular series; the walk makes it exact
  if (g > nr - 1) g = nr - 1;
  while (g < nr && p[g] < d) ++g;
  while (g > 0 && p[g - 1] >= d) --g;
  return g;
}
// the literal fold of wp_eval_counter with searched row ranges and stored sample times
template <int FN>
__device__ __forceinline__ double wp_eval_counter_irr(int n, const WpCtrChunk* K, const WpChunk* CD, const TileDrops* DR, const double* V, const int32_t* TSR,
                                                      int64_t qstep, int qinclusive, int64_t wStart, int64_t wEnd, double fdiv, double frcp, const TileCtrTab* tab) {
  const double NaNv = __longlong_as_double(0x7ff8000000000000LL);
  int32_t numSamples = 0; int64_t loT = INT64_MAX, hiT = 0; double loV = NaNv, hiV = NaNv;
  bool some = false; double corrLast = 0.0, corr = 0.0;
  for (int c = 0; c < n; ++c) {
    const WpCtrChunk& ch = K[c];
    if (ch.end_time < wStart) continue;                                // ChunkSetInfo.scala:481-510
    if (c > 0 && !(K[c - 1].end_time < wEnd)) continue;
    const int su = wp_irr_lower(TSR, ch, wStart);
    int eu = wp_irr_lower(TSR, ch, wEnd + 1) - 1; if (eu > ch.nrows - 1) eu = ch.nrows - 1;
    const double first = __longlong_as_double((long long)CD[c].first);
    if (FN != FN_DELTA && some) { if (first != first || first < corrLast) corr = corr + corrLast; }
    if (su <= eu) {
      const int64_t tS = ch.init + (int64_t)TSR[ch.rowpos + su], tE = ch.init + (int64_t)TSR[ch.rowpos + eu];
      const bool skip = FN != FN_DELTA && su == 0 && eu == 0 && first != first;      // RateFunctions.scala:255-256
      if (!skip && (tS < loT || tE > hiT)) {
        numSamples += eu - su + 1;
        const bool drp = FN != FN_DELTA && ch.kc.dropped;
        if (tS < loT) { loT = tS; const double b = wp_ctr_value(V, ch, su, DR[c], drp); loV = (FN != FN_DELTA && some) ? b + corr : b; }
        if (tE > hiT) { hiT = tE; const double b = wp_ctr_value(V, ch, eu, DR[c], drp); hiV = (FN != FN_DELTA && some) ? b + corr : b; }
      }
    }
    if (FN != FN_DELTA) {
      if (ch.kc.dropped) {                                               // CorrectingDoubleVectorReader.updateCorrection, :375-391
        int idx = ch.nrows - 1; double lastValue = 0.0;
        do { lastValue = wp_row(V, ch, idx); idx -= 1; } while (lastValue != lastValue && idx >= 0);
        corrLast = nan0(lastValue); corr = (some ? corr : 0.0) + drops_cum(DR[c], ch.nrows - 1);
      }
      else { corrLast = wp_row(V, ch, ch.nrows - 1); corr = some ? corr : 0.0; }
    }
    some = true;
  }
  const int64_t cws = qinclusive ? wStart : wStart - 1;                // RateFunctions.scala:270-285
  if (hiT > loT) return extrapolated_rate_tile<FN != FN_DELTA, FN == FN_RATE>(cws, wEnd, numSamples, loT, loV, hiT, hiV, fdiv, frcp, qstep, tab);
  return NaNv;
}

// NaN results are counted per window (rare: kept out of line so that the read-modify-write is not predicated into the common path)
#ifdef FILO_CUSIM
inline void wp_bump_u16(uint16_t* p) { *p = (uint16_t)(*p + 1); }
#else
static __device__ __noinline__ void wp_bump_u16(uint16_t* p) { *p = (uint16_t)(*p + 1); }
#endif
// one clamped single-chunk window
template <int FN>
__device__ __forceinline__ double wp_clamped_window(const double* V, const WpCtrChunk& ch, const TileDrops& D, bool drp, int kk, int64_t wEnd, int64_t cws, int64_t qstep,
                                                   double fdiv, double frcp, const TileCtrTab* tab) {
  int r1 = ch.s0 + kk; if (r1 < 0) r1 = 0;
  int r2 = ch.e0 + kk; if (r2 > ch.nrows - 1) r2 = ch.nrows - 1;
  if (!(r2 > r1)) return __longlong_as_double(0x7ff8000000000000LL);      // highestTime > lowestTime (RateFunctions.scala:271,284)
  double v1 = wp_row(V, ch, r1), v2 = wp_row(V, ch, r2);
  if (drp) { v1 = nan0(v1) + drops_cum(D, r1); v2 = nan0(v2) + drops_cum(D, r2); }
  return extrapolated_rate_tile<FN != FN_DELTA, FN == FN_RATE>(cws, wEnd, r2 - r1 + 1, ch.init + (int64_t)r1 * qstep, v1, ch.init + (int64_t)r2 * qstep, v2,
                                                              fdiv, frcp, qstep, tab);
}

// IRR: the table has timestamp vectors off the step grid (its own instantiation: the regular kernel keeps its code and register budget)
// MOM (with AGG, agg_op = AGG_SUM): stddev / stdvar moments, a second [T] row of Σv² in the warp's region behind the NaN counts
// (wp_ctr_layout sizes it only for this mode), its partial rows at pval + n_items * T
template <int FN, bool AGG, int NW, bool IRR = false, bool MOM = false>
__global__ void __launch_bounds__(NW * 32, 1)
scan_wp_ctr_kernel(const uint8_t* __restrict__ arena, const int64_t* __restrict__ rec_off, int64_t n_series, QueryParams q,
                   double* __restrict__ out, WpCtrSmem L, int64_t* __restrict__ fallback_list, unsigned long long* __restrict__ fallback_count,
                   unsigned long long* d_counters, int* d_err,
                   const int32_t* __restrict__ order, const int64_t* __restrict__ item_begin, int64_t n_items, int agg_op,
                   double* __restrict__ pval, uint32_t* __restrict__ pcnt) {
  extern __shared__ __align__(128) uint8_t smem[];
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t* wb = smem + (size_t)warp * L.per_warp;
  uint64_t* bar = reinterpret_cast<uint64_t*>(wb);
  WpChunk* CD = reinterpret_cast<WpChunk*>(wb + WP_OFF_DESC);
  uint64_t* xtab = reinterpret_cast<uint64_t*>(wb + WP_OFF_J);
  TileDrops* DR = reinterpret_cast<TileDrops*>(wb + WP_OFF_DROPS);
  uint8_t* R = wb + WP_OFF_REC;
  double* V = reinterpret_cast<double*>(wb + L.vals);
  WpCtrChunk* KC = reinterpret_cast<WpCtrChunk*>(wb + L.kc);
  double* ACC = reinterpret_cast<double*>(wb + L.acc);
  MomOnly<MOM, double*> ACC2;
  if constexpr (MOM) ACC2.v = reinterpret_cast<double*>(wb + L.nbad + align_up((uint32_t)q.T * 2u, 16));
  uint16_t* NBAD = reinterpret_cast<uint16_t*>(wb + L.nbad);
  int32_t* TSR = reinterpret_cast<int32_t*>(wb + L.tsr);                 // (L.tsr == 0: tables with const-DDV timestamps only; never read then)
  constexpr bool allow_irr = IRR;
  TileCtrTab* CTAB = reinterpret_cast<TileCtrTab*>(smem + L.tab);
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t gw = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  if (lane == 0) { mbar_init(bar, 1); mbar_fence_init(); }
  // extrapolation terms of RateFunctions.scala:74-77,92 for samples m steps apart: sampledInterval = (m * step) / 1000,
  // averageDurationBetweenSamples = sampledInterval / (numSamples - 1) with numSamples - 1 = m
  if ((int)threadIdx.x <= TILE_CTR_TABMAX) {
    const int m = threadIdx.x;
    TileCtrTab& e = CTAB[m];
    const double sI = (double)((int64_t)m * q.step) / 1000.0;
    const double avg = sI / ((double)(m + 1) - 1.0);
    e.sI = sI; e.thr = avg * 1.1; e.half = avg / 2.0; e.rcpSI = m > 0 ? 1.0 / sI : 0.0;
  }
  __syncthreads();                      // (the only CTA-wide barrier: the table is read-only from here on)

  int64_t winDur = q.inclusive ? q.window : q.window - 1; if (winDur < 0) winDur = 0;
  const double fdiv = (double)(q.inclusive ? winDur : winDur + 1), frcp = 1.0 / fdiv;
  const int64_t S0 = q.start - winDur, E0 = q.start;
  const int64_t lastEnd = q.start + (int64_t)(q.T - 1) * q.step;
  StepDiv sd; sd.init(q.step);
  const double NaNv = __longlong_as_double(0x7ff8000000000000LL);
  const double agg_ident = agg_op == AGG_MIN ? __longlong_as_double(0x7ff0000000000000LL)
                         : agg_op == AGG_MAX ? __longlong_as_double(0xfff0000000000000LL) : 0.0;

  // memo of the plan (lane c holds chunk c's key; the plan stays in KC / CD)
  int64_t m_init = 0, m_end = 0; int m_nrows = -1, m_n = -1, m_wire = -1, m_tlen = -1; bool m_ok = false;
  int dd_dst[2] = {0, 0}, dd_inf[2] = {0, 0};
  int64_t rows_scanned = 0, bytes_scanned = 0, pend_rows = 0, pend_bytes = 0;
  uint32_t parity = 0;

  // ---- walk: per-series mode = series gw, gw + nwarps, ...; AGG = items gw, gw + nwarps, ..., positions item_begin[it] .. item_begin[it + 1]
  // walk position = (item, position, item end); plain scalars (a struct handed to the helpers by reference ends up in local memory)
  int64_t c_it = 0, c_p = 0, c_pe = 0, x_it = 0, x_p = 0, x_pe = 0;
#define WP_ITEM_SEEK(it, p, pe, ok) { ok = false; while (it < n_items) { p = item_begin[it]; pe = item_begin[it + 1]; if (p < pe) { ok = true; break; } it += nwarps; } }
  // successor of (it, p, pe) into (it, p, pe); skip_item: the rest of the item is not wanted
#define WP_POS_NEXT(it, p, pe, skip_item, ok) { \
    if (AGG) { if (!(skip_item) && p + 1 < pe) { p += 1; ok = true; } else { it += nwarps; WP_ITEM_SEEK(it, p, pe, ok) } } \
    else { p += nwarps; ok = p < n_series; } }
  auto sid_at = [&](int64_t p) -> int64_t { return (AGG && order) ? (int64_t)order[p] : p; };
  auto issue = [&](int64_t off, uint32_t sz) { mbar_expect_tx(bar, sz); tma_load_1d(R, arena + off, sz, bar); };

  bool more;
  if (AGG) { c_it = gw; WP_ITEM_SEEK(c_it, c_p, c_pe, more) } else { c_p = gw; c_pe = n_series; more = c_p < n_series; }
  int64_t cur_sid = 0, cur_off = 0; uint32_t cur_sz = 0;
  if (more) { cur_sid = sid_at(c_p); cur_off = rec_off[cur_sid]; cur_sz = (uint32_t)(rec_off[cur_sid + 1] - cur_off); }
  if (more && cur_sz <= L.rec_cap && lane == 0) issue(cur_off, cur_sz);
  bool item_bad = false; int item_nser = 0;
  if (AGG) { for (int k = lane; k < q.T; k += 32) { ACC[k] = agg_ident; NBAD[k] = 0; if constexpr (MOM) ACC2.v[k] = 0.0; } __syncwarp(); }

  while (more) {
    // successor in walk order (its record is fetched as soon as R is dead)
    x_it = c_it; x_p = c_p; x_pe = c_pe; bool nmore;
    WP_POS_NEXT(x_it, x_p, x_pe, false, nmore)
    int64_t nxt_sid = 0, nxt_off = 0; uint32_t nxt_sz = 0;
    if (nmore) { nxt_sid = sid_at(x_p); nxt_off = rec_off[nxt_sid]; nxt_sz = (uint32_t)(rec_off[nxt_sid + 1] - nxt_off); }
    const bool staged = cur_sz <= L.rec_cap;
    if (staged) { mbar_wait(bar, parity); parity ^= 1; }
    const int64_t s = cur_sid;
    const bool skip = AGG && item_bad;                     // the item already failed: this record was in flight, drop it
    // ------------------------------------------------------------------------------------------------ setup
    const WpParsed P = wp_parse<false, IRR>(R, q, staged && !skip, lane);
    bool regular = P.regular;
    const bool irr = IRR && P.irr;
    const bool have = P.have; const int n = P.n, c = lane;
    const bool samec = !(c < n) || (P.init == m_init && P.nrows == m_nrows && P.end_time == m_end && P.vwire == m_wire && P.tlen == m_tlen);
    const bool same_all = __all_sync(FULL, samec);
    const bool same = m_ok && n == m_n && same_all && !irr;
    if (regular && !same) {
      m_init = P.init; m_end = P.end_time; m_nrows = P.nrows; m_n = n; m_wire = P.vwire; m_tlen = P.tlen; m_ok = false;
      const int64_t init = P.init, end_time = P.end_time; const int nrows = P.nrows, tlen = P.tlen;
      // three divisions per chunk: s0, e0 = unclamped first / last row of window 0; v4 = last window whose start is <= endTime.
      // (interval logic of the tile kernel's producer, scan_tile.cuh; chunk c = lane c)
      int64_t s0 = 0, e0 = 0, v4 = 0;
      if (have && !irr) { s0 = sd.ceil_div(S0 - init); e0 = sd.floor_div(E0 - init); v4 = sd.floor_div(end_time - S0); }
      const int64_t s0p = __shfl_up_sync(FULL, s0, 1), v4p = __shfl_up_sync(FULL, v4, 1), e0n = __shfl_down_sync(FULL, e0, 1);
      const int tlenp = __shfl_up_sync(FULL, tlen, 1);
      int64_t kA = -e0;
      if (c > 0) { int64_t x = v4p + 1; const int64_t y = (int64_t)tlenp - s0p; if (y > x) x = y; if (x > kA) kA = x; }
      int64_t kB = (int64_t)(nrows - 1) - s0;
      { const int64_t x = (c + 1 < n) ? -(e0n + 1) : (int64_t)q.T; if (x < kB) kB = x; }
      if (v4 < kB) kB = v4;
      if (kA < 0) kA = 0;
      if (kB > q.T - 1) kB = q.T - 1;
      const int64_t kA2 = kA, kB2 = kB;    // every single-chunk window of the chunk
      if (-s0 > kA) kA = -s0;              // [kA, kB]: only windows whose row range is not clamped by the chunk's ends
      { const int64_t x = (int64_t)(nrows - 1) - e0; if (x < kB) kB = x; }
      const int64_t sA = s0 + kA, eA = e0 + kA;
      const bool ok = have && !irr && kA <= kB && eA >= sA;
      const int Wr = ok ? (int)(eA - sA) : 0;
      const bool blocked = ok && Wr >= 1;  // two samples
      // row positions: 8 spare rows behind every chunk
      int rowpos;
      { const int z = have ? nrows + 8 : 0;
        const int a0 = __shfl_sync(FULL, z, 0), a1 = __shfl_sync(FULL, z, 1), a2 = __shfl_sync(FULL, z, 2), a3 = __shfl_sync(FULL, z, 3);
        rowpos = (c > 0 ? a0 : 0) + (c > 1 ? a1 : 0) + (c > 2 ? a2 : 0);
        const int pend = a0 + a1 + a2 + a3;
        if ((uint32_t)(pend + (pend >> 3) + 2) > L.vcap) regular = false; }
      if (regular) {
        if (c < WP_MAXC) {
          WpCtrChunk& d = KC[c];
          d.init = init; d.end_time = end_time; d.nrows = nrows; d.s0 = (int)s0; d.e0 = (int)e0; d.rowpos = rowpos;
          d.kA = blocked ? (int)kA : 0; d.kB = blocked ? (int)kB : -1;
          d.kA2 = (have && !irr && kA2 <= kB2) ? (int)kA2 : 0; d.kB2 = (have && !irr && kA2 <= kB2) ? (int)kB2 : -1;      // irregular: every window takes the literal fold
          if (irr) d.kc.pad = __float_as_int(have ? 1.0f / (float)P.tslope : 0.0f);
          if (blocked) {
            // RateFunctions.extrapolatedRate (RateFunctions.scala:72-111) for the chunk's unclamped single-chunk windows: the sample
            // times move with the window, so durationToStart / End, sampledInterval, numSamples are window-invariant
            const double dTS = (double)(init + s0 * q.step - S0 + (q.inclusive ? 0 : 1)) / 1000.0, dTE = (double)(E0 - (init + e0 * q.step)) / 1000.0;
            const double sI = (double)((e0 - s0) * q.step) / 1000.0;
            const double avg = sI / ((double)(Wr + 1) - 1.0), thr = avg * 1.1, half = avg / 2.0;
            const double endpart = dTE < thr ? dTE : half;
            const double eTI = (sI + (dTS < thr ? dTS : half)) + endpart;
            d.kc.dTS = dTS; d.kc.thr = thr; d.kc.half = half; d.kc.endpart = endpart; d.kc.sI = sI; d.kc.ratio0 = eTI / sI;
            d.kc.skipC = 2.0 * dTS / sI;      // v1 > delta * skipC  =>  durationToZero >= durationToStart (no zero-point clamp)
          }
          CD[c].rowpos = rowpos; CD[c].nrows = nrows;
        }
        __syncwarp();
        {
          const int gb1 = __shfl_sync(FULL, have ? P.grp_base : 0x7fffffff, 1), gb2 = __shfl_sync(FULL, have ? P.grp_base : 0x7fffffff, 2),
                    gb3 = __shfl_sync(FULL, have ? P.grp_base : 0x7fffffff, 3);
#pragma unroll
          for (int jj = 0; jj < 2; ++jj) {
            const int slot = jj * 32 + lane;
            const bool active = slot < P.ngroups;
            const int ci = active ? (slot >= gb1 ? 1 : 0) + (slot >= gb2 ? 1 : 0) + (slot >= gb3 ? 1 : 0) : 0;
            const int gbc = ci == 0 ? 0 : ci == 1 ? gb1 : ci == 2 ? gb2 : gb3;
            const int g = active ? slot - gbc : 0;
            const int pq = CD[ci].rowpos + 1 + g * 8;
            dd_dst[jj] = wp_vidx(pq);
            dd_inf[jj] = (active ? 1 : 0) | (ci << 1) | ((pq & 7) << 3) | (g << 8);
          }
        }
        m_ok = !irr;
      }
    }
    bool declined = !regular && !skip;
    if (regular) {
      // per-series parts of the descriptors
      if (c < WP_MAXC) {
        WpChunk& d = CD[c];
        d.grp_base = have ? P.grp_base : 0x7fffffff; d.ng = P.ng; d.wire = P.vwire; d.val_off = P.voff; d.dropped = have ? P.dropped : 0;
        if (have && P.vwire == WIRE_XOR) { const uint32_t po = P.w12 >> 16; d.first = ld64(R + P.voff + po); d.grp_off = P.voff + po + 8; d.tab_off = P.voff + XOR_OFF_GROUPTAB; }
        else { d.first = have ? ld64(R + P.voff + 8) : 0ull; d.grp_off = 0; d.tab_off = 0; }
        KC[c].kc.dropped = have ? P.dropped : 0;
        DR[c].n = 0;
      }
      __syncwarp();
      (void)wp_decode<FN != FN_DELTA>(R, V, CD, xtab, dd_dst, dd_inf, n, P.any_raw, lane, DR);
      if (IRR && irr) {                                    // row times: init + slope * r + residual (DeltaDeltaVector.scala:153-156), const chunks without residuals
        for (int ci = 0; ci < n; ++ci) {
          const uint32_t toff = __shfl_sync(FULL, P.toff, ci); const int tsl = __shfl_sync(FULL, P.tslope, ci);
          const uint8_t* tv = R + toff;
          const int nr = KC[ci].nrows; int32_t* dst = TSR + KC[ci].rowpos;
          if ((int)(ld32(tv + 4) & 0xffff) == WIRE_DDV) {
            const uint8_t* in = tv + 20; const uint32_t iw = ld32(in + 4);
            const int nbits = (iw >> 16) & 0x7f; const bool sgn = (iw >> 23) & 1;
            for (int r = lane; r < nr; r += 32) dst[r] = tsl * r + int_apply(in, nbits, sgn, r);
          } else for (int r = lane; r < nr; r += 32) dst[r] = tsl * r;
        }
      }
      __syncwarp();
      // more drops in one chunk than the list holds: the generic kernel takes the series
      bool overflow = false;
      if (FN != FN_DELTA) for (int ci = 0; ci < n; ++ci) overflow |= KC[ci].kc.dropped && DR[ci].n > TILE_MAXDROP;
      if (overflow) { regular = false; declined = true; }
    }
    // R is dead: fetch the successor's record behind the window phase
    if (AGG && (declined || item_bad) && !skip) {          // the item fails here: its remaining series are not wanted
      x_it = c_it; x_p = c_p; x_pe = c_pe;
      WP_POS_NEXT(x_it, x_p, x_pe, true, nmore)
      if (nmore) { nxt_sid = sid_at(x_p); nxt_off = rec_off[nxt_sid]; nxt_sz = (uint32_t)(rec_off[nxt_sid + 1] - nxt_off); }
    }
    __syncwarp();
    if (nmore && nxt_sz <= L.rec_cap && lane == 0) issue(nxt_off, nxt_sz);

    if (declined) {
      if (!AGG) { if (lane == 0) { const unsigned long long slot = atomicAdd(fallback_count, 1ull); fallback_list[slot] = s; } }
      else item_bad = true;
    }
    if (regular && !skip) {
      // scan counters (CountingChunkInfoIterator, ChunkSetInfo.scala:336-380): every chunk in range is pulled, except one that starts
      // after the last window end
      int cnt_rows = 0, cnt_bytes = 0;
      { const int64_t endp = __shfl_up_sync(FULL, P.end_time, 1);
        if (have && !(c > 0 && !(endp < lastEnd))) { cnt_rows = P.num_rows; cnt_bytes = P.vbytes; } }
#pragma unroll
      for (int o = 1; o < WP_MAXC; o <<= 1) { cnt_rows += __shfl_xor_sync(FULL, cnt_rows, o); cnt_bytes += __shfl_xor_sync(FULL, cnt_bytes, o); }
      if (lane == 0) { pend_rows += cnt_rows; pend_bytes += cnt_bytes; }
      // lane c: sort chunk c's drops by row and turn the amounts into running sums (reference order of additions)
      if (FN != FN_DELTA && lane < n && KC[lane].kc.dropped) {
        TileDrops& D = DR[lane];
        const int nd = D.n;
        for (int i = 1; i < nd; ++i) {
          const int pz = D.pos[i]; const double a = D.amt[i]; int j = i - 1;
          while (j >= 0 && D.pos[j] > pz) { D.pos[j + 1] = D.pos[j]; D.amt[j + 1] = D.amt[j]; --j; }
          D.pos[j + 1] = pz; D.amt[j + 1] = a;
        }
        double run = 0.0;
        for (int i = 0; i < nd; ++i) { run += D.amt[i]; D.amt[i] = run; }
      }
      __syncwarp();
      // ---------------------------------------------------------------------------------------------- windows
      double* gout = AGG ? nullptr : out + (size_t)s * q.T;
      const bool agg_add = agg_op == AGG_SUM || agg_op == AGG_AVG;
      auto emit = [&](int k, double v) {
        if (!AGG) { wp_store_result(gout + k, v); return; }
        if (v == v) {                                        // RowAggregators skip NaN (SumRowAggregator.scala:22-29 ...)
          if (agg_add) ACC[k] += v;
          // acc = min/maxIgnoreNaN(acc, v) (QueryUtils.scala:111-123): v replaces acc unless acc is strictly better, so of two equal
          // values (+0.0 / -0.0) the later one is kept
          else if (agg_op != AGG_COUNT) { const double a = ACC[k]; if (agg_op == AGG_MIN ? !(a < v) : !(a > v)) ACC[k] = v; }
          if constexpr (MOM) ACC2.v[k] += v * v;
        } else wp_bump_u16(NBAD + k);
      };
      for (int ci = 0; ci < n; ++ci) {
        const WpCtrChunk& ch = KC[ci];
        if (ch.kA2 > ch.kB2) continue;
        const bool hasfast = ch.kA <= ch.kB;
        const TileCtr kc = ch.kc;
        const TileDrops& D = DR[ci];
        const bool drp = FN != FN_DELTA && kc.dropped;
        // drops of this chunk (warp-uniform): none / one (position and amount in registers) / several (list walk)
        const int dn = drp ? D.n : 0;
        const int dpos0 = dn >= 1 ? D.pos[0] : 0x7fffffff;
        const double damt0 = dn >= 1 ? D.amt[0] : 0.0;
        // V index of row r0 + 32 m = index of row r0 + 36 m (one pad slot per 8 rows)
        const double* p1 = V + wp_vidx(ch.rowpos + ch.s0 + ch.kA + lane);
        const double* p2 = V + wp_vidx(ch.rowpos + ch.e0 + ch.kA + lane);
        // one window from its two samples (extrapolatedRate with the chunk's window-invariant terms)
        auto fast_one = [&](int kk, double v1, double v2) -> double {
          if (drp) {
            const int r1 = ch.s0 + kk, r2 = ch.e0 + kk;
            if (dn <= 1) { v1 = nan0(v1) + (r1 >= dpos0 ? damt0 : 0.0); v2 = nan0(v2) + (r2 >= dpos0 ? damt0 : 0.0); }
            else { v1 = nan0(v1) + drops_cum(D, r1); v2 = nan0(v2) + drops_cum(D, r2); }     // sorted running sums
          }
          const double delta = v2 - v1;
          double ratio = kc.ratio0;
          if (FN != FN_DELTA && delta > 0 && v1 >= 0 && !(v1 > delta * kc.skipC)) {      // zero-point clamp may apply (:84-90)
            const double dz = kc.sI * ddiv_rare(v1, delta);
            const double dts = dz < kc.dTS ? dz : kc.dTS;
            const double eTI = (kc.sI + (dts < kc.thr ? dts : kc.half)) + kc.endpart;
            ratio = ddiv_rare(eTI, kc.sI);
          }
          const double scaled = delta * ratio;
          return FN == FN_RATE ? __dmul_rn(div_invariant(scaled, fdiv, frcp), 1000.0) : scaled;
        };
#ifdef FILO_WP_CTR_PAIR
        // two windows per lane and iteration (kk and kk + 32): the kernel is latency bound, two independent
        // dependency chains per warp overlap
        for (int kk = ch.kA + lane; hasfast && kk <= ch.kB; kk += 64, p1 += 72, p2 += 72) {
          const bool two = kk + 32 <= ch.kB;
          const double a1 = *p1, a2 = *p2;
          const double b1 = two ? p1[36] : 0.0, b2 = two ? p2[36] : 0.0;
          const double ra = fast_one(kk, a1, a2);
          const double rb = two ? fast_one(kk + 32, b1, b2) : 0.0;
          emit(kk, ra);
          if (two) emit(kk + 32, rb);
        }
#else
        for (int kk = ch.kA + lane; hasfast && kk <= ch.kB; kk += 32, p1 += 36, p2 += 36) emit(kk, fast_one(kk, *p1, *p2));
#endif
        // the chunk's clamped single-chunk windows (window start before its first row or end after its last): the sample distance
        // varies with the window, the table supplies the terms that depend on it
        const int nlo = hasfast ? ch.kA - ch.kA2 : ch.kB2 - ch.kA2 + 1, nhi = hasfast ? ch.kB2 - ch.kB : 0;
        for (int u = lane; u < nlo + nhi; u += 32) {
          const int kk = u < nlo ? ch.kA2 + u : ch.kB + 1 + (u - nlo);
          const int64_t wEnd = q.start + (int64_t)kk * q.step, cws = wEnd - winDur - (q.inclusive ? 0 : 1);
          emit(kk, wp_clamped_window<FN>(V, ch, D, drp, kk, wEnd, cws, q.step, fdiv, frcp, CTAB));
        }
      }
      // windows outside every chunk's single-chunk interval (chunk junctions, no data): literal fold, lanes over the gaps
      {
        int prev = -1;
        for (int ci = 0; ci <= n; ++ci) {
          int gend = q.T;
          if (ci < n) { if (KC[ci].kA2 > KC[ci].kB2) continue; gend = KC[ci].kA2; }
          for (int k = prev + 1 + lane; k < gend; k += 32) {
            const int64_t wEnd = q.start + (int64_t)k * q.step, wStart = wEnd - winDur;
            if (IRR && irr) emit(k, wp_eval_counter_irr<FN>(n, KC, CD, DR, V, TSR, q.step, q.inclusive, wStart, wEnd, fdiv, frcp, CTAB));
            else emit(k, wp_eval_counter<FN>(n, KC, CD, DR, V, q.step, q.inclusive, wStart, wEnd, k, fdiv, frcp, CTAB));
          }
          if (ci < n) prev = KC[ci].kB2;
        }
      }
      if (!AGG && lane == 0) { rows_scanned += pend_rows; bytes_scanned += pend_bytes; pend_rows = 0; pend_bytes = 0; }
      if (AGG) item_nser += 1;
    }
    // ---------------------------------------------------------------------------------------------- item end (AGG)
    if (AGG) {
      const bool last_of_item = !nmore || x_it != c_it;
      if (last_of_item) {
        __syncwarp();
        if (!item_bad) {
          double* pv = pval + (size_t)c_it * q.T; uint32_t* pc = pcnt + (size_t)c_it * q.T;
          for (int k = lane; k < q.T; k += 32) { pv[k] = ACC[k]; pc[k] = (uint32_t)(item_nser - (int)NBAD[k]); }
          if constexpr (MOM) { double* pv2 = pval + (size_t)(n_items + c_it) * q.T; for (int k = lane; k < q.T; k += 32) pv2[k] = ACC2.v[k]; }
          if (lane == 0) { rows_scanned += pend_rows; bytes_scanned += pend_bytes; }
        } else if (lane == 0) {
          const unsigned long long slot = atomicAdd(fallback_count, 1ull); fallback_list[slot] = c_it;
        }
        for (int k = lane; k < q.T; k += 32) { ACC[k] = agg_ident; NBAD[k] = 0; if constexpr (MOM) ACC2.v[k] = 0.0; }
        pend_rows = 0; pend_bytes = 0; item_bad = false; item_nser = 0;
      }
    }
    __syncwarp();
    c_it = x_it; c_p = x_p; c_pe = x_pe; more = nmore; cur_sid = nxt_sid; cur_off = nxt_off; cur_sz = nxt_sz;
  }
  if (lane == 0 && (rows_scanned | bytes_scanned)) {
    atomicAdd(&d_counters[0], (unsigned long long)rows_scanned); atomicAdd(&d_counters[1], (unsigned long long)bytes_scanned);
  }
}

#undef WP_ITEM_SEEK
#undef WP_POS_NEXT

} // namespace filo
