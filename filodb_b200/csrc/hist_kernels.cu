// Histogram column scan (first version): hist rate / increase over SectDelta histogram vectors with counter correction,
// fused HistSum across series and histogram_quantile.
//
// Reference path: SectDeltaHistogramReader (vectors/HistogramVector.scala:628-738), SectionReader (Section.scala:146-227),
// NibblePack.DeltaSink (NibblePack.scala:208-230), HistogramRateFunctionBase (rangefn/RateFunctions.scala:330-418),
// CounterChunkedRangeFunction (rangefn/RangeFunction.scala:131-172), HistSumRowAggregator (aggregator/HistSumRowAggregator.scala),
// Histogram.quantile (vectors/Histogram.scala:65-108).
//
// One CTA walks work items (runs of series of one group).  Per series: every histogram row of the chunks in range is decoded
// once into shared memory as cumulative bucket counts with the chunk's own drop corrections applied (int64, exact); the
// corrections carried from chunk to chunk inside a window are prefix sums over the chunks (integer addition is associative,
// so correctedValue(n, meta) = row + carried(firstChunkOfWindow, chunk)); a per-window descriptor pass finds the lowest and
// highest sample; then one thread per (window, bucket) evaluates extrapolatedRate.
#include "kernels.h"
#include "scan_device.cuh"
#include "scan_fast.cuh"
#include "hist_phases.h"

namespace filo {

constexpr int HIST_THREADS = 1024;
constexpr int HIST_MAXC = 8;          // chunks in range per series
constexpr int HIST_MAXSECT = 96;      // sections per series

struct HistWin { int32_t lo_row, hi_row, a, lo_c, hi_c, num_samples; int64_t lo_t, hi_t;
                 double dTS, thr, half, endpart, sI, ratio0, skipC; };     // window-invariant terms of extrapolatedRate (all buckets share the sample times)
struct HistSect { int32_t chunk, start_row /*global row of the section's first histogram*/, n, type; uint32_t first_rec /*byte offset in record*/; };
struct HistChunkD { int32_t row_base, nrows, nsect, has_drop; int64_t end_time; int32_t sect, pad; };

// NibblePack.unpack8 (NibblePack.scala:395-447) over bytes in global memory; returns bytes consumed
__device__ __forceinline__ uint64_t rd_long(const uint8_t* p, int cap, int index) {
  uint64_t out = 0;
  for (int i = 0; i < 8 && index + i < cap; ++i) out |= (uint64_t)p[index + i] << (8 * i);
  return out;
}
__device__ int unpack8_dev(const uint8_t* buf, int cap, uint64_t out[8], bool& short_in) {
  const uint32_t nonzeroMask = buf[0];
  if (nonzeroMask == 0) { for (int i = 0; i < 8; ++i) out[i] = 0; return 1; }
  const int numNibblesU8 = buf[1];
  const int numBits = ((numNibblesU8 >> 4) + 1) * 4, trailingZeroes = (numNibblesU8 & 0x0f) * 4;
  const int total = 2 + (numBits * __popc(nonzeroMask) + 7) / 8;
  const uint64_t mask = numBits >= 64 ? ~0ull : ((1ull << numBits) - 1);
  int bufIndex = 2, bitCursor = 0;
  uint64_t inWord = rd_long(buf, cap, bufIndex); bufIndex += 8;
  for (int bit = 0; bit < 8; ++bit) {
    if (nonzeroMask & (1u << bit)) {
      const int remaining = 64 - bitCursor;
      uint64_t outWord = (inWord >> bitCursor) & mask;
      if (remaining <= numBits && bufIndex < total) {
        if (bufIndex < cap) { inWord = rd_long(buf, cap, bufIndex); bufIndex += 8; if (remaining < numBits) outWord |= (inWord << remaining) & mask; }
        else { short_in = true; return total; }
      }
      out[bit] = outWord << trailingZeroes;
      bitCursor = (bitCursor + numBits) % 64;
    } else out[bit] = 0;
  }
  return total;
}
// one histogram record (u16 length + NibblePack delta bytes) -> cumulative values (DeltaSink), added onto `base` when given
__device__ void decode_record(const uint8_t* rec, int nb, const int64_t* base, int64_t* out, bool& bad) {
  int cap = (int)(rec[0] | (rec[1] << 8));
  const uint8_t* p = rec + 2;
  int64_t current = 0; int i = 0;
  while (i < nb && cap > 0) {
    uint64_t data[8];
    const int used = unpack8_dev(p, cap, data, bad);
    const int m = nb - i < 8 ? nb - i : 8;
    for (int n = 0; n < m; ++n) { current += (int64_t)data[n]; out[i + n] = current + (base ? base[i + n] : 0); }
    i += 8;
    if (cap > used) { p += used; cap -= used; } else cap = 0;
  }
  for (; i < nb; ++i) out[i] = base ? base[i] : 0;          // input ran out: remaining deltas are zero (unpackToSink stops)
}

__device__ __forceinline__ int64_t ts_of(const uint8_t* tv, int twire, int r) {
  if (twire == WIRE_DDV_CONST) return (int64_t)ld64_a4(tv + 12) + (int64_t)(int32_t)((int32_t)ld32(tv + 20) * r);
  if (twire == WIRE_RAW64) return (int64_t)ld64(tv + 8 + 8 * (size_t)r);
  const uint8_t* in = tv + 20; const uint32_t iw = ld32(in + 4);
  return (int64_t)ld64(tv + 8) + (int64_t)(int32_t)ld32(tv + 16) * r + (int64_t)int_apply(in, (iw >> 16) & 0x7f, (iw >> 23) & 1, r);
}

// Per-phase cycle counters of hist_scan_kernel for profiling builds (-DFILO_HIST_PROF; scratch/hist_prof.py).
// Compiled out of the product build.
#ifdef FILO_HIST_PROF
__device__ unsigned long long g_hist_prof[16];
#define HPROF_DECL long long hp_t0 = clock64(), hp_acc[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
#define HPROF(i) { const long long hp_t1 = clock64(); hp_acc[i] += hp_t1 - hp_t0; hp_t0 = hp_t1; }
#define HPROF_FLUSH if (threadIdx.x == 0) { for (int hp_i = 0; hp_i < 12; ++hp_i) atomicAdd(&g_hist_prof[hp_i], (unsigned long long)hp_acc[hp_i]); atomicAdd(&g_hist_prof[15], 1ull); }
#else
#define HPROF_DECL
#define HPROF(i)
#define HPROF_FLUSH
#endif

struct HistLayout { uint32_t cv, ts, pt, pd, tot, lastraw, win, acc, any, sect, rec, total; };
__host__ __device__ inline HistLayout hist_layout(int max_rows, int nb, int T, bool agg, uint32_t max_rec) {
  HistLayout L; uint32_t o = 0;
  L.cv = o; o += (uint32_t)max_rows * nb * 8;
  L.ts = o; o += (uint32_t)max_rows * 8;
  L.pt = o; o += (HIST_MAXC + 1) * nb * 8;
  L.pd = o; o += (HIST_MAXC + 1) * nb * 8;
  L.tot = o; o += HIST_MAXC * nb * 8;
  L.lastraw = o; o += HIST_MAXC * nb * 8;
  L.win = o; o += (uint32_t)T * (uint32_t)sizeof(HistWin);
  L.acc = o; if (agg) o += (uint32_t)T * nb * 8;
  L.any = o; if (agg) o += ((uint32_t)T + 7) & ~7u;
  L.sect = o; o += HIST_MAXSECT * (uint32_t)sizeof(HistSect);
  o = (o + 15) & ~15u;
  L.rec = o; o += (max_rec + 15) & ~15u;               // the series' record, staged so that parsing and decoding read shared memory
  L.total = (o + 127) & ~127u;
  return L;
}

// err codes written to d_err[0]: 1 corrupt vector, 5 unsupported shape (too many chunks / sections / rows)
__global__ void __launch_bounds__(HIST_THREADS)
hist_scan_kernel(const uint8_t* __restrict__ arena, const int64_t* __restrict__ rec_off, int64_t n_series, QueryParams q, int nb, int max_rows, uint32_t max_rec,
                 const int32_t* __restrict__ order, const int64_t* __restrict__ item_begin, int64_t n_items, int agg,
                 double* __restrict__ out /* !agg: [S][T][nb] */, double* __restrict__ pval /* agg: [items][T][nb] */, uint8_t* __restrict__ pany,
                 unsigned long long* d_counters, int* d_err,
                 const double* __restrict__ tops = nullptr, double qtl = 0.0, int exp_buckets = 0, double* __restrict__ out_q = nullptr /* !agg: [S][T] */) {
  extern __shared__ __align__(16) uint8_t smem[];
  // per-series histogram_quantile (!agg, out_q given): each series' window rows are staged in acc[T][nb] (the fused mode's layout) and
  // presented by a thread per window; out, when given, receives the staged rows
  const bool pq = !agg && out_q != nullptr;
  const HistLayout L = hist_layout(max_rows, nb, q.T, agg != 0 || pq, max_rec);
  int64_t* cv = reinterpret_cast<int64_t*>(smem + L.cv);
  int64_t* tss = reinterpret_cast<int64_t*>(smem + L.ts);
  int64_t* PT = reinterpret_cast<int64_t*>(smem + L.pt);
  int64_t* PD = reinterpret_cast<int64_t*>(smem + L.pd);
  HistWin* W = reinterpret_cast<HistWin*>(smem + L.win);
  double* acc = reinterpret_cast<double*>(smem + L.acc);
  uint8_t* any = smem + L.any;
  HistSect* SE = reinterpret_cast<HistSect*>(smem + L.sect);
  __shared__ HistChunkD CH[HIST_MAXC];
  __shared__ int s_n, s_nsect, s_rows, s_err, s_cLo;
  __shared__ int LESS[HIST_MAXC];
  int64_t* TOT = reinterpret_cast<int64_t*>(smem + L.tot);
  int64_t* LASTRAW = reinterpret_cast<int64_t*>(smem + L.lastraw);
  const int tid = threadIdx.x;
  const double NaNv = __longlong_as_double(0x7ff8000000000000LL);
  int64_t winDur = q.inclusive ? q.window : q.window - 1; if (winDur < 0) winDur = 0;
  const int64_t n_work = agg ? n_items : n_series;
  int64_t rows_scanned = 0, bytes_scanned = 0;
  // sum mode: sum_over_time, and rate / increase on a delta-temporality schema (SumOverTimeChunkedFunctionH,
  // AggrOverTimeFunctions.scala:587-606; RateOverDeltaChunkedFunctionH, RateFunctions.scala:470-494)
  const bool last = q.fn == FN_LAST;
  const bool sum_mode = !last && (q.fn == FN_SUM || !q.cumulative);
  const double fdiv = (double)(q.inclusive ? winDur : winDur + 1), frcp = 1.0 / fdiv;       // windowEnd - curWindowStart

  HPROF_DECL
  for (int64_t it = blockIdx.x; it < n_work; it += gridDim.x) {
    const int64_t pb = agg ? item_begin[it] : it, pe = agg ? item_begin[it + 1] : it + 1;
    if (agg) { for (int i = tid; i < q.T * nb; i += HIST_THREADS) acc[i] = 0.0; for (int i = tid; i < q.T; i += HIST_THREADS) any[i] = 0; }
    __syncthreads();
    for (int64_t pos = pb; pos < pe; ++pos) {
      const int64_t sid = (agg && order) ? (int64_t)order[pos] : pos;
      const uint8_t* grec = arena + rec_off[sid];
      {                                                    // stage the record (16-byte aligned, rec_bytes multiple of 16)
        const uint32_t rb = reinterpret_cast<const RecordHeader*>(grec)->rec_bytes;
        const uint4* src = reinterpret_cast<const uint4*>(grec); uint4* dst = reinterpret_cast<uint4*>(smem + L.rec);
        for (uint32_t i = tid; i < (rb >> 4); i += HIST_THREADS) dst[i] = src[i];
      }
      __syncthreads();
      HPROF(0)                                             // record staged
      const uint8_t* rec = smem + L.rec;
      const RecordHeader* h = reinterpret_cast<const RecordHeader*>(rec);
      const ChunkEntry* E = reinterpret_cast<const ChunkEntry*>(rec + sizeof(RecordHeader));
      // ---- chunk range + section tables (thread 0; a few dozen sections per series)
      if (tid == 0) {
        const int nch = (int)h->n_chunks;
        const int64_t t1 = q.start - q.window, t2 = q.end;
        int cLo = 0; while (cLo < nch && E[cLo].end_time < t1) ++cLo;
        int cHi = cLo; while (cHi < nch && E[cHi].start_time <= t2) ++cHi;
        if (t1 > t2) cHi = cLo;
        int err = 0, rows = 0, nsect = 0;
        const int n = cHi - cLo;
        if (n > HIST_MAXC) err = 5;
        const int64_t lastEnd = q.start + (int64_t)(q.T - 1) * q.step;
        for (int c = 0; c < n && !err; ++c) {
          const ChunkEntry& e = E[cLo + c];
          const uint8_t* hv = rec + e.val_off;
          const int wire = ld32(hv + 4) & 0xffff;
          const int numHist = (int)(ld32(hv + 4) >> 16) & 0xffff;             // u16 at +6
          const int defBytes = (int)(hv[9] | (hv[10] << 8));
          const int vnb = (int)(hv[11] | (hv[12] << 8));
          // counter functions need the SectDelta reader (a RowHistogramReader is not a CounterVectorReader, RangeFunction.scala:142)
          if (!(wire == WIRE_H_SECTDELTA || (wire == WIRE_H_SIMPLE && (sum_mode || last))) || vnb != nb || numHist < e.num_rows) { err = 1; break; }
          HistChunkD d; d.sect = wire == WIRE_H_SECTDELTA; d.pad = 0; d.row_base = rows; d.nrows = e.num_rows; d.nsect = 0; d.has_drop = 0; d.end_time = e.end_time;
          const uint8_t* endp = hv + (int32_t)ld32(hv) + 4;
          const uint8_t* s = hv + 11 + defBytes; int start = 0;
          while (s + 4 <= endp && start < numHist) {
            const int sbytes = (int)(s[0] | (s[1] << 8)), sn = s[2], stype = s[3];
            if (s + 4 + sbytes > endp || sn == 0 || start >= e.num_rows) break;
            if (nsect >= HIST_MAXSECT) { err = 5; break; }
            SE[nsect] = HistSect{c, rows + start, sn < e.num_rows - start ? sn : e.num_rows - start, stype, (uint32_t)((s + 4) - rec)};   // rows past numRows are not read
            if (stype == 1 && start > 0) d.has_drop = 1;
            ++nsect; ++d.nsect; start += sn; s += 4 + sbytes;
          }
          if (start < e.num_rows) err = 1;
          CH[c] = d; rows += e.num_rows;
          // CountingChunkInfoIterator: a chunk the window iterator never pulls is not counted (ChunkSetInfo.scala:336-380)
          if (!(c > 0 && !(E[cLo + c - 1].end_time < lastEnd))) { rows_scanned += e.num_rows; bytes_scanned += (int64_t)ld32(rec + e.ts_off) + 4 + (int64_t)ld32(hv) + 4; }
        }
        if (rows > max_rows) err = 5;
        s_n = err ? 0 : n; s_nsect = err ? 0 : nsect; s_rows = err ? 0 : rows; s_err = err; s_cLo = cLo;
        if (err) { if (atomicCAS(&d_err[0], 0, err) == 0) { d_err[1] = (int)(sid & 0x7fffffff); d_err[2] = (int)(sid >> 31); } }
      }
      __syncthreads();
      HPROF(1)                                             // chunk range + section tables (thread 0)
      const int n = s_n, nsect = s_nsect, rows = s_rows, cLo = s_cLo;
      bool bad = false;
      // ---- timestamps of every row + section base histograms
      for (int r = tid; r < rows; r += HIST_THREADS) {
        int c = 0; while (c + 1 < n && r >= CH[c + 1].row_base) ++c;
        const ChunkEntry& e = E[cLo + c];
        const uint8_t* tv = rec + e.ts_off;
        tss[r] = ts_of(tv, ld32(tv + 4) & 0xffff, r - CH[c].row_base);
      }
      for (int si = tid; si < nsect; si += HIST_THREADS) decode_record(rec + SE[si].first_rec, nb, nullptr, cv + (size_t)SE[si].start_row * nb, bad);
      __syncthreads();
      HPROF(2)                                             // timestamps + section bases
      // ---- remaining rows: delta from the section's first histogram (SectDeltaHistogramReader.apply, :646-666)
      for (int r = tid; r < rows; r += HIST_THREADS) {
        int si = 0; while (si + 1 < nsect && r >= SE[si + 1].start_row) ++si;
        const HistSect S = SE[si];
        if (r == S.start_row || r >= S.start_row + S.n) continue;
        const uint8_t* p = rec + S.first_rec;
        for (int k = r - S.start_row; k > 0; --k) p += (int)(p[0] | (p[1] << 8)) + 2;      // SectionReader.skipAhead
        decode_record(p, nb, CH[S.chunk].sect ? cv + (size_t)S.start_row * nb : nullptr, cv + (size_t)r * nb, bad);
      }
      if (bad) { if (atomicCAS(&d_err[0], 0, 1) == 0) { d_err[1] = (int)(sid & 0x7fffffff); d_err[2] = (int)(sid >> 31); } }
      __syncthreads();
      HPROF(3)                                             // remaining rows decoded
      // per-series histogram_quantile of the staged rows (Histogram.quantile, hist_quantile in hist_phases.h; empty windows: NaN)
      auto present = [&]() {
        for (int k = tid; k < q.T; k += HIST_THREADS)
          out_q[(size_t)sid * q.T + k] = (any[k] && qtl == qtl) ? hist_quantile(acc + (size_t)k * nb, nb, tops, qtl, exp_buckets != 0) : NaNv;
        if (out) for (int i = tid; i < q.T * nb; i += HIST_THREADS) out[(size_t)sid * q.T * nb + i] = acc[i];
        __syncthreads();
      };
      if (last) {
        // LastSampleChunkedFunctionH (RangeFunction.scala:599-641): over the window's chunk set, the row endRowNum = min(ceilingIndex(end),
        // numRows - 1) of a chunk is kept when its timestamp is >= windowStart and > the one kept so far; the value is the raw reader value
        // (SectDelta base + delta, or the row of a simple vector), without counter correction
        for (int k = tid; k < q.T; k += HIST_THREADS) {
          const int64_t wEnd = q.start + (int64_t)k * q.step;
          const int row = hist_last_row(CH, n, tss, wEnd - winDur, wEnd);                // hist_phases.h, shared with the second kernel
          const int64_t* rv = row >= 0 ? cv + (size_t)row * nb : nullptr;
          if (!agg) {
            double* o = pq ? acc + (size_t)k * nb : out + ((size_t)sid * q.T + k) * nb;
            for (int b = 0; b < nb; ++b) o[b] = rv ? (double)rv[b] : NaNv;
            if (pq) any[k] = rv != nullptr;
          } else if (rv) {                                                    // HistSumRowAggregator: copy the first, MutableHistogram.add the others
            const bool firstm = any[k] == 0; double mx = 0.0;
            for (int b = 0; b < nb; ++b) {
              double nv = acc[(size_t)k * nb + b] + (double)rv[b];
              if (!firstm) { if (nv < mx || nv != nv) nv = mx; else if (nv > mx) mx = nv; }
              acc[(size_t)k * nb + b] = nv;
            }
            any[k] = firstm ? 1 : 2;
          }
        }
        __syncthreads();
        if (pq) present();
        continue;
      }
      if (sum_mode) {
        // per-bucket running sums over the rows of each chunk (int64, exact): the reference adds the rows as doubles
        // (RowHistogramReader.sum, HistogramVector.scala:613-621), which is the same number while the sums stay below 2^53
        for (int cb = tid; cb < n * nb; cb += HIST_THREADS) {
          const int c = cb / nb, b = cb - c * nb;
          const HistChunkD d = CH[c];
          int64_t run = 0;
          for (int r = d.row_base; r < d.row_base + d.nrows; ++r) { run += cv[(size_t)r * nb + b]; cv[(size_t)r * nb + b] = run; }
          if (run >= (1ll << 53) || run < 0) { if (atomicCAS(&d_err[0], 0, 5) == 0) { d_err[1] = (int)(sid & 0x7fffffff); d_err[2] = (int)(sid >> 31); } }
        }
        __syncthreads();
        // thread per window: chunks folded in order, h = sum.copy for the first, h.add(sum) (+ makeMonotonic) afterwards
        for (int k = tid; k < q.T; k += HIST_THREADS) {
          const int64_t wEnd = q.start + (int64_t)k * q.step, wStart = wEnd - winDur;
          double hv[64]; bool has = false;
          for (int c = 0; c < n; ++c) {
            const HistChunkD d = CH[c];
            if (d.end_time < wStart) continue;
            if (c > 0 && !(CH[c - 1].end_time < wEnd)) continue;
            const int64_t* t = tss + d.row_base;
            int lo = 0, hi = d.nrows;
            while (lo < hi) { const int m = (lo + hi) >> 1; if (t[m] < wStart) lo = m + 1; else hi = m; }
            const int s0 = lo;
            lo = 0; hi = d.nrows;
            while (lo < hi) { const int m = (lo + hi) >> 1; if (t[m] <= wEnd) lo = m + 1; else hi = m; }
            const int e0 = lo - 1;
            if (s0 > e0) continue;
            const int64_t* ce = cv + (size_t)(d.row_base + e0) * nb; const int64_t* cs = s0 > 0 ? cv + (size_t)(d.row_base + s0 - 1) * nb : nullptr;
            if (!has) { for (int b = 0; b < nb; ++b) hv[b] = (double)(ce[b] - (cs ? cs[b] : 0)); has = true; }
            else {
              for (int b = 0; b < nb; ++b) hv[b] += (double)(ce[b] - (cs ? cs[b] : 0));
              double mx = 0.0;                                                  // makeMonotonic, Histogram.scala:440-449
              for (int b = 0; b < nb; ++b) { if (hv[b] < mx || hv[b] != hv[b]) hv[b] = mx; else if (hv[b] > mx) mx = hv[b]; }
            }
          }
          if (has && q.fn == FN_RATE) for (int b = 0; b < nb; ++b) hv[b] = hv[b] / (double)(wEnd - wStart) * 1000.0;   // RateFunctions.scala:481 (raw windowStart)
          if (!agg) {
            double* o = pq ? acc + (size_t)k * nb : out + ((size_t)sid * q.T + k) * nb;
            for (int b = 0; b < nb; ++b) o[b] = has ? hv[b] : NaNv;
            if (pq) any[k] = has;
          }
          else if (has) {                                                     // HistSumRowAggregator: copy the first, MutableHistogram.add the others
            const bool firstm = any[k] == 0; double mx = 0.0;
            for (int b = 0; b < nb; ++b) {
              double nv = acc[(size_t)k * nb + b] + hv[b];
              if (!firstm) { if (nv < mx || nv != nv) nv = mx; else if (nv > mx) mx = nv; }
              acc[(size_t)k * nb + b] = nv;
            }
            any[k] = firstm ? 1 : 2;
          }
        }
        __syncthreads();
        if (pq) present();
        continue;
      }
      // ---- corrections.  Inside a chunk (lazy val corrections, :690-707; correctedValue :730-746): every Drop section starting
      //      at row ci > 0 adds the RAW histogram of row ci-1 to all rows >= ci.  Thread per (chunk, bucket), sequential over rows.
      for (int cb = tid; cb < n * nb; cb += HIST_THREADS) {
        const int c = cb / nb, b = cb - c * nb;
        const HistChunkD d = CH[c];
        int64_t run = 0, prev_raw = 0;
        if (d.has_drop) {
          int si = 0; while (si < nsect && SE[si].chunk != c) ++si;
          for (; si < nsect && SE[si].chunk == c; ++si) {
            const HistSect S = SE[si];
            if (S.type == 1 && S.start_row > d.row_base) run += prev_raw;
            for (int r = S.start_row; r < S.start_row + S.n && r < d.row_base + d.nrows; ++r) { const int64_t x = cv[(size_t)r * nb + b]; prev_raw = x; cv[(size_t)r * nb + b] = x + run; }
          }
        } else prev_raw = cv[(size_t)(d.row_base + d.nrows - 1) * nb + b];
        TOT[c * nb + b] = run; LASTRAW[c * nb + b] = prev_raw;
      }
      __syncthreads();
      HPROF(4)                                             // in-chunk corrections
      // ---- corrections carried across chunks: detectDropAndCorrection (:673-686, Histogram.compare Histogram.scala:197-208) adds the
      //      previous chunk's last raw histogram when this chunk's first one compares lower; updateCorrection (:717-728) adds the
      //      chunk's own total.  carried(a, c) = (PT[c] - PT[a]) + (PD[c] - PD[a]) for a window whose chunk set starts at a.
      if (tid < n) {
        const int c = tid; bool less = false;
        if (c > 0) {
          for (int b = nb - 1; b >= 0; --b) {
            const double f = (double)cv[(size_t)CH[c].row_base * nb + b], l = (double)LASTRAW[(c - 1) * nb + b];
            if (f != l) { less = f < l; break; }
          }
        }
        LESS[c] = less ? 1 : 0;
      }
      __syncthreads();
      for (int b = tid; b < nb; b += HIST_THREADS) {
        int64_t pt = 0, pd = 0;
        PT[b] = 0; PD[b] = 0;
        for (int c = 0; c < n; ++c) {
          if (c > 0 && LESS[c]) pd += LASTRAW[(c - 1) * nb + b];
          PD[(size_t)c * nb + b] = pd;                      // PD[c] = sum_{1 <= j <= c} D_j
          PT[(size_t)c * nb + b] = pt;                      // PT[c] = sum_{j < c} tot_j
          pt += TOT[c * nb + b];
        }
      }
      // ---- per window: chunk set, row ranges, lowest / highest sample (HistogramRateFunctionBase.addTimeChunks, RateFunctions.scala:349-364)
      for (int k = tid; k < q.T; k += HIST_THREADS) {
        const int64_t wEnd = q.start + (int64_t)k * q.step, wStart = wEnd - winDur;
        HistWin w; w.a = -1; w.num_samples = 0; w.lo_t = INT64_MAX; w.hi_t = 0; w.lo_row = w.hi_row = 0; w.lo_c = w.hi_c = 0;
        for (int c = 0; c < n; ++c) {
          const HistChunkD d = CH[c];
          if (d.end_time < wStart) continue;                                  // ChunkSetInfo.scala:481-510 (time-ordered chunks)
          if (c > 0 && !(CH[c - 1].end_time < wEnd)) continue;
          if (w.a < 0) w.a = c;
          const int64_t* t = tss + d.row_base;
          int lo = 0, hi = d.nrows;                                           // first row with ts >= wStart (binarySearch & 0x7fffffff)
          while (lo < hi) { const int m = (lo + hi) >> 1; if (t[m] < wStart) lo = m + 1; else hi = m; }
          const int s = lo;
          lo = 0; hi = d.nrows;                                               // rows with ts <= wEnd: ceilingIndex = count - 1
          while (lo < hi) { const int m = (lo + hi) >> 1; if (t[m] <= wEnd) lo = m + 1; else hi = m; }
          int e = lo - 1; if (e > d.nrows - 1) e = d.nrows - 1;
          if (s <= e) {
            const int64_t tS = t[s], tE = t[e];
            if (tS < w.lo_t || tE > w.hi_t) {
              w.num_samples += e - s + 1;
              if (tS < w.lo_t) { w.lo_t = tS; w.lo_row = d.row_base + s; w.lo_c = c; }
              if (tE > w.hi_t) { w.hi_t = tE; w.hi_row = d.row_base + e; w.hi_c = c; }
            }
          }
        }
        if (w.hi_t > w.lo_t) {                       // RateFunctions.scala:72-111 with the per-window terms evaluated once
          const int64_t cws = q.inclusive ? wStart : wStart - 1;
          const double dTS = (double)(w.lo_t - cws) / 1000.0, dTE = (double)(wEnd - w.hi_t) / 1000.0, sI = (double)(w.hi_t - w.lo_t) / 1000.0;
          const double avg = sI / ((double)w.num_samples - 1.0), thr = avg * 1.1, half = avg / 2.0;
          const double endpart = dTE < thr ? dTE : half;
          const double eTI = (sI + (dTS < thr ? dTS : half)) + endpart;
          w.dTS = dTS; w.thr = thr; w.half = half; w.endpart = endpart; w.sI = sI; w.ratio0 = eTI / sI; w.skipC = 2.0 * dTS / sI;
        }
        W[k] = w;
        if (pq) any[k] = w.hi_t > w.lo_t;
      }
      __syncthreads();
      HPROF(5)                                             // carried corrections + window descriptors
      // ---- one thread per (window, bucket): extrapolatedRate on the corrected bucket values (HistogramRateFunctionBase.apply, :366-407)
      for (int i = tid; i < q.T * nb; i += HIST_THREADS) {
        const int k = i / nb, b = i - k * nb;
        const HistWin w = W[k];
        double r = NaNv; bool has = false;
        if (w.hi_t > w.lo_t) {
          const int64_t clo = (PT[(size_t)w.lo_c * nb + b] - PT[(size_t)w.a * nb + b]) + (PD[(size_t)w.lo_c * nb + b] - PD[(size_t)w.a * nb + b]);
          const int64_t chi = (PT[(size_t)w.hi_c * nb + b] - PT[(size_t)w.a * nb + b]) + (PD[(size_t)w.hi_c * nb + b] - PD[(size_t)w.a * nb + b]);
          const double lo = (double)(cv[(size_t)w.lo_row * nb + b] + clo), hi = (double)(cv[(size_t)w.hi_row * nb + b] + chi);
          const double delta = hi - lo;
          double ratio = w.ratio0;
          if (delta > 0 && lo >= 0 && !(lo > delta * w.skipC)) {                  // the zero-point clamp may apply (:84-90)
            const double dz = w.sI * (lo / delta);
            const double dts = dz < w.dTS ? dz : w.dTS;
            ratio = ((w.sI + (dts < w.thr ? dts : w.half)) + w.endpart) / w.sI;
          }
          const double scaled = delta * ratio;
          r = q.fn == FN_RATE ? __dmul_rn(div_invariant(scaled, fdiv, frcp), 1000.0) : scaled;
          has = true;
        }
        if (pq) acc[i] = r;
        else if (!agg) out[((size_t)sid * q.T + k) * nb + b] = r;             // an empty histogram is returned as NaN buckets
        else if (has) {                                                       // HistSumRowAggregator: empty histograms are skipped
          acc[i] += r;                                                        // (MutableHistogram.addNoCorrection: NaN-seeded sums start at 0)
          if (b == 0) any[k] = any[k] ? 2 : 1;                                // 1: the item's first histogram for this window (copied), 2: a further one
        }
      }
      __syncthreads();
      if (agg) {      // MutableHistogram.add = addNoCorrection + makeMonotonic for every histogram but the first (Histogram.scala:428-449)
        for (int k = tid; k < q.T; k += HIST_THREADS) {
          if (any[k] == 2 && W[k].hi_t > W[k].lo_t) {
            double mx = 0.0; double* a = acc + (size_t)k * nb;
            for (int b = 0; b < nb; ++b) { if (a[b] < mx || a[b] != a[b]) a[b] = mx; else if (a[b] > mx) mx = a[b]; }
          }
        }
        __syncthreads();
      }
      if (pq) present();
      HPROF(6)                                             // (window, bucket) rates
    }
    if (agg) {
      double* pv = pval + (size_t)it * q.T * nb; uint8_t* pa = pany + (size_t)it * q.T;
      for (int i = tid; i < q.T * nb; i += HIST_THREADS) pv[i] = acc[i];
      for (int i = tid; i < q.T; i += HIST_THREADS) pa[i] = any[i] ? 1 : 0;
      __syncthreads();
      HPROF(7)                                             // item partial written
    }
  }
  HPROF_FLUSH
  if (rows_scanned | bytes_scanned) { atomicAdd(&d_counters[0], (unsigned long long)rows_scanned); atomicAdd(&d_counters[1], (unsigned long long)bytes_scanned); }
}


// Fold the partial rows of each group in item order (deterministic), MutableHistogram.add per item (Histogram.scala:428-449),
// then Histogram.quantile (:65-108, hist_quantile in hist_phases.h).  Thread per (group, window).
__global__ void hist_merge_kernel(const double* __restrict__ pval, const uint8_t* __restrict__ pany, const int64_t* __restrict__ gis,
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
    const double* pv = pval + ((size_t)it * T + k) * nb;
    if (!any) { for (int b = 0; b < nb; ++b) v[b] = pv[b]; any = true; continue; }
    hist_add_monotonic(v, pv, 1, nb);
  }
  const double qv = (any && qtl == qtl) ? hist_quantile(v, nb, tops, qtl, exp_buckets != 0) : NaNv;
  if (out_values) for (int b = 0; b < nb; ++b) out_values[(size_t)i * nb + b] = any ? v[b] : NaNv;
  if (out_q) out_q[i] = qv;
}

#ifndef FILO_CUSIM      // launchers need nvcc
#ifdef FILO_HIST_PROF
extern "C" int filo_debug_hist_prof(unsigned long long* out16, int reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out16, g_hist_prof, sizeof(unsigned long long) * 16);
  if (e == cudaSuccess && reset) { unsigned long long z[16] = {}; e = cudaMemcpyToSymbol(g_hist_prof, z, sizeof z); }
  return (int)e;
}
#endif

size_t hist_smem_bytes(int max_rows, int nb, int T, bool agg, uint32_t max_rec) { return hist_layout(max_rows, nb, T, agg, max_rec).total; }
cudaError_t launch_hist_scan(const ScanLaunch& L, int nb, int max_rows, uint32_t max_rec, const int32_t* order, const int64_t* item_begin, int64_t n_items, int agg,
                             double* out, double* pval, uint8_t* pany, const double* tops, double qtl, int exp_buckets, double* out_q) {
  const size_t smem = hist_layout(max_rows, nb, L.q.T, agg != 0 || (!agg && out_q), max_rec).total;
  cudaError_t e = cudaFuncSetAttribute(hist_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  hist_scan_kernel<<<L.grid, HIST_THREADS, smem, L.stream>>>(L.arena, L.rec_off, L.n_series, L.q, nb, max_rows, max_rec, order, item_begin, n_items, agg,
                                                             out, pval, pany, L.d_counters, L.d_err, tops, qtl, exp_buckets, out_q);
  return cudaGetLastError();
}
cudaError_t launch_hist_merge(const double* pval, const uint8_t* pany, const int64_t* gis, int n_groups, int T, int nb, int exp_buckets, const double* tops, double q,
                              double* out_values, double* out_q, cudaStream_t s) {
  const int64_t n = (int64_t)n_groups * T;
  if (n <= 0) return cudaSuccess;
  hist_merge_kernel<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(pval, pany, gis, n_groups, T, nb, exp_buckets, tops, q, out_values, out_q);
  return cudaGetLastError();
}

#endif // FILO_CUSIM

} // namespace filo
