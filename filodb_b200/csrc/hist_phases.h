// Histogram column scan, second version: the per-series phases of hist_scan2_kernel (hist_kernels2.cu).
//
// Every phase is a function of (thread id, thread count, H2Ctx) with a CTA-wide barrier between phases, and is written to compile for
// the device AND for the host: tests/cpp/hist_emul.cpp runs the very same phase functions on the CPU (one loop over the thread ids per
// phase) and compares them with the oracle, so the kernel's logic is checked without a GPU.  Only the barrier placement, the smem
// carve-up and the global-memory staging are device-specific (hist_kernels2.cu).
//
// Differences to the first version (hist_kernels.cu): word-wise NibblePack group decode (hist_decode.h); every row decoded in ONE pass
// (the SectDelta base is added afterwards, element-wise); a thread per WINDOW computes the window's extrapolation terms in
// registers and walks the buckets (no window table in shared memory); the fused sum's accumulators live in the item's partial row
// in global memory (L2-resident, bucket-major so that the lanes' read-modify-writes coalesce).  Shared memory per CTA drops from
// ~215 KB to ~100 KB for 480 rows x 20 buckets: two CTAs per SM overlap each other's serial phases.
//
// Reference path: see hist_kernels.cu (SectDeltaHistogramReader HistogramVector.scala:628-738, Section.scala:146-227, NibblePack
// DeltaSink NibblePack.scala:208-230, HistogramRateFunctionBase RateFunctions.scala:330-418, extrapolatedRate :72-111).
#pragma once
#include <cstdint>
#include <cstring>
#include <cmath>
#include "filo_record.h"
#include "scan_params.h"
#include "hist_decode.h"

namespace filo {

constexpr int H2_THREADS = 512;
constexpr int H2_MAXC = 8;          // chunks in range per series
constexpr int H2_MAXSECT = 96;      // sections per series
#ifndef FILO_H2_BATCH
#define FILO_H2_BATCH 4
#endif
constexpr int H2_BATCH = FILO_H2_BATCH;         // buckets whose partial sums are loaded ahead of the arithmetic

struct H2Sect { int32_t chunk, start_row /* row (over the series' chunks in range) of the section's first histogram */, n, type; uint32_t first_rec /* byte offset in record */; };
struct H2Chunk { int32_t row_base, nrows, nsect, has_drop, sect, ts_wire; int64_t end_time; uint32_t ts_off, pad /* slope of const-DDV timestamps when the closed-form row search applies, else 0 */; };
// control block (shared memory): written by thread 0 in h2_tables, read by everyone afterwards
struct H2Ctl {
  H2Chunk ch[H2_MAXC];
  int32_t less[H2_MAXC];
  int32_t n, nsect, rows, cLo, err, bad;
  int64_t rows_scanned, bytes_scanned;         // this series' contribution to the scan counters
};

struct H2Layout { uint32_t cv, ts, pt, pd, tot, lastraw, sect, rsec, ctl, rec, total; int32_t pitch; };
FILO_HD inline H2Layout h2_layout(int max_rows, int nb, uint32_t max_rec) {
  H2Layout L; uint32_t o = 0;
  L.pitch = nb | 1;                                    // odd pitch (in 8-byte units): a warp's rows fall into distinct banks
  L.cv = o; o += (uint32_t)max_rows * (uint32_t)L.pitch * 8;
  L.ts = o; o += (uint32_t)max_rows * 8;
  L.pt = o; o += (H2_MAXC + 1) * (uint32_t)nb * 8;
  L.pd = o; o += (H2_MAXC + 1) * (uint32_t)nb * 8;
  L.tot = o; o += H2_MAXC * (uint32_t)nb * 8;
  L.lastraw = o; o += H2_MAXC * (uint32_t)nb * 8;
  L.sect = o; o += H2_MAXSECT * (uint32_t)sizeof(H2Sect);
  L.rsec = o; o += ((uint32_t)max_rows * 2 + 15) & ~15u;
  o = (o + 15) & ~15u;
  L.ctl = o; o += ((uint32_t)sizeof(H2Ctl) + 15) & ~15u;
  L.rec = o; o += ((max_rec + 15) & ~15u) + 16;        // + slack: the word-wise group decoder may touch 15 bytes past a group
  L.total = (o + 127) & ~127u;
  return L;
}

struct H2Ctx {
  uint8_t* smem; H2Layout L;
  QueryParams q; int32_t nb;
  int64_t winDur; double fdiv, frcp;
  FILO_HD int64_t* cv() const { return reinterpret_cast<int64_t*>(smem + L.cv); }
  FILO_HD int64_t* ts() const { return reinterpret_cast<int64_t*>(smem + L.ts); }
  FILO_HD int64_t* PT() const { return reinterpret_cast<int64_t*>(smem + L.pt); }
  FILO_HD int64_t* PD() const { return reinterpret_cast<int64_t*>(smem + L.pd); }
  FILO_HD int64_t* TOT() const { return reinterpret_cast<int64_t*>(smem + L.tot); }
  FILO_HD int64_t* LASTRAW() const { return reinterpret_cast<int64_t*>(smem + L.lastraw); }
  FILO_HD H2Sect* SE() const { return reinterpret_cast<H2Sect*>(smem + L.sect); }
  FILO_HD uint16_t* rsec() const { return reinterpret_cast<uint16_t*>(smem + L.rsec); }
  FILO_HD H2Ctl* ctl() const { return reinterpret_cast<H2Ctl*>(smem + L.ctl); }
  FILO_HD const uint8_t* rec() const { return smem + L.rec; }
};
FILO_HD inline void h2_ctx_init(H2Ctx& X, uint8_t* smem, const H2Layout& L, const QueryParams& q, int nb) {
  X.smem = smem; X.L = L; X.q = q; X.nb = nb;
  int64_t wd = q.inclusive ? q.window : q.window - 1; if (wd < 0) wd = 0;
  X.winDur = wd;
  X.fdiv = (double)(q.inclusive ? wd : wd + 1); X.frcp = 1.0 / X.fdiv;          // windowEnd - curWindowStart (RateFunctions.scala:436-442)
}

// ---- little-endian loads from the staged record (4-byte aligned fields; 64-bit fields may be only 4-byte aligned)
FILO_HDI uint32_t h2_ld16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
FILO_HDI uint32_t h2_ld32(const uint8_t* p) {
#if defined(__CUDA_ARCH__)
  return *reinterpret_cast<const uint32_t*>(p);
#else
  uint32_t v; std::memcpy(&v, p, 4); return v;
#endif
}
FILO_HDI uint64_t h2_ld64_a4(const uint8_t* p) { return (uint64_t)h2_ld32(p) | ((uint64_t)h2_ld32(p + 4) << 32); }
FILO_HDI double h2_nan() {
#if defined(__CUDA_ARCH__)
  return __longlong_as_double(0x7ff8000000000000LL);
#else
  const uint64_t b = 0x7ff8000000000000ull; double d; std::memcpy(&d, &b, 8); return d;
#endif
}
// IntBinaryVector element (IntBinaryVector.scala:306-457); `in` = inner vector start
FILO_HDI int32_t h2_int_apply(const uint8_t* in, int nbits, bool sgn, int n) {
  const uint8_t* d = in + 8;
  switch (nbits) {
    case 32: return (int32_t)h2_ld32(d + 4 * (size_t)n);
    case 16: { const uint32_t h = h2_ld16(d + 2 * (size_t)n); return sgn ? (int32_t)(int16_t)h : (int32_t)h; }
    case 8:  { const uint8_t b = d[n]; return sgn ? (int32_t)(int8_t)b : (int32_t)b; }
    case 4:  return ((int32_t)(int8_t)d[n >> 1] >> ((n & 1) * 4)) & 0x0f;
    case 2:  return ((int32_t)(int8_t)d[n >> 2] >> ((n & 3) * 2)) & 0x03;
  }
  return 0;
}
// timestamp of row r of a chunk: const DDV (DeltaDeltaVector.scala:237-290), raw i64, DDV (:147-229)
FILO_HDI int64_t h2_ts_of(const uint8_t* tv, int twire, int r) {
  if (twire == WIRE_DDV_CONST) return (int64_t)h2_ld64_a4(tv + 12) + (int64_t)(int32_t)((int32_t)h2_ld32(tv + 20) * r);
  if (twire == WIRE_RAW64) return (int64_t)h2_ld64_a4(tv + 8 + 8 * (size_t)r);
  const uint8_t* in = tv + 20; const uint32_t iw = h2_ld32(in + 4);
  return (int64_t)h2_ld64_a4(tv + 8) + (int64_t)(int32_t)h2_ld32(tv + 16) * r + (int64_t)h2_int_apply(in, (iw >> 16) & 0x7f, (iw >> 23) & 1, r);
}

// NibblePack.unpack8 literally (NibblePack.scala:395-447), for a group the record length cuts short
FILO_HDI uint64_t h2_rd_long(const uint8_t* p, int cap, int index) {
  uint64_t out = 0;
  for (int i = 0; i < 8 && index + i < cap; ++i) out |= (uint64_t)p[index + i] << (8 * i);
  return out;
}
FILO_HD inline int h2_unpack8_literal(const uint8_t* buf, int cap, uint64_t out[8], bool& short_in) {
  const uint32_t nonzeroMask = buf[0];
  if (nonzeroMask == 0) { for (int i = 0; i < 8; ++i) out[i] = 0; return 1; }
  const int numNibblesU8 = cap > 1 ? buf[1] : 0;
  const int numBits = ((numNibblesU8 >> 4) + 1) * 4, trailingZeroes = (numNibblesU8 & 0x0f) * 4;
  const int total = 2 + (numBits * hd_popc(nonzeroMask) + 7) / 8;
  const uint64_t mask = numBits >= 64 ? ~0ull : ((1ull << numBits) - 1);
  int bufIndex = 2, bitCursor = 0;
  uint64_t inWord = h2_rd_long(buf, cap, bufIndex); bufIndex += 8;
  for (int bit = 0; bit < 8; ++bit) {
    if (nonzeroMask & (1u << bit)) {
      const int remaining = 64 - bitCursor;
      uint64_t outWord = (inWord >> bitCursor) & mask;
      if (remaining <= numBits && bufIndex < total) {
        if (bufIndex < cap) { inWord = h2_rd_long(buf, cap, bufIndex); bufIndex += 8; if (remaining < numBits) outWord |= (inWord << remaining) & mask; }
        else { short_in = true; for (int j = bit; j < 8; ++j) out[j] = 0; return total; }
      }
      out[bit] = outWord << trailingZeroes;
      bitCursor = (bitCursor + numBits) % 64;
    } else out[bit] = 0;
  }
  return total;
}
// one histogram record (u16 length + NibblePack delta bytes) -> cumulative bucket values of the record itself (DeltaSink)
FILO_HD inline void h2_decode_record(const uint8_t* rec, int nb, int64_t* out, bool& bad) {
  int cap = (int)h2_ld16(rec);
  const uint8_t* p = rec + 2;
  int64_t current = 0; int i = 0;
  while (i < nb && cap > 0) {
    uint64_t data[8];
    int used;
    if (p[0] == 0 || (cap >= 2 && nibble_group_bytes(p) <= cap)) used = nibble_unpack8_inbounds(p, data);
    else {
      uint64_t slow[8];
      used = h2_unpack8_literal(p, cap, slow, bad);
#pragma unroll
      for (int n = 0; n < 8; ++n) data[n] = slow[n];
    }
#pragma unroll
    for (int n = 0; n < 8; ++n) if (i + n < nb) { current += (int64_t)data[n]; out[i + n] = current; }
    i += 8;
    if (cap > used) { p += used; cap -= used; } else cap = 0;
  }
  for (; i < nb; ++i) out[i] = 0;                          // input ran out: remaining deltas are zero (unpackToSink stops)
}

// ---------------------------------------------------------------------------------------------------------------- phases
// P1 (thread 0): chunks in range, section table, scan counters.  err: 1 corrupt vector, 5 unsupported shape.
FILO_HD inline void h2_tables(int tid, const H2Ctx& X, int max_rows) {
  if (tid != 0) return;
  const uint8_t* rec = X.rec();
  const RecordHeader* h = reinterpret_cast<const RecordHeader*>(rec);
  const ChunkEntry* E = reinterpret_cast<const ChunkEntry*>(rec + sizeof(RecordHeader));
  H2Ctl* C = X.ctl(); H2Sect* SE = X.SE();
  const QueryParams& q = X.q; const int nb = X.nb;
  const int nch = (int)h->n_chunks;
  const int64_t t1 = q.start - q.window, t2 = q.end;
  int cLo = 0; while (cLo < nch && E[cLo].end_time < t1) ++cLo;
  int cHi = cLo; while (cHi < nch && E[cHi].start_time <= t2) ++cHi;
  if (t1 > t2) cHi = cLo;
  int err = 0, rows = 0, nsect = 0;
  int64_t rows_scanned = 0, bytes_scanned = 0;
  const int n = cHi - cLo;
  if (n > H2_MAXC) err = 5;
  const int64_t lastEnd = q.start + (int64_t)(q.T - 1) * q.step;
  for (int c = 0; c < n && !err; ++c) {
    const ChunkEntry& e = E[cLo + c];
    const uint8_t* hv = rec + e.val_off;
    const uint32_t w4 = h2_ld32(hv + 4);
    const int wire = (int)(w4 & 0xffff), numHist = (int)(w4 >> 16) & 0xffff;         // u16 wire at +4, u16 numHistograms at +6
    const int defBytes = (int)h2_ld16(hv + 9), vnb = (int)h2_ld16(hv + 11);
    // counter functions need the SectDelta reader (a RowHistogramReader is not a CounterVectorReader, RangeFunction.scala:142)
    if (wire != WIRE_H_SECTDELTA || vnb != nb || numHist < e.num_rows) { err = 1; break; }
    H2Chunk d; d.sect = 1; d.pad = 0; d.row_base = rows; d.nrows = e.num_rows; d.nsect = 0; d.has_drop = 0; d.end_time = e.end_time;
    d.ts_off = e.ts_off; d.ts_wire = (int)(h2_ld32(rec + e.ts_off + 4) & 0xffff);
    if (d.ts_wire == WIRE_DDV_CONST) {                    // regular timestamps: the window's row range in closed form (h2_window); slope kept when no int32 wrap can occur
      const int32_t slope = (int32_t)h2_ld32(rec + e.ts_off + 20);
      if (slope > 0 && (int64_t)slope * (int64_t)(e.num_rows > 0 ? e.num_rows - 1 : 0) < 0x7fffffffLL) d.pad = (uint32_t)slope;
    }
    const uint8_t* endp = hv + (int32_t)h2_ld32(hv) + 4;
    const uint8_t* s = hv + 11 + defBytes; int start = 0;
    while (s + 4 <= endp && start < numHist) {
      const uint32_t sh = (uint32_t)s[0] | ((uint32_t)s[1] << 8) | ((uint32_t)s[2] << 16) | ((uint32_t)s[3] << 24);
      const int sbytes = (int)(sh & 0xffff), sn = (int)((sh >> 16) & 0xff), stype = (int)(sh >> 24);
      if (s + 4 + sbytes > endp || sn == 0 || start >= e.num_rows) break;
      if (nsect >= H2_MAXSECT) { err = 5; break; }
      H2Sect S; S.chunk = c; S.start_row = rows + start; S.n = sn < e.num_rows - start ? sn : e.num_rows - start; S.type = stype; S.first_rec = (uint32_t)((s + 4) - rec);
      SE[nsect] = S;                                     // rows past numRows are not read
      if (stype == 1 && start > 0) d.has_drop = 1;
      ++nsect; ++d.nsect; start += sn; s += 4 + sbytes;
    }
    if (!err && start < e.num_rows) err = 1;
    C->ch[c] = d; rows += e.num_rows;
    // CountingChunkInfoIterator: a chunk the window iterator never pulls is not counted (ChunkSetInfo.scala:336-380)
    if (!(c > 0 && !(E[cLo + c - 1].end_time < lastEnd))) { rows_scanned += e.num_rows; bytes_scanned += (int64_t)h2_ld32(rec + e.ts_off) + 4 + (int64_t)h2_ld32(hv) + 4; }
  }
  if (!err && (rows > max_rows || rows > 65535)) err = 5;
  C->n = err ? 0 : n; C->nsect = err ? 0 : nsect; C->rows = err ? 0 : rows; C->err = err; C->cLo = cLo; C->bad = 0;
  C->rows_scanned = err ? 0 : rows_scanned; C->bytes_scanned = err ? 0 : bytes_scanned;
}

// P2 (thread per row): timestamp, the record's own cumulative buckets, and the row whose histogram is its SectDelta base
FILO_HD inline void h2_decode_rows(int tid, int nthreads, const H2Ctx& X) {
  H2Ctl* C = X.ctl(); const H2Sect* SE = X.SE(); const uint8_t* rec = X.rec();
  int64_t* cv = X.cv(); int64_t* tss = X.ts(); uint16_t* rsec = X.rsec();
  const int n = C->n, nsect = C->nsect, rows = C->rows, nb = X.nb, pitch = X.L.pitch;
  bool bad = false;
  for (int r = tid; r < rows; r += nthreads) {
    int c = 0; while (c + 1 < n && r >= C->ch[c + 1].row_base) ++c;
    const H2Chunk& d = C->ch[c];
    tss[r] = h2_ts_of(rec + d.ts_off, d.ts_wire, r - d.row_base);
    int si = 0; while (si + 1 < nsect && r >= SE[si + 1].start_row) ++si;
    const H2Sect S = SE[si];
    int64_t* o = cv + (size_t)r * pitch;
    if (r >= S.start_row + S.n) { rsec[r] = (uint16_t)r; for (int b = 0; b < nb; ++b) o[b] = 0; continue; }
    const uint8_t* p = rec + S.first_rec;
    for (int k = r - S.start_row; k > 0; --k) p += (int)h2_ld16(p) + 2;          // SectionReader.skipAhead
    h2_decode_record(p, nb, o, bad);
    rsec[r] = (uint16_t)S.start_row;                     // SectDelta: rows after a section's first hold the delta from it (:646-666)
  }
  if (bad) C->bad = 1;                                   // benign race: every writer stores 1
}
// P3 (thread per (row, bucket)): add the section's first histogram
FILO_HD inline void h2_add_base(int tid, int nthreads, const H2Ctx& X) {
  const H2Ctl* C = X.ctl(); int64_t* cv = X.cv(); const uint16_t* rsec = X.rsec();
  const int rows = C->rows, nb = X.nb, pitch = X.L.pitch;
  // i / nb = (i * magic) >> 32 with magic = ceil(2^32 / nb): exact while i * (magic * nb - 2^32) < 2^32, i.e. for every i < 2^26 at nb <= 64
  // (rows * nb <= 2^16 * 64 here); nb = 1 has no 32-bit magic
  const uint32_t magic = nb > 1 ? (uint32_t)((0x100000000ull + (uint32_t)nb - 1) / (uint32_t)nb) : 0u;
  for (int i = tid; i < rows * nb; i += nthreads) {
    const int r = nb > 1 ? (int)(((uint64_t)(uint32_t)i * magic) >> 32) : i, b = i - r * nb;
    const int r0 = rsec[r];
    if (r0 != r) cv[(size_t)r * pitch + b] += cv[(size_t)r0 * pitch + b];
  }
}
// P4 (thread per (chunk, bucket)): corrections inside a chunk (lazy val corrections, :690-707; correctedValue :730-746): every Drop
// section starting at row ci > 0 adds the RAW histogram of row ci-1 to all rows >= ci
FILO_HD inline void h2_chunk_corrections(int tid, int nthreads, const H2Ctx& X) {
  const H2Ctl* C = X.ctl(); const H2Sect* SE = X.SE(); int64_t* cv = X.cv();
  int64_t* TOT = X.TOT(); int64_t* LASTRAW = X.LASTRAW();
  const int n = C->n, nsect = C->nsect, nb = X.nb, pitch = X.L.pitch;
  for (int cb = tid; cb < n * nb; cb += nthreads) {
    const int c = cb / nb, b = cb - c * nb;
    const H2Chunk d = C->ch[c];
    int64_t run = 0, prev_raw = 0;
    if (d.has_drop) {
      int si = 0; while (si < nsect && SE[si].chunk != c) ++si;
      for (; si < nsect && SE[si].chunk == c; ++si) {
        const H2Sect S = SE[si];
        if (S.type == 1 && S.start_row > d.row_base) run += prev_raw;
        for (int r = S.start_row; r < S.start_row + S.n && r < d.row_base + d.nrows; ++r) { const int64_t x = cv[(size_t)r * pitch + b]; prev_raw = x; cv[(size_t)r * pitch + b] = x + run; }
      }
    } else prev_raw = cv[(size_t)(d.row_base + d.nrows - 1) * pitch + b];
    TOT[c * nb + b] = run; LASTRAW[c * nb + b] = prev_raw;
  }
}
// P5 (thread per chunk): does the chunk's first histogram compare lower than the previous chunk's last raw one
// (detectDropAndCorrection :673-686, Histogram.compare Histogram.scala:197-208: from the top bucket down)
FILO_HD inline void h2_chunk_less(int tid, const H2Ctx& X) {
  H2Ctl* C = X.ctl(); const int64_t* cv = X.cv(); const int64_t* LASTRAW = X.LASTRAW();
  const int n = C->n, nb = X.nb, pitch = X.L.pitch;
  if (tid >= n) return;
  const int c = tid; bool less = false;
  if (c > 0) {
    for (int b = nb - 1; b >= 0; --b) {
      const double f = (double)cv[(size_t)C->ch[c].row_base * pitch + b], l = (double)LASTRAW[(c - 1) * nb + b];
      if (f != l) { less = f < l; break; }
    }
  }
  C->less[c] = less ? 1 : 0;
}
// P6 (thread per bucket): corrections carried across chunks.  carried(a, c) = (PT[c] - PT[a]) + (PD[c] - PD[a]) (stored summed, see below) for a window whose
// chunk set starts at a (updateCorrection :717-728 adds the chunk's own total, detectDropAndCorrection the previous last raw value)
FILO_HD inline void h2_carried(int tid, int nthreads, const H2Ctx& X) {
  const H2Ctl* C = X.ctl(); int64_t* PT = X.PT(); int64_t* PD = X.PD(); const int64_t* TOT = X.TOT(); const int64_t* LASTRAW = X.LASTRAW();
  const int n = C->n, nb = X.nb;
  for (int b = tid; b < nb; b += nthreads) {
    int64_t pt = 0, pd = 0;
    PT[b] = 0; PD[b] = 0;
    for (int c = 0; c < n; ++c) {
      if (c > 0 && C->less[c]) pd += LASTRAW[(c - 1) * nb + b];
      PD[(size_t)c * nb + b] = pd;
      PT[(size_t)c * nb + b] = (int64_t)((uint64_t)pt + (uint64_t)pd);   // one table: (PT[c] - PT[a]) + (PD[c] - PD[a]) = (PT + PD)[c] - (PT + PD)[a] in the JVM's wrapping long arithmetic
      pt += TOT[c * nb + b];
    }
  }
}

FILO_HDI double h2_div_window(double x, double fdiv, double frcp) {
#if defined(__CUDA_ARCH__)
  // x / fdiv with the reciprocal precomputed: q0 = RN(x * rcp), one exact-remainder correction (Markstein); see scan_fast.cuh div_invariant
  const double q0 = __dmul_rn(x, frcp);
  const uint32_t ex = ((uint32_t)__double2hiint(q0) >> 20) & 0x7ff;
  if (ex > 64u && ex < 1983u) { const double r = __fma_rn(-q0, fdiv, x); return __fma_rn(r, frcp, q0); }
  if (x == 0.0) return q0;
  return x / fdiv;
#else
  (void)frcp; return x / fdiv;
#endif
}

// extrapolation ratio of a bucket whose zero point may lie inside the window (RateFunctions.scala:84-90: durationToZero = sampledInterval *
// (startValue / delta), durationToStart clamped to it).  Two IEEE divisions, needed for a few buckets near a series' start or a reset:
// kept out of line on the device (inline, the compiler if-converts them into every bucket of every window)
#if defined(__CUDACC__) && !defined(FILO_CUSIM)
static __host__ __device__ __noinline__ double h2_clamped_ratio(double sI, double lo, double delta, double dTS, double thr, double half, double endpart) {
#else
inline double h2_clamped_ratio(double sI, double lo, double delta, double dTS, double thr, double half, double endpart) {
#endif
  const double dz = sI * (lo / delta);
  const double dts = dz < dTS ? dz : dTS;
  return ((sI + (dts < thr ? dts : half)) + endpart) / sI;
}

// P7 (thread per window): chunk set, row ranges, lowest / highest sample (HistogramRateFunctionBase.addTimeChunks, RateFunctions.scala:349-364),
// then extrapolatedRate per bucket (:72-111, :366-407) folded into the item's partial row pv[b * T + k] (HistSumRowAggregator: empty
// histograms are skipped; `first`: no series of the item has produced a histogram for this window yet).  Returns true when the window produced a histogram.
// SERIES: the series' own window histogram is stored, bucket b at pv[b * ws] (pv already points at the window's first bucket).
template <bool SERIES = false>
FILO_HD inline bool h2_window(int k, const H2Ctx& X, double* pv, bool first, size_t ws = 0) {
  const H2Ctl* C = X.ctl(); const int64_t* cv = X.cv(); const int64_t* tss = X.ts(); const int64_t* PT = X.PT();
  const QueryParams& q = X.q; const int n = C->n, nb = X.nb, pitch = X.L.pitch;
  const int64_t wEnd = q.start + (int64_t)k * q.step, wStart = wEnd - X.winDur;
  int a = -1, num_samples = 0, lo_row = 0, hi_row = 0, lo_c = 0, hi_c = 0; int64_t lo_t = INT64_MAX, hi_t = 0;
  for (int c = 0; c < n; ++c) {
    const H2Chunk& d = C->ch[c];
    if (d.end_time < wStart) continue;                                  // ChunkSetInfo.scala:481-510 (time-ordered chunks)
    if (c > 0 && !(C->ch[c - 1].end_time < wEnd)) continue;
    if (a < 0) a = c;
    const int64_t* t = tss + d.row_base;
    int s, e;
    if (d.pad != 0 && d.nrows > 0) {                                    // t[r] = t[0] + slope * r: the same two row numbers without the searches
      const uint32_t slope = d.pad; const int64_t t0 = t[0], span = (int64_t)slope * (int64_t)(d.nrows - 1);
      const int64_t ds = wStart - t0, de = wEnd - t0;
      s = ds <= 0 ? 0 : ds > span ? d.nrows : (int)(((uint32_t)ds + slope - 1) / slope);
      e = de < 0 ? -1 : de >= span ? d.nrows - 1 : (int)((uint32_t)de / slope);
    } else {
      int lo = 0, hi = d.nrows;                                         // first row with ts >= wStart (binarySearch & 0x7fffffff)
      while (lo < hi) { const int m = (lo + hi) >> 1; if (t[m] < wStart) lo = m + 1; else hi = m; }
      s = lo;
      lo = 0; hi = d.nrows;                                             // rows with ts <= wEnd: ceilingIndex = count - 1
      while (lo < hi) { const int m = (lo + hi) >> 1; if (t[m] <= wEnd) lo = m + 1; else hi = m; }
      e = lo - 1; if (e > d.nrows - 1) e = d.nrows - 1;
    }
    if (s <= e) {
      const int64_t tS = t[s], tE = t[e];
      if (tS < lo_t || tE > hi_t) {
        num_samples += e - s + 1;
        if (tS < lo_t) { lo_t = tS; lo_row = d.row_base + s; lo_c = c; }
        if (tE > hi_t) { hi_t = tE; hi_row = d.row_base + e; hi_c = c; }
      }
    }
  }
  if (!(hi_t > lo_t)) return false;
  // RateFunctions.scala:72-111 with the per-window terms evaluated once (all buckets share the sample times)
  const int64_t cws = q.inclusive ? wStart : wStart - 1;
  const double dTS = (double)(lo_t - cws) / 1000.0, dTE = (double)(wEnd - hi_t) / 1000.0, sI = (double)(hi_t - lo_t) / 1000.0;
  const double avg = sI / ((double)num_samples - 1.0), thr = avg * 1.1, half = avg / 2.0;
  const double endpart = dTE < thr ? dTE : half;
  const double eTI = (sI + (dTS < thr ? dTS : half)) + endpart;
  const double ratio0 = eTI / sI, skipC = 2.0 * dTS / sI;
  const uint64_t* plo = reinterpret_cast<const uint64_t*>(PT) + (size_t)lo_c * nb; const uint64_t* pla = reinterpret_cast<const uint64_t*>(PT) + (size_t)a * nb;
  const uint64_t* phi = reinterpret_cast<const uint64_t*>(PT) + (size_t)hi_c * nb;
  const int64_t* rlo = cv + (size_t)lo_row * pitch; const int64_t* rhi = cv + (size_t)hi_row * pitch;
  const bool is_rate = q.fn == FN_RATE;
  const bool carried = (lo_c != a) | (hi_c != a);                         // false for a window inside one chunk: both differences are 0
  // buckets in batches of H2_BATCH: the partial row lives in global memory (L2); loading a batch's old sums before computing keeps
  // several loads in flight instead of one load -> add -> store chain per bucket
  // HistSumRowAggregator.reduceAggregate (HistSumRowAggregator.scala:25-36): the first histogram of the partial row is copied, every
  // further one goes through MutableHistogram.add = addNoCorrection + makeMonotonic (Histogram.scala:428-449): running maximum mx
  double mx = 0.0;
  double* pk = SERIES ? pv : pv + k;                                        // bucket b of window k at pk[b * T] (SERIES: pk[b * ws])
  const size_t Tq = SERIES ? ws : (size_t)q.T;
  for (int b0 = 0; b0 < nb; b0 += H2_BATCH, pk += (size_t)H2_BATCH * Tq) {
    double old[H2_BATCH];
#pragma unroll
    for (int j = 0; j < H2_BATCH; ++j) if (!SERIES && b0 + j < nb) old[j] = pk[(size_t)j * Tq];
#pragma unroll
    for (int j = 0; j < H2_BATCH; ++j) {
      const int b = b0 + j;
      if (b < nb) {
        int64_t clo = 0, chi = 0;                                          // corrections carried from earlier chunks of the window's chunk set
        if (carried) { const uint64_t base = pla[b]; clo = (int64_t)(plo[b] - base); chi = (int64_t)(phi[b] - base); }
        const double lo = (double)(rlo[b] + clo), hi = (double)(rhi[b] + chi);
        const double delta = hi - lo;
        double ratio = ratio0;
        if (delta > 0 && lo >= 0 && !(lo > delta * skipC))                  // the zero-point clamp may apply (:84-90): rare, out of line
          ratio = h2_clamped_ratio(sI, lo, delta, dTS, thr, half, endpart);
        const double scaled = delta * ratio;
        const double r = is_rate ? h2_div_window(scaled, X.fdiv, X.frcp) * 1000.0 : scaled;
        if (SERIES) { pk[(size_t)j * Tq] = r; continue; }
        double nv = old[j] + r;                                             // MutableHistogram.addNoCorrection: NaN-seeded sums start at 0
        if (!first) { nv = nv >= mx ? nv : mx; mx = nv > mx ? nv : mx; }    // makeMonotonic: below the running maximum (or NaN) -> the maximum
        pk[(size_t)j * Tq] = nv;
      }
    }
  }
  return true;
}

// `last` of one window, shared by both histogram kernels (ch: their chunk descriptors with row_base / nrows / end_time, tss: the decoded
// timestamps of the series' rows): LastSampleChunkedFunction.addChunks (RangeFunction.scala:599-614) keeps, over the window's chunk set
// (as h2_window), the row endRowNum = min(ceilingIndex(windowEnd), numRows - 1) of a chunk when its timestamp is >= windowStart and > the
// timestamp kept so far.  Returns that row, or -1 (Histogram.empty).
template <class Chunk>
FILO_HD inline int hist_last_row(const Chunk* ch, int n, const int64_t* tss, int64_t wStart, int64_t wEnd) {
  int64_t kept = -1; int row = -1;                                      // LastSampleChunkedFunction.timestamp starts at -1
  for (int c = 0; c < n; ++c) {
    const Chunk& d = ch[c];
    if (d.end_time < wStart) continue;                                  // ChunkSetInfo.scala:481-510 (time-ordered chunks)
    if (c > 0 && !(ch[c - 1].end_time < wEnd)) continue;
    const int64_t* t = tss + d.row_base;
    int lo = 0, hi = d.nrows;                                           // ceilingIndex: rows with ts <= wEnd, minus one
    while (lo < hi) { const int m = (lo + hi) >> 1; if (t[m] <= wEnd) lo = m + 1; else hi = m; }
    int e = lo - 1; if (e > d.nrows - 1) e = d.nrows - 1;
    if (e >= 0 && t[e] >= wStart && t[e] > kept) { kept = t[e]; row = d.row_base + e; }
  }
  return row;
}
// P7 for `last` (thread per window; P4-P6 do not run, the rows hold the raw reader values after P3)
FILO_HD inline int h2_last_row(int k, const H2Ctx& X) {
  const int64_t wEnd = X.q.start + (int64_t)k * X.q.step;
  return hist_last_row(X.ctl()->ch, X.ctl()->n, X.ts(), wEnd - X.winDur, wEnd);
}
// `last` of window k: LastSampleChunkedFunctionH.updateValue takes asHistReader(endRowNum), the raw value (no counter correction).
// Fused: folded into the partial row like h2_window; SERIES: stored at pv[b * ws].
template <bool SERIES = false>
FILO_HD inline bool h2_window_last(int k, const H2Ctx& X, double* pv, bool first, size_t ws = 0) {
  const int row = h2_last_row(k, X);
  if (row < 0) return false;
  const int64_t* r = X.cv() + (size_t)row * X.L.pitch;
  const int nb = X.nb;
  double* pk = SERIES ? pv : pv + k;
  const size_t Tq = SERIES ? ws : (size_t)X.q.T;
  double mx = 0.0;
  for (int b = 0; b < nb; ++b) {
    const double v = (double)r[b];
    if (SERIES) { pk[(size_t)b * Tq] = v; continue; }
    double nv = pk[(size_t)b * Tq] + v;                                 // HistSumRowAggregator fold, as in h2_window
    if (!first) { nv = nv >= mx ? nv : mx; mx = nv > mx ? nv : mx; }
    pk[(size_t)b * Tq] = nv;
  }
  return true;
}

// MutableHistogram.add of a further histogram p[b * ps] into the running sum v (Histogram.scala:428-449): addNoCorrection, a bucket-wise
// sum, then makeMonotonic: a bucket below the running maximum, or NaN, becomes that maximum.  The step of every merge kernel
// (hist_merge_kernel, hist_merge2_kernel, hist_merge_parts_kernel); the first histogram of a fold is copied, not added.
FILO_HDI void hist_add_monotonic(double* v, const double* p, size_t ps, int nb) {
  double mx = 0.0;
  for (int b = 0; b < nb; ++b) { double nv = v[b] + p[(size_t)b * ps]; if (nv < mx || nv != nv) nv = mx; else if (nv > mx) mx = nv; v[b] = nv; }
}

// Histogram.quantile (vectors/Histogram.scala:65-108; min = 0, max = +Inf, evenDistribution = false) over cumulative bucket sums v[b * vs]
// with bucket tops tops[nb]; exp_buckets: Base2ExpHistogramBuckets interpolate in log2 space except in the zero bucket (:97-104, log2 :111).
// No makeMonotonic: firstBucketGTE walks up from bucket 0 as the reference does, also over a non-monotonic per-series histogram.
FILO_HD inline double hist_quantile(const double* v, size_t vs, int nb, const double* tops, double qtl, bool exp_buckets) {
  const double NaNv = h2_nan(), Inf = HUGE_VAL;
  const double top = v[(size_t)(nb - 1) * vs];
  if (qtl < 0) return -Inf;
  if (qtl > 1) return Inf;
  if (nb < 2 || !(top > 0)) return NaNv;
  double rank = qtl * top;
  int bucket = 0; while (v[(size_t)bucket * vs] < rank) ++bucket;
  const double bucketStart = bucket == 0 ? 0.0 : tops[bucket - 1];
  const double bucketEnd = tops[bucket];
  if (bucket == nb - 1 && bucketEnd == Inf) return tops[nb - 2];
  if (bucket == 0 && tops[0] <= 0) return tops[0];
  const double count = bucket == 0 ? v[(size_t)bucket * vs] : v[(size_t)bucket * vs] - v[(size_t)(bucket - 1) * vs];
  rank -= (bucket == 0 ? 0.0 : v[(size_t)(bucket - 1) * vs]);
  const double fraction = rank / count;
  if (!exp_buckets || bucketStart == 0) return bucketStart + (bucketEnd - bucketStart) * fraction;
  const double ln2 = log(2.0), logEnd = log(bucketEnd) / ln2, logStart = log(bucketStart) / ln2;
  return pow(2.0, logStart + (logEnd - logStart) * fraction);
}
FILO_HD inline double hist_quantile(const double* v, int nb, const double* tops, double qtl, bool exp_buckets) {
  return hist_quantile(v, (size_t)1, nb, tops, qtl, exp_buckets);
}

} // namespace filo
