// The per-series and `last` modes of the histogram kernels on the CPU (test infrastructure; built and run by tests/test_hist_series_emul.py):
//   hist_scan2_kernel<SERIES = true, LAST> (hist_kernels2.cu) and hist_scan_kernel with its per-series quantile stage and `last`
//   (hist_kernels.cu, through tests/cpp/make_cusim_src.py), compiled for the host on the cusim emulator, and the fused `last`
//   (hist_scan2_kernel<false, true> + hist_merge2_kernel, hist_scan_kernel + hist_merge_kernel).
// Checked bit for bit, quantile bits included, against the oracle: periodicSamplesHist (oracle/filo_hist.hpp) for rate / increase /
// sum_over_time, the restatement of LastSampleChunkedFunctionH below for `last`, MutableHistogram.quantile for every quantile.
//     hist_series_emul [schedule seed]
#define FILO_CUSIM 1
#include "cusim.h"
namespace filo { alignas(128) uint8_t smem[232448]; }
#include "../../filodb_b200/csrc/hist_kernels2.cu"
#include HIST_V1_SRC                                             // hist_kernels.cu with function-scope __shared__ turned into static
#include "../../oracle/filo_hist.hpp"
#include <memory>
#include <random>

namespace H = fo::hist;
struct Chunk { std::vector<uint8_t> ts, hv, info; };
struct Series { std::vector<std::unique_ptr<Chunk>> chunks; std::vector<uint8_t> record; };

// the series builder of tests/cpp/hist_kernel_emul.cpp: cumulative bucket counts (resets inside chunks and at chunk starts) or per-row
// (delta) histograms, timestamps with optional jitter, encoded by the oracle's appenders into one device record
static void build_series(Series& S, std::mt19937_64& rng, const H::Buckets& b, int rows, const std::vector<int>& chunk_rows, int64_t t0, int step_ms, int jitter,
                         int reset_every, bool sect, bool cumulative) {
  const int nb = b.n;
  std::vector<int64_t> ts((size_t)rows), vals((size_t)rows * nb), cur((size_t)nb, 0);
  std::vector<char> boundary((size_t)rows + 1, 0);
  { int r0 = 0; for (int n : chunk_rows) { r0 += n; if (r0 < rows) boundary[(size_t)r0] = 1; } }
  for (int r = 0; r < rows; ++r) {
    ts[(size_t)r] = t0 + (int64_t)r * step_ms + (jitter ? (int64_t)(rng() % (uint64_t)(2 * jitter + 1)) - jitter : 0);
    if (!cumulative) std::fill(cur.begin(), cur.end(), 0);        // delta temporality: every row stands alone
    else if (reset_every && r > 0 && (rng() % (uint64_t)reset_every == 0 || (boundary[(size_t)r] && rng() % 2))) std::fill(cur.begin(), cur.end(), 0);
    std::vector<int64_t> inc((size_t)nb, 0);
    const int k = 1 + (int)(rng() % 3);
    for (int j = 0; j < k; ++j) inc[(size_t)(rng() % (uint64_t)nb)] += 1 + (int64_t)(rng() % 5);
    int64_t acc = 0;
    for (int i = 0; i < nb; ++i) { acc += inc[(size_t)i]; cur[(size_t)i] += acc; vals[(size_t)r * nb + i] = cur[(size_t)i]; }
  }
  int r0 = 0;
  for (int n : chunk_rows) {
    auto c = std::make_unique<Chunk>();
    c->ts = fo::enc::timestamps(ts.data() + r0, n);
    H::HistAppender app(sect, 60000);
    for (int r = 0; r < n; ++r) {
      std::vector<uint8_t> blob = H::bin::writeDelta(b, vals.data() + (size_t)(r0 + r) * nb, nb);
      if (app.addData(blob.data(), (int)blob.size()) != H::Ack) { std::printf("appender failed\n"); std::exit(2); }
    }
    c->hv = app.bytes();
    c->info.assign(fo::csi::OffsetVectors + 16, 0);
    fo::setLong(c->info.data() + fo::csi::OffsetChunkID, fo::csi::chunkID(ts[(size_t)r0], (ts[(size_t)(r0 + n - 1)] + 1000) / 1000));
    fo::setInt(c->info.data() + fo::csi::OffsetNumRows, n);
    fo::setLong(c->info.data() + fo::csi::OffsetIngestionTime, ts[(size_t)(r0 + n - 1)] + 1000);
    fo::setLong(c->info.data() + fo::csi::OffsetEndTime, ts[(size_t)(r0 + n - 1)]);
    fo::setLong(c->info.data() + fo::csi::OffsetVectors, (int64_t)(uintptr_t)c->ts.data());
    fo::setLong(c->info.data() + fo::csi::OffsetVectors + 8, (int64_t)(uintptr_t)c->hv.data());
    S.chunks.push_back(std::move(c));
    r0 += n;
  }
  const size_t nch = S.chunks.size(), off = sizeof(filo::RecordHeader) + nch * sizeof(filo::ChunkEntry);
  std::vector<filo::ChunkEntry> E(nch); std::vector<uint8_t> body; uint32_t row_base = 0;
  for (size_t i = 0; i < nch; ++i) {
    Chunk& c = *S.chunks[i];
    E[i].start_time = fo::csi::startTime(c.info.data()); E[i].end_time = fo::csi::endTime(c.info.data()); E[i].num_rows = fo::csi::numRows(c.info.data());
    auto put = [&](const std::vector<uint8_t>& v) { while ((off + body.size()) % 8) body.push_back(0); const uint32_t o = (uint32_t)(off + body.size()); body.insert(body.end(), v.begin(), v.end()); return o; };
    E[i].ts_off = put(c.ts); E[i].val_off = put(c.hv); E[i].row_base = row_base; row_base += (uint32_t)E[i].num_rows;
  }
  size_t total = off + body.size(); total = (total + 15) & ~(size_t)15;
  S.record.assign(total, 0);
  filo::RecordHeader h; h.rec_bytes = (uint32_t)total; h.n_chunks = (uint32_t)nch; h.n_rows = row_base; h.flags = filo::REC_HIST;
  std::memcpy(S.record.data(), &h, sizeof h);
  std::memcpy(S.record.data() + sizeof h, E.data(), nch * sizeof(filo::ChunkEntry));
  std::memcpy(S.record.data() + off, body.data(), body.size());
}
static bool same_bits(double a, double b) { uint64_t x, y; std::memcpy(&x, &a, 8); std::memcpy(&y, &b, 8); return x == y || (a != a && b != b); }

// LastSampleChunkedFunction.addChunks + LastSampleChunkedFunctionH.updateValue (RangeFunction.scala:599-614, 630-640), driven by the chunk set
// of WindowedChunkIterator for time-ordered chunks (ChunkSetInfo.scala:481-510, as periodicSamplesHist): per window the row
// endRowNum = min(ceilingIndex(endTime), numRows - 1) of each chunk of the window, kept when ts >= windowStart && ts > timestamp; the value
// is valReader.asHistReader(endRowNum), the raw reader value (no counter correction).  Histogram.empty otherwise.
static void last_samples_hist(const Series& S, int64_t start, int64_t step, int64_t end, int64_t window, bool inclusive, std::vector<H::MutHist>& out) {
  const int T = (int)((end - start) / step) + 1;
  out.assign((size_t)T, H::MutHist());
  const int64_t winDur = inclusive ? window : window - 1;
  for (int k = 0; k < T; ++k) {
    const int64_t wEnd = start + (int64_t)k * step, wStart = wEnd - (winDur < 0 ? 0 : winDur);
    int64_t timestamp = -1;
    for (size_t c = 0; c < S.chunks.size(); ++c) {
      fo::Ptr info = S.chunks[c]->info.data();
      if (fo::csi::endTime(info) < wStart) continue;
      if (c > 0 && !(fo::csi::endTime(S.chunks[c - 1]->info.data()) < wEnd)) continue;
      fo::Ptr tv = S.chunks[c]->ts.data();
      const fo::LongReader tr = fo::LongReader::of(tv);
      const int32_t endRowNum = std::min(tr.ceilingIndex(tv, wEnd), fo::csi::numRows(info) - 1);
      if (endRowNum >= 0) {
        const int64_t ts = tr.apply(tv, endRowNum);
        if (ts >= wStart && ts > timestamp) { timestamp = ts; out[(size_t)k] = H::MutHist::from(H::HistReader(S.chunks[c]->hv.data()).apply(endRowNum)); }
      }
    }
  }
}

int main(int argc, char** argv) {
  cusim::rng_state() = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 0;
  std::mt19937_64 rng(4242);
  long checked = 0, qchecked = 0; int cases = 0;
  enum { CUSTOM, GEOMETRIC, OTEL };
  struct Cfg { int nb, scheme; std::vector<int> chunks; int jitter, reset_every; bool sect, cumulative; int fn; int64_t window, step; int nser; int inclusive; double qtl; };
  const std::vector<Cfg> cfgs = {
    {20, CUSTOM, {400, 80}, 0, 0, true, true, filo::FN_RATE, 300000, 15000, 5, 1, 0.99},                       // C4 shape, per series
    {8, GEOMETRIC, {70, 50, 40}, 3000, 37, true, true, filo::FN_INCREASE, 120000, 15000, 7, 1, 0.5},           // resets in chunks and at chunk starts, jitter
    {12, OTEL, {90, 70}, 0, 41, true, true, filo::FN_RATE, 300000, 15000, 6, 1, 0.75},                         // otel buckets: log-space quantile
    {33, CUSTOM, {60, 90}, 1500, 53, true, true, filo::FN_RATE, 450000, 47000, 4, 0, 1.0},                     // 5 NibblePack groups, exclusive start, q = 1
    {10, GEOMETRIC, {20, 20, 20, 20, 20, 20, 20, 20}, 800, 29, true, true, filo::FN_INCREASE, 90000, 13000, 5, 1, 0.0},  // 8 chunks, q = 0
    {16, CUSTOM, {100, 60}, 0, 31, true, true, filo::FN_LAST, 300000, 15000, 6, 1, 0.9},                       // last over SectDelta (raw after Drop sections)
    {24, OTEL, {50, 50, 30}, 1500, 19, true, true, filo::FN_LAST, 0, 20000, 5, 1, 0.3},                        // last, default lookback, jitter, otel
    {9, GEOMETRIC, {20, 20, 20, 20, 20, 20, 20, 20}, 2500, 0, true, true, filo::FN_LAST, 40000, 7000, 4, 0, -0.5},      // 8 chunks, short window (empty windows), q < 0
    {12, GEOMETRIC, {80, 40}, 1000, 0, false, false, filo::FN_LAST, 200000, 30000, 6, 1, 1.5},                 // last over simple (delta) vectors: first kernel, q > 1
    {12, CUSTOM, {80, 40}, 0, 0, false, false, filo::FN_SUM, 300000, 15000, 5, 1, 0.9},                        // sum_over_time on simple vectors: first kernel's stage
    {12, GEOMETRIC, {80, 40}, 2000, 0, false, false, filo::FN_RATE, 200000, 30000, 5, 1, 0.6},                 // delta-temporality rate: first kernel's stage
    {6, CUSTOM, {30, 30}, 0, 17, true, true, filo::FN_RATE, 120000, 15000, 70, 1, 0.95},                       // 70 series: two runs of 64 per CTA
    {8, CUSTOM, {60, 40}, 0, 23, true, true, filo::FN_LAST, 10000, 5000, 3, 1, 0.9},                           // last: windows whose only row sits on windowStart
    {8, GEOMETRIC, {60, 40}, 0, 0, false, true, filo::FN_LAST, 10000, 5000, 3, 0, 0.9},                        // ... exclusive start: that row is out
  };
  for (size_t ci = 0; ci < cfgs.size(); ++ci) {
    const Cfg& c = cfgs[ci];
    std::vector<double> les; for (int i = 0; i < c.nb - 1; ++i) les.push_back(2.0 * std::pow(3.0, i)); les.push_back(INFINITY);
    const H::Buckets b = c.scheme == OTEL ? H::Buckets::exponential(3, -5, c.nb - 1) : c.scheme == GEOMETRIC ? H::Buckets::geometric(2.0, 2.0, c.nb)
                                                                                                           : H::Buckets::custom(les.data(), c.nb);
    int rows = 0; for (int n : c.chunks) rows += n;
    const int64_t t0 = 1700000000000LL;
    std::vector<Series> SS((size_t)c.nser); std::vector<int64_t> rec_off((size_t)c.nser + 1, 0); uint32_t max_rec = 0;
    for (int s = 0; s < c.nser; ++s) { build_series(SS[(size_t)s], rng, b, rows, c.chunks, t0, 15000, c.jitter, c.reset_every, c.sect, c.cumulative);
                                       rec_off[(size_t)s + 1] = rec_off[(size_t)s] + (int64_t)SS[(size_t)s].record.size(); max_rec = std::max<uint32_t>(max_rec, (uint32_t)SS[(size_t)s].record.size()); }
    std::vector<uint64_t> backing((size_t)rec_off.back() / 8 + 64, 0); uint8_t* arena = reinterpret_cast<uint8_t*>(backing.data());
    for (int s = 0; s < c.nser; ++s) std::memcpy(arena + rec_off[(size_t)s], SS[(size_t)s].record.data(), SS[(size_t)s].record.size());
    const bool last = c.fn == filo::FN_LAST;
    filo::QueryParams q{};
    q.start = t0 - 30000; q.step = c.step; q.end = t0 + (int64_t)rows * 15000 + 45000;
    q.window = c.window > 0 ? c.window : 5 * 60 * 1000 + 1;                         // last: filo_query_hist's default lookback
    q.T = (int)((q.end - q.start) / q.step) + 1;
    q.fn = c.fn; q.cumulative = c.cumulative; q.inclusive = c.inclusive;
    const int T = q.T, nb = c.nb, S = c.nser;
    // oracle per series
    std::vector<std::vector<H::MutHist>> ref((size_t)S);
    for (int s = 0; s < S; ++s) {
      if (last) { last_samples_hist(SS[(size_t)s], q.start, q.step, q.end, q.window, c.inclusive != 0, ref[(size_t)s]); continue; }
      H::HistSeries hs; for (auto& ch : SS[(size_t)s].chunks) hs.infos.push_back(ch->info.data());
      H::periodicSamplesHist(hs, c.fn == filo::FN_SUM ? fo::FN_SUM_OVER_TIME : c.fn, c.cumulative, q.start, q.step, q.end, q.window, c.inclusive != 0, ref[(size_t)s]);
    }
    std::vector<double> tops((size_t)nb); for (int i = 0; i < nb; ++i) tops[(size_t)i] = b.bucketTop(i);
    const int expb = b.kind == H::Buckets::EXP ? 1 : 0;
    int n_empty = 0, n_full = 0;
    auto check_series = [&](const char* what, const std::vector<double>* ov, const std::vector<double>& oq) -> bool {
      for (int s = 0; s < S; ++s) for (int k = 0; k < T; ++k) {
        const H::MutHist& h = ref[(size_t)s][(size_t)k];
        if (ov) for (int i = 0; i < nb; ++i) {
          const double e = h.numBuckets() ? h.values[(size_t)i] : std::nan(""), a = (*ov)[((size_t)s * T + k) * nb + i];
          if (!same_bits(a, e)) { std::printf("FAIL cfg %zu %s s %d window %d bucket %d: %.17g vs %.17g\n", ci, what, s, k, i, a, e); return false; }
          ++checked;
        }
        const double eq = h.numBuckets() ? h.quantile(c.qtl) : std::nan(""), aq = oq[(size_t)s * T + k];
        if (!same_bits(aq, eq)) { std::printf("FAIL cfg %zu %s s %d window %d quantile %g: %.17g vs %.17g\n", ci, what, s, k, c.qtl, aq, eq); return false; }
        ++qchecked; (h.numBuckets() ? n_full : n_empty) += 1;
      }
      return true;
    };
    unsigned long long counters[2]; int derr[4];
    std::string ran;
    // ---- second kernel, per series: rate / increase over cumulative SectDelta, last over SectDelta
    if (c.sect && (last || (c.cumulative && (c.fn == filo::FN_RATE || c.fn == filo::FN_INCREASE)))) {
      const int grid = 2;
      const int64_t n_items = (S + filo::H2_RUN - 1) / filo::H2_RUN;          // runs of H2_RUN consecutive series (launch_hist_scan2_series)
      for (int mode = 0; mode < 2; ++mode) {                        // 0: bucket rows + quantile, 1: quantile only (window columns in the CTA's scratch)
        std::vector<double> ov(mode == 0 ? (size_t)S * T * nb : 0, -1.0), oq((size_t)S * T, -1.0), scr((size_t)grid * T * nb, -1.0);
        const filo::H2Series HS{mode == 0 ? ov.data() : nullptr, oq.data(), mode == 0 ? nullptr : scr.data(), tops.data(), c.qtl, expb};
        counters[0] = counters[1] = 0; std::memset(derr, 0, sizeof derr);
        if (last) cusim::launch(dim3(grid), dim3(filo::H2_THREADS), [&] { filo::hist_scan2_kernel<true, true>(arena, rec_off.data(), q, nb, rows, max_rec, nullptr, nullptr, n_items, nullptr, nullptr, counters, derr, HS, S); });
        else cusim::launch(dim3(grid), dim3(filo::H2_THREADS), [&] { filo::hist_scan2_kernel<true, false>(arena, rec_off.data(), q, nb, rows, max_rec, nullptr, nullptr, n_items, nullptr, nullptr, counters, derr, HS, S); });
        if (derr[0]) { std::printf("FAIL cfg %zu: v2 per-series device error %d\n", ci, derr[0]); return 1; }
        if (!check_series(mode == 0 ? "v2 per series" : "v2 quantile only", mode == 0 ? &ov : nullptr, oq)) return 1;
        if ((int64_t)counters[0] != (int64_t)S * rows) { std::printf("FAIL cfg %zu: v2 samples_scanned %llu\n", ci, counters[0]); return 1; }
      }
      ran += "v2 per series, ";
    }
    // ---- first kernel, per series: bucket rows + its quantile stage, and the quantile alone
    for (int mode = 0; mode < 2; ++mode) {
      std::vector<double> ov(mode == 0 ? (size_t)S * T * nb : 0, -1.0), oq((size_t)S * T, -1.0);
      counters[0] = counters[1] = 0; std::memset(derr, 0, sizeof derr);
      cusim::launch(dim3(3), dim3(filo::HIST_THREADS), [&] { filo::hist_scan_kernel(arena, rec_off.data(), S, q, nb, rows, max_rec, nullptr, nullptr, 0, 0, mode == 0 ? ov.data() : nullptr,
                                                                                    nullptr, nullptr, counters, derr, tops.data(), c.qtl, expb, oq.data()); }, 128 * 1024);
      if (derr[0]) { std::printf("FAIL cfg %zu: v1 per-series device error %d\n", ci, derr[0]); return 1; }
      if (!check_series(mode == 0 ? "v1 per series" : "v1 quantile only", mode == 0 ? &ov : nullptr, oq)) return 1;
      if ((int64_t)counters[0] != (int64_t)S * rows) { std::printf("FAIL cfg %zu: v1 samples_scanned %llu\n", ci, counters[0]); return 1; }
    }
    ran += "v1 per series";
    // ---- fused last (+ quantile): items of 2 series in a shuffled order, folded as HistSumRowAggregator does at both levels
    if (last) {
      std::vector<int32_t> order((size_t)S); for (int s = 0; s < S; ++s) order[(size_t)s] = s; std::shuffle(order.begin(), order.end(), rng);
      std::vector<int64_t> item_begin; for (int64_t p = 0; p < S; p += 2) item_begin.push_back(p); item_begin.push_back(S);
      const int64_t n_items = (int64_t)item_begin.size() - 1; const int64_t gis[2] = {0, n_items};
      std::vector<double> exp_vals((size_t)T * nb, 0.0), exp_q((size_t)T, 0.0); std::vector<char> exp_any((size_t)T, 0);
      for (int k = 0; k < T; ++k) {
        H::MutHist tot; bool any = false;
        for (int64_t it = 0; it < n_items; ++it) {
          H::MutHist part; bool iany = false;
          for (int64_t p = item_begin[(size_t)it]; p < item_begin[(size_t)it + 1]; ++p) { const H::MutHist& h = ref[(size_t)order[(size_t)p]][(size_t)k]; if (h.numBuckets()) { if (!iany) { part = h; iany = true; } else part.add(h); } }
          if (iany) { if (!any) { tot = part; any = true; } else tot.add(part); }
        }
        exp_any[(size_t)k] = any;
        if (any) { exp_q[(size_t)k] = tot.quantile(c.qtl); for (int i = 0; i < nb; ++i) exp_vals[(size_t)k * nb + i] = tot.values[(size_t)i]; }
      }
      auto check_fused = [&](const char* what, const std::vector<double>& ov, const std::vector<double>& oq) -> bool {
        for (int k = 0; k < T; ++k) {
          for (int i = 0; i < nb; ++i) { const double e = exp_any[(size_t)k] ? exp_vals[(size_t)k * nb + i] : std::nan(""); if (!same_bits(ov[(size_t)k * nb + i], e)) { std::printf("FAIL cfg %zu %s window %d bucket %d: %.17g vs %.17g\n", ci, what, k, i, ov[(size_t)k * nb + i], e); return false; } ++checked; }
          const double eq = exp_any[(size_t)k] ? exp_q[(size_t)k] : std::nan("");
          if (!same_bits(oq[(size_t)k], eq)) { std::printf("FAIL cfg %zu %s window %d quantile: %.17g vs %.17g\n", ci, what, k, oq[(size_t)k], eq); return false; }
          ++qchecked;
        }
        return true;
      };
      if (c.sect) {
        std::vector<double> pval((size_t)n_items * T * nb, -1.0), ov((size_t)T * nb, -1.0), oq((size_t)T, -1.0); std::vector<uint8_t> pany((size_t)n_items * T + 16, 7);
        std::memset(derr, 0, sizeof derr);
        cusim::launch(dim3(2), dim3(filo::H2_THREADS), [&] { filo::hist_scan2_kernel<false, true>(arena, rec_off.data(), q, nb, rows, max_rec, order.data(), item_begin.data(), n_items, pval.data(), pany.data(), counters, derr); });
        if (derr[0]) { std::printf("FAIL cfg %zu: v2 fused last device error %d\n", ci, derr[0]); return 1; }
        cusim::launch(dim3((unsigned)((T + 127) / 128)), dim3(128), [&] { filo::hist_merge2_kernel(pval.data(), pany.data(), gis, 1, T, nb, expb, tops.data(), c.qtl, ov.data(), oq.data()); });
        if (!check_fused("v2 fused last", ov, oq)) return 1;
        ran += ", v2 fused last";
      }
      std::vector<double> pval((size_t)n_items * T * nb, -1.0), ov((size_t)T * nb, -1.0), oq((size_t)T, -1.0); std::vector<uint8_t> pany((size_t)n_items * T + 16, 7);
      std::memset(derr, 0, sizeof derr);
      cusim::launch(dim3(2), dim3(filo::HIST_THREADS), [&] { filo::hist_scan_kernel(arena, rec_off.data(), S, q, nb, rows, max_rec, order.data(), item_begin.data(), n_items, 1, nullptr, pval.data(), pany.data(), counters, derr); }, 128 * 1024);
      if (derr[0]) { std::printf("FAIL cfg %zu: v1 fused last device error %d\n", ci, derr[0]); return 1; }
      cusim::launch(dim3((unsigned)((T + 127) / 128)), dim3(128), [&] { filo::hist_merge_kernel(pval.data(), pany.data(), gis, 1, T, nb, expb, tops.data(), c.qtl, ov.data(), oq.data()); });
      if (!check_fused("v1 fused last", ov, oq)) return 1;
      ran += ", v1 fused last";
    }
    if (n_empty == 0 && c.window > 0 && c.window < 60000) { std::printf("FAIL cfg %zu: no empty window in a short-window case\n", ci); return 1; }
    if (n_full == 0) { std::printf("FAIL cfg %zu: no histogram\n", ci); return 1; }
    std::printf("cfg %zu ok (%s)\n", ci, ran.c_str());
    ++cases;
  }
  std::printf("OK %d cases, %ld bucket values and %ld quantiles bit-exact\n", cases, checked, qchecked);
  return 0;
}
