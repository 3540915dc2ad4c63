// The cross-GPU histogram sum on the CPU (test infrastructure; built and run by tests/test_hist_parts_emul.py): W tables cut from one
// series set, each one's SUM output produced by hist_scan2_kernel + hist_merge2_kernel (hist_kernels2.cu) and by hist_scan_kernel +
// hist_merge_kernel (hist_kernels.cu, through tests/cpp/make_cusim_src.py) on the cusim emulator, then folded by hist_merge_parts_kernel.
// Checked bit for bit, quantile bits included, against the oracle: periodicSamplesHist per series (oracle/filo_hist.hpp), folded with
// MutHist::add in (part, item, series) order -- this driver sets the item boundaries, so the reduction tree is known.  It also pins the
// invariant the merge relies on: a SUM output cell is NaN in every bucket exactly where no item of its group set pany, and has no NaN
// bucket anywhere else.
//     hist_parts_emul [schedule seed]
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

// cumulative bucket counts with resets inside chunks and at chunk starts, optional timestamp jitter, encoded by the oracle's appenders
// into one device record (the builder of tests/cpp/hist_series_emul.cpp, with the series' first timestamp as an argument)
static void build_series(Series& S, std::mt19937_64& rng, const H::Buckets& b, int rows, const std::vector<int>& chunk_rows, int64_t t0, int step_ms, int jitter,
                         int reset_every) {
  const int nb = b.n;
  std::vector<int64_t> ts((size_t)rows), vals((size_t)rows * nb), cur((size_t)nb, 0);
  std::vector<char> boundary((size_t)rows + 1, 0);
  { int r0 = 0; for (int n : chunk_rows) { r0 += n; if (r0 < rows) boundary[(size_t)r0] = 1; } }
  for (int r = 0; r < rows; ++r) {
    ts[(size_t)r] = t0 + (int64_t)r * step_ms + (jitter ? (int64_t)(rng() % (uint64_t)(2 * jitter + 1)) - jitter : 0);
    if (reset_every && r > 0 && (rng() % (uint64_t)reset_every == 0 || (boundary[(size_t)r] && rng() % 2))) std::fill(cur.begin(), cur.end(), 0);
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
    H::HistAppender app(true, 60000);
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

// one table: its series (global ids), grouped and cut into work items of at most `seg` series of one group, as the loader does
struct Part {
  std::vector<int> sids;                                         // global series ids, table order
  std::vector<int64_t> rec_off; std::vector<uint64_t> backing; uint32_t max_rec = 0;
  std::vector<int32_t> order; std::vector<int64_t> item_begin, gis;
};
static void build_part(Part& P, const std::vector<Series>& SS, const std::vector<int>& gid, int G, int seg) {
  const int n = (int)P.sids.size();
  P.rec_off.assign((size_t)n + 1, 0);
  for (int s = 0; s < n; ++s) { const size_t sz = SS[(size_t)P.sids[(size_t)s]].record.size(); P.rec_off[(size_t)s + 1] = P.rec_off[(size_t)s] + (int64_t)sz; P.max_rec = std::max<uint32_t>(P.max_rec, (uint32_t)sz); }
  P.backing.assign((size_t)P.rec_off.back() / 8 + 64, 0);
  uint8_t* arena = reinterpret_cast<uint8_t*>(P.backing.data());
  for (int s = 0; s < n; ++s) std::memcpy(arena + P.rec_off[(size_t)s], SS[(size_t)P.sids[(size_t)s]].record.data(), SS[(size_t)P.sids[(size_t)s]].record.size());
  P.order.clear(); P.item_begin.clear(); P.gis.assign((size_t)G + 1, 0);
  for (int g = 0; g < G; ++g) {
    P.gis[(size_t)g] = (int64_t)P.item_begin.size();
    int in_item = 0;
    for (int s = 0; s < n; ++s) {
      if (gid[(size_t)P.sids[(size_t)s]] != g) continue;
      if (in_item == 0) P.item_begin.push_back((int64_t)P.order.size());
      P.order.push_back(s); in_item = (in_item + 1) % seg;
    }
  }
  P.gis[(size_t)G] = (int64_t)P.item_begin.size();
  P.item_begin.push_back((int64_t)P.order.size());
}

// LastSampleChunkedFunction.addChunks + LastSampleChunkedFunctionH.updateValue (RangeFunction.scala:599-614, 630-640; the restatement of
// tests/cpp/hist_series_emul.cpp): per window the row min(ceilingIndex(windowEnd), numRows - 1) of each chunk of the window's chunk set,
// kept when its timestamp is >= windowStart and > the one kept so far; the raw reader value.  Histogram.empty otherwise.
static void last_samples_hist(const Series& S, int64_t start, int64_t step, int64_t end, int64_t window, std::vector<H::MutHist>& out) {
  const int T = (int)((end - start) / step) + 1;
  out.assign((size_t)T, H::MutHist());
  for (int k = 0; k < T; ++k) {
    const int64_t wEnd = start + (int64_t)k * step, wStart = wEnd - window;
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

// HistSumRowAggregator.reduceAggregate: the first non-empty histogram is copied, every further one goes through MutableHistogram.add
static void fold(H::MutHist& acc, const H::MutHist& h) { if (!h.numBuckets()) return; if (!acc.numBuckets()) acc = h; else acc.add(h); }

int main(int argc, char** argv) {
  cusim::rng_state() = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 0;
  std::mt19937_64 rng(777);
  long checked = 0, qchecked = 0, nonmono_copied = 0, cells_partial = 0; int cases = 0, cases_rank0_only = 0;
  enum { CUSTOM, GEOMETRIC, OTEL };
  // split: 0 contiguous series ranges, 1 interleaved (series s on table s % W)
  struct Cfg { int nb, scheme, W, S, G, seg, split; int fn; int64_t step; double qtl; };
  const std::vector<Cfg> cfgs = {
    {20, CUSTOM, 1, 10, 4, 2, 0, filo::FN_RATE, 60000, 0.99},           // one part: the merge is the copy of the part
    {20, CUSTOM, 2, 14, 4, 2, 0, filo::FN_RATE, 60000, 0.5},
    {12, GEOMETRIC, 3, 15, 5, 3, 1, filo::FN_INCREASE, 45000, 0.9},
    {8, OTEL, 8, 20, 4, 2, 1, filo::FN_RATE, 60000, 0.75},            // otel buckets: log2 interpolation; some ranks hold 2 series
    {20, OTEL, 8, 12, 5, 1, 0, filo::FN_RATE, 60000, 0.3},            // ranks 6 and 7 are empty tables
    {1, CUSTOM, 2, 8, 3, 2, 1, filo::FN_RATE, 60000, 0.5},            // nb = 1: the quantile is NaN
    {64, GEOMETRIC, 3, 9, 3, 2, 0, filo::FN_INCREASE, 90000, 0.95},   // nb = 64: 8 NibblePack groups
    {10, CUSTOM, 3, 9, 3, 2, 1, filo::FN_RATE, 5000, 0.6},            // T > 128 windows: the merge spans several thread blocks per group
    {6, GEOMETRIC, 2, 8, 3, 2, 0, filo::FN_SUM, 60000, NAN},          // quantile NaN: values only (first kernel only: sum_over_time)
    {6, CUSTOM, 3, 9, 3, 2, 1, filo::FN_RATE, 60000, -0.5},           // q < 0
    {6, OTEL, 3, 9, 3, 2, 0, filo::FN_RATE, 60000, 1.5},              // q > 1
    {16, CUSTOM, 3, 12, 4, 2, 1, filo::FN_LAST, 60000, 0.9},          // last: raw rows of the window's latest sample
    {8, OTEL, 8, 14, 3, 2, 0, filo::FN_LAST, 45000, 0.5},
  };
  const int ROWS = 120, STEP = 15000;
  const int64_t t0 = 1700000000000LL;
  for (size_t ci = 0; ci < cfgs.size(); ++ci) {
    const Cfg& c = cfgs[ci];
    std::vector<double> les; for (int i = 0; i < c.nb - 1; ++i) les.push_back(2.0 * std::pow(3.0, i)); les.push_back(INFINITY);
    const H::Buckets b = c.scheme == OTEL ? H::Buckets::exponential(3, -5, c.nb - 1) : c.scheme == GEOMETRIC ? H::Buckets::geometric(2.0, 2.0, c.nb)
                                                                                                           : H::Buckets::custom(les.data(), c.nb);
    const int nb = c.nb, S = c.S, G = c.G, W = c.W;
    // series start at three offsets, so that a window can be empty on one rank and not on another
    std::vector<Series> SS((size_t)S);
    for (int s = 0; s < S; ++s) build_series(SS[(size_t)s], rng, b, ROWS, {70, 50}, t0 + (int64_t)(s % 3) * 600000, STEP, (s % 4 == 1) ? 2000 : 0, 29);
    // parts and groups: group G - 1 has no series anywhere; group 0 has none on rank 0 (W > 1); the others are spread
    std::vector<Part> parts((size_t)W);
    const int per = (S + W - 1) / W;                               // contiguous: shard.series_range_of_rank
    for (int s = 0; s < S; ++s) parts[(size_t)(c.split == 0 ? s / per : s % W)].sids.push_back(s);
    std::vector<int> gid((size_t)S);
    for (int r = 0; r < W; ++r)
      for (size_t j = 0; j < parts[(size_t)r].sids.size(); ++j) {
        const int s = parts[(size_t)r].sids[j];
        gid[(size_t)s] = G == 1 ? 0 : (W > 1 && r == 0) ? 1 + (int)(j % (size_t)std::max(1, G - 2)) : (int)((j + (size_t)r) % (size_t)std::max(1, G - 1));
      }
    for (auto& P : parts) build_part(P, SS, gid, G, c.seg);
    filo::QueryParams q{};
    q.start = t0 - 30000; q.step = c.step; q.end = t0 + (int64_t)ROWS * STEP + 1200000 + 45000; q.window = 300000;
    q.T = (int)((q.end - q.start) / q.step) + 1;
    q.fn = c.fn; q.cumulative = 1; q.inclusive = 1;
    const int T = q.T;
    if (c.step == 5000 && T <= 128) { std::printf("FAIL cfg %zu: T = %d does not span several blocks\n", ci, T); return 1; }
    // oracle: per series, then folded in (part, item, series) order
    std::vector<std::vector<H::MutHist>> ref((size_t)S);
    for (int s = 0; s < S; ++s) {
      if (c.fn == filo::FN_LAST) { last_samples_hist(SS[(size_t)s], q.start, q.step, q.end, q.window, ref[(size_t)s]); continue; }
      H::HistSeries hs; for (auto& ch : SS[(size_t)s].chunks) hs.infos.push_back(ch->info.data());
      H::periodicSamplesHist(hs, c.fn == filo::FN_SUM ? fo::FN_SUM_OVER_TIME : c.fn, true, q.start, q.step, q.end, q.window, true, ref[(size_t)s]);
    }
    std::vector<H::MutHist> part_exp((size_t)W * G * T), tot_exp((size_t)G * T);
    for (int r = 0; r < W; ++r) {
      const Part& P = parts[(size_t)r];
      for (int g = 0; g < G; ++g)
        for (int k = 0; k < T; ++k) {
          H::MutHist& pe = part_exp[((size_t)r * G + g) * T + k];
          for (int64_t it = P.gis[(size_t)g]; it < P.gis[(size_t)g + 1]; ++it) {
            H::MutHist item;
            for (int64_t p = P.item_begin[(size_t)it]; p < P.item_begin[(size_t)it + 1]; ++p) fold(item, ref[(size_t)P.sids[(size_t)P.order[(size_t)p]]][(size_t)k]);
            fold(pe, item);
          }
          fold(tot_exp[(size_t)g * T + k], pe);
        }
    }
    std::vector<double> tops((size_t)nb); for (int i = 0; i < nb; ++i) tops[(size_t)i] = b.bucketTop(i);
    const int expb = b.kind == H::Buckets::EXP ? 1 : 0;
    const double NaNv = std::nan("");
    const bool v2_ok = c.fn == filo::FN_RATE || c.fn == filo::FN_INCREASE || c.fn == filo::FN_LAST;       // SectDelta vectors throughout
    unsigned long long counters[2]; int derr[4];
    std::string ran;
    for (int kernel = v2_ok ? 2 : 1; kernel >= 1; --kernel) {
      // ---- each table's SUM output, as filo_query_hist_device writes it
      std::vector<double> d_parts((size_t)W * G * T * nb, -1.0);
      std::vector<char> pany_any((size_t)W * G * T, 0);
      for (int r = 0; r < W; ++r) {
        Part& P = parts[(size_t)r];
        const int64_t n_items = (int64_t)P.item_begin.size() - 1;
        const uint8_t* arena = reinterpret_cast<const uint8_t*>(P.backing.data());
        std::vector<double> pval((size_t)std::max<int64_t>(n_items, 1) * T * nb, -1.0); std::vector<uint8_t> pany((size_t)std::max<int64_t>(n_items, 1) * T + 16, 7);
        double* out = d_parts.data() + (size_t)r * G * T * nb;
        counters[0] = counters[1] = 0; std::memset(derr, 0, sizeof derr);
        if (n_items > 0) {
          if (kernel == 2 && c.fn == filo::FN_LAST)                      // as launch_hist_scan2 selects the instantiation
            cusim::launch(dim3(2), dim3(filo::H2_THREADS), [&] { filo::hist_scan2_kernel<false, true>(arena, P.rec_off.data(), q, nb, ROWS, P.max_rec, P.order.data(), P.item_begin.data(), n_items, pval.data(), pany.data(), counters, derr); });
          else if (kernel == 2)
            cusim::launch(dim3(2), dim3(filo::H2_THREADS), [&] { filo::hist_scan2_kernel<false, false>(arena, P.rec_off.data(), q, nb, ROWS, P.max_rec, P.order.data(), P.item_begin.data(), n_items, pval.data(), pany.data(), counters, derr); });
          else
            cusim::launch(dim3(2), dim3(filo::HIST_THREADS), [&] { filo::hist_scan_kernel(arena, P.rec_off.data(), (int64_t)P.sids.size(), q, nb, ROWS, P.max_rec, P.order.data(), P.item_begin.data(), n_items, 1, nullptr, pval.data(), pany.data(), counters, derr); }, 128 * 1024);
          if (derr[0]) { std::printf("FAIL cfg %zu: kernel %d part %d device error %d\n", ci, kernel, r, derr[0]); return 1; }
        }
        const unsigned grid = (unsigned)(((int64_t)G * T + 127) / 128);
        if (kernel == 2) cusim::launch(dim3(grid), dim3(128), [&] { filo::hist_merge2_kernel(pval.data(), pany.data(), P.gis.data(), G, T, nb, expb, tops.data(), NaNv, out, nullptr); });
        else cusim::launch(dim3(grid), dim3(128), [&] { filo::hist_merge_kernel(pval.data(), pany.data(), P.gis.data(), G, T, nb, expb, tops.data(), NaNv, out, nullptr); });
        for (int g = 0; g < G; ++g)
          for (int64_t it = P.gis[(size_t)g]; it < P.gis[(size_t)g + 1]; ++it)
            for (int k = 0; k < T; ++k) if (pany[(size_t)it * T + k]) pany_any[((size_t)r * G + g) * T + k] = 1;
      }
      // ---- the parts: bit-exact against the oracle, and the invariant
      for (size_t cell = 0; cell < (size_t)W * G * T; ++cell) {
        const H::MutHist& h = part_exp[cell];
        const double* row = d_parts.data() + cell * nb;
        int nan_buckets = 0; bool mono = true;
        for (int i = 0; i < nb; ++i) {
          nan_buckets += row[i] != row[i];
          if (i > 0 && row[i] < row[i - 1]) mono = false;
          const double e = h.numBuckets() ? h.values[(size_t)i] : NaNv;
          if (!same_bits(row[i], e)) { std::printf("FAIL cfg %zu kernel %d part cell %zu bucket %d: %.17g vs %.17g\n", ci, kernel, cell, i, row[i], e); return 1; }
          ++checked;
        }
        const bool any = pany_any[cell] != 0;
        if (any ? nan_buckets != 0 : nan_buckets != nb) { std::printf("FAIL cfg %zu kernel %d part cell %zu: %d NaN buckets, pany %d\n", ci, kernel, cell, nan_buckets, (int)any); return 1; }
        if (any && !mono) ++nonmono_copied;
        cells_partial += any;
      }
      // ---- the rank-order fold
      std::vector<double> ov((size_t)G * T * nb, -1.0), oq((size_t)G * T, -1.0);
      const bool with_q = c.qtl == c.qtl;
      cusim::launch(dim3((unsigned)(((int64_t)G * T + 127) / 128)), dim3(128), [&] {
        filo::hist_merge_parts_kernel(d_parts.data(), W, (int64_t)G * T, nb, expb, tops.data(), c.qtl, ov.data(), with_q ? oq.data() : nullptr); });
      for (int g = 0; g < G; ++g)
        for (int k = 0; k < T; ++k) {
          const size_t cell = (size_t)g * T + k;
          const H::MutHist& h = tot_exp[cell];
          bool any = false; for (int r = 0; r < W; ++r) any |= pany_any[((size_t)r * G + g) * T + k] != 0;
          int nan_buckets = 0;
          for (int i = 0; i < nb; ++i) {
            const double e = h.numBuckets() ? h.values[(size_t)i] : NaNv, a = ov[cell * nb + i];
            nan_buckets += a != a;
            if (!same_bits(a, e)) { std::printf("FAIL cfg %zu kernel %d merge g %d window %d bucket %d: %.17g vs %.17g\n", ci, kernel, g, k, i, a, e); return 1; }
            ++checked;
          }
          if (any ? nan_buckets != 0 : nan_buckets != nb) { std::printf("FAIL cfg %zu kernel %d merge g %d window %d: %d NaN buckets, pany %d\n", ci, kernel, g, k, nan_buckets, (int)any); return 1; }
          const double eq = with_q ? (h.numBuckets() ? h.quantile(c.qtl) : NaNv) : -1.0;
          if (!same_bits(oq[cell], eq)) { std::printf("FAIL cfg %zu kernel %d merge g %d window %d quantile: %.17g vs %.17g\n", ci, kernel, g, k, oq[cell], eq); return 1; }
          ++qchecked;
        }
      // the coverage each case is there for
      int empty_g_every = 0, empty_g_rank0 = 0, empty_some = 0, full = 0;
      for (int g = 0; g < G; ++g) {
        bool any_rank = false, rank0 = false; int ranks = 0;
        for (int r = 0; r < W; ++r) { bool a = false; for (int k = 0; k < T; ++k) a |= pany_any[((size_t)r * G + g) * T + k] != 0; ranks += a; any_rank |= a; if (r == 0) rank0 = a; }
        empty_g_every += !any_rank; empty_g_rank0 += (W > 1 && !rank0 && ranks == W - 1); empty_some += (ranks > 0 && ranks < W);
        for (int k = 0; k < T; ++k) full += tot_exp[(size_t)g * T + k].numBuckets() > 0;
      }
      if (!empty_g_every || !full || (W > 1 && G > 2 && !empty_some)) { std::printf("FAIL cfg %zu: coverage (empty everywhere %d, empty on some ranks %d, full cells %d)\n", ci, empty_g_every, empty_some, full); return 1; }
      ran += kernel == 2 ? "second kernel " : "first kernel ";
      if (empty_g_rank0) { ran += "(a group empty on rank 0 only) "; ++cases_rank0_only; }
    }
    std::printf("cfg %zu ok: W %d, G %d, T %d, nb %d: %s\n", ci, W, G, T, nb, ran.c_str());
    ++cases;
  }
  if (!cases_rank0_only) { std::printf("FAIL: no case with a group empty on rank 0 only\n"); return 1; }
  // ---- a non-monotonic partial is copied as it is and made monotonic only by a second add; cells empty on some or every rank
  {
    const int W = 3, nb = 3, T = 4;
    const double N = std::nan(""), les[3] = {1.0, 10.0, INFINITY};
    const double P[W][T][nb] = {{{5, 3, 7}, {N, N, N}, {N, N, N}, {0, 2, 1}},
                                {{N, N, N}, {5, 3, 7}, {N, N, N}, {N, N, N}},
                                {{N, N, N}, {1, 1, -4}, {N, N, N}, {1, 0, 0}}};
    const H::Buckets b = H::Buckets::custom(les, nb);
    std::vector<double> ov((size_t)T * nb, -1.0), oq((size_t)T, -1.0);
    cusim::launch(dim3(1), dim3(128), [&] { filo::hist_merge_parts_kernel(&P[0][0][0], W, T, nb, 0, les, 0.5, ov.data(), oq.data()); });
    const double want[T][nb] = {{5, 3, 7}, {6, 6, 6}, {N, N, N}, {1, 2, 2}};
    for (int k = 0; k < T; ++k) {
      H::MutHist acc;
      for (int r = 0; r < W; ++r) if (P[r][k][0] == P[r][k][0]) { H::MutHist h; h.buckets = b; h.values.assign(P[r][k], P[r][k] + nb); fold(acc, h); }
      for (int i = 0; i < nb; ++i) {
        const double e = acc.numBuckets() ? acc.values[(size_t)i] : N;
        if (!same_bits(ov[(size_t)k * nb + i], e) || !same_bits(e, want[k][i])) { std::printf("FAIL hand-made window %d bucket %d: %.17g vs %.17g\n", k, i, ov[(size_t)k * nb + i], e); return 1; }
      }
      const double eq = acc.numBuckets() ? acc.quantile(0.5) : N;
      if (!same_bits(oq[(size_t)k], eq)) { std::printf("FAIL hand-made window %d quantile: %.17g vs %.17g\n", k, oq[(size_t)k], eq); return 1; }
    }
    ++cases;
  }
  std::printf("OK %d cases, %ld bucket values and %ld quantiles bit-exact; %ld non-empty part cells, %ld of them non-monotonic\n", cases, checked, qchecked,
              cells_partial, nonmono_copied);
  return 0;
}
