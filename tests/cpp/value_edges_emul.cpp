// The scan kernels at value edges, compiled for the host on the cusim SIMT emulator.  Test infrastructure: built and run by
// tests/test_value_edges.py.  The series builders and launch helpers are tile_emul.cpp's.
//   1. Fused min / max over signed-zero gauge tables: the v4 counter kernel (delta is the counter class even on a gauge), the v2
//      aggregate kernel (last, min_over_time), then merge_partials_kernel over more than 8 items of one group.  Every item's partial
//      row is the oracle's aggregate() over the item's series; the merged row is aggregate() over the series in the order
//      0, 8, 16, ..., 1, 9, ... of the items (the rule keeps the later of two equal values, so the 8-lane tree equals that fold).
//   2. The v4 SUM kernel over one bound value per series: it declines 2^513, nextafter(2^-511, 0), +-0, subnormals, DBL_MAX and
//      +-Inf, admits nextafter(2^513, 0) and 2^-511 (wp_decode's 2^-511 <= |v| < 2^513); every result is bit-exact after the v2 pass.
//   value_edges_emul [seed]     seed 0 = round-robin schedule, otherwise a pseudo-random fiber schedule
#define main tile_emul_main
#include "tile_emul.cpp"
#undef main
#include <cfloat>
#include <set>

static const int64_t kT0 = 1700000000000LL;
static const int kStep = 15000;

struct Table {
  std::vector<SeriesData> SS; std::vector<int64_t> rec_off; std::vector<uint64_t> backing; uint8_t* arena = nullptr; uint32_t max_rec = 0;
  V2Shape sh{0, 0, 0, false, false};
};
static void finish_table(Table& tb, int rows, int nchunks) {
  tb.rec_off.assign(tb.SS.size() + 1, 0);
  for (size_t s = 0; s < tb.SS.size(); ++s) tb.rec_off[s + 1] = tb.rec_off[s] + (int64_t)tb.SS[s].record.size();
  tb.backing.assign((size_t)tb.rec_off.back() / 8 + 64, 0);
  tb.arena = reinterpret_cast<uint8_t*>(tb.backing.data());
  for (size_t s = 0; s < tb.SS.size(); ++s) {
    std::memcpy(tb.arena + tb.rec_off[s], tb.SS[s].record.data(), tb.SS[s].record.size());
    tb.max_rec = std::max<uint32_t>(tb.max_rec, (uint32_t)tb.SS[s].record.size());
  }
  tb.sh = V2Shape{tb.max_rec, rows, nchunks, false, false};
  for (auto& S : tb.SS) { filo::RecordHeader h; std::memcpy(&h, S.record.data(), sizeof h); tb.sh.any_nonconst_ts |= !(h.flags & filo::REC_ALL_TS_CONST); tb.sh.any_drop |= (h.flags & filo::REC_ANY_DROP) != 0; }
}
static std::vector<double> oracle_rows(const Table& tb, const filo::QueryParams& q, int64_t* samples) {
  std::vector<double> ref(tb.SS.size() * (size_t)q.T);
  for (size_t s = 0; s < tb.SS.size(); ++s) {
    fo::Series os; for (auto& ch : tb.SS[s].chunks) os.infos.push_back(ch->info.data());
    fo::QueryStats st;
    fo::periodicSamples(os, oracle_fn(q.fn), q.cumulative != 0, q.start, q.step, q.end, q.window, fo::QueryConfig{true}, ref.data() + s * q.T, &st, 0, 0);
    if (samples) *samples += st.samplesScanned;
  }
  return ref;
}
static bool row_same(const double* a, const double* b, int T, int* at) {
  for (int k = 0; k < T; ++k) if (!same_bits(a[k], b[k])) { *at = k; return false; }
  return true;
}

// ---------------------------------------------------------------------------------------------------- 1. signed zeros, fused min / max
static int signed_zero_case(std::mt19937_64& rng, int fn, bool xor_enc, int nser, int per_item, long& checked, long& ties) {
  const std::vector<int> chunks = {400, 80};
  const int rows = 480;
  const double pal[4] = {0.0, -0.0, 1.0, -1.0};
  Table tb; tb.SS.resize((size_t)nser);
  std::vector<int64_t> ts((size_t)rows); for (int r = 0; r < rows; ++r) ts[(size_t)r] = kT0 + (int64_t)r * kStep;
  for (int s = 0; s < nser; ++s) {
    std::vector<double> v((size_t)rows);
    const int kind = s % 6;           // palettes {+0, -0}, {+0, -0, 1}, {+0, -0, -1}, all four; then all +0.0, all -0.0
    for (int r = 0; r < rows; r += 12) {
      double x;
      if (kind == 4) x = 0.0; else if (kind == 5) x = -0.0;
      else { const int np = kind == 3 ? 4 : kind == 0 ? 2 : 3; const int i = (int)(rng() % (uint64_t)np); x = (kind == 2 && i == 2) ? -1.0 : pal[i]; }
      for (int j = 0; j < 12; ++j) v[(size_t)(r + j)] = x;
    }
    build_series_from(tb.SS[(size_t)s], rng, ts, v, chunks, 0, xor_enc, 0);
  }
  finish_table(tb, rows, (int)chunks.size());
  filo::QueryParams q{};
  q.start = kT0 + 300000; q.step = kStep; q.end = kT0 + (int64_t)(rows - 1) * kStep; q.window = 300000;
  q.T = (int)((q.end - q.start) / q.step) + 1; q.fn = fn; q.cumulative = 0; q.inclusive = 1;
  int64_t exp_rows = 0;
  const std::vector<double> ref = oracle_rows(tb, q, &exp_rows);
  std::vector<int32_t> order((size_t)nser); for (int s = 0; s < nser; ++s) order[(size_t)s] = s;
  std::shuffle(order.begin(), order.end(), rng);
  std::vector<int64_t> item_begin; for (int64_t p = 0; p < nser; p += per_item) item_begin.push_back(p); item_begin.push_back(nser);
  const int64_t n_items = (int64_t)item_begin.size() - 1;
  const uint32_t wrows = (uint32_t)(q.window / q.step) + 1;
  const filo::TileSmem L = filo::tile_layout(tb.max_rec, (uint32_t)rows, (uint32_t)q.T, 2 * wrows + 16);
  for (int op : {filo::AGG_MIN, filo::AGG_MAX}) {
    std::vector<double> pval((size_t)n_items * q.T, -777.0); std::vector<uint32_t> pcnt((size_t)n_items * q.T, 12345u);
    std::vector<int64_t> flist((size_t)n_items + 8, -1); unsigned long long fcount = 0, counters[2] = {0, 0}; int derr[4] = {0, 0, 0, 0};
    Launch A{tb.arena, tb.rec_off.data(), nser, q, nullptr, L, 2, flist.data(), &fcount, counters, derr, order.data(), item_begin.data(), n_items, op, pval.data(), pcnt.data()};
    const char* kernel = "v2 aggregate";
    if (filo::fn_class_of(q.fn, q.cumulative) == filo::CLASS_COUNTER) {
      kernel = "v4 counter";
      filo::WpCtrSmem W = filo::wp_ctr_layout(tb.max_rec, (uint32_t)rows, (uint32_t)chunks.size(), (uint32_t)q.T, true, false);
      W.warps = 3; W.tab = W.per_warp * W.warps;
      if ((size_t)W.tab + 4096 > sizeof(filo::smem)) { std::printf("FAIL: wp ctr layout %u bytes per warp\n", W.per_warp); return 1; }
      cusim::launch(dim3((unsigned)A.grid), dim3(W.warps * 32), [&] {
        filo::scan_wp_ctr_kernel<filo::FN_DELTA, true, 16, false>(A.arena, A.rec_off, A.S, A.q, nullptr, W, A.flist, A.fcount, A.counters, A.derr, A.order, A.item_begin, A.n_items, A.agg_op, A.pval, A.pcnt);
      });
      if (derr[0]) { std::printf("FAIL signed zeros fn %d: device error %d (v4 counter kernel)\n", fn, derr[0]); return 1; }
      if (fcount) run_agg_v2(A, tb.sh, flist.data(), &fcount);
    } else run_agg_v2(A, tb.sh, nullptr, nullptr);
    if (derr[0]) { std::printf("FAIL signed zeros fn %d: device error %d\n", fn, derr[0]); return 1; }
    if ((int64_t)counters[0] != exp_rows) { std::printf("FAIL signed zeros fn %d: samples_scanned %llu vs %lld\n", fn, counters[0], (long long)exp_rows); return 1; }
    // every item's partial row: the oracle's aggregate() over the item's series in item order
    for (int64_t it = 0; it < n_items; ++it) {
      std::vector<const double*> rs;
      for (int64_t p = item_begin[(size_t)it]; p < item_begin[(size_t)it + 1]; ++p) rs.push_back(ref.data() + (size_t)order[(size_t)p] * q.T);
      const fo::AggResult e = fo::aggregate((fo::AggrOp)op, 0, rs, std::vector<int32_t>(rs.size(), 0), 1, q.T);
      int at = 0;
      if (!row_same(pval.data() + (size_t)it * q.T, e.values.data(), q.T, &at)) {
        std::printf("FAIL signed zeros fn %d op %d (%s kernel) item %lld window %d: %.17g vs %.17g\n", fn, op, kernel, (long long)it, at, pval[(size_t)it * q.T + at], e.values[(size_t)at]);
        return 1;
      }
      checked += q.T;
    }
    // merge_partials_kernel, one group of n_items > 8 items: aggregate() over the series in the order of the items 0, 8, 16, ..., 1, 9, ...
    const int64_t gis[2] = {0, n_items};
    std::vector<double> mv((size_t)q.T, -777.0); std::vector<int64_t> mc((size_t)q.T, -1);
    cusim::launch(dim3((unsigned)((q.T + 31) / 32)), dim3(256), [&] { filo::merge_partials_kernel(pval.data(), pcnt.data(), gis, 1, q.T, op, 0, mv.data(), mc.data()); });
    std::vector<const double*> rs;
    for (int j = 0; j < 8; ++j)
      for (int64_t it = j; it < n_items; it += 8)
        for (int64_t p = item_begin[(size_t)it]; p < item_begin[(size_t)it + 1]; ++p) rs.push_back(ref.data() + (size_t)order[(size_t)p] * q.T);
    const fo::AggResult e = fo::aggregate((fo::AggrOp)op, 0, rs, std::vector<int32_t>(rs.size(), 0), 1, q.T);
    int at = 0;
    if (!row_same(mv.data(), e.values.data(), q.T, &at)) {
      std::printf("FAIL signed zeros fn %d op %d (%s kernel) merged window %d: %.17g vs %.17g\n", fn, op, kernel, at, mv[(size_t)at], e.values[(size_t)at]);
      return 1;
    }
    // the case is meaningful only where the rule decides: zeros of both signs meet at the result
    for (int k = 0; k < q.T; ++k) {
      bool pz = false, nz = false;
      for (const double* r : rs) if (r[k] == e.values[(size_t)k]) { if (std::signbit(r[k])) nz = true; else pz = true; }
      if (e.values[(size_t)k] == 0.0 && pz && nz) ++ties;
    }
    checked += q.T;
  }
  std::printf("signed zeros fn %d (%s) ok: %d series in %lld items\n", fn, xor_enc ? "xor" : "raw", nser, (long long)n_items);
  return 0;
}

// ---------------------------------------------------------------------------------------------------- 2. the v4 SUM kernel's value bounds
static int bounds_case(std::mt19937_64& rng, int fn, bool xor_enc, long& checked) {
  const std::vector<int> chunks = {400, 80};
  const int rows = 480;
  const double hi = std::ldexp(1.0, 513), lo = std::ldexp(1.0, -511);
  struct Edge { double v; bool admitted; };
  std::vector<Edge> edges = {{hi, false}, {std::nextafter(hi, 0.0), true}, {lo, true}, {std::nextafter(lo, 0.0), false}};
  for (int i = 0; i < 4; ++i) edges.push_back({-edges[(size_t)i].v, edges[(size_t)i].admitted});
  for (double x : {0.0, -0.0, 5e-324, DBL_MAX, -DBL_MAX, (double)INFINITY, -(double)INFINITY}) edges.push_back({x, false});
  const int edge_rows[6] = {0, 137, 399, 400, 479, 250};
  Table tb;
  std::vector<bool> admitted;
  std::vector<int64_t> ts((size_t)rows); for (int r = 0; r < rows; ++r) ts[(size_t)r] = kT0 + (int64_t)r * kStep;
  std::normal_distribution<double> N(0.0, 1.0);
  for (size_t i = 0; i < edges.size(); ++i) {
    for (int rep = 0; rep < 2; ++rep) {
      std::vector<double> v((size_t)rows);
      for (int r = 0; r < rows; ++r) v[(size_t)r] = 15.0 + std::sin((double)(r + 1)) + N(rng);
      v[(size_t)edge_rows[(i + (size_t)rep * 3) % 6]] = edges[i].v;
      tb.SS.emplace_back(); build_series_from(tb.SS.back(), rng, ts, v, chunks, 0, xor_enc, 0); admitted.push_back(edges[i].admitted);
    }
  }
  for (double scale : {std::ldexp(1.0, 512), std::ldexp(1.0, -510)}) {          // whole series at the edges, mixed signs
    for (int rep = 0; rep < 2; ++rep) {
      std::vector<double> v((size_t)rows);
      for (int r = 0; r < rows; ++r) v[(size_t)r] = scale * (1.0 + (double)(rng() >> 11) * 0x1p-53) * (rng() & 1 ? -1.0 : 1.0);
      tb.SS.emplace_back(); build_series_from(tb.SS.back(), rng, ts, v, chunks, 0, xor_enc, 0); admitted.push_back(true);
    }
  }
  finish_table(tb, rows, (int)chunks.size());
  const int nser = (int)tb.SS.size();
  filo::QueryParams q{};
  q.start = kT0 + 300000; q.step = kStep; q.end = kT0 + (int64_t)(rows - 1) * kStep; q.window = 300000;
  q.T = (int)((q.end - q.start) / q.step) + 1; q.fn = fn; q.cumulative = 0; q.inclusive = 1;
  int64_t exp_rows = 0;
  const std::vector<double> ref = oracle_rows(tb, q, &exp_rows);
  const uint32_t wrows = (uint32_t)(q.window / q.step) + 1;
  const filo::TileSmem L = filo::tile_layout(tb.max_rec, (uint32_t)rows, (uint32_t)q.T, 2 * wrows + 16);
  std::vector<double> out((size_t)nser * q.T, -777.0);
  std::vector<int64_t> flist((size_t)nser + 8, -1); unsigned long long fcount = 0, counters[2] = {0, 0}; int derr[4] = {0, 0, 0, 0};
  Launch A{tb.arena, tb.rec_off.data(), nser, q, out.data(), L, 2, flist.data(), &fcount, counters, derr, nullptr, nullptr, 0, 0, nullptr, nullptr};
  const bool alias = filo::wp_max_items((uint32_t)chunks.size(), (uint32_t)q.T, wrows) <= 64;
  filo::WpSmem W = filo::wp_layout(tb.max_rec, (uint32_t)rows, (uint32_t)chunks.size(), (uint32_t)q.T, wrows, alias);
  W.warps = 3;
  if ((size_t)W.per_warp * W.warps > sizeof(filo::smem)) { std::printf("FAIL: wp layout %u bytes per warp\n", W.per_warp); return 1; }
  auto body = [&](auto fnc) {
    cusim::launch(dim3((unsigned)A.grid), dim3(W.warps * 32), [&] {
      filo::scan_wp_sum_kernel<decltype(fnc)::value, 16>(A.arena, A.rec_off, A.S, A.q, A.out, W, A.flist, A.fcount, A.counters, A.derr);
    });
  };
  if (fn == filo::FN_RATE) body(std::integral_constant<int, filo::FN_RATE>{});
  else if (fn == filo::FN_AVG) body(std::integral_constant<int, filo::FN_AVG>{});
  else if (fn == filo::FN_COUNT) body(std::integral_constant<int, filo::FN_COUNT>{});
  else body(std::integral_constant<int, filo::FN_SUM>{});
  if (derr[0]) { std::printf("FAIL bounds fn %d: device error %d (wp kernel)\n", fn, derr[0]); return 1; }
  const std::set<int64_t> declined(flist.begin(), flist.begin() + (int64_t)fcount);
  if (declined.size() != (size_t)fcount) { std::printf("FAIL bounds fn %d: a series declined twice\n", fn); return 1; }
  for (int s = 0; s < nser; ++s)
    if ((declined.count(s) != 0) == admitted[(size_t)s]) {
      std::printf("FAIL bounds fn %d: series %d %s (expected %s)\n", fn, s, declined.count(s) ? "declined" : "admitted", admitted[(size_t)s] ? "admitted" : "declined");
      return 1;
    }
  if (fcount) run_v2(A, tb.sh, flist.data(), &fcount);
  if (derr[0]) { std::printf("FAIL bounds fn %d: device error %d\n", fn, derr[0]); return 1; }
  for (int s = 0; s < nser; ++s) {
    int at = 0;
    if (!row_same(out.data() + (size_t)s * q.T, ref.data() + (size_t)s * q.T, q.T, &at)) {
      std::printf("FAIL bounds fn %d series %d window %d: %.17g vs %.17g\n", fn, s, at, out[(size_t)s * q.T + at], ref[(size_t)s * q.T + at]);
      return 1;
    }
    checked += q.T;
  }
  if ((int64_t)counters[0] != exp_rows) { std::printf("FAIL bounds fn %d: samples_scanned %llu vs %lld\n", fn, counters[0], (long long)exp_rows); return 1; }
  std::printf("bounds fn %d (%s) ok: %llu of %d series declined\n", fn, xor_enc ? "xor" : "raw", fcount, nser);
  return 0;
}

int main(int argc, char** argv) {
  const uint64_t seed = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 0;
  cusim::rng_state() = seed;
  std::mt19937_64 rng(2513);
  long checked = 0, ties = 0; int cases = 0;
  for (bool xe : {true, false}) {
    for (int fn : {filo::FN_DELTA, filo::FN_LAST, filo::FN_MIN}) {
      if (signed_zero_case(rng, fn, xe, 40, 3, checked, ties)) return 1;
      ++cases;
    }
  }
  if (ties == 0) { std::printf("FAIL: no window where zeros of both signs meet at the min / max\n"); return 1; }
  for (bool xe : {true, false}) {
    for (int fn : {filo::FN_SUM, filo::FN_RATE, filo::FN_AVG, filo::FN_COUNT}) {
      if (bounds_case(rng, fn, xe, checked)) return 1;
      ++cases;
    }
  }
  std::printf("OK %d cases, %ld values bit-exact, %ld signed-zero ties (schedule seed %llu)\n", cases, checked, ties, (unsigned long long)seed);
  return 0;
}
