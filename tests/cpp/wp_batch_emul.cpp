// The v4 SUM kernel with a CTA-wide record stream (scan_wp_batch_kernel, scan_wp.cuh), compiled for the host on the cusim SIMT emulator.
// Test infrastructure: built and run by tests/test_wp_batch_emul.py.  The series builders and launch helpers are tile_emul.cpp's.  A
// producer warp fetches batches of B consecutive records with one bulk copy each and parses their headers into per-series entries; the
// consumer warps take the CTA's series in turn and release each record on its buffer's `empty` barrier.  Cases: CTAs without series, a
// partial last batch, a batch of one series, records of different sizes in one batch (the table's largest among them), series declined
// by the header parse (five chunks), by the plan (a window over three chunks) and by the values (a NaN stale marker) at the first, middle and last position of a batch,
// consecutive series with different plans (memo misses inside a batch), sum / avg / count_over_time and rate on a delta schema,
// T = 20, 27, 481 and 630, with O in V's place (when the plan allows it) and apart, at several (consumers, B, buffers) shapes including
// the product's.  Every result is bit-exact against the oracle (declined series through the v2 kernel), and the scan counters match.
//   wp_batch_emul [seed]     seed 0 = round-robin schedule, otherwise a pseudo-random fiber schedule
#define main tile_emul_main
#include "tile_emul.cpp"
#undef main

static const int64_t kT0 = 1700000000000LL;
static const int kStep = 15000;
static const std::vector<int> kThreeChunks = {200, 10, 270};      // a 21-row window spans all three chunks: the plan declines the series
static const std::vector<int> kFiveChunks = {100, 100, 100, 100, 80};   // more than four chunks in range: the header parse declines the series

struct Case {
  int fn; std::vector<std::vector<int>> shapes;   // series s takes chunk shape s % shapes.size() (total rows may differ)
  int64_t window; int nser; int64_t start_off, end_off;
  std::vector<int> nan_series;                    // series with a NaN stale marker: declined by the values
  std::vector<int> plan_series;                   // series with kThreeChunks: declined by the plan
  std::vector<int> parse_series;                  // series with kFiveChunks: declined by the header parse (also on a memo hit)
  int grid;
  const char* what;
};
struct Shape { uint32_t consumers, B, nbuf; };

static bool has(const std::vector<int>& v, int s) { return std::find(v.begin(), v.end(), s) != v.end(); }

static int run_case(std::mt19937_64& rng, const Case& c, bool want_alias, const Shape& shp, long& checked, int& runs, bool fit_or_skip = false) {
  int rows = 0; for (int n : c.shapes[0]) rows += n;
  std::vector<SeriesData> SS((size_t)c.nser);
  std::normal_distribution<double> N(0.0, 1.0);
  int max_chunks = 0, max_rows = 0;
  for (int s = 0; s < c.nser; ++s) {
    const std::vector<int>& sh = has(c.plan_series, s) ? kThreeChunks : has(c.parse_series, s) ? kFiveChunks : c.shapes[(size_t)s % c.shapes.size()];
    int r_s = 0; for (int n : sh) r_s += n;
    max_chunks = std::max<int>(max_chunks, (int)sh.size()); max_rows = std::max(max_rows, r_s);
    std::vector<int64_t> ts((size_t)r_s); std::vector<double> v((size_t)r_s);
    for (int r = 0; r < r_s; ++r) { ts[(size_t)r] = kT0 + (int64_t)r * kStep; v[(size_t)r] = 15.0 + std::sin((double)(r + 1)) + N(rng); }
    if (has(c.nan_series, s)) v[(size_t)(r_s / 3)] = std::nan("");
    build_series_from(SS[(size_t)s], rng, ts, v, sh, 0, true, 0);
  }
  std::vector<int64_t> rec_off((size_t)c.nser + 1, 0);
  for (int s = 0; s < c.nser; ++s) rec_off[(size_t)s + 1] = rec_off[(size_t)s] + (int64_t)SS[(size_t)s].record.size();
  std::vector<uint64_t> backing((size_t)rec_off.back() / 8 + 64, 0);
  uint8_t* arena = reinterpret_cast<uint8_t*>(backing.data());
  uint32_t max_rec = 0;
  for (int s = 0; s < c.nser; ++s) { std::memcpy(arena + rec_off[(size_t)s], SS[(size_t)s].record.data(), SS[(size_t)s].record.size()); max_rec = std::max<uint32_t>(max_rec, (uint32_t)SS[(size_t)s].record.size()); }
  filo::QueryParams q{};
  q.start = kT0 + c.start_off; q.step = kStep; q.end = kT0 + (int64_t)(rows - 1) * kStep + c.end_off; q.window = c.window;
  q.T = (int)((q.end - q.start) / q.step) + 1; q.fn = c.fn; q.cumulative = 0; q.inclusive = 1;
  std::vector<double> ref((size_t)c.nser * q.T); int64_t exp_rows = 0;
  for (int s = 0; s < c.nser; ++s) {
    fo::Series os; for (auto& ch : SS[(size_t)s].chunks) os.infos.push_back(ch->info.data());
    fo::QueryStats st;
    fo::periodicSamples(os, oracle_fn(q.fn), false, q.start, q.step, q.end, q.window, fo::QueryConfig{true}, ref.data() + (size_t)s * q.T, &st, 0, 0);
    exp_rows += st.samplesScanned;
  }
  const uint32_t wrows = (uint32_t)(q.window / q.step) + 1;
  if (want_alias && filo::wp_max_items((uint32_t)max_chunks, (uint32_t)q.T, wrows) > 64) return 0;      // O in V's place needs one pass of <= 64 blocks
  const filo::TileSmem L = filo::tile_layout(max_rec, (uint32_t)max_rows, (uint32_t)q.T, 2 * wrows + 16);
  std::vector<double> out((size_t)c.nser * q.T, -777.0);
  std::vector<int64_t> flist((size_t)c.nser + 8, -1); unsigned long long fcount = 0, counters[2] = {0, 0}; int derr[4] = {0, 0, 0, 0};
  Launch A{arena, rec_off.data(), c.nser, q, out.data(), L, c.grid, flist.data(), &fcount, counters, derr, nullptr, nullptr, 0, 0, nullptr, nullptr};
  const filo::WpBatchSmem W = filo::wp_batch_layout(max_rec, (uint32_t)max_rows, (uint32_t)max_chunks, (uint32_t)q.T, wrows, want_alias, shp.B, shp.nbuf, shp.consumers);
  if (W.W.vals != filo::WP_OFF_REC || W.buf < W.W.per_warp * W.consumers || W.ent < W.buf + W.nbuf * W.buf_stride || W.bars < W.ent + W.nbuf * W.B * sizeof(filo::WpEntry)) {
    std::printf("FAIL %s: batch layout overlaps\n", c.what); return 1;
  }
  if ((size_t)W.total > sizeof(filo::smem) && fit_or_skip) return 0;      // (the product's shape with O apart: the host takes the per-warp kernel)
  if ((size_t)W.total > sizeof(filo::smem)) { std::printf("FAIL %s: batch layout %u bytes\n", c.what, W.total); return 1; }
  auto body = [&](auto fnc) {
    cusim::launch(dim3((unsigned)A.grid), dim3((W.consumers + 1) * 32), [&] {
      filo::scan_wp_batch_kernel<decltype(fnc)::value, filo::WP_BATCH_WARPS>(A.arena, A.rec_off, A.S, A.q, A.out, W, A.flist, A.fcount, A.counters, A.derr);
    });
  };
  if (c.fn == filo::FN_RATE) body(std::integral_constant<int, filo::FN_RATE>{});
  else if (c.fn == filo::FN_AVG) body(std::integral_constant<int, filo::FN_AVG>{});
  else if (c.fn == filo::FN_COUNT) body(std::integral_constant<int, filo::FN_COUNT>{});
  else body(std::integral_constant<int, filo::FN_SUM>{});
  if (derr[0]) { std::printf("FAIL %s: device error %d\n", c.what, derr[0]); return 1; }
  const size_t want_declined = c.nan_series.size() + c.plan_series.size() + c.parse_series.size();
  if (fcount != want_declined) { std::printf("FAIL %s: %llu series declined, expected %zu\n", c.what, fcount, want_declined); return 1; }
  if (fcount) {                                        // the fallback pass, as filo_query chains it
    V2Shape sh{max_rec, max_rows, max_chunks, false, false};
    run_v2(A, sh, flist.data(), &fcount);
    if (derr[0]) { std::printf("FAIL %s: device error %d (fallback)\n", c.what, derr[0]); return 1; }
  }
  const char* lay = want_alias ? "O in V" : "O apart";
  for (int s = 0; s < c.nser; ++s)
    for (int k = 0; k < q.T; ++k) {
      const double a = out[(size_t)s * q.T + k], r = ref[(size_t)s * q.T + k];
      if (!same_bits(a, r)) {
        std::printf("FAIL %s (%s, %u consumers, B = %u x %u) series %d window %d: %.17g vs %.17g\n", c.what, lay, shp.consumers, shp.B, shp.nbuf, s, k, a, r);
        return 1;
      }
      ++checked;
    }
  if ((int64_t)counters[0] != exp_rows) { std::printf("FAIL %s: samples_scanned %llu vs %lld\n", c.what, counters[0], (long long)exp_rows); return 1; }
  std::printf("%s (%s, %u consumers, B = %u x %u): %d series, T = %d ok\n", c.what, lay, shp.consumers, shp.B, shp.nbuf, c.nser, q.T);
  ++runs;
  return 0;
}

int main(int argc, char** argv) {
  const uint64_t seed = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 0;
  cusim::rng_state() = seed;
  std::mt19937_64 rng(4817);
  const std::vector<Case> cases = {
    // 2 CTAs, B = 3: 37 series end in a batch of one series
    {filo::FN_RATE, {{400, 80}}, 300000, 37, 0, 15000, {}, {}, {}, 2, "rate: C2 shape, T = 481, 37 series"},
    {filo::FN_RATE, {{400, 80}}, 300000, 1, 0, 15000, {}, {}, {}, 2, "rate: one series, a CTA without series"},
    {filo::FN_SUM, {{400, 80}}, 300000, 5, 0, 15000, {}, {}, {}, 4, "sum: 5 series over 4 CTAs, CTAs without series"},
    // records of 480, 280, 480 and 400 rows: different sizes in one batch, the largest (the table's maximum) several times
    {filo::FN_SUM, {{400, 80}, {200, 80}, {300, 180}, {400}}, 300000, 24, 0, 15000, {}, {}, {}, 2, "sum: different sizes and plans in one batch"},
    // value- and plan-declined series at positions 0, 1, 2 of the batches of B = 3 (and 0, 1 of B = 2)
    {filo::FN_AVG, {{300, 180}, {400, 80}}, 300000, 31, 0, 0, {0, 4, 8, 30}, {3, 13, 20}, {9, 16, 23}, 2, "avg: declined series at every batch position"},
    {filo::FN_COUNT, {{400, 80}}, 300000, 11, 0, 0, {5, 10}, {6}, {1}, 3, "count: declined middle and last series"},
    {filo::FN_SUM, {{20}}, 150000, 13, 0, 0, {0, 6}, {}, {}, 2, "sum: one chunk, T = 20, declined first series"},
    {filo::FN_COUNT, {{20}}, 150000, 7, 0, 0, {}, {}, {}, 2, "count: one chunk, T = 20"},
    {filo::FN_RATE, {{13, 14}, {14, 13}}, 135000, 18, 0, 0, {}, {}, {}, 2, "rate: one junction, T = 27"},
    {filo::FN_AVG, {{13, 14}, {14, 13}}, 135000, 9, 0, 0, {4}, {}, {}, 2, "avg: one junction, T = 27"},
    {filo::FN_AVG, {{400, 80}}, 300000, 19, -60 * 15000, 90 * 15000, {2, 8}, {}, {}, 2, "avg: T = 630, windows past 512"},
    {filo::FN_RATE, {{400, 80}, {300, 180}}, 300000, 14, -60 * 15000, 90 * 15000, {}, {7}, {}, 2, "rate: T = 630, different plans"},
  };
  const Shape shapes[] = {{3, 3, 2}, {3, 2, 3}};
  const Shape product{filo::WP_BATCH_WARPS - 1, filo::WP_BATCH_SERIES, filo::WP_BATCH_BUFS};
  long checked = 0; int runs = 0;
  for (size_t i = 0; i < cases.size(); ++i) {
    const Case& c = cases[i];
    for (bool alias : {true, false}) {
      for (const Shape& sh : shapes) if (run_case(rng, c, alias, sh, checked, runs)) return 1;
      if (i == 0 || i == 4 || i == 11) { if (run_case(rng, c, alias, product, checked, runs, true)) return 1; }
    }
  }
  std::printf("OK %d runs of %zu cases, %ld values bit-exact (schedule seed %llu)\n", runs, cases.size(), checked, (unsigned long long)seed);
  return 0;
}
