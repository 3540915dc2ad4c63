// The v4 SUM kernel (scan_wp_sum_kernel, scan_wp.cuh) with two record buffers per warp, compiled for the host on the cusim SIMT
// emulator.  Test infrastructure: built and run by tests/test_wp_rec2_emul.py.  The series builders and launch helpers are
// tile_emul.cpp's.  A warp's series alternate between the two buffers, each with its own mbarrier, and the record of the series two
// iterations ahead is issued into the buffer of the series just decoded.  Cases: series counts that leave warps with one, two and
// many series (odd and even), consecutive series with different window plans, declined series (a NaN stale marker, answered by the
// v2 kernel into the same output) in either buffer, sum / avg / count_over_time and rate on a delta schema, T = 20, 27, 481 and 630,
// with O in V's place (when the plan allows it) and apart.  Every result is bit-exact against the oracle, and the scan counters match.
//   wp_rec2_emul [seed]     seed 0 = round-robin schedule, otherwise a pseudo-random fiber schedule
#define main tile_emul_main
#include "tile_emul.cpp"
#undef main

static const int64_t kT0 = 1700000000000LL;
static const int kStep = 15000;

struct Case {
  int fn; std::vector<std::vector<int>> shapes;   // series s takes chunk shape s % shapes.size() (same total rows)
  int64_t window; int nser; int64_t start_off, end_off;
  std::vector<int> nan_series;                    // series with a NaN stale marker: declined to the fallback list
  const char* what;
};

static int run_case(std::mt19937_64& rng, const Case& c, bool want_alias, long& checked, int& runs) {
  int rows = 0; for (int n : c.shapes[0]) rows += n;
  int max_chunks = 0; for (auto& sh : c.shapes) max_chunks = std::max<int>(max_chunks, (int)sh.size());
  std::vector<SeriesData> SS((size_t)c.nser);
  std::normal_distribution<double> N(0.0, 1.0);
  for (int s = 0; s < c.nser; ++s) {
    std::vector<int64_t> ts((size_t)rows); std::vector<double> v((size_t)rows);
    for (int r = 0; r < rows; ++r) { ts[(size_t)r] = kT0 + (int64_t)r * kStep; v[(size_t)r] = 15.0 + std::sin((double)(r + 1)) + N(rng); }
    if (std::find(c.nan_series.begin(), c.nan_series.end(), s) != c.nan_series.end()) v[(size_t)(rows / 3)] = std::nan("");
    build_series_from(SS[(size_t)s], rng, ts, v, c.shapes[(size_t)s % c.shapes.size()], 0, true, 0);
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
  const filo::TileSmem L = filo::tile_layout(max_rec, (uint32_t)rows, (uint32_t)q.T, 2 * wrows + 16);
  std::vector<double> out((size_t)c.nser * q.T, -777.0);
  std::vector<int64_t> flist((size_t)c.nser + 8, -1); unsigned long long fcount = 0, counters[2] = {0, 0}; int derr[4] = {0, 0, 0, 0};
  Launch A{arena, rec_off.data(), c.nser, q, out.data(), L, 2, flist.data(), &fcount, counters, derr, nullptr, nullptr, 0, 0, nullptr, nullptr};
  filo::WpSmem W = filo::wp_layout(max_rec, (uint32_t)rows, (uint32_t)max_chunks, (uint32_t)q.T, wrows, want_alias, true);
  W.warps = 3;
  if (W.rec2 == 0 || W.rec2 < W.rec + W.rec_cap || W.vals < W.rec2 + W.rec_cap) { std::printf("FAIL %s: layout without a second record buffer\n", c.what); return 1; }
  if ((size_t)W.per_warp * W.warps > sizeof(filo::smem)) { std::printf("FAIL %s: wp layout %u bytes per warp\n", c.what, W.per_warp); return 1; }
  auto body = [&](auto fnc) {
    cusim::launch(dim3((unsigned)A.grid), dim3(W.warps * 32), [&] {
      filo::scan_wp_sum_kernel<decltype(fnc)::value, 16>(A.arena, A.rec_off, A.S, A.q, A.out, W, A.flist, A.fcount, A.counters, A.derr);
    });
  };
  if (c.fn == filo::FN_RATE) body(std::integral_constant<int, filo::FN_RATE>{});
  else if (c.fn == filo::FN_AVG) body(std::integral_constant<int, filo::FN_AVG>{});
  else if (c.fn == filo::FN_COUNT) body(std::integral_constant<int, filo::FN_COUNT>{});
  else body(std::integral_constant<int, filo::FN_SUM>{});
  if (derr[0]) { std::printf("FAIL %s: device error %d\n", c.what, derr[0]); return 1; }
  if (fcount != c.nan_series.size()) { std::printf("FAIL %s: %llu series declined, expected %zu\n", c.what, fcount, c.nan_series.size()); return 1; }
  if (fcount) {                                        // the fallback pass, as filo_query chains it
    V2Shape sh{max_rec, rows, max_chunks, false, false};
    run_v2(A, sh, flist.data(), &fcount);
    if (derr[0]) { std::printf("FAIL %s: device error %d (fallback)\n", c.what, derr[0]); return 1; }
  }
  const char* lay = want_alias ? "O in V" : "O apart";
  for (int s = 0; s < c.nser; ++s)
    for (int k = 0; k < q.T; ++k) {
      const double a = out[(size_t)s * q.T + k], r = ref[(size_t)s * q.T + k];
      if (!same_bits(a, r)) { std::printf("FAIL %s (%s) series %d window %d: %.17g vs %.17g\n", c.what, lay, s, k, a, r); return 1; }
      ++checked;
    }
  if ((int64_t)counters[0] != exp_rows) { std::printf("FAIL %s: samples_scanned %llu vs %lld\n", c.what, counters[0], (long long)exp_rows); return 1; }
  std::printf("%s (%s): %d series, T = %d ok\n", c.what, lay, c.nser, q.T);
  ++runs;
  return 0;
}

int main(int argc, char** argv) {
  const uint64_t seed = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 0;
  cusim::rng_state() = seed;
  std::mt19937_64 rng(4813);
  // 2 CTAs of 3 warps: 6 warps, so 5 series leave a warp without series, 7 and 11 give warps one and two series, 37 up to seven
  const std::vector<Case> cases = {
    {filo::FN_RATE, {{400, 80}}, 300000, 37, 0, 15000, {}, "rate: C2 shape, T = 481, 37 series"},
    {filo::FN_RATE, {{400, 80}}, 300000, 1, 0, 15000, {}, "rate: C2 shape, one series"},
    {filo::FN_SUM, {{400, 80}}, 300000, 5, 0, 15000, {}, "sum: 5 series, a warp without series"},
    {filo::FN_SUM, {{400, 80}, {300, 180}}, 300000, 24, 0, 15000, {}, "sum: consecutive series with different plans, 24 series"},
    {filo::FN_AVG, {{300, 180}, {400, 80}, {400, 80}}, 300000, 31, 0, 0, {3, 9, 10, 16, 30}, "avg: different plans, declined series in both buffers"},
    {filo::FN_COUNT, {{400, 80}}, 300000, 11, 0, 0, {6, 10}, "count: declined second and last series"},
    {filo::FN_SUM, {{20}}, 150000, 13, 0, 0, {0, 6}, "sum: one chunk, T = 20, declined first series"},
    {filo::FN_RATE, {{13, 14}, {14, 13}}, 135000, 18, 0, 0, {}, "rate: one junction, T = 27"},
    {filo::FN_AVG, {{400, 80}}, 300000, 19, -60 * 15000, 90 * 15000, {2, 8}, "avg: T = 630, windows past 512"},
  };
  long checked = 0; int runs = 0;
  for (const Case& c : cases)
    for (bool alias : {true, false})
      if (run_case(rng, c, alias, checked, runs)) return 1;
  std::printf("OK %d runs of %zu cases, %ld values bit-exact (schedule seed %llu)\n", runs, cases.size(), checked, (unsigned long long)seed);
  return 0;
}
