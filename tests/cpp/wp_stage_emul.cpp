// The window blocks of the v4 SUM kernel with a CTA-wide record stream (scan_wp_batch_kernel, scan_wp.cuh) write each finished window
// straight into the dense result row; raw tail sums go to the raw tail area behind the row, and a fix-up writes only the junction, raw
// and gap windows before the row's bulk store.  Compiled for the host on the cusim SIMT emulator.  Test infrastructure: built and run by
// tests/test_wp_stage_emul.py.  Cases: T = 1, 2, 3, 20, 27, 241, 480, 481 and 630; the output at a 16-byte-aligned base and at 8 mod 16
// (both row phases h); chunk junctions at several split points (block-aligned and not, so that raw tail blocks hold own windows too) with
// 2, 3 and 4 chunks; windows without rows in front of the data and in a time gap between chunks; sum / avg / count_over_time and rate;
// plan- and value-declined series as the next series of a warp that has just stored a row; a CTA's last batch partial; O in V's place
// (when the plan allows it) and apart.  Every result is bit-exact against the oracle (declined series through the v2 kernel), the scan
// counters match, and guard words on both sides of the output stay untouched.  The emulator defers every bulk copy as late as the
// program allows.
//   wp_stage_emul [seed]     seed 0 = round-robin schedule, otherwise a pseudo-random fiber schedule
#define main tile_emul_main
#include "tile_emul.cpp"
#undef main

static const int64_t kT0 = 1700000000000LL;
static const int kStep = 15000;
static const std::vector<int> kThreeChunks = {200, 10, 270};      // a 21-row window over rows 200 .. 209 spans all three chunks: declined by the plan

struct Case {
  int fn; std::vector<std::vector<int>> shapes;   // series s takes chunk shape s % shapes.size()
  int64_t window; int nser; int start_row; int T;
  int gap;                                        // steps without rows between the first chunk and the second
  std::vector<int> nan_series;                    // series with a NaN value: declined by the values
  std::vector<int> plan_series;                   // series with kThreeChunks: declined by the plan
  int grid;
  const char* what;
};
struct Shape { uint32_t consumers, B, nbuf; };

static bool has(const std::vector<int>& v, int s) { return std::find(v.begin(), v.end(), s) != v.end(); }

static int run_case(std::mt19937_64& rng, const Case& c, bool want_alias, const Shape& shp, int off8, long& checked, int& runs, bool fit_or_skip = false) {
  std::vector<SeriesData> SS((size_t)c.nser);
  std::normal_distribution<double> N(0.0, 1.0);
  int max_chunks = 0, max_rows = 0;
  for (int s = 0; s < c.nser; ++s) {
    const std::vector<int>& sh = has(c.plan_series, s) ? kThreeChunks : c.shapes[(size_t)s % c.shapes.size()];
    int r_s = 0; for (int n : sh) r_s += n;
    max_chunks = std::max<int>(max_chunks, (int)sh.size()); max_rows = std::max(max_rows, r_s);
    std::vector<int64_t> ts((size_t)r_s); std::vector<double> v((size_t)r_s);
    for (int r = 0; r < r_s; ++r) {
      ts[(size_t)r] = kT0 + (int64_t)(r + (r >= sh[0] ? c.gap : 0)) * kStep;
      v[(size_t)r] = 15.0 + std::sin((double)(r + 1)) + N(rng);
    }
    if (has(c.nan_series, s)) v[(size_t)(std::min(r_s - 1, c.start_row > 0 ? c.start_row - 3 : 5))] = std::nan("");
    build_series_from(SS[(size_t)s], rng, ts, v, sh, 0, true, 0);
  }
  std::vector<int64_t> rec_off((size_t)c.nser + 1, 0);
  for (int s = 0; s < c.nser; ++s) rec_off[(size_t)s + 1] = rec_off[(size_t)s] + (int64_t)SS[(size_t)s].record.size();
  std::vector<uint64_t> backing((size_t)rec_off.back() / 8 + 64, 0);
  uint8_t* arena = reinterpret_cast<uint8_t*>(backing.data());
  uint32_t max_rec = 0;
  for (int s = 0; s < c.nser; ++s) { std::memcpy(arena + rec_off[(size_t)s], SS[(size_t)s].record.data(), SS[(size_t)s].record.size()); max_rec = std::max<uint32_t>(max_rec, (uint32_t)SS[(size_t)s].record.size()); }
  filo::QueryParams q{};
  q.start = kT0 + (int64_t)c.start_row * kStep; q.step = kStep; q.end = q.start + (int64_t)(c.T - 1) * kStep; q.window = c.window;
  q.T = c.T; q.fn = c.fn; q.cumulative = 0; q.inclusive = 1;
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
  // the output: 16-byte-aligned storage, the rows from byte 8 * off8 of it on, guard words on both sides
  const size_t G = 6, nout = (size_t)c.nser * q.T;
  std::vector<uint64_t> store(2 * G + nout + 2);
  const uint64_t GUARD = 0x7ff4a5a5c3c3e1e1ull;                        // a signalling-NaN pattern no kernel writes
  for (auto& w : store) w = GUARD;
  if ((reinterpret_cast<uintptr_t>(store.data()) & 15) != 0) { std::printf("FAIL: output storage not 16-byte aligned\n"); return 1; }
  double* out = reinterpret_cast<double*>(store.data() + 2 * G + off8);
  for (size_t i = 0; i < nout; ++i) out[i] = -777.0;
  std::vector<int64_t> flist((size_t)c.nser + 8, -1); unsigned long long fcount = 0, counters[2] = {0, 0}; int derr[4] = {0, 0, 0, 0};
  Launch A{arena, rec_off.data(), c.nser, q, out, L, c.grid, flist.data(), &fcount, counters, derr, nullptr, nullptr, 0, 0, nullptr, nullptr};
  const filo::WpBatchSmem W = filo::wp_batch_layout(max_rec, (uint32_t)max_rows, (uint32_t)max_chunks, (uint32_t)q.T, wrows, want_alias, shp.B, shp.nbuf, shp.consumers);
  if ((size_t)W.total > sizeof(filo::smem) && fit_or_skip) return 0;      // (the product's shape with O apart: the host takes the per-warp kernel)
  if ((size_t)W.total > sizeof(filo::smem)) { std::printf("FAIL %s: batch layout %u bytes\n", c.what, W.total); return 1; }
  // poison the warps' regions: a window the kernel neither finishes in its block nor fixes up shows as a wrong result
  for (size_t i = 0; i < (size_t)W.W.per_warp * W.consumers; i += 8) { const uint64_t p = 0x7ff0dead0badf00dull; std::memcpy(filo::smem + i, &p, 8); }
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
  const size_t want_declined = c.nan_series.size() + c.plan_series.size();
  if (fcount != want_declined) { std::printf("FAIL %s: %llu series declined, expected %zu\n", c.what, fcount, want_declined); return 1; }
  if (fcount) {                                        // the fallback pass, as filo_query chains it
    V2Shape sh{max_rec, max_rows, max_chunks, false, false};
    run_v2(A, sh, flist.data(), &fcount);
    if (derr[0]) { std::printf("FAIL %s: device error %d (fallback)\n", c.what, derr[0]); return 1; }
  }
  const char* lay = want_alias ? "O in V" : "O apart";
  for (size_t i = 0; i < store.size(); ++i) {
    const bool row = i >= 2 * G + (size_t)off8 && i < 2 * G + (size_t)off8 + nout;
    if (!row && store[i] != GUARD) { std::printf("FAIL %s (%s, out + %d B): word %zd outside the rows written\n", c.what, lay, 8 * off8, (ptrdiff_t)i - (ptrdiff_t)(2 * G + off8)); return 1; }
  }
  for (int s = 0; s < c.nser; ++s)
    for (int k = 0; k < q.T; ++k) {
      const double a = out[(size_t)s * q.T + k], r = ref[(size_t)s * q.T + k];
      if (!same_bits(a, r)) {
        std::printf("FAIL %s (%s, out + %d B, %u consumers, B = %u x %u) series %d window %d: %.17g vs %.17g\n", c.what, lay, 8 * off8, shp.consumers, shp.B, shp.nbuf, s, k, a, r);
        return 1;
      }
      ++checked;
    }
  if ((int64_t)counters[0] != exp_rows) { std::printf("FAIL %s: samples_scanned %llu vs %lld\n", c.what, counters[0], (long long)exp_rows); return 1; }
  std::printf("%s (%s, out + %d B, %u consumers, B = %u x %u): %d series, T = %d ok\n", c.what, lay, 8 * off8, shp.consumers, shp.B, shp.nbuf, c.nser, q.T);
  ++runs;
  return 0;
}

int main(int argc, char** argv) {
  const uint64_t seed = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 0;
  cusim::rng_state() = seed;
  std::mt19937_64 rng(61017);
  // Series positions as in wp_bulk_store_emul: series 7, 8 and 31, 33 are the next series of warps that have just stored a row; with
  // 40 series CTA 0's last batch is partial for B = 15, CTA 1's for B = 3.  Junctions: 400 | 80 and 240 | 240 on the block grid of the
  // first chunk, 237 | 243 and 13 | 14 off it (the raw tail block of the first chunk then also holds own windows), three and four chunks.
  const std::vector<int> nan_s = {7, 31}, plan_s = {8, 33};
  const std::vector<Case> cases = {
    {filo::FN_RATE, {{400, 80}}, 300000, 40, 215, 1, 0, nan_s, plan_s, 2, "rate: T = 1"},
    {filo::FN_SUM, {{400, 80}, {237, 243}}, 300000, 40, 398, 2, 0, nan_s, {}, 2, "sum: junction, T = 2"},
    {filo::FN_AVG, {{400, 80}, {300, 180}}, 300000, 40, 213, 3, 0, nan_s, plan_s, 2, "avg: T = 3"},
    {filo::FN_COUNT, {{230, 250}, {237, 243}}, 300000, 40, 225, 20, 0, nan_s, {}, 2, "count: junction inside the row, T = 20"},
    {filo::FN_RATE, {{13, 14}, {14, 13}}, 135000, 40, 0, 27, 0, nan_s, {}, 2, "rate: one junction, T = 27"},
    {filo::FN_AVG, {{240, 240}, {237, 243}, {100, 190, 190}}, 300000, 40, 100, 241, 0, nan_s, plan_s, 2, "avg: two and three chunks, T = 241"},
    {filo::FN_SUM, {{60, 60, 60, 60}, {237, 3}}, 300000, 40, -20, 241, 0, nan_s, {}, 2, "sum: four chunks, T = 241"},
    {filo::FN_AVG, {{237, 243}}, 300000, 40, 0, 480, 0, nan_s, {}, 2, "avg: junction off the block grid, T = 480"},
    {filo::FN_RATE, {{400, 80}}, 300000, 40, 0, 481, 0, {7, 8, 31, 33}, {}, 2, "rate: C2 shape, T = 481"},
    {filo::FN_COUNT, {{200, 280}, {237, 243}}, 300000, 40, 0, 481, 45, nan_s, {}, 2, "count: gap between chunks, T = 481"},
    {filo::FN_RATE, {{120, 120, 120, 120}}, 300000, 40, -40, 481, 0, nan_s, {}, 2, "rate: four chunks, T = 481"},
    {filo::FN_SUM, {{400, 80}, {300, 180}}, 300000, 40, -60, 630, 0, nan_s, plan_s, 2, "sum: T = 630, windows past 512"},
    {filo::FN_AVG, {{150, 150, 180}, {237, 243}}, 300000, 19, -60, 630, 30, {2, 8}, {}, 3, "avg: T = 630, gap, three chunks"},
  };
  const Shape small{3, 3, 2};
  const Shape product{filo::WP_BATCH_WARPS - 1, filo::WP_BATCH_SERIES, filo::WP_BATCH_BUFS};
  long checked = 0; int runs = 0;
  for (const Case& c : cases)
    for (bool alias : {true, false})
      for (int off8 : {0, 1}) {
        if (run_case(rng, c, alias, small, off8, checked, runs)) return 1;
        if (run_case(rng, c, alias, product, off8, checked, runs, true)) return 1;
      }
  std::printf("OK %d runs of %zu cases, %ld values bit-exact, guards intact (schedule seed %llu)\n", runs, cases.size(), checked, (unsigned long long)seed);
  return 0;
}
