// The finish pass of the v4 SUM kernel (scan_wp_sum_kernel, scan_wp.cuh), compiled for the host on the cusim SIMT emulator.  Test
// infrastructure: built and run by tests/test_wp_finish_emul.py.  The series builders and launch helpers are tile_emul.cpp's.
// Every window class of the plan (finished by its window block, raw sum to finish, chunk junction, no rows) over every SUM-class
// function: 1-4 chunks, windows without rows in front, between chunks and behind, T < 32 and T not a multiple of 32, head shares
// longer than one block and than 32 windows, raw f64 chunks next to XOR chunks, blocks on and off O's 9-word grid, plans of more
// than 64 blocks (T > 512).  Each case runs with O in V's place (when the plan allows it) and with O apart; no series may be declined,
// and every result is bit-exact against the oracle.
//   wp_finish_emul [seed]     seed 0 = round-robin schedule, otherwise a pseudo-random fiber schedule
#define main tile_emul_main
#include "tile_emul.cpp"
#undef main

static const int64_t kT0 = 1700000000000LL;
static const int kStep = 15000;

// the arena record of a series from its chunks (as build_series_from writes it)
static void record_of(SeriesData& S) {
  const size_t nch = S.chunks.size();
  const size_t off = sizeof(filo::RecordHeader) + nch * sizeof(filo::ChunkEntry);
  std::vector<filo::ChunkEntry> E(nch); std::vector<uint8_t> body; uint32_t row_base = 0, flags = filo::REC_ALL_TS_CONST;
  for (size_t i = 0; i < nch; ++i) {
    Chunk& c = *S.chunks[i];
    E[i].start_time = fo::csi::startTime(c.info.data()); E[i].end_time = fo::csi::endTime(c.info.data()); E[i].num_rows = fo::csi::numRows(c.info.data());
    auto put = [&](const std::vector<uint8_t>& x) { while ((off + body.size()) % 8) body.push_back(0); const uint32_t o = (uint32_t)(off + body.size()); body.insert(body.end(), x.begin(), x.end()); return o; };
    E[i].ts_off = put(c.ts); E[i].val_off = put(c.vv); E[i].row_base = row_base;
    const int vwire = (int)(c.vv[4] | (c.vv[5] << 8));
    if (vwire == filo::WIRE_XOR) flags |= filo::REC_ANY_DECODE;
    row_base += (uint32_t)E[i].num_rows;
  }
  size_t total = off + body.size(); total = (total + 15) & ~(size_t)15;
  S.record.assign(total, 0);
  filo::RecordHeader h; h.rec_bytes = (uint32_t)total; h.n_chunks = (uint32_t)nch; h.n_rows = row_base; h.flags = flags;
  std::memcpy(S.record.data(), &h, sizeof h);
  std::memcpy(S.record.data() + sizeof h, E.data(), nch * sizeof(filo::ChunkEntry));
  std::memcpy(S.record.data() + off, body.data(), body.size());
}

struct Case {
  int fn; std::vector<int> chunks; int64_t window; int nser; int inclusive; int64_t start_off, end_off;
  int gap;      // steps without rows in front of every chunk but the first
  bool mix;     // every second chunk keeps raw f64 values (the others are XOR)
  const char* what;
};

static int run_case(std::mt19937_64& rng, const Case& c, bool want_alias, long& checked, int& runs) {
  int rows = 0; for (int n : c.chunks) rows += n;
  const int nch = (int)c.chunks.size();
  std::vector<SeriesData> SS((size_t)c.nser);
  std::normal_distribution<double> N(0.0, 1.0);
  for (int s = 0; s < c.nser; ++s) {
    std::vector<int64_t> ts((size_t)rows); std::vector<double> v((size_t)rows);
    for (int r = 0, ci = 0, cend = c.chunks[0]; r < rows; ++r) {
      while (r >= cend) cend += c.chunks[(size_t)++ci];
      ts[(size_t)r] = kT0 + (int64_t)(r + c.gap * ci) * kStep;
      v[(size_t)r] = 15.0 + std::sin((double)(r + 1)) + N(rng);
    }
    SeriesData& S = SS[(size_t)s];
    build_series_from(S, rng, ts, v, c.chunks, 0, true, 0);
    if (c.mix) {
      for (int ci = 1, r0 = c.chunks[0]; ci < nch; r0 += c.chunks[(size_t)ci], ++ci) {
        if (!(ci & 1)) continue;
        Chunk& ch = *S.chunks[(size_t)ci];
        ch.vv = fo::enc::doubles(v.data() + r0, c.chunks[(size_t)ci], false);
        fo::setLong(ch.info.data() + fo::csi::OffsetVectors + 8, (int64_t)(uintptr_t)ch.vv.data());
      }
      record_of(S);
    }
  }
  std::vector<int64_t> rec_off((size_t)c.nser + 1, 0);
  for (int s = 0; s < c.nser; ++s) rec_off[(size_t)s + 1] = rec_off[(size_t)s] + (int64_t)SS[(size_t)s].record.size();
  std::vector<uint64_t> backing((size_t)rec_off.back() / 8 + 64, 0);
  uint8_t* arena = reinterpret_cast<uint8_t*>(backing.data());
  uint32_t max_rec = 0;
  for (int s = 0; s < c.nser; ++s) { std::memcpy(arena + rec_off[(size_t)s], SS[(size_t)s].record.data(), SS[(size_t)s].record.size()); max_rec = std::max<uint32_t>(max_rec, (uint32_t)SS[(size_t)s].record.size()); }
  filo::QueryParams q{};
  q.start = kT0 + c.start_off; q.step = kStep; q.end = kT0 + (int64_t)(rows - 1 + c.gap * (nch - 1)) * kStep + c.end_off; q.window = c.window;
  q.T = (int)((q.end - q.start) / q.step) + 1; q.fn = c.fn; q.cumulative = 0; q.inclusive = c.inclusive;
  std::vector<double> ref((size_t)c.nser * q.T); int64_t exp_rows = 0;
  for (int s = 0; s < c.nser; ++s) {
    fo::Series os; for (auto& ch : SS[(size_t)s].chunks) os.infos.push_back(ch->info.data());
    fo::QueryStats st;
    fo::periodicSamples(os, oracle_fn(q.fn), false, q.start, q.step, q.end, q.window, fo::QueryConfig{q.inclusive != 0}, ref.data() + (size_t)s * q.T, &st, 0, 0);
    exp_rows += st.samplesScanned;
  }
  const uint32_t wrows = (uint32_t)(q.window / q.step) + 1;
  if (want_alias && filo::wp_max_items((uint32_t)nch, (uint32_t)q.T, wrows) > 64) return 0;      // O in V's place needs one pass of <= 64 blocks
  const filo::TileSmem L = filo::tile_layout(max_rec, (uint32_t)rows, (uint32_t)q.T, 2 * wrows + 16);
  std::vector<double> out((size_t)c.nser * q.T, -777.0);
  std::vector<int64_t> flist((size_t)c.nser + 8, -1); unsigned long long fcount = 0, counters[2] = {0, 0}; int derr[4] = {0, 0, 0, 0};
  Launch A{arena, rec_off.data(), c.nser, q, out.data(), L, 2, flist.data(), &fcount, counters, derr, nullptr, nullptr, 0, 0, nullptr, nullptr};
  filo::WpSmem W = filo::wp_layout(max_rec, (uint32_t)rows, (uint32_t)nch, (uint32_t)q.T, wrows, want_alias);
  W.warps = 3;
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
  if (fcount) { std::printf("FAIL %s: %llu of %d series declined (the case must run on the v4 SUM kernel)\n", c.what, fcount, c.nser); return 1; }
  for (int s = 0; s < c.nser; ++s)
    for (int k = 0; k < q.T; ++k) {
      const double a = out[(size_t)s * q.T + k], r = ref[(size_t)s * q.T + k];
      if (!same_bits(a, r)) { std::printf("FAIL %s (%s) series %d window %d: %.17g vs %.17g\n", c.what, want_alias ? "O in V" : "O apart", s, k, a, r); return 1; }
      ++checked;
    }
  if ((int64_t)counters[0] != exp_rows) { std::printf("FAIL %s: samples_scanned %llu vs %lld\n", c.what, counters[0], (long long)exp_rows); return 1; }
  std::printf("%s (%s): %d series, T = %d ok\n", c.what, want_alias ? "O in V" : "O apart", c.nser, q.T);
  ++runs;
  return 0;
}

int main(int argc, char** argv) {
  const uint64_t seed = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 0;
  cusim::rng_state() = seed;
  std::mt19937_64 rng(4811);
  const std::vector<Case> cases = {
    {filo::FN_RATE, {300, 100}, 300000, 9, 1, -330000, 330000, 0, false, "rate: windows without rows in front and behind"},
    {filo::FN_AVG, {150, 90, 110}, 300000, 8, 1, 0, 0, 30, true, "avg: windows without rows between chunks, raw next to XOR"},
    {filo::FN_COUNT, {200, 100, 60, 70}, 600000, 7, 0, 0, 0, 0, false, "count: four chunks, head shares of 40 windows"},
    {filo::FN_SUM, {20}, 150000, 5, 1, 0, 0, 0, false, "sum: one chunk, T = 20"},
    {filo::FN_RATE, {13, 14}, 135000, 6, 1, 0, 0, 0, false, "rate: one junction, T = 27"},
    {filo::FN_AVG, {200, 200, 200}, 600000, 5, 1, 0, 0, 0, true, "avg: head shares of 40 windows, T = 600, raw next to XOR"},
    {filo::FN_RATE, {250, 250, 250, 250}, 300000, 6, 1, 0, 0, 0, true, "rate: four chunks, T = 1000, raw next to XOR"},
    {filo::FN_SUM, {100, 37, 91}, 300000, 8, 0, -15000, 0, 3, true, "sum: short gaps inside windows, raw next to XOR"},
    {filo::FN_COUNT, {64, 64}, 300000, 6, 1, 0, 45000, 25, false, "count: windows without rows between chunks"},
    {filo::FN_RATE, {120, 120, 120, 120}, 300000, 7, 1, 0, 0, 0, false, "rate: four chunks on O's 9-word grid"},
    {filo::FN_AVG, {401, 79}, 300000, 9, 1, 7000, 0, 0, false, "avg: C2 shape off O's grid, unaligned start"},
  };
  long checked = 0; int runs = 0;
  for (const Case& c : cases)
    for (bool alias : {true, false})
      if (run_case(rng, c, alias, checked, runs)) return 1;
  std::printf("OK %d runs of %zu cases, %ld values bit-exact (schedule seed %llu)\n", runs, cases.size(), checked, (unsigned long long)seed);
  return 0;
}
