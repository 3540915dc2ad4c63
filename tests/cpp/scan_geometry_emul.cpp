// The per-series scan kernels across query geometry, on the cusim SIMT emulator.  Test infrastructure: built and run by
// tests/test_scan_geometry_emul.py, which writes the cases of tests/scan_geometry_cases.py to a file.  The series builders and the v2
// launch are tile_emul.cpp's.  Every query (a case in one range mode) runs on each kernel of its class, with the declined series
// chained to the v2 kernel the way filo_query chains them:
//   SUM class      scan_wp_batch_kernel with O on V (when the plan bound allows it) and O apart, at 3 consumers / B = 3 / 2 buffers and
//                  at the product's shape (on the cases that ask for it); scan_wp_sum_kernel with one and two record buffers; the tile kernel
//   counter class  scan_wp_ctr_kernel, const-DDV and irregular-timestamp instantiations
// Every value is bit-exact against fo::periodicSamples with QueryConfig{inclusive}, the scan counters are the oracle's, and each kernel
// declines exactly the series the case file predicts (the same series, not only as many).
//   scan_geometry_emul <seed> <cases file>     seed 0 = round-robin schedule, otherwise a pseudo-random fiber schedule
#define main tile_emul_main
#include "tile_emul.cpp"
#undef main
#include <fstream>
#include <map>

struct GChunk { char enc; std::vector<int64_t> ts; std::vector<double> v; };
struct GQuery {
  std::string name; int counter = 0, product = 0; filo::QueryParams q{}; std::vector<int> fns;
  std::vector<int64_t> exp_wp, exp_tile, exp_ctr_const, exp_ctr_irr;      // ids of the series each kernel is expected to decline
  std::vector<std::vector<GChunk>> series;
};

static bool read_queries(const char* path, std::vector<GQuery>& out) {
  std::ifstream f(path);
  int nq = 0;
  if (!(f >> nq)) return false;
  out.resize((size_t)nq);
  for (GQuery& g : out) {
    long long start, step, end, window; int T, incl, nf, ns;
    f >> g.name >> g.counter >> g.product >> start >> step >> end >> window >> T >> incl >> nf;
    g.q.start = start; g.q.step = step; g.q.end = end; g.q.window = window; g.q.T = T; g.q.inclusive = incl; g.q.cumulative = g.counter;
    g.fns.resize((size_t)nf); for (int& x : g.fns) f >> x;
    for (auto* ids : {&g.exp_wp, &g.exp_tile, &g.exp_ctr_const, &g.exp_ctr_irr}) {
      int nd = 0; f >> nd; ids->resize((size_t)std::max(nd, 0));
      for (int64_t& x : *ids) { long long y; f >> y; x = y; }
    }
    f >> ns;
    g.series.resize((size_t)ns);
    for (auto& S : g.series) {
      int nc; f >> nc; S.resize((size_t)nc);
      for (GChunk& c : S) {
        int n; f >> c.enc >> n; c.ts.resize((size_t)n); c.v.resize((size_t)n);
        for (int64_t& t : c.ts) { long long x; f >> x; t = x; }
        for (double& v : c.v) { std::string h; f >> h; const uint64_t b = std::strtoull(h.c_str(), nullptr, 16); std::memcpy(&v, &b, 8); }
      }
    }
    if (!f) return false;
  }
  return true;
}

struct Table {
  std::vector<SeriesData> SS; std::vector<int64_t> rec_off; std::vector<uint64_t> backing; uint8_t* arena = nullptr;
  uint32_t max_rec = 0; int max_rows = 0, max_chunks = 0;
};
static void build_table(std::mt19937_64& rng, const GQuery& g, Table& tb) {
  const int ns = (int)g.series.size();
  tb.SS.clear(); tb.SS.resize((size_t)ns); tb.rec_off.assign((size_t)ns + 1, 0);
  for (int s = 0; s < ns; ++s) {
    std::vector<int64_t> ts; std::vector<double> v; std::vector<int> rows; g_chunk_enc.clear();
    for (const GChunk& c : g.series[(size_t)s]) { ts.insert(ts.end(), c.ts.begin(), c.ts.end()); v.insert(v.end(), c.v.begin(), c.v.end()); rows.push_back((int)c.ts.size()); g_chunk_enc += c.enc; }
    build_series_from(tb.SS[(size_t)s], rng, ts, v, rows, g.counter, true, 0);
    tb.rec_off[(size_t)s + 1] = tb.rec_off[(size_t)s] + (int64_t)tb.SS[(size_t)s].record.size();
    tb.max_rows = std::max(tb.max_rows, (int)ts.size()); tb.max_chunks = std::max(tb.max_chunks, (int)rows.size());
  }
  g_chunk_enc.clear();
  tb.backing.assign((size_t)tb.rec_off.back() / 8 + 64, 0);
  tb.arena = reinterpret_cast<uint8_t*>(tb.backing.data());
  for (int s = 0; s < ns; ++s) {
    std::memcpy(tb.arena + tb.rec_off[(size_t)s], tb.SS[(size_t)s].record.data(), tb.SS[(size_t)s].record.size());
    tb.max_rec = std::max<uint32_t>(tb.max_rec, (uint32_t)tb.SS[(size_t)s].record.size());
  }
}

template <typename F> static void by_sum_fn(int fn, F&& f) {
  if (fn == filo::FN_RATE) f(std::integral_constant<int, filo::FN_RATE>{});
  else if (fn == filo::FN_INCREASE) f(std::integral_constant<int, filo::FN_INCREASE>{});
  else if (fn == filo::FN_AVG) f(std::integral_constant<int, filo::FN_AVG>{});
  else if (fn == filo::FN_COUNT) f(std::integral_constant<int, filo::FN_COUNT>{});
  else f(std::integral_constant<int, filo::FN_SUM>{});
}
template <typename F> static void by_ctr_fn(int fn, F&& f) {
  if (fn == filo::FN_RATE) f(std::integral_constant<int, filo::FN_RATE>{});
  else if (fn == filo::FN_INCREASE) f(std::integral_constant<int, filo::FN_INCREASE>{});
  else f(std::integral_constant<int, filo::FN_DELTA>{});
}

int main(int argc, char** argv) {
  if (argc < 3) { std::printf("usage: scan_geometry_emul <seed> <cases file>\n"); return 2; }
  const uint64_t seed = std::strtoull(argv[1], nullptr, 10);
  cusim::rng_state() = seed;
  std::vector<GQuery> qs;
  if (!read_queries(argv[2], qs)) { std::printf("FAIL: cannot read %s\n", argv[2]); return 1; }
  std::mt19937_64 rng(9157);
  long checked = 0, runs = 0, accepted_wp = 0, declined_wp = 0;
  std::map<std::string, long> per_kernel;
  for (const GQuery& g : qs) {
    Table tb; build_table(rng, g, tb);
    const int ns = (int)g.series.size();
    for (int fn : g.fns) {
      filo::QueryParams q = g.q; q.fn = fn;
      const char* mode = q.inclusive ? "inclusive" : "exclusive";
      std::vector<double> ref((size_t)ns * q.T); int64_t exp_rows = 0, exp_bytes = 0;
      for (int s = 0; s < ns; ++s) {
        fo::Series os; for (auto& ch : tb.SS[(size_t)s].chunks) os.infos.push_back(ch->info.data());
        fo::QueryStats st;
        fo::periodicSamples(os, oracle_fn(fn), q.cumulative != 0, q.start, q.step, q.end, q.window, fo::QueryConfig{q.inclusive != 0}, ref.data() + (size_t)s * q.T, &st, 0, 0);
        exp_rows += st.samplesScanned; exp_bytes += st.bytesScanned;
      }
      const uint32_t wrows = (uint32_t)(q.window / q.step) + 1;
      const filo::TileSmem L = filo::tile_layout(tb.max_rec, (uint32_t)tb.max_rows, (uint32_t)q.T, 2 * wrows + 16);
      V2Shape sh{tb.max_rec, tb.max_rows, tb.max_chunks, false, false};        // the v2 kernel's scratch, as filo_query sizes it
      for (auto& S : tb.SS) { filo::RecordHeader h; std::memcpy(&h, S.record.data(), sizeof h); sh.any_nonconst_ts |= !(h.flags & filo::REC_ALL_TS_CONST); sh.any_drop |= (h.flags & filo::REC_ANY_DROP) != 0; }
      // one kernel run: launch(A) fills out / the fallback list, the declined series go through the v2 kernel, then every check
      auto check = [&](const char* kernel, const std::vector<int64_t>& want_declined, auto&& launch) -> bool {
        std::vector<double> out((size_t)ns * q.T, -777.0);
        std::vector<int64_t> flist((size_t)ns + 8, -1); unsigned long long fcount = 0, counters[2] = {0, 0}; int derr[4] = {0, 0, 0, 0};
        Launch A{tb.arena, tb.rec_off.data(), ns, q, out.data(), L, 2, flist.data(), &fcount, counters, derr, nullptr, nullptr, 0, 0, nullptr, nullptr};
        launch(A);
        if (derr[0]) { std::printf("FAIL %s %s fn %d on %s: device error %d\n", g.name.c_str(), mode, fn, kernel, derr[0]); return false; }
        std::vector<int64_t> got(flist.begin(), flist.begin() + (std::ptrdiff_t)std::min<unsigned long long>(fcount, flist.size()));
        std::sort(got.begin(), got.end());
        if (fcount != want_declined.size() || got != want_declined) {
          std::printf("FAIL %s %s fn %d T %d window %lld on %s: declined series", g.name.c_str(), mode, fn, q.T, (long long)q.window, kernel);
          for (int64_t x : got) std::printf(" %lld", (long long)x);
          std::printf(", predicted");
          for (int64_t x : want_declined) std::printf(" %lld", (long long)x);
          std::printf("\n");
          return false;
        }
        if (fcount) { run_v2(A, sh, flist.data(), &fcount); if (derr[0]) { std::printf("FAIL %s: device error %d (v2 fallback)\n", g.name.c_str(), derr[0]); return false; } }
        for (int s = 0; s < ns; ++s)
          for (int k = 0; k < q.T; ++k) {
            const double a = out[(size_t)s * q.T + k], r = ref[(size_t)s * q.T + k];
            if (!same_bits(a, r)) {
              std::printf("FAIL %s %s fn %d T %d window %lld on %s: series %d window %d: %.17g vs %.17g\n", g.name.c_str(), mode, fn, q.T, (long long)q.window, kernel, s, k, a, r);
              return false;
            }
            ++checked;
          }
        if ((int64_t)counters[0] != exp_rows || (int64_t)counters[1] != exp_bytes) {
          std::printf("FAIL %s %s fn %d on %s: scan counters %llu / %llu vs %lld / %lld\n", g.name.c_str(), mode, fn, kernel, counters[0], counters[1], (long long)exp_rows, (long long)exp_bytes);
          return false;
        }
        ++runs; ++per_kernel[kernel];
        return true;
      };
      if (!g.counter) {
        // scan_wp_batch_kernel: O on V where filo_query allows it (one pass of <= 64 blocks), and O apart
        const bool alias_ok = filo::wp_max_items((uint32_t)tb.max_chunks, (uint32_t)q.T, wrows) <= 64;
        const struct { uint32_t consumers, B, nbuf; const char* name; } shapes[] = {{3, 3, 2, "3/3/2"}, {filo::WP_BATCH_WARPS - 1, filo::WP_BATCH_SERIES, filo::WP_BATCH_BUFS, "product"}};
        for (bool alias : {true, false}) {
          if (alias && !alias_ok) continue;
          for (const auto& shp : shapes) {
            if (shp.B == filo::WP_BATCH_SERIES && !g.product) continue;
            const filo::WpBatchSmem W = filo::wp_batch_layout(tb.max_rec, (uint32_t)tb.max_rows, (uint32_t)tb.max_chunks, (uint32_t)q.T, wrows, alias, shp.B, shp.nbuf, shp.consumers);
            if ((size_t)W.total > sizeof(filo::smem)) continue;                  // (filo_query takes scan_wp_sum_kernel there)
            const std::string kn = std::string("batch ") + (alias ? "O on V " : "O apart ") + shp.name;
            if (!check(kn.c_str(), g.exp_wp, [&](Launch& A) {
                  by_sum_fn(fn, [&](auto fnc) {
                    cusim::launch(dim3((unsigned)A.grid), dim3((W.consumers + 1) * 32), [&] {
                      filo::scan_wp_batch_kernel<decltype(fnc)::value, filo::WP_BATCH_WARPS>(A.arena, A.rec_off, A.S, A.q, A.out, W, A.flist, A.fcount, A.counters, A.derr);
                    });
                  });
                })) return 1;
          }
        }
        // scan_wp_sum_kernel: one and two record buffers
        for (bool two : {false, true}) {
          filo::WpSmem W = filo::wp_layout(tb.max_rec, (uint32_t)tb.max_rows, (uint32_t)tb.max_chunks, (uint32_t)q.T, wrows, alias_ok, two);
          W.warps = 3;
          if ((size_t)W.per_warp * W.warps > sizeof(filo::smem)) { std::printf("FAIL %s: wp layout %u bytes per warp\n", g.name.c_str(), W.per_warp); return 1; }
          if (!check(two ? "sum two record buffers" : "sum one record buffer", g.exp_wp, [&](Launch& A) {
                by_sum_fn(fn, [&](auto fnc) {
                  cusim::launch(dim3((unsigned)A.grid), dim3(W.warps * 32), [&] {
                    filo::scan_wp_sum_kernel<decltype(fnc)::value, 16>(A.arena, A.rec_off, A.S, A.q, A.out, W, A.flist, A.fcount, A.counters, A.derr);
                  });
                });
              })) return 1;
        }
        // the tile kernel
        if (L.total > sizeof(filo::smem)) { std::printf("FAIL %s: tile layout %u bytes\n", g.name.c_str(), L.total); return 1; }
        if (!check("tile", g.exp_tile, [&](Launch& A) { dispatch<false>(A); })) return 1;
      } else {
        // scan_wp_ctr_kernel: the const-DDV instantiation, and the irregular-timestamp one (what a table with DDV timestamps runs)
        for (bool irr : {false, true}) {
          filo::WpCtrSmem W = filo::wp_ctr_layout(tb.max_rec, (uint32_t)tb.max_rows, (uint32_t)tb.max_chunks, (uint32_t)q.T, false, irr);
          W.warps = 3; W.tab = W.per_warp * W.warps;
          if ((size_t)W.tab + 4096 > sizeof(filo::smem)) { std::printf("FAIL %s: wp ctr layout %u bytes per warp\n", g.name.c_str(), W.per_warp); return 1; }
          if (!check(irr ? "ctr irregular" : "ctr const", irr ? g.exp_ctr_irr : g.exp_ctr_const, [&](Launch& A) {
                by_ctr_fn(fn, [&](auto fnc) {
                  cusim::launch(dim3((unsigned)A.grid), dim3(W.warps * 32), [&] {
                    if (W.tsr) filo::scan_wp_ctr_kernel<decltype(fnc)::value, false, 16, true>(A.arena, A.rec_off, A.S, A.q, A.out, W, A.flist, A.fcount, A.counters, A.derr, nullptr, nullptr, 0, 0, nullptr, nullptr);
                    else filo::scan_wp_ctr_kernel<decltype(fnc)::value, false, 16, false>(A.arena, A.rec_off, A.S, A.q, A.out, W, A.flist, A.fcount, A.counters, A.derr, nullptr, nullptr, 0, 0, nullptr, nullptr);
                  });
                });
              })) return 1;
        }
      }
    }
    if (!g.counter) { declined_wp += (long)g.exp_wp.size(); accepted_wp += ns - (long)g.exp_wp.size(); }
  }
  for (const auto& kv : per_kernel) std::printf("%s: %ld runs\n", kv.first.c_str(), kv.second);
  std::printf("v4 SUM kernels: %ld series taken, %ld declined, as predicted\n", accepted_wp, declined_wp);
  std::printf("OK %zu queries, %ld runs, %ld values bit-exact (schedule seed %llu)\n", qs.size(), runs, checked, (unsigned long long)seed);
  return 0;
}
