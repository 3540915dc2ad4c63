// The fused aggregate kernels at steady state on the cusim SIMT emulator: work items of seg in {1, 7, 9, 64, 256} series laid out by
// build_groups_new's rule over groups of mixed sizes (1, seg - 1, seg, seg + 1, 8 seg, 8 seg + 1, an empty group), on a grid of one or
// two CTAs so that every warp (counter kernel) or CTA (tile kernel) folds at least six items.  Declining series are planted at an item's
// first, middle and last series, twice in one item, in every series of an item, at the first series a warp takes, in a warp's last item,
// in two consecutive items of one warp, in the only item of a small group and in every item of one group.
// Kernels: scan_wp_ctr_kernel<AGG> (const-DDV and IRR instantiations) and scan_tile_kernel<AGG>, each with and without the moments row,
// scan_agg_kernel_v2 over the fallback list, merge_partials_kernel over every group.  Checked:
// - the fallback list, sorted, equals the items holding a planted series;
// - every item's partial row: counts exact; sums exact on integer gauges (tile), within gamma_{m-1} * sum|v| of an exact sum on counters;
// - every group's merged row the same way, against a fold of the oracle's per-series rows;
// - samples_scanned / bytes_scanned equal the oracle's.
// Test infrastructure: built and run by tests/test_agg_items_emul.py.  The series builders and launch helpers are tile_emul.cpp's.
//   agg_items_emul [seed [variant]]     seed 0 = round-robin schedule, otherwise a pseudo-random fiber schedule; variant: run only the
//                                       variants whose name starts with it (ctr, tile)
#define main tile_emul_main
#include "tile_emul.cpp"
#undef main
#include <algorithm>
#include <set>

enum { OKS = 0, C_CHUNKS5 = 1, C_DDV = 2, C_RESETS = 3, C_JITTER = 4 };

static void run_agg_v2_any(const Launch& A, const V2Shape& sh, const int64_t* list, const unsigned long long* list_count, bool mom) {
  const bool need_corr2 = (A.q.fn == filo::FN_RATE || A.q.fn == filo::FN_INCREASE) && A.q.cumulative && sh.any_drop;
  uint32_t scratch = filo::align_up((uint32_t)sh.max_chunks * (uint32_t)filo::CHUNK_DESC_BYTES, 16) +
                     ((uint32_t)sh.max_rows + (uint32_t)sh.max_chunks * 8u) * 8u * (1u + (sh.any_nonconst_ts ? 1u : 0u) + (need_corr2 ? 1u : 0u));
  scratch = filo::align_up(scratch + 16, 128);                                   // as filo_query sizes it (capi.cu)
  const uint32_t rec_cap = filo::align_up(sh.max_rec + 16, 128), acc_bytes = filo::align_up((uint32_t)A.q.T * (mom ? 20u : 12u), 128);
  const size_t smem_bytes = (size_t)(filo::WARP_HDR_BYTES + rec_cap + filo::STAGE_BYTES + acc_bytes + scratch) * filo::FAST_WARPS;
  if (smem_bytes > sizeof(filo::smem)) { std::printf("FAIL: agg v2 shared memory %zu\n", smem_bytes); std::exit(1); }
  auto body = [&](auto cls) {
    cusim::launch(dim3((unsigned)A.grid), dim3(filo::FAST_WARPS * 32), [&] {
      if (mom) filo::scan_agg_kernel_v2<decltype(cls)::value, true>(A.arena, A.rec_off, A.order, A.item_begin, A.n_items, A.q, A.agg_op, A.pval, A.pcnt, rec_cap, scratch,
                                                                    acc_bytes, A.counters, A.derr, list, list_count);
      else filo::scan_agg_kernel_v2<decltype(cls)::value>(A.arena, A.rec_off, A.order, A.item_begin, A.n_items, A.q, A.agg_op, A.pval, A.pcnt, rec_cap, scratch, acc_bytes,
                                                          A.counters, A.derr, list, list_count);
    });
  };
  if (filo::fn_class_of(A.q.fn, A.q.cumulative, A.q.long_values) == filo::CLASS_COUNTER) body(std::integral_constant<int, filo::CLASS_COUNTER>{});
  else body(std::integral_constant<int, filo::CLASS_SUM>{});
}

// a sum's reference: exact (binary128) and the bound any order of m double additions keeps, gamma_{m-1} * sum |v|; a sum of m rounded
// squares keeps gamma_m * sum v^2
struct Ref { __float128 s = 0; double abs = 0; uint32_t n = 0; };
static bool within(double got, const Ref& r, bool squares = false) {
  const uint32_t m = squares ? r.n : (r.n ? r.n - 1 : 0);
  if (m == 0) return same_bits(got, (double)r.s);
  const double u = std::ldexp(1.0, -53), g = m * u / (1 - m * u);
  return std::fabs((double)((__float128)got - r.s)) <= g * r.abs * (1 + 4 * u);
}

struct Variant { const char* name; bool ctr, irr, mom; int fn; };

int main(int argc, char** argv) {
  const uint64_t seed = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 0;
  cusim::rng_state() = seed;
  const Variant variants[] = {
    {"ctr const-DDV", true, false, false, filo::FN_RATE}, {"ctr const-DDV moments", true, false, true, filo::FN_INCREASE},
    {"ctr IRR", true, true, false, filo::FN_INCREASE},    {"ctr IRR moments", true, true, true, filo::FN_RATE},
    {"tile", false, false, false, filo::FN_SUM},          {"tile moments", false, false, true, filo::FN_SUM},
  };
  const int segs[] = {1, 7, 9, 64, 256};
  const int64_t t0 = 1700000000000LL; const int step_ms = 15000, ROWS = 60;
  long checked = 0; int cases = 0;
  const std::string only = argc > 2 ? argv[2] : "";
  for (const Variant& V : variants) {
    if (std::string(V.name).compare(0, only.size(), only) != 0) continue;
    for (int seg : segs) {
      for (int grouped = 1; grouped >= 0; --grouped) {
        if (!grouped && seg != 9) continue;                       // the ungrouped table (order == nullptr) at one seg
        std::mt19937_64 rng(seed * 131 + (uint64_t)seg * 7 + (V.ctr ? 1 : 0) + (V.irr ? 2 : 0) + (V.mom ? 4 : 0) + (uint64_t)grouped * 1000);
        // workers: warps * grid (ctr, 3 warps per CTA below seg 64, fewer above) or grid (tile)
        const int warps = seg >= 256 ? 1 : seg >= 64 ? 2 : 3, grid = seg >= 64 ? 1 : 2;
        const int workers = V.ctr ? warps * grid : grid;
        // group sizes: 1, seg - 1, seg, seg + 1, 8 seg, 8 seg + 1, empty, then mixed sizes until every worker has >= 6 items
        std::vector<int> sizes;
        if (grouped) {
          for (int x : {1, seg - 1, seg, seg + 1, 8 * seg, 8 * seg + 1, 0}) if (x >= 0 && (seg <= 64 || x <= seg + 1)) sizes.push_back(x);
          auto items_of = [&]() { int64_t n = 0; for (int x : sizes) n += (x + seg - 1) / seg; return n; };
          while (items_of() < 6 * workers + 3) sizes.push_back(1 + (int)(rng() % (uint64_t)(3 * seg)));
        } else sizes.push_back(6 * workers * seg + seg / 2 + 1);
        const int G = (int)sizes.size();
        std::vector<int32_t> gid;
        for (int g = 0; g < G; ++g) for (int i = 0; i < sizes[(size_t)g]; ++i) gid.push_back(g);
        std::shuffle(gid.begin(), gid.end(), rng);                // ids interleaved: `order` gathers are scattered
        const int64_t S = (int64_t)gid.size();
        // build_groups_new: stable sort by group id, seg consecutive positions of one group per item
        std::vector<int32_t> order((size_t)S); for (int64_t s = 0; s < S; ++s) order[(size_t)s] = (int32_t)s;
        std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return gid[(size_t)a] < gid[(size_t)b]; });
        std::vector<int64_t> gstart((size_t)G + 1, 0), gis((size_t)G + 1, 0), item_begin;
        for (int g = 0; g < G; ++g) gstart[(size_t)g + 1] = gstart[(size_t)g] + sizes[(size_t)g];
        for (int g = 0; g < G; ++g) { gis[(size_t)g + 1] = gis[(size_t)g] + (sizes[(size_t)g] + seg - 1) / seg; for (int64_t p = gstart[(size_t)g]; p < gstart[(size_t)g + 1]; p += seg) item_begin.push_back(p); }
        item_begin.push_back(S);
        const int64_t n_items = (int64_t)item_begin.size() - 1;
        for (int w = 0; w < workers; ++w) if ((n_items - w + workers - 1) / workers < 6) { std::printf("FAIL: worker %d has fewer than 6 items\n", w); return 1; }
        // planted declines, by position in `order`
        std::vector<int> cause((size_t)S, OKS);
        const std::vector<int> causes = V.ctr ? (V.fn == filo::FN_DELTA ? std::vector<int>{C_CHUNKS5, C_DDV} : std::vector<int>{C_CHUNKS5, C_DDV, C_RESETS})
                                              : std::vector<int>{C_JITTER, C_DDV, C_CHUNKS5};
        int nc = 0;
        auto plant = [&](int64_t pos) { if (pos >= 0 && pos < S && cause[(size_t)order[(size_t)pos]] == OKS) cause[(size_t)order[(size_t)pos]] = causes[(size_t)(nc++ % causes.size())]; };
        auto ib = [&](int64_t it) { return item_begin[(size_t)it]; };
        auto ie = [&](int64_t it) { return item_begin[(size_t)it + 1]; };
        std::vector<int64_t> big;                                  // items of at least 3 series
        for (int64_t it = 0; it < n_items; ++it) if (ie(it) - ib(it) >= 3) big.push_back(it);
        if (big.size() >= 4) {
          plant(ib(big[0]));                                       // first series of an item
          plant((ib(big[1]) + ie(big[1])) / 2);                    // a middle one
          plant(ie(big[2]) - 1);                                   // the last one
          plant(ib(big[3])); plant(ie(big[3]) - 1);                // two in one item
        }
        { const int64_t it = n_items / 2; for (int64_t p = ib(it); p < ie(it); ++p) plant(p); }      // every series of an item
        plant(ib(workers > 1 ? 1 : 0));                            // the first series worker 1 (or 0) takes
        { const int64_t w = workers - 1, last = w + ((n_items - 1 - w) / workers) * workers; plant(ie(last) - 1); }   // worker's last item
        { const int64_t it = 2 * workers + (workers > 1 ? 1 : 0); plant(ib(it)); plant(ib(it + workers) + (ie(it + workers) - ib(it + workers)) / 2); }  // it, it + workers
        if (grouped) {
          plant(gstart[0]);                                        // the only item of the group of one series
          for (int g = 0; g < G; ++g)                              // every item of one group of several items
            if (gis[(size_t)g + 1] - gis[(size_t)g] >= 2 && g != 0) { for (int64_t it = gis[(size_t)g]; it < gis[(size_t)g + 1]; ++it) plant(ib(it) + (it % 3) * (ie(it) - ib(it) - 1) / 2); break; }
        }
        std::set<int64_t> bad;
        for (int64_t it = 0; it < n_items; ++it) for (int64_t p = ib(it); p < ie(it); ++p) if (cause[(size_t)order[(size_t)p]] != OKS) bad.insert(it);
        // series
        std::vector<SeriesData> SS((size_t)S);
        std::vector<int64_t> rec_off((size_t)S + 1, 0);
        bool any_irr = false, any_drop = false; int max_chunks = 0;
        for (int64_t s = 0; s < S; ++s) {
          const int c = cause[(size_t)s];
          const bool jit = c == C_JITTER || (V.irr && s % 3 == 1);
          std::vector<int64_t> ts((size_t)ROWS); std::vector<double> v((size_t)ROWS);
          for (int r = 0; r < ROWS; ++r) ts[(size_t)r] = t0 + (int64_t)r * step_ms + (jit ? (int64_t)(rng() % 4001) - 2000 : 0);
          double acc = 1000.0 + (double)(rng() % 1000);
          for (int r = 0; r < ROWS; ++r) {
            const double inc = (double)(rng() % 40);
            if (V.ctr) { acc += inc; if ((c == C_RESETS && r < 36 && r % 3 == 2) || (c == OKS && r == 17 && s % 5 == 0)) acc = inc; v[(size_t)r] = acc; }
            else v[(size_t)r] = inc - 12.0;                        // integers: window and item sums are exact in any order
          }
          const std::vector<int> chunks = c == C_CHUNKS5 ? std::vector<int>{12, 12, 12, 12, 12} : std::vector<int>{36, 24};
          g_chunk_enc = c == C_DDV ? "xr" : "";                   // 'r': DoubleVector.optimize, which makes integral values a DDV vector
          build_series_from(SS[(size_t)s], rng, ts, v, chunks, V.ctr ? 1 : 0, true, 0);
          g_chunk_enc.clear();
          rec_off[(size_t)s + 1] = rec_off[(size_t)s] + (int64_t)SS[(size_t)s].record.size();
          filo::RecordHeader h; std::memcpy(&h, SS[(size_t)s].record.data(), sizeof h);
          any_irr |= !(h.flags & filo::REC_ALL_TS_CONST); any_drop |= (h.flags & filo::REC_ANY_DROP) != 0;
          max_chunks = std::max(max_chunks, (int)chunks.size());
        }
        if (V.irr != any_irr && V.ctr) { std::printf("FAIL %s seg %d: the table's timestamps do not select the %s instantiation\n", V.name, seg, V.irr ? "IRR" : "const-DDV"); return 1; }
        std::vector<uint64_t> arena_backing((size_t)rec_off.back() / 8 + 64, 0);
        uint8_t* arena = reinterpret_cast<uint8_t*>(arena_backing.data());
        uint32_t max_rec = 0;
        for (int64_t s = 0; s < S; ++s) { std::memcpy(arena + rec_off[(size_t)s], SS[(size_t)s].record.data(), SS[(size_t)s].record.size()); max_rec = std::max<uint32_t>(max_rec, (uint32_t)SS[(size_t)s].record.size()); }
        filo::QueryParams q{};
        q.start = t0 + 75000; q.step = step_ms; q.end = t0 + (int64_t)(ROWS - 1) * step_ms; q.window = 75000;
        q.T = (int)((q.end - q.start) / q.step) + 1;
        q.fn = V.fn; q.cumulative = V.ctr ? 1 : 0; q.inclusive = 1;
        const uint32_t wrows = (uint32_t)(q.window / q.step) + 1;
        // oracle, per series
        std::vector<double> ref((size_t)S * q.T); int64_t exp_rows = 0, exp_bytes = 0;
        for (int64_t s = 0; s < S; ++s) {
          fo::Series os; for (auto& ch : SS[(size_t)s].chunks) os.infos.push_back(ch->info.data());
          fo::QueryStats st;
          fo::periodicSamples(os, oracle_fn(q.fn), q.cumulative != 0, q.start, q.step, q.end, q.window, fo::QueryConfig{true}, ref.data() + (size_t)s * q.T, &st, 0, 0);
          exp_rows += st.samplesScanned; exp_bytes += st.bytesScanned;
        }
        const int nparts = V.mom ? 2 : 1;
        std::vector<double> pval((size_t)nparts * n_items * q.T, -777.0); std::vector<uint32_t> pcnt((size_t)n_items * q.T, 12345u);
        std::vector<int64_t> flist((size_t)n_items + 8, -1); unsigned long long fcount = 0, counters[2] = {0, 0}; int derr[4] = {0, 0, 0, 0};
        const filo::TileSmem L = filo::tile_layout(max_rec, (uint32_t)ROWS, (uint32_t)q.T, 2 * wrows + 16);
        Launch A{arena, rec_off.data(), S, q, nullptr, L, grid, flist.data(), &fcount, counters, derr, grouped ? order.data() : nullptr, item_begin.data(), n_items,
                 filo::AGG_SUM, pval.data(), pcnt.data()};
        if (V.ctr) {
          filo::WpCtrSmem W = filo::wp_ctr_layout(max_rec, (uint32_t)ROWS, (uint32_t)max_chunks, (uint32_t)q.T, true, V.irr, V.mom);
          W.warps = (uint32_t)warps; W.tab = W.per_warp * W.warps;
          if ((size_t)W.tab + 4096 > sizeof(filo::smem)) { std::printf("FAIL: wp ctr layout %u bytes per warp\n", W.per_warp); return 1; }
          auto body = [&](auto fnc, auto irr, auto mom) {
            cusim::launch(dim3((unsigned)A.grid), dim3(W.warps * 32), [&] {
              filo::scan_wp_ctr_kernel<decltype(fnc)::value, true, 16, decltype(irr)::value, decltype(mom)::value>(A.arena, A.rec_off, A.S, A.q, nullptr, W, A.flist, A.fcount,
                  A.counters, A.derr, A.order, A.item_begin, A.n_items, A.agg_op, A.pval, A.pcnt);
            });
          };
          auto by_mom = [&](auto fnc, auto irr) { if (V.mom) body(fnc, irr, std::true_type{}); else body(fnc, irr, std::false_type{}); };
          auto by_irr = [&](auto fnc) { if (W.tsr) by_mom(fnc, std::true_type{}); else by_mom(fnc, std::false_type{}); };
          if (q.fn == filo::FN_RATE) by_irr(std::integral_constant<int, filo::FN_RATE>{});
          else by_irr(std::integral_constant<int, filo::FN_INCREASE>{});
        } else {
          if (L.total > sizeof(filo::smem)) { std::printf("FAIL: layout %u bytes\n", L.total); return 1; }
          cusim::launch(dim3((unsigned)A.grid), dim3(filo::TILE_LAUNCH_THREADS), [&] {
            if (V.mom) filo::scan_tile_kernel<filo::FN_SUM, true, true>(A.arena, A.rec_off, A.S, A.q, nullptr, A.L, A.flist, A.fcount, A.counters, A.derr, A.order, A.item_begin, A.n_items, A.agg_op, A.pval, A.pcnt);
            else filo::scan_tile_kernel<filo::FN_SUM, true>(A.arena, A.rec_off, A.S, A.q, nullptr, A.L, A.flist, A.fcount, A.counters, A.derr, A.order, A.item_begin, A.n_items, A.agg_op, A.pval, A.pcnt);
          });
        }
        const char* what = V.name;
        if (derr[0]) { std::printf("FAIL %s seg %d: device error %d\n", what, seg, derr[0]); return 1; }
        std::vector<int64_t> got_list(flist.begin(), flist.begin() + (std::ptrdiff_t)fcount); std::sort(got_list.begin(), got_list.end());
        const std::vector<int64_t> want(bad.begin(), bad.end());
        if (got_list != want) {
          std::printf("FAIL %s seg %d grouped %d: fallback list of %zu items, predicted %zu:", what, seg, grouped, got_list.size(), want.size());
          for (size_t i = 0; i < std::max(got_list.size(), want.size()) && i < 12; ++i)
            std::printf(" %lld/%lld", i < got_list.size() ? (long long)got_list[i] : -1LL, i < want.size() ? (long long)want[i] : -1LL);
          std::printf("\n"); return 1;
        }
        // the scan counters before the fallback pass: the good items' series only
        { int64_t good_rows = 0;
          for (int64_t it = 0; it < n_items; ++it) if (!bad.count(it)) for (int64_t p = ib(it); p < ie(it); ++p) {
            const int64_t s = grouped ? order[(size_t)p] : p;
            fo::Series os; for (auto& ch : SS[(size_t)s].chunks) os.infos.push_back(ch->info.data());
            fo::QueryStats st; std::vector<double> tmp((size_t)q.T);
            fo::periodicSamples(os, oracle_fn(q.fn), q.cumulative != 0, q.start, q.step, q.end, q.window, fo::QueryConfig{true}, tmp.data(), &st, 0, 0);
            good_rows += st.samplesScanned; }
          if ((int64_t)counters[0] != good_rows) { std::printf("FAIL %s seg %d: samples_scanned of the good items %llu vs %lld\n", what, seg, counters[0], (long long)good_rows); return 1; } }
        if (fcount) {
          V2Shape sh{max_rec, ROWS, max_chunks, any_irr, any_drop};
          Launch F = A; F.grid = 2;
          run_agg_v2_any(F, sh, flist.data(), &fcount, V.mom);
          if (derr[0]) { std::printf("FAIL %s seg %d: device error %d (fused fallback)\n", what, seg, derr[0]); return 1; }
        }
        if ((int64_t)counters[0] != exp_rows || (int64_t)counters[1] != exp_bytes) {
          std::printf("FAIL %s seg %d: scan counters (%llu, %llu) vs the oracle's (%lld, %lld)\n", what, seg, counters[0], counters[1], (long long)exp_rows, (long long)exp_bytes);
          return 1;
        }
        // every item's partial row (Σv, n; Σv² with moments)
        for (int64_t it = 0; it < n_items; ++it) {
          for (int k = 0; k < q.T; ++k) {
            Ref a, a2;
            for (int64_t p = ib(it); p < ie(it); ++p) {
              const double v = ref[(size_t)(grouped ? order[(size_t)p] : p) * q.T + k];
              if (v == v) { a.s += v; a.abs += std::fabs(v); a2.s += (__float128)v * v; a2.abs += v * v; ++a.n; ++a2.n; }
            }
            const size_t o = (size_t)it * q.T + k;
            const bool ok_v = V.ctr ? within(pval[o], a) : same_bits(pval[o], (double)a.s);
            const bool ok_v2 = !V.mom || (V.ctr ? within(pval[(size_t)(n_items + it) * q.T + k], a2, true) : same_bits(pval[(size_t)(n_items + it) * q.T + k], (double)a2.s));
            if (!ok_v || !ok_v2 || pcnt[o] != a.n) {
              std::printf("FAIL %s seg %d grouped %d item %lld (%s) window %d: (%.17g, %u) vs (%.17g, %u)\n", what, seg, grouped, (long long)it, bad.count(it) ? "fallback" : "fused", k,
                          pval[o], pcnt[o], (double)a.s, a.n);
              return 1;
            }
            ++checked;
          }
        }
        // merge_partials_kernel over every group: Σv (and Σv²) and n of the group's series
        {
          const int ktiles = (q.T + 31) / 32;
          const int op = V.mom ? filo::AGG_STDVAR : filo::AGG_SUM;
          std::vector<double> mv((size_t)nparts * G * q.T, -777.0); std::vector<int64_t> mc((size_t)G * q.T, -1);
          cusim::launch(dim3((unsigned)(G * ktiles)), dim3(256), [&] {
            if (V.mom) filo::merge_partials_kernel<filo::MERGE_MOMENTS>(pval.data(), pcnt.data(), gis.data(), G, q.T, op, 1, mv.data(), mc.data());
            else filo::merge_partials_kernel(pval.data(), pcnt.data(), gis.data(), G, q.T, op, 1, mv.data(), mc.data());
          });
          for (int g = 0; g < G; ++g) {
            for (int k = 0; k < q.T; ++k) {
              Ref a, a2;
              for (int64_t p = gstart[(size_t)g]; p < gstart[(size_t)g + 1]; ++p) {
                const double v = ref[(size_t)(grouped ? order[(size_t)p] : p) * q.T + k];
                if (v == v) { a.s += v; a.abs += std::fabs(v); a2.s += (__float128)v * v; a2.abs += v * v; ++a.n; ++a2.n; }
              }
              const size_t o = (size_t)g * q.T + k;
              const bool ok_v = V.ctr ? within(mv[o], a) : same_bits(mv[o], (double)a.s);
              const bool ok_v2 = !V.mom || (V.ctr ? within(mv[(size_t)G * q.T + o], a2, true) : same_bits(mv[(size_t)G * q.T + o], (double)a2.s));
              if (!ok_v || !ok_v2 || mc[o] != (int64_t)a.n) {
                std::printf("FAIL %s seg %d grouped %d merged group %d (%d series) window %d: (%.17g, %lld) vs (%.17g, %u)\n", what, seg, grouped, g, sizes[(size_t)g], k,
                            mv[o], (long long)mc[o], (double)a.s, a.n);
                return 1;
              }
              ++checked;
            }
          }
        }
        std::printf("%s seg %d%s: %lld series, %d groups, %lld items over %d %s, %zu to the fallback list\n", what, seg, grouped ? "" : " ungrouped", (long long)S, G,
                    (long long)n_items, workers, V.ctr ? "warps" : "CTAs", want.size());
        ++cases;
      }
    }
  }
  std::printf("OK %d cases, %ld cells checked (schedule seed %llu)\n", cases, checked, (unsigned long long)seed);
  return 0;
}
