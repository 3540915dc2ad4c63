// stddev / stdvar / group across series: the moments mode of the fused scan kernels (scan_tile_kernel<FN, true, true>,
// scan_wp_ctr_kernel<FN, true, NW, IRR, true>, scan_agg_kernel_v2<CLS, true>) and the merge / presentation kernels, compiled for the
// host on the cusim SIMT emulator.  Every (item, window) Σv, Σv² and count is checked bit-exact against the oracle's per-series rows
// folded in the item's series order; the merged and presented rows against the same fixed 8-lane tree on the host.
// Test infrastructure: built and run by tests/test_agg_moments.py.  The series builders and launch helpers are tile_emul.cpp's.
//   moments_emul [seed]     seed 0 = round-robin schedule, otherwise a pseudo-random fiber schedule
#define main tile_emul_main
#include "tile_emul.cpp"
#undef main

// the moments fallback: scan_agg_kernel_v2<CLS, true> over the listed items (a [T] Σv² row in the warp's accumulators)
static void run_agg_v2_mom(const Launch& A, const V2Shape& sh, const int64_t* list, const unsigned long long* list_count) {
  const bool need_corr2 = (A.q.fn == filo::FN_RATE || A.q.fn == filo::FN_INCREASE) && A.q.cumulative && sh.any_drop;
  uint32_t scratch = filo::align_up((uint32_t)sh.max_chunks * (uint32_t)filo::CHUNK_DESC_BYTES, 16) +
                     ((uint32_t)sh.max_rows + (uint32_t)sh.max_chunks * 8u) * 8u * (1u + (sh.any_nonconst_ts ? 1u : 0u) + (need_corr2 ? 1u : 0u));
  scratch = filo::align_up(scratch + 16, 128);
  const uint32_t rec_cap = filo::align_up(sh.max_rec + 16, 128), acc_bytes = filo::align_up((uint32_t)A.q.T * 20u, 128);      // as filo_query sizes it
  const size_t smem_bytes = (size_t)(filo::WARP_HDR_BYTES + rec_cap + filo::STAGE_BYTES + acc_bytes + scratch) * filo::FAST_WARPS;
  if (smem_bytes > sizeof(filo::smem)) { std::printf("FAIL: agg v2 shared memory %zu\n", smem_bytes); std::exit(1); }
  auto body = [&](auto cls) {
    cusim::launch(dim3((unsigned)A.grid), dim3(filo::FAST_WARPS * 32), [&] {
      filo::scan_agg_kernel_v2<decltype(cls)::value, true>(A.arena, A.rec_off, A.order, A.item_begin, A.n_items, A.q, filo::AGG_SUM, A.pval, A.pcnt, rec_cap, scratch, acc_bytes,
                                                           A.counters, A.derr, list, list_count);
    });
  };
  switch (filo::fn_class_of(A.q.fn, A.q.cumulative, A.q.long_values)) {
    case filo::CLASS_SUM: body(std::integral_constant<int, filo::CLASS_SUM>{}); break;
    case filo::CLASS_MINMAX: body(std::integral_constant<int, filo::CLASS_MINMAX>{}); break;
    case filo::CLASS_COUNTER: body(std::integral_constant<int, filo::CLASS_COUNTER>{}); break;
    default: body(std::integral_constant<int, filo::CLASS_POINT>{}); break;
  }
}

// present_cell on the host (the presentation rules of include/filo_b200.h)
static double host_present(int op, double s, double s2, unsigned long long c) {
  if (c == 0) return std::nan("");
  if (op == filo::AGG_GROUP) return 1.0;
  const double m = s / (double)c, var = s2 / (double)c - m * m;
  if (op == filo::AGG_STDVAR) return var;
  if (var < 0.0) return var == -INFINITY ? INFINITY : std::nan("");
  return var == 0.0 ? 0.0 : std::sqrt(var);
}

int main(int argc, char** argv) {
  const uint64_t seed = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 0;
  cusim::rng_state() = seed;
  std::mt19937_64 rng(9191);
  enum { K_TILE = 0, K_CTR = 1, K_V2 = 2 };
  struct MCfg { int kernel; int kind; bool xor_enc; int fn; std::vector<int> chunks; int nan_ppm, reset_every; int64_t window; int nser, per_item, jitter, grid; };
  const std::vector<MCfg> cfgs = {
    {K_TILE, 0, true, filo::FN_SUM, {400, 80}, 300000, 0, 300000, 26, 9, 0, 2},        // gauge sum_over_time, NaN markers, items of two tiles
    {K_TILE, 0, true, filo::FN_RATE, {150, 90}, 0, 0, 300000, 17, 17, 0, 1},           // delta-temporality rate, one item of three tiles
    {K_TILE, 0, false, filo::FN_AVG, {200, 40}, 100000, 0, 120000, 11, 4, 0, 3},       // raw f64 vectors
    {K_TILE, 0, true, filo::FN_COUNT, {100, 50, 50, 50, 50}, 0, 0, 300000, 12, 5, 0, 2}, // five chunks: every item declined -> v2
    {K_TILE, 0, true, filo::FN_SUM, {200, 100}, 0, 0, 300000, 10, 3, 3000, 2},         // irregular scrapes: declined -> v2
    {K_CTR, 1, true, filo::FN_RATE, {400, 80}, 200000, 61, 300000, 13, 5, 0, 2},       // counter rate: resets (drop lists) + NaN markers
    {K_CTR, 1, true, filo::FN_INCREASE, {120, 120, 60}, 0, 41, 60000, 12, 12, 0, 1},  // one item, three chunks
    {K_CTR, 1, false, filo::FN_DELTA, {200, 100}, 0, 0, 300000, 9, 4, 0, 2},           // raw vectors
    {K_CTR, 1, true, filo::FN_RATE, {240, 240}, 100000, 97, 300000, 11, 4, 3000, 2},   // irregular timestamps (IRR instantiation)
    {K_CTR, 1, true, filo::FN_RATE, {150, 90}, 0, 7, 300000, 10, 5, 0, 2},            // frequent resets: drop-list overflow -> v2
    {K_V2, 0, true, filo::FN_MAX, {150, 90}, 100000, 0, 300000, 9, 4, 0, 2},           // max_over_time: the v2 kernel only
    {K_V2, 0, true, filo::FN_LAST, {200, 40}, 50000, 0, 300000, 7, 3, 4000, 1},        // last sample, jittered timestamps
  };
  long checked = 0; int cases = 0;
  for (size_t ci = 0; ci < cfgs.size(); ++ci) {
    const MCfg& c = cfgs[ci];
    int rows = 0; for (int n : c.chunks) rows += n;
    const int64_t t0 = 1700000000000LL; const int step_ms = 15000;
    std::vector<SeriesData> SS((size_t)c.nser);
    std::vector<int64_t> rec_off((size_t)c.nser + 1, 0);
    g_jitter_ms = c.jitter; g_integral = false; g_long_col = 0;
    for (int s = 0; s < c.nser; ++s) {
      build_series(SS[(size_t)s], rng, rows, c.chunks, t0, step_ms, c.kind, c.xor_enc, c.nan_ppm, c.reset_every);
      rec_off[(size_t)s + 1] = rec_off[(size_t)s] + (int64_t)SS[(size_t)s].record.size();
    }
    std::vector<uint64_t> arena_backing((size_t)rec_off.back() / 8 + 64, 0);
    uint8_t* arena = reinterpret_cast<uint8_t*>(arena_backing.data());
    uint32_t max_rec = 0;
    for (int s = 0; s < c.nser; ++s) { std::memcpy(arena + rec_off[(size_t)s], SS[(size_t)s].record.data(), SS[(size_t)s].record.size()); max_rec = std::max<uint32_t>(max_rec, (uint32_t)SS[(size_t)s].record.size()); }
    filo::QueryParams q{};
    q.start = t0; q.step = 15000; q.end = t0 + (int64_t)(rows - 1) * step_ms; q.window = c.window;
    q.T = (int)((q.end - q.start) / q.step) + 1;
    q.fn = c.fn; q.cumulative = c.kind == 1; q.inclusive = 1;
    const uint32_t wrows = (uint32_t)(q.window / q.step) + 1;
    const filo::TileSmem L = filo::tile_layout(max_rec, (uint32_t)rows, (uint32_t)q.T, 2 * wrows + 16);
    std::vector<double> ref((size_t)c.nser * q.T);
    for (int s = 0; s < c.nser; ++s) {
      fo::Series os; for (auto& ch : SS[(size_t)s].chunks) os.infos.push_back(ch->info.data());
      fo::QueryStats st;
      fo::periodicSamples(os, oracle_fn(q.fn), q.cumulative != 0, q.start, q.step, q.end, q.window, fo::QueryConfig{true}, ref.data() + (size_t)s * q.T, &st, 0, 0);
    }
    // items of per_item series in a shuffled order (one group, as build_groups lays it out)
    std::vector<int32_t> order((size_t)c.nser); for (int s = 0; s < c.nser; ++s) order[(size_t)s] = s;
    std::shuffle(order.begin(), order.end(), rng);
    std::vector<int64_t> item_begin; for (int64_t p = 0; p < c.nser; p += c.per_item) item_begin.push_back(p); item_begin.push_back(c.nser);
    const int64_t n_items = (int64_t)item_begin.size() - 1;
    std::vector<double> pval((size_t)2 * n_items * q.T, -777.0); std::vector<uint32_t> pcnt((size_t)n_items * q.T, 12345u);
    std::vector<int64_t> flist((size_t)n_items + 8, -1); unsigned long long fcount = 0, counters[2] = {0, 0}; int derr[4] = {0, 0, 0, 0};
    Launch A{arena, rec_off.data(), c.nser, q, nullptr, L, c.grid, flist.data(), &fcount, counters, derr, order.data(), item_begin.data(), n_items, filo::AGG_SUM, pval.data(), pcnt.data()};
    V2Shape sh{max_rec, rows, (int)c.chunks.size(), false, false};
    for (auto& S : SS) { filo::RecordHeader h; std::memcpy(&h, S.record.data(), sizeof h); sh.any_nonconst_ts |= !(h.flags & filo::REC_ALL_TS_CONST); sh.any_drop |= (h.flags & filo::REC_ANY_DROP) != 0; }
    if (c.kernel == K_TILE) {
      if (L.total > sizeof(filo::smem)) { std::printf("FAIL: layout %u bytes\n", L.total); return 1; }
      auto body = [&](auto fnc) {
        cusim::launch(dim3((unsigned)A.grid), dim3(filo::TILE_LAUNCH_THREADS), [&] {
          filo::scan_tile_kernel<decltype(fnc)::value, true, true>(A.arena, A.rec_off, A.S, A.q, nullptr, A.L, A.flist, A.fcount, A.counters, A.derr, A.order, A.item_begin, A.n_items, A.agg_op, A.pval, A.pcnt);
        });
      };
      if (q.fn == filo::FN_RATE) body(std::integral_constant<int, filo::FN_RATE>{});
      else if (q.fn == filo::FN_AVG) body(std::integral_constant<int, filo::FN_AVG>{});
      else if (q.fn == filo::FN_COUNT) body(std::integral_constant<int, filo::FN_COUNT>{});
      else body(std::integral_constant<int, filo::FN_SUM>{});
    } else if (c.kernel == K_CTR) {
      filo::WpCtrSmem W = filo::wp_ctr_layout(max_rec, (uint32_t)rows, (uint32_t)c.chunks.size(), (uint32_t)q.T, true, c.jitter != 0, true);
      W.warps = 3; W.tab = W.per_warp * W.warps;
      if ((size_t)W.tab + 4096 > sizeof(filo::smem)) { std::printf("FAIL: wp ctr layout %u bytes per warp\n", W.per_warp); return 1; }
      auto body = [&](auto fnc) {
        cusim::launch(dim3((unsigned)A.grid), dim3(W.warps * 32), [&] {
          if (W.tsr) filo::scan_wp_ctr_kernel<decltype(fnc)::value, true, 16, true, true>(A.arena, A.rec_off, A.S, A.q, nullptr, W, A.flist, A.fcount, A.counters, A.derr, A.order, A.item_begin, A.n_items, A.agg_op, A.pval, A.pcnt);
          else filo::scan_wp_ctr_kernel<decltype(fnc)::value, true, 16, false, true>(A.arena, A.rec_off, A.S, A.q, nullptr, W, A.flist, A.fcount, A.counters, A.derr, A.order, A.item_begin, A.n_items, A.agg_op, A.pval, A.pcnt);
        });
      };
      if (q.fn == filo::FN_RATE) body(std::integral_constant<int, filo::FN_RATE>{});
      else if (q.fn == filo::FN_INCREASE) body(std::integral_constant<int, filo::FN_INCREASE>{});
      else body(std::integral_constant<int, filo::FN_DELTA>{});
    } else run_agg_v2_mom(A, sh, nullptr, nullptr);
    if (derr[0]) { std::printf("FAIL cfg %zu: device error %d\n", ci, derr[0]); return 1; }
    if (fcount) {
      run_agg_v2_mom(A, sh, flist.data(), &fcount);
      if (derr[0]) { std::printf("FAIL cfg %zu: device error %d (fused fallback)\n", ci, derr[0]); return 1; }
    }
    if (c.chunks.size() > 4 && fcount != (unsigned long long)n_items) { std::printf("FAIL cfg %zu: items with five chunks were not declined\n", ci); return 1; }
    // partial rows: Σv, Σv², n of the item's series in order
    for (int64_t it = 0; it < n_items; ++it) {
      for (int k = 0; k < q.T; ++k) {
        double a = 0.0, a2 = 0.0; uint32_t n = 0;
        for (int64_t p = item_begin[(size_t)it]; p < item_begin[(size_t)it + 1]; ++p) {
          const double v = ref[(size_t)order[(size_t)p] * q.T + k];
          if (v == v) { a += v; a2 += v * v; ++n; }
        }
        const size_t o = (size_t)it * q.T + k, o2 = (size_t)(n_items + it) * q.T + k;
        if (!same_bits(pval[o], a) || !same_bits(pval[o2], a2) || pcnt[o] != n) {
          std::printf("FAIL cfg %zu item %lld window %d: (%.17g, %.17g, %u) vs (%.17g, %.17g, %u)\n", ci, (long long)it, k, pval[o], pval[o2], pcnt[o], a, a2, n);
          return 1;
        }
        checked += 3;
      }
    }
    // merge (one group over all items) and presentation: the fixed 8-lane tree, then present_kernel over the partial form
    const int64_t gis[2] = {0, n_items};
    const int ktiles = (q.T + 31) / 32;
    for (int op : {filo::AGG_STDDEV, filo::AGG_STDVAR, filo::AGG_GROUP}) {
      std::vector<double> mv((size_t)q.T, -777.0), mp((size_t)2 * q.T, -777.0), pr((size_t)q.T, -777.0); std::vector<int64_t> mc((size_t)q.T, -1), mpc((size_t)q.T, -1);
      // the instantiation launch_merge_partials picks for the operator
      auto merge = [&](int partial_out, double* ov, int64_t* oc) {
        cusim::launch(dim3((unsigned)ktiles), dim3(256), [&] {
          if (op == filo::AGG_GROUP) filo::merge_partials_kernel<filo::MERGE_GROUP>(pval.data(), pcnt.data(), gis, 1, q.T, op, partial_out, ov, oc);
          else filo::merge_partials_kernel<filo::MERGE_MOMENTS>(pval.data(), pcnt.data(), gis, 1, q.T, op, partial_out, ov, oc);
        });
      };
      merge(0, mv.data(), mc.data());
      merge(1, mp.data(), mpc.data());
      cusim::launch(dim3((unsigned)((q.T + 255) / 256)), dim3(256), [&] { filo::present_kernel(op, q.T, mp.data(), mpc.data(), pr.data()); });
      for (int k = 0; k < q.T; ++k) {
        double la[8], la2[8]; unsigned long long lc[8];
        for (int j = 0; j < 8; ++j) {
          double a = 0.0, a2 = 0.0; unsigned long long n = 0;
          for (int64_t it = j; it < n_items; it += 8) { const size_t o = (size_t)it * q.T + k;
            if (pcnt[o]) { a += pval[o]; a2 += pval[(size_t)(n_items + it) * q.T + k]; n += pcnt[o]; } }
          la[j] = a; la2[j] = a2; lc[j] = n;
        }
        double a = la[0], a2 = la2[0]; unsigned long long n = lc[0];
        for (int j = 1; j < 8; ++j) if (lc[j]) { a += la[j]; a2 += la2[j]; n += lc[j]; }
        const double e = host_present(op, a, a2, n);
        const bool mom = op != filo::AGG_GROUP;
        if (!same_bits(mv[(size_t)k], e) || mc[(size_t)k] != (int64_t)n || !same_bits(mp[(size_t)k], a) || (mom && !same_bits(mp[(size_t)q.T + k], a2)) ||
            mpc[(size_t)k] != (int64_t)n || !same_bits(pr[(size_t)k], e)) {
          std::printf("FAIL cfg %zu op %d window %d: presented %.17g / %.17g vs %.17g, partial (%.17g, %.17g, %lld) vs (%.17g, %.17g, %llu)\n", ci, op, k,
                      mv[(size_t)k], pr[(size_t)k], e, mp[(size_t)k], mp[(size_t)q.T + k], (long long)mpc[(size_t)k], a, a2, n);
          return 1;
        }
        checked += 2;
      }
    }
    std::printf("cfg %zu ok: %d series in %lld items (%llu to the fallback list), T=%d\n", ci, c.nser, (long long)n_items, fcount, q.T);
    ++cases;
  }
  std::printf("OK %d cases, %ld values bit-exact (schedule seed %llu)\n", cases, checked, (unsigned long long)seed);
  return 0;
}
