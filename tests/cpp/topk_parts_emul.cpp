// topk / bottomk across GPUs on the CPU (test infrastructure; built and run by tests/test_topk_parts_emul.py): one series set cut into W
// parts (contiguous ranges as shard.series_range_of_rank, or series s on part s % W as the modulo shard map), each part's candidates
// computed by the oracle's aggregate() over its series with the ids mapped to global ordinals, merged by topk_merge_parts_kernel
// (scan_kernels.cu through tests/cpp/make_cusim_src.py) on the cusim emulator, and checked bit for bit, values and ids, against
// aggregate() over the union of the series.  Every part's candidates are also produced by topk_kernel and must equal the oracle's.
// Parts whose tables list their series in a shuffled order (a local -> global map that is not increasing, so equal values inside a part
// are not in ordinal order) are checked against a restatement of the merge rule over the parts' candidates instead.  A mutation of the
// merge rule (ties broken by part order instead of ordinal) must disagree with the oracle somewhere.
//     topk_parts_emul [schedule seed]
#define FILO_CUSIM 1
#include "cusim.h"
namespace filo { alignas(128) uint8_t smem[232448]; }
#include SCAN_SRC
#include "../../oracle/filo_query.hpp"
#include <algorithm>
#include <cfloat>
#include <random>
#include <string>

static bool same_bits(double a, double b) { uint64_t x, y; std::memcpy(&x, &a, 8); std::memcpy(&y, &b, 8); return x == y; }

// values: 0 gaussian, 1 integers in [-2, 2] with zeros of both signs (heavy ties), 2 edges (±Inf, ±DBL_MAX next to the padding, ±0, 1);
// NaN at random and in every series at window 0 (a window with only NaN inputs)
static std::vector<double> make_rows(std::mt19937_64& rng, int S, int T, int kind) {
  std::vector<double> v((size_t)S * T);
  std::normal_distribution<double> N(0.0, 10.0);
  const double edges[8] = {INFINITY, -INFINITY, DBL_MAX, -DBL_MAX, 0.0, -0.0, 1.0, -1.0};
  for (int s = 0; s < S; ++s)
    for (int t = 0; t < T; ++t) {
      double x;
      if (t == 0 || rng() % 7 == 0) x = std::nan("");
      else if (kind == 0) x = N(rng);
      else if (kind == 1) { const int i = (int)(rng() % 6); x = i == 5 ? -0.0 : (double)(i - 2); }
      else x = edges[rng() % 8];
      v[(size_t)s * T + t] = x;
    }
  return v;
}

// the merge rule restated: per cell the k best slots of all parts with id >= 0 and a non-NaN value, larger (topk) / smaller (bottomk)
// value first, among equal values the smaller ordinal -- or, as a mutation, the part listed first (the order an arrival-order fold
// would give) -- written worst first and padded
static void merge_rule(const std::vector<double>& pv, const std::vector<int64_t>& pid, int W, size_t n_cells, int k, bool bottom, bool by_part,
                       std::vector<double>& ov, std::vector<int64_t>& oi) {
  ov.assign(n_cells * k, bottom ? DBL_MAX : -DBL_MAX); oi.assign(n_cells * k, -1);
  for (size_t c = 0; c < n_cells; ++c) {
    std::vector<std::pair<double, std::pair<int, int64_t>>> all;           // value, (part, id)
    for (int p = 0; p < W; ++p)
      for (int s = 0; s < k; ++s) { const size_t i = ((size_t)p * n_cells + c) * k + s; if (pid[i] >= 0 && pv[i] == pv[i]) all.push_back({pv[i], {p, pid[i]}}); }
    std::stable_sort(all.begin(), all.end(), [&](const auto& a, const auto& b) {
      if (a.first != b.first) return bottom ? a.first < b.first : a.first > b.first;
      return by_part ? a.second.first < b.second.first : a.second.second < b.second.second;
    });
    const int m = std::min<int>(k, (int)all.size());
    for (int j = 0; j < m; ++j) { ov[c * k + j] = all[(size_t)(m - 1 - j)].first; oi[c * k + j] = all[(size_t)(m - 1 - j)].second.second; }
  }
}

int main(int argc, char** argv) {
  cusim::rng_state() = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 0;
  std::mt19937_64 rng(4242);
  struct Cfg { int W, S, G, T, k, split, kind, shuffle = 0; };  // split: 0 contiguous, 1 modulo; shuffle: tables list their series in a random order
  const std::vector<Cfg> cfgs = {
    {1, 12, 3, 9, 3, 0, 0},                                      // one part: the merge reproduces it
    {2, 20, 4, 11, 3, 0, 1},
    {2, 20, 4, 11, 3, 1, 1},
    {3, 25, 5, 10, 1, 1, 1},                                     // k = 1
    {3, 25, 5, 10, 32, 0, 2},                                    // k = 32: every group smaller than k
    {8, 30, 4, 7, 3, 1, 1},
    {8, 30, 4, 7, 32, 0, 0},
    {8, 5, 3, 6, 3, 0, 2},                                       // parts 3..7 hold no series
    {64, 90, 4, 5, 3, 1, 1},                                     // more parts than lanes: the strided pass
    {64, 40, 4, 5, 32, 0, 2},                                    // 64 parts, 24 of them empty
    {64, 200, 3, 4, 32, 1, 1},
    {1, 12, 3, 9, 3, 0, 1, 1},                                   // non-increasing local -> global maps with ties inside a part
    {3, 25, 5, 10, 5, 1, 1, 1},
    {8, 30, 4, 7, 32, 0, 1, 1},
    {64, 200, 3, 4, 32, 1, 1, 1},
  };
  long checked = 0; int cases = 0, mutation_caught = 0, ties_at_cut = 0, unordered_ties = 0;
  for (size_t ci = 0; ci < cfgs.size(); ++ci) {
    const Cfg& c = cfgs[ci];
    const int W = c.W, S = c.S, G = c.G, T = c.T, k = c.k;
    const std::vector<double> rows = make_rows(rng, S, T, c.kind);
    std::vector<std::vector<int>> sids((size_t)W);
    const int per = (S + W - 1) / W;
    for (int s = 0; s < S; ++s) sids[(size_t)(c.split == 0 ? s / per : s % W)].push_back(s);
    if (c.shuffle) for (auto& v : sids) std::shuffle(v.begin(), v.end(), rng);
    // group G - 1 has no series, group 0 none on part 0; the others at random
    std::vector<int32_t> gid((size_t)S);
    for (int s = 0; s < S; ++s) {
      const bool on_part0 = (c.split == 0 ? s / per : s % W) == 0;
      gid[(size_t)s] = G <= 2 ? 0 : (W > 1 && on_part0) ? 1 + (int32_t)(rng() % (uint64_t)(G - 2)) : (int32_t)(rng() % (uint64_t)(G - 1));
    }
    const size_t n_cells = (size_t)G * T;
    std::vector<const double*> all_rows; for (int s = 0; s < S; ++s) all_rows.push_back(rows.data() + (size_t)s * T);
    bool empty_part = false, group_empty_somewhere = false;
    for (int op : {fo::AGG_TOPK, fo::AGG_BOTTOMK}) {
      const bool bottom = op == fo::AGG_BOTTOMK;
      std::vector<double> pv((size_t)W * n_cells * k, -777.0); std::vector<int64_t> pid((size_t)W * n_cells * k, -777);
      for (int p = 0; p < W; ++p) {
        const std::vector<int>& ids = sids[(size_t)p];
        empty_part |= ids.empty();
        std::vector<const double*> rs; std::vector<int32_t> gs;
        for (int s : ids) { rs.push_back(rows.data() + (size_t)s * T); gs.push_back(gid[(size_t)s]); }
        for (int g = 0; g < G - 1; ++g) group_empty_somewhere |= std::find(gs.begin(), gs.end(), g) == gs.end();
        const fo::AggResult e = fo::aggregate((fo::AggrOp)op, k, rs, gs, G, T);
        // topk_kernel over the part's table (series in table order, grouped by a stable sort) gives the oracle's candidates
        std::vector<double> per_series((size_t)std::max<size_t>(ids.size(), 1) * T);
        for (size_t j = 0; j < ids.size(); ++j) std::memcpy(per_series.data() + j * T, rs[j], (size_t)T * 8);
        std::vector<int32_t> order((size_t)ids.size()); for (size_t j = 0; j < ids.size(); ++j) order[j] = (int32_t)j;
        std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return gs[(size_t)a] < gs[(size_t)b]; });
        std::vector<int64_t> gstart((size_t)G + 1, 0);
        for (int g = 0; g <= G; ++g) { int64_t n = 0; for (int32_t x : gs) n += x < g; gstart[(size_t)g] = n; }
        std::vector<double> kv(n_cells * k, -777.0); std::vector<int64_t> ki(n_cells * k, -777);
        cusim::launch(dim3((unsigned)((n_cells + 127) / 128)), dim3(128), [&] {
          filo::topk_kernel(per_series.data(), order.data(), gstart.data(), G, T, k, bottom, kv.data(), ki.data()); });
        for (size_t i = 0; i < n_cells * (size_t)k; ++i)
          if (!same_bits(kv[i], e.values[i]) || ki[i] != e.aux[i]) {
            std::printf("FAIL cfg %zu op %d part %d slot %zu: topk_kernel (%.17g, %lld) vs oracle (%.17g, %lld)\n", ci, op, p, i, kv[i], (long long)ki[i],
                        e.values[i], (long long)e.aux[i]);
            return 1;
          }
        for (size_t i = 0; i < n_cells * (size_t)k; ++i) {
          pv[(size_t)p * n_cells * k + i] = e.values[i];
          pid[(size_t)p * n_cells * k + i] = e.aux[i] < 0 ? -1 : ids[(size_t)e.aux[i]];        // local -> global ordinal
        }
      }
      // a shuffled part may list equal values with the smaller ordinal first: what a merge that assumed ordinal order inside a part missed
      for (size_t i = 0; i + 1 < pid.size(); ++i)
        unordered_ties += c.shuffle && (i + 1) % (size_t)k != 0 && pid[i] >= 0 && pid[i + 1] >= 0 && pv[i] == pv[i + 1] && pid[i] < pid[i + 1];
      fo::AggResult want;
      if (c.shuffle) merge_rule(pv, pid, W, n_cells, k, bottom, false, want.values, want.aux);
      else {
        want = fo::aggregate((fo::AggrOp)op, k, all_rows, gid, G, T);
        std::vector<double> rv; std::vector<int64_t> ri;                 // the restatement agrees with the oracle over the union
        merge_rule(pv, pid, W, n_cells, k, bottom, false, rv, ri);
        for (size_t i = 0; i < n_cells * (size_t)k; ++i)
          if (!same_bits(rv[i], want.values[i]) || ri[i] != want.aux[i]) { std::printf("FAIL cfg %zu op %d slot %zu: the merge rule restated differs from the oracle\n", ci, op, i); return 1; }
      }
      std::vector<double> ov(n_cells * k, -777.0); std::vector<int64_t> oi(n_cells * k, -777);
      cusim::launch(dim3((unsigned)((n_cells + 7) / 8)), dim3(256), [&] {
        filo::topk_merge_parts_kernel(pv.data(), pid.data(), W, (int64_t)n_cells, k, bottom, ov.data(), oi.data()); });
      for (size_t i = 0; i < n_cells * (size_t)k; ++i) {
        if (!same_bits(ov[i], want.values[i]) || oi[i] != want.aux[i]) {
          std::printf("FAIL cfg %zu op %d cell %zu slot %zu: merged (%.17g, %lld) vs expected (%.17g, %lld)\n", ci, op, i / k, i % k, ov[i], (long long)oi[i],
                      want.values[i], (long long)want.aux[i]);
          return 1;
        }
        ++checked;
      }
      // the mutation: on a modulo split with ties, part order differs from ordinal order and the check above would catch it
      std::vector<double> mv; std::vector<int64_t> mi;
      merge_rule(pv, pid, W, n_cells, k, bottom, true, mv, mi);
      bool differs = false;
      for (size_t i = 0; i < n_cells * (size_t)k; ++i) differs |= !same_bits(mv[i], want.values[i]) || mi[i] != want.aux[i];
      if (!c.shuffle && c.split == 1 && c.kind == 1 && W > 1 && k > 1) {
        if (!differs) { std::printf("FAIL cfg %zu op %d: ties broken by part order pass the check\n", ci, op); return 1; }
        ++mutation_caught;
      }
      // ties that straddle the cut: an equal value inside and outside the kept k of a cell
      for (size_t cl = 0; cl < n_cells && !c.shuffle; ++cl) {
        if (want.aux[cl * k] < 0) continue;
        const double worst = want.values[cl * k];
        int eq = 0; for (int s = 0; s < S; ++s) eq += gid[(size_t)s] == (int32_t)(cl / T) && rows[(size_t)s * T + cl % T] == worst;
        int kept_eq = 0; for (int j = 0; j < k; ++j) kept_eq += want.aux[cl * k + j] >= 0 && want.values[cl * k + j] == worst;
        ties_at_cut += eq > kept_eq;
      }
    }
    if (G > 1 && W > 1 && !group_empty_somewhere) { std::printf("FAIL cfg %zu: no group empty on a part\n", ci); return 1; }
    std::printf("cfg %zu ok: W %d (%s%s%s), S %d, G %d, T %d, k %d\n", ci, W, c.split ? "modulo" : "contiguous", c.shuffle ? ", shuffled tables" : "",
                empty_part ? ", empty parts" : "", S, G, T, k);
    ++cases;
  }
  // hand-made: a part listing equal values with the smaller ordinal first (local series 0 -> global 9, 1 -> global 3), and a NaN value
  // with an id, which is skipped like an empty slot
  {
    const double NaN = std::nan("");
    const double v1[2] = {5.0, 5.0}; const int64_t i1[2] = {3, 9};
    const double v2[2 * 3] = {1.0, 5.0, -DBL_MAX, NaN, 5.0, 7.0}; const int64_t i2[2 * 3] = {4, 6, -1, 8, 1, 2};
    struct Hand { int W, k; const double* v; const int64_t* id; std::vector<double> wv; std::vector<int64_t> wi; };
    const Hand hs[2] = {{1, 2, v1, i1, {5.0, 5.0}, {9, 3}}, {2, 3, v2, i2, {5.0, 5.0, 7.0}, {6, 1, 2}}};
    for (const Hand& h : hs) {
      std::vector<double> ov((size_t)h.k, -777.0); std::vector<int64_t> oi((size_t)h.k, -777);
      cusim::launch(dim3(1), dim3(256), [&] { filo::topk_merge_parts_kernel(h.v, h.id, h.W, 1, h.k, 0, ov.data(), oi.data()); });
      for (int j = 0; j < h.k; ++j)
        if (!same_bits(ov[(size_t)j], h.wv[(size_t)j]) || oi[(size_t)j] != h.wi[(size_t)j]) {
          std::printf("FAIL hand-made W %d slot %d: (%.17g, %lld) vs (%.17g, %lld)\n", h.W, j, ov[(size_t)j], (long long)oi[(size_t)j], h.wv[(size_t)j], (long long)h.wi[(size_t)j]);
          return 1;
        }
    }
    ++cases;
  }
  if (!mutation_caught || !ties_at_cut || !unordered_ties) {
    std::printf("FAIL: coverage (mutation caught %d, ties at the cut %d, unordered ties in shuffled parts %d)\n", mutation_caught, ties_at_cut, unordered_ties);
    return 1;
  }
  std::printf("OK %d cases, %ld slots bit-exact (values and ids); part-order mutation caught %d times; %d cells with a tie at the cut; "
              "%d unordered ties in shuffled parts\n", cases, checked, mutation_caught, ties_at_cut, unordered_ties);
  return 0;
}
