// GPU driver for the C++ operator mirror (include/filo_b200.hpp) over histogram columns (test infrastructure; built and run by
// tests/test_gpu_hist_series.py).  Chunks come from the oracle's histogram store (oracle/hist_capi.cpp, libfilo_oracle.so):
//   1. PeriodicSamplesMapper with functionId unset (LastSample) over a histogram column -> [series][T][buckets], the raw rows;
//   2. PeriodicSamplesMapper(Rate) + HistogramQuantileMapper(q) without an AggregateMapReduce -> [series][T], Histogram.quantile of each
//      series' own rate histogram (the oracle's periodic samples + quantile).
#include "filo_b200.hpp"
#include <cstdio>
#include <cstring>
#include <random>

extern "C" {
void* fo_hstore_new();
void fo_hstore_free(void*);
int64_t fo_hstore_add_series(void*);
int32_t fo_hstore_add_chunk(void*, int64_t, const int64_t*, int32_t, int, double, double, int, const double*, int32_t, const int64_t*, int32_t, int32_t);
int64_t fo_hstore_num_chunks(void*, int64_t);
void fo_hstore_info_addrs(void*, int64_t, uint64_t*);
int32_t fo_hstore_query(void*, int32_t, int32_t, int64_t, int64_t, int64_t, int64_t, int32_t, int32_t, const int32_t*, int32_t, int32_t, double,
                        double*, uint8_t*, double*);
double fo_hist_quantile(int, double, double, int, const double*, int, const double*, double);
}

static bool same_bits(double a, double b) { uint64_t x, y; std::memcpy(&x, &a, 8); std::memcpy(&y, &b, 8); return x == y || (a != a && b != b); }

int main() {
  const int S = 6, rows = 240, nb = 12, kind = 1 /* geometric */;
  const double first = 2.0, mult = 2.0;
  const int64_t t0 = 1700000000000LL;
  void* st = fo_hstore_new();
  std::mt19937_64 rng(7);
  std::vector<std::vector<int64_t>> vals((size_t)S);
  std::vector<filo::RawDataRangeVector> src((size_t)S);
  for (int s = 0; s < S; ++s) {
    std::vector<int64_t> ts((size_t)rows), cur((size_t)nb, 0);
    vals[(size_t)s].resize((size_t)rows * nb);
    for (int r = 0; r < rows; ++r) {
      ts[(size_t)r] = t0 + (int64_t)r * 15000;
      if (r == 70 + 13 * s) std::fill(cur.begin(), cur.end(), 0);                        // a counter reset (a Drop section)
      int64_t run = 0;
      for (int b = 0; b < nb; ++b) { run += (int64_t)(rng() % 7); cur[(size_t)b] += run; vals[(size_t)s][(size_t)r * nb + b] = cur[(size_t)b]; }
    }
    const int64_t si = fo_hstore_add_series(st);
    const int chunks[2] = {160, 80}; int off = 0;
    for (int n : chunks) {
      if (fo_hstore_add_chunk(st, si, ts.data() + off, n, kind, first, mult, 0, nullptr, nb, vals[(size_t)s].data() + (size_t)off * nb, 1, 15000) != 0) { std::printf("FAIL add_chunk\n"); return 1; }
      off += n;
    }
    src[(size_t)s].chunkInfoAddrs.resize((size_t)fo_hstore_num_chunks(st, si));
    fo_hstore_info_addrs(st, si, src[(size_t)s].chunkInfoAddrs.data());
  }
  const int64_t start = t0 + 300000, step = 15000, end = t0 + (int64_t)(rows - 1) * 15000, window = 300000;
  const int T = filo_num_windows(start, step, end);
  int bad = 0;
  try {
    filo::FusedGpuExec ex(0);
    // 1. LastSample: windows end on the scrape times, so window k holds row 20 + k as appended (raw, also after the reset)
    filo::PeriodicSamplesMapper psm_last(start, step, end, std::nullopt, std::nullopt);
    const filo::QueryResult rl = ex.execute(src, psm_last, nullptr, nullptr, 1, true, true);
    if (rl.rows != S || rl.windows != T || rl.buckets != nb) { std::printf("FAIL last shape %d %d %d\n", rl.rows, rl.windows, rl.buckets); return 1; }
    for (int s = 0; s < S; ++s)
      for (int k = 0; k < T; ++k)
        for (int b = 0; b < nb; ++b)
          if (!same_bits(rl.values[((size_t)s * T + k) * nb + b], (double)vals[(size_t)s][(size_t)(20 + k) * nb + b])) ++bad;
    // 2. per-series histogram_quantile(0.9, rate(h[5m]))
    filo::PeriodicSamplesMapper psm_rate(start, step, end, window, filo::InternalRangeFunction::Rate);
    filo::HistogramQuantileMapper hq(0.9);
    const filo::QueryResult rq = ex.execute(src, psm_rate, nullptr, &hq, 1, true, true);
    if (rq.rows != S || rq.windows != T || rq.buckets != 0 || rq.values.size() != (size_t)S * T) { std::printf("FAIL quantile shape\n"); return 1; }
    std::vector<double> ov((size_t)S * T * nb); std::vector<uint8_t> oe((size_t)S * T);
    if (fo_hstore_query(st, FILO_FN_RATE, 1, start, step, end, window, 1, 0, nullptr, 1, nb, 0.9, ov.data(), oe.data(), nullptr) != 0) { std::printf("FAIL oracle\n"); return 1; }
    int finite = 0;
    for (size_t i = 0; i < (size_t)S * T; ++i) {
      const double e = oe[i] ? std::nan("") : fo_hist_quantile(kind, first, mult, 0, nullptr, nb, ov.data() + i * nb, 0.9);
      const double g = rq.values[i];
      if ((e != e) != (g != g) || (e == e && std::fabs(g - e) > 1e-9 * std::fabs(e))) ++bad;
      finite += e == e;
    }
    if (finite == 0) { std::printf("FAIL no finite quantile\n"); return 1; }
  } catch (const std::exception& e) { std::printf("FAIL %s\n", e.what()); return 1; }
  fo_hstore_free(st);
  if (bad) { std::printf("FAIL %d mismatches\n", bad); return 1; }
  std::printf("OK hist mirror: last %d x %d x %d, per-series quantile %d x %d\n", S, T, nb, S, T);
  return 0;
}
