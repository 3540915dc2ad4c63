// scan_tile_kernel on the CPU: the kernel's own source (filodb_b200/csrc/scan_tile.cuh) compiled for the host on top of the cusim
// SIMT emulator (tests/cpp/cusim.h), fed with arena records built from the oracle's encoders and checked bit-exact against the
// oracle's ChunkedWindowIterator.  Test infrastructure: built and run by tests/test_abi.py.
//   tile_emul [seed]     seed 0 = round-robin schedule, otherwise a pseudo-random fiber schedule
#define FILO_CUSIM 1
#include "cusim.h"
namespace filo { alignas(128) uint8_t smem[232448]; }          // `extern __shared__ ... smem[]` of the kernels
#ifdef SCAN_SRC
#include SCAN_SRC                                             // scan_kernels.cu through tests/cpp/make_cusim_src.py (function-scope __shared__ -> static)
#define HAVE_MERGE_KERNEL 1
#else
#include "../../filodb_b200/csrc/scan_kernels.cu"          // every scan kernel (the launchers are compiled out under FILO_CUSIM)
#endif
#include "../../oracle/filo_query.hpp"
#include <cassert>
#include <memory>
#include <random>
#include <string>

struct Chunk { std::vector<uint8_t> ts, vv, info; };
struct SeriesData { std::vector<std::unique_ptr<Chunk>> chunks; std::vector<uint8_t> record; };

static long g_wp_declined = 0, g_wp_series = 0;
static int g_long_col = 0;          // 1: Long value column through LongBinaryVector.optimize (DDV / const DDV), 2: raw 64-bit longs
static int g_jitter_ms = 0; static bool g_integral = false;      // irregular scrapes (DDV timestamps) / integral values (DoubleVector.optimize -> DDV longs)
static bool g_signed_zero = false;  // gauge values +0.0 / -0.0 in runs of 12 rows: min / max meet equal zeros of both signs
static std::string g_chunk_enc;     // when set: chunk c's values XOR ('x') or raw f64 ('r'), in place of xor_enc
// chunks of the given rows (nan_ppm: a stale marker at a chunk end) and the arena record, from timestamps and values
static void build_series_from(SeriesData& S, std::mt19937_64& rng, const std::vector<int64_t>& ts, const std::vector<double>& v, const std::vector<int>& chunk_rows,
                              int kind /*0 gauge 1 counter*/, bool xor_enc, int nan_ppm) {
  int r0 = 0;
  for (int n : chunk_rows) {
    if (!g_chunk_enc.empty()) { assert(g_chunk_enc.size() == chunk_rows.size()); xor_enc = g_chunk_enc[S.chunks.size()] == 'x'; }
    auto c = std::make_unique<Chunk>();
    std::vector<double> cv(v.begin() + r0, v.begin() + r0 + n);
    if (nan_ppm && (int)(rng() % 1000000) < nan_ppm) cv[(size_t)n - 1] = std::nan("");          // stale marker at the chunk end
    c->ts = fo::enc::timestamps(ts.data() + r0, n);
    if (g_long_col) {
      std::vector<int64_t> lv((size_t)n);
      for (int i = 0; i < n; ++i) lv[(size_t)i] = (int64_t)std::floor(v[(size_t)(r0 + i)] * (g_long_col == 2 ? 1e15 : (r0 % 3 == 1 ? 0.0 : 1.0)));      // some chunks constant (const DDV, slope 0)
      c->vv = g_long_col == 2 ? fo::enc::rawLongs(lv.data(), n) : fo::enc::longs(lv.data(), n);
    } else
    c->vv = xor_enc ? fo::enc::doublesXor(cv.data(), n, kind == 1) : fo::enc::doubles(cv.data(), n, kind == 1);
    c->info.assign(fo::csi::OffsetVectors + 16, 0);
    fo::setLong(c->info.data() + fo::csi::OffsetChunkID, fo::csi::chunkID(ts[(size_t)r0], (ts[(size_t)(r0 + n - 1)] + 1000) / 1000));
    fo::setInt(c->info.data() + fo::csi::OffsetNumRows, n);
    fo::setLong(c->info.data() + fo::csi::OffsetIngestionTime, ts[(size_t)(r0 + n - 1)] + 1000);
    fo::setLong(c->info.data() + fo::csi::OffsetEndTime, ts[(size_t)(r0 + n - 1)]);
    fo::setLong(c->info.data() + fo::csi::OffsetVectors, (int64_t)(uintptr_t)c->ts.data());
    fo::setLong(c->info.data() + fo::csi::OffsetVectors + 8, (int64_t)(uintptr_t)c->vv.data());
    S.chunks.push_back(std::move(c));
    r0 += n;
  }
  // arena record (filo_record.h), as filo_load_series writes it
  const size_t nch = S.chunks.size();
  const size_t off = sizeof(filo::RecordHeader) + nch * sizeof(filo::ChunkEntry);
  std::vector<filo::ChunkEntry> E(nch); std::vector<uint8_t> body; uint32_t row_base = 0, flags = filo::REC_ALL_TS_CONST;
  for (size_t i = 0; i < nch; ++i) {
    Chunk& c = *S.chunks[i];
    E[i].start_time = fo::csi::startTime(c.info.data()); E[i].end_time = fo::csi::endTime(c.info.data()); E[i].num_rows = fo::csi::numRows(c.info.data());
    auto put = [&](const std::vector<uint8_t>& x) { while ((off + body.size()) % 8) body.push_back(0); const uint32_t o = (uint32_t)(off + body.size()); body.insert(body.end(), x.begin(), x.end()); return o; };
    E[i].ts_off = put(c.ts); E[i].val_off = put(c.vv); E[i].row_base = row_base;
    const int twire = (int)(c.ts[4] | (c.ts[5] << 8)), vwire = (int)(c.vv[4] | (c.vv[5] << 8));
    if (twire != filo::WIRE_DDV_CONST) flags &= ~filo::REC_ALL_TS_CONST;
    if (c.vv[7] & 0x80) flags |= filo::REC_ANY_DROP;
    if (vwire == filo::WIRE_XOR || vwire == filo::WIRE_DDV || vwire == filo::WIRE_DDV_CONST) flags |= filo::REC_ANY_DECODE;
    uint32_t vlen = (uint32_t)E[i].num_rows;
    row_base += vlen;
  }
  size_t total = off + body.size(); total = (total + 15) & ~(size_t)15;
  S.record.assign(total, 0);
  filo::RecordHeader h; h.rec_bytes = (uint32_t)total; h.n_chunks = (uint32_t)nch; h.n_rows = row_base; h.flags = flags;
  std::memcpy(S.record.data(), &h, sizeof h);
  std::memcpy(S.record.data() + sizeof h, E.data(), nch * sizeof(filo::ChunkEntry));
  std::memcpy(S.record.data() + off, body.data(), body.size());
}
static void build_series(SeriesData& S, std::mt19937_64& rng, int rows, const std::vector<int>& chunk_rows, int64_t t0, int step_ms, int kind /*0 gauge 1 counter*/,
                         bool xor_enc, int nan_ppm, int reset_every) {
  std::vector<int64_t> ts((size_t)rows); std::vector<double> v((size_t)rows);
  std::normal_distribution<double> N(0.0, 1.0);
  double acc = 0.0, zrun = 0.0;
  for (int r = 0; r < rows; ++r) {
    ts[(size_t)r] = t0 + (int64_t)r * step_ms + (g_jitter_ms ? (int64_t)(rng() % (uint64_t)(2 * g_jitter_ms + 1)) - g_jitter_ms : 0);
    double g = 15.0 + std::sin((double)(r + 1)) + N(rng);
    if (g_integral) g = std::floor(g);
    if (g_signed_zero) { if (r % 12 == 0) zrun = rng() & 1 ? -0.0 : 0.0; g = zrun; }
    if (kind == 0) v[(size_t)r] = g;
    else { if (reset_every && r > 0 && rng() % (uint64_t)reset_every == 0) acc = 0.0; acc += g > 0 ? g : 0.0; v[(size_t)r] = acc; }
  }
  build_series_from(S, rng, ts, v, chunk_rows, kind, xor_enc, nan_ppm);
}

static bool same_bits(double a, double b) { uint64_t x, y; std::memcpy(&x, &a, 8); std::memcpy(&y, &b, 8); return x == y || (a != a && b != b); }

struct Launch {
  const uint8_t* arena; const int64_t* rec_off; int64_t S; filo::QueryParams q; double* out; filo::TileSmem L; int grid;
  int64_t* flist; unsigned long long* fcount; unsigned long long* counters; int* derr;
  const int32_t* order; const int64_t* item_begin; int64_t n_items; int agg_op; double* pval; uint32_t* pcnt;
};
template <int FN, bool AGG> static void run_kernel(const Launch& A) {
  cusim::launch(dim3((unsigned)A.grid), dim3(filo::TILE_LAUNCH_THREADS), [&] {
    filo::scan_tile_kernel<FN, AGG>(A.arena, A.rec_off, A.S, A.q, A.out, A.L, A.flist, A.fcount, A.counters, A.derr, A.order, A.item_begin, A.n_items, A.agg_op, A.pval, A.pcnt);
  });
}
template <bool AGG> static void dispatch(const Launch& A) {          // the instantiations launch_tile_any makes (scan_kernels.cu)
  const int fn = A.q.fn;
  if (fn == filo::FN_RATE) run_kernel<filo::FN_RATE, AGG>(A);
  else if (fn == filo::FN_AVG) run_kernel<filo::FN_AVG, AGG>(A);
  else if (fn == filo::FN_COUNT) run_kernel<filo::FN_COUNT, AGG>(A);
  else run_kernel<filo::FN_SUM, AGG>(A);
}
// the v2 warp-per-series kernel (every function / encoding; also the fallback pass over the series the tile kernel declined)
struct V2Shape { uint32_t max_rec; int max_rows, max_chunks; bool any_nonconst_ts, any_drop; };
static void run_v2(const Launch& A, const V2Shape& sh, const int64_t* list, const unsigned long long* list_count) {
  const bool need_corr2 = (A.q.fn == filo::FN_RATE || A.q.fn == filo::FN_INCREASE) && A.q.cumulative && sh.any_drop;
  uint32_t scratch = filo::align_up((uint32_t)sh.max_chunks * (uint32_t)filo::CHUNK_DESC_BYTES, 16) +
                     ((uint32_t)sh.max_rows + (uint32_t)sh.max_chunks * 8u) * 8u * (1u + (sh.any_nonconst_ts ? 1u : 0u) + (need_corr2 ? 1u : 0u));
  scratch = filo::align_up(scratch + 16, 128);                        // as filo_query sizes it (capi.cu)
  const uint32_t rec_cap = filo::align_up(sh.max_rec + 16, 128);
  const size_t smem_bytes = (size_t)(filo::WARP_HDR_BYTES + rec_cap + filo::STAGE_BYTES + scratch) * filo::FAST_WARPS;
  if (smem_bytes > sizeof(filo::smem)) { std::printf("FAIL: v2 shared memory %zu\n", smem_bytes); std::exit(1); }
  auto body = [&](auto cls) {
    cusim::launch(dim3((unsigned)A.grid), dim3(filo::FAST_WARPS * 32), [&] {
      filo::scan_series_kernel_v2<decltype(cls)::value>(A.arena, A.rec_off, A.S, A.q, A.out, rec_cap, scratch, A.counters, A.derr, list, list_count);
    });
  };
  switch (filo::fn_class_of(A.q.fn, A.q.cumulative, A.q.long_values)) {
    case filo::CLASS_SUM: body(std::integral_constant<int, filo::CLASS_SUM>{}); break;
    case filo::CLASS_MINMAX: body(std::integral_constant<int, filo::CLASS_MINMAX>{}); break;
    case filo::CLASS_COUNTER: body(std::integral_constant<int, filo::CLASS_COUNTER>{}); break;
    default: body(std::integral_constant<int, filo::CLASS_POINT>{}); break;
  }
}
// the fused fallback: scan_agg_kernel_v2 over the items the tile kernel declined
static void run_agg_v2(const Launch& A, const V2Shape& sh, const int64_t* list, const unsigned long long* list_count) {
  const bool need_corr2 = (A.q.fn == filo::FN_RATE || A.q.fn == filo::FN_INCREASE) && A.q.cumulative && sh.any_drop;
  uint32_t scratch = filo::align_up((uint32_t)sh.max_chunks * (uint32_t)filo::CHUNK_DESC_BYTES, 16) +
                     ((uint32_t)sh.max_rows + (uint32_t)sh.max_chunks * 8u) * 8u * (1u + (sh.any_nonconst_ts ? 1u : 0u) + (need_corr2 ? 1u : 0u));
  scratch = filo::align_up(scratch + 16, 128);
  const uint32_t rec_cap = filo::align_up(sh.max_rec + 16, 128), acc_bytes = filo::align_up((uint32_t)A.q.T * 12u, 128);
  const size_t smem_bytes = (size_t)(filo::WARP_HDR_BYTES + rec_cap + filo::STAGE_BYTES + acc_bytes + scratch) * filo::FAST_WARPS;
  if (smem_bytes > sizeof(filo::smem)) { std::printf("FAIL: agg v2 shared memory %zu\n", smem_bytes); std::exit(1); }
  auto body = [&](auto cls) {
    cusim::launch(dim3((unsigned)A.grid), dim3(filo::FAST_WARPS * 32), [&] {
      filo::scan_agg_kernel_v2<decltype(cls)::value>(A.arena, A.rec_off, A.order, A.item_begin, A.n_items, A.q, A.agg_op, A.pval, A.pcnt, rec_cap, scratch, acc_bytes,
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
static fo::RangeFn oracle_fn(int fn) {
  switch (fn) { case filo::FN_SUM: return fo::FN_SUM_OVER_TIME; case filo::FN_AVG: return fo::FN_AVG_OVER_TIME; case filo::FN_COUNT: return fo::FN_COUNT_OVER_TIME;
                case filo::FN_MIN: return fo::FN_MIN_OVER_TIME; case filo::FN_MAX: return fo::FN_MAX_OVER_TIME; case filo::FN_TIMESTAMP: return fo::FN_TIMESTAMP; default: return (fo::RangeFn)fn; }
}

int main(int argc, char** argv) {
  const uint64_t seed = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 0;
  cusim::rng_state() = seed;
  std::mt19937_64 rng(4242);
  long checked = 0; int cases = 0;
  struct Cfg { int kind = 0; bool xor_enc = true; int fn = 0; std::vector<int> chunks; int nan_ppm = 0, reset_every = 0; int64_t window = 300000; int nser = 1; int inclusive = 1;
               int64_t start_off = 0, end_off = 0; int agg_op = 0; int grid = 1; int jitter = 0; bool integral = false; bool v2_only = false; bool wp = false; bool hetero = false; int long_col = 0; double p0 = 0, p1 = 0; bool szero = false; };
  std::vector<Cfg> all_ext;
  const std::vector<Cfg> cfgs = {
    {0, true, filo::FN_RATE, {400, 80}, 200000, 0, 300000, 11, 1, 0, 0, 0, 2},           // C2: gauge, delta-temporality rate (CLASS_SUM), NaN stale markers
    {0, true, filo::FN_SUM, {150, 90}, 0, 0, 300000, 37, 1, -90000, 45000, 0, 2},        // several tiles per CTA, a partial last tile, windows before / after the data
    {0, true, filo::FN_SUM, {150, 90}, 0, 0, 300000, 13, 1, -90000, 45000, 0, 2},        // the same, two tiles
    {0, false, filo::FN_AVG, {200, 40}, 100000, 0, 120000, 5, 0, 0, 0, 0, 1},             // raw f64 vectors, exclusive range start
    {0, true, filo::FN_COUNT, {60, 60, 60, 60}, 300000, 0, 600000, 9, 1, 30000, 0, 0, 3}, // four chunks, long windows over several chunk junctions
    {0, true, filo::FN_RATE, {100, 50, 50, 50, 50}, 0, 0, 300000, 10, 1, 0, 0, 0, 2},     // five chunks: declined (fallback list)
    {0, true, filo::FN_AVG, {100, 100, 100}, 30000, 0, 300000, 24, 1, 0, 0, 0, 2},        // two junctions per series, NaN rows in some tiles only
    {0, true, filo::FN_COUNT, {90, 70, 50, 30}, 0, 0, 240000, 16, 0, 15000, 0, 0, 2},     // three junctions, exclusive range start, a chunk barely longer than the window
    {0, false, filo::FN_SUM, {64, 200}, 0, 0, 420000, 9, 1, 0, 0, 0, 1},                  // raw vectors, a 29-window junction
    {0, true, filo::FN_RATE, {400, 80}, 200000, 0, 300000, 19, 1, 0, 0, 0, 2},           // C2 shape with NaN markers, three tiles
    {0, true, filo::FN_AVG, {100, 100, 100}, 30000, 0, 300000, 24, 1, -30000, 30000, 0, 2},  // three chunks, windows before / after the data
    {0, true, filo::FN_SUM, {33, 150, 7, 90}, 0, 0, 240000, 11, 0, 0, 0, 0, 3},           // a 7-row chunk inside the windows, raw + XOR mixes
    // the v4 warp-pipeline kernel (scan_wp.cuh) for the SUM class, declines chained to the v2 kernel
    {0, true, filo::FN_RATE, {400, 80}, 200000, 0, 300000, 23, 1, 0, 0, 0, 2, 0, false, false, true},                 // C2 shape, NaN stale markers (declined)
    {0, true, filo::FN_SUM, {150, 90}, 0, 0, 300000, 37, 1, -90000, 45000, 0, 2, 0, false, false, true},              // windows before / after the data
    {0, false, filo::FN_AVG, {200, 40}, 0, 0, 180000, 9, 0, 0, 0, 0, 1, 0, false, false, true},                       // raw f64, exclusive range start
    {0, true, filo::FN_COUNT, {60, 60, 60, 60}, 0, 0, 600000, 9, 1, 30000, 0, 0, 3, 0, false, false, true},           // four chunks, windows over three chunks (declined)
    {0, true, filo::FN_AVG, {100, 100, 100}, 0, 0, 300000, 24, 1, 0, 0, 0, 2, 0, false, false, true},                 // two junctions
    {0, true, filo::FN_COUNT, {90, 70, 50, 30}, 0, 0, 240000, 16, 0, 15000, 0, 0, 2, 0, false, false, true},          // three junctions, exclusive start
    {0, false, filo::FN_SUM, {64, 200}, 0, 0, 420000, 9, 1, 0, 0, 0, 1, 0, false, false, true},
    {0, true, filo::FN_RATE, {100, 50, 50, 50, 50}, 0, 0, 300000, 10, 1, 0, 0, 0, 2, 0, false, false, true},          // five chunks: declined
    {0, true, filo::FN_SUM, {33, 150, 7, 90}, 0, 0, 240000, 11, 0, 0, 0, 0, 3, 0, false, false, true},                // a 7-row chunk inside the windows
    {0, false, filo::FN_RATE, {500, 400}, 0, 0, 300000, 7, 1, 0, 0, 0, 1, 0, false, false, true},                      // more than 64 blocks per series: second pass
    {0, true, filo::FN_SUM, {150, 90}, 0, 0, 300000, 29, 1, -90000, 45000, 0, 2, 0, false, false, true, true},          // chunk shapes differ from series to series: the plan memo is invalidated
    {0, false, filo::FN_AVG, {200, 100}, 0, 0, 180000, 21, 0, 0, 0, 0, 1, 0, false, false, true, true},
    // the v4 counter-class kernel (scan_wp_ctr.cuh): per-series and fused, resets (drop lists), raw vectors, delta
    {1, true, filo::FN_RATE, {400, 80}, 0, 0, 300000, 10, 1, 0, 0, 0, 2, 0, false, false, true},
    {1, true, filo::FN_INCREASE, {120, 120, 60}, 0, 41, 60000, 19, 1, -30000, 30000, 0, 2, 0, false, false, true},
    {1, false, filo::FN_DELTA, {200, 100}, 0, 0, 300000, 6, 0, 0, 0, 0, 1, 0, false, false, true},
    {1, true, filo::FN_RATE, {400, 80}, 200000, 61, 300000, 13, 1, 0, 0, 0, 2, 0, false, false, true},                  // NaN markers + resets
    {1, true, filo::FN_RATE, {400, 80}, 0, 61, 300000, 13, 1, 0, 0, 0, 2, 0, false, false, true},                       // resets without NaN markers
    {1, true, filo::FN_RATE, {150, 90}, 0, 7, 300000, 21, 1, 0, 0, 0, 2, 0, false, false, true, true},                   // frequent resets (drop list overflow -> declined), shapes differ
    {1, true, filo::FN_INCREASE, {120, 120, 60}, 0, 41, 60000, 12, 1, -30000, 30000, filo::AGG_SUM, 2, 0, false, false, true},   // fused
    {1, true, filo::FN_RATE, {240, 240}, 0, 97, 300000, 17, 1, 0, 0, filo::AGG_MAX, 2, 0, false, false, true},
    {1, true, filo::FN_RATE, {100, 50, 50, 50, 50}, 0, 0, 300000, 12, 1, 0, 0, filo::AGG_SUM, 2, 0, false, false, true},  // fused, every item declined
    // irregular scrapes (DDV timestamps with residuals) on the v4 counter kernel: searched row ranges, literal fold per window
    {1, true, filo::FN_RATE, {400, 80}, 0, 61, 300000, 9, 1, 0, 0, 0, 2, 2000, false, false, true},
    {1, true, filo::FN_INCREASE, {120, 120, 60}, 50000, 41, 60000, 11, 0, -30000, 30000, 0, 2, 4000, false, false, true},
    {1, false, filo::FN_DELTA, {200, 100}, 0, 0, 300000, 6, 1, 0, 0, 0, 1, 700, false, false, true},
    {1, true, filo::FN_INCREASE, {150, 150}, 0, 45, 60000, 14, 1, 0, 0, filo::AGG_SUM, 2, 2000, false, false, true},      // fused (BASELINE C3 shape)
    {1, true, filo::FN_RATE, {240, 240}, 100000, 97, 300000, 13, 1, 15000, 0, filo::AGG_MAX, 2, 3000, false, false, true, true},
    // the v2 warp-per-series kernel on its own: every function class, irregular scrapes (DDV timestamps), integral values (DDV longs)
    {0, true, filo::FN_MIN, {150, 90}, 100000, 0, 300000, 9, 1, -30000, 15000, 0, 2, 0, false, true},
    {0, false, filo::FN_MAX, {64, 64, 64, 64, 64}, 0, 0, 200000, 7, 0, 0, 0, 0, 1, 0, false, true},
    {0, true, filo::FN_LAST, {200, 40}, 50000, 0, 300000, 6, 1, 0, 0, 0, 1, 4000, false, true},
    {0, true, filo::FN_TIMESTAMP, {100, 100}, 0, 0, 120000, 5, 1, 0, 0, 0, 1, 4000, false, true},
    {0, true, filo::FN_SUM, {120, 120}, 30000, 0, 300000, 8, 1, 0, 0, 0, 2, 4000, false, true},
    {1, false, filo::FN_RATE, {150, 150}, 0, 45, 300000, 8, 1, 0, 0, 0, 2, 0, true, true},         // integral counters with resets: DDV-long value vectors
    {1, true, filo::FN_INCREASE, {100, 100, 100}, 0, 60, 60000, 8, 1, 0, 0, 0, 2, 4000, false, true},
    // tile kernel + fallback pass: irregular scrapes make the tile kernel decline every series
    {0, true, filo::FN_RATE, {200, 100}, 0, 0, 300000, 10, 1, 0, 0, 0, 2, 4000, false, false},
    {0, true, filo::FN_RATE, {400, 80}, 100000, 0, 300000, 26, 1, 0, 0, filo::AGG_SUM, 2},   // fused sum: items of 5 series in shuffled order
    // fused min / max over +0.0 / -0.0 gauges (delta: the v4 counter kernel): of equal values the later one is kept (QueryUtils.scala:111-123)
    {0, true, filo::FN_DELTA, {400, 80}, 0, 0, 300000, 26, 1, 0, 0, filo::AGG_MIN, 2, 0, false, false, false, false, 0, 0, 0, true},
    {0, false, filo::FN_DELTA, {400, 80}, 0, 0, 300000, 26, 1, 0, 0, filo::AGG_MAX, 2, 0, false, false, false, false, 0, 0, 0, true},
  };
  // the remaining chunked range functions and the Long-column variants: window by window on the v2 kernel (eval_window_ext)
  {
    auto ext = [&](int fn, std::vector<int> chunks, int nan_ppm, int64_t window, int nser, int jitter, bool xor_enc, bool integral, int long_col, double p0, double p1, int inclusive = 1) {
      Cfg c; c.kind = 0; c.xor_enc = xor_enc; c.fn = fn; c.chunks = chunks; c.nan_ppm = nan_ppm; c.window = window; c.nser = nser; c.inclusive = inclusive;
      c.start_off = -30000; c.end_off = 30000; c.grid = 2; c.jitter = jitter; c.integral = integral; c.v2_only = true; c.long_col = long_col; c.p0 = p0; c.p1 = p1;
      all_ext.push_back(c);
    };
    const int fns[] = {filo::FN_STDDEV, filo::FN_STDVAR, filo::FN_ZSCORE, filo::FN_CHANGES, filo::FN_QUANTILE, filo::FN_MAD, filo::FN_HOLT_WINTERS, filo::FN_PREDICT_LINEAR, filo::FN_PRESENT};
    for (int fn : fns) {
      const double p0 = fn == filo::FN_QUANTILE ? 0.73 : fn == filo::FN_HOLT_WINTERS ? 0.3 : 600.0, p1 = 0.1;
      ext(fn, {100, 60, 40}, 400000, 300000, 5, 0, true, false, 0, p0, p1);                   // XOR doubles, NaN markers at chunk ends, windows over two chunks
      ext(fn, {64, 64}, 0, 120000, 4, 3000, false, false, 0, p0, p1, 0);                        // raw doubles, jittered (DDV) timestamps, exclusive range start
      ext(fn, {90, 50}, 0, 200000, 4, 0, false, true, 0, p0, p1);                               // integral doubles: DoubleLongWrap readers (DDV / const DDV)
    }
    ext(filo::FN_QUANTILE, {80, 80}, 300000, 300000, 3, 0, true, false, 0, -0.5, 0);          // q < 0 / q > 1
    ext(filo::FN_QUANTILE, {80, 80}, 300000, 300000, 3, 0, true, false, 0, 1.5, 0);
    ext(filo::FN_QUANTILE, {80, 80}, 0, 300000, 3, 0, true, false, 0, 0.0, 0);
    ext(filo::FN_QUANTILE, {80, 80}, 0, 300000, 3, 0, true, false, 0, 1.0, 0);
    const int lfns[] = {filo::FN_LAST, filo::FN_COUNT, filo::FN_SUM, filo::FN_AVG, filo::FN_MIN, filo::FN_MAX, filo::FN_STDDEV, filo::FN_STDVAR, filo::FN_CHANGES, filo::FN_QUANTILE,
                        filo::FN_PREDICT_LINEAR, filo::FN_MAD};
    for (int fn : lfns) {
      ext(fn, {70, 50, 40}, 0, 240000, 4, 0, false, false, 1, fn == filo::FN_QUANTILE ? 0.4 : 120.0, 0);     // LongBinaryVector.optimize: DDV / const DDV
      ext(fn, {70, 50}, 0, 150000, 3, 2000, false, false, 2, fn == filo::FN_QUANTILE ? 0.9 : 120.0, 0);       // raw 64-bit longs, jittered timestamps
    }
  }
  // `tile_emul <seed> fuzz <n>`: n random shapes on top of the fixed list (chunk counts / sizes, windows, offsets, functions, NaN and reset rates)
  std::vector<Cfg> all = cfgs;
  all.insert(all.end(), all_ext.begin(), all_ext.end());
  if (argc > 3 && std::string(argv[2]) == "fuzz") {
    std::mt19937_64 fr(seed * 7919 + 13);
    const int n = std::atoi(argv[3]);
    for (int i = 0; i < n; ++i) {
      Cfg c;
      c.kind = (int)(fr() % 3 == 0);
      c.xor_enc = fr() % 4 != 0;
      const int sumfns[] = {filo::FN_RATE, filo::FN_SUM, filo::FN_AVG, filo::FN_COUNT, filo::FN_INCREASE}, ctrfns[] = {filo::FN_RATE, filo::FN_INCREASE, filo::FN_DELTA};
      c.fn = c.kind ? ctrfns[fr() % 3] : sumfns[fr() % 5];
      const int nch = 1 + (int)(fr() % 4);
      int rows = 0; for (int j = 0; j < nch; ++j) { const int r = 16 + (int)(fr() % 150); c.chunks.push_back(r); rows += r; }
      c.nan_ppm = fr() % 3 == 0 ? (int)(fr() % 300000) : 0;
      c.reset_every = c.kind && fr() % 2 ? 20 + (int)(fr() % 100) : 0;
      c.window = 15000 * (int64_t)(1 + fr() % 45) + (fr() % 2 ? 0 : (int64_t)(fr() % 15000));
      c.nser = 1 + (int)(fr() % 20);
      c.inclusive = (int)(fr() % 2);
      c.start_off = (int64_t)(fr() % 7) * 15000 - 45000 + (fr() % 3 == 0 ? (int64_t)(fr() % 15000) : 0);
      c.end_off = (int64_t)(fr() % 5) * 15000 - 15000;
      c.agg_op = fr() % 5 == 0 ? (fr() % 2 ? filo::AGG_SUM : filo::AGG_MIN) : 0;
      c.grid = 1 + (int)(fr() % 3);
      c.jitter = fr() % 5 == 0 ? 300 + (int)(fr() % 5000) : 0;
      c.integral = fr() % 6 == 0; if (c.integral) c.xor_enc = false;
      c.v2_only = fr() % 4 == 0;
      fr(); fr();                      // two unused draws: a seed keeps drawing the shapes it always drew
      c.wp = fr() % 2 == 0;            // SUM class: v4 or tile kernel (the counter class always takes the v4 counter kernel)
      c.hetero = fr() % 3 == 0;
      if (c.v2_only) { const int fns[] = {filo::FN_MIN, filo::FN_MAX, filo::FN_LAST, filo::FN_TIMESTAMP, c.fn, c.fn}; c.fn = fns[fr() % 6]; c.agg_op = 0; }
      all.push_back(c);
    }
  }
  const bool quiet = all.size() > cfgs.size();
  for (size_t ci = 0; ci < all.size(); ++ci) {
    Cfg c = all[ci];
    int rows = 0; for (int n : c.chunks) rows += n;
    const int64_t t0 = 1700000000000LL; const int step_ms = 15000;
    std::vector<SeriesData> SS((size_t)c.nser);
    std::vector<int64_t> rec_off((size_t)c.nser + 1, 0);
    g_jitter_ms = c.jitter; g_integral = c.integral; g_long_col = c.long_col; g_signed_zero = c.szero;
    for (int s = 0; s < c.nser; ++s) {
      std::vector<int> cr = c.chunks; int64_t ts0 = t0; bool xe = c.xor_enc;
      if (c.hetero) {      // series-dependent chunk split, start time and encoding (runs of equal shapes in between)
        const int v = (s / 2) % 4;
        if (cr.size() >= 2) { const int mv = 8 * v + (v == 3 ? 3 : 0); if (cr[0] > mv + 8) { cr[0] -= mv; cr[1] += mv; } }
        if (v == 2) ts0 += step_ms;
        if ((s / 3) % 3 == 1) xe = !xe;
      }
      build_series(SS[(size_t)s], rng, rows, cr, ts0, step_ms, c.kind, xe, c.nan_ppm, c.reset_every); rec_off[(size_t)s + 1] = rec_off[(size_t)s] + (int64_t)SS[(size_t)s].record.size(); }
    std::vector<uint64_t> arena_backing((size_t)rec_off.back() / 8 + 64, 0);
    uint8_t* arena = reinterpret_cast<uint8_t*>(arena_backing.data());
    uint32_t max_rec = 0;
    for (int s = 0; s < c.nser; ++s) { std::memcpy(arena + rec_off[(size_t)s], SS[(size_t)s].record.data(), SS[(size_t)s].record.size()); max_rec = std::max<uint32_t>(max_rec, (uint32_t)SS[(size_t)s].record.size()); }
    filo::QueryParams q{};
    q.start = t0 + c.start_off; q.step = 15000; q.end = t0 + (int64_t)(rows - 1) * step_ms + c.end_off; q.window = c.window; q.T = (int)((q.end - q.start) / q.step) + 1;
    if (q.end < q.start) q.end = q.start;
    q.T = (int)((q.end - q.start) / q.step) + 1;
    q.fn = c.fn; q.cumulative = c.kind == 1; q.inclusive = c.inclusive; q.long_values = c.long_col ? 1 : 0; q.p0 = c.p0; q.p1 = c.p1;
    if (c.agg_op && q.T > filo::TILE_AGG_ACC * filo::TILE_THREADS) c.agg_op = 0;      // the fused tile / v4 counter paths serve T <= 512 (filo_query picks the v2 kernel beyond)
    const uint32_t wrows = (uint32_t)(q.window / q.step) + 1;
    const filo::TileSmem L = filo::tile_layout(max_rec, (uint32_t)rows, (uint32_t)q.T, 2 * wrows + 16);
    if (L.total > sizeof(filo::smem)) { std::printf("FAIL: layout %u bytes\n", L.total); return 1; }
    // oracle, per series
    std::vector<double> ref((size_t)c.nser * q.T); std::vector<int64_t> oracle_rows((size_t)c.nser, 0);
    for (int s = 0; s < c.nser; ++s) {
      fo::Series os; for (auto& ch : SS[(size_t)s].chunks) os.infos.push_back(ch->info.data());
      os.longCol = c.long_col != 0;
      fo::QueryStats st;
      fo::periodicSamples(os, oracle_fn(q.fn), q.cumulative != 0, q.start, q.step, q.end, q.window, fo::QueryConfig{q.inclusive != 0}, ref.data() + (size_t)s * q.T, &st, q.p0, q.p1);
      oracle_rows[(size_t)s] = st.samplesScanned;
    }
    std::vector<double> out((size_t)c.nser * q.T, -777.0);
    std::vector<int64_t> flist((size_t)c.nser + 8, -1); unsigned long long fcount = 0, counters[2] = {0, 0}; int derr[4] = {0, 0, 0, 0};
    Launch A{arena, rec_off.data(), c.nser, q, out.data(), L, c.grid, flist.data(), &fcount, counters, derr, nullptr, nullptr, 0, 0, nullptr, nullptr};
    if (!c.agg_op) {
      V2Shape sh{max_rec, rows, (int)c.chunks.size(), false, false};
      for (auto& S : SS) { filo::RecordHeader h; std::memcpy(&h, S.record.data(), sizeof h); sh.any_nonconst_ts |= !(h.flags & filo::REC_ALL_TS_CONST); sh.any_drop |= (h.flags & filo::REC_ANY_DROP) != 0; }
      const int cls = filo::fn_class_of(q.fn, q.cumulative, q.long_values);
      const bool tile_ok = !c.v2_only && (cls == filo::CLASS_SUM || cls == filo::CLASS_COUNTER);
      if (tile_ok && c.wp && cls == filo::CLASS_SUM) {
        const bool alias = filo::wp_max_items((uint32_t)c.chunks.size(), (uint32_t)q.T, wrows) <= 64 && !(ci % 5 == 0);      // as filo_query decides (every fifth case keeps O apart)
        filo::WpSmem W = filo::wp_layout(max_rec, (uint32_t)rows, (uint32_t)c.chunks.size(), (uint32_t)q.T, wrows, alias);
        W.warps = 3;
        if ((size_t)W.per_warp * W.warps > sizeof(filo::smem)) { std::printf("FAIL: wp layout %u bytes per warp\n", W.per_warp); return 1; }
        auto body = [&](auto fnc) {
          cusim::launch(dim3((unsigned)A.grid), dim3(W.warps * 32), [&] {
            filo::scan_wp_sum_kernel<decltype(fnc)::value, 16>(A.arena, A.rec_off, A.S, A.q, A.out, W, A.flist, A.fcount, A.counters, A.derr);
          });
        };
        if (q.fn == filo::FN_RATE) body(std::integral_constant<int, filo::FN_RATE>{});
        else if (q.fn == filo::FN_AVG) body(std::integral_constant<int, filo::FN_AVG>{});
        else if (q.fn == filo::FN_COUNT) body(std::integral_constant<int, filo::FN_COUNT>{});
        else body(std::integral_constant<int, filo::FN_SUM>{});
        if (derr[0]) { std::printf("FAIL cfg %zu: device error %d (wp kernel)\n", ci, derr[0]); return 1; }
        g_wp_declined += (long)fcount; g_wp_series += c.nser;
        if (fcount) run_v2(A, sh, flist.data(), &fcount);
      } else if (tile_ok && cls == filo::CLASS_COUNTER) {
        filo::WpCtrSmem W = filo::wp_ctr_layout(max_rec, (uint32_t)rows, (uint32_t)c.chunks.size(), (uint32_t)q.T, false, c.jitter != 0);
        W.warps = 3; W.tab = W.per_warp * W.warps;
        if ((size_t)W.tab + 4096 > sizeof(filo::smem)) { std::printf("FAIL: wp ctr layout %u bytes per warp\n", W.per_warp); return 1; }
        auto body = [&](auto fnc) {
          cusim::launch(dim3((unsigned)A.grid), dim3(W.warps * 32), [&] {
            if (W.tsr) filo::scan_wp_ctr_kernel<decltype(fnc)::value, false, 16, true>(A.arena, A.rec_off, A.S, A.q, A.out, W, A.flist, A.fcount, A.counters, A.derr, nullptr, nullptr, 0, 0, nullptr, nullptr);
            else filo::scan_wp_ctr_kernel<decltype(fnc)::value, false, 16, false>(A.arena, A.rec_off, A.S, A.q, A.out, W, A.flist, A.fcount, A.counters, A.derr, nullptr, nullptr, 0, 0, nullptr, nullptr);
          });
        };
        if (q.fn == filo::FN_RATE) body(std::integral_constant<int, filo::FN_RATE>{});
        else if (q.fn == filo::FN_INCREASE) body(std::integral_constant<int, filo::FN_INCREASE>{});
        else body(std::integral_constant<int, filo::FN_DELTA>{});
        if (derr[0]) { std::printf("FAIL cfg %zu: device error %d (wp ctr kernel)\n", ci, derr[0]); return 1; }
        g_wp_declined += (long)fcount; g_wp_series += c.nser;
        if (fcount) run_v2(A, sh, flist.data(), &fcount);
      } else if (tile_ok) {
        dispatch<false>(A);
        if (derr[0]) { std::printf("FAIL cfg %zu: device error %d (tile kernel)\n", ci, derr[0]); return 1; }
        if (fcount) run_v2(A, sh, flist.data(), &fcount);               // the fallback pass, as filo_query chains it
      } else run_v2(A, sh, nullptr, nullptr);
      if (derr[0]) { std::printf("FAIL cfg %zu: device error %d\n", ci, derr[0]); return 1; }
      int64_t exp_rows = 0;
      for (int s = 0; s < c.nser; ++s) {
        exp_rows += oracle_rows[(size_t)s];
        for (int k = 0; k < q.T; ++k) {
          const double a = out[(size_t)s * q.T + k], r = ref[(size_t)s * q.T + k];
          if (!same_bits(a, r)) { std::printf("FAIL cfg %zu series %d window %d: %.17g vs %.17g\n", ci, s, k, a, r); return 1; }
          ++checked;
        }
      }
      if ((int64_t)counters[0] != exp_rows) { std::printf("FAIL cfg %zu: samples_scanned %llu vs %lld\n", ci, counters[0], (long long)exp_rows); return 1; }
      if (tile_ok && c.chunks.size() > (size_t)filo::TILE_MAXC && fcount != (unsigned long long)c.nser) { std::printf("FAIL cfg %zu: series with too many chunks were not declined\n", ci); return 1; }
      if (!quiet) std::printf("cfg %zu ok: %d series (%llu to the fallback list), T=%d\n", ci, c.nser, fcount, q.T);
    } else {
      // items of <= 5 series in a shuffled order (what build_groups produces for one group)
      std::vector<int32_t> order((size_t)c.nser); for (int s = 0; s < c.nser; ++s) order[(size_t)s] = s;
      std::shuffle(order.begin(), order.end(), rng);
      std::vector<int64_t> item_begin; for (int64_t p = 0; p < c.nser; p += 5) item_begin.push_back(p); item_begin.push_back(c.nser);
      const int64_t n_items = (int64_t)item_begin.size() - 1;
      std::vector<double> pval((size_t)n_items * q.T, -777.0); std::vector<uint32_t> pcnt((size_t)n_items * q.T, 12345u);
      A.order = order.data(); A.item_begin = item_begin.data(); A.n_items = n_items; A.agg_op = c.agg_op; A.pval = pval.data(); A.pcnt = pcnt.data(); A.out = nullptr;
      if (filo::fn_class_of(q.fn, q.cumulative) == filo::CLASS_COUNTER) {
        filo::WpCtrSmem W = filo::wp_ctr_layout(max_rec, (uint32_t)rows, (uint32_t)c.chunks.size(), (uint32_t)q.T, true, c.jitter != 0);
        W.warps = 3; W.tab = W.per_warp * W.warps;
        if ((size_t)W.tab + 4096 > sizeof(filo::smem)) { std::printf("FAIL: wp ctr layout %u bytes per warp\n", W.per_warp); return 1; }
        auto body = [&](auto fnc) {
          cusim::launch(dim3((unsigned)A.grid), dim3(W.warps * 32), [&] {
            if (W.tsr) filo::scan_wp_ctr_kernel<decltype(fnc)::value, true, 16, true>(A.arena, A.rec_off, A.S, A.q, nullptr, W, A.flist, A.fcount, A.counters, A.derr, A.order, A.item_begin, A.n_items, A.agg_op, A.pval, A.pcnt);
            else filo::scan_wp_ctr_kernel<decltype(fnc)::value, true, 16, false>(A.arena, A.rec_off, A.S, A.q, nullptr, W, A.flist, A.fcount, A.counters, A.derr, A.order, A.item_begin, A.n_items, A.agg_op, A.pval, A.pcnt);
          });
        };
        if (q.fn == filo::FN_RATE) body(std::integral_constant<int, filo::FN_RATE>{});
        else if (q.fn == filo::FN_INCREASE) body(std::integral_constant<int, filo::FN_INCREASE>{});
        else body(std::integral_constant<int, filo::FN_DELTA>{});
      } else dispatch<true>(A);
      if (derr[0]) { std::printf("FAIL cfg %zu: device error %d\n", ci, derr[0]); return 1; }
      if (fcount) {                                                     // declined items: the fused v2 kernel, as filo_query chains it
        V2Shape sh{max_rec, rows, (int)c.chunks.size(), false, false};
        for (auto& S : SS) { filo::RecordHeader h; std::memcpy(&h, S.record.data(), sizeof h); sh.any_nonconst_ts |= !(h.flags & filo::REC_ALL_TS_CONST); sh.any_drop |= (h.flags & filo::REC_ANY_DROP) != 0; }
        run_agg_v2(A, sh, flist.data(), &fcount);
        if (derr[0]) { std::printf("FAIL cfg %zu: device error %d (fused fallback)\n", ci, derr[0]); return 1; }
      }
      for (int64_t it = 0; it < n_items; ++it) {
        for (int k = 0; k < q.T; ++k) {
          double a = c.agg_op == filo::AGG_MIN ? INFINITY : c.agg_op == filo::AGG_MAX ? -INFINITY : 0.0; uint32_t n = 0;
          for (int64_t p = item_begin[(size_t)it]; p < item_begin[(size_t)it + 1]; ++p) {
            const double v = ref[(size_t)order[(size_t)p] * q.T + k];
            if (v == v) { if (c.agg_op == filo::AGG_MIN) a = fo::minIgnoreNaN(a, v); else if (c.agg_op == filo::AGG_MAX) a = fo::maxIgnoreNaN(a, v); else if (c.agg_op != filo::AGG_COUNT) a += v; ++n; }
          }
          if (!same_bits(pval[(size_t)it * q.T + k], a) || pcnt[(size_t)it * q.T + k] != n) { std::printf("FAIL cfg %zu item %lld window %d: %.17g (%u) vs %.17g (%u)\n", ci, (long long)it, k, pval[(size_t)it * q.T + k], pcnt[(size_t)it * q.T + k], a, n); return 1; }
          ++checked;
        }
      }
#ifdef HAVE_MERGE_KERNEL
      {   // merge_partials_kernel: one group over all items; thread (window, lane j) folds items j, j+8, ... and the 8 lanes fold in order
        const int64_t gis[2] = {0, n_items};
        std::vector<double> mv((size_t)q.T, -777.0); std::vector<int64_t> mc((size_t)q.T, -1);
        const int ktiles = (q.T + 31) / 32;
        cusim::launch(dim3((unsigned)ktiles), dim3(256), [&] { filo::merge_partials_kernel(pval.data(), pcnt.data(), gis, 1, q.T, c.agg_op, 0, mv.data(), mc.data()); });
        for (int k = 0; k < q.T; ++k) {
          const double ident = c.agg_op == filo::AGG_MIN ? INFINITY : c.agg_op == filo::AGG_MAX ? -INFINITY : 0.0;
          double lane_a[8]; unsigned long long lane_c[8];
          for (int j = 0; j < 8; ++j) {
            double a = ident; unsigned long long n = 0;
            for (int64_t it = j; it < n_items; it += 8) { const double v = pval[(size_t)it * q.T + k]; const uint32_t m = pcnt[(size_t)it * q.T + k];
              if (m) { if (c.agg_op == filo::AGG_MIN) a = fo::minIgnoreNaN(a, v); else if (c.agg_op == filo::AGG_MAX) a = fo::maxIgnoreNaN(a, v); else a += v; n += m; } }
            lane_a[j] = a; lane_c[j] = n;
          }
          double a = lane_a[0]; unsigned long long n = lane_c[0];
          for (int j = 1; j < 8; ++j) if (lane_c[j]) { const double v = lane_a[j]; if (c.agg_op == filo::AGG_MIN) a = fo::minIgnoreNaN(a, v); else if (c.agg_op == filo::AGG_MAX) a = fo::maxIgnoreNaN(a, v); else a += v; n += lane_c[j]; }
          const double e = n == 0 ? std::nan("") : c.agg_op == filo::AGG_AVG ? a / (double)n : c.agg_op == filo::AGG_COUNT ? (double)n : a;
          if (!same_bits(mv[(size_t)k], e) || mc[(size_t)k] != (int64_t)n) { std::printf("FAIL cfg %zu merged window %d: %.17g (%lld) vs %.17g (%llu)\n", ci, k, mv[(size_t)k], (long long)mc[(size_t)k], e, n); return 1; }
          ++checked;
        }
      }
#endif
      if (!quiet) std::printf("cfg %zu ok: %d series in %lld items (%llu to the fallback list), T=%d\n", ci, c.nser, (long long)n_items, fcount, q.T);
    }
    ++cases;
  }
  std::printf("wp kernel: %ld of %ld series declined\n", g_wp_declined, g_wp_series);
  std::printf("OK %d cases, %ld values bit-exact (schedule seed %llu)\n", cases, checked, (unsigned long long)seed);
  return 0;
}
