// C++ host-side mirror of the reference's operator interface for this path, over the C-ABI of filo_b200.h.
//
// The reference's host code is Scala; no JVM toolchain exists where this repo is built, so the operator surface is restated in
// C++ with the reference's names, argument meaning and error behaviour:
//   RangeVectorTransformer            query/src/main/scala/filodb/query/exec/RangeVectorTransformer.scala:36-55
//   PeriodicSamplesMapper             query/src/main/scala/filodb/query/exec/PeriodicSamplesMapper.scala:27-76
//   AggregateMapReduce                query/src/main/scala/filodb/query/exec/AggrOverRangeVectors.scala:119-182
//   InstantVectorFunctionMapper(HistogramQuantile)   query/src/main/scala/filodb/query/exec/RangeVectorTransformer.scala:61-110
//   RawDataRangeVector.chunkInfos     core/src/main/scala/filodb.core/query/RangeVector.scala:365-389
// A query is the same chain of transformers the planner builds (ExecPlan.addRangeVectorTransformer); FusedGpuExec.execute()
// recognises the chain [PeriodicSamplesMapper, AggregateMapReduce?, InstantVectorFunctionMapper(HistogramQuantile)?] and runs
// it as one call into the device library.  Illegal arguments throw std::invalid_argument (Scala `require`), engine errors
// throw filo::QueryError carrying the C-ABI status and message (the JNI shim maps them to RuntimeException).
#pragma once
#include "filo_b200.h"

#include <cmath>
#include <cstdint>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <vector>

namespace filo {

struct QueryError : std::runtime_error {
  int32_t status;
  QueryError(int32_t st, const std::string& msg) : std::runtime_error(msg), status(st) {}
};

// InternalRangeFunction (query/src/main/scala/filodb/query/exec/RangeFunctionId.scala) subset served by the device path
enum class InternalRangeFunction : int32_t {
  LastSample = FILO_FN_LAST, Rate = FILO_FN_RATE, Increase = FILO_FN_INCREASE, Delta = FILO_FN_DELTA,
  SumOverTime = FILO_FN_SUM_OVER_TIME, AvgOverTime = FILO_FN_AVG_OVER_TIME, CountOverTime = FILO_FN_COUNT_OVER_TIME,
  MinOverTime = FILO_FN_MIN_OVER_TIME, MaxOverTime = FILO_FN_MAX_OVER_TIME, Timestamp = FILO_FN_TIMESTAMP,
  StdDevOverTime = FILO_FN_STDDEV_OVER_TIME, StdVarOverTime = FILO_FN_STDVAR_OVER_TIME, Changes = FILO_FN_CHANGES,
  QuantileOverTime = FILO_FN_QUANTILE_OVER_TIME, ZScore = FILO_FN_ZSCORE, HoltWinters = FILO_FN_HOLT_WINTERS,
  PredictLinear = FILO_FN_PREDICT_LINEAR, MedianAbsoluteDeviationOverTime = FILO_FN_MAD_OVER_TIME, PresentOverTime = FILO_FN_PRESENT_OVER_TIME,
  AvgWithSumAndCountOverTime = 1000     // downsample schemas (RangeFunction.downsampleRangeFunction): two value columns, filo_query_avg_sum_count
};
// AggregationOperator (query/src/main/scala/filodb/query/PlanEnums.scala) subset
enum class AggregationOperator : int32_t {
  Sum = FILO_AGG_SUM, Avg = FILO_AGG_AVG, Min = FILO_AGG_MIN, Max = FILO_AGG_MAX, Count = FILO_AGG_COUNT,
  TopK = FILO_AGG_TOPK, BottomK = FILO_AGG_BOTTOMK, Stddev = FILO_AGG_STDDEV, Stdvar = FILO_AGG_STDVAR, Group = FILO_AGG_GROUP
};

// RawDataRangeVector: one partition's chunks for the query range (ChunkSetInfo native addresses in chunkID order) + the group
// ordinal its RangeVectorKey maps to under the query's by/without clause (AggrOverRangeVectors.scala:150-159).
struct RawDataRangeVector {
  std::vector<uint64_t> chunkInfoAddrs;
  int32_t group = 0;
};

struct RangeVectorTransformer { virtual ~RangeVectorTransformer() = default; };

struct PeriodicSamplesMapper : RangeVectorTransformer {
  int64_t startMs, stepMs, endMs;
  std::optional<int64_t> window;
  std::optional<InternalRangeFunction> functionId;
  std::vector<double> funcParams;              // StaticFuncArgs scalars: quantile_over_time(q), holt_winters(sf, tf), predict_linear(seconds)
  PeriodicSamplesMapper(int64_t start, int64_t step, int64_t end, std::optional<int64_t> windowMs, std::optional<InternalRangeFunction> fn,
                        std::vector<double> params = {})
      : startMs(start), stepMs(step), endMs(end), window(windowMs), functionId(fn), funcParams(std::move(params)) {
    // PeriodicSamplesMapper.scala:45-49
    if (!(start <= end)) throw std::invalid_argument("requirement failed: start " + std::to_string(start) + " should be <= end " + std::to_string(end));
    if (!(start == end || step > 0)) throw std::invalid_argument("requirement failed: step should be > 0 for range query");
    if (fn && fn != InternalRangeFunction::LastSample && fn != InternalRangeFunction::Timestamp && !(windowMs && *windowMs > 0))
      throw std::invalid_argument("requirement failed: Need positive window lengths to apply range function");
  }
};

struct AggregateMapReduce : RangeVectorTransformer {
  AggregationOperator aggrOp; std::vector<double> aggrParams; int32_t numGroups;
  AggregateMapReduce(AggregationOperator op, std::vector<double> params, int32_t nGroups) : aggrOp(op), aggrParams(std::move(params)), numGroups(nGroups) {
    if ((op == AggregationOperator::TopK || op == AggregationOperator::BottomK) && aggrParams.size() != 1)
      throw std::invalid_argument("requirement failed: topk/bottomk need one parameter");
  }
};

struct HistogramQuantileMapper : RangeVectorTransformer {      // InstantVectorFunctionMapper(InstantFunctionId.HistogramQuantile, Seq(q))
  double q;
  explicit HistogramQuantileMapper(double quantile) : q(quantile) {}
};

struct QueryResult {
  int32_t rows = 0, windows = 0, buckets = 0;     // rows = series (no aggregate) or groups; buckets > 0: histogram rows
  std::vector<double> values;                     // [rows * windows (* k | * buckets)]
  std::vector<int64_t> aux;                       // avg counts / topk series ordinals
  filo_stats stats{};
  int64_t timestamp(int i, int64_t startMs, int64_t stepMs) const { (void)windows; return startMs + (int64_t)i * stepMs; }   // RvRange
};

// One shard's query context on one GPU.
class FusedGpuExec {
 public:
  explicit FusedGpuExec(int device = 0, const filo_cfg* cfg = nullptr) {
    const int32_t rc = filo_ctx_create(device, cfg, &ctx_);
    if (rc != FILO_OK) throw QueryError(rc, "filo_ctx_create failed (is there a CUDA device?)");
  }
  ~FusedGpuExec() { filo_ctx_destroy(ctx_); }
  FusedGpuExec(const FusedGpuExec&) = delete;
  FusedGpuExec& operator=(const FusedGpuExec&) = delete;

  // ExecPlan.execute step 2 for the chain of transformers over the shard's raw range vectors (timestamp column 0, value column
  // `valueColumn`); `cumulative` = the schema's counter flag, `histogram` = the value column is a histogram column.
  QueryResult execute(const std::vector<RawDataRangeVector>& source, const PeriodicSamplesMapper& psm, const AggregateMapReduce* aggr = nullptr,
                      const HistogramQuantileMapper* quantile = nullptr, int valueColumn = 1, bool cumulative = false, bool histogram = false) {
    std::vector<int32_t> nChunks; std::vector<uint64_t> addrs; std::vector<int32_t> groups;
    for (const auto& rv : source) { nChunks.push_back((int32_t)rv.chunkInfoAddrs.size()); addrs.insert(addrs.end(), rv.chunkInfoAddrs.begin(), rv.chunkInfoAddrs.end()); groups.push_back(rv.group); }
    const int32_t nGroups = aggr ? aggr->numGroups : 0;
    if (psm.functionId == InternalRangeFunction::AvgWithSumAndCountOverTime) {
      // AvgWithSumAndCountOverTimeFuncD(schema.colIDs(2)) (RangeFunction.scala:360-362): sum column = valueColumn, count column = the next one
      if (aggr || histogram) throw QueryError(FILO_ERR_UNSUPPORTED, "AvgWithSumAndCountOverTime: per-series rows of double columns only");
      filo_table *ts = nullptr, *tc = nullptr;
      check(filo_load_series(ctx_, (int64_t)source.size(), nChunks.data(), addrs.data(), 0, valueColumn, nullptr, 0, 0, &ts));
      struct Free { filo_ctx* c; filo_table* t; ~Free() { filo_table_free(c, t); } } gs{ctx_, ts};
      check(filo_load_series(ctx_, (int64_t)source.size(), nChunks.data(), addrs.data(), 0, valueColumn + 1, nullptr, 0, 0, &tc));
      Free gc{ctx_, tc};
      QueryResult r; r.windows = filo_num_windows(psm.startMs, psm.stepMs, psm.endMs); r.rows = (int32_t)source.size();
      r.values.assign((size_t)r.rows * r.windows, 0.0);
      check(filo_query_avg_sum_count(ctx_, ts, tc, psm.startMs, psm.stepMs, psm.endMs, psm.window.value_or(0), r.values.data(), &r.stats));
      return r;
    }
    filo_table* t = nullptr;
    check(filo_load_series(ctx_, (int64_t)source.size(), nChunks.data(), addrs.data(), 0, valueColumn, aggr ? groups.data() : nullptr, nGroups,
                           cumulative ? FILO_SCHEMA_CUMULATIVE : 0, &t));
    struct Free { filo_ctx* c; filo_table* t; ~Free() { filo_table_free(c, t); } } guard{ctx_, t};
    const int32_t fn = (int32_t)psm.functionId.value_or(InternalRangeFunction::LastSample);
    const int64_t window = psm.window.value_or(0);
    check(filo_ctx_set_fn_args(ctx_, psm.funcParams.size() > 0 ? psm.funcParams[0] : 0.0, psm.funcParams.size() > 1 ? psm.funcParams[1] : 0.0));
    QueryResult r; r.windows = filo_num_windows(psm.startMs, psm.stepMs, psm.endMs);
    if (histogram) {
      filo_table_info ti{}; filo_table_get_info(t, &ti);
      r.rows = aggr ? nGroups : (int32_t)source.size();
      if (aggr && aggr->aggrOp != AggregationOperator::Sum) throw QueryError(FILO_ERR_UNSUPPORTED, "histogram aggregates: sum only");
      if (quantile) {                             // [rows][T]: the quantile of each group's sum, or of each series' own histogram
        r.values.assign((size_t)r.rows * r.windows, 0.0);
        check(filo_query_hist(ctx_, t, fn, psm.startMs, psm.stepMs, psm.endMs, window, aggr ? FILO_AGG_SUM : FILO_AGG_NONE, quantile->q, nullptr, r.values.data(), &r.stats));
      } else {
        r.buckets = ti.hist_buckets; r.values.assign((size_t)r.rows * r.windows * r.buckets, 0.0);
        check(filo_query_hist(ctx_, t, fn, psm.startMs, psm.stepMs, psm.endMs, window, aggr ? FILO_AGG_SUM : FILO_AGG_NONE, std::nan(""), r.values.data(), nullptr, &r.stats));
      }
      return r;
    }
    if (!aggr) {                                  // plain PeriodicSamplesMapper: the pipelined load + scan + read-back call
      r.rows = (int32_t)source.size(); r.values.assign((size_t)r.rows * r.windows, 0.0);
      check(filo_scan_series(ctx_, (int64_t)source.size(), nChunks.data(), addrs.data(), 0, valueColumn, cumulative ? FILO_SCHEMA_CUMULATIVE : 0,
                             fn, psm.startMs, psm.stepMs, psm.endMs, window, r.values.data(), &r.stats));
      return r;
    }
    int32_t k = 0, op = FILO_AGG_NONE;
    if (aggr) { op = (int32_t)aggr->aggrOp; if (op == FILO_AGG_TOPK || op == FILO_AGG_BOTTOMK) k = (int32_t)aggr->aggrParams[0]; }
    r.rows = aggr ? nGroups : (int32_t)source.size();
    const size_t n = (size_t)r.rows * r.windows * (k ? k : 1);
    r.values.assign(n, 0.0);
    if (op == FILO_AGG_AVG || k) r.aux.assign(n, 0);
    check(filo_query(ctx_, t, fn, psm.startMs, psm.stepMs, psm.endMs, window, op, k, 0, r.values.data(), r.aux.empty() ? nullptr : r.aux.data(), &r.stats));
    return r;
  }

 private:
  void check(int32_t rc) {
    if (rc == FILO_OK) return;
    char msg[512]; filo_last_error(ctx_, msg, (int32_t)sizeof msg);
    if (rc == FILO_ERR_INVALID_ARG) throw std::invalid_argument(std::string("requirement failed: ") + msg);
    throw QueryError(rc, msg);
  }
  filo_ctx* ctx_ = nullptr;
};

} // namespace filo
