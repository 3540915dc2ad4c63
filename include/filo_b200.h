/*
 * filo_b200.h — C-ABI of the H100-native chunk-scan + range-vector aggregation engine for FiloDB.
 *
 * This is the drop-in boundary: a JVM (FiloDB) process binds these symbols through the JNI shim
 * (filodb_b200/csrc/jni_shim.cpp, see INTEGRATION.md) exactly the way the reference binds its existing
 * native seam on this path:
 *     core/src/main/scala/filodb.memory/format/vectors/SimdNativeMethods.scala:68-86   (@native simdSumDouble/...)
 *     core/src/rust/filodb_core/src/simd_vectors.rs:163-200                            (Java_..._simdSumDouble)
 * Conventions mirrored from that seam (core/src/rust/filodb_core/src/exec.rs:15-61, errors.rs:36-47, lib.rs:5-17):
 *   - primitives and raw addresses only (jlong addresses of off-heap BinaryVectors / ChunkSetInfos);
 *   - no exception/abort ever crosses the boundary: every entry returns an int32 status (0 = OK, <0 = error) and
 *     the message is fetched with filo_last_error(); the JNI shim turns non-zero into java.lang.RuntimeException;
 *   - the callee COPIES chunk bytes during filo_load_series and never retains host pointers: the caller holds the
 *     partition ChunkMap shared locks + shard eviction lock only for the duration of that call
 *     (core/src/main/scala/filodb.memory/data/ChunkMap.scala:17-41, EvictionLock.scala:24-32).
 *
 * What the entry points replace (reference file:line):
 *   filo_load_series  <- RawDataRangeVector.chunkInfos / WindowedChunkIterator chunk resolution
 *                        core/src/main/scala/filodb.core/query/RangeVector.scala:365-399
 *                        core/src/main/scala/filodb.core/store/ChunkSetInfo.scala:445-529 (ChunkSetInfo layout :133-154)
 *   filo_query        <- PeriodicSamplesMapper.apply -> ChunkedWindowIteratorD.doNext -> ChunkedRangeFunction.addChunks/apply
 *                        query/src/main/scala/filodb/query/exec/PeriodicSamplesMapper.scala:61-190, 256-347
 *                        query/src/main/scala/filodb/query/exec/rangefn/RangeFunction.scala:84-242, 595-724
 *                        query/src/main/scala/filodb/query/exec/rangefn/RateFunctions.scala:72-111, 230-322, 424-445
 *                        query/src/main/scala/filodb/query/exec/rangefn/AggrOverTimeFunctions.scala:40-116, 553-572, 924-1015
 *                        + AggregateMapReduce.apply / RangeVectorAggregator.mapReduce / RowAggregators
 *                        query/src/main/scala/filodb/query/exec/AggrOverRangeVectors.scala:119-182, 214-378
 *                        query/src/main/scala/filodb/query/exec/aggregator/{Sum,Min,Max,Count,Avg,TopBottomK}RowAggregator.scala
 *   filo_synth_table  <- (bench/test only) TestTimeseriesProducer + the appenders' optimize()
 *                        gateway/src/main/scala/filodb/timeseries/TestTimeseriesProducer.scala:147,196-198
 *
 * Output timestamps are implicit: window i ends at start_ms + i*step_ms (RvRange, PeriodicSamplesMapper.scala:48).
 * There is NO CPU fallback: every query runs the sm_90a kernels; a missing/failed device is an error.
 */
#ifndef FILO_B200_H
#define FILO_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct filo_ctx filo_ctx;
typedef struct filo_table filo_table;

/* status codes */
enum {
  FILO_OK = 0,
  FILO_ERR_INVALID_ARG = -1,
  FILO_ERR_CUDA = -2,
  FILO_ERR_CORRUPT_VECTOR = -3,     /* CorruptVectorException, ChunkSetInfo.scala:424-429 */
  FILO_ERR_UNSUPPORTED = -4,        /* encoding/ordering the device path does not handle; caller keeps the JVM path */
  FILO_ERR_QUERY_LIMIT = -5,        /* QueryLimitException: scanned-bytes / group-by cardinality limits */
  FILO_ERR_BAD_QUERY = -6,          /* BadQueryException: step below min-step */
  FILO_ERR_OOM = -7
};

/* InternalRangeFunction subset on this path (query/.../exec/InternalRangeFunction.scala:11-70) */
enum {
  FILO_FN_LAST = 0,                 /* None / Last                 -> LastSampleChunkedFunctionD */
  FILO_FN_RATE = 1,                 /* Rate      (CumlDeltaToggler: counter -> ChunkedRateFunction, else RateOverDelta) */
  FILO_FN_INCREASE = 2,             /* Increase  (counter -> ChunkedIncreaseFunction, else SumOverTime) */
  FILO_FN_DELTA = 3,                /* ChunkedDeltaFunction */
  FILO_FN_SUM_OVER_TIME = 4,
  FILO_FN_AVG_OVER_TIME = 5,
  FILO_FN_COUNT_OVER_TIME = 6,
  FILO_FN_MIN_OVER_TIME = 7,
  FILO_FN_MAX_OVER_TIME = 8,
  FILO_FN_TIMESTAMP = 9,
  /* the other chunked range functions of RangeFunction.doubleChunkedFunction (RangeFunction.scala:341-375); static arguments
   * (funcParams) come from filo_ctx_set_fn_args */
  FILO_FN_STDDEV_OVER_TIME = 10,    /* StdDevOverTimeChunkedFunctionD / L   AggrOverTimeFunctions.scala:1082-1183 */
  FILO_FN_STDVAR_OVER_TIME = 11,
  FILO_FN_CHANGES = 12,             /* ChangesChunkedFunctionD / L          :1185-1225 */
  FILO_FN_QUANTILE_OVER_TIME = 13,  /* arg0 = q                             :1227-1344 */
  FILO_FN_ZSCORE = 14,              /* ZScoreChunkedFunctionD               :1592-1604 */
  FILO_FN_HOLT_WINTERS = 15,        /* arg0 = sf, arg1 = tf, both in [0,1]  :1361-1453 */
  FILO_FN_PREDICT_LINEAR = 16,      /* arg0 = duration in seconds           :1496-1590 */
  FILO_FN_MAD_OVER_TIME = 17,       /* MedianAbsoluteDeviationOverTime      :1248-1359 */
  FILO_FN_PRESENT_OVER_TIME = 18    /* PresentOverTimeChunkedFunctionD      RangeFunction.scala:725-748 */
};

/* AggregationOperator subset (query/src/main/scala/filodb/query/PlanEnums.scala:99-114) */
enum {
  FILO_AGG_NONE = 0, FILO_AGG_SUM = 1, FILO_AGG_AVG = 2, FILO_AGG_MIN = 3, FILO_AGG_MAX = 4,
  FILO_AGG_COUNT = 5, FILO_AGG_TOPK = 6, FILO_AGG_BOTTOMK = 7,
  /* RowAggregator.apply (aggregator/RowAggregator.scala:133,138-139): StddevRowAggregator.scala:39-58,
   * StdvarRowAggregator.scala:52-72 (sumSquare/count - mean^2, sqrt of it for stddev), GroupRowAggregator.scala:23-29
   * (1.0 where any input is non-NaN).  Scalar tables only: histogram tables answer FILO_ERR_UNSUPPORTED. */
  FILO_AGG_STDDEV = 8, FILO_AGG_STDVAR = 9, FILO_AGG_GROUP = 10
};

/* schema_flags of filo_load_series */
enum {
  FILO_SCHEMA_CUMULATIVE = 1,       /* schema.hasCumulativeTemporalityColumn (detectDrops column), Schemas.scala:190-193 */
  FILO_SCHEMA_LONG_VALUES = 2       /* the value column is a LongColumn: LongBinaryVector readers and the *L chunked functions
                                       (RangeFunction.scala:300-339); functions without an L variant answer FILO_ERR_UNSUPPORTED */
};

/* query flags */
enum {
  FILO_Q_PARTIAL = 1                /* aggregates are returned in mergeable form for the cross-GPU reduce (see filo_query_device) */
};

typedef struct {
  int32_t inclusive_range;            /* filodb.query.inclusive-range (filodb-defaults.conf:590), default 1 */
  int32_t group_by_cardinality_limit; /* enforcedLimits.groupByCardinality, 0 = unlimited (AggrOverRangeVectors.scala:237-246) */
  int64_t min_step_ms;                /* filodb.query.min-step (filodb-defaults.conf:626), 0 = not enforced */
  int64_t max_data_per_shard_query;   /* bytes, 0 = unlimited (ChunkSetInfo.scala:361-368) */
} filo_cfg;

typedef struct {
  int64_t bytes_scanned;              /* Σ totalBytes(ts)+totalBytes(value) of chunks scanned (dataBytesScannedCtr) */
  int64_t samples_scanned;            /* Σ numRows of chunks scanned (samplesScannedCtr, ChunkSetInfo.scala:360) */
  int64_t kernel_ns;                  /* device time of the kernels of this call (CUDA events) */
  int64_t h2d_bytes;
  int64_t d2h_bytes;
  int64_t kernel_launches;
} filo_stats;

typedef struct {
  int64_t n_series;
  int64_t n_chunks;
  int64_t n_samples;                  /* Σ numRows */
  int64_t arena_bytes;                /* device bytes of the chunk arena (records + index) */
  int64_t algorithmic_bytes;          /* Σ chunks (28 + 8*ncols + totalBytes(ts) + totalBytes(value)), SURVEY §8(d) */
  int32_t max_rows_per_series;
  int32_t max_chunks_per_series;
  int32_t n_groups;
  int32_t schema_flags;
  int32_t hist_buckets;               /* > 0: histogram table with this many buckets */
  int32_t reserved;
} filo_table_info;

/* Synthetic table spec (bench + tests): the reference's own generator shapes, encoded on the GPU.
 * value_kind: 0 gauge  15 + sin(n+1) + N(0,1)            (TestTimeseriesProducer.scala:147)
 *             1 counter v += max(0, 15 + sin + N(0,1))    (TestTimeseriesProducer.scala:196-198), resets ~1/reset_period rows
 *             2 integral counter (values rounded -> DeltaDeltaVector-as-long encoding, DoubleVector.scala:86-96)
 * value_enc:  0 raw f64 (DoubleVector.optimize for non-integral data), 1 XOR-NibblePack container, 2 DoubleVector.optimize (DDV if integral)
 * ts_jitter_ms: 0 -> regular scrapes (const DDV, 24 bytes); >250 -> DeltaDeltaVector with residuals */
typedef struct {
  int64_t n_series;
  int32_t rows_per_series;
  int32_t rows_per_chunk;             /* max-chunks-size (400) */
  int64_t t0_ms;
  int32_t interval_ms;
  int32_t ts_jitter_ms;
  int32_t value_kind;
  int32_t value_enc;
  int32_t reset_period;               /* counters: expected rows between resets (0 = never) */
  int32_t nan_per_million;            /* stale markers: probability (ppm) that a chunk's last row is NaN */
  int32_t n_groups;                   /* group id = hash(series) % n_groups (0 -> no grouping) */
  int32_t schema_flags;
  uint64_t seed;
  int64_t series_id_base;             /* global id of series 0 of this table (multi-GPU shards generate disjoint ids) */
  const double* sin_table;            /* host pointer, rows_per_series doubles: sin(n+1) as computed by the caller */
} filo_synth_spec;

int32_t filo_ctx_create(int32_t device_ordinal, const filo_cfg* cfg /* NULL = defaults */, filo_ctx** out);
void    filo_ctx_destroy(filo_ctx* ctx);
/* Static arguments of the range function of the following queries on this ctx -- the reference's funcParams: Seq[StaticFuncArgs]
 * (RangeFunction.generatorFor, RangeFunction.scala:283-313): quantile_over_time(arg0), holt_winters(arg0 = sf, arg1 = tf),
 * predict_linear(arg0 = seconds).  Other functions ignore them. */
int32_t filo_ctx_set_fn_args(filo_ctx* ctx, double arg0, double arg1);
/* Waits for the non-synchronising queries issued on this ctx (filo_query_device with stats == NULL) and returns the first device-side
 * error among them (CorruptVector, scratch overflow), FILO_OK otherwise.  Such errors are also returned by the next call on the ctx
 * that finds them complete. */
int32_t filo_ctx_check(filo_ctx* ctx);
/* Copies the last error message of this ctx (thread-local when ctx is NULL) into buf; returns its length. */
int32_t filo_last_error(filo_ctx* ctx, char* buf, int32_t len);

/* Ingest a set of time series into a device chunk arena.
 *  n_chunks[i]        chunks of series i, in increasing chunkID order (what partition.infos yields)
 *  chunk_info_addrs   Σ n_chunks native addresses of ChunkSetInfo blocks (ChunkSetInfo.scala:133-154); vector pointers
 *                     inside them are dereferenced for columns ts_col / val_col
 *  group_ids          per-series group ordinal in [0, n_groups) for a later across-series aggregate, or NULL */
int32_t filo_load_series(filo_ctx* ctx, int64_t n_series, const int32_t* n_chunks, const uint64_t* chunk_info_addrs,
                         int32_t ts_col, int32_t val_col, const int32_t* group_ids, int32_t n_groups,
                         int32_t schema_flags, filo_table** out);
/* Incremental arena: appends new chunks to the series of a resident table (same series, in the table's order; n_chunks[i] may be 0) --
 * what TimeSeriesPartition.switchBuffers / encodeOneChunkset produce at a flush (TimeSeriesPartition.scala:251-288).  Only the new
 * chunks cross PCIe; the records are re-packed on the device into a new arena that is byte-identical to filo_load_series over all the
 * chunks (old arena + new arena are resident during the call).  New chunks must follow the resident ones in time (else
 * FILO_ERR_UNSUPPORTED and the table is unchanged).  The handle, its grouping and queries in flight on other streams: the caller
 * serialises appends against queries of the same table. */
int32_t filo_table_append(filo_ctx* ctx, filo_table* t, const int32_t* n_chunks, const uint64_t* chunk_info_addrs, int32_t ts_col, int32_t val_col);
int32_t filo_synth_table(filo_ctx* ctx, const filo_synth_spec* spec, filo_table** out);
/* GPU-side encode of an ingest batch: raw samples -- timestamps / values row-major [n_series][rows_per_series] in HOST memory, strictly
 * increasing timestamps per series -- are encoded on the device into the chunk vectors the reference's appenders + optimize() write
 * (timestamps: DeltaDeltaVector.fromLongVector incl. the +-250 ms approximate-const rule, DeltaDeltaVector.scala:20-80; values by
 * value_enc: 0 raw doubles, 1 XOR-NibblePack container, 2 DoubleVector.optimize, DoubleVector.scala:86-96; counter drop flag with
 * FILO_SCHEMA_CUMULATIVE, DoubleVector.scala:456-466), one chunk per rows_per_chunk rows, into a resident table (same bytes as
 * filo_load_series over the JVM-encoded chunks).  group_ids may be NULL. */
int32_t filo_encode_table(filo_ctx* ctx, const int64_t* timestamps, const double* values, int64_t n_series, int32_t rows_per_series,
                          int32_t rows_per_chunk, int32_t value_enc, int32_t schema_flags, const int32_t* group_ids, int32_t n_groups,
                          filo_table** out);
/* Histogram columns written on the device: SectDelta HistogramVectors (AppendableSectDeltaHistVector.appendHist, HistogramVector.scala:
 * 489-545; Section.scala:91-145; NibblePack.scala:296-345), byte-identical to the JVM appender.  bucket_def = the bucket definition as a
 * BinaryHistogram carries it (u16 length prefix + body; format_code 0x03 / 0x04 geometric, 0x05 custom, 0x09 otel exponential), 1..64 buckets.
 *   filo_encode_hist_table: an ingest batch -- cumulative bucket counts [n_series][rows][n_buckets] and timestamps [n_series][rows] in HOST
 *     memory -- encoded into a resident table (one chunk per rows_per_chunk rows);
 *   filo_synth_hist_table: the bench / test generator (row r adds 1 + hash % 3 observations to bucket (r + series) % n_buckets,
 *     TestTimeseriesProducer.scala:229-248; series with id % reset_period == 0 restart at 5/8 of the rows), counter schema. */
int32_t filo_encode_hist_table(filo_ctx* ctx, const int64_t* timestamps, const int64_t* bucket_counts, int64_t n_series, int32_t rows_per_series,
                               int32_t rows_per_chunk, int32_t n_buckets, int32_t format_code, const uint8_t* bucket_def, int32_t bucket_def_bytes,
                               int32_t schema_flags, const int32_t* group_ids, int32_t n_groups, filo_table** out);
int32_t filo_synth_hist_table(filo_ctx* ctx, int64_t n_series, int32_t rows_per_series, int32_t rows_per_chunk, int64_t t0_ms, int32_t interval_ms,
                              int32_t n_buckets, int32_t format_code, const uint8_t* bucket_def, int32_t bucket_def_bytes,
                              int32_t reset_period, int32_t n_groups, uint64_t seed, int64_t series_id_base, filo_table** out);
int32_t filo_table_set_groups(filo_ctx* ctx, filo_table* t, const int32_t* group_ids, int32_t n_groups);
int32_t filo_table_get_info(const filo_table* t, filo_table_info* out);
/* Copies the device arena record of one series back to the host (tests: byte parity of the GPU encoder). */
int64_t filo_table_read_record(filo_ctx* ctx, const filo_table* t, int64_t series, uint8_t* out, int64_t cap);
/* Copies the arena records of series [first, first+n) to the host: `out` receives the record bytes back to back,
 * rec_off_out receives n+1 byte offsets relative to out.  Returns the byte count, or -(bytes needed) when cap is too small.
 * (bench/test: host-side mirror of the chunk memory a FiloDB shard would hold off-heap.) */
int64_t filo_table_read_arena(filo_ctx* ctx, const filo_table* t, int64_t first, int64_t n, uint8_t* out, int64_t cap,
                              int64_t* rec_off_out);
void    filo_table_free(filo_ctx* ctx, filo_table* t);

/* Number of output windows: first window always, then while window_end + step <= end (ChunkSetInfo.scala:462). */
int32_t filo_num_windows(int64_t start_ms, int64_t step_ms, int64_t end_ms);

/* PeriodicSamplesMapper (+ AggregateMapReduce when aggr_op != NONE) over a loaded table; results to HOST buffers.
 *  out_values: aggr NONE -> [n_series * T]; SUM/AVG/MIN/MAX/COUNT/STDDEV/STDVAR/GROUP -> [n_groups * T]; TOPK/BOTTOMK -> [n_groups * T * k];
 *              STDDEV/STDVAR with FILO_Q_PARTIAL -> [2 * n_groups * T] (see filo_query_device)
 *  out_aux:    AVG -> counts [n_groups*T]; TOPK/BOTTOMK -> series ordinals [n_groups*T*k] (-1 = empty); else may be NULL
 *  STDVAR presents NaN where no input is non-NaN, else Σv²/n - m*m with m = Σv/n; STDDEV presents sqrt of that, NaN when the
 *  variance rounds below zero (Math.pow(negative, 0.5)); GROUP presents 1.0 or NaN.  Their counts go to out_aux when it is not NULL. */
int32_t filo_query(filo_ctx* ctx, const filo_table* t, int32_t range_fn,
                   int64_t start_ms, int64_t step_ms, int64_t end_ms, int64_t window_ms,
                   int32_t aggr_op, int32_t k, int32_t flags,
                   double* out_values, int64_t* out_aux, filo_stats* stats);
/* Same, results left in DEVICE buffers (d_out_values / d_out_aux are device pointers), enqueued on cuda_stream
 * (a cudaStream_t, may be NULL = ctx stream); does not synchronize unless stats != NULL.
 * With FILO_Q_PARTIAL: SUM/AVG/COUNT -> values = Σ of non-NaN inputs (0 when none), aux = contributing count;
 * MIN/MAX -> values = min/max with +Inf/-Inf identity, aux = count.  Merge across GPUs with ncclSum / ncclMin /
 * ncclMax on values and ncclSum on aux, then call filo_present_partials.
 * STDDEV/STDVAR with FILO_Q_PARTIAL -> values = [2 * n_groups * T]: the Σv block, then the Σv² block (0 when no input), aux = count
 * (required); both blocks merge with ncclSum.  GROUP with FILO_Q_PARTIAL is exactly the COUNT partial.  For a cross-node
 * ReduceAggregateExec the adapter turns a (Σv, Σv², n) cell into the reference's reduction schema (stdvar|stddev, mean, count)
 * (StdvarRowAggregator.scala:76-79): mean = Σv/n, stdvar = Σv²/n - mean*mean (stddev = sqrt of it), count = n; a cell with n = 0
 * becomes (NaN, NaN, 0). */
int32_t filo_query_device(filo_ctx* ctx, const filo_table* t, int32_t range_fn,
                          int64_t start_ms, int64_t step_ms, int64_t end_ms, int64_t window_ms,
                          int32_t aggr_op, int32_t k, int32_t flags,
                          void* d_out_values, void* d_out_aux, void* cuda_stream, filo_stats* stats);
/* AvgWithSumAndCountOverTimeFuncD / FuncL (query/exec/rangefn/AggrOverTimeFunctions.scala:820-893): avg_over_time over downsampled data
 * (RangeFunction.downsampleRangeFunction, RangeFunction.scala:272-279) = sum_over_time(sum column) / sum_over_time(count column); with a
 * Long sum column (FILO_SCHEMA_LONG_VALUES on t_sum) the divisor is count_over_time of the count column, as FuncL has it.  t_sum and
 * t_count are the two value columns of the same series, loaded as two tables over the same ChunkSetInfo lists (filo_load_series with
 * val_col = the sum / the count column): the windows' row ranges come from the shared timestamp column.  out_values [n_series * T]. */
int32_t filo_query_avg_sum_count(filo_ctx* ctx, const filo_table* t_sum, const filo_table* t_count,
                                 int64_t start_ms, int64_t step_ms, int64_t end_ms, int64_t window_ms, double* out_values, filo_stats* stats);
/* Histogram value columns (HistogramVector.scala: H_SIMPLE / H_SECTDELTA vectors).  filo_load_series accepts them as the value
 * column when every series of the table uses ONE bucket scheme: 1..64 geometric, custom or otel exponential buckets
 * (Base2ExpHistogramBuckets stored in these vectors, format code 0x09: what a counter=true histogram column holds,
 * TimeSeriesStore.scala:278-285; histogram_quantile then interpolates in log2 space, Histogram.scala:97-104).  Row-wise
 * ExpHistogramVector columns (wire 0x1309, a scheme per row) and the XOR-packed codes 0x08 / 0x0a / 0x10 are declined with
 * FILO_ERR_UNSUPPORTED; filo_table_info.schema_flags keeps the caller's flags.  filo_query_hist runs
 *   HistRateFunction / HistIncreaseFunction (RateFunctions.scala:330-418) over cumulative SectDelta histograms with counter
 *   correction (SectDeltaHistogramReader, HistogramVector.scala:628-738), sum_over_time (and rate / increase over a delta-temporality
 *   schema), or LastSampleChunkedFunctionH (range_fn FILO_FN_LAST, RangeFunction.scala:595-641: per window the latest row of the
 *   window's chunks, the raw reader value without counter correction; window_ms <= 0 takes the 5 min + 1 ms default lookback),
 *   optionally HistSumRowAggregator (aggregator/HistSumRowAggregator.scala) over the table's groups, and HistogramQuantileImpl
 *   (InstantFunction.scala:362-368).
 *  aggr NONE: out_values [n_series * T * buckets] (an empty histogram = NaN buckets) or NULL, out_quantile [n_series * T] or NULL:
 *             the quantile of each series' own window histogram (Histogram.quantile, no makeMonotonic), NaN for an empty one
 *  aggr SUM : out_values [n_groups * T * buckets] or NULL, out_quantile [n_groups * T] or NULL (quantile in [0,1])
 *  At least one of the two outputs is given; a quantile < 0 gives -Inf, > 1 gives +Inf (for a non-empty histogram).
 * The sum follows HistSumRowAggregator.reduceAggregate (HistSumRowAggregator.scala:25-36): the first histogram of a partial aggregate
 * is copied, every further one goes through MutableHistogram.add = addNoCorrection + makeMonotonic (Histogram.scala:428-449).  That
 * holds inside a work item (a run of series of one group, in series order) and across the items of a group (item order) -- the
 * same two-level reduction the reference runs (per-shard AggregateMapReduce, then ReduceAggregateExec), with a fixed tree. */
int32_t filo_query_hist(filo_ctx* ctx, const filo_table* t, int32_t range_fn,
                        int64_t start_ms, int64_t step_ms, int64_t end_ms, int64_t window_ms,
                        int32_t aggr_op, double quantile, double* out_values, double* out_quantile, filo_stats* stats);
/* Same, results left in DEVICE buffers (d_out_values / d_out_quantile are device pointers, either may be NULL as above), enqueued on
 * cuda_stream (a cudaStream_t, may be NULL = ctx stream) with its temporaries stream-ordered on it; does not synchronize unless
 * stats != NULL.  Device-side errors of a call with stats == NULL (CorruptVector, or a series with more chunks / sections / rows in
 * range than the device path holds) are returned by the next call on the ctx that finds them complete, or by filo_ctx_check, with the
 * status and message the synchronous call returns.  filo_query_hist runs the same code into device temporaries (allocated only once the
 * arguments have been checked) and copies them to the host before its one synchronisation.
 * aggr SUM without a quantile gives the per-GPU partial of the cross-GPU histogram sum: [n_groups * T * buckets], NaN in every bucket
 * of an empty cell, never NaN in bucket 0 of a non-empty one (the device path reads integer-count histograms only, and makeMonotonic
 * replaces NaN).  Gather the partials of all ranks (not an all-reduce: the fold below is not a sum) and call filo_merge_hist_partials. */
int32_t filo_query_hist_device(filo_ctx* ctx, const filo_table* t, int32_t range_fn,
                               int64_t start_ms, int64_t step_ms, int64_t end_ms, int64_t window_ms,
                               int32_t aggr_op, double quantile, void* d_out_values, void* d_out_quantile, void* cuda_stream, filo_stats* stats);
/* ReduceAggregateExec of histogram sums across GPUs: d_parts holds n_parts aggr SUM outputs of filo_query_hist_device back to back,
 * [n_parts][n_groups][n_windows][buckets] doubles in DEVICE memory, in rank order.  For every (group, window) the parts are folded in
 * that order with HistSumRowAggregator.reduceAggregate: empty cells (bucket 0 NaN) are skipped, the first non-empty one is copied and
 * every further one goes through MutableHistogram.add (bucket-wise sum + makeMonotonic, Histogram.scala:428-449); then
 * histogram_quantile.  d_out_values [n_groups * n_windows * buckets] (NaN buckets for a cell empty on every rank) and
 * d_out_quantile [n_groups * n_windows] as filo_query_hist's SUM outputs; either may be NULL, and a NaN quantile writes the values alone.
 * Caller's contract: t is any rank's table over the same bucket scheme and the same group numbering (n_groups, the bucket count, the
 * bucket tops and the exponential flag come from it), and every part was computed with the same start / step / end.
 * Enqueued on cuda_stream (NULL = ctx stream), no synchronisation.  FILO_ERR_INVALID_ARG for n_parts < 1, n_windows < 1, a table that
 * is not a histogram table, or no output; FILO_ERR_UNSUPPORTED for more than 64 buckets. */
int32_t filo_merge_hist_partials(filo_ctx* ctx, const filo_table* t, int32_t n_parts, int32_t n_windows, double quantile,
                                 const void* d_parts, void* d_out_values, void* d_out_quantile, void* cuda_stream);
/* ReduceAggregateExec of topk / bottomk across GPUs: d_part_values / d_part_ids hold n_parts outputs of filo_query_device with
 * aggr_op TOPK or BOTTOMK back to back, [n_parts][n_groups][n_windows][k] doubles and int64 in DEVICE memory, in rank order; every
 * cell lists its k slots worst first, the way the query writes them.  For every (group, window) the k best non-empty candidates over
 * all parts go to d_out_values / d_out_ids [n_groups * n_windows * k] in that same form: worst first, unused slots padded with
 * -DBL_MAX (topk) / +DBL_MAX (bottomk) and id -1.  Better = larger value for topk, smaller for bottomk; values compare with ==
 * (+0.0 ties -0.0), and among equal values the smaller id is better.  A slot is empty iff its id is -1 (the padding value is also a
 * legal value); value bits pass through unchanged.  The order of the slots inside a part does not matter: the result is the k best of
 * all non-empty slots under that rule, whatever local -> global map produced the ids.  filo_query_device never writes a NaN value with
 * an id (NaN inputs are skipped); a NaN value with an id is skipped like an empty slot.
 * Caller's contract: the ids are global series ordinals (map each rank's local ordinals through its local -> global table first;
 * -1 stays -1), every part was computed with the same aggr_op, k, group numbering (n_groups) and start / step / end, and no series is
 * in two parts.  When every part's table lists its series in increasing global ordinal (a contiguous split or the modulo shard map),
 * the result is bit for bit the query over the union of the series, values and ids.  With another map a part keeps, among equal values
 * at its cut, its earlier series rather than the smaller ordinals, so the merged ties may name other (equally valued) series.
 * Enqueued on cuda_stream (NULL = ctx stream), no synchronisation.  FILO_ERR_INVALID_ARG for an operator other than TOPK / BOTTOMK,
 * k outside [1, 32], n_parts < 1, n_groups < 1, n_windows < 1, or a NULL pointer. */
int32_t filo_merge_topk_partials(filo_ctx* ctx, int32_t aggr_op, int32_t k, int32_t n_parts, int32_t n_groups, int32_t n_windows,
                                 const void* d_part_values, const void* d_part_ids, void* d_out_values, void* d_out_ids, void* cuda_stream);

/* Registers a region of host memory that holds chunk vectors (FiloDB's off-heap block memory, BlockManager pages) for direct
 * device access: pinned + mapped once, like the reference maps its blocks once at start-up.  filo_scan_series then lets the
 * GPU gather the vectors of a call straight out of the region (no staging copy on the host) whenever every vector of the
 * call lies inside registered regions; otherwise it stages through pinned slabs as before.  Unregister before freeing. */
int32_t filo_host_register(filo_ctx* ctx, const void* base, int64_t bytes);
int32_t filo_host_unregister(filo_ctx* ctx, const void* base);

/* PeriodicSamplesMapper over host-resident chunks in ONE pipelined call: filo_load_series + filo_query (aggr NONE) +
 * result read-back, processed in batches so that the host gather of batch b, the H2D copy and the kernels of batch b-1
 * and the D2H of batch b-2 overlap (pinned staging kept in the context).  Same argument meaning, validation and errors as
 * filo_load_series / filo_query; out_values: host [n_series * T] (pinned memory lets the D2H copies overlap).
 * Replaces the per-partition ChunkedWindowIterator loop of PeriodicSamplesMapper.apply (PeriodicSamplesMapper.scala:78-146)
 * for a whole shard's RawDataRangeVectors.  stats->kernel_ns is not filled (batches overlap). */
int32_t filo_scan_series(filo_ctx* ctx, int64_t n_series, const int32_t* n_chunks, const uint64_t* chunk_info_addrs,
                         int32_t ts_col, int32_t val_col, int32_t schema_flags,
                         int32_t range_fn, int64_t start_ms, int64_t step_ms, int64_t end_ms, int64_t window_ms,
                         double* out_values, filo_stats* stats);
/* RowAggregator "present" after a cross-GPU merge: n = n_groups*T cells; writes NaN where count == 0, Σ/n for AVG.
 * STDDEV/STDVAR read the Σv² block at d_values + n (the FILO_Q_PARTIAL layout); GROUP writes 1.0 where count > 0. */
int32_t filo_present_partials(filo_ctx* ctx, int32_t aggr_op, int64_t n, void* d_values, void* d_counts,
                              void* d_out_values, void* cuda_stream);

/* Result wire format: the rows (start + k*step, values[row][k]) of a query result encoded as BinaryRecord v2 records in 4096-byte
 * RecordContainers -- the bytes SerializedRangeVector.apply writes through ONE RecordBuilder shared by all range vectors of a result
 * (core/src/main/scala/filodb.core/query/RangeVector.scala:427-476,511-586; binaryrecord2/RecordBuilder.scala:109-175,461-480,589-621;
 * RecordContainer.scala:13-57).  NaN rows are not encoded unless start == end (canRemoveEmptyRows); 204 records of 20 bytes per
 * container.  Range vector i is (rows_serialized[i], start_record_no[i], first_container[i]): its records are records
 * [start_record_no, start_record_no + rows_serialized) of the containers from first_container on.  container_ts_ms is the server
 * timestamp of the container headers.  The *_device form reads and writes device memory on cuda_stream (containers: capacity
 * filo_result_max_containers(n_rows, T) * 4096 bytes always suffices; bytes of the last container past its records are not written). */
int64_t filo_result_max_containers(int64_t n_rows, int32_t n_windows);
int32_t filo_encode_result_device(filo_ctx* ctx, const void* d_values, int64_t n_rows, int64_t start_ms, int64_t step_ms, int64_t end_ms,
                                  int64_t container_ts_ms, void* d_containers, int64_t containers_cap_bytes,
                                  void* d_rows_serialized /* int32[n_rows] */, void* d_start_record_no /* int32[n_rows] */,
                                  void* d_first_container /* int64[n_rows] */, int64_t* n_containers_out, int64_t* n_records_out, void* cuda_stream);
int32_t filo_encode_result(filo_ctx* ctx, const double* values, int64_t n_rows, int64_t start_ms, int64_t step_ms, int64_t end_ms,
                           int64_t container_ts_ms, uint8_t* out_containers, int64_t containers_cap_bytes, int32_t* rows_serialized,
                           int32_t* start_record_no, int64_t* first_container, int64_t* n_containers_out, int64_t* n_records_out);

#ifdef __cplusplus
}
#endif
#endif /* FILO_B200_H */
