"""Host-side mirror of the reference's operator interface for this path, over the C-ABI (Python twin of include/filo_b200.hpp).

    RangeVectorTransformer / PeriodicSamplesMapper   query/src/main/scala/filodb/query/exec/PeriodicSamplesMapper.scala:27-76
    AggregateMapReduce                               query/src/main/scala/filodb/query/exec/AggrOverRangeVectors.scala:119-182
    InstantVectorFunctionMapper(HistogramQuantile)   query/src/main/scala/filodb/query/exec/RangeVectorTransformer.scala:61-110
    RawDataRangeVector.chunkInfos                    core/src/main/scala/filodb.core/query/RangeVector.scala:365-389

Same names, argument meaning and error behaviour: Scala `require` failures are ValueError("requirement failed: ..."), engine
errors are capi.FiloError (what the JNI shim raises as RuntimeException).  There is no CPU path: everything ends in libfilo_b200.so.
"""
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

from . import capi


class RangeVectorTransformer:
    funcParams: Sequence[float] = ()


@dataclass
class RawDataRangeVector:
    """One partition's chunks for the query range (ChunkSetInfo native addresses in chunkID order) and the ordinal of the group its
    RangeVectorKey maps to under the query's by / without clause (AggrOverRangeVectors.scala:150-159)."""
    chunkInfoAddrs: List[int]
    group: int = 0


FN_AVG_WITH_SUM_AND_COUNT_OVER_TIME = 1000      # InternalRangeFunction.AvgWithSumAndCountOverTime: not a scan function id, served by filo_query_avg_sum_count


@dataclass
class PeriodicSamplesMapper(RangeVectorTransformer):
    startMs: int
    stepMs: int
    endMs: int
    window: Optional[int] = None
    functionId: Optional[int] = None            # capi.FN_*; None = last sample
    funcParams: Sequence[float] = ()            # StaticFuncArgs scalars (quantile; sf, tf; duration)

    def __post_init__(self):                     # PeriodicSamplesMapper.scala:45-49
        if not self.startMs <= self.endMs:
            raise ValueError("requirement failed: start %d should be <= end %d" % (self.startMs, self.endMs))
        if not (self.startMs == self.endMs or self.stepMs > 0):
            raise ValueError("requirement failed: step should be > 0 for range query")
        if self.functionId not in (None, capi.FN_LAST, capi.FN_TIMESTAMP) and not (self.window and self.window > 0):
            raise ValueError("requirement failed: Need positive window lengths to apply range function")


@dataclass
class AggregateMapReduce(RangeVectorTransformer):
    aggrOp: int                                  # capi.AGG_*
    aggrParams: Sequence[float] = ()
    numGroups: int = 1

    def __post_init__(self):
        if self.aggrOp in (capi.AGG_TOPK, capi.AGG_BOTTOMK) and len(self.aggrParams) != 1:
            raise ValueError("requirement failed: topk/bottomk need one parameter")


@dataclass
class HistogramQuantileMapper(RangeVectorTransformer):      # InstantVectorFunctionMapper(InstantFunctionId.HistogramQuantile, Seq(q))
    q: float


@dataclass
class QueryResult:
    values: np.ndarray
    aux: Optional[np.ndarray] = None
    stats: dict = field(default_factory=dict)


class FusedGpuExec:
    """One shard's query context on one GPU: ExecPlan.execute step 2 for the transformer chain
    [PeriodicSamplesMapper, AggregateMapReduce?, HistogramQuantileMapper?] as one call into the device library."""

    def __init__(self, device=0, **cfg):
        self.ctx = capi.Context(device, **cfg)

    def close(self):
        self.ctx.close()

    def execute(self, source: Sequence[RawDataRangeVector], psm: PeriodicSamplesMapper, aggr: Optional[AggregateMapReduce] = None,
                quantile: Optional[HistogramQuantileMapper] = None, valueColumn=1, cumulative=False, histogram=False, longValues=False) -> QueryResult:
        nch = np.array([len(rv.chunkInfoAddrs) for rv in source], np.int32)
        addrs = np.array([a for rv in source for a in rv.chunkInfoAddrs], np.uint64)
        flags = (capi.SCHEMA_CUMULATIVE if cumulative else 0) | (capi.SCHEMA_LONG_VALUES if longValues else 0)
        fn = capi.FN_LAST if psm.functionId is None else psm.functionId
        window = psm.window or 0
        if psm.functionId == FN_AVG_WITH_SUM_AND_COUNT_OVER_TIME:
            # AvgWithSumAndCountOverTimeFuncD / FuncL(schema.colIDs(2)) (RangeFunction.scala:325-326,360-362): sum column = valueColumn, count column next to it
            if aggr is not None or histogram:
                raise capi.FiloError(capi.ERR_UNSUPPORTED, "AvgWithSumAndCountOverTime: per-series rows of scalar columns only")
            t_sum = self.ctx.load_series(nch, addrs, val_col=valueColumn, schema_flags=capi.SCHEMA_LONG_VALUES if longValues else 0)
            try:
                t_cnt = self.ctx.load_series(nch, addrs, val_col=valueColumn + 1)
                try:
                    out = self.ctx.query_avg_sum_count(t_sum, t_cnt, psm.startMs, psm.stepMs, psm.endMs, window)
                    return QueryResult(out, None, dict(self.ctx.last_stats))
                finally:
                    t_cnt.free()
            finally:
                t_sum.free()
        self.ctx.set_fn_args(*(tuple(psm.funcParams) + (0.0, 0.0))[:2])
        try:
            if aggr is None and not histogram:          # bare PeriodicSamplesMapper: the pipelined load + scan + read-back call
                out = self.ctx.scan_series(nch, addrs, fn, psm.startMs, psm.stepMs, psm.endMs, window, val_col=valueColumn, schema_flags=flags)
                return QueryResult(out, None, dict(self.ctx.last_stats))
            groups = np.array([rv.group for rv in source], np.int32) if aggr else None
            tab = self.ctx.load_series(nch, addrs, val_col=valueColumn, group_ids=groups, n_groups=aggr.numGroups if aggr else 0, schema_flags=flags)
            try:
                if histogram:
                    if aggr and aggr.aggrOp != capi.AGG_SUM:
                        raise capi.FiloError(capi.ERR_UNSUPPORTED, "histogram aggregates: sum only")
                    res = self.ctx.query_hist(tab, fn, psm.startMs, psm.stepMs, psm.endMs, window, aggr=capi.AGG_SUM if aggr else capi.AGG_NONE,
                                              quantile=quantile.q if quantile else None, want_values=quantile is None)
                    # [rows, T, buckets], or with the quantile [rows, T]; rows = groups, or series without an aggregate
                    return QueryResult(res, None, dict(self.ctx.last_stats))
                k = int(aggr.aggrParams[0]) if aggr.aggrOp in (capi.AGG_TOPK, capi.AGG_BOTTOMK) else 0
                res = self.ctx.query(tab, fn, psm.startMs, psm.stepMs, psm.endMs, window, aggr=aggr.aggrOp, k=k)
                vals, aux = res if isinstance(res, tuple) else (res, None)
                return QueryResult(vals, aux, dict(self.ctx.last_stats))
            finally:
                tab.free()
        finally:
            self.ctx.set_fn_args(0.0, 0.0)
