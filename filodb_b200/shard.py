"""Host-side multi-GPU logic: FiloDB shard -> GPU assignment and the one cross-shard exchange of an aggregate query.

One process per GPU.  Series are independent until the across-series aggregate (SURVEY.md §8e), so the data path has no
collective for per-series queries; aggregates merge `[G x T]` partials (FILO_Q_PARTIAL form, include/filo_b200.h) with
one all-reduce, the role `LocalPartitionReduceAggregateExec` + `RowAggregator.reduceAggregate` play in the reference
(query/exec/AggrOverRangeVectors.scala:119-182; aggregator/*RowAggregator.scala).  Histogram sums are gathered instead
(gather_hist_partials) and folded in rank order on the device by filo_merge_hist_partials; topk / bottomk candidates are mapped
to global series ordinals (topk_ids_to_global), gathered (gather_topk_partials) and selected again by filo_merge_topk_partials.

Works on CUDA tensors over NCCL (product) and on CPU tensors over gloo (tests/test_multi_gpu_gloo.py).
"""
from __future__ import annotations

AGG_NONE, AGG_SUM, AGG_AVG, AGG_MIN, AGG_MAX, AGG_COUNT, AGG_TOPK, AGG_BOTTOMK, AGG_STDDEV, AGG_STDVAR, AGG_GROUP = range(11)


def shards_of_rank(num_shards: int, rank: int, world: int) -> list[int]:
    """GPU g owns shards {s : s mod nGPU == g}: FiloDB's spread bits are the upper bits of the shard number
    (coordinator/ShardMapper.scala:26-48,93-102), so the modulo spreads one shard key's shards over all GPUs."""
    if num_shards & (num_shards - 1):
        raise ValueError("numShards must be a power of two (ShardMapper.scala:26-31)")
    if not 0 <= rank < world:
        raise ValueError("rank out of range")
    return [s for s in range(num_shards) if s % world == rank]


def series_range_of_rank(n_series_total: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous [begin, end) series-id range of a rank when series (not shards) are split evenly (synthetic bench)."""
    per = (n_series_total + world - 1) // world
    b = min(n_series_total, rank * per)
    return b, min(n_series_total, b + per)


def merge_partials(values, counts, aggr_op: int, dist) -> None:
    """In-place cross-rank merge of FILO_Q_PARTIAL results: values [G*T] f64 ([2*G*T] for stddev / stdvar: the Σv and Σv² blocks),
    counts [G*T] i64.  sum/avg/count/group: Σ values, Σ counts; stddev/stdvar: Σ of both value blocks, Σ counts (the moments add up);
    min/max: min/max of values (identity ±Inf), Σ counts."""
    if aggr_op in (AGG_SUM, AGG_AVG, AGG_COUNT, AGG_GROUP, AGG_STDDEV, AGG_STDVAR):
        dist.all_reduce(values, op=dist.ReduceOp.SUM)
    elif aggr_op == AGG_MIN:
        dist.all_reduce(values, op=dist.ReduceOp.MIN)
    elif aggr_op == AGG_MAX:
        dist.all_reduce(values, op=dist.ReduceOp.MAX)
    else:
        raise ValueError("aggregate %d has no all-reduce merge (topk merges gathered candidates)" % aggr_op)
    dist.all_reduce(counts, op=dist.ReduceOp.SUM)


def gather_hist_partials(values, dist):
    """Every rank's histogram SUM partial (filo_query_hist_device with aggr SUM, [G, T, nb] f64, NaN buckets = empty) -> [W, G, T, nb]
    in rank order, for filo_merge_hist_partials.  all_gather into views of one preallocated tensor, so the same code runs on gloo
    (CPU tensors) and NCCL (CUDA tensors)."""
    import torch
    # A gather, not an all-reduce: HistSumRowAggregator.reduceAggregate copies the first non-empty histogram and makes every later sum
    # monotonic (MutableHistogram.add, Histogram.scala:428-451), so the merge is an ordered fold that a reduction op cannot express.
    out = torch.empty((dist.get_world_size(),) + tuple(values.shape), dtype=values.dtype, device=values.device)
    dist.all_gather(list(out.unbind(0)), values.contiguous())
    return out


def topk_ids_to_global(ids, global_of_local):
    """A rank's topk / bottomk ids (filo_query_device with aggr TOPK / BOTTOMK: ordinals of its table's series, -1 = empty slot) ->
    global series ordinals through its local -> global table (a tensor on the ids' device); -1 stays -1.  Runs where the tensors are.
    A rank whose table holds no series has only empty slots: its ids come back unchanged."""
    import torch
    if global_of_local.numel() == 0:
        return ids.clone()
    g = global_of_local.to(device=ids.device, dtype=torch.int64)
    return torch.where(ids >= 0, g[ids.clamp(min=0)], ids)


def gather_topk_partials(values, ids, dist):
    """Every rank's topk / bottomk candidates ([G, T, k] f64 values and i64 global ordinals) -> two [W, G, T, k] tensors in rank order,
    for filo_merge_topk_partials.  all_gather into views of preallocated tensors, so the same code runs on gloo and NCCL."""
    import torch
    # A gather, not an all-reduce: the merge selects the k best (value, ordinal) pairs of the union, which no reduction op expresses.
    W = dist.get_world_size()
    out_v = torch.empty((W,) + tuple(values.shape), dtype=values.dtype, device=values.device)
    out_i = torch.empty((W,) + tuple(ids.shape), dtype=ids.dtype, device=ids.device)
    dist.all_gather(list(out_v.unbind(0)), values.contiguous())
    dist.all_gather(list(out_i.unbind(0)), ids.contiguous())
    return out_v, out_i


def max_over_ranks(x: float, dist, device) -> float:
    """Device-timed durations are reported as the max over ranks."""
    import torch
    t = torch.tensor([x], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())
