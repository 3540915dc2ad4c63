"""TEST INFRASTRUCTURE: the reference's stddev / stdvar / group aggregators restated literally, vectorised over the windows.

    StdvarRowAggregator   query/src/main/scala/filodb/query/exec/aggregator/StdvarRowAggregator.scala:52-79
    StddevRowAggregator   query/src/main/scala/filodb/query/exec/aggregator/StddevRowAggregator.scala:39-58
    GroupRowAggregator    query/src/main/scala/filodb/query/exec/aggregator/GroupRowAggregator.scala:23-29

The inputs are the per-series window results of the CPU oracle (oracle.Store.query with AGG_NONE), folded in series (arrival)
order: `map` turns a sample v into the row (0, v, v is NaN ? 0 : 1), `reduceAggregate` folds a row into the holder, NaN reseeding
of acc.mean / acc.stdVar included.  `math.pow(x, 2)` is x*x; `Math.pow(x, 0.5)` is java_pow_half.  numpy's float64 element-wise
operations are single IEEE operations (no contraction), as the JVM's are.
"""
import numpy as np

STDDEV, STDVAR, GROUP = 8, 9, 10          # include/filo_b200.h FILO_AGG_*


def java_pow_half(x):
    """Math.pow(x, 0.5): sqrt for x >= +0.0; NaN below zero and for NaN; pow(-0.0, 0.5) = +0.0 and pow(-Inf, 0.5) = +Inf."""
    x = np.asarray(x, np.float64)
    with np.errstate(invalid="ignore"):
        r = np.sqrt(np.where(x < 0, np.nan, x))
    r = np.where(x == 0.0, 0.0, r)                      # -0.0 -> +0.0
    return np.where(x == -np.inf, np.inf, r)


class Holder:
    """StdvarHolder / StddevHolder over T windows: (stat, mean, count) with the reference's zero (NaN, NaN, 0)."""

    def __init__(self, T):
        self.stat = np.full(T, np.nan)
        self.mean = np.full(T, np.nan)
        self.count = np.zeros(T, np.int64)

    def row(self):
        return self.stat.copy(), self.mean.copy(), self.count.copy()


def reduce_aggregate(op, acc, stat, mean, count):
    """StdvarRowAggregator / StddevRowAggregator.reduceAggregate for every window at once (the windows are independent)."""
    ok = ~np.isnan(stat) & ~np.isnan(mean)
    a_mean = np.where(ok & np.isnan(acc.mean), 0.0, acc.mean)
    a_stat = np.where(ok & np.isnan(acc.stat), 0.0, acc.stat)
    ac = acc.count.astype(np.float64); gc = count.astype(np.float64)          # Long operands widen to Double
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        new_mean = (a_mean * ac + mean * gc) / (ac + gc)
        if op == STDVAR:
            acc_sq = (a_stat + a_mean * a_mean) * ac
            agg_sq = (stat + mean * mean) * gc
            new_stat = (acc_sq + agg_sq) / (ac + gc) - new_mean * new_mean
        else:
            acc_sq = (a_stat * a_stat + a_mean * a_mean) * ac
            agg_sq = (stat * stat + mean * mean) * gc
            new_stat = java_pow_half((acc_sq + agg_sq) / (ac + gc) - new_mean * new_mean)
    acc.stat = np.where(ok, new_stat, a_stat)
    acc.mean = np.where(ok, new_mean, a_mean)
    acc.count = np.where(ok, acc.count + count, acc.count)
    # (a_mean / a_stat differ from acc's only where ok: the reseeding happens inside the `if`)


def map_row(v):
    """map: (timestamp, 0, v, v is NaN ? 0 : 1)."""
    v = np.asarray(v, np.float64)
    return np.zeros_like(v), v, np.where(np.isnan(v), 0, 1).astype(np.int64)


def leaf(op, rows):
    """mapReduce(skipMapPhase = false) of one group: rows = the group's per-series window results [n, T] in arrival order."""
    rows = np.asarray(rows, np.float64)
    T = rows.shape[1]
    if op == GROUP:
        return np.where((~np.isnan(rows)).any(axis=0), 1.0, np.nan) if len(rows) else np.full(T, np.nan)
    acc = Holder(T)
    for v in rows:
        reduce_aggregate(op, acc, *map_row(v))
    return acc


def two_level(op, leaves):
    """mapReduce(skipMapPhase = true) over leaf results of one group (e.g. one per shard): their rows folded into a fresh holder."""
    if op == GROUP:
        stack = np.array(leaves)
        return np.where((stack == 1.0).any(axis=0), 1.0, np.nan)
    acc = Holder(leaves[0].stat.size)
    for lf in leaves:
        reduce_aggregate(op, acc, *lf.row())
    return acc


def aggregate(op, per_series, group_ids, n_groups):
    """AggregateMapReduce over per-series results [S, T] with the group of each series: presented values [G, T] and the
    non-NaN counts [G, T].  The series of a group are folded in increasing series ordinal (the arrival order)."""
    per_series = np.asarray(per_series, np.float64)
    S, T = per_series.shape
    g = np.zeros(S, np.int64) if group_ids is None else np.asarray(group_ids)
    vals = np.full((n_groups, T), np.nan); cnts = np.zeros((n_groups, T), np.int64)
    for k in range(n_groups):
        rows = per_series[g == k]
        cnts[k] = (~np.isnan(rows)).sum(axis=0)
        if op == GROUP:
            vals[k] = leaf(op, rows)
        elif len(rows):
            vals[k] = leaf(op, rows).stat
    return vals, cnts


def group_means(per_series, group_ids, n_groups):
    """m of the cancellation bound: mean of the group's non-NaN inputs per window (NaN where none)."""
    per_series = np.asarray(per_series, np.float64)
    g = np.zeros(per_series.shape[0], np.int64) if group_ids is None else np.asarray(group_ids)
    out = np.full((n_groups, per_series.shape[1]), np.nan)
    for k in range(n_groups):
        rows = per_series[g == k]
        if len(rows):
            with np.errstate(invalid="ignore", divide="ignore"):
                out[k] = np.nansum(rows, axis=0) / (~np.isnan(rows)).sum(axis=0)
    return out


def moment_partials(per_series, group_ids, n_groups):
    """The FILO_Q_PARTIAL form of stddev / stdvar built on the host: (Σv, Σv²) [2, G, T] and counts [G, T], series in order."""
    per_series = np.asarray(per_series, np.float64)
    g = np.zeros(per_series.shape[0], np.int64) if group_ids is None else np.asarray(group_ids)
    T = per_series.shape[1]
    vals = np.zeros((2, n_groups, T)); cnts = np.zeros((n_groups, T), np.int64)
    for row, k in zip(per_series, g):
        ok = ~np.isnan(row)
        v = np.where(ok, row, 0.0)
        vals[0, k] = np.where(ok, vals[0, k] + v, vals[0, k])
        vals[1, k] = np.where(ok, vals[1, k] + v * v, vals[1, k])
        cnts[k] += ok
    return vals, cnts


def present_moments(op, s, s2, c):
    """What the device presents from merged moments (filo_present_partials): NaN where c == 0, else Σv²/c - m*m with m = Σv/c
    (stdvar), Math.pow of it to 0.5 (stddev), 1.0 (group)."""
    s = np.asarray(s, np.float64); s2 = np.asarray(s2, np.float64); c = np.asarray(c)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        cf = c.astype(np.float64)
        m = s / cf
        var = s2 / cf - m * m
    r = 1.0 if op == GROUP else var if op == STDVAR else java_pow_half(var)
    return np.where(c == 0, np.nan, r)


def assert_moments_close(op, got, exp, means, ref_var, what=""):
    """|got - exp| <= 1e-9 |exp| + 1e-12 m^2 per cell (stddev compared squared); identical NaN pattern except in cells the
    reference marks as cancellation-dominated (|stdvar| <= 1e-12 m^2, ref_var = the reference's stdvar of the same cells)."""
    got = np.asarray(got, np.float64); exp = np.asarray(exp, np.float64)
    g2, e2 = (got * got, exp * exp) if op == STDDEV else (got, exp)
    bound = 1e-12 * means * means
    cancel = np.abs(ref_var) <= bound
    nan_ok = (np.isnan(got) == np.isnan(exp)) | cancel
    assert nan_ok.all(), "%s: NaN pattern differs at %s" % (what, np.argwhere(~nan_ok)[:5].tolist())
    m = ~np.isnan(got) & ~np.isnan(exp)
    err = np.abs(g2[m] - e2[m]); lim = 1e-9 * np.abs(e2[m]) + bound[m]
    assert (err <= lim).all(), "%s: %d cells outside the bound, worst %r vs %r" % (what, int((err > lim).sum()), g2[m][np.argmax(err - lim)], e2[m][np.argmax(err - lim)])
