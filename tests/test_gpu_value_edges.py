"""GPU: the scan and aggregate kernels at value edges, against the CPU oracle on the same chunk bytes.

Every suite table elsewhere holds moderate non-zero values; the kernels take shortcuts that are exact only because of claims about
values.  This module feeds them the values those claims are about:
- signed zeros, where min / max across series must keep the later of two equal values (QueryUtils.minIgnoreNaN / maxIgnoreNaN,
  QueryUtils.scala:111-123), in every fused kernel and in merge_partials_kernel;
- the decode bounds of the v4 SUM kernel (wp_decode admits 2^-511 <= |v| < 2^513 and declines the series otherwise);
- counters above 2^53, near DBL_MAX with resets, +Inf samples, series starting at +-0.0, and rows on the boundary of the v4 counter
  kernel's zero-point skip test (v1 > delta * skipC) and of the reference's `durationToZero < durationToStart` (RateFunctions.scala:84-90).
Per-series results and min / max / count across series are compared bit for bit (the sign of zero counts), with the scan counters."""
import sys
import zlib

import numpy as np
import pytest

from tests import agg_moments_ref as R
from tests.test_gpu_agg_moments import check_moments
from tests.test_gpu_parity import ALL_FNS, assert_same, same_bits

pytestmark = pytest.mark.gpu
T0 = 1_700_000_000_000
ROWS = 480
TS = T0 + np.arange(ROWS, dtype=np.int64) * 15000
Q5M = (T0 + 300000, 15000, T0 + 479 * 15000, 300000)          # [5m] windows, 15 s step (BASELINE C2 shape)
Q1M = (T0 + 60000, 15000, T0 + 479 * 15000 + 30000, 60000)
# window k covers rows k + 1 .. k + 20: durationToStart = 5 s, durationToEnd = 10 s, sampledInterval = 285 s
QOFF = (T0 + 310000, 15000, T0 + 470 * 15000, 300000)
DTS, SI = 5.0, 285.0


@pytest.fixture(scope="module", params=["v4", "v3", "v2", "v1"])
def gpu(request):
    """v4: the default selection (v4 SUM kernel per series, tile kernel fused, v4 counter kernel for the counter class, the v2 kernel
    behind each); v3: the tile kernel for the SUM class; v2: the TMA-staged warp-per-series kernel; v1: the generic kernel."""
    import os
    import filodb_b200.capi as capi
    if request.param == "v4": os.environ.pop("FILO_KERNEL", None)
    else: os.environ["FILO_KERNEL"] = request.param
    ctx = capi.Context(0)
    yield capi, ctx
    ctx.close()
    os.environ.pop("FILO_KERNEL", None)


def same_stats(ctx, st, what):
    assert ctx.last_stats["samples_scanned"] == st.last_stats["samples_scanned"], what + ": samples_scanned"
    assert ctx.last_stats["bytes_scanned"] == st.last_stats["bytes_scanned"], what + ": bytes_scanned"


# ---- the reference's min / max fold and the device's fold order
def fold_minmax(rows, op_min, keep_later=True):
    """acc = minIgnoreNaN(acc, v) / maxIgnoreNaN(acc, v) over `rows` in order (QueryUtils.scala:111-123), from NaN.
    keep_later=False is the rule the kernels had before: of two equal values the earlier one stays."""
    acc = None
    for r in rows:
        r = np.asarray(r, np.float64)
        if acc is None:
            acc = r.copy(); continue
        if keep_later: keep = acc < r if op_min else acc > r
        else: keep = acc <= r if op_min else acc >= r
        acc = np.where(np.isnan(acc), r, np.where(np.isnan(r) | keep, acc, r))
    return acc


def items_per_group_seg(S):
    """Series per work item: S / (SMs * 64 * 4), at least 1, at most 256 (build_groups_new, capi.cu:205-212)."""
    import torch
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    return int(min(max(S // (sm * 256), 1), 256))


def device_fold_order(members, seg):
    """The series of one group in the order the device's min / max fold sees them: items of `seg` consecutive series in group order
    (a stable sort by group id); merge_partials_kernel folds items j, j + 8, ... in lane j and then lanes 0 .. 7 in order, which for an
    associative rule is one sequential fold over the items 0, 8, 16, ..., 1, 9, ..., each item's series in group order."""
    items = [members[i:i + seg] for i in range(0, len(members), seg)]
    return [s for j in range(8) for it in items[j::8] for s in it]


def expected_minmax(per, groups, G, op_min, seg, keep_later=True):
    T = per.shape[1]
    out = np.full((G, T), np.nan)
    for g in range(G):
        members = list(np.nonzero(groups == g)[0])
        if members:
            out[g] = fold_minmax([per[s] for s in device_fold_order(members, seg)], op_min, keep_later)
    return out


def tie_orders(per, groups, G, op_min, seg):
    """Cells where the kept-later rule gives -0.0 and the kept-earlier rule +0.0 (arrival +0 then -0), and the other way round."""
    a = expected_minmax(per, groups, G, op_min, seg, True)
    b = expected_minmax(per, groups, G, op_min, seg, False)
    z = (a == 0) & (b == 0)
    return int((z & np.signbit(a) & ~np.signbit(b)).sum()), int((z & ~np.signbit(a) & np.signbit(b)).sum())


# ---- signed zeros
ZP = np.array([0.0, -0.0, 1.0, -1.0])
PALETTES = [ZP[[0, 1]], ZP[[0, 1, 2]], ZP[[0, 1, 3]], ZP]


def signed_zero_store(o, rng, n_series, val_mode):
    """Gauge series of +-0.0 / +-1.0 in runs of 12 rows (a [5m] window sees two or three runs), and series entirely +0.0 and -0.0."""
    st = o.Store()
    for s in range(n_series):
        kind = s % 6
        if kind == 4: v = np.zeros(ROWS)
        elif kind == 5: v = np.full(ROWS, -0.0)
        else:
            pal = PALETTES[kind]
            v = np.repeat(pal[rng.integers(0, len(pal), ROWS // 12)], 12)
        st.add_series_rows(TS, v, [400, 80], val_mode=val_mode)
    return st


FUSED_FNS = ("FN_LAST", "FN_MIN_OVER_TIME", "FN_DELTA", "FN_SUM_OVER_TIME")


def check_fused(capi, ctx, o, st, tab, groups, G, seg, fn_name, q, what, need_ties):
    fn, ofn = getattr(capi, fn_name), getattr(o, fn_name)
    per = st.query(ofn, *q)
    ints = fn_name != "FN_DELTA"                            # per-series values are small integers: sums are exact
    for op_min in (True, False):
        name = "AGG_MIN" if op_min else "AGG_MAX"
        if need_ties:
            a, b = tie_orders(per, groups, G, op_min, seg)
            assert a > 0 and b > 0, "%s %s: the table has no signed-zero tie in some arrival order (%d, %d)" % (what, name, a, b)
        got = ctx.query(tab, fn, *q, aggr=getattr(capi, name))
        same_stats(ctx, st, "%s %s %s" % (what, fn_name, name))
        assert_same(got, expected_minmax(per, groups, G, op_min, seg), "%s %s %s" % (what, fn_name, name))
        if seg == 1 and np.bincount(groups, minlength=G).max() <= 8:       # the device's order is the arrival order: the oracle itself
            exp = st.query(ofn, *q, aggr=getattr(o, name), group_ids=groups, n_groups=G)
            assert_same(got, exp, "%s %s %s (oracle)" % (what, fn_name, name))
        # partial form + present on the device
        check_partial_present_plain(capi, ctx, tab, fn, q, getattr(capi, name), got)
    gs = ctx.query(tab, fn, *q, aggr=capi.AGG_SUM)
    es = st.query(ofn, *q, aggr=o.AGG_SUM, group_ids=groups, n_groups=G)
    if ints: assert_same(gs, es, "%s %s sum" % (what, fn_name))
    else: np.testing.assert_allclose(gs, es, rtol=1e-9, atol=0, equal_nan=True)
    gc = ctx.query(tab, fn, *q, aggr=capi.AGG_COUNT)
    assert_same(gc, st.query(ofn, *q, aggr=o.AGG_COUNT, group_ids=groups, n_groups=G), "%s %s count" % (what, fn_name))
    (gv, gn), (ev, en) = ctx.query(tab, fn, *q, aggr=capi.AGG_AVG), st.query(ofn, *q, aggr=o.AGG_AVG, group_ids=groups, n_groups=G)
    assert (gn == en).all()
    np.testing.assert_allclose(gv, ev, rtol=1e-9, atol=1e-300, equal_nan=True)
    check_moments(capi, ctx, tab, per, groups, G, fn, q, "%s %s" % (what, fn_name))


def check_partial_present_plain(capi, ctx, tab, fn, q, aggr, presented):
    import torch
    pv, pc = ctx.query(tab, fn, *q, aggr=aggr, flags=capi.Q_PARTIAL)
    n = presented.size
    dv = torch.from_numpy(pv.reshape(-1).copy()).cuda(); dc = torch.from_numpy(pc.reshape(-1).copy()).cuda()
    do = torch.empty(n, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    ctx.present_partials(aggr, n, dv.data_ptr(), dc.data_ptr(), do.data_ptr())
    torch.cuda.synchronize()
    assert same_bits(do.cpu().numpy().reshape(presented.shape), presented), "partial + present differs from the presented form"


@pytest.mark.parametrize("val_mode", [1, 2], ids=["xor", "raw"])
def test_signed_zeros(gpu, oracle, val_mode):
    """Per-series ALL_FNS, then min / max / sum / avg / count / group / stddev / stdvar across groups of <= 8 series over last and
    min_over_time (the v2 aggregate kernel), delta (the counter class even on a gauge: the fused v4 counter kernel) and sum_over_time
    (the tile kernel).  Ties of +0.0 and -0.0 occur at the min and at the max in both arrival orders."""
    capi, ctx = gpu; o = oracle
    rng = np.random.default_rng(zlib.crc32(b"signed zeros %d" % val_mode))
    S, G = 48, 8
    st = signed_zero_store(o, rng, S, val_mode)
    groups = (np.arange(S) * 5 % G).astype(np.int32)         # six series per group, mixed kinds
    tab = ctx.load_series(*st.all_info_addrs(), group_ids=groups, n_groups=G)
    for q in (Q5M, Q1M):
        for name in ALL_FNS:
            got = ctx.query(tab, getattr(capi, name), *q)
            assert_same(got, st.query(getattr(o, name), *q), "%s q=%s" % (name, q))
            same_stats(ctx, st, name)
    seg = items_per_group_seg(S)
    for fn_name in FUSED_FNS:
        check_fused(capi, ctx, o, st, tab, groups, G, seg, fn_name, Q5M, "signed zeros", fn_name in ("FN_LAST", "FN_MIN_OVER_TIME", "FN_DELTA"))
    tab.free()


def test_signed_zeros_group_of_many_items(gpu, oracle):
    """One group of 40 series (more than 8 work items): min / max fold the oracle's per-series rows in the device's item order."""
    capi, ctx = gpu; o = oracle
    rng = np.random.default_rng(4040)
    S, G = 60, 3
    st = signed_zero_store(o, rng, S, 1)
    groups = np.where(np.arange(S) < 40, 0, 1 + np.arange(S) % 2).astype(np.int32)
    groups = groups[rng.permutation(S)]
    tab = ctx.load_series(*st.all_info_addrs(), group_ids=groups, n_groups=G)
    seg = items_per_group_seg(S)
    assert -(-40 // seg) > 8
    for fn_name in ("FN_LAST", "FN_MIN_OVER_TIME", "FN_DELTA"):
        per = st.query(getattr(o, fn_name), *Q5M)
        for op_min in (True, False):
            name = "AGG_MIN" if op_min else "AGG_MAX"
            got = ctx.query(tab, getattr(capi, fn_name), *Q5M, aggr=getattr(capi, name))
            assert_same(got, expected_minmax(per, groups, G, op_min, seg), "%s %s" % (fn_name, name))
            same_stats(ctx, st, fn_name + " " + name)
    tab.free()


def test_topk_bottomk_zero_ties_and_infinities(gpu, oracle):
    capi, ctx = gpu; o = oracle
    rng = np.random.default_rng(99)
    S, G = 30, 4
    st = o.Store()
    pal = np.array([0.0, -0.0, np.inf, -np.inf, 1.0])
    for s in range(S):
        v = np.repeat(pal[rng.integers(0, 2 if s % 3 else 5, ROWS // 12)], 12)
        st.add_series_rows(TS, v, [400, 80], val_mode=2 if s % 2 else 1)
    groups = (np.arange(S) % G).astype(np.int32)
    tab = ctx.load_series(*st.all_info_addrs(), group_ids=groups, n_groups=G)
    per = st.query(o.FN_LAST, *Q5M)
    for aggr_name in ("AGG_TOPK", "AGG_BOTTOMK"):
        for k in (1, 3):
            gv, gi = ctx.query(tab, capi.FN_LAST, *Q5M, aggr=getattr(capi, aggr_name), k=k)
            ev, ei = st.query(o.FN_LAST, *Q5M, aggr=getattr(o, aggr_name), k=k, group_ids=groups, n_groups=G)
            same_stats(ctx, st, aggr_name)
            assert_same(gv, ev, "%s k=%d values" % (aggr_name, k))
            ok = gi >= 0
            assert (ok == (ei >= 0)).all()
            g_, t_, j_ = np.nonzero(ok)
            assert (groups[gi[ok]] == g_).all()
            assert same_bits(per[gi[ok], t_], gv[g_, t_, j_])
    tab.free()


# ---- the v4 SUM kernel's value bounds (C2 shape: XOR doubles, chunks of 400 and 80 rows, [5m] windows, 15 s step)
B_HI, B_LO = 2.0 ** 513, 2.0 ** -511
EDGES = [B_HI, float(np.nextafter(B_HI, 0)), B_LO, float(np.nextafter(B_LO, 0))]
EDGES += [-x for x in EDGES] + [0.0, -0.0, 5e-324, sys.float_info.max, np.inf, -np.inf]
EDGE_ROWS = (0, 137, 399, 400, 479, 250)


def bound_store(o, val_mode):
    rng = np.random.default_rng(513 + val_mode)
    st = o.Store()
    for i, e in enumerate(EDGES):
        v = 15 + np.sin(np.arange(1, ROWS + 1)) + rng.normal(0, 1, ROWS)
        v[EDGE_ROWS[i % len(EDGE_ROWS)]] = e
        st.add_series_rows(TS, v, [400, 80], val_mode=val_mode)
    for scale in (2.0 ** 512, 2.0 ** -510):               # whole series at the edges, mixed signs: window sums cancel
        for _ in range(3):
            v = scale * (1.0 + rng.random(ROWS)) * np.where(rng.random(ROWS) < 0.5, -1.0, 1.0)
            st.add_series_rows(TS, v, [400, 80], val_mode=val_mode)
    return st


@pytest.mark.parametrize("val_mode", [1, 2], ids=["xor", "raw"])
def test_sum_kernel_value_bounds(gpu, oracle, val_mode):
    capi, ctx = gpu; o = oracle
    st = bound_store(o, val_mode)
    tab = ctx.load_series(*st.all_info_addrs())
    for q in (Q5M, Q1M):
        for name in ("FN_SUM_OVER_TIME", "FN_AVG_OVER_TIME", "FN_COUNT_OVER_TIME", "FN_RATE", "FN_INCREASE"):
            got = ctx.query(tab, getattr(capi, name), *q)
            assert_same(got, st.query(getattr(o, name), *q), "%s q=%s" % (name, q))
            same_stats(ctx, st, name)
    tab.free()


# ---- counters at the edges
def _ramp(R, v1, v2):
    """A non-decreasing counter with v[R] = v1 and v[R + 19] = v2 (the first and last rows of window R - 1 of QOFF)."""
    v = np.empty(ROWS)
    v[:R + 1] = v1 * np.arange(R + 1) / R
    v[R:R + 20] = v1 + (v2 - v1) * np.arange(20) / 19
    v[R + 19:] = v2 + (v2 - v1) * np.arange(ROWS - R - 19) / 19
    v[R], v[R + 19] = v1, v2
    return v


def skip_boundary_values():
    """(v1, v2) with v1 == (v2 - v1) * skipC exactly, skipC = 2 * durationToStart / sampledInterval (scan_wp_ctr.cuh), and v1 one ulp
    either side with the same delta."""
    skipC = 2.0 * DTS / SI
    c = 0.5 + 3 * 2.0 ** -30
    d = c / skipC
    for _ in range(200): d = float(np.nextafter(d, -np.inf))
    for _ in range(400):
        vs = [c, float(np.nextafter(c, np.inf)), float(np.nextafter(c, -np.inf))]
        if d * skipC == c and all((v + d) - v == d for v in vs):
            assert vs[1] > d * skipC > vs[2]
            return [(v, v + d) for v in vs]
        d = float(np.nextafter(d, np.inf))
    raise AssertionError("no exact skip-test boundary found")


def zero_point_boundary_values():
    """(v1, v2) with durationToZero = sampledInterval * (v1 / delta) equal to durationToStart (RateFunctions.scala:84-90 compares with
    a literal <), and one ulp either side of it."""
    out = {}
    d = 57.0
    for _ in range(60): d = float(np.nextafter(d, -np.inf))
    for _ in range(120):
        dz = SI * (1.0 / d)
        if (1.0 + d) - 1.0 == d:
            if dz == DTS: out.setdefault(0, d)
            elif dz == float(np.nextafter(DTS, np.inf)): out.setdefault(1, d)
            elif dz == float(np.nextafter(DTS, -np.inf)): out.setdefault(-1, d)
        d = float(np.nextafter(d, np.inf))
    assert sorted(out) == [-1, 0, 1], out
    return [(1.0, 1.0 + out[k]) for k in (-1, 0, 1)]


def counter_edge_series(rng):
    base = np.cumsum(rng.uniform(0, 30, ROWS))
    out = []
    out.append(2.0 ** 55 + np.cumsum(rng.uniform(0, 6, ROWS)))              # increments below one ulp (8)
    out.append(2.0 ** 53 + np.arange(ROWS) * 0.5)                           # half-ulp steps: round to even
    v = (np.arange(ROWS) % 60 + 1) * 2.9e306                               # near DBL_MAX, a reset every 60 rows: the correction overflows
    out.append(v)
    out.append(1e300 * (1 + np.arange(ROWS) % 45))
    v = base.copy(); v[200] = np.inf; out.append(v)                         # +Inf sample, then a drop
    v = base.copy(); v[399] = np.inf; out.append(v)                         # +Inf at a chunk end
    v = base.copy(); v[460:] = np.inf; out.append(v)                        # trailing +Inf
    v = base - base[0]; v[0] = 0.0; out.append(v)                           # starts at +0.0
    v = base - base[0]; v[0] = -0.0; out.append(v)                          # starts at -0.0
    v = np.zeros(ROWS); v[0] = -0.0; v[300:] = 5.0; out.append(v)
    for R_, (v1, v2) in zip((101, 230, 350), skip_boundary_values()):      # skip test: ==, +1 ulp, -1 ulp
        out.append(_ramp(R_, v1, v2))
    for R_, (v1, v2) in zip((120, 260, 370), zero_point_boundary_values()):
        out.append(_ramp(R_, v1, v2))
    return out


@pytest.mark.parametrize("val_mode", [1, 2], ids=["xor", "raw"])
def test_counters_at_value_edges(gpu, oracle, val_mode):
    capi, ctx = gpu; o = oracle
    rng = np.random.default_rng(53 + val_mode)
    series = counter_edge_series(rng)
    st = o.Store()
    for v in series:
        st.add_series_rows(TS, v, [400, 80], val_mode=val_mode, detect_drops=True)
    S = len(series); G = (S + 3) // 4
    groups = (np.arange(S) // 4).astype(np.int32)            # neighbours share a group: four series each
    tab = ctx.load_series(*st.all_info_addrs(), group_ids=groups, n_groups=G, schema_flags=capi.SCHEMA_CUMULATIVE)
    seg = items_per_group_seg(S)
    for q in (Q5M, QOFF):
        for name in ("FN_RATE", "FN_INCREASE", "FN_DELTA"):
            fn, ofn = getattr(capi, name), getattr(o, name)
            per = st.query(ofn, *q, cumulative=True)
            assert_same(ctx.query(tab, fn, *q), per, "%s q=%s" % (name, q))
            same_stats(ctx, st, name)
            for op_min in (True, False):
                aggr = "AGG_MIN" if op_min else "AGG_MAX"
                got = ctx.query(tab, fn, *q, aggr=getattr(capi, aggr))
                same_stats(ctx, st, name + " " + aggr)
                assert_same(got, expected_minmax(per, groups, G, op_min, seg), "%s %s q=%s" % (name, aggr, q))
                assert_same(got, st.query(ofn, *q, cumulative=True, aggr=getattr(o, aggr), group_ids=groups, n_groups=G), name + " (oracle)")
            gs = ctx.query(tab, fn, *q, aggr=capi.AGG_SUM)
            with np.errstate(invalid="ignore", over="ignore"):
                np.testing.assert_allclose(gs, st.query(ofn, *q, cumulative=True, aggr=o.AGG_SUM, group_ids=groups, n_groups=G), rtol=1e-9, atol=0, equal_nan=True)
    tab.free()
