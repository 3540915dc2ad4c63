"""GPU: stddev / stdvar / group across series (FILO_AGG_STDDEV / STDVAR / GROUP) against the literal restatement of the reference's
RowAggregators (tests/agg_moments_ref.py) over the oracle's per-series rows of the same chunk bytes.

The device folds the moments (Σv, Σv², n) per work item and per group and presents Σv²/n - m*m once; the reference folds the running
(stdvar, mean, count) pairwise in arrival order.  Counts and group are bit-exact with identical NaN patterns; stdvar (and stddev
squared) hold |gpu - ref| <= 1e-9 |ref| + 1e-12 m^2 per cell, m the group mean, and the NaN patterns agree except in cells the
reference marks as cancellation-dominated."""
import zlib

import numpy as np
import pytest

from tests import agg_moments_ref as R
from tests.test_gpu_parity import build_store, same_bits

pytestmark = pytest.mark.gpu
T0 = 1_700_000_000_000
OPS = (R.STDDEV, R.STDVAR, R.GROUP)


@pytest.fixture(scope="module", params=["v4", "v3", "v2", "v1"])
def gpu(request):
    """v4: the default selection (tile kernel for the SUM class, v4 counter kernel for counters, the v2 kernel behind both);
    v3: the tile kernel for the SUM class; v2: the TMA-staged warp-per-series kernel; v1: the generic kernel."""
    import os
    import filodb_b200.capi as capi
    if request.param == "v4": os.environ.pop("FILO_KERNEL", None)
    else: os.environ["FILO_KERNEL"] = request.param
    ctx = capi.Context(0)
    yield capi, ctx
    ctx.close()
    os.environ.pop("FILO_KERNEL", None)


_REF = {}


def reference(per, groups, n_groups, key=None):
    """{op: (presented, counts)} and the group means of the restatement (kept per key: the kernel generations share it)."""
    if key is not None and key in _REF:
        return _REF[key]
    ref = {op: R.aggregate(op, per, groups, n_groups) for op in OPS}, R.group_means(per, groups, n_groups)
    if key is not None:
        _REF[key] = ref
    return ref


def check_moments(capi, ctx, tab, per, groups, n_groups, fn, q, what, key=None):
    """All three operators on the device against the reference restatement over per-series rows `per` [S, T]."""
    refs, means = reference(per, groups, n_groups, key)
    ref_var = refs[R.STDVAR][0]
    for op in OPS:
        gv, gc = ctx.query(tab, fn, *q, aggr=op)
        exp, cnt = refs[op]
        assert (gc == cnt).all(), "%s op %d: counts" % (what, op)
        if op == R.GROUP:
            assert same_bits(gv, exp), "%s: group" % what
        else:
            R.assert_moments_close(op, gv, exp, means, ref_var, "%s op %d" % (what, op))
        if op != R.GROUP:                                   # presented from the partial form on the device: bit for bit
            check_partial_present(capi, ctx, tab, fn, q, op, gv, gc)
    # group's partial form is exactly the count partial
    pg = ctx.query(tab, fn, *q, aggr=capi.AGG_GROUP, flags=capi.Q_PARTIAL)
    pc = ctx.query(tab, fn, *q, aggr=capi.AGG_COUNT, flags=capi.Q_PARTIAL)
    assert same_bits(pg[0], pc[0]) and (pg[1] == pc[1]).all()


def check_partial_present(capi, ctx, tab, fn, q, op, presented, counts):
    import torch
    pv, pc = ctx.query(tab, fn, *q, aggr=op, flags=capi.Q_PARTIAL)
    assert pv.shape == (2,) + presented.shape and (pc == counts).all()
    n = presented.size
    dv = torch.from_numpy(pv.reshape(-1).copy()).cuda(); dc = torch.from_numpy(pc.reshape(-1).copy()).cuda()
    do = torch.empty(n, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    ctx.present_partials(op, n, dv.data_ptr(), dc.data_ptr(), do.data_ptr())
    torch.cuda.synchronize()
    assert same_bits(do.cpu().numpy().reshape(presented.shape), presented), "partial + present differs from the presented form"


def _groups(rng, S, G):
    g = rng.integers(0, G - 2, S).astype(np.int32)           # group G-2 stays empty
    g[S // 2] = G - 1                                         # group G-1 holds one series
    return g


SUM_CASES = [("gauge", 1, 0, False, 0.02), ("gauge", 2, 0, False, 0.0), ("linear", 0, 0, False, 0.0)]


@pytest.mark.parametrize("case", SUM_CASES, ids=[("%s-v%d-nan%g" % (c[0], c[1], c[4])) for c in SUM_CASES])
def test_sum_class_sum_over_time(gpu, oracle, case):
    """Gauge sum_over_time / avg_over_time: the tile kernel's moments mode under v4 / v3."""
    capi, ctx = gpu; o = oracle
    kind, val_mode, jitter, cumulative, nan_frac = case
    rng = np.random.default_rng(zlib.crc32(repr(case).encode()))
    S, G = 120, 7
    st = build_store(o, rng, S, kind, val_mode, jitter, cumulative, nan_frac)
    groups = _groups(rng, S, G)
    tab = ctx.load_series(*st.all_info_addrs(), group_ids=groups, n_groups=G)
    for name in ("FN_SUM_OVER_TIME", "FN_AVG_OVER_TIME"):
        q = (T0 + 300000, 15000, T0 + 479 * 15000, 300000)
        per = st.query(getattr(o, name), *q)
        check_moments(capi, ctx, tab, per, groups, G, getattr(capi, name), q, "%s %s" % (case, name))
    tab.free()


def test_counter_rate_with_resets(gpu, oracle):
    """rate / increase over counters with resets and drop flags: the v4 counter kernel's moments mode under v4."""
    capi, ctx = gpu; o = oracle
    rng = np.random.default_rng(77)
    S, G = 100, 6
    st = build_store(o, rng, S, "counter", 1, 0, True, 0.01)
    groups = _groups(rng, S, G)
    tab = ctx.load_series(*st.all_info_addrs(), group_ids=groups, n_groups=G, schema_flags=capi.SCHEMA_CUMULATIVE)
    for name, q in (("FN_RATE", (T0 + 300000, 15000, T0 + 479 * 15000, 300000)), ("FN_INCREASE", (T0 + 60000, 15000, T0 + 479 * 15000, 60000))):
        per = st.query(getattr(o, name), *q, cumulative=True)
        check_moments(capi, ctx, tab, per, groups, G, getattr(capi, name), q, name)
    tab.free()


DECLINED = [  # kind, val_mode, jitter, cumulative, nan_frac, function, params
    ("gauge", 1, 3000, False, 0.02, "FN_SUM_OVER_TIME", ()),      # jittered timestamps: the tile kernel declines, the v2 kernel takes them
    ("gauge", 1, 0, False, 0.05, "FN_MAX_OVER_TIME", ()),         # NaN markers, a MINMAX-class function: v2 only
    ("intcounter", 0, 0, True, 0.0, "FN_RATE", ()),               # DDV-long values
    ("gauge", 2, 0, False, 0.02, "FN_QUANTILE_OVER_TIME", (0.9,)),
    ("counter", 1, 2000, True, 0.01, "FN_RATE", ()),              # irregular counters
]


@pytest.mark.parametrize("case", DECLINED, ids=["%s-j%d-%s" % (c[0], c[2], c[5]) for c in DECLINED])
def test_declined_shapes(gpu, oracle, case):
    capi, ctx = gpu; o = oracle
    kind, val_mode, jitter, cumulative, nan_frac, name, params = case
    rng = np.random.default_rng(zlib.crc32(repr(case).encode()))
    S, G = 60, 5
    st = build_store(o, rng, S, kind, val_mode, jitter, cumulative, nan_frac)
    groups = _groups(rng, S, G)
    tab = ctx.load_series(*st.all_info_addrs(), group_ids=groups, n_groups=G, schema_flags=capi.SCHEMA_CUMULATIVE if cumulative else 0)
    q = (T0 + 300000, 15000, T0 + 479 * 15000, 300000)
    ctx.set_fn_args(*(tuple(params) + (0.0, 0.0))[:2])
    try:
        per = st.query(getattr(o, name), *q, cumulative=cumulative, params=tuple(params) + (0.0, 0.0))
        check_moments(capi, ctx, tab, per, groups, G, getattr(capi, name), q, str(case))
    finally:
        ctx.set_fn_args(0.0, 0.0)
    tab.free()


def test_infinite_input_gives_nan(gpu, oracle):
    """A series holding +Inf makes its group's stdvar and stddev NaN in every window that sees it (Σv² - ... = Inf - Inf)."""
    capi, ctx = gpu; o = oracle
    rng = np.random.default_rng(5)
    S, G = 30, 3
    st = o.Store()
    for s in range(S):
        ts = T0 + np.arange(480, dtype=np.int64) * 15000
        v = 15 + np.sin(np.arange(1, 481)) + rng.normal(0, 1, 480)
        if s == 4: v[200] = np.inf
        st.add_series_rows(ts, v, [400, 80], val_mode=2)
    groups = (np.arange(S) % G).astype(np.int32)
    tab = ctx.load_series(*st.all_info_addrs(), group_ids=groups, n_groups=G)
    q = (T0 + 300000, 15000, T0 + 479 * 15000, 300000)
    per = st.query(o.FN_SUM_OVER_TIME, *q)
    inf_cells = np.isinf(per[4])
    assert inf_cells.any()
    for op in (R.STDDEV, R.STDVAR):
        gv, gc = ctx.query(tab, capi.FN_SUM_OVER_TIME, *q, aggr=op)
        assert np.isnan(gv[groups[4]][inf_cells]).all()
        assert not np.isnan(gv[groups[4]][~inf_cells]).any()
        assert not np.isnan(gv[[g for g in range(G) if g != groups[4]]]).any()
    tab.free()


_BIG = {}


def test_large_table_multi_series_items(gpu, oracle):
    """70 000 gauge series in 40 groups: work items of several series (build_groups_new: S / (SMs * 256) per item on a 132-SM H100)
    through the tile kernel, and counters through the v4 counter kernel; the oracle reads the same arena bytes."""
    capi, ctx = gpu; o = oracle
    S, G, ROWS = 70_000, 40, 240
    q = (T0 + 300000, 15000, T0 + (ROWS - 1) * 15000, 300000)
    for label, kw, name in (("gauge", dict(value_kind=0, value_enc=1, nan_per_million=20000), "FN_SUM_OVER_TIME"),
                            ("counter", dict(value_kind=1, value_enc=1, reset_period=60, schema_flags=capi.SCHEMA_CUMULATIVE), "FN_RATE")):
        tab = ctx.synth_table(S, ROWS, 400, T0, 15000, n_groups=G, seed=11, **kw)
        if label not in _BIG:
            arena, rec_off = tab.read_arena(0, S)
            ost = o.Store(); ost.add_from_arena(arena, rec_off, S)
            per = ost.query(getattr(o, name), *q, cumulative=label == "counter", threads=8)
            _BIG[label] = (per, o.synth_group_ids(11, 0, S, G), (arena, ost))
        per, groups, _ = _BIG[label]
        assert np.bincount(groups, minlength=G).min() > 1000
        check_moments(capi, ctx, tab, per, groups, G, getattr(capi, name), q, "large " + label, key=label)
        tab.free()


def test_fused_gpu_exec_stddev(oracle):
    """FusedGpuExec with AggregateMapReduce(AGG_STDDEV): PeriodicSamplesMapper + stddev by group end to end."""
    from filodb_b200 import capi, exec as fx
    o = oracle
    rng = np.random.default_rng(9)
    S, G = 40, 4
    st = build_store(o, rng, S, "gauge", 1, 0, False, 0.02)
    groups = (np.arange(S) * 3 % G).astype(np.int32)
    source = [fx.RawDataRangeVector(list(st.info_addrs(s)), int(groups[s])) for s in range(S)]
    q = (T0 + 300000, 15000, T0 + 479 * 15000, 300000)
    ex = fx.FusedGpuExec(0)
    try:
        psm = fx.PeriodicSamplesMapper(*q[:3], window=q[3], functionId=capi.FN_SUM_OVER_TIME)
        r = ex.execute(source, psm, fx.AggregateMapReduce(capi.AGG_STDDEV, numGroups=G))
    finally:
        ex.close()
    per = st.query(o.FN_SUM_OVER_TIME, *q)
    exp, cnt = R.aggregate(R.STDDEV, per, groups, G)
    ref_var, _ = R.aggregate(R.STDVAR, per, groups, G)
    assert (r.aux == cnt).all()
    R.assert_moments_close(R.STDDEV, r.values, exp, R.group_means(per, groups, G), ref_var, "FusedGpuExec stddev")
