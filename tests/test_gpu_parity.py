"""GPU parity: the CUDA path (through the C-ABI) vs the CPU oracle on the same chunk bytes.

Per-series results (PeriodicSamplesMapper) must be BIT-EXACT: the kernels follow the reference's operation order and are
compiled without FMA contraction.  Across-series aggregates: min/max/count bit-exact; sum/avg within 1e-9 relative (the
reference folds in arrival order, the device folds per work item then per group — SURVEY.md §7 "FP parity")."""
import math
import zlib
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
NaN = float("nan")


@pytest.fixture(scope="module", params=["v4", "v3", "v2", "v1"])
def gpu(request):
    """Every test runs against every kernel generation: v4 (the default: warp-pipeline kernels scan_wp_sum / scan_wp_ctr, with the v2 kernel
    behind them for what they decline), v3 (round-1 tile kernel), v2 (TMA-staged warp per series), v1 (generic, global-memory reads)."""
    import os
    import filodb_b200.capi as capi
    if request.param == "v4": os.environ.pop("FILO_KERNEL", None)
    else: os.environ["FILO_KERNEL"] = request.param
    ctx = capi.Context(0)
    yield capi, ctx
    ctx.close()
    os.environ.pop("FILO_KERNEL", None)


def same_bits(a, b):
    a = np.ascontiguousarray(a, np.float64); b = np.ascontiguousarray(b, np.float64)
    an, bn = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and (an == bn).all() and (a[~an].view(np.uint64) == b[~bn].view(np.uint64)).all()


def assert_same(a, b, what=""):
    if not same_bits(a, b):
        a = np.ascontiguousarray(a, np.float64); b = np.ascontiguousarray(b, np.float64)
        if a.shape != b.shape:
            raise AssertionError("%s: shapes %s vs %s" % (what, a.shape, b.shape))
        bad = np.argwhere(~((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))))      # bits: +0.0 != -0.0
        i = tuple(bad[0])
        raise AssertionError("%s: %d mismatches, first at %s: gpu=%r oracle=%r" % (what, len(bad), i, a[i], b[i]))


ALL_FNS = ["FN_LAST", "FN_RATE", "FN_INCREASE", "FN_DELTA", "FN_SUM_OVER_TIME", "FN_AVG_OVER_TIME", "FN_COUNT_OVER_TIME",
           "FN_MIN_OVER_TIME", "FN_MAX_OVER_TIME", "FN_TIMESTAMP"]


def build_store(o, rng, n_series, kind, val_mode, jitter, detect_drops, nan_frac=0.0, rows=480, chunks=(400, 80), t0=1_700_000_000_000, interval=15000):
    st = o.Store()
    for s in range(n_series):
        ts = t0 + np.arange(rows, dtype=np.int64) * interval
        if jitter:
            ts = ts + rng.integers(-jitter, jitter + 1, rows)
        if kind == "gauge":
            v = 15 + np.sin(np.arange(1, rows + 1)) + rng.normal(0, 1, rows)
        elif kind == "counter":
            v = np.cumsum(np.maximum(0, 15 + np.sin(np.arange(1, rows + 1)) + rng.normal(0, 1, rows)))
            for r in np.nonzero(rng.random(rows) < 0.01)[0]:
                if r > 0: v[r:] = v[r:] - v[r] + rng.random() * 5
        elif kind == "intcounter":
            v = np.cumsum(rng.integers(0, 40, rows)).astype(float)
            for r in np.nonzero(rng.random(rows) < 0.01)[0]:
                if r > 0: v[r:] = v[r:] - v[r] + float(rng.integers(0, 5))
        elif kind == "linear":
            v = np.arange(1, rows + 1, dtype=float) * (s + 1)
        else:
            raise ValueError(kind)
        if nan_frac:
            v = v.copy(); v[rng.random(rows) < nan_frac] = NaN
        st.add_series_rows(ts, v, list(chunks), val_mode=val_mode, detect_drops=detect_drops)
    return st


CASES = [
    # kind, val_mode, jitter, cumulative/detectDrops, nan_frac
    ("gauge", 2, 0, False, 0.0),
    ("gauge", 1, 0, False, 0.02),
    ("gauge", 0, 3000, False, 0.02),
    ("counter", 2, 0, True, 0.01),
    ("counter", 1, 2000, True, 0.01),
    ("intcounter", 0, 0, True, 0.0),
    ("intcounter", 0, 100, True, 0.0),
    ("linear", 0, 0, False, 0.0),
    ("gauge", 1, 0, True, 0.05),
]


@pytest.mark.parametrize("case", CASES, ids=[("%s-v%d-j%d-%s-nan%g" % c) for c in CASES])
def test_per_series_bit_exact(gpu, oracle, case):
    capi, ctx = gpu; o = oracle
    kind, val_mode, jitter, cumulative, nan_frac = case
    rng = np.random.default_rng(zlib.crc32(repr(case).encode()))      # reproducible across processes (str hashes are salted)
    st = build_store(o, rng, 40, kind, val_mode, jitter, cumulative, nan_frac)
    nch, addrs = st.all_info_addrs()
    tab = ctx.load_series(nch, addrs, schema_flags=capi.SCHEMA_CUMULATIVE if cumulative else 0)
    ti = tab.info()
    assert ti.n_series == 40 and ti.n_samples == 40 * 480
    assert ti.algorithmic_bytes == st.algorithmic_bytes()
    t0 = 1_700_000_000_000
    queries = [(t0 + 300000, 15000, t0 + 479 * 15000, 300000),      # BASELINE shape: [5m] step 15s
               (t0 + 60000, 15000, t0 + 479 * 15000 + 90000, 60000),  # [1m], runs past the data
               (t0 - 100000, 47000, t0 + 480 * 15000, 333333),        # unaligned step/window
               (t0 + 5999000, 1, t0 + 5999000, 300000)]               # instant query
    for (start, step, end, window) in queries:
        for name in ALL_FNS:
            fn = getattr(capi, name)
            got = ctx.query(tab, fn, start, step, end, window)
            exp = st.query(getattr(o, name), start, step, end, window, cumulative=cumulative)
            assert_same(got, exp, "%s %s q=%s" % (case, name, (start, step, end, window)))
            assert ctx.last_stats["samples_scanned"] == st.last_stats["samples_scanned"]
            assert ctx.last_stats["bytes_scanned"] == st.last_stats["bytes_scanned"]
    tab.free()


def test_golden_known_answers_on_gpu(gpu, oracle):
    """The reference's own known-answer tests, through the CUDA path (WindowIteratorSpec.scala:219-284, RateFunctionsSpec.scala:58-158)."""
    capi, ctx = gpu; o = oracle
    from tests.test_oracle_golden import PROM_SAMPLES, PROM_EXPECTED, OT_SAMPLES, COUNTER_SAMPLES, _store_one
    st = _store_one(o, PROM_SAMPLES)
    tab = ctx.load_series(*st.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE)
    start, step, end, window = 1548191496000, 15000, 1548191796000, 300000
    out = ctx.query(tab, capi.FN_RATE, start, step, end, window)[0]
    for k, v in enumerate(out):
        if start + k * step in PROM_EXPECTED:
            assert v == pytest.approx(PROM_EXPECTED[start + k * step], abs=1e-10)
    samples = [(1614821996000, NaN), (1614821996100, 489.0), (1614821997000, NaN), (1614822566000, 19.0),
               (1614822596000, 26.0), (1614822626000, 26.0), (1614822656000, 26.0), (1614822686000, 26.0),
               (1614822716000, 26.0), (1614822717000, NaN), (1614822866000, 5.0)]
    st = _store_one(o, samples)
    tab = ctx.load_series(*st.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE)
    assert ctx.query(tab, capi.FN_RATE, 1614822880000, 15000, 1614822880000, 900000)[0, 0] == 0.5870753512132821
    st = _store_one(o, OT_SAMPLES, detect_drops=False)
    tab = ctx.load_series(*st.all_info_addrs())
    out = ctx.query(tab, capi.FN_SUM_OVER_TIME, 50000, 100000, 1100000, 100000)[0]
    assert [(50000 + 100000 * k, v) for k, v in enumerate(out) if not math.isnan(v)] == \
        [(150000, 1.0), (250000, 5.0), (350000, 12.0), (450000, 13.0), (750000, 17.0)]
    # drops in the middle of chunks, 1 and 2 chunks (RateFunctionsSpec.scala:117-158)
    reset1 = [(8072000, 4419.0), (8082100, 4511.0), (8092196, 4614.0), (8102215, 4724.0), (8112223, 4909.0),
              (8122388, 948.0), (8132570, 1000.0), (8142822, 1095.0), (8152858, 1102.0), (8162999, 1201.0)]
    reset2 = [(8173000, 1325.0), (8183000, 1511.0), (8193000, 214.0), (8203000, 324.0), (8213000, 409.0)]
    expected = (409.0 + 4909.0 + 1511.0 - 4419.0) / (8213000 - 8072000) * 1000
    for rows in ([10, 5], [15]):
        st = _store_one(o, reset1 + reset2, chunk_rows=rows)
        tab = ctx.load_series(*st.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE)
        assert ctx.query(tab, capi.FN_RATE, 8213070, 10000, 8213070, 8213070 - 8071950)[0, 0] == pytest.approx(expected, abs=1e-7)


def test_edge_cases(gpu, oracle):
    capi, ctx = gpu; o = oracle
    rng = np.random.default_rng(77)
    st = o.Store()
    t0 = 1_700_000_000_000
    # ragged: 1-row chunks, single-NaN chunk, 2-row chunk (raw long timestamps), many small chunks, a gap between chunks
    st.add_series_rows([t0], [5.0], [1], val_mode=2, detect_drops=True)
    st.add_series_rows([t0, t0 + 15000, t0 + 30000], [1.0, 2.0, NaN], [2, 1], val_mode=2, detect_drops=True)
    ts = t0 + np.arange(100) * 15000
    st.add_series_rows(ts, rng.random(100), [7] * 14 + [2], val_mode=1)
    ts2 = np.concatenate([t0 + np.arange(50) * 15000, t0 + 3_000_000 + np.arange(50) * 15000])
    st.add_series_rows(ts2, np.cumsum(rng.random(100)), [50, 50], val_mode=2, detect_drops=True)
    st.add_series_rows(ts, np.full(100, NaN), [60, 40], val_mode=2)          # all NaN
    st.add_series_rows(ts, np.zeros(100), [60, 40], val_mode=0)              # constant 0 -> const DDV values
    st.add_series_rows(ts, -np.arange(100.0), [60, 40], val_mode=0, detect_drops=True)   # decreasing integral counter
    st.add_series_rows(ts, np.where(np.arange(100) % 2 == 0, -0.0, 0.0), [100], val_mode=2)
    for cumulative in (False, True):
        tab = ctx.load_series(*st.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE if cumulative else 0)
        for (start, step, end, window) in [(t0, 15000, t0 + 100 * 15000, 60000), (t0 - 10**6, 7000, t0 + 4 * 10**6, 123456),
                                           (t0 + 10**7, 15000, t0 + 10**7 + 60000, 30000)]:
            for name in ALL_FNS:
                got = ctx.query(tab, getattr(capi, name), start, step, end, window)
                exp = st.query(getattr(o, name), start, step, end, window, cumulative=cumulative)
                assert_same(got, exp, "%s cumulative=%s q=%s" % (name, cumulative, (start, step, end, window)))
        tab.free()
    # empty table
    tab = ctx.load_series(np.zeros(0, np.int32), np.zeros(0, np.uint64))
    assert ctx.query(tab, capi.FN_SUM_OVER_TIME, t0, 15000, t0 + 60000, 30000).shape == (0, 5)
    # non-inclusive range config (filodb.query.inclusive-range = false)
    ctx2 = capi.Context(0, inclusive_range=False)
    tab = ctx2.load_series(*st.all_info_addrs())
    for name in ("FN_SUM_OVER_TIME", "FN_RATE", "FN_LAST"):
        got = ctx2.query(tab, getattr(capi, name), t0, 15000, t0 + 100 * 15000, 60000)
        exp = st.query(getattr(o, name), t0, 15000, t0 + 100 * 15000, 60000, inclusive=False)
        assert_same(got, exp, name + " non-inclusive")
    ctx2.close()


def test_many_chunks_and_long_series(gpu, oracle):
    """Series far larger than the shared-memory scratch (global-scratch path) and > 8 chunks (binary chunk search)."""
    capi, ctx = gpu; o = oracle
    rng = np.random.default_rng(5)
    rows = 6000
    t0 = 1_700_000_000_000
    st = o.Store()
    for s in range(6):
        ts = t0 + np.arange(rows, dtype=np.int64) * 10000 + (rng.integers(-2000, 2001, rows) if s % 2 else 0)
        v = np.cumsum(rng.random(rows) * 10)
        st.add_series_rows(ts, v, [400] * 15, val_mode=s % 3, detect_drops=True)
    tab = ctx.load_series(*st.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE)
    for (start, step, end, window) in [(t0 + 600000, 60000, t0 + rows * 10000, 600000), (t0, 3600000, t0 + rows * 10000, 7200000)]:
        for name in ("FN_RATE", "FN_SUM_OVER_TIME", "FN_MAX_OVER_TIME", "FN_LAST", "FN_COUNT_OVER_TIME"):
            got = ctx.query(tab, getattr(capi, name), start, step, end, window)
            exp = st.query(getattr(o, name), start, step, end, window, cumulative=True)
            assert_same(got, exp, name)


def test_aggregates(gpu, oracle):
    capi, ctx = gpu; o = oracle
    rng = np.random.default_rng(123)
    S, G = 300, 7
    st = build_store(o, rng, S, "counter", 1, 0, True, 0.01)
    groups = rng.integers(0, G, S).astype(np.int32)
    groups[groups == 3] = 2      # leave group 3 empty
    nch, addrs = st.all_info_addrs()
    tab = ctx.load_series(nch, addrs, group_ids=groups, n_groups=G, schema_flags=capi.SCHEMA_CUMULATIVE)
    t0 = 1_700_000_000_000
    start, step, end, window = t0 + 60000, 15000, t0 + 479 * 15000, 60000
    for fn_name in ("FN_INCREASE", "FN_RATE", "FN_COUNT_OVER_TIME"):
        fn = getattr(capi, fn_name); ofn = getattr(o, fn_name)
        for aggr_name in ("AGG_SUM", "AGG_MIN", "AGG_MAX", "AGG_COUNT", "AGG_AVG"):
            aggr = getattr(capi, aggr_name)
            got = ctx.query(tab, fn, start, step, end, window, aggr=aggr)
            exp = st.query(ofn, start, step, end, window, cumulative=True, aggr=getattr(o, aggr_name), group_ids=groups, n_groups=G)
            if aggr_name == "AGG_AVG":
                (gv, gc), (ev, ec) = got, exp
                assert (gc == ec).all()
                assert np.isnan(gv[3]).all()
                np.testing.assert_allclose(gv, ev, rtol=1e-9, atol=0, equal_nan=True)
            elif aggr_name == "AGG_SUM":
                np.testing.assert_allclose(got, exp, rtol=1e-9, atol=0, equal_nan=True)
            else:
                assert_same(got, exp, fn_name + " " + aggr_name)
    # no grouping: one group
    tab.set_groups(None, 1)
    got = ctx.query(tab, capi.FN_RATE, start, step, end, window, aggr=capi.AGG_SUM)
    exp = st.query(o.FN_RATE, start, step, end, window, cumulative=True, aggr=o.AGG_SUM, n_groups=1)
    np.testing.assert_allclose(got, exp, rtol=1e-9, equal_nan=True)
    # partial (mergeable) form + present
    tab.set_groups(groups, G)
    pv, pc = ctx.query(tab, capi.FN_RATE, start, step, end, window, aggr=capi.AGG_AVG, flags=capi.Q_PARTIAL)
    ev, ec = st.query(o.FN_RATE, start, step, end, window, cumulative=True, aggr=o.AGG_AVG, group_ids=groups, n_groups=G)
    assert (pc == ec).all()
    with np.errstate(invalid="ignore", divide="ignore"):
        np.testing.assert_allclose(np.where(pc > 0, pv / pc, np.nan), ev, rtol=1e-9, equal_nan=True)
    # topk / bottomk
    for aggr_name, rev in (("AGG_TOPK", True), ("AGG_BOTTOMK", False)):
        gv, gi = ctx.query(tab, capi.FN_RATE, start, step, end, window, aggr=getattr(capi, aggr_name), k=3)
        ev, ei = st.query(o.FN_RATE, start, step, end, window, cumulative=True, aggr=getattr(o, aggr_name), k=3, group_ids=groups, n_groups=G)
        assert_same(gv, ev, aggr_name + " values")
        per = st.query(o.FN_RATE, start, step, end, window, cumulative=True)
        ok = gi >= 0
        assert (ok == (ei >= 0)).all()
        gs, ts_ = np.nonzero(ok.any(axis=2))
        for g, t in zip(gs, ts_):
            for j in range(3):
                if gi[g, t, j] >= 0:
                    assert groups[gi[g, t, j]] == g and same_bits(per[gi[g, t, j], t], gv[g, t, j])
    tab.free()


def test_error_paths(gpu, oracle):
    capi, ctx = gpu; o = oracle
    t0 = 1_700_000_000_000
    st = o.Store()
    ts = t0 + np.arange(10) * 15000
    st.add_series_rows(ts, np.arange(10.0) + 0.5, [10], val_mode=2)
    # corrupt wire format -> CorruptVectorException equivalent (ChunkSetInfo.scala:424-429)
    bad = st.vector_bytes(0, 0, 1).copy(); bad[4] = 0x07
    s2 = o.Store(); s2.add_series(); s2.add_chunk_raw(0, int(ts[0]), int(ts[-1]), 10, st.vector_bytes(0, 0, 0), bad)
    with pytest.raises(capi.FiloError) as e:
        ctx.load_series(*s2.all_info_addrs())
    assert e.value.code == capi.ERR_CORRUPT_VECTOR
    # numRows larger than the vectors
    s3 = o.Store(); s3.add_series(); s3.add_chunk_raw(0, int(ts[0]), int(ts[-1]), 11, st.vector_bytes(0, 0, 0), st.vector_bytes(0, 0, 1))
    with pytest.raises(capi.FiloError) as e:
        ctx.load_series(*s3.all_info_addrs())
    assert e.value.code == capi.ERR_CORRUPT_VECTOR
    # chunks out of time order -> unsupported (caller keeps the JVM path)
    s4 = o.Store(); s4.add_series()
    s4.add_chunk(0, ts + 10**6, np.arange(10.0)); s4.add_chunk(0, ts, np.arange(10.0))
    with pytest.raises(capi.FiloError) as e:
        ctx.load_series(*s4.all_info_addrs())
    assert e.value.code == capi.ERR_UNSUPPORTED
    tab = ctx.load_series(*st.all_info_addrs())
    for args, code in (((capi.FN_SUM_OVER_TIME, t0 + 100, 15000, t0, 1000), capi.ERR_INVALID_ARG),       # start > end
                       ((capi.FN_SUM_OVER_TIME, t0, 0, t0 + 1000, 1000), capi.ERR_INVALID_ARG),            # step 0 on a range
                       ((capi.FN_SUM_OVER_TIME, t0, 15000, t0 + 1000, 0), capi.ERR_INVALID_ARG),           # window 0
                       ((99, t0, 15000, t0 + 1000, 1000), capi.ERR_INVALID_ARG)):
        with pytest.raises(capi.FiloError) as e:
            ctx.query(tab, *args)
        assert e.value.code == code
    # a device-detected error of a non-synchronising query (stats == NULL) is not lost: filo_ctx_check, or the next call, returns it.
    # XOR doubles under a Long-column schema are only seen by the kernel (the wire type is valid for the loader).
    import torch
    sx = o.Store(); sx.add_series_rows(ts, np.arange(10.0) + 0.25, [10], val_mode=1)
    tabx = ctx.load_series(*sx.all_info_addrs(), schema_flags=capi.SCHEMA_LONG_VALUES)
    T = capi.num_windows(t0, 15000, t0 + 135000)
    dout = torch.empty(T, dtype=torch.float64, device="cuda")
    with pytest.raises(capi.FiloError) as e:
        ctx.query_device(tabx, capi.FN_SUM_OVER_TIME, t0, 15000, t0 + 135000, 60000, dout.data_ptr(), want_stats=True)
    assert e.value.code == capi.ERR_CORRUPT_VECTOR
    ctx.query_device(tabx, capi.FN_SUM_OVER_TIME, t0, 15000, t0 + 135000, 60000, dout.data_ptr(), want_stats=False)      # returns before the kernel ran
    with pytest.raises(capi.FiloError) as e:
        ctx.check()
    assert e.value.code == capi.ERR_CORRUPT_VECTOR
    ctx.check()                                             # reported once
    ctx.query_device(tabx, capi.FN_SUM_OVER_TIME, t0, 15000, t0 + 135000, 60000, dout.data_ptr(), want_stats=False)
    torch.cuda.synchronize()
    with pytest.raises(capi.FiloError) as e:                # ... or by the next call on the ctx
        ctx.query(tab, capi.FN_SUM_OVER_TIME, t0, 15000, t0 + 135000, 60000)
    assert e.value.code == capi.ERR_CORRUPT_VECTOR
    tabx.free()
    ctx3 = capi.Context(0, min_step_ms=5000, group_by_cardinality_limit=2, max_data_per_shard_query=10)
    with pytest.raises(capi.FiloError) as e:
        ctx3.load_series(*st.all_info_addrs())
    assert e.value.code == capi.ERR_QUERY_LIMIT
    ctx3.close()
    ctx4 = capi.Context(0, min_step_ms=5000, group_by_cardinality_limit=2)
    tab4 = ctx4.load_series(*st.all_info_addrs())
    with pytest.raises(capi.FiloError) as e:
        ctx4.query(tab4, capi.FN_SUM_OVER_TIME, t0, 1000, t0 + 60000, 30000)
    assert e.value.code == capi.ERR_BAD_QUERY
    with pytest.raises(capi.FiloError) as e:
        tab4.set_groups(np.zeros(1, np.int32), 3)
    assert e.value.code == capi.ERR_QUERY_LIMIT
    ctx4.close()


SYNTH_CASES = [
    dict(value_kind=0, value_enc=0, ts_jitter_ms=0),
    dict(value_kind=0, value_enc=1, ts_jitter_ms=0, nan_per_million=200000),
    dict(value_kind=1, value_enc=1, ts_jitter_ms=2000, reset_period=100, schema_flags=1, nan_per_million=100000),
    dict(value_kind=2, value_enc=2, ts_jitter_ms=100, reset_period=150, schema_flags=1),
    dict(value_kind=1, value_enc=0, ts_jitter_ms=0, reset_period=50, schema_flags=1),
    dict(value_kind=2, value_enc=2, ts_jitter_ms=0, schema_flags=1, nan_per_million=300000),
]


@pytest.mark.parametrize("case", SYNTH_CASES, ids=[str(i) for i in range(len(SYNTH_CASES))])
def test_gpu_encoder_matches_reference_appenders(gpu, oracle, case):
    """The GPU generator/encoder writes exactly the bytes FiloDB's appenders' optimize() would (oracle restatement)."""
    capi, ctx = gpu; o = oracle
    from tests import synth_ref as sr
    rows, rpc, S, seed, base = 173, 64, 24, 99, 1000
    t0, interval = 1_700_000_000_000, 15000
    tab = ctx.synth_table(S, rows, rows_per_chunk=rpc, t0_ms=t0, interval_ms=interval, seed=seed, series_id_base=base, n_groups=5, **case)
    st_tab = capi.sin_table(rows)
    cumulative = bool(case.get("schema_flags", 0) & 1)
    val_mode = {0: o.VAL_RAW, 1: o.VAL_XOR, 2: o.VAL_OPTIMIZE}[case["value_enc"]]
    st = o.Store()
    for s in range(S):
        ts, vals = sr.gen_series(seed, base + s, rows, rpc, t0, interval, case.get("ts_jitter_ms", 0), case["value_kind"],
                                 case.get("reset_period", 0), case.get("nan_per_million", 0), st_tab)
        st.add_series_rows(ts, vals, sr.chunk_rows(rows, rpc), val_mode=val_mode, detect_drops=cumulative)
    alg = 0
    for s in range(S):
        rec = tab.read_record(s)
        hdr = np.frombuffer(rec[:16].tobytes(), np.uint32)
        assert hdr[0] == rec.size and hdr[1] == len(sr.chunk_rows(rows, rpc)) and hdr[2] == rows
        for c in range(int(hdr[1])):
            e = rec[16 + 32 * c: 48 + 32 * c].tobytes()
            start_t, end_t = np.frombuffer(e[:16], np.int64)
            nrows, ts_off, val_off, row_base = np.frombuffer(e[16:], np.uint32)
            tsb, vb = st.vector_bytes(s, c, 0), st.vector_bytes(s, c, 1)
            assert rec[ts_off:ts_off + tsb.size].tobytes() == tsb.tobytes(), "ts vector bytes series %d chunk %d" % (s, c)
            assert rec[val_off:val_off + vb.size].tobytes() == vb.tobytes(), "value vector bytes series %d chunk %d" % (s, c)
            alg += 28 + 16 + tsb.size + vb.size
    assert tab.info().algorithmic_bytes == alg == st.algorithmic_bytes()
    # and queries over the synthetic table agree with the oracle over the re-built chunks
    start, step, end, window = t0 + 60000, 15000, t0 + rows * interval, 120000
    for name in ("FN_RATE", "FN_SUM_OVER_TIME", "FN_LAST"):
        got = ctx.query(tab, getattr(capi, name), start, step, end, window)
        exp = st.query(getattr(o, name), start, step, end, window, cumulative=cumulative)
        assert_same(got, exp, name)
    groups = np.array([sr.group_id(seed, base + s, 5) for s in range(S)], np.int32)
    got = ctx.query(tab, capi.FN_SUM_OVER_TIME, start, step, end, window, aggr=capi.AGG_MAX)
    exp = st.query(o.FN_SUM_OVER_TIME, start, step, end, window, cumulative=cumulative, aggr=o.AGG_MAX, group_ids=groups, n_groups=5)
    assert_same(got, exp, "group max over synthetic table")


def test_scan_series_pipelined_matches_oracle(gpu, oracle):
    """filo_scan_series (ingest + query + read-back in one pipelined call) returns what load + query returns, bit for bit,
    with the same scan counters; errors surface the same way."""
    capi, ctx = gpu; o = oracle
    rng = np.random.default_rng(5)
    t0 = 1_700_000_000_000
    for kind, cumulative, nan_frac in (("gauge", False, 0.02), ("counter", True, 0.01)):
        st = build_store(o, rng, 300, kind, 2, 0, cumulative, nan_frac)
        nch, addrs = st.all_info_addrs()
        flags = capi.SCHEMA_CUMULATIVE if cumulative else 0
        for (start, step, end, window) in [(t0, 15000, t0 + 7200000, 300000), (t0 + 60000, 47000, t0 + 480 * 15000, 333333)]:
            for name in ("FN_RATE", "FN_SUM_OVER_TIME", "FN_MAX_OVER_TIME", "FN_LAST"):
                got = ctx.scan_series(nch, addrs, getattr(capi, name), start, step, end, window, schema_flags=flags)
                stats = dict(ctx.last_stats)
                exp = st.query(getattr(o, name), start, step, end, window, cumulative=cumulative)
                assert_same(got, exp, "scan_series %s %s" % (kind, name))
                assert stats["samples_scanned"] == st.last_stats["samples_scanned"]
                assert stats["bytes_scanned"] == st.last_stats["bytes_scanned"]
                assert stats["d2h_bytes"] == got.size * 8
    with pytest.raises(capi.FiloError):
        ctx.scan_series(nch, addrs, capi.FN_RATE, t0 + 10, 15000, t0, 300000)          # start > end
    empty = ctx.scan_series(np.zeros(0, np.int32), np.zeros(0, np.uint64), capi.FN_RATE, t0, 15000, t0 + 60000, 300000)
    assert empty.shape == (0, 5)


def test_scan_series_zero_copy_gather(gpu, oracle):
    """With the chunk memory registered (filo_host_register) the GPU gathers the vectors itself: same bits, same counters, and
    the arena it builds is byte-identical to the staged one (filo_load_series)."""
    capi, ctx = gpu; o = oracle
    t0 = 1_700_000_000_000
    S = 700
    tab = ctx.synth_table(S, 480, 400, t0, 15000, value_kind=1, value_enc=1, reset_period=200, nan_per_million=20000, schema_flags=1, seed=7)
    arena, rec_off = tab.read_arena(0, S)
    import bench
    nch, addrs, keep = bench.host_chunk_infos(arena, rec_off, S)
    start, step, end, window = t0, 15000, t0 + 7200000, 300000
    staged = ctx.scan_series(nch, addrs, capi.FN_RATE, start, step, end, window, schema_flags=capi.SCHEMA_CUMULATIVE)
    st_staged = dict(ctx.last_stats)
    ctx.host_register(arena)
    try:
        for name in ("FN_RATE", "FN_SUM_OVER_TIME", "FN_LAST"):
            got = ctx.scan_series(nch, addrs, getattr(capi, name), start, step, end, window, schema_flags=capi.SCHEMA_CUMULATIVE)
            st = dict(ctx.last_stats)
            exp = ctx.query(tab, getattr(capi, name), start, step, end, window)
            assert_same(got, exp, "zero-copy scan %s" % name)
            assert st["samples_scanned"] == ctx.last_stats["samples_scanned"] and st["bytes_scanned"] == ctx.last_stats["bytes_scanned"]
        got = ctx.scan_series(nch, addrs, capi.FN_RATE, start, step, end, window, schema_flags=capi.SCHEMA_CUMULATIVE)
        assert_same(got, staged, "zero-copy vs staged")
        assert ctx.last_stats["samples_scanned"] == st_staged["samples_scanned"]
        assert ctx.last_stats["h2d_bytes"] >= st_staged["h2d_bytes"]         # the records still cross PCIe (device-side reads) + the gather lists
    finally:
        ctx.host_unregister(arena)
    tab.free()


@pytest.mark.parametrize("slots", [2, 3, 6])
def test_scan_series_many_plan_chunks_and_batches(gpu, oracle, slots, monkeypatch):
    """The pipeline of filo_scan_series with small bounds: several plan chunks (1,024 series each), several batches per chunk (1 MB of
    records), 2 / 3 / 6 slots in flight -- staged and zero-copy -- returns what the resident table returns, with the same counters; an
    error in a later plan chunk surfaces after the batches in flight have drained."""
    capi, ctx = gpu
    monkeypatch.setenv("FILO_SCAN_PLAN_CHUNK", "1024"); monkeypatch.setenv("FILO_SCAN_SLAB_MB", "1"); monkeypatch.setenv("FILO_SCAN_SLOTS", str(slots))
    t0, S = 1_700_000_000_000, 3500
    tab = ctx.synth_table(S, 480, 400, t0, 15000, value_kind=1, value_enc=1, reset_period=173, nan_per_million=5000, schema_flags=1, seed=11)
    arena, rec_off = tab.read_arena(0, S)
    import bench
    nch, addrs, keep = bench.host_chunk_infos(arena, rec_off, S)
    q = (t0 + 60000, 15000, t0 + 7200000, 300000)
    exp = {name: ctx.query(tab, getattr(capi, name), *q) for name in ("FN_RATE", "FN_SUM_OVER_TIME")}
    want = dict(ctx.last_stats)
    for registered in (False, True):
        if registered: ctx.host_register(arena)
        try:
            for name in exp:
                got = ctx.scan_series(nch, addrs, getattr(capi, name), *q, schema_flags=capi.SCHEMA_CUMULATIVE)
                assert_same(got, exp[name], "scan_series slots=%d registered=%s %s" % (slots, registered, name))
                assert ctx.last_stats["samples_scanned"] == want["samples_scanned"] and ctx.last_stats["bytes_scanned"] == want["bytes_scanned"]
                assert ctx.last_stats["d2h_bytes"] == got.size * 8
            bad = nch.copy(); bad[2500] = -1                                  # third plan chunk
            with pytest.raises(capi.FiloError) as e:
                ctx.scan_series(bad, addrs, capi.FN_RATE, *q, schema_flags=capi.SCHEMA_CUMULATIVE)
            assert e.value.code == capi.ERR_INVALID_ARG
            got = ctx.scan_series(nch, addrs, capi.FN_RATE, *q, schema_flags=capi.SCHEMA_CUMULATIVE)     # the context is usable afterwards
            assert_same(got, exp["FN_RATE"], "scan_series after an error")
        finally:
            if registered: ctx.host_unregister(arena)
    tab.free()


@pytest.mark.parametrize("long_sum", [False, True])
def test_avg_with_sum_and_count_over_downsampled_columns(gpu, oracle, long_sum):
    """AvgWithSumAndCountOverTimeFuncD / FuncL (AggrOverTimeFunctions.scala:820-893): avg_over_time over a downsample schema = the window sum
    of the `sum` column over the window sum of the `count` column (FuncL: a Long sum column over count_over_time of the count column), both
    over the row range of the shared timestamp column.  The ChunkSetInfos here hold three vectors (timestamp, sum, count); the two value
    columns are loaded as two tables (val_col 1 and 2).  Expected: the oracle's two chunked functions, divided (the reference's apply())."""
    import ctypes
    capi, ctx = gpu; o = oracle
    rng = np.random.default_rng(77)
    t0, rows, S = 1_700_000_000_000, 200, 40
    a, b = o.Store(), o.Store()
    for s in range(S):
        a.add_series(); b.add_series()
        ts = t0 + np.arange(rows, dtype=np.int64) * 60000 + (rng.integers(-900, 901, rows) if s % 3 == 1 else 0)
        cnt = rng.integers(1, 5, rows).astype(np.float64)
        if s % 5 == 2: cnt[rng.integers(0, rows, 6)] = NaN                     # rows the count column does not have
        sums = np.round(rng.normal(50, 20, rows) * cnt, 3)
        if s % 7 == 3: sums[rng.integers(0, rows, 4)] = NaN
        for lo, hi in ((0, 90), (90, 150), (150, rows)):
            if long_sum: a.add_chunk_longs(s, ts[lo:hi], np.nan_to_num(sums[lo:hi]).astype(np.int64))
            else: a.add_chunk(s, ts[lo:hi], sums[lo:hi])
            b.add_chunk(s, ts[lo:hi], cnt[lo:hi])
    nch, addr_a = a.all_info_addrs(); _, addr_b = b.all_info_addrs()
    # three-column ChunkSetInfo blocks: the 28 header bytes and the two vector pointers of store a, then store b's value vector
    infos = np.zeros((addr_a.size, 52), np.uint8)
    for i in range(addr_a.size):
        infos[i, :44] = np.frombuffer(ctypes.string_at(int(addr_a[i]), 44), np.uint8)
        infos[i, 44:52] = np.frombuffer(ctypes.string_at(int(addr_b[i]) + 36, 8), np.uint8)
    addrs = (infos.ctypes.data + 52 * np.arange(addr_a.size)).astype(np.uint64)
    t_sum = ctx.load_series(nch, addrs, ts_col=0, val_col=1, schema_flags=capi.SCHEMA_LONG_VALUES if long_sum else 0)
    t_cnt = ctx.load_series(nch, addrs, ts_col=0, val_col=2)
    seen_finite = seen_nan = False
    try:
        for (start, step, end, window) in [(t0 + 600000, 60000, t0 + (rows - 1) * 60000, 300000), (t0 - 3000000, 171000, t0 + (rows + 5) * 60000, 1234567)]:
            num = a.query(o.FN_SUM_OVER_TIME, start, step, end, window, long_column=long_sum)
            den = b.query(o.FN_COUNT_OVER_TIME if long_sum else o.FN_SUM_OVER_TIME, start, step, end, window)
            with np.errstate(all="ignore"):
                exp = num / den
            got = ctx.query_avg_sum_count(t_sum, t_cnt, start, step, end, window)
            assert_same(got, exp, "avg over sum/count columns long_sum=%s q=%s" % (long_sum, (start, step, end, window)))
            seen_finite |= bool(np.isfinite(got).any()); seen_nan |= bool(np.isnan(got).any())
        assert seen_finite and seen_nan                                        # windows without samples (NaN / NaN) are part of the data
        # the operator mirror: PeriodicSamplesMapper(functionId = AvgWithSumAndCountOverTime) over the three-column range vectors
        from filodb_b200 import exec as X
        ex = X.FusedGpuExec.__new__(X.FusedGpuExec); ex.ctx = ctx
        src, pos = [], 0
        for n_ in nch:
            src.append(X.RawDataRangeVector([int(x) for x in addrs[pos:pos + int(n_)]])); pos += int(n_)
        psm = X.PeriodicSamplesMapper(start, step, end, window, X.FN_AVG_WITH_SUM_AND_COUNT_OVER_TIME)
        res = ex.execute(src, psm, valueColumn=1, longValues=long_sum)
        assert_same(np.asarray(res.values), exp, "operator mirror AvgWithSumAndCountOverTime")
        with pytest.raises(capi.FiloError):
            ctx.query_avg_sum_count(t_sum, ctx.load_series(nch[:3], addrs[:int(nch[:3].sum())], val_col=2), t0, 60000, t0 + 600000, 300000)
    finally:
        t_sum.free(); t_cnt.free()


# ---------------------------------------------------------------------------------------------------------------------
# histogram columns (SURVEY §8 A8 / A16 / A18 HistSum / A19)
# ---------------------------------------------------------------------------------------------------------------------
def _hist_series(rng, rows, nb, resets=()):
    inc = np.cumsum(rng.integers(0, 20, (rows, nb)), axis=1)
    out = np.cumsum(inc, axis=0).astype(np.int64)
    for r in resets:
        out[r:] = np.cumsum(inc[r:], axis=0)
    return out


@pytest.mark.parametrize("kernel", ["v2", "v1"])
@pytest.mark.parametrize("scheme", ["custom", "geometric", "otel"])
def test_hist_rate_sum_quantile(gpu, oracle, scheme, kernel, monkeypatch):
    """hist rate / increase (SectDelta, counter correction inside and across chunks), fused sum by group, histogram_quantile.
    kernel: the fused sum runs on hist_scan2_kernel by default; FILO_HIST_V2=0 keeps it on the first kernel."""
    monkeypatch.setenv("FILO_HIST_V2", "1" if kernel == "v2" else "0")
    capi, ctx = gpu; o = oracle
    from oracle import hist as H
    rng = np.random.default_rng(21)
    t0, rows = 1_700_000_000_000, 240
    if scheme == "custom":
        b = H.Buckets.custom([2.0 * 3 ** i for i in range(19)] + [float("inf")])      # TestTimeseriesProducer.scala:229-235
    elif scheme == "otel":
        # Base2ExpHistogramBuckets in SectDelta vectors (format code 0x09): what a `counter = true` histogram column holds for otel
        # exponential histograms (TimeSeriesStore.scala:278-285); scale 3, buckets 0 | 2^(-4/8) .. 2^(10/8)
        b = H.Buckets.exponential(3, -5, 15)
    else:
        b = H.Buckets.geometric(2.0, 2.0, 12)
    st = H.HistStore(b)
    S = 37
    for s in range(S):
        jit = rng.integers(-200, 201, rows) if s % 5 == 1 else 0                     # some irregular scrapes (DDV timestamps)
        ts = t0 + np.arange(rows, dtype=np.int64) * 15000 + jit
        resets = () if s % 3 else (int(rng.integers(20, 100)), int(rng.integers(130, 230)))
        chunks = [100, 100, 40] if s % 2 else [160, 80]
        st.add_series(ts, _hist_series(rng, rows, b.n, resets), chunks)
    nch, addrs = st.all_info_addrs()
    gids = np.arange(S, dtype=np.int32) % 4
    tab = ctx.load_series(nch, addrs, group_ids=gids, n_groups=4, schema_flags=capi.SCHEMA_CUMULATIVE)
    assert tab.info().hist_buckets == b.n
    queries = [(t0 + 300000, 15000, t0 + (rows - 1) * 15000, 300000), (t0 - 60000, 47000, t0 + rows * 15000 + 90000, 333333),
               (t0 + 2000000, 1, t0 + 2000000, 600000)]
    nonmono_cells = 0
    for (start, step, end, window) in queries:
        for name in ("FN_RATE", "FN_INCREASE"):
            exp, empty = st.query(getattr(o, name), start, step, end, window)
            got = ctx.query_hist(tab, getattr(capi, name), start, step, end, window)
            exp = exp.copy(); exp[empty] = NaN
            assert_same(got, exp, "hist %s per series q=%s" % (name, (start, step, end, window)))
            aexp, aempty, qexp = st.query(getattr(o, name), start, step, end, window, aggr=True, group_ids=gids, n_groups=4, q=0.99)
            agot, qgot = ctx.query_hist(tab, getattr(capi, name), start, step, end, window, aggr=capi.AGG_SUM, quantile=0.99)
            assert (np.isnan(agot[:, :, 0]) == aempty).all()
            # HistSumRowAggregator.reduceAggregate copies the first histogram and runs MutableHistogram.add (sum + makeMonotonic) for every
            # further one (HistSumRowAggregator.scala:25-36, Histogram.scala:428-449); the device does the same inside a work item and
            # across the items of a group, in series order -- here every series is its own item, so the fold is the oracle's, cell by cell
            # (also where member histograms are not monotonic over their buckets: extrapolation around a counter reset)
            live = ~aempty
            np.testing.assert_allclose(agot[live], aexp[live], rtol=1e-9, atol=0)
            assert (np.isnan(qgot) == np.isnan(qexp)).all()
            np.testing.assert_allclose(qgot[live], qexp[live], rtol=1e-9, atol=0)
            mono = np.ones((4, exp.shape[1]), bool)
            for sidx in range(S):
                d = np.diff(np.nan_to_num(exp[sidx], nan=0.0), axis=1)
                mono[gids[sidx]] &= (d >= 0).all(axis=1) | empty[sidx]
            nonmono_cells += int((live & ~mono).sum())
    assert nonmono_cells > 0          # the case the per-add correction exists for is part of the data
    # scalar entry points decline histogram tables and vice versa
    with pytest.raises(capi.FiloError):
        ctx.query(tab, capi.FN_RATE, *queries[0])
    with pytest.raises(capi.FiloError):
        ctx.query_hist(tab, capi.FN_MIN_OVER_TIME, *queries[0])
    tab.free()


def test_row_wise_exp_histogram_vectors_are_declined(gpu, oracle):
    """ExpHistogramVector (wire 0x1309: a BinaryHistogram blob with its own scheme per row, ExpHistogramVector.scala:19-35) is not on the
    device path: the load answers FILO_ERR_UNSUPPORTED and the caller keeps the JVM path (the reference has no counter reader for it and
    its rate over differing schemes is unimplemented, RateFunctions.scala:387-399)."""
    capi, ctx = gpu; o = oracle
    from oracle import hist as H
    app = H.Appender(2, 1024)                                                   # sect == 2: AppendableExpHistogramVector
    for sch, vals in (((3, -3, 1), [0, 3]), ((20, -3, 9), [0, 4, 5, 6, 7, 8, 9, 10, 11, 12])):
        assert app.add(H.Buckets.exponential(*sch).write_delta(vals)) == H.ACK
    hv = app.bytes()
    st = o.Store(); st.add_series()
    tsv = o.Store(); tsv.add_series(); tsv.add_chunk(0, np.array([1000, 2000], np.int64), np.zeros(2))
    st.add_chunk_raw(0, 1000, 2000, 2, tsv.vector_bytes(0, 0, 0), hv)
    with pytest.raises(capi.FiloError) as e:
        ctx.load_series(*st.all_info_addrs())
    assert e.value.code == capi.ERR_UNSUPPORTED


def test_hist_sum_over_time_and_delta_schema(gpu, oracle):
    """SumOverTimeChunkedFunctionH over SectDelta vectors, and delta-temporality histograms in simple (row) vectors."""
    capi, ctx = gpu; o = oracle
    from oracle import hist as H
    rng = np.random.default_rng(22)
    t0, rows = 1_700_000_000_000, 240
    b = H.Buckets.geometric(2.0, 2.0, 12)
    st = H.HistStore(b)
    S = 9
    for s in range(S):
        ts = t0 + np.arange(rows, dtype=np.int64) * 15000
        st.add_series(ts, _hist_series(rng, rows, b.n, () if s % 3 else (77,)), [160, 80])
    nch, addrs = st.all_info_addrs()
    tab = ctx.load_series(nch, addrs, schema_flags=capi.SCHEMA_CUMULATIVE)
    queries = [(t0 + 300000, 15000, t0 + (rows - 1) * 15000, 300000), (t0 - 60000, 47000, t0 + rows * 15000 + 90000, 333333)]
    # sum_over_time over the same (cumulative) vectors: SumOverTimeChunkedFunctionH
    for (start, step, end, window) in queries[:2]:
        exp, empty = st.query(o.FN_SUM_OVER_TIME, start, step, end, window)
        got = ctx.query_hist(tab, capi.FN_SUM_OVER_TIME, start, step, end, window)
        exp = exp.copy(); exp[empty] = NaN
        assert_same(got, exp, "hist sum_over_time q=%s" % ((start, step, end, window),))
    tab.free()
    # delta-temporality histograms in simple (row) vectors: rate = sum / window * 1000, increase = sum (RateFunctions.scala:470-494)
    st2 = H.HistStore(b)
    for s in range(11):
        ts = t0 + np.arange(rows, dtype=np.int64) * 15000
        obs = np.cumsum(rng.integers(0, 9, (rows, b.n)), axis=1).astype(np.int64)       # per-row (delta) histograms, cumulative over buckets
        st2.add_series(ts, obs, [100, 100, 40], sect=False)
    nch2, addrs2 = st2.all_info_addrs()
    tab2 = ctx.load_series(nch2, addrs2, schema_flags=0)
    for (start, step, end, window) in queries[:2]:
        for name in ("FN_RATE", "FN_INCREASE", "FN_SUM_OVER_TIME"):
            exp, empty = st2.query(getattr(o, name), start, step, end, window, cumulative=False)
            got = ctx.query_hist(tab2, getattr(capi, name), start, step, end, window)
            exp = exp.copy(); exp[empty] = NaN
            assert_same(got, exp, "delta hist %s q=%s" % (name, (start, step, end, window)))
        aexp, aempty, qexp = st2.query(o.FN_RATE, start, step, end, window, cumulative=False, aggr=True, group_ids=np.zeros(11, np.int32), n_groups=1, q=0.5)
        agot, qgot = ctx.query_hist(tab2, capi.FN_RATE, start, step, end, window, aggr=capi.AGG_SUM, quantile=0.5)
        m = ~aempty
        np.testing.assert_allclose(agot[m], aexp[m], rtol=1e-9, atol=0)
        np.testing.assert_allclose(qgot[~np.isnan(qexp)], qexp[~np.isnan(qexp)], rtol=1e-9, atol=0)
    tab2.free()


# ------------------------------------------------------------------------------------------------------------------
# the remaining chunked range functions, Long value columns, masked vectors
# ------------------------------------------------------------------------------------------------------------------
EXT_FNS = [("FN_STDDEV_OVER_TIME", ()), ("FN_STDVAR_OVER_TIME", ()), ("FN_ZSCORE", ()), ("FN_CHANGES", ()), ("FN_QUANTILE_OVER_TIME", (0.73,)),
           ("FN_QUANTILE_OVER_TIME", (0.0,)), ("FN_QUANTILE_OVER_TIME", (1.0,)), ("FN_QUANTILE_OVER_TIME", (-0.1,)), ("FN_QUANTILE_OVER_TIME", (1.5,)),
           ("FN_MAD_OVER_TIME", ()), ("FN_HOLT_WINTERS", (0.3, 0.1)), ("FN_PREDICT_LINEAR", (600.0,)), ("FN_PRESENT_OVER_TIME", ())]
EXT_CASES = [("gauge", 1, 0, False, 0.05), ("gauge", 2, 3000, False, 0.02), ("intcounter", 0, 0, False, 0.0), ("linear", 0, 200, False, 0.0)]


@pytest.mark.parametrize("case", EXT_CASES, ids=[("%s-v%d-j%d-%s-nan%g" % c) for c in EXT_CASES])
def test_extended_range_functions(gpu, oracle, case):
    """stddev / stdvar / zscore / changes / quantile / mad / holt_winters / predict_linear / present_over_time
    (AggrOverTimeFunctions.scala:1082-1604, RangeFunction.scala:725-748): bit-exact per series against the oracle."""
    capi, ctx = gpu; o = oracle
    kind, val_mode, jitter, cumulative, nan_frac = case
    rng = np.random.default_rng(zlib.crc32(repr(case).encode()))
    st = build_store(o, rng, 12, kind, val_mode, jitter, cumulative, nan_frac, rows=300, chunks=(140, 100, 60))
    nch, addrs = st.all_info_addrs()
    tab = ctx.load_series(nch, addrs)
    t0 = 1_700_000_000_000
    queries = [(t0 + 300000, 15000, t0 + 299 * 15000, 300000), (t0 - 50000, 47000, t0 + 320 * 15000, 111111)]
    try:
        for (start, step, end, window) in queries:
            for name, args in EXT_FNS:
                ctx.set_fn_args(*args)
                got = ctx.query(tab, getattr(capi, name), start, step, end, window)
                exp = st.query(getattr(o, name), start, step, end, window, params=args)
                assert_same(got, exp, "%s %s%s q=%s" % (case, name, args, (start, step, end, window)))
                assert ctx.last_stats["samples_scanned"] == st.last_stats["samples_scanned"]
        ctx.set_fn_args(1.5, 0.1)
        with pytest.raises(capi.FiloError) as ei:
            ctx.query(tab, capi.FN_HOLT_WINTERS, *queries[0])
        assert ei.value.code == capi.ERR_INVALID_ARG
    finally:
        ctx.set_fn_args(0.0, 0.0)
        tab.free()


LONG_FNS = [("FN_LAST", ()), ("FN_COUNT_OVER_TIME", ()), ("FN_SUM_OVER_TIME", ()), ("FN_AVG_OVER_TIME", ()), ("FN_MIN_OVER_TIME", ()), ("FN_MAX_OVER_TIME", ()),
            ("FN_STDDEV_OVER_TIME", ()), ("FN_STDVAR_OVER_TIME", ()), ("FN_CHANGES", ()), ("FN_QUANTILE_OVER_TIME", (0.4,)), ("FN_PREDICT_LINEAR", (120.0,)),
            ("FN_MAD_OVER_TIME", ())]


@pytest.mark.parametrize("shape", ["ddv", "const", "flat", "raw"])
def test_long_column_functions(gpu, oracle, shape):
    """Long value columns: LongBinaryVector readers (DDV, const DDV, raw 64-bit) and the *L chunked functions
    (AggrOverTimeFunctions.scala:60-116,574-585,924-938,1019-1028,1144-1183,1211-1225,1322-1359), bit-exact."""
    capi, ctx = gpu; o = oracle
    rng = np.random.default_rng({"ddv": 1, "const": 2, "flat": 3, "raw": 4}[shape])
    t0 = 1_700_000_000_000; rows = 260
    st = o.Store()
    for s in range(10):
        ts = t0 + np.arange(rows, dtype=np.int64) * 15000 + (rng.integers(-2000, 2001, rows) if s % 2 else 0)
        if shape == "ddv": v = (np.cumsum(rng.integers(0, 50, rows)) + 1000 * s).astype(np.int64)
        elif shape == "const": v = (7 * s + (3 + s) * np.arange(rows)).astype(np.int64)
        elif shape == "flat": v = np.full(rows, 42 + s, np.int64)
        else: v = rng.integers(-2 ** 62, 2 ** 62, rows).astype(np.int64)
        si = st.add_series()
        for a, b in ((0, 120), (120, 200), (200, rows)):
            st.add_chunk_longs(si, ts[a:b], v[a:b], raw=(shape == "raw"))
    nch, addrs = st.all_info_addrs()
    tab = ctx.load_series(nch, addrs, schema_flags=capi.SCHEMA_LONG_VALUES)
    try:
        for (start, step, end, window) in [(t0 + 300000, 15000, t0 + (rows - 1) * 15000, 300000), (t0 - 50000, 47000, t0 + (rows + 20) * 15000, 111111)]:
            for name, args in LONG_FNS:
                ctx.set_fn_args(*args)
                got = ctx.query(tab, getattr(capi, name), start, step, end, window)
                exp = st.query(getattr(o, name), start, step, end, window, long_column=True, params=args)
                assert_same(got, exp, "long %s %s%s q=%s" % (shape, name, args, (start, step, end, window)))
        with pytest.raises(capi.FiloError) as ei:      # no chunked L variant: the caller keeps the iterating JVM path
            ctx.query(tab, capi.FN_RATE, t0, 15000, t0 + 600000, 300000)
        assert ei.value.code == capi.ERR_UNSUPPORTED
    finally:
        ctx.set_fn_args(0.0, 0.0)
        tab.free()


def _masked(inner, n, na_rows=()):
    """BitmapMaskAppendableVector layout (BinaryVector.scala:614-660): +0 numBytes, +4 wire BINSIMPLE/PRIMITIVE, +8 offset of the
    subvector (12 + bitmap bytes), +12 NA bitmap in 64-bit words, then the subvector."""
    inner = np.ascontiguousarray(inner, np.uint8)
    bm = np.zeros((n + 63) // 64, np.uint64)
    for r in na_rows: bm[r >> 6] |= np.uint64(1) << np.uint64(r & 63)
    hdr = np.zeros(12, np.uint8)
    hdr[0:4] = np.frombuffer(np.int32(8 + bm.nbytes + inner.size).tobytes(), np.uint8)
    hdr[4] = 0x06; hdr[5] = 0x00
    hdr[8:12] = np.frombuffer(np.int32(12 + bm.nbytes).tobytes(), np.uint8)
    return np.concatenate([hdr, bm.view(np.uint8), inner])


def test_masked_vectors(gpu, oracle):
    """Masked (NA-bitmap) vectors: MaskedDoubleDataReader / MaskedLongDataReader delegate to the subvector (DoubleVector.scala:397-417,
    LongBinaryVector.scala:270-293, BinaryVector.scala:193-227); the counter drop bit lives on the outer vector."""
    capi, ctx = gpu; o = oracle
    rng = np.random.default_rng(77)
    t0 = 1_700_000_000_000; rows = 200
    st = o.Store()
    for s in range(8):
        ts = t0 + np.arange(rows, dtype=np.int64) * 15000 + (rng.integers(-1500, 1501, rows) if s % 2 else 0)
        v = np.cumsum(np.maximum(0, 15 + rng.normal(0, 3, rows)))
        if s % 3 == 0:
            v[120:] = v[120:] - v[120] + 1.0                       # a counter reset inside the second chunk
        v[rng.random(rows) < 0.03] = NaN
        si = st.add_series()
        for a, b in ((0, 110), (110, rows)):
            tsv = o.encode_timestamps(ts[a:b]) if s % 4 else _masked(o.encode_timestamps(ts[a:b]), b - a)
            inner = o.encode_doubles(v[a:b], detect_drops=True, mode=o.VAL_RAW)
            drop = bool(o.Vec(inner).dropped())
            inner = np.array(inner, np.uint8); inner[7] &= 0x7f        # the appender marks the drop on the OUTER vector
            mv = _masked(inner, b - a, na_rows=[int(i) for i in np.nonzero(np.isnan(v[a:b]))[0]])
            if drop: mv[7] |= 0x80
            st.add_chunk_raw(si, int(ts[a]), int(ts[b - 1]), b - a, tsv, mv)
    nch, addrs = st.all_info_addrs()
    tab = ctx.load_series(nch, addrs, schema_flags=capi.SCHEMA_CUMULATIVE)
    try:
        for (start, step, end, window) in [(t0 + 300000, 15000, t0 + (rows - 1) * 15000, 300000), (t0 - 50000, 47000, t0 + (rows + 20) * 15000, 111111)]:
            for name in ALL_FNS:
                got = ctx.query(tab, getattr(capi, name), start, step, end, window)
                exp = st.query(getattr(o, name), start, step, end, window, cumulative=True)
                assert_same(got, exp, "masked %s q=%s" % (name, (start, step, end, window)))
                assert ctx.last_stats["samples_scanned"] == st.last_stats["samples_scanned"]
    finally:
        tab.free()


def test_host_mirror_and_jni_shim_on_gpu(tmp_path):
    """The C++ operator mirror (include/filo_b200.hpp: FusedGpuExec::execute over PeriodicSamplesMapper [+ AggregateMapReduce]) and the
    JNI shim (filodb_b200/csrc/jni_shim.cpp, driven through a host JNIEnv) on the GPU against the oracle: tests/cpp/host_mirror_gpu.cpp."""
    import os, subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.join(root, "filodb_b200")
    assert os.path.exists(os.path.join(libdir, "libfilo_b200_jni.so")), "build the JNI shim first (filodb_b200/build.py)"
    exe = str(tmp_path / "host_mirror_gpu")
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", os.path.join(root, "tests", "cpp", "host_mirror_gpu.cpp"), "-o", exe,
                    "-L", libdir, "-lfilo_b200_jni", "-lfilo_b200", "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "OK host mirror + JNI shim" in r.stdout, r.stdout + r.stderr


def test_python_operator_mirror(oracle):
    """filodb_b200/exec.py: the reference's transformer chain as objects (PeriodicSamplesMapper [+ AggregateMapReduce]) -> one device call."""
    import filodb_b200.capi as capi
    from filodb_b200 import exec as fx
    o = oracle
    rng = np.random.default_rng(5)
    st = build_store(o, rng, 20, "gauge", 1, 0, False, 0.02)
    t0 = 1_700_000_000_000
    src = [fx.RawDataRangeVector([int(a) for a in st.info_addrs(s)], s % 3) for s in range(20)]
    ex = fx.FusedGpuExec(0)
    try:
        psm = fx.PeriodicSamplesMapper(t0 + 300000, 15000, t0 + 479 * 15000, 300000, capi.FN_QUANTILE_OVER_TIME, funcParams=(0.9,))
        r = ex.execute(src, psm)
        assert_same(r.values, st.query(o.FN_QUANTILE_OVER_TIME, t0 + 300000, 15000, t0 + 479 * 15000, 300000, params=(0.9,)), "mirror quantile_over_time")
        psm = fx.PeriodicSamplesMapper(t0 + 300000, 15000, t0 + 479 * 15000, 300000, capi.FN_SUM_OVER_TIME)
        r = ex.execute(src, psm, fx.AggregateMapReduce(capi.AGG_MAX, (), 3))
        exp = st.query(o.FN_SUM_OVER_TIME, t0 + 300000, 15000, t0 + 479 * 15000, 300000, aggr=o.AGG_MAX, group_ids=np.arange(20) % 3, n_groups=3)
        assert_same(r.values, exp, "mirror max(sum_over_time)")
        with pytest.raises(ValueError):
            fx.PeriodicSamplesMapper(t0, 15000, t0 + 1000, None, capi.FN_RATE)
        with pytest.raises(ValueError):
            fx.PeriodicSamplesMapper(t0 + 10, 15000, t0, 1000, capi.FN_RATE)
    finally:
        ex.close()


def test_result_wire_format(oracle):
    """filo_encode_result: the result rows as BinaryRecord v2 records in RecordContainers, byte for byte what SerializedRangeVector.apply
    writes through one shared RecordBuilder (RangeVector.scala:427-476,511-586; RecordBuilder.scala:109-175,461-480,589-621)."""
    import filodb_b200.capi as capi
    o = oracle
    ctx = capi.Context(0)
    try:
        rng = np.random.default_rng(31)
        for (n, T, nan_frac) in ((1, 11, 0.6), (201, 11, 0.6), (37, 481, 0.02), (5, 481, 1.0), (64, 204, 0.0), (3, 1, 0.5)):
            v = rng.normal(0, 1e3, (n, T))
            v[rng.random((n, T)) < nan_frac] = NaN
            start, step = 1_700_000_000_000, 15000
            end = start + (T - 1) * step
            c, rs, sr, fc = ctx.encode_result(v, start, step, end, container_ts_ms=1234567)
            ce, rse, sre, fce = o.serialize_result(v, start, step, end, now_ms=1234567)
            assert (rs == rse).all() and (sr == sre).all() and (fc == fce).all(), (n, T)
            assert c.shape == ce.shape and (c == ce).all(), (n, T)
            for i in (0, n // 2, n - 1):
                ts, vals = o.result_rows(c, rs[i], sr[i], fc[i], start, step, end)
                assert len(ts) == T and same_bits(vals, v[i])
        # instant query: NaN rows stay (canRemoveEmptyRows is false for start == end)
        c, rs, sr, fc = ctx.encode_result(np.array([[NaN], [2.0]]), 5000, 0, 5000)
        ce, rse, _, _ = o.serialize_result(np.array([[NaN], [2.0]]), 5000, 1, 5000)
        assert list(rs) == [1, 1] and (c == ce).all()
        # a query result straight into the wire format
        st = build_store(o, rng, 9, "gauge", 1, 0, False, 0.05)
        t0 = 1_700_000_000_000
        tab = ctx.load_series(*st.all_info_addrs())
        q = (t0 - 100000, 15000, t0 + 480 * 15000, 60000)          # windows before the data: NaN rows that are not encoded
        got = ctx.query(tab, capi.FN_SUM_OVER_TIME, *q)
        c, rs, sr, fc = ctx.encode_result(got, q[0], q[1], q[2])
        exp = st.query(o.FN_SUM_OVER_TIME, *q)
        assert (rs == (~np.isnan(exp)).sum(axis=1)).all() and rs.sum() < exp.size
        for i in range(9):
            ts, vals = o.result_rows(c, rs[i], sr[i], fc[i], q[0], q[1], q[2])
            assert same_bits(vals, exp[i])
        tab.free()
    finally:
        ctx.close()


def test_incremental_arena_append(gpu, oracle):
    """filo_table_append: chunks arrive flush by flush (TimeSeriesPartition.switchBuffers, TimeSeriesPartition.scala:251-288); the re-packed
    arena is byte-identical to filo_load_series over all the chunks and queries agree with the oracle at every stage."""
    capi, ctx = gpu; o = oracle
    rng = np.random.default_rng(41)
    S, t0 = 33, 1_700_000_000_000
    st = build_store(o, rng, S, "counter", 1, 0, True, 0.01, rows=420, chunks=(150, 150, 120))
    for s in range(S):                                   # irregular timestamps and raw vectors in some series
        pass
    per = [st.info_addrs(s) for s in range(S)]
    gids = np.arange(S, dtype=np.int32) % 5
    # stage 1: first chunk of every series; stage 2: second chunk of two thirds of them; stage 3: the rest
    tab = ctx.load_series(np.ones(S, np.int32), np.array([p[0] for p in per], np.uint64), group_ids=gids, n_groups=5, schema_flags=capi.SCHEMA_CUMULATIVE)
    have = np.ones(S, np.int32)
    q = (t0 + 300000, 15000, t0 + 419 * 15000, 300000)

    def check(stage):
        sub = o.Store()
        for s in range(S):
            si = sub.add_series()
            for c in range(have[s]):
                ch_ts = st.vector_bytes(s, c, 0); ch_v = st.vector_bytes(s, c, 1)
                rows_c = (150, 150, 120)[c]; r0 = (0, 150, 300)[c]
                sub.add_chunk_raw(si, t0 + r0 * 15000, t0 + (r0 + rows_c - 1) * 15000, rows_c, ch_ts, ch_v)
        for name in ("FN_RATE", "FN_SUM_OVER_TIME", "FN_LAST"):
            assert_same(ctx.query(tab, getattr(capi, name), *q), sub.query(getattr(o, name), *q, cumulative=True), "append stage %d %s" % (stage, name))
        got = ctx.query(tab, capi.FN_RATE, *q, aggr=capi.AGG_SUM)
        exp = sub.query(o.FN_RATE, *q, cumulative=True, aggr=o.AGG_SUM, group_ids=gids, n_groups=5)
        np.testing.assert_allclose(got, exp, rtol=1e-9, equal_nan=True)
        # byte equality with a fresh load of the same chunks
        nch = have.copy(); addrs = np.array([a for s in range(S) for a in per[s][:have[s]]], np.uint64)
        ref = ctx.load_series(nch, addrs, schema_flags=capi.SCHEMA_CUMULATIVE)
        a1, o1 = tab.read_arena(0, S); a2, o2 = ref.read_arena(0, S)
        assert (o1 == o2).all() and a1.size == a2.size and (a1 == a2).all(), "arena bytes differ at stage %d" % stage
        i1, i2 = tab.info(), ref.info()
        assert (i1.n_chunks, i1.n_samples, i1.algorithmic_bytes, i1.max_rows_per_series, i1.max_chunks_per_series) == \
               (i2.n_chunks, i2.n_samples, i2.algorithmic_bytes, i2.max_rows_per_series, i2.max_chunks_per_series)
        ref.free()

    check(1)
    add = np.array([1 if s % 3 else 0 for s in range(S)], np.int32)
    tab.append(add, np.array([per[s][1] for s in range(S) if add[s]], np.uint64)); have += add
    check(2)
    add = np.array([3 - have[s] for s in range(S)], np.int32)
    tab.append(add, np.array([a for s in range(S) for a in per[s][have[s]:3]], np.uint64)); have += add
    check(3)
    # a chunk older than the resident ones is refused and leaves the table as it was
    with pytest.raises(capi.FiloError) as e:
        one = np.zeros(S, np.int32); one[0] = 1
        tab.append(one, np.array([per[0][0]], np.uint64))
    assert e.value.code == capi.ERR_UNSUPPORTED
    check(4)
    tab.free()


@pytest.mark.parametrize("value_enc", [0, 1, 2])
def test_encode_ingest_batch_on_gpu(gpu, oracle, value_enc):
    """filo_encode_table: raw samples encoded on the device into the appenders' bytes (DeltaDeltaVector.fromLongVector incl. the +-250 ms
    rule, DoubleVector.optimize / raw / XOR container, counter drop flag), byte for byte the oracle's encoders; queries agree."""
    capi, ctx = gpu; o = oracle
    rng = np.random.default_rng(50 + value_enc)
    S, rows, rpc, t0 = 21, 230, 100, 1_700_000_000_000
    ts = np.zeros((S, rows), np.int64); vals = np.zeros((S, rows), np.float64)
    for s in range(S):
        jit = (0, 100, 3000)[s % 3]
        ts[s] = t0 + np.arange(rows) * 15000 + (rng.integers(-jit, jit + 1, rows) if jit else 0)
        if s % 2: v = np.cumsum(rng.integers(0, 30, rows)).astype(float)              # integral counters (DDV longs under optimize)
        else: v = np.cumsum(np.maximum(0, 15 + rng.normal(0, 2, rows)))
        for r in np.nonzero(rng.random(rows) < 0.01)[0]:
            if r > 0: v[r:] = v[r:] - v[r] + 1.0                                       # counter resets
        if s % 5 == 0: v[rng.random(rows) < 0.02] = NaN
        vals[s] = v
    gids = np.arange(S, dtype=np.int32) % 4
    tab = ctx.encode_table(ts, vals, rows_per_chunk=rpc, value_enc=value_enc, schema_flags=capi.SCHEMA_CUMULATIVE, group_ids=gids, n_groups=4)
    val_mode = {0: o.VAL_RAW, 1: o.VAL_XOR, 2: o.VAL_OPTIMIZE}[value_enc]
    st = o.Store()
    chunk_rows = [100, 100, 30]
    for s in range(S):
        st.add_series_rows(ts[s], vals[s], chunk_rows, val_mode=val_mode, detect_drops=True)
    ref = ctx.load_series(*st.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE)
    a1, o1 = tab.read_arena(0, S); a2, o2 = ref.read_arena(0, S)
    assert (o1 == o2).all() and (a1 == a2).all(), "device-encoded arena differs from the appenders' bytes"
    assert tab.info().algorithmic_bytes == st.algorithmic_bytes()
    q = (t0 + 300000, 15000, t0 + (rows - 1) * 15000, 300000)
    for name in ("FN_RATE", "FN_SUM_OVER_TIME", "FN_LAST"):
        assert_same(ctx.query(tab, getattr(capi, name), *q), st.query(getattr(o, name), *q, cumulative=True), "encoded table %s" % name)
    got = ctx.query(tab, capi.FN_RATE, *q, aggr=capi.AGG_SUM)
    np.testing.assert_allclose(got, st.query(o.FN_RATE, *q, cumulative=True, aggr=o.AGG_SUM, group_ids=gids, n_groups=4), rtol=1e-9, equal_nan=True)
    with pytest.raises(capi.FiloError):
        bad = ts.copy(); bad[0, 5] = bad[0, 4]
        ctx.encode_table(bad, vals)
    tab.free(); ref.free()


@pytest.mark.parametrize("scheme", ["geometric", "custom", "otel"])
def test_histogram_vectors_encoded_on_gpu(gpu, oracle, scheme):
    """filo_encode_hist_table / filo_synth_hist_table: SectDelta HistogramVectors written on the device are byte for byte the JVM appender's
    (AppendableSectDeltaHistVector.appendHist incl. section roll-over every 16 records and Drop sections; oracle restatement), and queries agree."""
    capi, ctx = gpu; o = oracle
    from oracle import hist as H
    from tests import synth_ref as sr
    rng = np.random.default_rng(61)
    t0, rows, rpc, nb = 1_700_000_000_000, 230, 100, (20 if scheme == "geometric" else 13)
    if scheme == "geometric":
        b = H.Buckets.geometric(2.0, 3.0, nb); bdef, fmt = capi.geometric_bucket_def(2.0, 3.0, nb)
        assert (bdef == b.serialize()).all()
    elif scheme == "otel":
        b = H.Buckets.exponential(-1, -3, nb - 1); bdef, fmt = capi.exp_bucket_def(-1, -3, nb - 1)       # base 4, tops 0 | 4^-2 .. 4^9
        assert (bdef == b.serialize()).all()
    else:
        les = [0.5 * 2 ** i for i in range(nb - 1)] + [float("inf")]
        b = H.Buckets.custom(les); bdef, fmt = capi.custom_bucket_def(les)
        assert (bdef == b.serialize()).all()
    S = 17
    ts = np.zeros((S, rows), np.int64); counts = np.zeros((S, rows, nb), np.int64)
    for s in range(S):
        ts[s] = t0 + np.arange(rows) * 15000 + (rng.integers(-300, 301, rows) if s % 4 == 1 else 0)
        counts[s] = _hist_series(rng, rows, nb, () if s % 3 else (int(rng.integers(20, 90)), int(rng.integers(120, 220))))
    gids = np.arange(S, dtype=np.int32) % 3
    tab = ctx.encode_hist_table(ts, counts, bdef, fmt, rows_per_chunk=rpc, group_ids=gids, n_groups=3)
    st = H.HistStore(b)
    for s in range(S):
        st.add_series(ts[s], counts[s], [100, 100, 30])
    ref = ctx.load_series(*st.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE)
    a1, o1 = tab.read_arena(0, S); a2, o2 = ref.read_arena(0, S)
    assert (o1 == o2).all() and (a1 == a2).all(), "device-encoded histogram vectors differ from the appender's bytes"
    assert tab.info().hist_buckets == nb and tab.info().algorithmic_bytes == ref.info().algorithmic_bytes
    q = (t0 + 300000, 15000, t0 + (rows - 1) * 15000, 300000)
    exp, empty = st.query(o.FN_RATE, *q)
    exp = exp.copy(); exp[empty] = NaN
    assert_same(ctx.query_hist(tab, capi.FN_RATE, *q), exp, "rate over device-encoded histograms")
    aexp, aempty, qexp = st.query(o.FN_RATE, *q, aggr=True, group_ids=gids, n_groups=3, q=0.9)
    agot, qgot = ctx.query_hist(tab, capi.FN_RATE, *q, aggr=capi.AGG_SUM, quantile=0.9)
    np.testing.assert_allclose(qgot[~aempty], qexp[~aempty], rtol=1e-9)
    tab.free(); ref.free()
    # the generator: same encoder over hash-generated rows
    S2, seed, base = 11, 5, 194
    gtab = ctx.synth_hist_table(S2, rows, bdef, fmt, nb, rows_per_chunk=rpc, t0_ms=t0, reset_period=97, seed=seed, series_id_base=base)
    st2 = H.HistStore(b)
    tsr = t0 + np.arange(rows, dtype=np.int64) * 15000
    for s in range(S2):
        st2.add_series(tsr, sr.gen_hist_series(seed, base + s, rows, nb, 97), [100, 100, 30])
    ref2 = ctx.load_series(*st2.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE)
    a1, o1 = gtab.read_arena(0, S2); a2, o2 = ref2.read_arena(0, S2)
    assert (o1 == o2).all() and (a1 == a2).all(), "generated histogram table differs from the appender's bytes"
    gtab.free(); ref2.free()
