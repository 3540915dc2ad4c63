"""GPU: histogram `last` (LastSampleChunkedFunctionH) and per-series histogram_quantile through filo_query_hist, on both histogram scan
kernels (FILO_HIST_V2=1: hist_scan2_kernel where it serves the shape; FILO_HIST_V2=0: hist_scan_kernel), against the CPU restatement in
tests/hist_series_ref.py and the oracle's histogram path."""
import numpy as np
import pytest

from tests import hist_series_ref as R

pytestmark = pytest.mark.gpu
NaN = float("nan")
T0 = 1_700_000_000_000
ROWS = 240


def same_bits(a, b):
    a = np.ascontiguousarray(a, np.float64); b = np.ascontiguousarray(b, np.float64)
    an, bn = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and (an == bn).all() and (a[~an].view(np.uint64) == b[~bn].view(np.uint64)).all()


def assert_same(a, b, what=""):
    assert same_bits(a, b), "%s: %s" % (what, np.argwhere(~(np.isclose(a, b, rtol=0, atol=0) | (np.isnan(a) & np.isnan(b))))[:5].tolist())


@pytest.fixture(scope="module")
def gpu():
    import filodb_b200.capi as capi
    ctx = capi.Context(0)
    yield capi, ctx
    ctx.close()


def _buckets(H, scheme):
    if scheme == "custom":
        return H.Buckets.custom([2.0 * 3 ** i for i in range(19)] + [float("inf")])
    if scheme == "otel":
        return H.Buckets.exponential(3, -5, 15)
    return H.Buckets.geometric(2.0, 2.0, 12)


def _hist_rows(rng, rows, nb, resets=()):
    inc = np.cumsum(rng.integers(0, 20, (rows, nb)), axis=1)
    out = np.cumsum(inc, axis=0).astype(np.int64)
    for r in resets:
        out[r:] = np.cumsum(inc[r:], axis=0)
    return out


def _store(H, b, S, seed, sect=True, delta=False):
    """S series of ROWS rows: some jittered timestamps, counter resets inside chunks and at chunk starts, 1-3 chunks."""
    rng = np.random.default_rng(seed)
    st = H.HistStore(b); ts_l, ch_l = [], []
    for s in range(S):
        jit = rng.integers(-200, 201, ROWS) if s % 5 == 1 else 0
        ts = T0 + np.arange(ROWS, dtype=np.int64) * 15000 + jit
        chunks = [[100, 100, 40], [160, 80], [ROWS]][s % 3]
        if delta:
            vals = np.cumsum(rng.integers(0, 9, (ROWS, b.n)), axis=1).astype(np.int64)
        else:
            resets = () if s % 3 == 2 else ((int(rng.integers(20, 90)), 160) if s % 3 == 1 else (100, int(rng.integers(110, 230))))
            vals = _hist_rows(rng, ROWS, b.n, resets)
        st.add_series(ts, vals, chunks, sect=sect)
        ts_l.append(ts); ch_l.append(chunks)
    return st, ts_l, ch_l


def check_counters(ctx, st, ts_l, ch_l, q):
    """the call's scan counters equal CountingChunkInfoIterator's (tests/hist_series_ref.py scan_counters)"""
    samples, nbytes = R.scan_counters(st, ts_l, ch_l, *q)
    assert (ctx.last_stats["samples_scanned"], ctx.last_stats["bytes_scanned"]) == (samples, nbytes), (ctx.last_stats, samples, nbytes, q)


QUERIES = [(T0 + 300000, 15000, T0 + (ROWS - 1) * 15000, 300000), (T0 - 60000, 47000, T0 + ROWS * 15000 + 90000, 333333),
           (T0 + 2000000, 1, T0 + 2000000, 600000), (T0 - 60000, 61000, T0 + ROWS * 15000 + 400000, 0)]


@pytest.mark.parametrize("v2", ["1", "0"])
@pytest.mark.parametrize("sect", [True, False], ids=["sectdelta", "simple"])
def test_hist_last_per_series_and_sum(gpu, oracle, sect, v2, monkeypatch):
    """last per series (bit-exact, raw values after Drop sections), fused sum(last) by group with the quantile, scan counters."""
    monkeypatch.setenv("FILO_HIST_V2", v2)
    capi, ctx = gpu
    from oracle import hist as H
    b = _buckets(H, "custom")
    S, G = 23, 3
    st, ts_l, ch_l = _store(H, b, S, 31, sect=sect)
    gids = (np.arange(S) % G).astype(np.int32)
    tab = ctx.load_series(*st.all_info_addrs(), group_ids=gids, n_groups=G, schema_flags=capi.SCHEMA_CUMULATIVE)
    try:
        for q in QUERIES:
            exp, empty = R.last_store(st, ts_l, ch_l, b.n, *q)
            got = ctx.query_hist(tab, capi.FN_LAST, *q)
            assert_same(got, exp, "last per series q=%s" % (q,))
            check_counters(ctx, st, ts_l, ch_l, q)
            aexp, aempty = R.hist_sum(b.n, exp, empty, gids, G)
            qexp = R.quantiles(b, aexp, aempty, 0.9)
            agot, qgot = ctx.query_hist(tab, capi.FN_LAST, *q, aggr=capi.AGG_SUM, quantile=0.9)
            check_counters(ctx, st, ts_l, ch_l, q)
            assert (np.isnan(agot[:, :, 0]) == aempty).all()
            assert_same(agot, aexp, "sum(last) q=%s" % (q,))                     # integer counts: every order of the fold is exact
            assert (np.isnan(qgot) == np.isnan(qexp)).all()
            np.testing.assert_allclose(qgot[~np.isnan(qexp)], qexp[~np.isnan(qexp)], rtol=1e-9, atol=0)
    finally:
        tab.free()


FNS = ["FN_RATE", "FN_INCREASE", "FN_SUM_OVER_TIME", "FN_LAST"]


@pytest.mark.parametrize("v2", ["1", "0"])
@pytest.mark.parametrize("scheme", ["custom", "geometric", "otel"])
def test_hist_quantile_per_series(gpu, oracle, scheme, v2, monkeypatch):
    """histogram_quantile(q, f(h[w])) without an aggregate: Histogram.quantile of each series' own window histogram; the bucket rows of the
    same call bit-exact, the quantile-only call equal to it, NaN / +-Inf exactly where the reference has them."""
    monkeypatch.setenv("FILO_HIST_V2", v2)
    capi, ctx = gpu; o = oracle
    from oracle import hist as H
    b = _buckets(H, scheme)
    S = 19
    st, ts_l, ch_l = _store(H, b, S, 32)
    tab = ctx.load_series(*st.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE)
    nonmono = 0
    try:
        for q in QUERIES[:3]:
            for name in FNS:
                if name == "FN_LAST":
                    exp, empty = R.last_store(st, ts_l, ch_l, b.n, *q)
                else:
                    exp, empty = st.query(getattr(o, name), *q); exp = exp.copy(); exp[empty] = NaN
                for qt in (0.99, 0.5, 0.0, 1.0, -0.1, 1.5):
                    qexp = R.quantiles(b, exp, empty, qt)
                    vals, qgot = ctx.query_hist(tab, getattr(capi, name), *q, quantile=qt)
                    assert_same(vals, exp, "%s rows with quantile q=%s" % (name, q))
                    what = "%s %s quantile %g q=%s" % (scheme, name, qt, q)
                    assert (np.isnan(qgot) == np.isnan(qexp)).all(), what
                    assert (np.isinf(qgot) == np.isinf(qexp)).all() and (np.sign(qgot[np.isinf(qgot)]) == np.sign(qexp[np.isinf(qexp)])).all(), what
                    f = np.isfinite(qexp)
                    np.testing.assert_allclose(qgot[f], qexp[f], rtol=1e-9, atol=0, err_msg=what)
                    qonly = ctx.query_hist(tab, getattr(capi, name), *q, quantile=qt, want_values=False)
                    assert_same(qonly, qgot, what + " quantile only")
                    check_counters(ctx, st, ts_l, ch_l, q)
                if name == "FN_RATE":
                    d = np.diff(np.nan_to_num(exp, nan=0.0), axis=2)
                    nonmono += int(((d < 0).any(axis=2) & ~empty).sum())
        assert nonmono > 0                   # per-series rate histograms that are not monotonic over their buckets are part of the data
    finally:
        tab.free()


@pytest.mark.parametrize("v2", ["1", "0"])
def test_hist_quantile_per_series_delta_schema(gpu, oracle, v2, monkeypatch):
    """Delta-temporality histograms in simple vectors: per-series quantile of rate / increase / sum_over_time / last."""
    monkeypatch.setenv("FILO_HIST_V2", v2)
    capi, ctx = gpu; o = oracle
    from oracle import hist as H
    b = _buckets(H, "geometric")
    st, ts_l, ch_l = _store(H, b, 11, 33, sect=False, delta=True)
    tab = ctx.load_series(*st.all_info_addrs(), schema_flags=0)
    try:
        for q in QUERIES[:2]:
            for name in FNS:
                if name == "FN_LAST":
                    exp, empty = R.last_store(st, ts_l, ch_l, b.n, *q)
                else:
                    exp, empty = st.query(getattr(o, name), *q, cumulative=False); exp = exp.copy(); exp[empty] = NaN
                qexp = R.quantiles(b, exp, empty, 0.75)
                vals, qgot = ctx.query_hist(tab, getattr(capi, name), *q, quantile=0.75)
                assert_same(vals, exp, "delta %s q=%s" % (name, q))
                check_counters(ctx, st, ts_l, ch_l, q)
                assert (np.isnan(qgot) == np.isnan(qexp)).all()
                np.testing.assert_allclose(qgot[~np.isnan(qexp)], qexp[~np.isnan(qexp)], rtol=1e-9, atol=0)
    finally:
        tab.free()


def test_reference_known_answer_on_the_device(gpu, oracle):
    """InstantFunctionSpec.scala:315-327 through the device: histogram_quantile(0.4, h) per series over linearHistSeries (last at each
    sample) gives 0.8, 1.6, 2.4, 3.2, 4.0, 5.6, 7.2, 9.6 (the reference compares with +- 0.0001)."""
    capi, ctx = gpu
    from oracle import hist as H
    from tests.test_hist_series_oracle import linear_hist_series
    b = H.Buckets.geometric(2.0, 2.0, 8)
    st = H.HistStore(b)
    ts = 100000 + np.arange(10, dtype=np.int64) * 1000
    st.add_series(ts, linear_hist_series(10), [10])
    tab = ctx.load_series(*st.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE)
    try:
        qs = ctx.query_hist(tab, capi.FN_LAST, 100000, 1000, 107000, 0, quantile=0.4, want_values=False)
        np.testing.assert_allclose(qs[0], [0.8, 1.6, 2.4, 3.2, 4.0, 5.6, 7.2, 9.6], rtol=1e-15, atol=0)
    finally:
        tab.free()


def test_operator_mirrors(gpu, oracle, tmp_path):
    """exec.FusedGpuExec and include/filo_b200.hpp: PeriodicSamplesMapper(functionId unset = LastSample) over a histogram column, and
    HistogramQuantileMapper without an aggregate -> [series, T]."""
    capi, ctx = gpu
    from oracle import hist as H
    from filodb_b200 import exec as fx
    b = _buckets(H, "custom")
    S = 7
    st, ts_l, ch_l = _store(H, b, S, 34)
    nch, addrs = st.all_info_addrs()
    src, pos = [], 0
    for n in nch:
        src.append(fx.RawDataRangeVector([int(a) for a in addrs[pos:pos + int(n)]])); pos += int(n)
    q = QUERIES[0]
    exp, empty = R.last_store(st, ts_l, ch_l, b.n, *q)
    ex = fx.FusedGpuExec(0)
    try:
        res = ex.execute(src, fx.PeriodicSamplesMapper(q[0], q[1], q[2], None, None), cumulative=True, histogram=True)
        assert_same(np.asarray(res.values), exp, "exec last")
        res = ex.execute(src, fx.PeriodicSamplesMapper(q[0], q[1], q[2], q[3], capi.FN_RATE), quantile=fx.HistogramQuantileMapper(0.99),
                         cumulative=True, histogram=True)
        rexp, rempty = st.query(oracle.FN_RATE, *q); rexp = rexp.copy(); rexp[rempty] = NaN
        qexp = R.quantiles(b, rexp, rempty, 0.99)
        got = np.asarray(res.values)
        assert got.shape == (S, rexp.shape[1]) and (np.isnan(got) == np.isnan(qexp)).all()
        np.testing.assert_allclose(got[~np.isnan(qexp)], qexp[~np.isnan(qexp)], rtol=1e-9, atol=0)
    finally:
        ex.close()
    # the C++ mirror: LastSample and the per-series quantile through FusedGpuExec::execute (tests/cpp/hist_mirror_gpu.cpp)
    import os, subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir, odir = os.path.join(root, "filodb_b200"), os.path.join(root, "oracle", "_build")
    exe = str(tmp_path / "hist_mirror_gpu")
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-I", os.path.join(root, "include"), os.path.join(root, "tests", "cpp", "hist_mirror_gpu.cpp"),
                    "-o", exe, "-L", libdir, "-L", odir, "-lfilo_b200", "-lfilo_oracle", "-Wl,-rpath," + libdir + ":" + odir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "OK hist mirror" in r.stdout, r.stdout + r.stderr


def test_hist_quantile_per_series_at_scale(gpu, oracle, monkeypatch):
    """histogram_quantile(0.99, rate(h[5m])) per series over 1 M synthetic series (20 buckets, 2 h at 15 s, T = 481): [S][T][nb] would
    be 77 GB, the call returns [S][T] without it.  Spot checks at three offsets (2,100 series) against tables built with series_id_base:
    the same quantiles, Histogram.quantile of the bucket rows on the host, and the first kernel."""
    capi, ctx = gpu
    from oracle import hist as H
    S, nb, rows = 1_000_000, 20, 480
    les = [2.0 * 3 ** i for i in range(nb - 1)] + [float("inf")]
    bdef, bfmt = capi.custom_bucket_def(les)
    b = H.Buckets.custom(les)
    q = (T0, 15000, T0 + 7200000, 300000)
    monkeypatch.setenv("FILO_HIST_V2", "1")
    tab = ctx.synth_hist_table(S, rows, bdef, bfmt, nb, rows_per_chunk=400, t0_ms=T0, interval_ms=15000, reset_period=97, seed=42)
    try:
        big = ctx.query_hist(tab, capi.FN_RATE, *q, quantile=0.99, want_values=False)
        assert ctx.last_stats["samples_scanned"] == tab.info().n_samples
    finally:
        tab.free()
    assert big.shape == (S, 481) and np.isfinite(big).mean() > 0.9
    for base in (0, 500_000, S - 700):
        sm = ctx.synth_hist_table(700, rows, bdef, bfmt, nb, rows_per_chunk=400, t0_ms=T0, interval_ms=15000, reset_period=97, seed=42, series_id_base=base)
        try:
            monkeypatch.setenv("FILO_HIST_V2", "1")
            vals, qs = ctx.query_hist(sm, capi.FN_RATE, *q, quantile=0.99)
            assert_same(qs, big[base:base + 700], "per-series quantile at series %d" % base)
            empty = np.isnan(vals[:, :, 0])
            host = R.quantiles(b, vals, empty, 0.99)
            assert (np.isnan(host) == np.isnan(qs)).all()
            np.testing.assert_allclose(qs[~np.isnan(host)], host[~np.isnan(host)], rtol=1e-9, atol=0)
            monkeypatch.setenv("FILO_HIST_V2", "0")
            v1 = ctx.query_hist(sm, capi.FN_RATE, *q, quantile=0.99, want_values=False)
            assert (np.isnan(v1) == np.isnan(qs)).all()
            np.testing.assert_allclose(v1[~np.isnan(qs)], qs[~np.isnan(qs)], rtol=1e-9, atol=0)
        finally:
            sm.free()


def test_hist_quantile_per_series_many_windows(gpu, oracle, monkeypatch):
    """The first kernel stages a series' [T][nb] window rows in shared memory, the second kernel does not: 3,601 windows x 20 buckets
    (563 KB) run per series on the second kernel, and the first kernel declines them with FILO_ERR_UNSUPPORTED."""
    capi, ctx = gpu; o = oracle
    from oracle import hist as H
    b = _buckets(H, "custom")
    st, ts_l, ch_l = _store(H, b, 4, 35)
    tab = ctx.load_series(*st.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE)
    q = (T0, 1000, T0 + 3600000, 300000)
    try:
        exp, empty = st.query(o.FN_RATE, *q); exp = exp.copy(); exp[empty] = NaN
        qexp = R.quantiles(b, exp, empty, 0.9)
        monkeypatch.setenv("FILO_HIST_V2", "1")
        qgot = ctx.query_hist(tab, capi.FN_RATE, *q, quantile=0.9, want_values=False)
        assert qgot.shape == (4, 3601) and (np.isnan(qgot) == np.isnan(qexp)).all()
        np.testing.assert_allclose(qgot[~np.isnan(qexp)], qexp[~np.isnan(qexp)], rtol=1e-9, atol=0)
        check_counters(ctx, st, ts_l, ch_l, q)
        monkeypatch.setenv("FILO_HIST_V2", "0")
        with pytest.raises(capi.FiloError) as ei:
            ctx.query_hist(tab, capi.FN_RATE, *q, quantile=0.9, want_values=False)
        assert ei.value.code == capi.ERR_UNSUPPORTED
    finally:
        tab.free()
