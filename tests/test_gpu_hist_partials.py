"""GPU: the cross-GPU histogram sum.  filo_query_hist_device (device outputs on a torch stream, with and without stats) against
filo_query_hist, and filo_merge_hist_partials over the SUM partials of W tables cut from one series set, against a numpy rank fold of
those partials (bitwise) and the oracle over the unsharded series; on both histogram scan kernels (FILO_HIST_V2 = 1 and 0)."""
import numpy as np
import pytest

from tests import hist_series_ref as R

pytestmark = pytest.mark.gpu
T0 = 1_700_000_000_000
ROWS = 160


def same_bits(a, b):
    a = np.ascontiguousarray(a, np.float64); b = np.ascontiguousarray(b, np.float64)
    an, bn = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and (an == bn).all() and (a[~an].view(np.uint64) == b[~bn].view(np.uint64)).all()


def close_quantiles(got, exp, what):
    assert (np.isnan(got) == np.isnan(exp)).all(), what
    f = ~np.isnan(exp)
    np.testing.assert_allclose(got[f], exp[f], rtol=1e-9, atol=0, err_msg=what)


@pytest.fixture(scope="module")
def gpu():
    import torch
    import filodb_b200.capi as capi
    ctx = capi.Context(0)
    yield capi, ctx, torch
    ctx.close()


def _buckets(H, scheme):
    if scheme == "custom":
        return H.Buckets.custom([2.0 * 3 ** i for i in range(19)] + [float("inf")])
    if scheme == "otel":
        return H.Buckets.exponential(3, -5, 15)
    return H.Buckets.geometric(2.0, 2.0, 12)


def _series_set(b, S, seed, base=0, resets=False):
    """S series: jittered timestamps for some, late starts for others (windows empty on some tables only), 1-3 chunks; with resets,
    counter resets inside chunks and at chunk starts."""
    rng = np.random.default_rng(seed)
    out = []
    for s in range(S):
        jit = rng.integers(-200, 201, ROWS) if s % 5 == 1 else 0
        ts = T0 + np.arange(ROWS, dtype=np.int64) * 15000 + jit + (600000 * (s % 4 == 3))
        inc = np.cumsum(rng.integers(0, 20, (ROWS, b.n)), axis=1)
        vals = np.cumsum(inc, axis=0)
        if resets and s % 3 == 1:
            vals[90:] = np.cumsum(inc[90:], axis=0)
        out.append((ts, (base + vals).astype(np.int64), [[60, 60, 40], [100, 60], [ROWS]][s % 3]))
    return out


def _store(H, b, series):
    st = H.HistStore(b)
    for ts, vals, chunks in series:
        st.add_series(ts, vals, chunks)
    return st


def _gids(S, G):
    """group G - 1 has no series, group G - 2 only series 0 (empty on every table but the first); the others are spread"""
    return np.array([G - 2 if s == 0 else (s * 5 + 2) % (G - 2) for s in range(S)], np.int32)


Q = (T0 + 300000, 15000, T0 + (ROWS + 30) * 15000, 300000)


def _dev(torch, shape):
    t = torch.full(shape, -7.0, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()                 # the fill is done before a kernel on another stream writes the buffer
    return t


@pytest.mark.parametrize("v2", ["1", "0"])
def test_query_hist_device_matches_query_hist(gpu, oracle, v2, monkeypatch):
    """rate and last, aggr NONE (rows and the per-series quantile) and SUM (rows and quantile): the device call on a torch stream returns
    the bits of the host call, with stats and without (then filo_ctx_check returns OK)."""
    monkeypatch.setenv("FILO_HIST_V2", v2)
    capi, ctx, torch = gpu
    from oracle import hist as H
    b = _buckets(H, "custom")
    S, G = 21, 4
    st = _store(H, b, _series_set(b, S, 11, resets=True))
    tab = ctx.load_series(*st.all_info_addrs(), group_ids=_gids(S, G), n_groups=G, schema_flags=capi.SCHEMA_CUMULATIVE)
    T = capi.num_windows(Q[0], Q[1], Q[2])
    stream = torch.cuda.Stream()
    try:
        for fn in (capi.FN_RATE, capi.FN_LAST):
            for aggr, rows in ((capi.AGG_NONE, S), (capi.AGG_SUM, G)):
                vals, qs = ctx.query_hist(tab, fn, *Q, aggr=aggr, quantile=0.9)
                for want_stats in (True, False):
                    dv, dq = _dev(torch, (rows, T, b.n)), _dev(torch, (rows, T))
                    with torch.cuda.stream(stream):
                        ctx.query_hist_device(tab, fn, *Q, d_values=dv.data_ptr(), d_quantile=dq.data_ptr(), aggr=aggr, quantile=0.9,
                                              stream=stream.cuda_stream, want_stats=want_stats)
                    if not want_stats:
                        ctx.check()
                    stream.synchronize()
                    what = "fn %d aggr %d stats %s" % (fn, aggr, want_stats)
                    assert same_bits(dv.cpu().numpy(), vals), what
                    assert same_bits(dq.cpu().numpy(), qs), what
                # quantile alone and rows alone
                dq = _dev(torch, (rows, T))
                ctx.query_hist_device(tab, fn, *Q, d_quantile=dq.data_ptr(), aggr=aggr, quantile=0.9, stream=stream.cuda_stream)
                stream.synchronize()
                assert same_bits(dq.cpu().numpy(), qs)
                dv = _dev(torch, (rows, T, b.n))
                ctx.query_hist_device(tab, fn, *Q, d_values=dv.data_ptr(), aggr=aggr, stream=stream.cuda_stream)
                stream.synchronize()
                assert same_bits(dv.cpu().numpy(), vals)
                assert ctx.last_stats["samples_scanned"] > 0 and ctx.last_stats["d2h_bytes"] == 0
    finally:
        tab.free()


def _subset(nch, addrs, ids):
    off = np.concatenate([[0], np.cumsum(nch)])
    return nch[ids], np.concatenate([addrs[off[i]:off[i + 1]] for i in ids]) if len(ids) else np.zeros(1, np.uint64)


def _rank_fold(parts, nb):
    """ReduceAggregateExec over the parts [W, G, T, nb] in rank order (tests/hist_series_ref.py hist_sum; empty = NaN bucket 0)."""
    W, G, T, _ = parts.shape
    rows = parts.reshape(W * G, T, nb)
    return R.hist_sum(nb, rows, np.isnan(rows[:, :, 0]), np.tile(np.arange(G), W), G)


@pytest.mark.parametrize("v2", ["1", "0"])
def test_merge_of_one_part_is_the_sum(gpu, oracle, v2, monkeypatch):
    """W = 1: the merge of one SUM partial gives filo_query_hist's SUM values and quantile, bit for bit."""
    monkeypatch.setenv("FILO_HIST_V2", v2)
    capi, ctx, torch = gpu
    from oracle import hist as H
    b = _buckets(H, "otel")
    S, G = 17, 4
    st = _store(H, b, _series_set(b, S, 12, resets=True))
    tab = ctx.load_series(*st.all_info_addrs(), group_ids=_gids(S, G), n_groups=G, schema_flags=capi.SCHEMA_CUMULATIVE)
    T = capi.num_windows(Q[0], Q[1], Q[2])
    try:
        for fn in (capi.FN_RATE, capi.FN_INCREASE, capi.FN_LAST):
            vals, qs = ctx.query_hist(tab, fn, *Q, aggr=capi.AGG_SUM, quantile=0.75)
            part = _dev(torch, (1, G, T, b.n))
            ctx.query_hist_device(tab, fn, *Q, d_values=part.data_ptr(), aggr=capi.AGG_SUM)
            mv, mq = _dev(torch, (G, T, b.n)), _dev(torch, (G, T))
            ctx.merge_hist_partials(tab, 1, T, part.data_ptr(), mv.data_ptr(), mq.data_ptr(), quantile=0.75)
            torch.cuda.synchronize()
            assert same_bits(part[0].cpu().numpy(), vals)
            assert same_bits(mv.cpu().numpy(), vals) and same_bits(mq.cpu().numpy(), qs), fn
    finally:
        tab.free()


@pytest.mark.parametrize("v2", ["1", "0"])
@pytest.mark.parametrize("scheme", ["custom", "geometric", "otel"])
@pytest.mark.parametrize("split", ["contiguous", "interleaved"])
def test_merge_of_sharded_partials(gpu, oracle, scheme, split, v2, monkeypatch):
    """W = 2, 4, 8 tables on one device, cut by contiguous series ranges (shard.series_range_of_rank) or by shard (s % W): the merge equals
    a numpy rank fold of the device partials bitwise, its quantile the oracle's quantile of that fold, and both are within 1e-9 of the
    oracle over the unsharded series (whose rates are monotonic per series, so that the fold tree changes rounding only)."""
    monkeypatch.setenv("FILO_HIST_V2", v2)
    capi, ctx, torch = gpu
    from filodb_b200 import shard
    from oracle import hist as H
    o = oracle
    b = _buckets(H, scheme)
    S, G, QT = 29, 5, 0.95
    series = _series_set(b, S, 13, base=1_000_000)
    st = _store(H, b, series)
    gids = _gids(S, G)
    nch, addrs = st.all_info_addrs()
    T = capi.num_windows(Q[0], Q[1], Q[2])
    exp, eempty, eq = st.query(o.FN_RATE, *Q, aggr=True, group_ids=gids, n_groups=G, q=QT)
    exp = exp.copy(); exp[eempty] = np.nan; eq = np.where(eempty, np.nan, eq)
    for W in (2, 4, 8):
        ids = [list(range(*shard.series_range_of_rank(S, r, W))) if split == "contiguous" else list(range(r, S, W)) for r in range(W)]
        tabs = [ctx.load_series(*_subset(nch, addrs, i), group_ids=gids[i], n_groups=G, schema_flags=capi.SCHEMA_CUMULATIVE) for i in ids]
        try:
            parts = _dev(torch, (W, G, T, b.n))
            for r, t in enumerate(tabs):
                ctx.query_hist_device(t, capi.FN_RATE, *Q, d_values=parts[r].data_ptr(), aggr=capi.AGG_SUM, want_stats=False)
            mv, mq = _dev(torch, (G, T, b.n)), _dev(torch, (G, T))
            ctx.merge_hist_partials(tabs[-1], W, T, parts.data_ptr(), mv.data_ptr(), mq.data_ptr(), quantile=QT)
            ctx.check()
            torch.cuda.synchronize()
            hp, got, gq = parts.cpu().numpy(), mv.cpu().numpy(), mq.cpu().numpy()
            what = "%s %s W=%d" % (scheme, split, W)
            assert (np.isnan(hp) == np.isnan(hp[..., :1])).all(), what        # a partial cell is all-NaN or has no NaN
            e = np.isnan(hp[..., 0])
            assert (e.any(axis=0) & ~e.all(axis=0)).any(), what              # cells empty on some tables and not on others
            fold, fempty = _rank_fold(hp, b.n)
            assert same_bits(got, fold), what
            close_quantiles(gq, R.quantiles(b, fold, fempty, QT), what)
            assert (np.isnan(got) == np.isnan(exp)).all(), what
            m = ~np.isnan(exp)
            np.testing.assert_allclose(got[m], exp[m], rtol=1e-9, atol=0, err_msg=what)
            close_quantiles(gq, eq, what)
            mv2 = _dev(torch, (G, T, b.n))                                    # values only: NaN quantile
            ctx.merge_hist_partials(tabs[0], W, T, parts.data_ptr(), mv2.data_ptr(), mq.data_ptr())
            torch.cuda.synchronize()
            assert same_bits(mv2.cpu().numpy(), got) and same_bits(mq.cpu().numpy(), gq), what
        finally:
            for t in tabs:
                t.free()


def test_error_paths(gpu, oracle):
    """Statuses of the two entry points, and a device-side error of a call without stats reported by filo_ctx_check with the status and
    message of the synchronous call."""
    capi, ctx, torch = gpu
    from oracle import hist as H
    b = _buckets(H, "geometric")
    st = _store(H, b, _series_set(b, 3, 14))
    tab = ctx.load_series(*st.all_info_addrs(), group_ids=np.array([0, 1, 0], np.int32), n_groups=2, schema_flags=capi.SCHEMA_CUMULATIVE)
    scalar = ctx.synth_table(4, 100, 50, T0, 15000)
    T = capi.num_windows(Q[0], Q[1], Q[2])
    parts, mv, mq = _dev(torch, (2, 2, T, b.n)), _dev(torch, (2, T, b.n)), _dev(torch, (2, T))

    def status(f):
        with pytest.raises(capi.FiloError) as ei:
            f()
        return ei.value.code, str(ei.value)

    try:
        assert status(lambda: ctx.merge_hist_partials(tab, 0, T, parts.data_ptr(), mv.data_ptr()))[0] == capi.ERR_INVALID_ARG
        assert status(lambda: ctx.merge_hist_partials(tab, 2, 0, parts.data_ptr(), mv.data_ptr()))[0] == capi.ERR_INVALID_ARG
        assert status(lambda: ctx.merge_hist_partials(scalar, 2, T, parts.data_ptr(), mv.data_ptr()))[0] == capi.ERR_INVALID_ARG
        assert status(lambda: ctx.merge_hist_partials(tab, 2, T, parts.data_ptr()))[0] == capi.ERR_INVALID_ARG
        assert status(lambda: ctx.merge_hist_partials(tab, 2, T, parts.data_ptr(), 0, mq.data_ptr()))[0] == capi.ERR_INVALID_ARG   # q NaN
        assert status(lambda: ctx.merge_hist_partials(tab, 2, T, 0, mv.data_ptr()))[0] == capi.ERR_INVALID_ARG
        assert status(lambda: ctx.query_hist_device(tab, capi.FN_RATE, *Q, aggr=capi.AGG_SUM))[0] == capi.ERR_INVALID_ARG
        assert status(lambda: ctx.query_hist_device(scalar, capi.FN_RATE, *Q, d_values=mv.data_ptr()))[0] == capi.ERR_INVALID_ARG
        assert status(lambda: ctx.query_hist_device(tab, capi.FN_RATE, *Q, d_values=mv.data_ptr(), aggr=capi.AGG_AVG))[0] == capi.ERR_UNSUPPORTED
        ctx.merge_hist_partials(tab, 2, T, parts.data_ptr(), mv.data_ptr(), mq.data_ptr(), quantile=0.5)
        ctx.check()
        # a series with more chunks in range than the device path holds: code 5 of the kernels
        many = _store(H, b, [(T0 + np.arange(ROWS, dtype=np.int64) * 15000, np.cumsum(np.ones((ROWS, b.n), np.int64), axis=0), [16] * 10)])
        mt = ctx.load_series(*many.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE)
        q = (T0, 15000, T0 + ROWS * 15000, 300000)
        try:
            sync = status(lambda: ctx.query_hist(mt, capi.FN_RATE, *q, aggr=capi.AGG_SUM))
            assert sync[0] == capi.ERR_UNSUPPORTED
            ctx.query_hist_device(mt, capi.FN_RATE, *q, d_values=mv.data_ptr(), aggr=capi.AGG_SUM, want_stats=False)
            assert status(ctx.check) == sync
            ctx.check()                                                      # reported once
        finally:
            mt.free()
    finally:
        tab.free(); scalar.free()


def test_invalid_query_is_refused_before_any_allocation(gpu, oracle):
    """filo_query_hist checks its arguments before it sizes any device buffer: a range query with step <= 0, or with a step below min-step,
    over ten days (one window per millisecond: hundreds of GB of output) returns INVALID_ARG / BAD_QUERY with the reference's message,
    not an allocation failure; the device form returns the same."""
    import ctypes as C
    capi, _, torch = gpu
    from oracle import hist as H
    b = _buckets(H, "geometric")
    st = _store(H, b, _series_set(b, 3, 15))
    start, end = T0, T0 + 10 * 86400 * 1000
    for min_step, step, code, msg in ((0, 0, capi.ERR_INVALID_ARG, "step should be > 0"), (0, -5, capi.ERR_INVALID_ARG, "step should be > 0"),
                                      (60000, 1, capi.ERR_BAD_QUERY, "min-step")):
        ctx = capi.Context(0, min_step_ms=min_step)
        tab = ctx.load_series(*st.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE)
        try:
            small = np.zeros(16, np.float64)              # never written: the call fails before any result exists
            for aggr in (capi.AGG_NONE, capi.AGG_SUM):
                rc = capi.lib().filo_query_hist(ctx.h, tab.h, capi.FN_RATE, start, step, end, 300000, aggr, 0.9,
                                                small.ctypes.data, small.ctypes.data, C.byref(capi.Stats()))
                buf = C.create_string_buffer(1024); capi.lib().filo_last_error(ctx.h, buf, 1024)
                assert rc == code and msg in buf.value.decode(), (step, aggr, rc, buf.value)
                with pytest.raises(capi.FiloError) as ei:
                    ctx.query_hist_device(tab, capi.FN_RATE, start, step, end, 300000, d_values=int(small.ctypes.data), aggr=aggr)
                assert ei.value.code == code and msg in str(ei.value)
            assert not small.any()
        finally:
            tab.free(); ctx.close()
