"""Pins the CPU restatement of histogram `last` (LastSampleChunkedFunctionH) and per-series histogram_quantile (tests/hist_series_ref.py)
to the reference's rules and known answers.  CPU only."""
import numpy as np
import pytest

from tests import hist_series_ref as R

T0 = 1_700_000_000_000


def linear_hist_series(n, num_buckets=8):
    """TestData.linearHistSeries (core/src/test/scala/filodb.core/TestData.scala:375-395): sample n adds 1 to the buckets from
    n % numBuckets up, GeometricBuckets(2.0, 2.0, numBuckets)."""
    buckets = np.zeros(num_buckets, np.int64); rows = []
    for i in range(n):
        buckets[i % num_buckets:] += 1
        rows.append(buckets.copy())
    return np.array(rows)


@pytest.fixture(scope="module")
def H(oracle):
    from oracle import hist
    return hist


def test_reference_known_answer_histogram_quantile_per_series(H):
    """InstantFunctionSpec.scala:315-327: histogram_quantile(0.4) over the histogram RV of linearHistSeries (the reference compares
    with +- 0.0001, :449-451; 2.4 comes out as 2.4000000000000004 in double arithmetic)."""
    b = H.Buckets.geometric(2.0, 2.0, 8)
    rows = linear_hist_series(10).astype(np.float64)
    got = [b.quantile(rows[i], 0.4) for i in range(8)]
    np.testing.assert_allclose(got, [0.8, 1.6, 2.4, 3.2, 4.0, 5.6, 7.2, 9.6], rtol=1e-15, atol=0)


def test_quantile_of_a_non_monotonic_histogram_is_literal(H):
    """Histogram.quantile walks firstBucketGTE from bucket 0 over the histogram as it is (no makeMonotonic)."""
    b = H.Buckets.custom([1.0, 2.0, 4.0, 8.0, float("inf")])
    v = np.array([4.0, 2.0, 6.0, 6.0, 10.0])
    # rank 5: bucket 2 (6 >= 5), count = 6 - 2, rank - 2 = 3 -> 2 + (4 - 2) * 0.75
    assert b.quantile(v, 0.5) == 3.5
    assert b.quantile(H.make_monotonic(v), 0.5) == 3.0                      # what a makeMonotonic would have changed
    assert b.quantile(v, -0.1) == -np.inf and b.quantile(v, 1.5) == np.inf
    assert np.isnan(b.quantile(np.zeros(5), 0.5))                              # top bucket 0: NaN
    assert b.quantile(v, 1.0) == 8.0                                            # the +Inf bucket answers the last finite top
    e = R.quantiles(b, v.reshape(1, 1, 5).repeat(2, axis=1), np.array([[False, True]]), 0.5)
    assert e[0, 0] == 3.5 and np.isnan(e[0, 1])                                # Histogram.empty: NaN


def _store(H, b, series):
    st = H.HistStore(b)
    for ts, vals, chunks, sect in series:
        st.add_series(ts, vals, chunks, sect=sect)
    return st


def test_last_rules(H):
    b = H.Buckets.geometric(2.0, 2.0, 6)
    rows = 40
    ts = T0 + np.arange(rows, dtype=np.int64) * 15000
    inc = np.cumsum(np.ones((rows, 6), np.int64), axis=1)
    vals = np.cumsum(inc, axis=0)
    vals[25:] = np.cumsum(inc[25:], axis=0)                                    # counter reset at row 25: a Drop section
    st = _store(H, b, [(ts, vals, [20, 20], True), (ts, vals, [20, 20], False)])
    rd = H.Reader(st.vector_bytes(0, 1))
    assert 1 in rd.section_types()[1:]                                          # the reset is a Drop section inside chunk 1
    # the raw value after the drop (asHistReader) is the appended histogram, the corrected value is not
    assert (rd(5) == vals[25]).all() and not (rd.corrected(5) == vals[25]).all()
    for s in (0, 1):
        sc = R.SeriesChunks(st, s, ts, [20, 20])
        # every row: an instant query at a row's timestamp returns that row, raw
        for r in (0, 19, 20, 25, 39):
            v, e = R.last_series(sc, 6, int(ts[r]), 0, int(ts[r]), 60000)
            assert not e[0] and (v[0] == vals[r]).all()
        # a window across the chunk boundary: the later chunk's row wins (ts > kept timestamp)
        v, _ = R.last_series(sc, 6, int(ts[20]) + 1000, 0, int(ts[20]) + 1000, 60000)
        assert (v[0] == vals[20]).all()
        # a window ending before chunk 1's first row: chunk 1 is in the chunk set but has no row <= end, chunk 0's last row is kept
        v, _ = R.last_series(sc, 6, int(ts[19]) + 5000, 0, int(ts[19]) + 5000, 60000)
        assert (v[0] == vals[19]).all()
        # a window without a sample (the row is older than windowStart): Histogram.empty
        v, e = R.last_series(sc, 6, int(ts[39]) + 200000, 0, int(ts[39]) + 200000, 60000)
        assert e[0] and np.isnan(v[0]).all()
        # the default lookback: window <= 0 is 5 min + 1 ms
        q = (int(ts[0]) - 30000, 7000, int(ts[39]) + 400000)
        a, ea = R.last_series(sc, 6, *q, 0)
        b2, eb = R.last_series(sc, 6, *q, R.DEFAULT_LOOKBACK_MS)
        assert (ea == eb).all() and np.array_equal(a, b2, equal_nan=True) and ea.any() and not ea.all()
