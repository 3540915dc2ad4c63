"""Value edges, CPU side: the oracle's min / max across series pinned to the reference's QueryUtils rule, and the scan kernels at
value edges on the SIMT emulator (tests/cpp/value_edges_emul.cpp): signed-zero ties through the fused v4 counter kernel, the v2
aggregate kernel and merge_partials_kernel, and the v4 SUM kernel's decode bounds."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T0 = 1_700_000_000_000
NaN = float("nan")


def _last_of_each(o, values):
    """One series per value, each holding it in all of its rows: last() is the value in every window."""
    st = o.Store()
    ts = T0 + np.arange(4, dtype=np.int64) * 15000
    for v in values:
        st.add_series_rows(ts, np.full(4, v), [4], val_mode=o.VAL_RAW)
    return st


@pytest.mark.parametrize("values, exp_min, exp_max", [
    ([0.0, -0.0], -0.0, -0.0),
    ([-0.0, 0.0], 0.0, 0.0),
    ([0.0, NaN, -0.0], -0.0, -0.0),
    ([-0.0, NaN, NaN, 0.0], 0.0, 0.0),
    ([NaN, -0.0, 0.0, NaN], 0.0, 0.0),
    ([1.0, 0.0, -0.0, -1.0], -1.0, 1.0),
    ([-1.0, -0.0, 0.0], -1.0, 0.0),
    ([1.0, 0.0, -0.0], -0.0, 1.0),
])
def test_oracle_min_max_keep_the_later_of_equal_values(oracle, values, exp_min, exp_max):
    """MinRowAggregator / MaxRowAggregator fold acc = minIgnoreNaN(acc, v) / maxIgnoreNaN(acc, v) (MinRowAggregator.scala:24,
    QueryUtils.scala:111-123): `if (a < b) a else b`, so of +0.0 and -0.0 the later one is kept; NaNs in between are skipped."""
    o = oracle
    st = _last_of_each(o, values)
    q = (T0 + 45000, 15000, T0 + 45000, 60000)
    for aggr, exp in ((o.AGG_MIN, exp_min), (o.AGG_MAX, exp_max)):
        got = st.query(o.FN_LAST, *q, aggr=aggr, n_groups=1)
        assert got.shape == (1, 1)
        assert got[0, 0] == exp and np.signbit(got[0, 0]) == np.signbit(exp), (values, aggr, got[0, 0])


def test_oracle_min_max_over_only_nan_is_nan(oracle):
    o = oracle
    st = _last_of_each(o, [NaN, NaN])
    for aggr in (o.AGG_MIN, o.AGG_MAX):
        assert np.isnan(st.query(o.FN_LAST, T0 + 45000, 15000, T0 + 45000, 60000, aggr=aggr, n_groups=1)[0, 0])


def test_value_edges_on_the_simt_emulator(tmp_path):
    """tests/cpp/value_edges_emul.cpp: fused min / max over signed-zero tables (the v4 counter kernel over delta, the v2 aggregate kernel
    over last and min_over_time, merge_partials_kernel over 14 items of one group) against the oracle's aggregate(), bit for bit; the v4
    SUM kernel declines exactly the series holding a value outside 2^-511 <= |v| < 2^513 and every result is bit-exact after the v2
    pass; in-order and pseudo-random fiber schedules."""
    src = str(tmp_path / "scan_kernels_cusim.cu")
    subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cpp", "make_cusim_src.py"), os.path.join(ROOT, "filodb_b200", "csrc", "scan_kernels.cu"), src], check=True)
    exe = str(tmp_path / "value_edges_emul")
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", "-I", "/usr/local/cuda/include",
                    "-I", os.path.join(ROOT, "filodb_b200", "csrc"), '-DSCAN_SRC="%s"' % src,
                    os.path.join(ROOT, "tests", "cpp", "value_edges_emul.cpp"), "-o", exe], check=True)
    for seed in ("0", "20261016"):
        r = subprocess.run([exe, seed], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "OK 14 cases" in r.stdout and "bit-exact" in r.stdout, r.stdout
