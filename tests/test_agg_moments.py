"""stddev / stdvar / group across series (FILO_AGG_STDDEV / STDVAR / GROUP), CPU side: the literal restatement of the reference's
RowAggregators (tests/agg_moments_ref.py) pinned to the reference's own known answers, the moment form the device uses held to it,
the C-ABI constants, a two-rank gloo merge of moment partials, and the moments mode of the scan kernels on the SIMT emulator."""
import os
import re
import socket
import subprocess
import sys

import numpy as np
import pytest

from tests import agg_moments_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERROR = 1e-7                  # AggrOverRangeVectorsSpec.scala:20 (compareIter :961-968)
NaN = float("nan")


def _close(got, exp):
    got = np.asarray(got, np.float64); exp = np.asarray(exp, np.float64)
    assert (np.isnan(got) == np.isnan(exp)).all()
    m = ~np.isnan(exp)
    assert (np.abs(got[m] - exp[m]) < ERROR).all(), (got, exp)


# AggrOverRangeVectorsSpec.scala:387-419 ("stdvar and stddev should work for with NaN Test case 2"): 11 series, one group
NAN_CASE = [[3247.0, 3297.0]] + [[NaN, NaN]] * 6 + [[5173.0, 5173.0], [NaN, NaN], [11583.0, 11583.0], [NaN, NaN]]
# :780-815 ("should aggregate correctly when grouping is applied"), without(a): b=1 <- series 0; b=2 <- series 1, 2
GROUP_CASE = ([[1.5, 5.6], [2.4, 4.4], [3.2, 5.4]], [0, 1, 1])


@pytest.mark.parametrize("op, expected", [(R.STDVAR, [12698496.88888889, 12585030.222222222]), (R.STDDEV, [3563.4950384263, 3547.5386146203])])
def test_reference_known_answers_with_nan_series(op, expected):
    """The spec's two levels: the leaf mapReduce over the samples, then mapReduce(skipMapPhase = true) over the leaf result."""
    lf = R.leaf(op, np.array(NAN_CASE))
    _close(R.two_level(op, [lf]).stat, expected)
    # the device's moment form of the same cells: (Σv, Σv², n) presented once
    (vals, cnts) = R.moment_partials(np.array(NAN_CASE), None, 1)
    _close(R.present_moments(op, vals[0], vals[1], cnts)[0], expected)


@pytest.mark.parametrize("op, b1, b2", [(R.GROUP, [1.0, 1.0], [1.0, 1.0]), (R.STDDEV, [0.0, 0.0], [0.4, 0.5]), (R.STDVAR, [0.0, 0.0], [0.16, 0.25])])
def test_reference_known_answers_grouped(op, b1, b2):
    rows, gids = GROUP_CASE
    rows = np.array(rows); gids = np.array(gids)
    for g, exp in ((0, b1), (1, b2)):
        lf = R.leaf(op, rows[gids == g])
        top = R.two_level(op, [lf])
        _close(top if op == R.GROUP else top.stat, exp)
    vals, cnts = R.moment_partials(rows, gids, 2)
    _close(R.present_moments(op, vals[0], vals[1], cnts), [b1, b2])
    # one leaf per shard: the series of group b=2 split over two leaves merge to the same answer
    if op != R.GROUP:
        top = R.two_level(op, [R.leaf(op, rows[1:2]), R.leaf(op, rows[2:3])])
        _close(top.stat, b2)


def test_java_pow_half_special_cases():
    x = np.array([-0.0, 0.0, -np.inf, np.inf, -1e-300, NaN, 0.25])
    r = R.java_pow_half(x)
    assert r[0] == 0.0 and not np.signbit(r[0]) and r[1] == 0.0
    assert r[2] == np.inf and r[3] == np.inf and np.isnan(r[4]) and np.isnan(r[5]) and r[6] == 0.5


def test_reference_reseeds_nan_after_inf():
    """+Inf then -Inf make the reference's running mean NaN; the next finite sample reseeds mean and variance to 0, so the result
    depends on where the infinities arrive.  The device's moment form gives NaN for any infinite input in the group (DESIGN §2)."""
    a = R.leaf(R.STDVAR, np.array([[np.inf], [-np.inf], [1.0], [2.0]])).stat[0]
    b = R.leaf(R.STDVAR, np.array([[1.0], [2.0], [np.inf], [-np.inf]])).stat[0]
    assert not np.isnan(a) and np.isnan(b)
    vals, cnts = R.moment_partials(np.array([[np.inf], [-np.inf], [1.0], [2.0]]), None, 1)
    assert np.isnan(R.present_moments(R.STDVAR, vals[0], vals[1], cnts)).all()


def test_abi_constants():
    hdr = open(os.path.join(ROOT, "include", "filo_b200.h")).read()
    for name, v in (("FILO_AGG_STDDEV", 8), ("FILO_AGG_STDVAR", 9), ("FILO_AGG_GROUP", 10), ("FILO_AGG_BOTTOMK", 7), ("FILO_AGG_SUM", 1)):
        assert re.search(r"\b%s = %d\b" % (name, v), hdr), name
    hpp = open(os.path.join(ROOT, "include", "filo_b200.hpp")).read()
    assert "Stddev = FILO_AGG_STDDEV" in hpp and "Stdvar = FILO_AGG_STDVAR" in hpp and "Group = FILO_AGG_GROUP" in hpp
    from filodb_b200 import capi, shard
    assert (capi.AGG_STDDEV, capi.AGG_STDVAR, capi.AGG_GROUP) == (8, 9, 10) == (shard.AGG_STDDEV, shard.AGG_STDVAR, shard.AGG_GROUP)
    assert (capi.AGG_TOPK, capi.AGG_BOTTOMK) == (6, 7)
    kh = open(os.path.join(ROOT, "filodb_b200", "csrc", "kernels.h")).read()
    assert "AGG_STDDEV = 8, AGG_STDVAR = 9, AGG_GROUP = 10" in kh
    # the JNI shim hands aggrOp to filo_query untouched
    shim = open(os.path.join(ROOT, "filodb_b200", "csrc", "jni_shim.cpp")).read()
    assert re.search(r"filo_query\(C\(ctx\), T\(table\), rangeFn, startMs, stepMs, endMs, windowMs, aggrOp,", shim)


# ---- two-rank merge of moment partials (filodb_b200/shard.py), like tests/test_multi_gpu_gloo.py
T0, STEP, ROWS = 1_700_000_000_000, 15000, 120
N_SERIES, N_GROUPS = 26, 5
QUERY = (T0 + 300000, STEP, T0 + (ROWS - 1) * STEP, 300000)


def _series(i):
    rng = np.random.default_rng(2000 + i)
    ts = T0 + np.arange(ROWS, dtype=np.int64) * STEP
    v = 1e3 + 15 * np.sin(np.arange(1, ROWS + 1)) + rng.normal(0, 1, ROWS)
    v[rng.random(ROWS) < 0.05] = np.nan
    if i % 9 == 4:
        v[:] = np.nan
    return ts, v


def _group(i):
    return 4 if i == 7 else (i * 3 + 1) % 4          # group 4 holds a single series


def _store(o, ids):
    st = o.Store()
    for i in ids:
        ts, v = _series(i)
        st.add_series_rows(ts, v, [80, 40], val_mode=1, detect_drops=False)
    return st


def _worker(rank, world, port, q):
    try:
        import torch
        import torch.distributed as dist
        from filodb_b200 import shard
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        from oracle import oracle as o
        b, e = shard.series_range_of_rank(N_SERIES, rank, world)
        ids = list(range(b, e))
        per = _store(o, ids).query(o.FN_SUM_OVER_TIME, *QUERY)
        vals, cnts = R.moment_partials(per, [_group(i) for i in ids], N_GROUPS)
        res = {}
        for op in (R.STDDEV, R.STDVAR, R.GROUP):
            if op == R.GROUP:                                   # the count partial
                tv, tc = torch.zeros(N_GROUPS * per.shape[1], dtype=torch.float64), torch.from_numpy(cnts.reshape(-1).copy())
            else:
                tv, tc = torch.from_numpy(vals.reshape(-1).copy()), torch.from_numpy(cnts.reshape(-1).copy())
            shard.merge_partials(tv, tc, op, dist)
            c = tc.numpy().reshape(N_GROUPS, -1)
            v = tv.numpy().reshape(-1, N_GROUPS, c.shape[1])
            res[op] = (R.present_moments(op, v[0], v[-1], c), c)
        q.put((rank, res))
        dist.barrier()
        dist.destroy_process_group()
    except Exception as ex:
        q.put((rank, repr(ex)))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.timeout(120)
def test_two_rank_moment_merge_matches_unsharded_reference(oracle):
    import torch.multiprocessing as mp
    o = oracle
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs: p.start()
    got = [q.get(timeout=100) for _ in range(world)]
    for p in procs: p.join(timeout=30)
    for rank, res in got:
        assert not isinstance(res, str), "rank %d failed: %s" % (rank, res)
    per = _store(o, range(N_SERIES)).query(o.FN_SUM_OVER_TIME, *QUERY)
    gids = np.array([_group(i) for i in range(N_SERIES)])
    means = R.group_means(per, gids, N_GROUPS)
    ref_var, ref_cnt = R.aggregate(R.STDVAR, per, gids, N_GROUPS)
    for op in (R.STDDEV, R.STDVAR, R.GROUP):
        exp, cnt = R.aggregate(op, per, gids, N_GROUPS)
        for rank, res in got:
            a, c = res[op]
            assert (c == cnt).all()
            if op == R.GROUP:
                assert (np.isnan(a) == np.isnan(exp)).all() and (a[~np.isnan(a)] == 1.0).all()
            else:
                R.assert_moments_close(op, a, exp, means, ref_var, "rank %d op %d" % (rank, op))


# ---- the moments mode of the scan kernels on the CPU SIMT emulator
def test_moment_kernels_run_on_the_simt_emulator(tmp_path):
    """scan_tile_kernel, scan_wp_ctr_kernel and scan_agg_kernel_v2 in their moments mode, plus merge_partials_kernel and
    present_kernel for stddev / stdvar / group, compiled for the host on the cusim emulator (tests/cpp/moments_emul.cpp): every
    (item, window) Σv, Σv² and count bit-exact against the oracle's per-series rows folded in the item's series order; NaN markers,
    counter resets, multi-tile items, declined items through the v2 kernel; in-order and pseudo-random fiber schedules."""
    src = str(tmp_path / "scan_kernels_cusim.cu")
    subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cpp", "make_cusim_src.py"), os.path.join(ROOT, "filodb_b200", "csrc", "scan_kernels.cu"), src], check=True)
    exe = str(tmp_path / "moments_emul")
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", "-I", "/usr/local/cuda/include",
                    "-I", os.path.join(ROOT, "filodb_b200", "csrc"), '-DSCAN_SRC="%s"' % src,
                    os.path.join(ROOT, "tests", "cpp", "moments_emul.cpp"), "-o", exe], check=True)
    for seed in ("0", "20261016"):
        out = subprocess.run([exe, seed], check=True, capture_output=True, text=True).stdout
        assert "OK 12 cases" in out and "bit-exact" in out, out
