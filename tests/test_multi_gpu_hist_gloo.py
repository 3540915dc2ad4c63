"""World-2 and world-3 CPU tests (gloo) of the cross-GPU histogram sum: every rank's HistSumRowAggregator partial over its series is
gathered in rank order by shard.gather_hist_partials, and the rank-order fold of the gathered partials (the reduceAggregate restatement
of tests/hist_series_ref.py, the fold filo_merge_hist_partials runs on the device) agrees with the oracle over the unsharded series."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from filodb_b200 import shard
from tests import hist_series_ref as R

T0, STEP, ROWS = 1_700_000_000_000, 15000, 120
N_SERIES, N_GROUPS, NB = 11, 5, 10                  # group 4 has no series: empty on every rank
QUERY = (T0 + 300000, STEP, T0 + (ROWS - 1) * STEP, 300000)
QTL = 0.9


def _group(i):
    return 3 if i == 5 else i % 3                   # series 5 alone in group 3: its cells are empty on every other rank


def _buckets(H):
    return H.Buckets.custom([2.0 * 3 ** i for i in range(NB - 1)] + [float("inf")])


def _store(H, ids):
    """Cumulative bucket counts over a large base (every window's rate is extrapolated without the zero-point clamp, so the per-series
    rates are monotonic and the sharded fold differs from the unsharded one by rounding only); series 5 starts late."""
    st = H.HistStore(_buckets(H))
    for i in ids:
        rng = np.random.default_rng(500 + i)
        ts = T0 + np.arange(ROWS, dtype=np.int64) * STEP + (900000 if i == 5 else 0)
        inc = np.cumsum(rng.integers(0, 20, (ROWS, NB)), axis=1)
        st.add_series(ts, 1_000_000 + np.cumsum(inc, axis=0).astype(np.int64), [80, 40])
    return st


def _partial(o, H, ids):
    """HistSumRowAggregator over `ids` by group: [G, T, nb], NaN buckets where a group has no histogram (the SUM output's form)."""
    vals, empty, _ = _store(H, ids).query(o.FN_RATE, *QUERY, aggr=True, group_ids=[_group(i) for i in ids], n_groups=N_GROUPS)
    vals = vals.copy(); vals[empty] = np.nan
    return vals


def _worker(rank, world, port, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        from oracle import hist as H
        from oracle import oracle as o
        b, e = shard.series_range_of_rank(N_SERIES, rank, world)
        part = _partial(o, H, range(b, e))
        gathered = shard.gather_hist_partials(torch.from_numpy(part), dist)
        q.put((rank, part, gathered.numpy().copy()))
        dist.barrier()
        dist.destroy_process_group()
    except Exception as ex:            # surface the failure in the parent instead of hanging it
        q.put((rank, repr(ex), None))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def same_bits(a, b):
    an, bn = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and (an == bn).all() and (a[~an].view(np.uint64) == b[~bn].view(np.uint64)).all()


@pytest.mark.timeout(180)
@pytest.mark.parametrize("world", [2, 3])
def test_gathered_hist_partials_fold_to_the_unsharded_sum(oracle, world):
    o = oracle
    from oracle import hist as H
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs: p.start()
    got = sorted([q.get(timeout=150) for _ in range(world)], key=lambda x: x[0])
    for p in procs: p.join(timeout=30)
    for rank, part, _ in got:
        assert not isinstance(part, str), "rank %d failed: %s" % (rank, part)
    parts = [part for _, part, _ in got]
    for rank, _, gathered in got:
        assert gathered.shape == (world,) + parts[0].shape
        for r in range(world):
            assert same_bits(gathered[r], parts[r]), "rank %d: gathered[%d] differs from rank %d's partial" % (rank, r, r)
    gathered = got[0][2]
    # ReduceAggregateExec: rows = the gathered partials in rank order, empty = their all-NaN cells
    rows = gathered.reshape(world * N_GROUPS, -1, NB)
    empty = np.isnan(rows).all(axis=2)
    assert (empty == np.isnan(rows[:, :, 0])).all()                  # all-NaN exactly where bucket 0 is NaN
    acc, aempty = R.hist_sum(NB, rows, empty, np.tile(np.arange(N_GROUPS), world), N_GROUPS)
    assert aempty[N_GROUPS - 1].all()                                   # the group without series stays empty
    e = np.isnan(gathered[..., 0])
    assert (e.any(axis=0) & ~e.all(axis=0)).any()                      # cells empty on some ranks and not on others
    exp, eempty, eq = _store(H, range(N_SERIES)).query(o.FN_RATE, *QUERY, aggr=True, group_ids=[_group(i) for i in range(N_SERIES)], n_groups=N_GROUPS, q=QTL)
    assert (aempty == eempty).all()
    np.testing.assert_allclose(acc[~aempty], exp[~eempty], rtol=1e-9, atol=0)
    qs = R.quantiles(_buckets(H), acc, aempty, QTL)
    eq = np.where(eempty, np.nan, eq)
    assert (np.isnan(qs) == np.isnan(eq)).all()
    np.testing.assert_allclose(qs[~np.isnan(eq)], eq[~np.isnan(eq)], rtol=1e-9, atol=0)
