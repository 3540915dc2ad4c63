"""World-2 and world-3 CPU tests (gloo) of topk / bottomk across GPUs: every rank's candidates over its series (the oracle, with its
series split contiguously or by the modulo shard map), mapped to global ordinals by shard.topk_ids_to_global and gathered in rank order
by shard.gather_topk_partials; a numpy restatement of the merge rule filo_merge_topk_partials runs on the device (k best by value, ties to
the smaller global ordinal, written worst first) over the gathered tensors equals the oracle's unsharded topk / bottomk bit for bit."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from filodb_b200 import shard

T0, STEP, ROWS = 1_700_000_000_000, 15000, 120
N_SERIES, N_GROUPS, K = 23, 4, 3                   # group 3 has no series: empty on every rank
QUERY = (T0 + 300000, STEP, T0 + (ROWS - 1) * STEP, 300000)
QUERY_T = (QUERY[2] - QUERY[0]) // QUERY[1] + 1
PAD = np.finfo(np.float64).max


def _series(i):
    """Integer values in [-2, 2] with zeros of both signs (heavy ties at the cut), NaN at random; series 4 only NaN."""
    rng = np.random.default_rng(2000 + i)
    ts = T0 + np.arange(ROWS, dtype=np.int64) * STEP
    v = rng.integers(-2, 3, ROWS).astype(np.float64)
    v[rng.random(ROWS) < 0.3] = -0.0
    v[rng.random(ROWS) < 0.1] = np.nan
    if i == 4:
        v[:] = np.nan
    return ts, v


def _group(i):
    return (i * 5 + 1) % (N_GROUPS - 1)


def _ids_of_rank(split, rank, world, n_series):
    return list(range(*shard.series_range_of_rank(n_series, rank, world))) if split == "contiguous" else list(range(rank, n_series, world))


def _candidates(o, ids, aggr):
    """The oracle's topk / bottomk over `ids` (ids: ordinals among them), what filo_query_device writes for that table."""
    st = o.Store()
    for i in ids:
        st.add_series_rows(*_series(i), [80, 40], val_mode=1, detect_drops=False)
    return st.query(o.FN_LAST, *QUERY, aggr=aggr, k=K, group_ids=[_group(i) for i in ids], n_groups=N_GROUPS)


def _worker(rank, world, port, split, n_series, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        from oracle import oracle as o
        ids = _ids_of_rank(split, rank, world, n_series)
        res = {}
        for aggr in (o.AGG_TOPK, o.AGG_BOTTOMK):
            v, local = _candidates(o, ids, aggr)
            glob = shard.topk_ids_to_global(torch.from_numpy(local), torch.tensor(ids, dtype=torch.int64))
            gv, gi = shard.gather_topk_partials(torch.from_numpy(v), glob, dist)
            res[aggr] = (v, glob.numpy().copy(), gv.numpy().copy(), gi.numpy().copy())
        q.put((rank, res))
        dist.barrier()
        dist.destroy_process_group()
    except Exception as ex:            # surface the failure in the parent instead of hanging it
        q.put((rank, repr(ex)))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def same_bits(a, b):
    return a.shape == b.shape and (a.view(np.uint64) == b.view(np.uint64)).all()


def merge_rule(values, ids, bottom):
    """filo_merge_topk_partials restated: per cell the k best non-empty (id >= 0, value not NaN) candidates of all parts, better = larger value for
    topk and smaller for bottomk, values compared with == (+0.0 ties -0.0), equal values ordered by the smaller id; written worst first,
    padded with -DBL_MAX / +DBL_MAX and id -1."""
    W, G, T, k = values.shape
    out_v = np.full((G, T, k), PAD if bottom else -PAD); out_i = np.full((G, T, k), -1, np.int64)
    for g in range(G):
        for t in range(T):
            c = [(values[p, g, t, j], int(ids[p, g, t, j])) for p in range(W) for j in range(k)
                 if ids[p, g, t, j] >= 0 and values[p, g, t, j] == values[p, g, t, j]]
            c.sort(key=lambda x: (x[0] if bottom else -x[0], x[1]))
            best = c[:k][::-1]
            for j, (v, i) in enumerate(best):
                out_v[g, t, j] = v; out_i[g, t, j] = i
    return out_v, out_i


def test_topk_ids_to_global_keeps_empty_slots():
    ids = torch.tensor([[2, 0, -1], [-1, -1, 1]], dtype=torch.int64)
    got = shard.topk_ids_to_global(ids, torch.tensor([5, 9, 17], dtype=torch.int64))
    assert got.tolist() == [[17, 5, -1], [-1, -1, 9]]
    empty = torch.full((2, 3), -1, dtype=torch.int64)                  # a rank whose table holds no series
    assert shard.topk_ids_to_global(empty, torch.zeros(0, dtype=torch.int64)).tolist() == empty.tolist()


def _run_world(o, world, split, n_series):
    """Every rank's candidates, gathered; checks that each rank holds every rank's tensors in rank order and that the merge rule over them
    gives the oracle's unsharded topk / bottomk.  Returns the number of cells where the tie rule decides."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, split, n_series, q)) for r in range(world)]
    for p in procs: p.start()
    got = sorted([q.get(timeout=150) for _ in range(world)], key=lambda x: x[0])
    for p in procs: p.join(timeout=30)
    for rank, res in got:
        assert not isinstance(res, str), "rank %d failed: %s" % (rank, res)
    all_ids = list(range(n_series))
    ties = 0
    for aggr in (o.AGG_TOPK, o.AGG_BOTTOMK):
        for rank, res in got:
            gv, gi = res[aggr][2], res[aggr][3]
            assert gv.shape == (world, N_GROUPS, QUERY_T, K) and gi.shape == gv.shape
            for r in range(world):
                assert same_bits(gv[r], got[r][1][aggr][0]), "rank %d: gathered values[%d] differ from rank %d's" % (rank, r, r)
                assert (gi[r] == got[r][1][aggr][1]).all(), "rank %d: gathered ids[%d] differ from rank %d's" % (rank, r, r)
        gv, gi = got[0][1][aggr][2], got[0][1][aggr][3]
        assert (gi[:, N_GROUPS - 1] == -1).all()                               # the group without series is empty everywhere
        mv, mi = merge_rule(gv, gi, aggr == o.AGG_BOTTOMK)
        ev, ei = _candidates(o, all_ids, aggr)
        assert same_bits(mv, ev) and (mi == ei).all(), "world %d %s aggr %d" % (world, split, aggr)
        # the rule decides somewhere: cells where a window's last samples hold the cut value more often than the kept slots do
        for g in range(N_GROUPS - 1):
            for t in range(QUERY_T):
                if ei[g, t, 0] < 0:
                    continue
                col = np.array([_series(i)[1][t + 20] for i in all_ids if _group(i) == g])
                ties += int((col == ev[g, t, 0]).sum() > (ev[g, t][ei[g, t] >= 0] == ev[g, t, 0]).sum())
    return ties


@pytest.mark.timeout(180)
@pytest.mark.parametrize("split", ["contiguous", "modulo"])
@pytest.mark.parametrize("world", [2, 3])
def test_gathered_topk_candidates_merge_to_the_unsharded_topk(oracle, world, split):
    assert _run_world(oracle, world, split, N_SERIES) > 0


@pytest.mark.timeout(180)
def test_a_rank_without_series(oracle):
    """World 3 over 2 series split contiguously: rank 2's table holds no series, its candidates are all empty slots."""
    assert _ids_of_rank("contiguous", 2, 3, 2) == []
    _run_world(oracle, 3, "contiguous", 2)

