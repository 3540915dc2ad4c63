"""GPU: topk / bottomk across GPUs.  W tables cut from one series set (contiguous ranges or the modulo shard map), each queried with
filo_query_device into torch buffers on a non-default stream without stats, the ids mapped to global ordinals (shard.topk_ids_to_global),
then filo_merge_topk_partials: bitwise equal, values and ids, to filo_query topk / bottomk over the whole table, and matching the oracle
under the checks test_gpu_parity.py applies to topk."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
T0, STEP, ROWS = 1_700_000_000_000, 15000, 240
S, G = 60, 5                                   # group G - 1 has no series; the others about 15 series each (fewer than k = 32)
Q = (T0 + 300000, STEP, T0 + (ROWS - 1) * STEP, 300000)


def same_bits(a, b):
    a = np.ascontiguousarray(a, np.float64); b = np.ascontiguousarray(b, np.float64)
    an, bn = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and (an == bn).all() and (a[~an].view(np.uint64) == b[~bn].view(np.uint64)).all()


@pytest.fixture(scope="module")
def gpu():
    import torch
    import filodb_b200.capi as capi
    ctx = capi.Context(0)
    yield capi, ctx, torch
    ctx.close()


# name: (range function, cumulative, value encoding, timestamp jitter, values)
CASES = {
    "xor_gauge_sum": ("FN_SUM_OVER_TIME", False, "VAL_XOR", 0, "ints"),          # SUM class on XOR doubles: the v4 SUM kernel
    "counter_rate": ("FN_RATE", True, "VAL_OPTIMIZE", 0, "counter"),
    "irregular_avg": ("FN_AVG_OVER_TIME", False, "VAL_XOR", 2000, "ints"),         # jittered timestamps: declined to the v2 kernel
    "signed_zero_last": ("FN_LAST", False, "VAL_XOR", 0, "zeros"),                 # ties of +0.0 and -0.0 at the cut
}


def _series_set(o, kind, jitter, val_mode, cumulative):
    rng = np.random.default_rng(77)
    st = o.Store()
    for s in range(S):
        ts = T0 + np.arange(ROWS, dtype=np.int64) * STEP
        if jitter:
            ts = ts + rng.integers(-jitter, jitter + 1, ROWS)
        if kind == "counter":
            v = np.cumsum(rng.integers(0, 4, ROWS)).astype(np.float64)
            if s % 7 == 2:
                v[150:] -= v[150]                                        # a reset
        elif kind == "zeros":
            v = rng.choice([0.0, -0.0, 1.0, -1.0], ROWS)
        else:
            v = rng.integers(-3, 4, ROWS).astype(np.float64)
            v[rng.random(ROWS) < 0.05] = np.nan
        if s == 9:
            v[:] = np.nan                                                # a series without a value
        st.add_series_rows(ts, v, [120, 120], val_mode=getattr(o, val_mode), detect_drops=cumulative)
    return st


def _gids():
    return np.array([(s * 7 + 3) % (G - 1) for s in range(S)], np.int32)


def _subset(nch, addrs, ids):
    off = np.concatenate([[0], np.cumsum(nch)])
    return nch[ids], np.concatenate([addrs[off[i]:off[i + 1]] for i in ids]) if len(ids) else np.zeros(1, np.uint64)


def _parity_with_oracle(gv, gi, ev, ei, per, gids, what):
    """test_gpu_parity.py's topk checks: the oracle's values bit for bit, the same empty slots, and each id names a series of the cell's
    group whose window value is the slot's value."""
    assert same_bits(gv, ev), what
    ok = gi >= 0
    assert (ok == (ei >= 0)).all(), what
    for g, t, j in zip(*np.nonzero(ok)):
        assert gids[gi[g, t, j]] == g and same_bits(per[gi[g, t, j], t], gv[g, t, j]), what


@pytest.mark.parametrize("split", ["contiguous", "modulo"])
@pytest.mark.parametrize("case", list(CASES))
def test_merged_topk_partials_equal_the_whole_table(gpu, oracle, case, split):
    capi, ctx, torch = gpu
    from filodb_b200 import shard
    o = oracle
    fn_name, cumulative, val_mode, jitter, kind = CASES[case]
    fn = getattr(capi, fn_name)
    flags = capi.SCHEMA_CUMULATIVE if cumulative else 0
    st = _series_set(o, kind, jitter, val_mode, cumulative)
    gids = _gids()
    nch, addrs = st.all_info_addrs()
    T = capi.num_windows(Q[0], Q[1], Q[2])
    whole = ctx.load_series(nch, addrs, group_ids=gids, n_groups=G, schema_flags=flags)
    per = st.query(getattr(o, fn_name), *Q, cumulative=cumulative)
    stream = torch.cuda.Stream()
    ties = 0
    try:
        for W in (2, 3, 8):
            ids = [list(range(*shard.series_range_of_rank(S, r, W))) if split == "contiguous" else list(range(r, S, W)) for r in range(W)]
            tabs = [ctx.load_series(*_subset(nch, addrs, i), group_ids=gids[i], n_groups=G, schema_flags=flags) for i in ids]
            tables = [torch.tensor(i, dtype=torch.int64, device="cuda") for i in ids]
            try:
                for k in (1, 5, 32):
                    for aggr in (capi.AGG_TOPK, capi.AGG_BOTTOMK):
                        what = "%s %s W=%d k=%d aggr %d" % (case, split, W, k, aggr)
                        pv = torch.full((W, G, T, k), -7.0, dtype=torch.float64, device="cuda")
                        pi = torch.full((W, G, T, k), -7, dtype=torch.int64, device="cuda")
                        mv = torch.full((G, T, k), -7.0, dtype=torch.float64, device="cuda")
                        mi = torch.full((G, T, k), -7, dtype=torch.int64, device="cuda")
                        torch.cuda.synchronize()          # the fills are done before the other stream writes the buffers
                        with torch.cuda.stream(stream):
                            for r, t in enumerate(tabs):
                                ctx.query_device(t, fn, *Q, pv[r].data_ptr(), pi[r].data_ptr(), aggr=aggr, k=k, stream=stream.cuda_stream, want_stats=False)
                                pi[r] = shard.topk_ids_to_global(pi[r], tables[r])
                            ctx.merge_topk_partials(aggr, k, W, G, T, pv.data_ptr(), pi.data_ptr(), mv.data_ptr(), mi.data_ptr(), stream=stream.cuda_stream)
                        ctx.check()
                        stream.synchronize()
                        gv, gi = mv.cpu().numpy(), mi.cpu().numpy()
                        wv, wi = ctx.query(whole, fn, *Q, aggr=aggr, k=k)
                        assert same_bits(gv, wv) and (gi == wi).all(), what
                        ev, ei = st.query(getattr(o, fn_name), *Q, cumulative=cumulative, aggr=getattr(o, "AGG_TOPK" if aggr == capi.AGG_TOPK else "AGG_BOTTOMK"),
                                          k=k, group_ids=gids, n_groups=G)
                        _parity_with_oracle(gv, gi, ev, ei, per, gids, what)
                        assert (gi[G - 1] == -1).all(), what
                        # the tie rule decides: a kept value equal to one of a series left out of the cell
                        for g in range(G - 1):
                            for t in range(T):
                                if gi[g, t, 0] >= 0:
                                    col = per[gids == g, t]
                                    ties += int((col == gv[g, t, 0]).sum() > (gv[g, t][gi[g, t] >= 0] == gv[g, t, 0]).sum())
            finally:
                for t in tabs:
                    t.free()
    finally:
        whole.free()
    if case in ("xor_gauge_sum", "signed_zero_last"):
        assert ties > 0


def test_merge_of_one_part_is_the_query(gpu, oracle):
    """W = 1: the merge reproduces filo_query's topk / bottomk cell for cell."""
    capi, ctx, torch = gpu
    st = _series_set(oracle, "ints", 0, "VAL_XOR", False)
    tab = ctx.load_series(*st.all_info_addrs(), group_ids=_gids(), n_groups=G)
    T = capi.num_windows(Q[0], Q[1], Q[2])
    try:
        for aggr in (capi.AGG_TOPK, capi.AGG_BOTTOMK):
            wv, wi = ctx.query(tab, capi.FN_MAX_OVER_TIME, *Q, aggr=aggr, k=4)
            pv = torch.tensor(wv, device="cuda")[None]; pi = torch.tensor(wi, device="cuda")[None]
            mv = torch.empty_like(pv[0]); mi = torch.empty_like(pi[0])
            ctx.merge_topk_partials(aggr, 4, 1, G, T, pv.data_ptr(), pi.data_ptr(), mv.data_ptr(), mi.data_ptr())
            torch.cuda.synchronize()
            assert same_bits(mv.cpu().numpy(), wv) and (mi.cpu().numpy() == wi).all()
    finally:
        tab.free()


def test_error_paths(gpu):
    capi, ctx, torch = gpu
    v = torch.zeros((2, 3, 4, 5), dtype=torch.float64, device="cuda")
    i = torch.full((2, 3, 4, 5), -1, dtype=torch.int64, device="cuda")
    ov, oi = v[0].clone(), i[0].clone()
    p = (v.data_ptr(), i.data_ptr(), ov.data_ptr(), oi.data_ptr())

    def code(aggr, k, n_parts, n_groups, n_windows, ptrs):
        with pytest.raises(capi.FiloError) as ei:
            ctx.merge_topk_partials(aggr, k, n_parts, n_groups, n_windows, *ptrs)
        return ei.value.code

    for aggr in (capi.AGG_SUM, capi.AGG_MAX, capi.AGG_NONE, 99):
        assert code(aggr, 5, 2, 3, 4, p) == capi.ERR_INVALID_ARG
    for k in (0, 33, -1):
        assert code(capi.AGG_TOPK, k, 2, 3, 4, p) == capi.ERR_INVALID_ARG
    assert code(capi.AGG_TOPK, 5, 0, 3, 4, p) == capi.ERR_INVALID_ARG
    assert code(capi.AGG_BOTTOMK, 5, 2, 0, 4, p) == capi.ERR_INVALID_ARG
    assert code(capi.AGG_TOPK, 5, 2, 3, 0, p) == capi.ERR_INVALID_ARG
    for n in range(4):
        assert code(capi.AGG_TOPK, 5, 2, 3, 4, tuple(0 if j == n else x for j, x in enumerate(p))) == capi.ERR_INVALID_ARG
    ctx.merge_topk_partials(capi.AGG_BOTTOMK, 5, 2, 3, 4, *p)             # every slot empty: the output is padding
    torch.cuda.synchronize()
    ctx.check()
    assert (oi == -1).all() and (ov == np.finfo(np.float64).max).all()
