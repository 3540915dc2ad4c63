"""GPU: the fused aggregate kernels at steady state, where work items hold many series and every warp (counter kernel) or CTA (tile
kernel) folds several items.  Tables are sized from the device's SM count, S = seg * SMs * 256 + r, so that build_groups_new gives items
of `seg` series (tests/fused_items.py restates the layout); before any comparison each query asserts filo_query's fused choice, grid,
seg and items per warp (scan_path, through tests/cpp/scan_path.cpp on the table's real record bytes).

Tables: counters (scan_wp_ctr_kernel<AGG>: rate / increase / delta) with const-DDV timestamps, and again with one jittered series (the
IRR instantiation); integer-valued gauges (scan_tile_kernel<AGG>: sum / count_over_time) at a seg that is not a multiple of 8 (a partial
last tile) and at one that is.  One table holds groups of 1, seg - 1, seg, seg + 1, 8 seg and 8 seg + 1 series, one of about 40 % of
the series, an empty one and about 2,000 of mixed sizes, with ids interleaved at random; the ungrouped form (order == nullptr) runs too.
Series that decline (five chunks in range, a DDV value chunk, more than eight resets in one chunk, jittered timestamps on the tile kernel)
sit at an item's first, middle and last series, twice in one item, in every series of an item, at the first series a warp takes, in a
warp's last item, in two consecutive items of one warp, in the only item of a small group and in every item of one group.

Every table is a few dozen distinct prototype series repeated, so references are folds of the oracle's prototype rows weighted by how
often each appears in a group; none depends on the device's fold order.  Integer gauges: sum / count / group / min / max bit-exact (and
sum against the oracle's own aggregate), avg = exact sum / count.  Counters: |gpu - ref| <= gamma_{m-1} * sum |v| with an extended
precision reference, on data whose smallest |v| per cell is 1e3 times the bound; min / max / count bit-exact.  stddev / stdvar through
agg_moments_ref; the partial form presented on the device bit for bit; topk / bottomk values and series ids; the scan counters on every
query.  Queries at T = 512 (the last the fused kernels take) and T = 513 (the v2 aggregate kernel alone) too."""
import os
import time
import zlib

import numpy as np
import pytest

from tests.fused_items import Items, seg_for
from tests.test_gpu_agg_moments import check_moments
from tests.test_gpu_parity import same_bits
from tests.test_gpu_steady_state import table_shape
from tests.test_gpu_value_edges import check_partial_present_plain
from tests.test_scan_path import build_scan_path, scan_path

pytestmark = pytest.mark.gpu
T0, STEP, ROWS = 1_700_000_000_000, 15000, 120
U = 2.0 ** -53
# (T, first window's end row, window in steps)
QUERIES = [(80, 40, 20), (512, 20, 20), (513, 20, 20)]     # every one reaches all five chunks of a five-chunk series
TABLES = {
    "ctr const-DDV": dict(counter=True, seg=9, jitter=False, kernel="ctr"),
    "ctr IRR": dict(counter=True, seg=9, jitter=True, kernel="ctr"),
    "tile seg 9": dict(counter=False, seg=9, jitter=False, kernel="tile"),
    "tile seg 8": dict(counter=False, seg=8, jitter=False, kernel="tile"),
}
N_REG = 24                                   # regular prototypes


def proto_chunks(rng, counter, cause):
    """(ts, values, val_mode, rows per chunk) of one prototype.  Counters: increments in [lo, lo + 10) with lo in [10, 100) per series, so
    rates are within a factor of ten of each other (the sum bound needs that) and spread widely enough that a group's variance is not
    lost to cancellation in Σv² / n - mean² (one reset in some series); gauges: integers in [0, 40)."""
    import oracle.oracle as o
    ts = T0 + np.arange(ROWS, dtype=np.int64) * STEP
    if cause == "jitter":
        ts = ts + rng.integers(-2000, 2001, ROWS)
    if counter:
        lo = rng.uniform(10, 100)
        inc = rng.uniform(lo, lo + 10, ROWS)
        if cause == "resets":                # a reset every 5 rows of chunk 0: 12 drops where the list holds 8
            v = np.cumsum(inc)
            for r in range(5, 70, 5): v[r:] -= v[r] - inc[r]
        else:
            v = 1e4 + np.cumsum(inc)
            if rng.random() < 0.3: r = int(rng.integers(10, ROWS)); v[r:] -= v[r] - inc[r]
        if cause == "ddv": v = np.round(v)
    else:
        v = rng.integers(0, 40, ROWS).astype(np.float64)
    split = [24] * 5 if cause == "chunks5" else [70, 50]
    mode = o.VAL_OPTIMIZE if cause == "ddv" else o.VAL_XOR      # the last chunk's integral values through optimize(): a DDV vector
    return ts, v, mode, split


def add_proto(st, rng, counter, cause):
    import oracle.oracle as o
    ts, v, mode, split = proto_chunks(rng, counter, cause)
    s = st.add_series()
    c0 = 0
    for i, n in enumerate(split):
        st.add_chunk(s, ts[c0:c0 + n], v[c0:c0 + n], val_mode=mode if i == len(split) - 1 else o.VAL_XOR, detect_drops=counter)
        c0 += n


def group_layout(rng, S, seg):
    sizes = [1, seg - 1, seg, seg + 1, 8 * seg, 8 * seg + 1, 0, int(0.4 * S)]
    rest = S - sum(sizes)
    mixed = rng.integers(1, 2 * rest // 2000, 2000)
    mixed = np.maximum(1, (mixed * rest / mixed.sum()).astype(np.int64))
    mixed[-1] += rest - mixed.sum()
    assert mixed[-1] > 0
    sizes = np.concatenate([sizes, mixed]).astype(np.int64)
    G = sizes.size
    groups = np.repeat(np.arange(G, dtype=np.int32), sizes)
    return groups[rng.permutation(S)], G


def plant(items, workers):
    """Positions in `order` of the declining series."""
    ib, n = items.item_begin, items.n_items
    sz = np.diff(ib)
    big = np.nonzero(sz >= 3)[0]
    pos = [ib[big[0]], (ib[big[1]] + ib[big[1] + 1]) // 2, ib[big[2] + 1] - 1, ib[big[3]], ib[big[3] + 1] - 1]
    it = big[len(big) // 2]; pos += list(range(ib[it], ib[it + 1]))                       # every series of an item
    pos.append(ib[1 % workers])                                                          # the first series warp 1 takes
    w = workers - 1; last = w + ((n - 1 - w) // workers) * workers; pos.append(ib[last + 1] - 1)   # a warp's last item
    it = 2 * workers + 1; pos += [ib[it], ib[it + workers] + sz[it + workers] // 2]      # items it, it + workers of one warp
    one = np.nonzero(np.diff(items.group_start) == 1)[0][0]; pos.append(items.group_start[one])     # the only item of a group of one
    g = int(np.argmax((np.diff(items.gis) >= 3) & (np.diff(items.gis) <= 40)))          # every item of one group
    for it in range(items.gis[g], items.gis[g + 1]): pos.append(ib[it] + (it % 3) * (sz[it] - 1) // 2)
    return np.unique(np.array(pos, np.int64))


@pytest.fixture(scope="module")
def env(tmp_path_factory, oracle):
    import torch
    import filodb_b200.capi as capi
    exe = build_scan_path(tmp_path_factory.mktemp("scan_path"))
    ctx = capi.Context(0)
    props = torch.cuda.get_device_properties(0)
    sms = props.multi_processor_count
    smem = min(props.shared_memory_per_block_optin, 227 * 1024)
    t_start = time.time()
    e = dict(capi=capi, ctx=ctx, exe=exe, sms=sms, smem=smem, o=oracle, tables={}, refs={})
    yield e
    for tb in e["tables"].values(): tb["tab"].free()
    ctx.close()
    print("\ntest_gpu_fused_steady_state: %.1f s" % (time.time() - t_start))


def get_table(env, name):
    """Built once per module: (table, prototype store, prototype of every series, groups, G, items, proto shape)."""
    if name in env["tables"]:
        return env["tables"][name]
    capi, ctx, o, sms = env["capi"], env["ctx"], env["o"], env["sms"]
    t = TABLES[name]
    seg = t["seg"]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    S = seg * sms * 256 + 37
    assert seg_for(S, sms) == seg
    groups, G = group_layout(rng, S, seg)
    items = Items(groups, G, seg)
    causes = ["chunks5", "ddv", "resets"] if t["counter"] else ["jitter", "ddv", "chunks5"]
    st = o.Store()
    for _ in range(N_REG): add_proto(st, rng, t["counter"], None)
    for c in causes: add_proto(st, rng, t["counter"], c)
    if t["jitter"]: add_proto(st, rng, True, "jitter")           # a jittered series the counter kernel's IRR instantiation takes
    P = st.num_series
    pid = rng.integers(0, N_REG, S)
    # the warps (ctr) or CTAs (tile) the items are strided over, from the choice for the prototypes' shape
    small = ctx.load_series(*st.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE if t["counter"] else 0)
    rec, rows, chunks, irr = table_shape(small); small.free()
    p = scan_path(env["exe"], rec=rec, rows=rows, chunks=chunks, T=80, wrows=21, n=S, cls="counter" if t["counter"] else "sum", fused=1, irr=int(irr),
                  items=items.n_items, sms=sms, smem=env["smem"])
    workers = p["fused_grid"] * (p["warps"] if t["kernel"] == "ctr" else 1)
    planted = items.order[plant(items, workers)]
    pid[planted] = N_REG + np.arange(planted.size) % len(causes)
    if t["jitter"]: pid[items.order[items.item_begin[5]]] = P - 1
    nch = np.array([st.num_chunks(i) for i in range(P)], np.int32)
    addr = [st.info_addrs(i) for i in range(P)]
    tab = ctx.load_series(nch[pid], np.concatenate([addr[i] for i in pid]), group_ids=groups, n_groups=G,
                          schema_flags=capi.SCHEMA_CUMULATIVE if t["counter"] else 0)
    C = np.zeros((G, P), np.int64)
    np.add.at(C, (groups, pid), 1)
    out = dict(tab=tab, st=st, pid=pid, groups=groups, G=G, items=items, C=C, S=S, P=P, n_planted=planted.size)
    env["tables"][name] = out
    return out


def proto_rows(env, tb, fn_name, q, counter):
    key = (id(tb["st"]), fn_name, q)
    if key not in env["refs"]:
        o = env["o"]
        rows = tb["st"].query(getattr(o, fn_name), *q, cumulative=counter)
        stats = np.zeros((tb["P"], 2), np.int64)
        for p in range(tb["P"]):
            tb["st"].query(getattr(o, fn_name), *q, cumulative=counter, series_begin=p, series_end=p + 1)
            stats[p] = tb["st"].last_stats["samples_scanned"], tb["st"].last_stats["bytes_scanned"]
        n_per = np.bincount(tb["pid"], minlength=tb["P"])
        env["refs"][key] = (rows, tuple(int(x) for x in n_per @ stats))
    return env["refs"][key]


def query_of(T, first, w):
    start = T0 + first * STEP
    return (start, STEP, start + (T - 1) * STEP, w * STEP)


@pytest.fixture(params=["v4", "v3", "v2", "v1"])
def gen(request):
    """v4: the default selection; v3: the tile kernel for the SUM class, the v2 kernel for counters; v2 / v1: the v2 / v1 aggregate
    kernels alone."""
    if request.param == "v4": os.environ.pop("FILO_KERNEL", None)
    else: os.environ["FILO_KERNEL"] = request.param
    yield request.param
    os.environ.pop("FILO_KERNEL", None)


def check_path(env, t, tb, T, gen):
    rec, rows, chunks, irr = table_shape(tb["tab"])
    assert irr == (t["jitter"] or not t["counter"])             # the tile table's jittered series decline; the counter kernel takes them
    p = scan_path(env["exe"], rec=rec, rows=rows, chunks=chunks, T=T, wrows=21, n=tb["S"], cls="counter" if t["counter"] else "sum", fused=1, irr=int(irr),
                  items=tb["items"].n_items, sms=env["sms"], smem=env["smem"])
    what = "%s T=%d: %s" % (t, T, p)
    if T > 512:
        assert p["fused_kernel"] == "v2", what
        return
    assert p["fused_kernel"] == t["kernel"], what
    assert p["fused_grid"] in ((env["sms"],) if t["kernel"] == "ctr" else (env["sms"], 2 * env["sms"])), what
    assert p["items_per_warp"] >= 3, what
    assert tb["items"].seg == t["seg"] and tb["items"].n_items == int(np.ceil(np.bincount(tb["groups"], minlength=tb["G"]) / t["seg"]).sum()), what
    if gen == "v4": print("%s T=%d: %s, grid %d, seg %d, %d items, >= %d items per %s" % (t["kernel"], T, p["fused_kernel"], p["fused_grid"], t["seg"],
                                                                                    tb["items"].n_items, p["items_per_warp"], "warp" if t["kernel"] == "ctr" else "CTA"))


def sums(C, rows):
    """Extended-precision Σv, Σ|v| and counts per (group, window) from prototype rows and group multiplicities."""
    ok = ~np.isnan(rows)
    r = np.where(ok, rows, 0.0).astype(np.longdouble)
    Cl = C.astype(np.longdouble)
    return Cl @ r, Cl @ np.abs(r), C @ ok.astype(np.int64)


def fold_minmax(C, rows, op_min):
    acc = np.full((C.shape[0], rows.shape[1]), np.nan)
    for p in range(C.shape[1]):
        m = C[:, p] > 0
        acc[m] = (np.fmin if op_min else np.fmax)(acc[m], rows[p])
    return acc


def topk_best(env, tb, key, rows, bottom, kmax=32):
    """Per (group, window) the kmax best non-NaN values best first and their series ids; ties keep the lower series id (the device
    scans a group's series in ascending id).  Cached per table, function and query."""
    ck = ("topk",) + key + (bottom,)
    if ck in env["refs"]:
        return env["refs"][ck]
    G, T = tb["G"], rows.shape[1]
    val = np.full((G, T, kmax), np.nan); ids = np.full((G, T, kmax), -1, np.int64); ngood = np.zeros((G, T), np.int64)
    order, gs, pid = tb["items"].order, tb["items"].group_start, tb["pid"]
    for g in range(G):
        mem = order[gs[g]:gs[g + 1]]
        if mem.size == 0: continue
        v = rows[pid[mem]]                                       # [m, T], members in ascending id
        keyv = np.where(np.isnan(v), np.inf, v if bottom else -v)
        best = np.argsort(keyv, axis=0, kind="stable")[:kmax]    # [<= kmax, T]
        ngood[g] = np.minimum((~np.isnan(v)).sum(axis=0), kmax)
        val[g, :, :best.shape[0]] = v[best, np.arange(T)].T
        ids[g, :, :best.shape[0]] = mem[best].T
    env["refs"][ck] = (val, ids, ngood)
    return env["refs"][ck]


def topk_expected(best, k, bottom):
    """topk_kernel's output: the kept values worst first, then (+-DBL_MAX, -1)."""
    val, ids, ngood = best
    G, T, _ = val.shape
    ev = np.full((G, T, k), np.finfo(np.float64).max if bottom else -np.finfo(np.float64).max); ei = np.full((G, T, k), -1, np.int64)
    n = np.minimum(ngood, k)
    for j in range(k):
        src = n - 1 - j                                          # slot j holds the (n - 1 - j)-th best
        g, t = np.nonzero(src >= 0)
        ev[g, t, j] = val[g, t, src[g, t]]; ei[g, t, j] = ids[g, t, src[g, t]]
    return ev, ei


FNS = {True: ("FN_RATE", "FN_INCREASE", "FN_DELTA"), False: ("FN_SUM_OVER_TIME", "FN_COUNT_OVER_TIME")}


@pytest.mark.parametrize("name", list(TABLES))
def test_fused_aggregates_at_steady_state(env, gen, name):
    capi, ctx, o = env["capi"], env["ctx"], env["o"]
    t = TABLES[name]
    tb = get_table(env, name)
    tab, C, G = tb["tab"], tb["C"], tb["G"]
    cum = t["counter"]

    def stats_ok(exp, what):
        assert (ctx.last_stats["samples_scanned"], ctx.last_stats["bytes_scanned"]) == exp, what + ": scan counters"

    for T, first, w in QUERIES:
        q = query_of(T, first, w)
        if gen == "v4": check_path(env, t, tb, T, gen)
        for fn_name in FNS[cum]:
            if T != 80 and fn_name not in ("FN_RATE", "FN_SUM_OVER_TIME"): continue
            fn = getattr(capi, fn_name)
            rows, exp_stats = proto_rows(env, tb, fn_name, q, cum)
            s, a, n = sums(C, rows)
            what = "%s %s %s T=%d" % (gen, name, fn_name, T)
            got = ctx.query(tab, fn, *q, aggr=capi.AGG_SUM); stats_ok(exp_stats, what + " sum")
            gc = ctx.query(tab, fn, *q, aggr=capi.AGG_COUNT); stats_ok(exp_stats, what + " count")
            assert same_bits(gc, np.where(n > 0, n.astype(np.float64), np.nan)), what + " count"
            empty = n == 0
            assert np.isnan(got[empty]).all(), what + " sum of empty cells"
            if cum:
                m = n[~empty]
                bound = (m - 1) * U / (1 - (m - 1) * U) * a[~empty].astype(np.float64) + 64 * 2.0 ** -64 * a[~empty].astype(np.float64)
                err = np.abs(got[~empty].astype(np.longdouble) - s[~empty]).astype(np.float64)
                assert (err <= bound).all(), "%s sum: %d cells off by more than gamma_{m-1} sum|v|" % (what, int((err > bound).sum()))
                if fn_name != "FN_DELTA":           # delta over a reset is near zero: its series are held by count, min and max
                    smallest = np.nanmin(np.abs(rows))
                    assert smallest >= 1e3 * bound.max(), "%s: a dropped or doubled series could hide under the bound" % what
                gv, gn = ctx.query(tab, fn, *q, aggr=capi.AGG_AVG)
                assert (gn == n).all()
                ref_avg = (s[~empty] / m).astype(np.float64)
                assert (np.abs(gv[~empty] - ref_avg) <= bound / m + 4 * U * np.abs(ref_avg)).all(), what + " avg"
            else:
                exact = s.astype(np.float64)
                assert same_bits(got[~empty], exact[~empty]), what + " sum"
                gv, gn = ctx.query(tab, fn, *q, aggr=capi.AGG_AVG)
                assert (gn == n).all() and same_bits(gv[~empty], exact[~empty] / n[~empty]), what + " avg"
                if T == 80:
                    ost = tb.setdefault("ost", None)
                    if ost is None:
                        arena, off = tab.read_arena(0, tb["S"])
                        ost = o.Store(); ost.add_from_arena(arena, off, tb["S"]); tb["ost"] = ost
                    ok = ("oracle sum", name, fn_name, q)
                    if ok not in env["refs"]:
                        es = ost.query(getattr(o, fn_name), *q, aggr=o.AGG_SUM, group_ids=tb["groups"], n_groups=G, threads=os.cpu_count() or 1)
                        assert (ost.last_stats["samples_scanned"], ost.last_stats["bytes_scanned"]) == exp_stats
                        env["refs"][ok] = es
                    assert same_bits(got, env["refs"][ok]), what + " sum against the oracle's aggregate"
            stats_ok(exp_stats, what + " avg")
            for op_min in (True, False):
                aggr = capi.AGG_MIN if op_min else capi.AGG_MAX
                gm = ctx.query(tab, fn, *q, aggr=aggr); stats_ok(exp_stats, what + " min/max")
                assert same_bits(gm, fold_minmax(C, rows, op_min)), what + (" min" if op_min else " max")
                if T == 80: check_partial_present_plain(capi, ctx, tab, fn, q, aggr, gm)
            if T == 80:
                check_partial_present_plain(capi, ctx, tab, fn, q, capi.AGG_SUM, got)
                if fn_name in ("FN_RATE", "FN_SUM_OVER_TIME"):
                    check_moments(capi, ctx, tab, rows[tb["pid"]], tb["groups"], G, fn, q, what, key=("fused steady state", name, fn_name, q))
                    stats_ok(exp_stats, what + " moments")
                    sizes = np.bincount(tb["groups"], minlength=G)
                    kbig = int(sorted(sizes[sizes > 0])[2]) + 2          # larger than the small groups
                    for aggr, bottom in ((capi.AGG_TOPK, False), (capi.AGG_BOTTOMK, True)):
                        for k in (1, 5, min(kbig, 32)):
                            gv_, gi_ = ctx.query(tab, fn, *q, aggr=aggr, k=k); stats_ok(exp_stats, what + " topk")
                            ev, ei = topk_expected(topk_best(env, tb, (id(tb["st"]), fn_name, q), rows, bottom), k, bottom)
                            assert same_bits(gv_, ev), "%s %s k=%d values" % (what, "bottomk" if bottom else "topk", k)
                            assert (gi_ == ei).all(), "%s %s k=%d series ids" % (what, "bottomk" if bottom else "topk", k)
    # the ungrouped table: one group, positions are series ids
    if gen in ("v4", "v2"):
        try:
            tab.set_groups(None, 1)
            items = Items(np.zeros(tb["S"], np.int32), 1, tb["items"].seg)
            assert items.n_items > 8 * env["sms"]
            q = query_of(*QUERIES[0])
            fn_name = FNS[cum][0]
            rows, exp_stats = proto_rows(env, tb, fn_name, q, cum)
            C1 = C.sum(axis=0, keepdims=True)
            s, a, n = sums(C1, rows)
            got = ctx.query(tab, getattr(capi, fn_name), *q, aggr=capi.AGG_SUM); stats_ok(exp_stats, "ungrouped sum")
            gc = ctx.query(tab, getattr(capi, fn_name), *q, aggr=capi.AGG_COUNT)
            assert same_bits(gc, n.astype(np.float64)), "ungrouped count"
            if cum:
                bound = (n - 1) * U / (1 - (n - 1) * U) * a.astype(np.float64) + 64 * 2.0 ** -64 * a.astype(np.float64)
                assert (np.abs(got.astype(np.longdouble) - s).astype(np.float64) <= bound).all(), "ungrouped sum"
            else:
                assert same_bits(got, s.astype(np.float64)), "ungrouped sum"
            assert same_bits(ctx.query(tab, getattr(capi, fn_name), *q, aggr=capi.AGG_MAX), fold_minmax(C1, rows, False)), "ungrouped max"
        finally:
            tab.set_groups(tb["groups"], G)
