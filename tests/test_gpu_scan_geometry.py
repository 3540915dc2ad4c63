"""GPU: the per-series scan kernels across query geometry (tests/scan_geometry_cases.py), bit-exact against the CPU oracle.  One table per
kernel path (the table shapes of tests/test_gpu_steady_state.py, which reach scan_wp_batch_kernel with O on V and O apart,
scan_wp_sum_kernel with two record buffers and with one, the tile kernel, and scan_wp_ctr_kernel with const-DDV and irregular
timestamps), with later chunks moved off chunk 0's grid by 1 ms, half a step, a step - 1 ms and a gap plus 7 s.  Each query runs with
inclusive and with exclusive ranges (`Context(0, inclusive_range=...)`), at start phases 0, +1 ms, half a step and a step - 1 ms, with
windows of k steps - 1 ms, k steps, k steps + 1 ms and k steps + half a step; the counter tables also run a step of twice the scrape
interval.  A table holds one full round of the grid and a partial one.  The path is asserted with filo_query's own choice before each
query; rows are written into a guarded buffer at 16-byte and 8 mod 16 alignment.  The same queries run under FILO_KERNEL=v2 and v1, and
fused `sum by` / `max by` on the tile and counter tables.

test_case_table_on_the_gpu runs every case of tests/scan_geometry_cases.py itself: the case's series repeated into a table of one grid
round and a partial one (the plan's 9-row bound, the J-capacity windows, T from 1 to 630, 1 s and 60 s scrapes, steps that are not the
scrape interval, NaN stale markers), its query in both range modes, with the path scan_path gives for the table asserted: the v4 SUM
kernels (O on V exactly where a series' blocks fit one pass) for the SUM class, scan_wp_ctr_kernel for counters, once on the case's
const-DDV table and once with one jittered series added, which moves the table to the irregular-timestamp instantiation."""
import os
import time
import zlib

import numpy as np
import pytest

from tests import scan_geometry_cases as G
from tests.test_gpu_parity import assert_same
from tests.test_gpu_steady_state import TABLES as STEADY, table_shape
from tests.test_scan_path import build_scan_path, scan_path

pytestmark = pytest.mark.gpu
STEP = G.SCRAPE
GUARD = 0x7FF4A5A5C3C3E1E1          # a signalling-NaN pattern no kernel writes
GW = 8                              # guard words on each side
THREADS = os.cpu_count() or 1
SHIFTS = (1, STEP // 2, STEP - 1, 7000, 0)      # chunk phases (ms, on top of the shape's gap of whole steps)
PATHS = ("batch O on V", "batch O apart", "sum two record buffers", "sum one record buffer", "tile", "ctr const timestamps",
         "ctr jittered timestamps")


def series_count(t, sms):
    """One full round of the grid (every warp, or every tile slot of every CTA, takes one series) and a partial one: two warps more per
    CTA than the steady-state table's, since the shifted chunks can change a record's size and with it the warps of a CTA by one."""
    return (t["warps"] + 2) * t["per_sm"] * sms + 3


def build(o, name, n):
    """The oracle store: series s takes shape s % len of the steady-state table's regular and declined shapes (those set the table's
    largest record and chunk count, and with them its kernel path), its later chunks shifted by SHIFTS[(s // len) % 5] on top of the
    shape's gap.  The irregular-timestamp table ends with one series of jittered timestamps, which selects that instantiation for every
    series."""
    t = STEADY[name]
    st = o.Store()
    reg = list(t["regular"]) + [t["declined"][k] for k in sorted(t["declined"])]
    jitter = bool(t.get("jitter"))
    for s in range(n):
        si = st.add_series()
        rows, enc, gap = reg[s % len(reg)]
        ph = SHIFTS[(s // len(reg)) % len(SHIFTS)]
        sh = G.shape(rows, enc, tuple(gap * STEP + ph if c == 0 else gap * STEP for c in range(len(rows) - 1)))
        chunks = G.series_chunks(sh, t["counter"], zlib.crc32(repr((name, s)).encode()))
        if jitter and s == n - 1:
            rng = np.random.default_rng(7)
            chunks = [(ts + rng.integers(-2000, 2001, len(ts)), v, e) for ts, v, e in chunks]
        for ts, v, e in chunks:
            if e == "d":                  # integral values, optimized to a DDV vector: the v4 and tile kernels decline the series
                v = np.round(v * (1 if t["counter"] else 10))
            st.add_chunk(si, ts, v, val_mode={"x": o.VAL_XOR, "r": o.VAL_RAW, "d": o.VAL_OPTIMIZE}[e], detect_drops=t["counter"])
    return st


def queries(t):
    """(start, step, T, window, fns) per query: each of the table's queries at two (start phase, window variant) pairs that take turns
    over the four phases and the four window variants; the counter tables add a step of twice the scrape interval."""
    out = []
    fns = G.CTR_FNS if t["counter"] else G.SUM_FNS
    for i, (T, first, wsteps) in enumerate(t["queries"]):
        for j in (0, 1):
            u = 2 * i + j
            ph = ("0", "+1", "half", "step-1")[(u + u // 4) % 4]
            wv = ("-1", "0", "+1", "+half")[u % 4]
            k = wsteps + 1 if wv == "-1" else wsteps          # (k + 1) steps - 1 ms: the table's window / step + 1, so its kernel path
            out.append((G.T0 + first * STEP + G._phase_ms(ph, STEP), STEP, T, G._window_ms(k, wv, STEP), (fns[u % len(fns)], fns[(u + 2) % len(fns)])))
    if t["counter"]:
        T, first, wsteps = t["queries"][0]
        out.append((G.T0 + first * STEP + 7500, 2 * STEP, T, wsteps * STEP + 1, fns))
    return out


@pytest.fixture(scope="module")
def env(tmp_path_factory):
    import torch
    import filodb_b200.capi as capi
    exe = build_scan_path(tmp_path_factory.mktemp("scan_path"))
    ctxs = {1: capi.Context(0, inclusive_range=True), 0: capi.Context(0, inclusive_range=False)}
    props = torch.cuda.get_device_properties(0)
    sms = props.multi_processor_count
    smem = min(props.shared_memory_per_block_optin, 227 * 1024)
    t_start = time.time()
    yield capi, ctxs, exe, sms, smem
    for c in ctxs.values():
        c.close()
    print("\ntest_gpu_scan_geometry: %.1f s" % (time.time() - t_start))


def check_path(exe, t, tab, n, sms, smem, T, wrows, fused=False):
    rec, rows, chunks, irr = table_shape(tab)
    p = scan_path(exe, rec=rec, rows=rows, chunks=chunks, T=T, wrows=wrows, n=n, sms=sms, smem=smem,
                  cls="counter" if t["counter"] else "sum", irr=int(irr), fused=int(fused))
    what = "T=%d wrows=%d rec=%d rows=%d chunks=%d irr=%d: %s" % (T, wrows, rec, rows, chunks, irr, p)
    assert p["kernel"] == t["kernel"], what
    assert irr == bool(t.get("jitter")), what
    if "alias" in t: assert p["alias"] == t["alias"], what
    if "rec_bufs" in t: assert p["rec_bufs"] == t["rec_bufs"], what
    assert p["series_per_warp"] >= 1 and (t["kernel"] == "tile" or p["rounds"] >= 0), what


@pytest.mark.parametrize("name", PATHS)
def test_scan_geometry_rows_match_the_oracle(env, oracle, name, monkeypatch):
    capi, ctxs, exe, sms, smem = env
    t = STEADY[name]
    n = series_count(t, sms)
    st = build(oracle, name, n)
    tab = ctxs[1].load_series(*st.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE if t["counter"] else 0)
    tab0 = ctxs[0].load_series(*st.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE if t["counter"] else 0)
    try:
        per_ctx = {1: _Bound(ctxs[1], tab), 0: _Bound(ctxs[0], tab0)}       # each range mode queries the table its context loaded
        run(per_ctx, st, t, n, name, exe, sms, smem)
        # the same queries on the v2 and v1 kernels
        for force in ("v2", "v1"):
            monkeypatch.setenv("FILO_KERNEL", force)
            run(per_ctx, st, t, n, "%s (FILO_KERNEL=%s)" % (name, force))
        monkeypatch.delenv("FILO_KERNEL")
    finally:
        tab.free(); tab0.free()


class _Bound:
    """A context with the table it loaded."""
    def __init__(self, ctx, tab): self.ctx, self.tab = ctx, tab


def run(per_ctx, st, t, n, name, exe=None, sms=0, smem=0, fixed=None):
    """Every query of the table (or the `fixed` ones) in both range modes; with exe, the kernel path is asserted before each query."""
    import torch
    cum = t["counter"]
    for start, step, T, window, fns in fixed if fixed is not None else queries(t):
        end = start + (T - 1) * step
        if exe: check_path(exe, t, per_ctx[1].tab, n, sms, smem, T, window // step + 1)
        buf = torch.empty((2 * GW + n * T + 2,), dtype=torch.int64, device="cuda")
        for incl in (1, 0):
            ctx, tab = per_ctx[incl].ctx, per_ctx[incl].tab
            for fn in fns:
                exp = st.query(fn, start, step, end, window, cumulative=cum, inclusive=bool(incl), threads=THREADS)
                for off in (0, 1):        # rows at a 16-byte-aligned address, or at 8 mod 16
                    buf.fill_(GUARD)
                    rows = buf[GW + off:GW + off + n * T].view(torch.float64)
                    ctx.query_device(tab, fn, start, step, end, window, rows.data_ptr())
                    torch.cuda.synchronize()
                    h = buf.cpu().numpy()
                    what = "%s: %s %s T=%d start=+%d step=%d window=%d out+%dB" % (name, G.FN_NAMES[fn], "inclusive" if incl else "exclusive", T,
                                                                                  start - G.T0, step, window, 8 * off)
                    outside = np.concatenate([h[:GW + off], h[GW + off + n * T:]])
                    assert (outside == GUARD).all(), what + ": words outside the rows were written"
                    assert_same(h[GW + off:GW + off + n * T].view(np.float64).reshape(n, T), exp, what)
                    assert ctx.last_stats["samples_scanned"] == st.last_stats["samples_scanned"], what
                    assert ctx.last_stats["bytes_scanned"] == st.last_stats["bytes_scanned"], what


@pytest.mark.parametrize("name", ["tile", "ctr const timestamps", "ctr jittered timestamps"])
def test_scan_geometry_fused_sum_and_max_by(env, oracle, name):
    """Fused `sum by` / `max by` (the tile and counter kernels fold partial rows): sums within 1e-9 of the oracle's per-series rows
    summed, max bit-exact, at the table's first queries in both range modes."""
    capi, ctxs, exe, sms, smem = env
    t = STEADY[name]
    n = series_count(t, sms)
    ng = 7
    groups = (np.arange(n) * 3 % ng).astype(np.int32)
    st = build(oracle, name, n)
    cum = t["counter"]
    for incl in (1, 0):
        ctx = ctxs[incl]
        tab = ctx.load_series(*st.all_info_addrs(), group_ids=groups, n_groups=ng, schema_flags=capi.SCHEMA_CUMULATIVE if cum else 0)
        try:
            for start, step, T, window, fns in queries(t)[:3]:
                end = start + (T - 1) * step
                # the tile kernel folds a fused SUM-class query up to TILE_AGG_ACC * TILE_THREADS windows; the counter kernel, its path
                check_path(exe, t, tab, n, sms, smem, T, window // step + 1, fused=True)
                assert T <= 512
                for fn in fns:
                    exp = st.query(fn, start, step, end, window, cumulative=cum, inclusive=bool(incl), threads=THREADS)
                    what = "%s: %s %s T=%d start=+%d window=%d" % (name, G.FN_NAMES[fn], "inclusive" if incl else "exclusive", T, start - G.T0, window)
                    for op in (capi.AGG_SUM, capi.AGG_MAX):
                        gv = np.asarray(ctx.query(tab, fn, start, step, end, window, aggr=op)).reshape(ng, T)
                        for g in range(ng):
                            rows = exp[groups == g]
                            have = ~np.isnan(rows)
                            ref = np.full(T, np.nan)
                            any_ = have.any(axis=0)
                            if op == capi.AGG_SUM:
                                ref[any_] = np.where(have, rows, 0.0).sum(axis=0)[any_]
                                assert (np.isnan(gv[g]) == ~any_).all(), what
                                np.testing.assert_allclose(gv[g][any_], ref[any_], rtol=1e-9, atol=0, err_msg=what)
                            else:
                                ref[any_] = np.where(have, rows, -np.inf).max(axis=0)[any_]
                                assert_same(gv[g][None, :], ref[None, :], what + " max")
        finally:
            tab.free()


def _wp_alias(chunks, T, wrows):
    """filo_query's choice of O on V (scan_path, scan_wp_layout.h wp_max_items): every series' blocks fit one pass of 64."""
    c = max(1, min(chunks, G.WP_MAXC))
    return (T + (c - 1) * (wrows - 1) + 7 * c) // 8 <= 64


@pytest.mark.parametrize("cls", ["sum", "counter"])
def test_case_table_on_the_gpu(env, oracle, cls):
    capi, ctxs, exe, sms, smem = env
    n = 21 * sms + 9           # one round and a partial one of every per-series kernel: at most 20 warps per CTA, one CTA per SM
    seen = set()
    for case in [c for c in G.CASES if c["counter"] == (cls == "counter")]:
        base = G.case_series(case)
        for irr in ((False, True) if case["counter"] else (False,)):
            series = [base[s % len(base)] for s in range(n - 1 if irr else n)]
            if irr:                # timestamps off the step grid by up to an eighth of the scrape interval: DDV timestamps
                jit = max(1, case["shapes"][0]["scrape"] // 8)
                rng = np.random.default_rng(zlib.crc32(case["name"].encode()))
                series.append([(ts + rng.integers(-jit, jit + 1, len(ts)), v, e) for ts, v, e in base[0]])
            st = oracle.Store()
            for chunks in series:
                si = st.add_series()
                for ts, v, e in chunks:
                    st.add_chunk(si, ts, v, val_mode={"x": oracle.VAL_XOR, "r": oracle.VAL_RAW}[e], detect_drops=case["counter"])
            flags = capi.SCHEMA_CUMULATIVE if case["counter"] else 0
            tabs = {k: ctxs[k].load_series(*st.all_info_addrs(), schema_flags=flags) for k in (1, 0)}
            try:
                start, step, end, window, T, _ = G.query_of(case, 1)
                wrows = window // step + 1
                rec, rows, chunks, tirr = table_shape(tabs[1])
                p = scan_path(exe, rec=rec, rows=rows, chunks=chunks, T=T, wrows=wrows, n=n, sms=sms, smem=smem, cls=cls, irr=int(tirr))
                what = "%s (%s) T=%d wrows=%d rec=%d rows=%d chunks=%d irr=%d: %s" % (case["name"], case["what"], T, wrows, rec, rows, chunks, tirr, p)
                assert tirr == irr, what
                if case["counter"]:
                    assert p["kernel"] == "ctr", what
                    path = "ctr irregular" if irr else "ctr const"
                else:
                    assert p["kernel"] in ("batch", "sum") and p["alias"] == int(_wp_alias(chunks, T, wrows)), what
                    path = "%s O %s" % (p["kernel"], "on V" if p["alias"] else "apart")
                assert p["series_per_warp"] >= 1 and p["rounds"] >= 0, what
                seen.add(path)
                run({k: _Bound(ctxs[k], tabs[k]) for k in (1, 0)}, st, dict(counter=case["counter"]), n,
                    "%s (%s, %s)" % (case["name"], case["what"], path), fixed=[(start, step, T, window, case["fns"])])
            finally:
                for tb in tabs.values():
                    tb.free()
    want = {"ctr const", "ctr irregular"} if cls == "counter" else {"batch O on V", "batch O apart"}
    assert want <= seen, seen
    print("\n%s cases on the GPU: %s" % (cls, sorted(seen)))
