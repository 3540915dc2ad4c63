"""GPU: the per-series scan kernels at steady state, where every warp (or CTA) of the persistent grid takes many series, bit-exact
against the CPU oracle.  Each table reaches one kernel, asserted with filo_query's own choice (scan_path, run through the host program
tests/cpp/scan_path.cpp on the table's real record bytes and the device's SM count), at a depth derived from the SM count:
scan_wp_batch_kernel with O on V and O apart (every batch buffer in its third round), scan_wp_sum_kernel with two record buffers and with
one, the tile kernel, and scan_wp_ctr_kernel with const-DDV and jittered timestamps; and one table built with filo_table_append.

Series of one warp alternate between plan-memo hits and misses (chunk shapes with different row counts and splits, a time gap between
chunks, XOR and raw f64 value chunks mixed in one series and one batch).  Declined series (a NaN stale marker, five chunks in range, a
window spanning three chunks, a DDV value chunk) sit at the first and last slot of batches and at the first series of later rounds; the
v2 kernel answers them into the same rows.  Queries run at odd and even T, through filo_query_device into a buffer with guard words on both sides whose rows
start 16-byte aligned or at 8 mod 16; nothing outside the rows may change, and the scan counters must equal the oracle's."""
import os
import time
import zlib

import numpy as np
import pytest

from tests.test_gpu_parity import assert_same
from tests.test_scan_path import build_scan_path, scan_path

pytestmark = pytest.mark.gpu
T0 = 1_700_000_000_000
STEP = 15000
GUARD = 0x7FF4A5A5C3C3E1E1          # a signalling-NaN pattern no kernel writes
G = 8                               # guard words on each side
THREADS = os.cpu_count() or 1
SUM_FNS = ("FN_SUM_OVER_TIME", "FN_AVG_OVER_TIME", "FN_COUNT_OVER_TIME", "FN_RATE", "FN_INCREASE")   # the SUM class on a gauge schema
CTR_FNS = ("FN_RATE", "FN_INCREASE", "FN_DELTA")                                                     # the counter class

# A shape is (rows per chunk, value encoding per chunk, gap in steps before every chunk after the first): x = XOR, r = raw f64,
# d = DDV (integral values, optimized; the v4 and tile kernels take XOR and raw f64 values only, so a DDV chunk declines its series).
# `regular` shapes are the ones the kernel takes; they take turns.  `declined` shapes, by cause, replace a regular one at the declined
# positions (a NaN marker keeps the regular shape).  kernel: scan_path's name; warps: series per round of one CTA (warps that take
# series; series per tile); depth: series per warp (tiles per CTA) to require; rounds: the buffer round every warp must reach.
# queries: (T, first window's row, window in steps).
TABLES = {
    "batch O on V": dict(
        kernel="batch", alias=1, warps=15, per_sm=1, depth=5, rounds=2, counter=False,
        regular=[((300, 60), "xx", 0), ((150, 110, 100), "xrx", 0), ((180, 180), "xr", 45), ((120, 120, 120), "rxx", 0), ((80, 140, 140), "xxr", 20)],
        declined=dict(chunks5=((72, 72, 72, 72, 72), "xxxxx", 0), span3=((175, 10, 175), "xxx", 0), ddv=((200, 160), "xd", 0)),
        queries=[(2, 299, 20), (27, 0, 20), (240, 100, 20), (431, -10, 20), (300, 60, 40)]),
    "batch O apart": dict(
        kernel="batch", alias=0, warps=15, per_sm=1, depth=5, rounds=2, counter=False,
        regular=[((100, 100), "xx", 0), ((97, 103), "xr", 0), ((70, 70, 60), "rxx", 10), ((50, 150), "rx", 0)],
        declined=dict(chunks5=((40, 40, 40, 40, 40), "xxxxx", 0), span3=((95, 10, 95), "xrx", 0), ddv=((100, 100), "dx", 0)),
        queries=[(630, 5, 20), (631, -200, 20)]),
    # at most three chunks: four would leave too little shared memory for two record buffers; windows of 89 rows
    "sum two record buffers": dict(
        kernel="sum", alias=0, warps=16, per_sm=1, depth=4, rounds=1, rec_bufs=2, counter=False,
        regular=[((120,), "r", 0), ((60, 60), "xr", 0), ((50, 70), "rx", 12), ((110,), "x", 0)],
        declined=dict(span3=((55, 10, 55), "rrr", 0), ddv=((60, 60), "dr", 0)),
        queries=[(630, 3, 88), (631, -150, 88)]),
    # records of about 4 KB (raw f64 series of 480 rows): 13 warps of one record buffer
    "sum one record buffer": dict(
        kernel="sum", alias=0, warps=13, per_sm=1, depth=3, rounds=2, rec_bufs=1, counter=False,
        regular=[((400, 80), "xx", 0), ((237, 243), "xr", 0), ((200, 150, 130), "xrx", 30), ((240, 240), "rr", 0)],
        declined=dict(chunks5=((96, 96, 96, 96, 96), "xxxxx", 0), span3=((230, 10, 240), "xxx", 0), ddv=((240, 240), "dx", 0)),
        queries=[(630, -60, 20), (631, 7, 20)]),
    # windows of 3001 rows: the positions of V in the v4 SUM layouts (rows plus zero gaps of a window's rows around every chunk) leave
    # room for fewer than four warps, and the tile kernel (with checked loads) takes the table
    "tile": dict(
        kernel="tile", warps=8, per_sm=2, depth=3, counter=False,
        regular=[((400, 80), "xx", 0), ((237, 243), "xr", 0), ((160, 160, 160), "rxx", 30)],
        declined=dict(chunks5=((96, 96, 96, 96, 96), "xxxxx", 0), span3=((230, 10, 240), "xxx", 0), ddv=((240, 240), "dx", 0)),
        queries=[(27, 0, 3000), (40, 300, 3000)]),
    "ctr const timestamps": dict(
        kernel="ctr", warps=20, per_sm=1, depth=3, rounds=2, counter=True, jitter=0,
        regular=[((400, 80), "xx", 0), ((237, 243), "xr", 0), ((160, 160, 160), "rxx", 30), ((300, 180), "rx", 0)],
        declined=dict(chunks5=((96, 96, 96, 96, 96), "xxxxx", 0), span3=((230, 10, 240), "xxx", 0), ddv=((237, 243), "xd", 0)),
        queries=[(27, 0, 20), (240, 101, 20), (481, 0, 20)]),
    "ctr jittered timestamps": dict(
        kernel="ctr", warps=16, per_sm=1, depth=3, rounds=2, counter=True, jitter=2000,
        regular=[((400, 80), "xx", 0), ((237, 243), "xr", 0), ((160, 160, 160), "rxx", 30), ((300, 180), "rx", 0)],
        declined=dict(chunks5=((96, 96, 96, 96, 96), "xxxxx", 0), span3=((230, 10, 240), "xxx", 0), ddv=((237, 243), "xd", 0)),
        queries=[(27, 0, 20), (241, 100, 20), (480, 0, 20)]),
}


def table_size(t, sms):
    """Series of a table: `depth` full rounds of every CTA's warps and a partial one."""
    return t["depth"] * t["warps"] * t["per_sm"] * sms + t["warps"] // 2 + 3


def plan(t, n, sms):
    """Per series: (shape, decline cause or None).  Shapes go A A B B .. along a warp's series (a memo hit after a different series, then a
    miss) and differ between neighbours; declines sit at a batch's first and last slot and at the first series of rounds 2 and 4."""
    P = t["warps"] * t["per_sm"] * sms          # series per round of the grid: consecutive series of one warp are s and s + P
    reg, dec = t["regular"], t["declined"]
    causes = ["nan"] + sorted(dec)
    out, nd = [], 0
    for s in range(n):
        k, pos = divmod(s, P)
        shape = reg[(k // 2 + pos) % len(reg)]
        cause = None
        if ((s // 15) % 5 == 2 and s % 15 in (0, 14)) or s in (2 * P, 4 * P, 2 * P + P // 2):
            cause = causes[nd % len(causes)]; nd += 1          # the causes take turns
            shape = dec.get(cause, shape)
        out.append((shape, cause))
    return out


def _chunks(rng, shape, counter, jitter, cause, shape_seed):
    """(ts, values, val_mode) per chunk.  The timestamps of a shape are the same in every series (so its plan can be memoised)."""
    import oracle.oracle as o
    rows, enc, gap = shape
    total = sum(rows)
    r = np.arange(total, dtype=np.int64)
    cstart = np.cumsum((0,) + tuple(rows))
    shift = np.zeros(total, np.int64)
    for c in range(1, len(rows)):
        shift[cstart[c]:] += gap
    ts = T0 + (r + shift) * STEP
    if jitter:
        ts = ts + np.random.default_rng(shape_seed).integers(-jitter, jitter + 1, total)
    if counter:
        v = np.cumsum(rng.integers(0, 40, total)).astype(np.float64)
        for q in np.nonzero(rng.random(total) < 0.01)[0]:
            if q > 0: v[q:] = v[q:] - v[q] + float(rng.integers(0, 5))
    else:
        v = 15 + np.sin(np.arange(1, total + 1)) + rng.normal(0, 1, total)
    out = []
    for c, e in enumerate(enc):
        a, b = cstart[c], cstart[c + 1]
        vc = v[a:b].copy()
        if e == "d":
            vc = np.round(vc * (1 if counter else 10))
        mode = {"x": o.VAL_XOR, "r": o.VAL_RAW, "d": o.VAL_OPTIMIZE}[e]
        out.append((ts[a:b], vc, mode))
    if cause == "nan":
        c = 0; vc = out[c][1]; vc[len(vc) // 2] = np.nan
    return out


def build(o, name, n, sms, only_first=False):
    """The oracle store of a table (with only_first: every series' first chunk alone, for the append table)."""
    t = TABLES[name]
    rng = np.random.default_rng(zlib.crc32(repr(("steady", name)).encode()))
    st = o.Store()
    for s, (shape, cause) in enumerate(plan(t, n, sms)):
        si = st.add_series()
        sseed = zlib.crc32(repr(shape).encode())
        for c, (ts, v, mode) in enumerate(_chunks(rng, shape, t["counter"], t.get("jitter", 0), cause, sseed)):
            if only_first and c > 0: break
            st.add_chunk(si, ts, v, val_mode=mode, detect_drops=t["counter"])
    return st


@pytest.fixture(scope="module")
def env(tmp_path_factory):
    import torch
    import filodb_b200.capi as capi
    exe = build_scan_path(tmp_path_factory.mktemp("scan_path"))
    ctx = capi.Context(0)
    props = torch.cuda.get_device_properties(0)
    sms = props.multi_processor_count
    smem = min(props.shared_memory_per_block_optin, 227 * 1024)     # the shared memory filo_query lets one CTA opt into
    t_start = time.time()
    yield capi, ctx, exe, sms, smem
    ctx.close()
    print("\ntest_gpu_steady_state: %.1f s" % (time.time() - t_start))


def table_shape(tab):
    """(max record bytes, max rows, max chunks, whether some series has timestamps that are not const-DDV) of a loaded table."""
    ti = tab.info()
    arena, off = tab.read_arena(0, ti.n_series)
    flags = arena[off[:-1, None] + np.arange(12, 16)].copy().view(np.uint32).ravel()    # RecordHeader.flags
    irr = bool(((flags & 1) == 0).any())                                                 # REC_ALL_TS_CONST
    return int(np.diff(off).max()), int(ti.max_rows_per_series), int(ti.max_chunks_per_series), irr


def check_path(exe, t, tab, n, sms, smem, T, wrows):
    rec, rows, chunks, irr = table_shape(tab)
    p = scan_path(exe, rec=rec, rows=rows, chunks=chunks, T=T, wrows=wrows, n=n, sms=sms, smem=smem,
                  cls="counter" if t["counter"] else "sum", irr=int(irr))
    what = "T=%d wrows=%d rec=%d rows=%d chunks=%d irr=%d: %s" % (T, wrows, rec, rows, chunks, irr, p)
    assert p["kernel"] == t["kernel"], what
    assert irr == bool(t.get("jitter")), what
    if "alias" in t: assert p["alias"] == t["alias"], what
    if "rec_bufs" in t: assert p["rec_bufs"] == t["rec_bufs"], what
    if t["kernel"] == "batch": assert p["B"] == 15 and p["rec_bufs"] == 2, what
    # the series of one warp are `warps * grid` apart, the stride plan() lays the shapes and declines out with
    assert (p["warps"] if t["kernel"] != "tile" else 8) == t["warps"], what
    assert p["grid"] == t["per_sm"] * sms, what
    assert p["series_per_warp"] >= t["depth"], what
    if "rounds" in t: assert p["rounds"] >= t["rounds"], what
    o_at = (" O on V" if p["alias"] else " O apart") if t["kernel"] in ("batch", "sum") else ""
    print("%s%s: %s series, T=%d: %d series per warp%s, buffer round %d" % (t["kernel"], o_at, n, T,
          p["series_per_warp"], "" if t["kernel"] != "tile" else " (tiles per CTA)", p["rounds"]))
    return p


def run_queries(capi, ctx, o, st, tab, t, n, exe, sms, smem, name, check=True):
    import torch
    cum = t["counter"]
    fns = CTR_FNS if cum else SUM_FNS
    for T, first, wsteps in t["queries"]:
        start, window = T0 + first * STEP, wsteps * STEP
        end = start + (T - 1) * STEP
        if check: check_path(exe, t, tab, n, sms, smem, T, wsteps + 1)
        buf = torch.empty((2 * G + n * T + 2,), dtype=torch.int64, device="cuda")
        assert buf.data_ptr() % 16 == 0
        for fn in fns:
            exp = st.query(getattr(o, fn), start, STEP, end, window, cumulative=cum, threads=THREADS)
            for off in (0, 1):        # the rows start at a 16-byte-aligned address, or at 8 mod 16
                buf.fill_(GUARD)
                rows = buf[G + off:G + off + n * T].view(torch.float64)
                ctx.query_device(tab, getattr(capi, fn), start, STEP, end, window, rows.data_ptr())
                torch.cuda.synchronize()
                h = buf.cpu().numpy()
                what = "%s: %s T=%d window=%d out+%dB" % (name, fn, T, window, 8 * off)
                outside = np.concatenate([h[:G + off], h[G + off + n * T:]])
                assert (outside == GUARD).all(), what + ": words outside the rows were written"
                assert_same(h[G + off:G + off + n * T].view(np.float64).reshape(n, T), exp, what)
                assert ctx.last_stats["samples_scanned"] == st.last_stats["samples_scanned"], what
                assert ctx.last_stats["bytes_scanned"] == st.last_stats["bytes_scanned"], what


@pytest.mark.parametrize("name", list(TABLES))
def test_steady_state_rows_match_the_oracle(env, oracle, name):
    capi, ctx, exe, sms, smem = env
    t = TABLES[name]
    n = table_size(t, sms)
    st = build(oracle, name, n, sms)
    tab = ctx.load_series(*st.all_info_addrs(), schema_flags=capi.SCHEMA_CUMULATIVE if t["counter"] else 0)
    try:
        run_queries(capi, ctx, oracle, st, tab, t, n, exe, sms, smem, name)
    finally:
        tab.free()


def test_appended_table_at_batch_depth(env, oracle):
    """filo_table_append re-packs the arena with every series' later chunks: the table's records grow, and with them the batch kernel's
    layout; the rows of the first chunks alone and of the whole series match the oracle."""
    capi, ctx, exe, sms, smem = env
    name = "batch O on V"
    t = TABLES[name]
    n = table_size(t, sms)
    st = build(oracle, name, n, sms)
    st1 = build(oracle, name, n, sms, only_first=True)
    per = [st.info_addrs(s) for s in range(n)]
    tab = ctx.load_series(np.ones(n, np.int32), np.array([p[0] for p in per], np.uint64))
    try:
        before = table_shape(tab)
        first = dict(t, queries=[(27, 0, 20), (240, 60, 20)])
        run_queries(capi, ctx, oracle, st1, tab, first, n, exe, sms, smem, name + " (first chunks)", check=False)
        p1 = check_path(exe, first, tab, n, sms, smem, 240, 21)
        tab.append(np.array([len(p) - 1 for p in per], np.int32), np.array([a for p in per for a in p[1:]], np.uint64))
        after = table_shape(tab)
        assert after[0] > before[0] and after[2] > before[2], (before, after)
        p2 = check_path(exe, first, tab, n, sms, smem, 240, 21)
        assert p2["smem"] > p1["smem"], (p1, p2)
        run_queries(capi, ctx, oracle, st, tab, t, n, exe, sms, smem, name + " (appended)")
    finally:
        tab.free()
