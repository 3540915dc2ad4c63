"""Query-geometry cases of the per-series scan kernels, shared by the emulator test (tests/test_scan_geometry_emul.py) and the GPU
test (tests/test_gpu_scan_geometry.py), and a brute-force predictor of which series the two kernels built on `wp_plan_series`
(scan_wp_batch_kernel and scan_wp_sum_kernel) take.

The v4 kernels never walk rows: they work out every window's row range in closed form from the query and each chunk's first timestamp
(`StepDiv` in `wp_plan_series`, the `(q.inclusive ? 0 : 1)` term of the counter kernel's extrapolation).  Every term depends on where the
query start falls on each chunk's timestamp grid, on whether the window is a whole number of steps, on the range mode and on whether a
later chunk is on the first chunk's grid.  The cases below combine those axes:
  * start phase against chunk 0's grid: 0, +1 ms, half a step, a step - 1 ms; starts before the data and ends past it;
  * windows of k steps - 1 ms, k steps, k steps + 1 ms and k steps + half a step, with k around the plan's 9-row bound (7, 8, 9), C2's 20,
    k large enough for O apart, and k at the J capacity (127 / 128: a window of 128 rows fits WP_J_DOUBLES, 129 do not);
  * later chunks shifted off chunk 0's grid by 1 ms, half a step, a step - 1 ms and a step + 7 s (with a gap of whole steps too);
  * T = 1, 2, 7, 8, 9, 63, 64, 65, 481, 630 (both row phases of the batch kernel's staged store);
  * scrape intervals of 15 s, 1 s and 60 s, and query steps of 2x, 4x and 1/3 of the scrape interval;
and every case runs with inclusive and with exclusive ranges.
"""
import itertools
import zlib

import numpy as np

T0 = 1_700_000_000_000
SCRAPE = 15000
# function codes (filo::FN_* in scan_params.h; the oracle and capi use the same numbers)
FN_RATE, FN_INCREASE, FN_DELTA, FN_SUM, FN_AVG, FN_COUNT = 1, 2, 3, 4, 5, 6
SUM_FNS = (FN_SUM, FN_AVG, FN_COUNT, FN_RATE, FN_INCREASE)      # SUM class (rate / increase on a gauge schema)
CTR_FNS = (FN_RATE, FN_INCREASE, FN_DELTA)                      # counter class
FN_NAMES = {FN_RATE: "FN_RATE", FN_INCREASE: "FN_INCREASE", FN_DELTA: "FN_DELTA", FN_SUM: "FN_SUM_OVER_TIME",
            FN_AVG: "FN_AVG_OVER_TIME", FN_COUNT: "FN_COUNT_OVER_TIME"}
WP_MAXC, WP_MAXG, WP_J_DOUBLES, WP_R = 4, 64, 128, 8         # scan_wp_layout.h


def shape(rows, enc, shifts=(), scrape=SCRAPE, nan=False):
    """A series shape: rows per chunk, value encoding per chunk (x = XOR, r = raw f64), a time shift in ms added to every chunk from
    chunk c + 1 on (cumulative, so chunk c + 1 leaves chunk c's grid when the shift is not a whole number of scrapes), the scrape
    interval, and a NaN stale marker in the middle of chunk 0."""
    assert len(enc) == len(rows) and len(shifts) == len(rows) - 1
    return dict(rows=tuple(rows), enc=enc, shifts=tuple(shifts), scrape=scrape, nan=nan)


def series_chunks(sh, counter, seed):
    """[(timestamps int64, values float64, encoding)] per chunk of a shape.  Gauges: 15 + sin + N(0, 1) (finite, normal, non-zero);
    counters: fractional increments (an encoder that optimizes keeps them f64) with two resets (at most two drops per chunk, far below
    the drop list's 8)."""
    rng = np.random.default_rng(seed)
    rows = sh["rows"]
    total = sum(rows)
    r = np.arange(total, dtype=np.int64)
    cstart = np.cumsum((0,) + rows)
    shift = np.zeros(total, np.int64)
    for c in range(1, len(rows)):
        shift[cstart[c]:] += sh["shifts"][c - 1]
    ts = T0 + r * sh["scrape"] + shift
    if counter:
        v = np.cumsum(rng.uniform(0.5, 40.0, total))
        for q in (total // 3, (2 * total) // 3 + 1):
            v[q:] = v[q:] - v[q] + rng.uniform(1.0, 5.0)
    else:
        v = 15 + np.sin(np.arange(1, total + 1)) + rng.normal(0, 1, total)
    out = []
    for c, e in enumerate(sh["enc"]):
        a, b = cstart[c], cstart[c + 1]
        out.append((ts[a:b].copy(), v[a:b].copy(), e))
    if sh["nan"]:
        vc = out[0][1]; vc[len(vc) // 2] = np.nan
    return out


def query_of(case, inclusive):
    """(start, step, end, window, T, inclusive) of a case."""
    return (case["start"], case["step"], case["start"] + (case["T"] - 1) * case["step"], case["window"], case["T"], inclusive)


def _lattice_count(init, step, S0, E0):
    """Points init + r * step (any integer r) in [S0, E0]: floor((E0 - init) / step) - ceil((S0 - init) / step) + 1."""
    return (E0 - init) // step - (-((S0 - init) // -step)) + 1


def wp_accepts(chunks, q):
    """Whether scan_wp_batch_kernel / scan_wp_sum_kernel take a series (chunks as series_chunks gives them) for query q.  Brute force
    over the rows; each rule names the check of scan_wp.cuh it restates.  The capacity checks the host sizes for (V's positions,
    O on V's 64 items, the batch kernel's raw tail area) are left out on purpose: the layouts say they cannot decline."""
    start, step, end, window, T, inclusive = q
    # header parse (scan_wp.cuh:185-192): the chunks in range end at or after start - window and start at or before end; at most four
    inr = [c for c in chunks if c[0][-1] >= start - window and c[0][0] <= end]
    if not inr or len(inr) > WP_MAXC:
        return False
    for ts, v, enc in inr:
        # timestamps: const DDV with slope = the query step (scan_wp.cuh:184, 166)
        if len(ts) > 1 and not (np.diff(ts) == step).all():
            return False
        # values: XOR or raw f64 (scan_wp.cuh:163-165), finite, normal and non-zero, so no NaN stale marker (scan_wp.cuh:1109-1120)
        if enc not in "xr" or not np.isfinite(v).all() or not ((np.abs(v) >= 2.0 ** -511) & (np.abs(v) < 2.0 ** 513)).all():
            return False
    # NibblePack groups of the XOR chunks in range: at most 64 (scan_wp.cuh:212)
    if sum((len(ts) + 6) // 8 for ts, v, enc in inr if enc == "x") > WP_MAXG:
        return False
    win_dur = max(window if inclusive else window - 1, 0)          # WpQuery::init, scan_wp.cuh:396-398
    S0, E0 = start - win_dur, start
    # rows per window on each chunk's own grid: the same for every chunk in range (scan_wp.cuh:438), at least 9 (Wr0 < 8 declines) and
    # at most WP_J_DOUBLES (Wr0 + 1 > jcap declines, scan_wp.cuh:439)
    counts = {_lattice_count(int(ts[0]), step, S0, E0) for ts, v, enc in inr}
    if len(counts) != 1:
        return False
    cnt = counts.pop()
    if cnt < 9 or cnt > WP_J_DOUBLES:
        return False
    # windows touched by each chunk (rows of the chunk inside window k), brute force
    k = np.arange(T, dtype=np.int64)
    lo, hi = S0 + k * step, E0 + k * step
    touch = []
    for ts, v, enc in inr:
        n_in = np.searchsorted(ts, hi, side="right") - np.searchsorted(ts, lo, side="left")
        w = np.nonzero(n_in > 0)[0]
        touch.append((int(w[0]), int(w[-1])) if len(w) else None)
    tm = [t is not None for t in touch]
    # touched chunks are contiguous (scan_wp.cuh:442)
    first = tm.index(True) if any(tm) else 0
    last = len(tm) - 1 - tm[::-1].index(True) if any(tm) else -1
    if any(not t for t in tm[first:last + 1]):
        return False
    # no window takes rows from three chunks (scan_wp.cuh:445)
    for c in range(2, len(touch)):
        if touch[c] and touch[c - 2] and not touch[c - 2][1] < touch[c][0]:
            return False
    # head shares (windows of chunk c that also take rows from chunk c - 1), in whole blocks of 8 windows: they may not reach into the
    # block of the chunk's raw tail (scan_wp.cuh:449-454), and their J slots take at most WP_J_DOUBLES (scan_wp.cuh:461)
    jtot = 0
    for c, t in enumerate(touch):
        if not t:
            continue
        kT0, kT1 = t
        own_lo = max(kT0, touch[c - 1][1] + 1) if c > 0 and touch[c - 1] else kT0
        own_hi = min(kT1, touch[c + 1][0] - 1) if c + 1 < len(touch) and touch[c + 1] else kT1
        hs = own_lo - kT0
        nblk = (kT1 - kT0 + WP_R) // WP_R
        jzb = (hs + WP_R - 1) // WP_R
        tb = (own_hi + 1 - kT0) // WP_R if own_hi < kT1 else nblk
        if jzb > tb:
            return False
        jtot += jzb * WP_R
    return jtot <= WP_J_DOUBLES


# ------------------------------------------------------------------------------------------------------------------------------------
# the case table
PHASES = ("0", "+1", "half", "step-1")


def _phase_ms(p, step):
    return {"0": 0, "+1": 1, "half": step // 2, "step-1": step - 1}[p]


def _window_ms(k, v, step):
    return {"-1": k * step - 1, "0": k * step, "+1": k * step + 1, "+half": k * step + step // 2}[v]


WINDOWS = ("-1", "0", "+1", "+half")


def _case(name, counter, shapes, nser, k, wv, phase, T, start_row, step=None, fns=None, scrape=None, tile_declined=0, ctr_declined=(0, 0)):
    """One case: `nser` series taking `shapes` in turn; the query's window is k steps with variant wv, its start is row `start_row` of
    chunk 0's grid (negative: before the data) plus the phase; T windows.  tile_declined / ctr_declined: the series the tile kernel and
    the counter kernel (const-DDV and irregular instantiations) are expected to decline, with the cause next to the case."""
    scrape = scrape or shapes[0]["scrape"]
    step = step or scrape
    start = T0 + start_row * scrape + _phase_ms(phase, step)
    return dict(name=name, counter=counter, shapes=shapes, nser=nser, step=step, window=_window_ms(k, wv, step), start=start, T=T,
                fns=fns or (CTR_FNS if counter else SUM_FNS), tile_declined=tile_declined, ctr_declined=ctr_declined,
                what="k=%d%s phase=%s T=%d" % (k, wv if wv != "0" else "", phase, T))


def _split_shapes(rows_total, nchunks, variant, scrape=SCRAPE):
    """Chunk splits of 2, 3 or 4 chunks with junctions on (multiples of 8 rows) and off the 8-window block grid."""
    if nchunks == 2:
        a = (rows_total // 2) & ~7
        rows = (a, rows_total - a) if variant % 2 == 0 else (a + 3, rows_total - a - 3)
    elif nchunks == 3:
        a = (rows_total // 3) & ~7
        rows = (a, a, rows_total - 2 * a) if variant % 2 == 0 else (a + 5, a - 2, rows_total - 2 * a - 3)
    else:
        a = (rows_total // 4) & ~7
        rows = (a, a, a, rows_total - 3 * a) if variant % 2 == 0 else (a + 1, a + 6, a - 3, rows_total - 3 * a - 4)
    return rows


def _shift_set(step):
    """Chunk phases: on the grid, 1 ms, half a step, a step - 1 ms, and a step + 7 s after a gap of three steps."""
    return (0, 1, step // 2, step - 1, 4 * step + 7000)


def _sum_cases():
    out = []
    Ts = (1, 2, 7, 8, 9, 63, 64, 65, 481, 630)
    # k around the 9-row bound and C2's 20: every (window variant, phase) pair once, with the chunk phase, the chunk count, the
    # encodings and T rotating along
    for i, (k, wv) in enumerate(itertools.product((7, 8, 9, 20), WINDOWS)):
        phase = PHASES[(i + i // 4) % 4]
        T = Ts[i % len(Ts)]
        nch = 2 + i % 3
        sh = _shift_set(SCRAPE)[i % 5]
        total = 480 if T >= 481 else 240
        rows = _split_shapes(total, nch, i // 3)
        shifts = tuple(sh if j == 0 else (0 if i % 2 else sh) for j in range(nch - 1))
        encs = ("xr" * 3)[: nch] if i % 2 else "x" * nch
        shapes = [shape(rows, encs, shifts), shape(rows, "x" * nch, tuple(0 for _ in shifts)), shape(rows, "r" + "x" * (nch - 1), shifts)]
        if i % 4 == 1:
            shapes.append(shape(rows, encs, shifts, nan=True))
        # small T: the windows sit over the first junction; T >= 481: from before the data to past it
        start_row = -60 if T >= 481 else rows[0] - T // 2 - (3 if i % 2 else 0)
        out.append(_case("sum %d" % i, False, shapes, 5, k, wv, phase, T, start_row))
    # O apart: four chunks and windows of 70 steps (wp_max_items > 64 at any T); the last junction off the block grid
    for j, (wv, phase, T) in enumerate((("0", "half", 65), ("+half", "+1", 9), ("-1", "step-1", 64), ("+1", "0", 481))):
        rows = (120, 124, 117, 119)
        shifts = ((0, 1, 0), (SCRAPE // 2, 0, SCRAPE - 1), (0, 0, 0), (4 * SCRAPE + 7000, 0, 0))[j]
        shapes = [shape(rows, "xxrx", shifts), shape(rows, "xxxx", (0, 0, 0)), shape((240, 240), "xr", (shifts[0],))]
        out.append(_case("apart %d" % j, False, shapes, 4, 70, wv, phase, T, -40 if T >= 481 else 150 - T // 2))
    # O apart through T on records of 200 rows: the batch kernel's layout fits (it does not for the 480-row records above, where the
    # per-warp kernel takes the table)
    for j, (rows, enc, shifts, wv, phase, T) in enumerate((((97, 103), "xr", (SCRAPE // 2,), "+half", "+1", 630),
                                                           ((70, 70, 60), "rxx", (1, 0), "-1", "step-1", 481))):
        shapes = [shape(rows, enc, shifts), shape(rows, "x" * len(rows), tuple(0 for _ in shifts))]
        out.append(_case("apart batch %d" % j, False, shapes, 4, 20, wv, phase, T, -200 if T > 600 else -100))
    # J capacity: 128 rows fit WP_J_DOUBLES, 129 do not (inclusive k = 128 on the grid); one junction of 127 windows
    for j, (k, wv, phase, T) in enumerate(((127, "0", "0", 200), (127, "+half", "half", 63), (128, "0", "0", 130), (128, "-1", "+1", 200),
                                           (126, "+1", "step-1", 300))):
        rows = (200, 200) if j % 2 == 0 else (203, 197)
        shifts = ((0,), (1,), (SCRAPE // 2,), (0,), (SCRAPE - 1,))[j]
        shapes = [shape(rows, "xr", shifts), shape(rows, "xx", (0,)), shape((130, 140, 130), "xxx", (0, 0))]
        out.append(_case("jcap %d" % j, False, shapes, 3, k, wv, phase, T, 200 - T // 2 - 50))
    # scrape intervals of 1 s and 60 s
    for j, (scr, k, wv, phase, T, nch) in enumerate(((1000, 20, "+half", "half", 65, 3), (1000, 9, "-1", "step-1", 8, 2),
                                                     (60000, 20, "+1", "+1", 481, 2), (60000, 8, "0", "half", 9, 4))):
        total = 480 if T >= 481 else 240
        rows = _split_shapes(total, nch, j)
        shifts = tuple((scr // 2, scr - 1, 1)[u % 3] if u == 0 else 0 for u in range(nch - 1))
        shapes = [shape(rows, "x" * nch, shifts, scrape=scr), shape(rows, "r" * nch, tuple(0 for _ in shifts), scrape=scr)]
        out.append(_case("scrape %d %d" % (scr, j), False, shapes, 4, k, wv, phase, T, -60 if T >= 481 else rows[0] - T // 2))
    # query step != scrape interval: every series goes to the v2 kernel (timestamp slope != step: scan_wp.cuh:166, scan_tile.cuh:212)
    for j, (mul, k, wv, phase, T) in enumerate(((2, 10, "0", "0", 65), (4, 9, "+half", "half", 30), (1 / 3, 30, "-1", "+1", 100))):
        step = int(SCRAPE * mul)
        rows = (200, 160)
        shapes = [shape(rows, "xr", (0,)), shape(rows, "xx", (SCRAPE // 2,))]
        c = _case("step %s" % mul, False, shapes, 4, k, wv, phase, T, 20, step=step, tile_declined=4)
        out.append(c)
    return out


def _ctr_cases():
    out = []
    Ts = (1, 2, 7, 8, 9, 63, 64, 65, 481, 630)
    for i, (k, wv) in enumerate(itertools.product((4, 8, 20), WINDOWS)):
        phase = PHASES[(i + i // 4) % 4]
        T = Ts[(3 * i) % len(Ts)]
        nch = 2 + i % 3
        sh = _shift_set(SCRAPE)[i % 5]
        total = 480 if T >= 481 else 240
        rows = _split_shapes(total, nch, i // 3)
        shifts = tuple(sh if j == 0 else (0 if i % 2 else sh) for j in range(nch - 1))
        encs = ("xr" * 3)[: nch] if i % 2 else "x" * nch
        shapes = [shape(rows, encs, shifts), shape(rows, "x" * nch, tuple(0 for _ in shifts))]
        start_row = -60 if T >= 481 else rows[0] - T // 2 - (2 if i % 2 else 0)
        out.append(_case("ctr %d" % i, True, shapes, 4, k, wv, phase, T, start_row))
    # query step != scrape interval: the const-DDV instantiation declines every series (slope != step, scan_wp.cuh:166); the
    # irregular one takes them all
    for j, (mul, k, wv, phase, T) in enumerate(((2, 10, "0", "half", 65), (4, 6, "+1", "0", 30), (1 / 3, 30, "+half", "step-1", 100))):
        step = int(SCRAPE * mul)
        rows = (200, 160)
        shapes = [shape(rows, "xr", (0,)), shape(rows, "xx", (SCRAPE // 2,))]
        out.append(_case("ctr step %s" % mul, True, shapes, 4, k, wv, phase, T, 20, step=step, ctr_declined=(4, 0)))
    # 1 s and 60 s scrapes
    for j, (scr, k, wv, phase, T) in enumerate(((1000, 20, "+half", "half", 65), (60000, 5, "-1", "+1", 481))):
        rows = (240, 240)
        shapes = [shape(rows, "xr", (scr // 2,), scrape=scr), shape(rows, "xx", (0,), scrape=scr)]
        out.append(_case("ctr scrape %d" % scr, True, shapes, 4, k, wv, phase, T, -60 if T >= 481 else 240 - T // 2))
    return out


def _rotate(cases):
    """Two functions per case, taking turns over the class's functions, and the batch kernel at the product's shape (15 consumer warps,
    B = 15, 2 buffers) on every third case: the emulator runs 512 fibers per CTA there."""
    for i, c in enumerate(cases):
        fns = c["fns"]
        c["fns"] = (fns[i % len(fns)], fns[(i + 2) % len(fns)])
        c["product"] = i % 3 == 0
    return cases


CASES = _rotate(_sum_cases() + _ctr_cases())


def case_series(case):
    """[chunks per series] of a case; series s takes shape s % len(shapes); the values depend on the case and the series."""
    out = []
    for s in range(case["nser"]):
        sh = case["shapes"][s % len(case["shapes"])]
        out.append(series_chunks(sh, case["counter"], zlib.crc32(repr((case["name"], s)).encode())))
    return out


def wp_declined_ids(case, inclusive, series=None):
    """The series of a case the v4 SUM kernels are predicted to decline."""
    series = series if series is not None else case_series(case)
    q = query_of(case, inclusive)
    return [s for s, ch in enumerate(series) if not wp_accepts(ch, q)]


def wp_declined(case, inclusive, series=None):
    """How many series of a case the v4 SUM kernels are predicted to decline."""
    return len(wp_declined_ids(case, inclusive, series))


def _all_or_none(case, count):
    """The ids of a per-case decline count: the tile and counter kernels decline every series of a case or none."""
    assert count in (0, case["nser"]), (case["name"], count)
    return list(range(count))


def write_cases(path, cases=CASES):
    """The cases as the emulator driver (tests/cpp/scan_geometry_emul.cpp) reads them: whitespace-separated numbers, one query per
    (case, range mode) with the series each kernel is expected to decline (v4 SUM, tile, counter const-DDV, counter irregular: a count
    and the series ids), then the series' chunks (timestamps, value bits as hex)."""
    lines = ["%d" % (2 * len(cases))]
    for case in cases:
        series = case_series(case)
        for inclusive in (1, 0):
            start, step, end, window, T, _ = query_of(case, inclusive)
            lines.append("%s %d %d %d %d %d %d %d %d" % (case["name"].replace(" ", "_"), int(case["counter"]), int(case["product"]), start, step, end,
                                                       window, T, inclusive))
            lines.append("%d %s" % (len(case["fns"]), " ".join(str(f) for f in case["fns"])))
            for ids in (wp_declined_ids(case, inclusive, series), _all_or_none(case, case["tile_declined"]),
                        _all_or_none(case, case["ctr_declined"][0]), _all_or_none(case, case["ctr_declined"][1])):
                lines.append(" ".join(str(x) for x in [len(ids)] + ids))
            lines.append("%d" % len(series))
            for chunks in series:
                lines.append("%d" % len(chunks))
                for ts, v, enc in chunks:
                    lines.append("%s %d" % (enc, len(ts)))
                    lines.append(" ".join(str(int(t)) for t in ts))
                    lines.append(" ".join("%x" % b for b in v.view(np.uint64)))
    with open(path, "w") as f:
        f.write("\n".join(lines) + "\n")
