"""GPU: the v4 SUM kernel with a CTA-wide record stream (scan_wp_batch_kernel) writes finished windows straight into the staged result
row from its window blocks and fixes up only junction, raw and gap windows.  filo_query_device writes into a caller's buffer whose base
is 16-byte aligned or 8 mod 16; chunk junctions on and off the block grid with 2, 3 and 4 chunks, a time gap between chunks and windows
before the data; the rows must be bit-exact against the CPU oracle and nothing outside them may change.  Each table has two full rounds
of series per CTA and a partial third, so every warp stores at least two rows back to back (asserted with filo_query's kernel choice).
Series of 480 rows in four chunks take too much shared memory for the batch buffers: that table runs on scan_wp_sum_kernel (one record
buffer per warp, O on V), which finishes and stores its rows straight from the window blocks."""
import os
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
# Tables sized so that the batch kernel takes them (400 rows where a series has four chunks): O on V where every plan is one pass (two
# chunks up to T = 481, four up to T = 424), and records small enough for its batch buffers with O apart (T = 630).  (name, chunk shapes,
# gap in steps after the first chunk, queries as (T, first window's row), the kernel filo_query picks, series per round of one CTA)
TABLES = [
    ("two chunks", [(400, 80), (237, 243), (240, 240)], 0, [(1, 400), (2, 399), (3, 236), (20, 225), (27, 0), (241, 100), (480, 0), (481, 0)], "batch", 15),
    ("three and four chunks", [(80, 160, 160), (100, 100, 100, 100), (60, 60, 60, 60)], 0, [(1, 120), (20, 110), (241, -20), (400, 0)], "batch", 15),
    ("gap between chunks", [(200, 280), (237, 243)], 45, [(27, 210), (241, 100), (481, 0)], "batch", 15),
    ("windows past 512", [(120, 120), (117, 123)], 0, [(630, -60)], "batch", 15),
    ("480 rows in four chunks", [(100, 190, 190), (120, 120, 120, 120), (60, 60, 60, 60)], 0, [(1, 120), (20, 110), (241, -20), (400, 0)], "sum", 20),
]


@pytest.fixture(scope="module")
def gpu(tmp_path_factory):
    import torch
    import filodb_b200.capi as capi
    ctx = capi.Context(0)
    yield capi, ctx, build_scan_path(tmp_path_factory.mktemp("scan_path")), torch.cuda.get_device_properties(0).multi_processor_count
    ctx.close()


def _store(o, rng, n, shapes, gap, nan_frac):
    st = o.Store()
    for s in range(n):
        chunks = list(shapes[s % len(shapes)])
        rows = sum(chunks)
        r = np.arange(rows, dtype=np.int64)
        ts = T0 + (r + np.where(r >= chunks[0], gap, 0)) * STEP
        v = 15 + np.sin(np.arange(1, rows + 1)) + rng.normal(0, 1, rows)
        if nan_frac:
            v[rng.random(rows) < nan_frac] = np.nan
        st.add_series_rows(ts, v, chunks, val_mode=o.VAL_XOR, detect_drops=False)
    return st


@pytest.mark.parametrize("nan_frac", [0.0, 0.002], ids=["regular", "declined"])
@pytest.mark.parametrize("table", TABLES, ids=[t[0] for t in TABLES])
def test_staged_windows_and_fixup_at_both_alignments(gpu, oracle, table, nan_frac):
    import torch
    capi, ctx, exe, sms = gpu; o = oracle
    tname, shapes, gap, queries, kernel, per_cta = table
    n = 2 * per_cta * sms + 7         # two full rounds per CTA and a partial third on some: every warp stores rows back to back
    rng = np.random.default_rng(zlib.crc32(repr(("wp_stage", tname, nan_frac)).encode()))
    st = _store(o, rng, n, shapes, gap, nan_frac)
    tab = ctx.load_series(*st.all_info_addrs())
    ti = tab.info()
    rec = int(np.diff(tab.read_arena(0, n)[1]).max())
    for T, first in queries:
        start, window = T0 + first * STEP, 300000
        end = start + (T - 1) * STEP
        p = scan_path(exe, rec=rec, rows=ti.max_rows_per_series, chunks=ti.max_chunks_per_series, T=T, wrows=window // STEP + 1, n=n, sms=sms)
        assert p["kernel"] == kernel and p["series_per_warp"] >= 2, (tname, T, p)
        if kernel == "batch": assert p["warps"] == per_cta == p["B"], (tname, T, p)
        for name in ("FN_SUM_OVER_TIME", "FN_AVG_OVER_TIME", "FN_COUNT_OVER_TIME", "FN_RATE"):
            exp = st.query(getattr(o, name), start, STEP, end, window, threads=os.cpu_count() or 1)
            for off in (0, 1):        # the rows start at a 16-byte-aligned address, or at 8 mod 16
                buf = torch.full((2 * G + n * T + 2,), GUARD, dtype=torch.int64, device="cuda")
                assert buf.data_ptr() % 16 == 0
                rows = buf[G + off:G + off + n * T].view(torch.float64)
                ctx.query_device(tab, getattr(capi, name), start, STEP, end, window, rows.data_ptr())
                torch.cuda.synchronize()
                h = buf.cpu().numpy()
                what = "%s: %s T=%d out+%dB" % (tname, name, T, 8 * off)
                outside = np.concatenate([h[:G + off], h[G + off + n * T:]])
                assert (outside == GUARD).all(), what + ": words outside the rows were written"
                assert_same(h[G + off:G + off + n * T].view(np.float64).reshape(n, T), exp, what)
                assert ctx.last_stats["samples_scanned"] == st.last_stats["samples_scanned"], what
    tab.free()
