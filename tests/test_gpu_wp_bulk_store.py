"""GPU: result rows of the v4 SUM kernel with a CTA-wide record stream (scan_wp_batch_kernel), which stores each row's 16-byte-aligned
span with one bulk copy and the window outside it directly.  filo_query_device writes into a caller's buffer whose base is 16-byte
aligned or 8 mod 16, at odd and even T; the rows must be bit-exact against the CPU oracle and nothing outside them may change.  The table
has two full batches per CTA and a partial third, so every consumer warp stores at least two rows back to back (asserted with filo_query's
kernel choice)."""
import os
import zlib

import numpy as np
import pytest

from tests.test_gpu_parity import assert_same, build_store
from tests.test_scan_path import build_scan_path, scan_path

pytestmark = pytest.mark.gpu
T0 = 1_700_000_000_000
GUARD = 0x7FF4A5A5C3C3E1E1          # a signalling-NaN pattern no kernel writes
G = 8                               # guard words on each side


@pytest.fixture(scope="module")
def gpu(tmp_path_factory):
    import torch
    import filodb_b200.capi as capi
    ctx = capi.Context(0)
    yield capi, ctx, build_scan_path(tmp_path_factory.mktemp("scan_path")), torch.cuda.get_device_properties(0).multi_processor_count
    ctx.close()


@pytest.mark.parametrize("nan_frac", [0.0, 0.002], ids=["regular", "declined"])
def test_bulk_result_rows_at_both_alignments(gpu, oracle, nan_frac):
    import torch
    capi, ctx, exe, sms = gpu; o = oracle
    n = 2 * 15 * sms + 7              # two full batches of 15 per CTA and a partial third on some: every consumer warp stores rows back to back
    rng = np.random.default_rng(zlib.crc32(repr(("wp_bulk_store", nan_frac)).encode()))
    st = build_store(o, rng, n, "gauge", o.VAL_XOR, 0, False, nan_frac)
    tab = ctx.load_series(*st.all_info_addrs())
    ti = tab.info()
    rec = int(np.diff(tab.read_arena(0, n)[1]).max())
    for T in (1, 2, 27, 460, 461):
        start, step, window = T0 + 300000, 15000, 300000
        end = start + (T - 1) * step
        p = scan_path(exe, rec=rec, rows=ti.max_rows_per_series, chunks=ti.max_chunks_per_series, T=T, wrows=window // step + 1, n=n, sms=sms)
        assert p["kernel"] == "batch" and p["series_per_warp"] >= 2, (T, p)
        for name in ("FN_SUM_OVER_TIME", "FN_AVG_OVER_TIME", "FN_COUNT_OVER_TIME"):
            exp = st.query(getattr(o, name), start, step, end, window, threads=os.cpu_count() or 1)
            for off in (0, 1):        # the rows start at a 16-byte-aligned address, or at 8 mod 16
                buf = torch.full((2 * G + n * T + 2,), GUARD, dtype=torch.int64, device="cuda")
                assert buf.data_ptr() % 16 == 0
                rows = buf[G + off:G + off + n * T].view(torch.float64)
                ctx.query_device(tab, getattr(capi, name), start, step, end, window, rows.data_ptr())
                torch.cuda.synchronize()
                h = buf.cpu().numpy()
                what = "%s T=%d out+%dB" % (name, T, 8 * off)
                outside = np.concatenate([h[:G + off], h[G + off + n * T:]])
                assert (outside == GUARD).all(), what + ": words outside the rows were written"
                assert_same(h[G + off:G + off + n * T].view(np.float64).reshape(n, T), exp, what)
                assert ctx.last_stats["samples_scanned"] == st.last_stats["samples_scanned"], what
    tab.free()
