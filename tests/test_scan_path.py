"""The per-series kernel choice of filo_query (scan_path, scan_wp_layout.h), through the host program tests/cpp/scan_path.cpp: the C2 shape
(480 rows in chunks of 400 + 80, T = 481, rate()[5m] step 15s on a gauge) runs on scan_wp_batch_kernel with O on V, 15 series per batch
in two batch buffers, one CTA per SM."""
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_scan_path(out_dir):
    exe = os.path.join(str(out_dir), "scan_path")
    subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Wextra", "-I", os.path.join(ROOT, "filodb_b200", "csrc"),
                    os.path.join(ROOT, "tests", "cpp", "scan_path.cpp"), "-o", exe], check=True)
    return exe


def scan_path(exe, **kw):
    """The choice for one table shape, as a dict of ints (and the kernel's name)."""
    r = subprocess.run([exe] + ["%s=%s" % (k, v) for k, v in kw.items()], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    out = dict(line.split("=", 1) for line in r.stdout.split())
    return {k: (v if k in ("kernel", "fused_kernel") else int(v)) for k, v in out.items()}


def test_c2_shape_selects_the_batch_kernel_with_o_on_v(tmp_path):
    exe = build_scan_path(tmp_path)
    # C2's records: 16-byte header, two chunk entries, a const-DDV timestamp vector and an XOR value vector per chunk, ~3.8 KB
    for rec in (3712, 3808, 3904):
        p = scan_path(exe, rec=rec, rows=480, chunks=2, T=481, wrows=21, n=5_000_000, cls="sum", sms=132)
        assert p["kernel"] == "batch" and p["alias"] == 1, p
        assert p["B"] == 15 and p["warps"] == 15 and p["rec_bufs"] == 2 and p["grid"] == 132, p
        assert p["smem"] <= 227 * 1024, p
    # depth: 5 * 15 * 132 series give every consumer warp five series, the last in round u = 4 // 2 = 2; one series fewer leaves the
    # last CTA's batch 4 empty
    assert scan_path(exe, rec=3808, rows=480, chunks=2, T=481, wrows=21, n=5 * 15 * 132)["series_per_warp"] == 5
    assert scan_path(exe, rec=3808, rows=480, chunks=2, T=481, wrows=21, n=5 * 15 * 132)["rounds"] == 2
    assert scan_path(exe, rec=3808, rows=480, chunks=2, T=481, wrows=21, n=5 * 15 * 132 - 1)["rounds"] == 1
    # rate on a counter schema runs on the counter kernel; without the v2 kernel no per-series kernel runs in front of it
    assert scan_path(exe, rec=3808, rows=480, chunks=2, T=481, wrows=21, n=5_000_000, cls="counter")["kernel"] == "ctr"
    assert scan_path(exe, rec=3808, rows=480, chunks=2, T=481, wrows=21, n=5_000_000, v2=0)["kernel"] == "v2"


def c5_items(S, G, sms):
    """Work items of a table of S series in G groups of near-equal size (C5: synth_group_ids hashes series over 100 clusters)."""
    from tests.fused_items import seg_for
    seg = seg_for(S, sms)
    sizes = [S // G + (1 if g < S % G else 0) for g in range(G)]
    return seg, sum((n + seg - 1) // seg for n in sizes)


def test_c5_shape_folds_items_of_147_series_on_the_counter_kernel(tmp_path):
    exe = build_scan_path(tmp_path)
    seg, items = c5_items(5_000_000, 100, 132)
    assert seg == 147 and items == 34_100
    p = scan_path(exe, rec=3808, rows=480, chunks=2, T=481, wrows=21, n=5_000_000, cls="counter", fused=1, items=items, sms=132)
    # the accumulator row of 481 windows (and its NaN counts) leaves room for 15 warps per SM
    assert p["fused_kernel"] == "ctr" and p["warps"] == 15 and p["fused_grid"] == 132, p
    assert p["items_per_warp"] == items // (132 * 15) == 17, p
    # C3-const: increase()[1m] by 1000 jobs; C3's jittered timestamps take the <= 16-warp irregular instantiation
    seg3, items3 = c5_items(5_000_000, 1000, 132)
    p = scan_path(exe, rec=3808, rows=480, chunks=2, T=481, wrows=5, n=5_000_000, cls="counter", fused=1, items=items3, sms=132)
    assert seg3 == 147 and p["fused_kernel"] == "ctr" and p["fused_grid"] == 132 and p["items_per_warp"] == items3 // (132 * p["warps"]), p
    p = scan_path(exe, rec=3808, rows=480, chunks=2, T=481, wrows=5, n=5_000_000, cls="counter", fused=1, irr=1, items=items3, sms=132)
    assert p["fused_kernel"] == "ctr" and p["warps"] <= 16, p


def test_fused_path_leaves_tile_and_counter_kernels_above_512_windows(tmp_path):
    """The tile kernel's accumulators hold TILE_AGG_ACC * TILE_THREADS = 512 windows; the counter kernel's fused mode takes the same
    bound: at T = 513 both classes go to the v2 aggregate kernel alone."""
    exe = build_scan_path(tmp_path)
    for cls, kernel in (("counter", "ctr"), ("sum", "tile")):
        for moments in (0, 1):
            kw = dict(rec=1200, rows=120, chunks=3, wrows=21, n=300_000, cls=cls, fused=1, moments=moments, items=40_000, sms=132)
            p = scan_path(exe, T=512, **kw)
            assert p["fused_kernel"] == kernel and p["fused_grid"] in (132, 264), p
            p = scan_path(exe, T=513, **kw)
            assert p["fused_kernel"] == "v2" and p["fused_grid"] == 0 and p["items_per_warp"] == -1, p
    # min / max / last over time: no fused ctr / tile kernel at any T
    assert scan_path(exe, rec=1200, rows=120, chunks=3, T=40, wrows=21, n=1000, cls="minmax", fused=1, items=1000)["fused_kernel"] == "v2"


def test_fused_grid_matches_the_inline_rule_it_replaced(tmp_path):
    """Over a sweep of shapes the fused grid is the one filo_query computed inline before scan_path returned it:
    ctr: max(1, min(ceil(n_items / warps), SMs)); tile: max(1, min(n_items, SMs * tile CTAs per SM))."""
    exe = build_scan_path(tmp_path)
    rng = np.random.default_rng(17)
    seen = set()
    for _ in range(60):
        cls = ["counter", "sum"][int(rng.integers(2))]
        rows = int(rng.integers(30, 2000)); chunks = int(rng.integers(1, 6)); rec = 16 + chunks * 48 + rows * int(rng.integers(1, 9))
        T = int(rng.choice([1, 7, 100, 481, 511, 512, 513, 900])); wrows = int(rng.choice([2, 5, 21, 89, 3001]))
        n = int(rng.integers(1, 6_000_000)); sms = int(rng.choice([1, 8, 114, 132]))
        items = int(rng.integers(1, max(2, n)))
        for moments in (0, 1):
            p = scan_path(exe, rec=rec, rows=rows, chunks=chunks, T=T, wrows=wrows, n=n, cls=cls, fused=1, moments=moments, irr=int(rng.integers(2)),
                          items=items, sms=sms)
            k = p["fused_kernel"]
            seen.add(k)
            if k == "ctr":
                assert p["fused_grid"] == max(1, min(-(-items // p["warps"]), sms)), p
            elif k == "tile":
                assert p["fused_grid"] in (max(1, min(items, sms)), max(1, min(items, 2 * sms))) and T <= 512, p
            else:
                assert p["fused_grid"] == 0 and (T > 512 or cls == "counter" or p["kernel"] == "v2"), p
    assert seen == {"ctr", "tile", "v2"}, seen
