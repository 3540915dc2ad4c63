"""The per-series scan kernels across query geometry on the SIMT emulator (tests/cpp/scan_geometry_emul.cpp): the cases of
tests/scan_geometry_cases.py (start phases, windows on and off the step grid, exclusive ranges, later chunks off chunk 0's grid, odd and
even T, 1 s / 15 s / 60 s scrapes, steps that are not the scrape interval) in both range modes, on scan_wp_batch_kernel (O on V and O
apart, a small shape and the product's), scan_wp_sum_kernel (one and two record buffers), the tile kernel and both instantiations of
scan_wp_ctr_kernel.  Every value is bit-exact against the oracle, the scan counters match, and every kernel declines exactly the series
predicted (the brute-force predictor of the case table for the two v4 SUM kernels, a per-case count for the others)."""
import os
import subprocess
import sys

import numpy as np

from tests import scan_geometry_cases as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_case_table_spans_the_geometry_axes():
    """The table combines the axes it promises, and the predictor both takes and declines series in each range mode."""
    Ts = {c["T"] for c in G.CASES}
    assert {1, 2, 7, 8, 9, 63, 64, 65, 481, 630} <= Ts
    assert {1000, 15000, 60000} <= {s["scrape"] for c in G.CASES for s in c["shapes"]}
    assert {30000, 60000, 5000} <= {c["step"] for c in G.CASES if c["step"] != c["shapes"][0]["scrape"]}
    phases = {(c["start"] - G.T0) % c["step"] for c in G.CASES if c["step"] == G.SCRAPE}
    assert {0, 1, G.SCRAPE // 2, G.SCRAPE - 1} <= phases
    assert {0, 1, G.SCRAPE // 2, G.SCRAPE - 1} <= {c["window"] % c["step"] for c in G.CASES if c["step"] == G.SCRAPE}
    shifts = {x % G.SCRAPE for c in G.CASES for s in c["shapes"] for x in s["shifts"] if s["scrape"] == G.SCRAPE}
    assert {1, G.SCRAPE // 2, G.SCRAPE - 1, 7000} <= shifts
    assert {2, 3, 4} <= {len(s["rows"]) for c in G.CASES for s in c["shapes"]}
    for inclusive in (1, 0):
        d = [G.wp_declined(c, inclusive) for c in G.CASES if not c["counter"]]
        n = [c["nser"] for c in G.CASES if not c["counter"]]
        assert 0 < sum(d) < sum(n)
    # cases where only the range mode decides: a shifted chunk keeps its row count in one mode and not in the other
    assert any(G.wp_declined(c, 1) != G.wp_declined(c, 0) for c in G.CASES if not c["counter"])


def test_predictor_counts_rows_on_each_chunk_grid():
    """[5m] at a 15 s step on the grid: 21 rows inclusive, 20 exclusive; a chunk half a step off the grid has 20 in both modes, so the
    series is declined inclusive and taken exclusive; a window of 8 steps on the grid holds 9 rows (taken), 8 exclusive (declined)."""
    ts0 = G.T0 + np.arange(200, dtype=np.int64) * G.SCRAPE
    ts1 = G.T0 + np.arange(200, 400, dtype=np.int64) * G.SCRAPE + G.SCRAPE // 2
    v = np.full(200, 15.5)
    two = [(ts0, v, "x"), (ts1, v, "x")]
    q = lambda window, incl: (G.T0 + 150 * G.SCRAPE, G.SCRAPE, G.T0 + 250 * G.SCRAPE, window, 101, incl)
    assert not G.wp_accepts(two, q(300000, 1)) and G.wp_accepts(two, q(300000, 0))
    assert G.wp_accepts(two[:1], q(120000, 1)) and not G.wp_accepts(two[:1], q(120000, 0))


def test_scan_geometry_on_the_simt_emulator(tmp_path):
    """In-order and pseudo-random fiber schedules; each seed runs the table in two halves, the four runs side by side."""
    src = str(tmp_path / "scan_kernels_cusim.cu")          # function-scope __shared__ (merge_partials_kernel) -> static
    subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cpp", "make_cusim_src.py"), os.path.join(ROOT, "filodb_b200", "csrc", "scan_kernels.cu"), src], check=True)
    exe = str(tmp_path / "scan_geometry_emul")
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", "-I", "/usr/local/cuda/include",
                    "-I", os.path.join(ROOT, "filodb_b200", "csrc"), '-DSCAN_SRC="%s"' % src,
                    os.path.join(ROOT, "tests", "cpp", "scan_geometry_emul.cpp"), "-o", exe], check=True)
    halves = []
    for h in (0, 1):
        path = str(tmp_path / ("cases%d.txt" % h))
        G.write_cases(path, G.CASES[h::2])
        halves.append(path)
    procs = [(seed, path, subprocess.Popen([exe, seed, path], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
             for seed in ("0", "20261018") for path in halves]
    runs = 0
    kernels = set()
    for seed, path, p in procs:
        out, _ = p.communicate()
        assert p.returncode == 0, "seed %s, %s:\n%s" % (seed, os.path.basename(path), out)
        assert "bit-exact" in out and "as predicted" in out, out
        runs += int(out.split(" runs, ")[0].split()[-1])
        kernels |= {line.split(":")[0] for line in out.splitlines() if line.endswith(" runs")}
    assert kernels == {"batch O on V 3/3/2", "batch O on V product", "batch O apart 3/3/2", "batch O apart product",
                       "sum one record buffer", "sum two record buffers", "tile", "ctr const", "ctr irregular"}, kernels
    assert runs >= 2 * 800, runs
