"""Finished windows of the v4 SUM kernel with a CTA-wide record stream written straight into the staged result row by the window blocks,
and a fix-up of only the junction, raw and gap windows, on the SIMT emulator (tests/cpp/wp_stage_emul.cpp).  T = 1 .. 630, both row
phases, chunk junctions on and off the block grid with 2, 3 and 4 chunks, gap windows, sum / avg / count_over_time and rate, declined
series right after a stored row, partial last batches, O in V's place and apart; bit-exact against the oracle, equal scan counters,
nothing written outside the rows."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_wp_batch_staged_windows_on_the_simt_emulator(tmp_path):
    """In-order and pseudo-random fiber schedules; bulk copies are deferred as late as the program allows."""
    src = str(tmp_path / "scan_kernels_cusim.cu")          # function-scope __shared__ (merge_partials_kernel) -> static
    subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cpp", "make_cusim_src.py"), os.path.join(ROOT, "filodb_b200", "csrc", "scan_kernels.cu"), src], check=True)
    exe = str(tmp_path / "wp_stage_emul")
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", "-I", "/usr/local/cuda/include",
                    "-I", os.path.join(ROOT, "filodb_b200", "csrc"), '-DSCAN_SRC="%s"' % src,
                    os.path.join(ROOT, "tests", "cpp", "wp_stage_emul.cpp"), "-o", exe], check=True)
    for seed in ("0", "20261017"):
        r = subprocess.run([exe, seed], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "bit-exact, guards intact" in r.stdout, r.stdout
        for t in (1, 2, 3, 20, 27, 241, 480, 481, 630):
            assert "T = %d ok" % t in r.stdout, (t, r.stdout)
        for lay in ("O in V, out + 0 B", "O in V, out + 8 B", "O apart, out + 0 B", "O apart, out + 8 B"):
            assert lay in r.stdout, (lay, r.stdout)
        for what in ("three chunks", "four chunks", "gap between chunks", "junction off the block grid"):
            assert what in r.stdout, (what, r.stdout)
        assert "rate: C2 shape, T = 481 (O in V, out + 8 B, 15 consumers, B = 15 x 2): 40 series, T = 481 ok" in r.stdout, r.stdout
