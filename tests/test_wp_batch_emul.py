"""The v4 SUM kernel with a CTA-wide record stream on the SIMT emulator (tests/cpp/wp_batch_emul.cpp): a producer warp copies batches
of consecutive records and parses their headers, consumer warps take the series in turn.  CTAs without series, partial batches and a
batch of one series, records of different sizes in one batch, plan- and value-declined series at every batch position, memo misses
inside a batch, sum / avg / count_over_time and rate on a delta schema, T from 20 to 630, with O in V's place and apart, bit-exact
against the oracle."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_wp_batch_record_stream_on_the_simt_emulator(tmp_path):
    """In-order and pseudo-random fiber schedules, bulk copies deferred adversarially; the scan counters must match the oracle's."""
    src = str(tmp_path / "scan_kernels_cusim.cu")          # function-scope __shared__ (merge_partials_kernel) -> static
    subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cpp", "make_cusim_src.py"), os.path.join(ROOT, "filodb_b200", "csrc", "scan_kernels.cu"), src], check=True)
    exe = str(tmp_path / "wp_batch_emul")
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", "-I", "/usr/local/cuda/include",
                    "-I", os.path.join(ROOT, "filodb_b200", "csrc"), '-DSCAN_SRC="%s"' % src,
                    os.path.join(ROOT, "tests", "cpp", "wp_batch_emul.cpp"), "-o", exe], check=True)
    for seed in ("0", "20261017"):
        r = subprocess.run([exe, seed], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "OK 41 runs of 12 cases" in r.stdout and "bit-exact" in r.stdout, r.stdout
        assert "T = 630 ok" in r.stdout and "T = 481 ok" in r.stdout and "T = 27 ok" in r.stdout and "T = 20 ok" in r.stdout, r.stdout
        assert "15 consumers, B = 15 x 2" in r.stdout, r.stdout
