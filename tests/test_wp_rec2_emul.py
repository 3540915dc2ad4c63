"""The v4 SUM kernel with two record buffers per warp on the SIMT emulator (tests/cpp/wp_rec2_emul.cpp): warps with zero, one, two
and many series, consecutive series with different plans, declined series in either buffer, sum / avg / count_over_time and rate on a
delta schema, T from 20 to 630, with O in V's place and apart, bit-exact against the oracle."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_wp_two_record_buffers_on_the_simt_emulator(tmp_path):
    """In-order and pseudo-random fiber schedules; the scan counters must match the oracle's."""
    src = str(tmp_path / "scan_kernels_cusim.cu")          # function-scope __shared__ (merge_partials_kernel) -> static
    subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cpp", "make_cusim_src.py"), os.path.join(ROOT, "filodb_b200", "csrc", "scan_kernels.cu"), src], check=True)
    exe = str(tmp_path / "wp_rec2_emul")
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", "-I", "/usr/local/cuda/include",
                    "-I", os.path.join(ROOT, "filodb_b200", "csrc"), '-DSCAN_SRC="%s"' % src,
                    os.path.join(ROOT, "tests", "cpp", "wp_rec2_emul.cpp"), "-o", exe], check=True)
    for seed in ("0", "20261017"):
        r = subprocess.run([exe, seed], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "OK 17 runs of 9 cases" in r.stdout and "bit-exact" in r.stdout, r.stdout
        assert "T = 630 ok" in r.stdout and "T = 481 ok" in r.stdout, r.stdout
