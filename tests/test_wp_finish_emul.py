"""The finish pass of the v4 SUM kernel on the SIMT emulator (tests/cpp/wp_finish_emul.cpp): every window class of the plan
(finished by its window block, raw sum to finish, chunk junction, no rows) over sum / avg / count_over_time and rate on a delta
schema, with O in V's place and apart, bit-exact against the oracle."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_wp_finish_pass_on_the_simt_emulator(tmp_path):
    """1-4 chunks; windows without rows in front, between chunks and behind; T = 20 and 27 (< 32) and T not a multiple of 32; head
    shares of 20 and 40 windows (longer than one block and than 32 windows); raw f64 chunks next to XOR chunks; chunk blocks on and
    off O's 9-word grid; plans of more than 64 blocks (T = 600, 1000: two window passes and windows past 512).  No series may be
    declined; in-order and pseudo-random fiber schedules."""
    src = str(tmp_path / "scan_kernels_cusim.cu")          # function-scope __shared__ (merge_partials_kernel) -> static
    subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cpp", "make_cusim_src.py"), os.path.join(ROOT, "filodb_b200", "csrc", "scan_kernels.cu"), src], check=True)
    exe = str(tmp_path / "wp_finish_emul")
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", "-I", "/usr/local/cuda/include",
                    "-I", os.path.join(ROOT, "filodb_b200", "csrc"), '-DSCAN_SRC="%s"' % src,
                    os.path.join(ROOT, "tests", "cpp", "wp_finish_emul.cpp"), "-o", exe], check=True)
    for seed in ("0", "20261016"):
        r = subprocess.run([exe, seed], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "OK 18 runs of 11 cases" in r.stdout and "bit-exact" in r.stdout, r.stdout
