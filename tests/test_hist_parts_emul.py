"""The cross-GPU histogram sum on the SIMT emulator (tests/cpp/hist_parts_emul.cpp): the SUM outputs of W tables cut from one series set,
from both histogram scan kernels, folded in rank order by hist_merge_parts_kernel, bit-exact against the oracle with the quantile bits
included; and the invariant the merge's emptiness test rests on (a SUM output cell is all-NaN exactly where its group produced nothing)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_hist_partials_merge_on_the_simt_emulator(tmp_path):
    """W = 1, 2, 3, 8 (contiguous and interleaved splits, empty tables); groups empty on some ranks, on rank 0 only and on every rank;
    custom, geometric and otel buckets; nb = 1, 6-20 and 64; T over several thread blocks; q NaN, < 0, > 1; a non-monotonic partial
    copied and made monotonic only by a second add; rate, increase, sum_over_time and last; in-order and pseudo-random fiber schedules."""
    v1 = str(tmp_path / "hist_kernels_cusim.cu")
    subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cpp", "make_cusim_src.py"), os.path.join(ROOT, "filodb_b200", "csrc", "hist_kernels.cu"), v1], check=True)
    exe = str(tmp_path / "hist_parts_emul")
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", "-I", "/usr/local/cuda/include",
                    "-I", os.path.join(ROOT, "filodb_b200", "csrc"), '-DHIST_V1_SRC="%s"' % v1,
                    os.path.join(ROOT, "tests", "cpp", "hist_parts_emul.cpp"), "-o", exe], check=True)
    for seed in ("0", "5"):
        r = subprocess.run([exe, seed], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "OK 14 cases" in r.stdout and "bit-exact" in r.stdout, r.stdout
