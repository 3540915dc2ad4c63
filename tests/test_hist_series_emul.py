"""The per-series and `last` modes of both histogram kernels on the SIMT emulator (tests/cpp/hist_series_emul.cpp), bit-exact against the
oracle with the quantile bits included: hist_scan2_kernel<SERIES, LAST> (bucket rows + quantile, and the quantile alone through the CTA's
window columns), the first kernel's `last` and per-series quantile stage, and the fused `last` + quantile on both kernels."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_hist_series_modes_on_the_simt_emulator(tmp_path):
    """rate / increase / last / sum_over_time / delta rate; custom, geometric and otel buckets; resets inside chunks and at chunk starts;
    jittered timestamps; 1-8 chunks; the default lookback; windows without a sample; a window whose only row sits on its start (inclusive and exclusive); q in {0, 1, < 0, > 1}; 70 series (two runs of 64 per
    CTA); in-order and pseudo-random fiber schedules."""
    v1 = str(tmp_path / "hist_kernels_cusim.cu")
    subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cpp", "make_cusim_src.py"), os.path.join(ROOT, "filodb_b200", "csrc", "hist_kernels.cu"), v1], check=True)
    exe = str(tmp_path / "hist_series_emul")
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", "-I", "/usr/local/cuda/include",
                    "-I", os.path.join(ROOT, "filodb_b200", "csrc"), '-DHIST_V1_SRC="%s"' % v1,
                    os.path.join(ROOT, "tests", "cpp", "hist_series_emul.cpp"), "-o", exe], check=True)
    for seed in ("0", "11"):
        r = subprocess.run([exe, seed], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "OK 14 cases" in r.stdout and "bit-exact" in r.stdout, r.stdout
