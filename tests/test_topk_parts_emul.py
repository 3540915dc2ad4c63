"""topk / bottomk across GPUs on the SIMT emulator (tests/cpp/topk_parts_emul.cpp): the per-part candidates of the oracle (and of
topk_kernel, which must agree with them) with global ordinals, merged by topk_merge_parts_kernel, bit-exact in values and ids against the
oracle over the union of the series; a merge that breaks ties by part order instead of ordinal is shown to fail that check."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_topk_partials_merge_on_the_simt_emulator(tmp_path):
    """W = 1, 2, 3, 8, 64 (contiguous and modulo splits, parts without series), groups empty on some parts and on all; k = 1, 3, 32 with
    groups smaller than k; windows with only NaN inputs; integer-valued ties with +0.0 / -0.0, ±Inf and real ±DBL_MAX next to the padding;
    tables listing their series in a shuffled order (a non-increasing local -> global map, equal values out of ordinal order inside a
    part) and a NaN value with an id; in-order and pseudo-random fiber schedules."""
    src = str(tmp_path / "scan_kernels_cusim.cu")
    subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cpp", "make_cusim_src.py"), os.path.join(ROOT, "filodb_b200", "csrc", "scan_kernels.cu"), src], check=True)
    exe = str(tmp_path / "topk_parts_emul")
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", "-I", "/usr/local/cuda/include",
                    "-I", os.path.join(ROOT, "filodb_b200", "csrc"), '-DSCAN_SRC="%s"' % src,
                    os.path.join(ROOT, "tests", "cpp", "topk_parts_emul.cpp"), "-o", exe], check=True)
    for seed in ("0", "20261017"):
        r = subprocess.run([exe, seed], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "OK 16 cases" in r.stdout and "bit-exact" in r.stdout, r.stdout
