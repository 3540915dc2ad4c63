"""CPU checks of the drop-in boundary: the C-ABI library builds, loads and exports every entry point include/filo_b200.h declares,
the product refuses to run without a CUDA device (no CPU fallback), and nothing under filodb_b200/ touches the oracle."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_functions():
    src = open(os.path.join(ROOT, "include", "filo_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"^\s*(?:int32_t|int64_t|void|const char\*)\s+(filo_[a-z0-9_]+)\s*\(", src, flags=re.M)))


def test_header_declares_the_documented_entry_points():
    names = _declared_functions()
    for must in ("filo_ctx_create", "filo_load_series", "filo_query", "filo_query_device", "filo_scan_series", "filo_query_hist",
                 "filo_present_partials", "filo_host_register", "filo_table_free", "filo_last_error"):
        assert must in names


def test_library_exports_every_declared_symbol():
    from filodb_b200 import build, capi
    path = build.build(force=False)                      # nvcc cross-compiles sm_90a without a GPU
    lib = C.CDLL(path)
    missing = [n for n in _declared_functions() if not hasattr(lib, n)]
    assert not missing, "declared in include/filo_b200.h but not exported: %s" % missing
    assert sorted(capi.EXPORTS) == sorted(_declared_functions())      # the ctypes mirror covers the whole header


def test_num_windows_matches_periodic_samples_mapper():
    """Host-only entry point: windows of [start, end] by step (PeriodicSamplesMapper / RvRange semantics)."""
    from filodb_b200 import capi
    assert capi.num_windows(0, 15000, 7200000) == 481
    assert capi.num_windows(100, 47000, 100 + 47000 * 3 + 46999) == 4
    assert capi.num_windows(5, 1, 5) == 1
    assert capi.num_windows(5, 0, 5) == 1                 # instant query: step 0 is adjusted to 1


def test_no_cpu_fallback_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA device present")
    from filodb_b200 import capi
    with pytest.raises(capi.FiloError):
        capi.Context(0)


def test_product_never_imports_the_oracle():
    bad = []
    for dirpath, _, files in os.walk(os.path.join(ROOT, "filodb_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                if re.search(r"^\s*(from|import)\s+oracle\b|#include\s+\"[./]*oracle/|libfilo_oracle", txt, flags=re.M):
                    bad.append(os.path.join(dirpath, f))
    assert not bad, "product files reference the oracle: %s" % bad


def test_cpp_operator_mirror_compiles_and_keeps_reference_requirements(tmp_path):
    """include/filo_b200.hpp (PeriodicSamplesMapper / AggregateMapReduce / FusedGpuExec over the C-ABI) builds as C++17, its
    constructors reject what the Scala `require`s reject (PeriodicSamplesMapper.scala:45-49), and without a CUDA device the
    executor throws instead of falling back."""
    import subprocess
    from filodb_b200 import build
    lib = build.build(force=False)
    exe = str(tmp_path / "mirror")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "operator_mirror_requires.cpp"), "-o", exe,
                    "-L", os.path.dirname(lib), "-lfilo_b200", "-Wl,-rpath," + os.path.dirname(lib)], check=True)
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    assert "start 100 should be <= end 50" in out
    assert "step should be > 0" in out
    assert "Need positive window lengths" in out
    import torch
    if not torch.cuda.is_available():
        assert "QueryError -2" in out and "ok=4" in out


def _build_and_run_cpp(tmp_path, name, flags=(), args=()):
    import subprocess
    exe = str(tmp_path / name)
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-Wno-unknown-pragmas", *flags,
                    os.path.join(ROOT, "tests", "cpp", name + ".cpp"), "-o", exe], check=True)
    return subprocess.run([exe, *args], check=True, capture_output=True, text=True).stdout


def test_hist_group_decoder_matches_nibblepack_on_cpu(tmp_path):
    """filodb_b200/csrc/hist_decode.h (the histogram kernel's word-wise NibblePack group decoder) compiled for the host:
    every group alignment, bit width and trailing-zero count against the oracle's pack8 / unpack8."""
    assert "OK 200000 groups" in _build_and_run_cpp(tmp_path, "hist_decode_check")


def test_hist_scan2_phases_match_oracle_on_cpu(tmp_path):
    """filodb_b200/csrc/hist_phases.h — the phase functions hist_scan2_kernel is made of — run thread id by thread id on the CPU:
    hist rate / increase over SectDelta chunks with resets inside chunks and at chunk starts, regular and jittered timestamps,
    8 / 20 / 33 buckets, several series folded into one partial row; bit-exact against the oracle (tests/cpp/hist_emul.cpp)."""
    for seed in ((), ("3",)):                      # default histories, and another draw of chunk layouts / resets
        out = _build_and_run_cpp(tmp_path, "hist_emul", args=seed)
        assert out.startswith("OK 81 cases") and "bit-exact" in out


def test_scan_kernels_run_on_the_simt_emulator(tmp_path):
    """The scan kernels themselves (filodb_b200/csrc/scan_kernels.cu: scan_tile_kernel with its producer warp, TMA + mbarriers, named
    barriers and warp shuffles; the v4 kernels scan_wp_sum_kernel and scan_wp_ctr_kernel; scan_series_kernel_v2 / scan_agg_kernel_v2,
    which also take the series and items the other kernels decline) compiled for the host on
    the cusim fiber emulator (tests/cpp/cusim.h) and checked bit-exact against the oracle, scan counters included: every range
    function, raw / XOR / DDV-long vectors, const and irregular timestamps, 1-5 chunks, NaN markers, counter resets, several tiles per
    CTA, the fused aggregate mode; under the in-order schedule and a pseudo-random one.  The emulator aborts on deadlocks and on warp collectives reached from different call
    sites, and performs bulk copies as late as the program allows."""
    import subprocess, sys
    src = str(tmp_path / "scan_kernels_cusim.cu")          # function-scope __shared__ (merge_partials_kernel) -> static
    subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cpp", "make_cusim_src.py"), os.path.join(ROOT, "filodb_b200", "csrc", "scan_kernels.cu"), src], check=True)
    exe = str(tmp_path / "tile_emul")
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", "-I", "/usr/local/cuda/include",
                    "-I", os.path.join(ROOT, "filodb_b200", "csrc"), '-DSCAN_SRC="%s"' % src,
                    os.path.join(ROOT, "tests", "cpp", "tile_emul.cpp"), "-o", exe], check=True)
    for seed in ("0", "20260922"):
        out = subprocess.run([exe, seed], check=True, capture_output=True, text=True).stdout
        assert "OK 104 cases" in out and "bit-exact" in out, out
    # random shapes: chunk counts and sizes, windows, offsets, functions, NaN / reset rates, per-series and fused modes
    out = subprocess.run([exe, "7", "fuzz", "60"], check=True, capture_output=True, text=True).stdout
    assert "OK 164 cases" in out and "bit-exact" in out, out


def test_histogram_kernels_run_on_the_simt_emulator(tmp_path):
    """hist_scan2_kernel (with its cp.async record prefetch) + hist_merge2_kernel and hist_scan_kernel + hist_merge_kernel compiled for
    the host on the cusim emulator: fused sum + histogram_quantile on both kernels, per-series rate / increase, sum_over_time and the
    delta-temporality rate, SectDelta and simple vectors, resets inside chunks and at chunk starts, irregular scrapes; bit-exact
    against the oracle (the checker folds series and items in the kernels' order)."""
    import subprocess, sys
    v1 = str(tmp_path / "hist_kernels_cusim.cu")
    subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cpp", "make_cusim_src.py"), os.path.join(ROOT, "filodb_b200", "csrc", "hist_kernels.cu"), v1], check=True)
    exe = str(tmp_path / "hist_kernel_emul")
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", "-I", "/usr/local/cuda/include",
                    "-I", os.path.join(ROOT, "filodb_b200", "csrc"), '-DHIST_V1_SRC="%s"' % v1,
                    os.path.join(ROOT, "tests", "cpp", "hist_kernel_emul.cpp"), "-o", exe], check=True)
    for seed in ("0", "5"):
        out = subprocess.run([exe, seed], check=True, capture_output=True, text=True).stdout
        assert "OK 11 cases" in out and "bit-exact" in out, out


def test_jni_shim_exports_the_reference_naming():
    """filodb_b200/libfilo_b200_jni.so (csrc/jni_shim.cpp) exports one Java_filodb_gpu_FiloB200NativeMethods_00024_<method> per @native
    method of INTEGRATION.md §2 -- the naming of the reference's own JNI crate for Scala objects (simd_vectors.rs:164,186) -- and
    nothing else; it needs the C-ABI library only."""
    import subprocess
    from filodb_b200 import build as b
    b.build()
    so = b.JNI_OUT if os.path.exists(b.JNI_OUT) else b.build_jni()
    syms = subprocess.run(["nm", "-D", "--defined-only", so], check=True, capture_output=True, text=True).stdout.split("\n")
    names = sorted(l.split()[-1] for l in syms if " T " in l)
    want = sorted("Java_filodb_gpu_FiloB200NativeMethods_00024_" + m for m in
                  ("ctxCreate", "ctxDestroy", "ctxSetFnArgs", "ctxCheck", "hostRegister", "hostUnregister", "loadSeries", "tableFree", "numWindows",
                   "query", "queryAvgSumCount", "queryHist", "scanSeries"))
    assert names == want, names
    needed = subprocess.run(["readelf", "-d", so], check=True, capture_output=True, text=True).stdout
    assert "libfilo_b200.so" in needed
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    for m in ("ctxCreate", "loadSeries", "query", "scanSeries", "queryHist", "tableFree"):
        assert "def %s(" % m in doc, m
