"""The fused aggregate kernels over work items of many series on the SIMT emulator (tests/cpp/agg_items_emul.cpp): items of 1, 7, 9, 64
and 256 series laid out by build_groups_new's rule, every warp / CTA folding at least six of them, declines planted at item and warp
boundaries.  The fallback list must name exactly the items holding a planted series; partial rows, merged rows and the scan counters
must match the oracle, under the round-robin schedule and a seeded random one."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fused_items_on_the_simt_emulator(tmp_path):
    src = str(tmp_path / "scan_cusim.cu")
    subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cpp", "make_cusim_src.py"), os.path.join(ROOT, "filodb_b200", "csrc", "scan_kernels.cu"), src], check=True)
    exe = str(tmp_path / "agg_items_emul")
    subprocess.run(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes", "-I", "/usr/local/cuda/include",
                    "-I", os.path.join(ROOT, "filodb_b200", "csrc"), '-DSCAN_SRC="%s"' % src,
                    os.path.join(ROOT, "tests", "cpp", "agg_items_emul.cpp"), "-o", exe], check=True)
    runs = [subprocess.Popen([exe, seed], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for seed in ("0", "7")]     # the two schedules at once
    for seed, p in zip(("0", "7"), runs):
        out = p.communicate()[0]
        assert p.returncode == 0 and "OK 36 cases" in out, "schedule seed %s:\n%s" % (seed, out[-3000:])
        assert "ctr IRR moments seg 256" in out and "tile seg 9 ungrouped" in out, out[-3000:]
