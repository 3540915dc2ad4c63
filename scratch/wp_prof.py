"""Per-phase cycle profile of the v4 SUM-class kernels, scan_wp_sum_kernel or scan_wp_batch_kernel (profiling build, -DFILO_WP_PROF).
    FILO_NVCC_EXTRA=-DFILO_WP_PROF FILO_BUILD_OUT=scratch/libfilo_b200_wp_prof.so python -m filodb_b200.build --force
    python scratch/wp_prof.py [workload] [series]       # on a GPU; workload: a SUM-class one, c2 (default) or c1
(FILO_LIB_PATH: another profiling build, e.g. of an earlier commit.)
Prints, per phase, the cycles a warp spends on one series (lane 0's SM clock, summed over warps and divided by the series the
warps took up) and the share of the warp's time.  Warps of one SM run side by side: divide by the warps per SM for SM cycles.
scan_wp_batch_kernel: "wait" is the wait for the entry and the record, "parse" the read of the entry, and slot 8 the wait for the
warp's previous result row to have left shared memory (its bulk store); the producer warp's cycles
per batch follow (stalled on the empty barrier, offsets + copy issue + copy wait, header parse + entries)."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import filodb_b200.capi as capi
capi.LIB_PATH = os.environ.get("FILO_LIB_PATH") or os.path.join(HERE, "libfilo_b200_wp_prof.so")
import bench

workload = sys.argv[1] if len(sys.argv) > 1 else "c2"
series = sys.argv[2] if len(sys.argv) > 2 else "5000000"
L = capi.lib()
L.filo_debug_wp_prof.argtypes = [C.c_void_p, C.c_int]
out = np.zeros(32, np.uint64)
sys.argv = ["bench.py", "--workload", workload, "--series", series, "--steps", "4", "--warmup", "2", "--no-e2e", "--no-cpu", "--no-extra", "--no-c5"]
L.filo_debug_wp_prof(out.ctypes.data, 1)
bench.main()
L.filo_debug_wp_prof(out.ctypes.data, 0)
names = ["wait: record (mbarrier)", "parse", "memo check (+ window plan on a miss)", "per-series descriptors, scan counters", "decode",
         "zero rows", "window blocks", "finish and store (batch kernel: fix-up and store)", "wait: previous row's bulk store", "loop head, declined series"]
# slot 8: scan_wp_batch_kernel's wait for its previous result row's bulk store (before the decode); zero for scan_wp_sum_kernel
ns = float(out[10])
tot = float(out[:10].sum())
print("SUM kernel: %d consumer warps, %d series taken up, %d memo misses, %d declined by the plan, %d declined by the values"
      % (int(out[15]), int(ns), int(out[11]), int(out[12]), int(out[13])))
print("  %-40s %10s %7s" % ("phase", "cyc/series", "share"))
for i, n in enumerate(names):
    if i == 8 and out[i] == 0:
        continue
    print("  %-40s %10.1f %6.1f %%" % (n, float(out[i]) / ns, 100.0 * float(out[i]) / tot))
print("  %-40s %10.1f" % ("total", tot / ns))
if out[20]:
    nb = float(out[19])
    ptot = float(out[16:19].sum())
    print("producer: %d warps, %d batches" % (int(out[20]), int(nb)))
    for i, n in enumerate(["stalled on the empty barrier", "offsets, copy issue, copy wait", "header parse, entries"]):
        print("  %-40s %10.1f %6.1f %%" % (n, float(out[16 + i]) / nb, 100.0 * float(out[16 + i]) / ptot))
    print("  %-40s %10.1f" % ("total", ptot / nb))
