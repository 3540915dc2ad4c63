"""Per-phase cycle profile of the tile kernel's consumer warps (profiling build, -DFILO_TILE_PROF).
    FILO_NVCC_EXTRA="-DFILO_HIST_PROF -DFILO_TILE_PROF" FILO_BUILD_OUT=scratch/libfilo_b200_prof.so python -m filodb_b200.build --force
    FILO_KERNEL=v3 python scratch/tile_prof.py [workload] [series]       # on the GPU box; workload: a SUM-class one, c2 (default) or c1"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import filodb_b200.capi as capi
capi.LIB_PATH = os.path.join(HERE, "libfilo_b200_prof.so")
import bench

workload = sys.argv[1] if len(sys.argv) > 1 else "c2"
series = sys.argv[2] if len(sys.argv) > 2 else "3000000"
L = capi.lib()
L.filo_debug_tile_prof.argtypes = [C.c_void_p, C.c_int]
out = np.zeros(16, np.uint64)
sys.argv = ["bench.py", "--workload", workload, "--series", series, "--steps", "4", "--warmup", "2", "--no-e2e", "--no-cpu"]
L.filo_debug_tile_prof(out.ctypes.data, 1)
bench.main()
L.filo_debug_tile_prof(out.ctypes.data, 0)
names = ["wait: tile descriptors / bytes ready", "decode: field extraction + in-warp prefix", "wait: cross-warp exchange barrier", "decode: prefixes applied, rows stored",
         "wait: barrier B", "windows: blocked items", "windows: literal per-window folds", "wait: windows-end barrier", "-",
         "results (fold / bulk store), loop overhead"]
tot = float(out[:10].sum())
print("tile kernel, consumer warps (lane 0 of each): %d warps reported, all launches of the run" % int(out[15]))
for i, n in enumerate(names):
    if n != "-": print("  %-48s %6.1f %%" % (n, 100.0 * float(out[i]) / tot))
