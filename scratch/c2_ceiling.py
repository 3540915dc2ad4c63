"""Bandwidth ceiling of C2: a plain device copy with C2's byte mix, as a yardstick for scan_wp_sum_kernel.
    python scratch/c2_ceiling.py [rows] [out.json]          # on a GPU; rows = series (default 5,000,000, as bench.py's C2)
Every row reads 3,762 B (one C2 record: ChunkEntries + 4 XOR vectors of 120 rows, packed back to back) and writes 3,848 B (481 f64
results), so 5 M rows read 18.8 GB and write 19.2 GB, as C2 does.  One warp per row, 16-byte loads, lane-consecutive 8-byte
streaming stores (the kernel's result stores).  Prints the card's name, power limit and SM clocks beside the time and the rate
against the 3.35 TB/s of the H100 SXM data sheet.  The kernel is compiled with nvcc into a temporary directory."""
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile

READ_B, WRITE_B = 3762, 3848
SRC = r"""
#include <cstdint>
#include <cuda_runtime.h>
__global__ void __launch_bounds__(640) c2_copy(const uint4* __restrict__ src, double* __restrict__ dst, long long rows) {
  const int lane = threadIdx.x & 31;
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long s = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < rows; s += nw) {
    // row s reads the 16-byte words that start inside its bytes [s * 3762, (s + 1) * 3762): the words of all rows tile the buffer
    const long long w0 = (s * 3762 + 15) / 16, w1 = ((s + 1) * 3762 + 15) / 16;
    unsigned long long acc = 0;
    for (long long w = w0 + lane; w < w1; w += 32) { const uint4 v = __ldcs(src + w); acc ^= ((unsigned long long)v.x | ((unsigned long long)v.y << 32)) ^ v.z ^ ((unsigned long long)v.w << 17); }
    double* o = dst + s * 481;
    for (int i = lane; i < 481; i += 32) __stcs(o + i, (double)(acc + (unsigned long long)i));
  }
}
extern "C" int c2_run(long long rows, int warmup, int reps, float* ms_out, char* name, int name_len) {
  cudaDeviceProp p; if (cudaGetDeviceProperties(&p, 0) != cudaSuccess) return -1;
  for (int i = 0; i < name_len - 1 && p.name[i]; ++i) { name[i] = p.name[i]; name[i + 1] = 0; }
  const size_t rb = (size_t)rows * 3762 + 64, wb = (size_t)rows * 3848;
  uint4* src = nullptr; double* dst = nullptr;
  if (cudaMalloc(&src, rb) != cudaSuccess) return -2;
  if (cudaMalloc(&dst, wb) != cudaSuccess) { cudaFree(src); return -3; }
  cudaMemset(src, 0x5a, rb);
  const int grid = p.multiProcessorCount;                     // one persistent CTA of 20 warps per SM, as the C2 kernel runs
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  for (int i = 0; i < warmup; ++i) c2_copy<<<grid, 640>>>(src, dst, rows);
  for (int i = 0; i < reps; ++i) {
    cudaEventRecord(a); c2_copy<<<grid, 640>>>(src, dst, rows); cudaEventRecord(b); cudaEventSynchronize(b);
    cudaEventElapsedTime(ms_out + i, a, b);
  }
  const cudaError_t e = cudaGetLastError();
  cudaEventDestroy(a); cudaEventDestroy(b); cudaFree(src); cudaFree(dst);
  return e == cudaSuccess ? 0 : -4;
}
"""


def smi():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {}


def main():
    rows = int(sys.argv[1]) if len(sys.argv) > 1 else 5_000_000
    tmp = tempfile.mkdtemp(prefix="c2_ceiling_")
    cu, so = os.path.join(tmp, "c2_copy.cu"), os.path.join(tmp, "c2_copy.so")
    with open(cu, "w") as f:
        f.write(SRC)
    subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-shared", "-Xcompiler", "-fPIC", cu, "-o", so], check=True)
    lib = C.CDLL(so)
    reps = 10
    ms = (C.c_float * reps)()
    name = C.create_string_buffer(128)
    before = smi()
    rc = lib.c2_run(C.c_longlong(rows), 3, reps, ms, name, 128)
    after = smi()
    if rc != 0:
        raise SystemExit("c2_ceiling: CUDA error %d (no GPU, or not enough memory for %d rows)" % (rc, rows))
    t = sorted(ms)
    rd, wr = rows * READ_B, rows * WRITE_B
    med = statistics.median(t)
    res = {"gpu": name.value.decode(), "smi_before": before, "smi_after": after, "rows": rows, "read_bytes": rd, "write_bytes": wr,
           "ms_min": t[0], "ms_median": med, "ms_max": t[-1], "tb_per_s_median": (rd + wr) / (med * 1e-3) / 1e12}
    res["share_of_3_35_tb_s"] = res["tb_per_s_median"] / 3.35
    print("%s, power limit %s, max SM clock %s (SM clock %s after the runs)" % (res["gpu"], after.get("power.limit", "?"),
          after.get("clocks.max.sm", "?"), after.get("clocks.sm", "?")))
    print("C2 byte mix (%d rows: read %.1f GB, write %.1f GB): %.2f ms median (%.2f-%.2f over %d runs), %.2f TB/s = %.0f %% of 3.35 TB/s"
          % (rows, rd / 1e9, wr / 1e9, med, t[0], t[-1], reps, res["tb_per_s_median"], 100 * res["share_of_3_35_tb_s"]))
    if len(sys.argv) > 2:
        with open(sys.argv[2], "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
