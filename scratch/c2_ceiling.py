"""Bandwidth ceiling of C2: copies with C2's byte mix in several traffic shapes, as yardsticks for scan_wp_sum_kernel.
    python scratch/c2_ceiling.py [rows] [out.json]          # on a GPU; rows = series (default 5,000,000, as bench.py's C2)
Every row reads 3,762 B (one C2 record: ChunkEntries + 4 XOR vectors of 120 rows, packed back to back) and writes 3,848 B (481 f64
results), so 5 M rows read 18.8 GB and write 19.2 GB, as C2 does.  The shapes, timed alternately (one launch of each per round,
10 rounds after 2 warm-up rounds):
  copy        one warp per row, 20 warps per SM, 16-byte loads, lane-consecutive 8-byte streaming stores (the kernel's result stores)
  read        the same loads, no stores (a reduction whose result is never stored): read-only bandwidth
  write       the same stores, no loads: write-only bandwidth
  pf_l2       `copy` plus one cp.async.bulk.prefetch.L2 of the row two series ahead of each warp
  pair_v2     one warp per pair of rows (2k, 2k + 1): the pair's bytes in one load loop, its two result rows (7,696 B, 16-byte aligned)
              with 16-byte streaming stores
  warp_tma2   one warp per row, each row fetched into the warp's shared memory by one cp.async.bulk, two rows in flight per warp
  bulk8_s3    CTA-cooperative, one CTA of 8 warps per SM: one cp.async.bulk per batch of 8 consecutive rows (30 KB), 3 batches in flight
              on mbarriers; the batch's 8 result rows (30.8 KB, 16-byte aligned) leave as one cp.async.bulk store from shared memory,
              2 stores in flight
  bulk4_s3x2  the same with batches of 4 rows and 2 CTAs of 4 warps per SM
  copy_v2     `copy` with the results stored by 16-byte streaming stores: an odd row starts at 8 mod 16, so it stores window 0 alone and
              windows (2j - 1, 2j) in pairs, an even row windows (2j, 2j + 1) in pairs and window 480 alone
  warp_tma1   `warp_tma2` with one row in flight per warp, the next copy issued once the row is read (the C2 kernel's record stream)
  warp_tma1_v2, warp_tma2_v2   the two above with `copy_v2`'s 16-byte result stores
  batch15     the C2 kernel's record stream: one CTA of 15 consumer warps and 1 producer warp per SM; the producer fetches batches of 15
              consecutive rows into two buffers with one cp.async.bulk each (full / empty mbarriers); warp w takes row w of every batch,
              releases the buffer once the row is read and stores its results with lane-consecutive 8-byte streaming stores
  batch15_rowbulk  `batch15` with every result row staged densely in the warp's own shared memory (at offset h = 1 when the row starts
              at 8 mod 16) and stored as one cp.async.bulk of its 16-byte-aligned span; the window outside the span (window 0 or 480)
              is stored directly.  The warp waits for its previous row's store to have read the staging area before it reads the next row
Prints the card's name, power limit and SM clocks beside each time and the rate against the 3.35 TB/s of the H100 SXM data sheet.
The kernels are compiled with nvcc into a temporary directory."""
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile

READ_B, WRITE_B = 3762, 3848
SHAPES = ["copy", "read", "write", "pf_l2", "pair_v2", "warp_tma2", "bulk8_s3", "bulk4_s3x2", "copy_v2", "warp_tma1", "warp_tma1_v2",
          "warp_tma2_v2", "batch15", "batch15_rowbulk"]
SRC = r"""
#include <cstdint>
#include <cuda_runtime.h>
#define RB 3762LL
#define NT 481

__device__ __forceinline__ unsigned long long mix(uint4 v) { return ((unsigned long long)v.x | ((unsigned long long)v.y << 32)) ^ v.z ^ ((unsigned long long)v.w << 17); }
// row s reads the 16-byte words that start inside its bytes [s * 3762, (s + 1) * 3762): the words of all rows tile the buffer
__device__ __forceinline__ long long w_lo(long long s) { return (s * RB + 15) / 16; }
__device__ __forceinline__ uint32_t sa(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bar_init(uint64_t* b) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(sa(b)) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void bulk_load(void* d, const void* g, uint32_t bytes, uint64_t* b) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sa(b)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(sa(d)), "l"(g), "r"(bytes), "r"(sa(b)) : "memory");
}
__device__ __forceinline__ void bar_init_n(uint64_t* b, uint32_t n) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sa(b)), "r"(n) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void bar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(sa(b)) : "memory"); }
__device__ __forceinline__ void bar_wait(uint64_t* b, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(sa(b)), "r"(parity) : "memory");
  } while (!ok);
}

__global__ void __launch_bounds__(640) c2_copy(const uint4* __restrict__ src, double* __restrict__ dst, long long rows, int pf) {
  const int lane = threadIdx.x & 31;
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long s = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < rows; s += nw) {
    if (pf && lane == 0 && s + 2 * nw < rows) {
      const long long a = w_lo(s + 2 * nw), b = w_lo(s + 2 * nw + 1);
      asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src + a), "r"((uint32_t)(b - a) * 16u) : "memory");
    }
    const long long w0 = w_lo(s), w1 = w_lo(s + 1);
    unsigned long long acc = 0;
    for (long long w = w0 + lane; w < w1; w += 32) acc ^= mix(__ldcs(src + w));
    double* o = dst + s * NT;
    for (int i = lane; i < NT; i += 32) __stcs(o + i, (double)(acc + (unsigned long long)i + 1));
  }
}

__global__ void __launch_bounds__(640) c2_read(const uint4* __restrict__ src, double* __restrict__ dst, long long rows) {
  const int lane = threadIdx.x & 31;
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  unsigned long long acc = 0;
  for (long long s = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < rows; s += nw)
    for (long long w = w_lo(s) + lane, w1 = w_lo(s + 1); w < w1; w += 32) acc ^= mix(__ldcs(src + w));
  if (acc == 0x0123456789abcdefull) dst[threadIdx.x] = (double)acc;         // never true for the data the survey writes
}

__global__ void __launch_bounds__(640) c2_write(const uint4* __restrict__ src, double* __restrict__ dst, long long rows) {
  const int lane = threadIdx.x & 31;
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long s = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < rows; s += nw) {
    double* o = dst + s * NT;
    for (int i = lane; i < NT; i += 32) __stcs(o + i, (double)(s + i + 1));
  }
}

__global__ void __launch_bounds__(640) c2_pair(const uint4* __restrict__ src, double* __restrict__ dst, long long rows) {
  const int lane = threadIdx.x & 31;
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5), np = rows / 2;
  for (long long p = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); p < np; p += nw) {
    const long long w0 = w_lo(2 * p), w1 = w_lo(2 * p + 2);
    unsigned long long acc = 0;
    for (long long w = w0 + lane; w < w1; w += 32) acc ^= mix(__ldcs(src + w));
    double2* o = reinterpret_cast<double2*>(dst + 2 * p * NT);                 // 2 * 481 * 8 = 7,696 = 16 * 481: 16-byte aligned
    for (int i = lane; i < NT; i += 32) __stcs(o + i, make_double2((double)(acc + 2 * i + 1), (double)(acc + 2 * i + 2)));
  }
}

// 481 results of row s from 16-byte-aligned stores: row s starts at 8 mod 16 when s is odd, so its window 0 is stored alone and
// windows (2j - 1, 2j) in pairs; an even row stores windows (2j, 2j + 1) in pairs and its window 480 alone
__device__ __forceinline__ void row_v2(double* dst, long long s, unsigned long long acc, int lane) {
  const int h = (int)(s & 1);
  double2* vb = reinterpret_cast<double2*>(dst + s * NT - h);                 // virtual window v = k + h; v = 2j, 2j + 1 at vb[j]
  for (int j = lane; j <= NT / 2; j += 32) {
    const double lo = (double)(acc + 2 * j + 1), hi = (double)(acc + 2 * j + 2);
    const bool vlo = 2 * j >= h, vhi = 2 * j + 1 < NT + h;
    if (vlo && vhi) __stcs(vb + j, make_double2(lo, hi));
    else if (vlo) __stcs(reinterpret_cast<double*>(vb + j), lo);
    else if (vhi) __stcs(reinterpret_cast<double*>(vb + j) + 1, hi);
  }
}

__global__ void __launch_bounds__(640) c2_copy_v2(const uint4* __restrict__ src, double* __restrict__ dst, long long rows) {
  const int lane = threadIdx.x & 31;
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long s = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < rows; s += nw) {
    unsigned long long acc = 0;
    for (long long w = w_lo(s) + lane, w1 = w_lo(s + 1); w < w1; w += 32) acc ^= mix(__ldcs(src + w));
    row_v2(dst, s, acc, lane);
  }
}

// one warp per row, each row fetched into the warp's shared memory by one cp.async.bulk, NB rows in flight per warp (NB x 3,808 B
// + the mbarriers); the next copy is issued as soon as the row is read, before its results are stored (as the C2 kernel does)
#define WT_BUF 3808
template <int NB, bool V2>
__global__ void __launch_bounds__(640) c2_warp_tma(const uint4* __restrict__ src, double* __restrict__ dst, long long rows) {
  extern __shared__ __align__(128) uint8_t sm[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t* base = sm + (size_t)warp * (NB * WT_BUF + 16);
  uint64_t* bar = reinterpret_cast<uint64_t*>(base + NB * WT_BUF);
  const long long nw = (long long)gridDim.x * (blockDim.x >> 5);
  long long s = (long long)blockIdx.x * (blockDim.x >> 5) + warp;
  if (lane == 0) for (int j = 0; j < NB; ++j) bar_init(bar + j);
  __syncwarp();
  for (int j = 0; j < NB; ++j)
    if (lane == 0 && s + j * nw < rows) { const long long a = w_lo(s + j * nw); bulk_load(base + j * WT_BUF, src + a, (uint32_t)(w_lo(s + j * nw + 1) - a) * 16u, bar + j); }
  for (int it = 0; s < rows; s += nw, ++it) {
    const int st = it % NB;
    bar_wait(bar + st, (uint32_t)(it / NB) & 1u);
    const long long w0 = w_lo(s), w1 = w_lo(s + 1);
    const uint4* r = reinterpret_cast<const uint4*>(base + st * WT_BUF);
    unsigned long long acc = 0;
    for (int w = lane; w < (int)(w1 - w0); w += 32) acc ^= mix(r[w]);
    __syncwarp();
    if (lane == 0 && s + NB * nw < rows) { const long long a = w_lo(s + NB * nw); bulk_load(base + st * WT_BUF, src + a, (uint32_t)(w_lo(s + NB * nw + 1) - a) * 16u, bar + st); }
    if (V2) row_v2(dst, s, acc, lane);
    else { double* o = dst + s * NT; for (int i = lane; i < NT; i += 32) __stcs(o + i, (double)(acc + (unsigned long long)i + 1)); }
  }
}

// CTA-cooperative: batches of B consecutive rows, ST loads and OST stores in flight; warp w of the CTA takes row w of a batch
template <int B, int ST, int OST>
__global__ void __launch_bounds__(B * 32) c2_bulk(const uint4* __restrict__ src, double* __restrict__ dst, long long rows) {
  constexpr int LB = ((B * 3762 + 32 + 15) / 16) * 16, OB = B * NT * 8;
  extern __shared__ __align__(128) uint8_t sm[];
  uint8_t* ld = sm;                                   // ST x LB
  double* ob = reinterpret_cast<double*>(sm + ST * LB); // OST x OB
  uint64_t* bar = reinterpret_cast<uint64_t*>(sm + ST * LB + OST * OB);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long nb = rows / B;
  auto issue = [&](long long b, int st) {
    const long long a = b * B * RB / 16, e = ((b + 1) * B * RB + 15) / 16;
    bulk_load(ld + st * LB, src + a, (uint32_t)(e - a) * 16u, bar + st);
  };
  if (threadIdx.x == 0) { for (int i = 0; i < ST; ++i) bar_init(bar + i); }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int j = 0; j < ST; ++j) if (blockIdx.x + (long long)j * gridDim.x < nb) issue(blockIdx.x + (long long)j * gridDim.x, j);
  int j = 0;
  for (long long b = blockIdx.x; b < nb; b += gridDim.x, ++j) {
    const int st = j % ST, os = j % OST;
    bar_wait(bar + st, (uint32_t)(j / ST) & 1u);
    if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(OST - 1) : "memory");   // store j - OST has left ob[os]
    __syncthreads();
    const long long s = b * B + warp, a = b * B * RB / 16;
    const uint4* r = reinterpret_cast<const uint4*>(ld + st * LB);
    unsigned long long acc = 0;
    for (long long w = w_lo(s) + lane, w1 = w_lo(s + 1); w < w1; w += 32) acc ^= mix(r[w - a]);
    double* o = ob + (size_t)os * (B * NT) + warp * NT;
    for (int i = lane; i < NT; i += 32) o[i] = (double)(acc + (unsigned long long)i + 1);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (threadIdx.x == 0) {
      asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst + b * B * NT), "r"(sa(ob + (size_t)os * (B * NT))), "r"((uint32_t)OB) : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      if (b + (long long)ST * gridDim.x < nb) issue(b + (long long)ST * gridDim.x, st);
    }
  }
  if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}
template <int B, int ST, int OST> constexpr int bulk_smem() { return ST * (((B * 3762 + 32 + 15) / 16) * 16) + OST * B * NT * 8 + 8 * ST; }

// the C2 kernel's record stream (scan_wp_batch_kernel): batches of 15 consecutive rows, two batch buffers, warp 15 fetches them (one
// cp.async.bulk per batch), consumer warp w takes row w of each batch and releases the buffer on `empty` once it has read the row.
// ROWBULK: the result row is staged at stg[k + h] (h = 1 when the row starts at 8 mod 16) and its 16-byte-aligned span of windows
// [h, h + ((481 - h) & ~1)) leaves as one cp.async.bulk store; the window outside it is stored directly
constexpr int BT_B = 15, BT_NBUF = 2, BT_LB = ((BT_B * 3762 + 32 + 15) / 16) * 16, BT_SB = (((NT + 1) * 8 + 15) / 16) * 16;
constexpr int batch_smem() { return BT_NBUF * BT_LB + BT_B * BT_SB + 2 * BT_NBUF * 8; }
template <bool ROWBULK>
__global__ void __launch_bounds__(512, 1) c2_batch(const uint4* __restrict__ src, double* __restrict__ dst, long long rows) {
  extern __shared__ __align__(128) uint8_t sm[];
  uint64_t* full = reinterpret_cast<uint64_t*>(sm + BT_NBUF * BT_LB + BT_B * BT_SB);
  uint64_t* empty = full + BT_NBUF;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  auto first = [&](long long i) -> long long { return ((long long)blockIdx.x + i * gridDim.x) * BT_B; };
  if (threadIdx.x == 0) for (int b = 0; b < BT_NBUF; ++b) { bar_init_n(full + b, 1); bar_init_n(empty + b, BT_B); }
  __syncthreads();
  if (warp == BT_B) {                                 // producer
    if (lane == 0)
      for (long long i = 0; first(i) < rows; ++i) {
        const int b = (int)(i % BT_NBUF);
        if (i >= BT_NBUF) bar_wait(empty + b, (uint32_t)(i / BT_NBUF - 1) & 1u);
        const long long s1 = first(i) + BT_B < rows ? first(i) + BT_B : rows;
        const long long a = first(i) * RB / 16, e = (s1 * RB + 15) / 16;
        bulk_load(sm + b * BT_LB, src + a, (uint32_t)(e - a) * 16u, full + b);
      }
    return;
  }
  double* stg = reinterpret_cast<double*>(sm + BT_NBUF * BT_LB + warp * BT_SB);
  for (long long i = 0;; ++i) {
    const long long s = first(i) + warp;
    if (s >= rows) break;
    const int b = (int)(i % BT_NBUF);
    bar_wait(full + b, (uint32_t)(i / BT_NBUF) & 1u);
    if (ROWBULK && lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // the previous row's store has read stg
    const long long a = first(i) * RB / 16;
    const uint4* r = reinterpret_cast<const uint4*>(sm + b * BT_LB);
    unsigned long long acc = 0;
    for (long long w = w_lo(s) + lane, w1 = w_lo(s + 1); w < w1; w += 32) acc ^= mix(r[w - a]);
    __syncwarp();
    if (lane == 0) bar_arrive(empty + b);
    double* o = dst + s * NT;
    if (!ROWBULK) { for (int k = lane; k < NT; k += 32) __stcs(o + k, (double)(acc + (unsigned long long)k + 1)); continue; }
    const int h = (int)((reinterpret_cast<uintptr_t>(o) >> 3) & 1), nb = (NT - h) & ~1;
    for (int k = lane; k < NT; k += 32) {
      const double v = (double)(acc + (unsigned long long)k + 1);
      if (k >= h && k < h + nb) stg[k + h] = v; else __stcs(o + k, v);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncwarp();
    if (lane == 0) {
      asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(o + h), "r"(sa(stg + 2 * h)), "r"((uint32_t)nb * 8u) : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
  }
  if (ROWBULK && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// shape k, one launch
static int launch(int k, int sms, const uint4* src, double* dst, long long rows) {
  switch (k) {
    case 0: c2_copy<<<sms, 640>>>(src, dst, rows, 0); break;
    case 1: c2_read<<<sms, 640>>>(src, dst, rows); break;
    case 2: c2_write<<<sms, 640>>>(src, dst, rows); break;
    case 3: c2_copy<<<sms, 640>>>(src, dst, rows, 1); break;
    case 4: c2_pair<<<sms, 640>>>(src, dst, rows); break;
    case 5: c2_warp_tma<2, false><<<sms, 640, 20 * (2 * WT_BUF + 16)>>>(src, dst, rows); break;
    case 6: c2_bulk<8, 3, 2><<<sms, 256, bulk_smem<8, 3, 2>()>>>(src, dst, rows); break;
    case 7: c2_bulk<4, 3, 2><<<2 * sms, 128, bulk_smem<4, 3, 2>()>>>(src, dst, rows); break;
    case 8: c2_copy_v2<<<sms, 640>>>(src, dst, rows); break;
    case 9: c2_warp_tma<1, false><<<sms, 640, 20 * (WT_BUF + 16)>>>(src, dst, rows); break;
    case 10: c2_warp_tma<1, true><<<sms, 640, 20 * (WT_BUF + 16)>>>(src, dst, rows); break;
    case 11: c2_warp_tma<2, true><<<sms, 640, 20 * (2 * WT_BUF + 16)>>>(src, dst, rows); break;
    case 12: c2_batch<false><<<sms, 512, batch_smem()>>>(src, dst, rows); break;
    case 13: c2_batch<true><<<sms, 512, batch_smem()>>>(src, dst, rows); break;
    default: return -1;
  }
  return 0;
}

// nshapes shapes, `reps` rounds of one launch each (after `warmup` rounds): ms_out[k * reps + i].  Before the rounds, every shape
// that stores results runs once on a zeroed output and `check_out[k]` counts the sampled result slots it left at zero.
extern "C" int c2_run(long long rows, int nshapes, int warmup, int reps, float* ms_out, long long* check_out, char* name, int name_len) {
  cudaDeviceProp p; if (cudaGetDeviceProperties(&p, 0) != cudaSuccess) return -1;
  for (int i = 0; i < name_len - 1 && p.name[i]; ++i) { name[i] = p.name[i]; name[i + 1] = 0; }
  if (rows % 8 != 0) return -5;                       // the bulk shapes store whole batches
  const size_t rb = (size_t)rows * 3762 + 64, wb = (size_t)rows * 3848;
  uint4* src = nullptr; double* dst = nullptr;
  if (cudaMalloc(&src, rb) != cudaSuccess) return -2;
  if (cudaMalloc(&dst, wb) != cudaSuccess) { cudaFree(src); return -3; }
  cudaMemset(src, 0x5a, rb);
  cudaFuncSetAttribute(c2_warp_tma<2, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 20 * (2 * WT_BUF + 16));
  cudaFuncSetAttribute(c2_warp_tma<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 20 * (2 * WT_BUF + 16));
  cudaFuncSetAttribute(c2_warp_tma<1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 20 * (WT_BUF + 16));
  cudaFuncSetAttribute(c2_warp_tma<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 20 * (WT_BUF + 16));
  cudaFuncSetAttribute(c2_bulk<8, 3, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, bulk_smem<8, 3, 2>());
  cudaFuncSetAttribute(c2_bulk<4, 3, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, bulk_smem<4, 3, 2>());
  cudaFuncSetAttribute(c2_batch<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, batch_smem());
  cudaFuncSetAttribute(c2_batch<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, batch_smem());
  const int sms = p.multiProcessorCount;
  for (int k = 0; k < nshapes; ++k) {
    check_out[k] = -1;
    if (k == 1) continue;
    cudaMemset(dst, 0, wb);
    if (launch(k, sms, src, dst, rows) != 0) return -6;
    if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) return -100 - k;
    long long zeros = 0;
    for (int i = 0; i < 4096; ++i) {                  // spread over the rows, both parities, first and last slots included
      const long long r = i == 4095 ? rows - 1 : (long long)((unsigned long long)i * 2654435761ull % (unsigned long long)rows);
      const int c = i % 3 == 0 ? 0 : i % 3 == 1 ? NT - 1 : (i * 37) % NT;
      double v = 0.0; cudaMemcpy(&v, dst + r * NT + c, 8, cudaMemcpyDeviceToHost);
      zeros += v == 0.0;
    }
    check_out[k] = zeros;
  }
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  for (int i = 0; i < warmup; ++i) for (int k = 0; k < nshapes; ++k) launch(k, sms, src, dst, rows);
  for (int i = 0; i < reps; ++i)
    for (int k = 0; k < nshapes; ++k) {
      cudaEventRecord(a); launch(k, sms, src, dst, rows); cudaEventRecord(b); cudaEventSynchronize(b);
      cudaEventElapsedTime(ms_out + k * reps + i, a, b);
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
    reps, ns = 10, len(SHAPES)
    ms = (C.c_float * (reps * ns))()
    chk = (C.c_longlong * ns)()
    name = C.create_string_buffer(128)
    before = smi()
    rc = lib.c2_run(C.c_longlong(rows), ns, 2, reps, ms, chk, name, 128)
    after = smi()
    if rc != 0:
        raise SystemExit("c2_ceiling: CUDA error %d (no GPU, rows not a multiple of 8, not enough memory for %d rows, or -100 - k: shape k "
                         "did not run)" % (rc, rows))
    rd, wr = rows * READ_B, rows * WRITE_B
    res = {"gpu": name.value.decode(), "smi_before": before, "smi_after": after, "rows": rows, "read_bytes": rd, "write_bytes": wr,
           "reps": reps, "shapes": {}}
    print("%s, power limit %s, max SM clock %s (SM clock %s before, %s after the runs)" % (res["gpu"], after.get("power.limit", "?"),
          after.get("clocks.max.sm", "?"), before.get("clocks.sm", "?"), after.get("clocks.sm", "?")))
    print("%d rows: read %.1f GB, write %.1f GB; %d alternated rounds" % (rows, rd / 1e9, wr / 1e9, reps))
    for k, sh in enumerate(SHAPES):
        t = sorted(ms[k * reps:(k + 1) * reps])
        med = statistics.median(t)
        by = (rd if sh != "write" else 0) + (wr if sh != "read" else 0)
        tbs = by / (med * 1e-3) / 1e12
        res["shapes"][sh] = {"ms": list(ms[k * reps:(k + 1) * reps]), "ms_min": t[0], "ms_median": med, "ms_max": t[-1], "bytes": by,
                             "tb_per_s_median": tbs, "share_of_3_35_tb_s": tbs / 3.35, "sampled_zero_results": chk[k]}
        print("  %-11s %7.2f ms median (%.2f-%.2f)  %5.2f TB/s = %3.0f %% of 3.35 TB/s%s" % (sh, med, t[0], t[-1], tbs, 100 * tbs / 3.35,
              "" if chk[k] <= 0 else "  CHECK FAILED: %d of 4096 sampled results not written" % chk[k]))
    if len(sys.argv) > 2:
        with open(sys.argv[2], "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
