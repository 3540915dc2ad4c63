"""Device time of topk / bottomk across GPUs (filo_query_device candidates + topk_ids_to_global + filo_merge_topk_partials), CUDA events:

    merge kernel alone       W = 8 parts, T = 481, k = 5 and 32, G = 1, 100 and 1000 (topk_merge_parts_kernel)
    sharded C5 on one card   C5's table (counters, rate()[5m], 100 clusters) cut into 8 contiguous tables: eight topk(5) partial queries,
                             the id mapping and the merge, against one topk(5) query over the whole table, alternated; the merged values
                             and ids must equal the whole-table query bit for bit.  The merge alone on these candidates is timed too.

Tables as bench.py's C5: filo_synth_table, XOR counters with resets, 480 rows at 15 s (chunks 400 + 80), T = 481, 100 groups; table r holds
series ids [r * S / 8, (r + 1) * S / 8), i.e. the same series as the whole table.  Prints the card, its power limit and SM clock; writes
JSON when given a path.

    python scratch/topk_parts_bench.py [--reps 5] [--series 5000000] [out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

T0, ROWS, RPC, INTERVAL = 1_700_000_000_000, 480, 400, 15000
C5 = dict(value_kind=1, value_enc=1, reset_period=1000, schema_flags=1)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:            # noqa: BLE001 -- reported, not fatal
        return "nvidia-smi unavailable: %s" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--series", type=int, default=5_000_000)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import filodb_b200.capi as capi
    from filodb_b200 import shard
    info = card(); print(info, flush=True)
    ctx = capi.Context(0)
    q = (T0, 15000, T0 + ROWS * INTERVAL, 300000)
    T = capi.num_windows(q[0], q[1], q[2])
    res = {"card": info, "reps": a.reps, "windows": T}
    stream = torch.cuda.Stream()              # a stream of its own: the events and every call are on it (0 would mean the ctx stream)
    ev = lambda: torch.cuda.Event(enable_timing=True)          # noqa: E731

    def timed(f, n):
        torch.cuda.synchronize()
        for _ in range(3): f()
        times = []
        for _ in range(a.reps):
            e0, e1 = ev(), ev(); e0.record(stream)
            for _ in range(n): f()
            e1.record(stream); torch.cuda.synchronize(); times.append(e0.elapsed_time(e1) / n)
        return times

    # ---- merge kernel alone: 8 parts of sorted candidates with unique ids, every 7th window holding 2 of its k slots at most
    W = 8
    for k in (5, 32):
        for G in (1, 100, 1000):
            g = torch.Generator(device="cuda"); g.manual_seed(G * 100 + k)
            pv = torch.rand((W, G, T, k), dtype=torch.float64, device="cuda", generator=g).sort(dim=3).values
            pi = torch.arange(W * G * T * k, dtype=torch.int64, device="cuda").reshape(W, G, T, k)
            pi[:, :, ::7, 2:] = -1
            mv = torch.empty((G, T, k), dtype=torch.float64, device="cuda"); mi = torch.empty((G, T, k), dtype=torch.int64, device="cuda")
            run = lambda: ctx.merge_topk_partials(capi.AGG_TOPK, k, W, G, T, pv.data_ptr(), pi.data_ptr(), mv.data_ptr(), mi.data_ptr(), stream=stream.cuda_stream)  # noqa: E731
            times = timed(run, 200 if G < 1000 else 50)
            nbytes = (W + 1) * G * T * k * 16
            res["merge k=%d G=%d" % (k, G)] = {"ms": times, "bytes": nbytes, "GB/s": nbytes / (min(times) / 1e3) / 1e9}
            print("merge W=8 T=%d k=%-2d G=%-5d %s ms  (%.0f GB/s at the best)" % (T, k, G, " ".join("%.4f" % x for x in times), nbytes / (min(times) / 1e3) / 1e9), flush=True)
            del pv, pi, mv, mi

    # ---- C5 cut into 8 tables: 8 partial topk queries + id mapping + merge against one topk query over the whole table
    S, K, G = a.series, 5, 100
    per = S // W
    whole = ctx.synth_table(S, ROWS, RPC, T0, INTERVAL, n_groups=G, seed=42, **C5)
    tabs = [ctx.synth_table(per, ROWS, RPC, T0, INTERVAL, n_groups=G, seed=42, series_id_base=r * per, **C5) for r in range(W)]
    glob = [torch.arange(r * per, (r + 1) * per, dtype=torch.int64, device="cuda") for r in range(W)]
    pv = torch.empty((W, G, T, K), dtype=torch.float64, device="cuda"); pi = torch.empty((W, G, T, K), dtype=torch.int64, device="cuda")
    mv = torch.empty((G, T, K), dtype=torch.float64, device="cuda"); mi = torch.empty((G, T, K), dtype=torch.int64, device="cuda")
    wv = torch.empty((G, T, K), dtype=torch.float64, device="cuda"); wi = torch.empty((G, T, K), dtype=torch.int64, device="cuda")

    def partials():
        with torch.cuda.stream(stream):
            for r, t in enumerate(tabs):
                ctx.query_device(t, capi.FN_RATE, *q, pv[r].data_ptr(), pi[r].data_ptr(), aggr=capi.AGG_TOPK, k=K, stream=stream.cuda_stream, want_stats=False)
                pi[r] = shard.topk_ids_to_global(pi[r], glob[r])

    def merge():
        ctx.merge_topk_partials(capi.AGG_TOPK, K, W, G, T, pv.data_ptr(), pi.data_ptr(), mv.data_ptr(), mi.data_ptr(), stream=stream.cuda_stream)

    def sharded():
        partials(); merge()

    def one():
        ctx.query_device(whole, capi.FN_RATE, *q, wv.data_ptr(), wi.data_ptr(), aggr=capi.AGG_TOPK, k=K, stream=stream.cuda_stream, want_stats=False)

    out = {"sharded": [], "whole": []}
    torch.cuda.synchronize()
    for f in (sharded, one): f(); f()
    torch.cuda.synchronize(); ctx.check()
    for r in range(a.reps):
        for name, f in ((("sharded", sharded), ("whole", one)) if r % 2 == 0 else (("whole", one), ("sharded", sharded))):
            e0, e1 = ev(), ev(); e0.record(stream); f(); e1.record(stream); torch.cuda.synchronize()
            out[name].append(e0.elapsed_time(e1))
    ctx.check()
    same = bool(torch.equal(mv.view(torch.int64), wv.view(torch.int64)) and torch.equal(mi, wi))
    filled = int((wi >= 0).sum())
    one_partial = timed(lambda: ctx.query_device(tabs[0], capi.FN_RATE, *q, pv[0].data_ptr(), pi[0].data_ptr(), aggr=capi.AGG_TOPK, k=K,
                                                 stream=stream.cuda_stream, want_stats=False), 3)
    partials(); torch.cuda.synchronize()
    merge_only = timed(merge, 50)
    res["c5 sharded"] = dict(out, bit_equal=same, filled_slots=filled, slots=G * T * K, one_partial_query_ms=one_partial, merge_ms=merge_only)
    print("C5 %d series, topk(5) by 100 clusters: 8 x %d partial queries + id mapping + merge %s ms; one query %s ms; bit-equal %s (%d of %d slots filled)" %
          (S, per, " ".join("%.2f" % x for x in out["sharded"]), " ".join("%.2f" % x for x in out["whole"]), same, filled, G * T * K), flush=True)
    print("  one partial query %s ms; merge alone %s ms" % (" ".join("%.3f" % x for x in one_partial), " ".join("%.4f" % x for x in merge_only)), flush=True)
    for t in tabs: t.free()
    whole.free(); ctx.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    if not same:
        raise SystemExit("the sharded topk differs from the whole-table topk")


if __name__ == "__main__":
    main()
