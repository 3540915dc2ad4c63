"""Device time of the cross-GPU histogram sum (filo_query_hist_device partials + filo_merge_hist_partials), CUDA events:

    merge kernel alone       W = 8 partials, T = 481, nb = 20, G = 1 and G = 1000 (hist_merge_parts_kernel)
    sharded C4 on one card   C4's 1 M series cut into 8 tables of 125 k: eight SUM partial queries + the merge, against one
                             SUM query over the whole table (histogram_quantile(0.99, sum(rate(h[5m])))), alternated
    gather over NCCL         shard.gather_hist_partials of [1000, 481, 20] f64 partials across the visible GPUs (>= 2), else "not measured"

Tables as C4: filo_synth_hist_table, 20 custom buckets 2 * 3^i .. +Inf, 480 rows at 15 s (chunks 400 + 80), T = 481; the 8 tables hold
series ids [r * 125 k, (r + 1) * 125 k), i.e. the same series as the whole table.  Prints the card, its power limit and SM clock; writes
JSON when given a path.

    python scratch/hist_parts_bench.py [--reps 5] [out.json]
"""
import argparse
import json
import os
import socket
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

T0, ROWS, RPC, INTERVAL = 1_700_000_000_000, 480, 400, 15000
NB = 20


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:            # noqa: BLE001 -- reported, not fatal
        return "nvidia-smi unavailable: %s" % e


def _gather_worker(rank, world, port, reps, q):
    import torch
    import torch.distributed as dist
    from filodb_b200 import shard
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    part = torch.full((1000, 481, NB), float(rank), dtype=torch.float64, device="cuda")
    for _ in range(3):
        shard.gather_hist_partials(part, dist)
    torch.cuda.synchronize(); dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        out = shard.gather_hist_partials(part, dist)
    e1.record(); torch.cuda.synchronize()
    ok = all(bool((out[r] == float(r)).all()) for r in range(world))
    if rank == 0:
        q.put({"world": world, "ms": e0.elapsed_time(e1) / reps, "bytes_per_rank": part.numel() * 8, "ok": ok})
    dist.barrier(); dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--series", type=int, default=1_000_000)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import filodb_b200.capi as capi
    info = card(); print(info, flush=True)
    bdef, bfmt = capi.custom_bucket_def([2.0 * 3 ** i for i in range(NB - 1)] + [float("inf")])
    ctx = capi.Context(0)
    q = (T0, 15000, T0 + 7200000, 300000)
    T = capi.num_windows(q[0], q[1], q[2])
    res = {"card": info, "reps": a.reps}
    stream = torch.cuda.Stream()              # a stream of its own: the events and every call are on it (0 would mean the ctx stream)
    ev = lambda: torch.cuda.Event(enable_timing=True)          # noqa: E731

    # ---- merge kernel alone: 8 partials of monotonic rows, a few cells empty
    W = 8
    for G in (1, 1000):
        tab = ctx.synth_hist_table(2 * G, 24, bdef, bfmt, NB, rows_per_chunk=24, t0_ms=T0, interval_ms=INTERVAL, seed=1, n_groups=G)
        assert tab.info().n_groups == G
        g = torch.Generator(device="cuda"); g.manual_seed(G)
        parts = torch.rand((W, G, T, NB), dtype=torch.float64, device="cuda", generator=g).cumsum(dim=3)
        parts[:, :, ::7, :] = float("nan")
        mv = torch.empty((G, T, NB), dtype=torch.float64, device="cuda"); mq = torch.empty((G, T), dtype=torch.float64, device="cuda")
        run = lambda: ctx.merge_hist_partials(tab, W, T, parts.data_ptr(), mv.data_ptr(), mq.data_ptr(), quantile=0.99, stream=stream.cuda_stream)  # noqa: E731
        torch.cuda.synchronize()
        for _ in range(5): run()
        n = 200 if G == 1 else 50
        times = []
        for _ in range(a.reps):
            e0, e1 = ev(), ev(); e0.record(stream)
            for _ in range(n): run()
            e1.record(stream); torch.cuda.synchronize(); times.append(e0.elapsed_time(e1) / n)
        nbytes = (W * G * T * NB + G * T * (NB + 1)) * 8
        res["merge G=%d" % G] = {"ms": times, "bytes": nbytes, "GB/s": nbytes / (min(times) / 1e3) / 1e9}
        print("merge W=8 T=%d nb=%d G=%-5d %s ms  (%.0f GB/s at the best)" % (T, NB, G, " ".join("%.4f" % x for x in times), nbytes / (min(times) / 1e3) / 1e9), flush=True)
        tab.free()

    # ---- C4 cut into 8 tables: 8 partials + merge against one query over the whole table
    S = a.series; per = S // W
    whole = ctx.synth_hist_table(S, ROWS, bdef, bfmt, NB, rows_per_chunk=RPC, t0_ms=T0, interval_ms=INTERVAL, reset_period=97, seed=42)
    tabs = [ctx.synth_hist_table(per, ROWS, bdef, bfmt, NB, rows_per_chunk=RPC, t0_ms=T0, interval_ms=INTERVAL, reset_period=97, seed=42, series_id_base=r * per)
            for r in range(W)]
    parts = torch.empty((W, 1, T, NB), dtype=torch.float64, device="cuda")
    mq = torch.empty((1, T), dtype=torch.float64, device="cuda"); wq = torch.empty((1, T), dtype=torch.float64, device="cuda")

    def sharded():
        for r, t in enumerate(tabs):
            ctx.query_hist_device(t, capi.FN_RATE, *q, d_values=parts[r].data_ptr(), aggr=capi.AGG_SUM, stream=stream.cuda_stream, want_stats=False)
        ctx.merge_hist_partials(tabs[0], W, T, parts.data_ptr(), 0, mq.data_ptr(), quantile=0.99, stream=stream.cuda_stream)

    def one():
        ctx.query_hist_device(whole, capi.FN_RATE, *q, d_quantile=wq.data_ptr(), aggr=capi.AGG_SUM, quantile=0.99, stream=stream.cuda_stream, want_stats=False)

    out = {"sharded": [], "whole": []}
    torch.cuda.synchronize()
    for f in (sharded, one): f(); f()
    torch.cuda.synchronize(); ctx.check()
    for r in range(a.reps):
        for name, f in ((("sharded", sharded), ("whole", one)) if r % 2 == 0 else (("whole", one), ("sharded", sharded))):
            e0, e1 = ev(), ev(); e0.record(stream); f(); e1.record(stream); torch.cuda.synchronize()
            out[name].append(e0.elapsed_time(e1))
    ctx.check()
    a_q, b_q = mq.cpu().numpy(), wq.cpu().numpy()
    rel = float(np.nanmax(np.abs(a_q - b_q) / np.maximum(np.abs(b_q), 1e-300)))
    res["c4 sharded"] = dict(out, quantile_nan_pattern_equal=bool((np.isnan(a_q) == np.isnan(b_q)).all()), quantile_max_rel_diff=rel)
    print("C4 %d series: 8 x %d partial queries + merge %s ms; one query %s ms; quantile max rel diff %.2e" %
          (S, per, " ".join("%.2f" % x for x in out["sharded"]), " ".join("%.2f" % x for x in out["whole"]), rel), flush=True)
    for t in tabs: t.free()
    whole.free(); ctx.close()

    # ---- gather over NCCL
    ng = torch.cuda.device_count()
    if ng >= 2:
        import torch.multiprocessing as mp
        with socket.socket() as s:
            s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]
        mctx = mp.get_context("spawn"); qq = mctx.Queue()
        procs = [mctx.Process(target=_gather_worker, args=(r, min(ng, 8), port, 20, qq)) for r in range(min(ng, 8))]
        try:
            for p in procs: p.start()
            res["gather nccl"] = qq.get(timeout=300)
            for p in procs: p.join(timeout=60)
        finally:                              # no worker outlives the script, whatever happened above
            for p in procs:
                if p.is_alive(): p.terminate()
            for p in procs:
                if p.pid is not None: p.join()
    else:
        res["gather nccl"] = "not measured: %d GPU visible" % ng
    print("gather:", res["gather nccl"], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
