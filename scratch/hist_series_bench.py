"""Device time of the per-series histogram query shapes on both histogram scan kernels (FILO_HIST_V2=1 / 0, alternated):

    histogram_quantile(0.99, rate(h[5m]))            per series, 1 M series (quantile only: [S][T])
    rate(h[5m]) bucket rows                          per series, --rows-series series ([S][T][nb] read back)
    histogram_quantile(0.99, sum(last(h)) by (g))    fused, 1 M series in --groups groups

Tables as C4: filo_synth_hist_table, 20 custom buckets 2 * 3^i .. +Inf, 480 rows at 15 s (chunks 400 + 80), T = 481.
Prints the card, its power limit and SM clock; writes JSON when given a path.

    python scratch/hist_series_bench.py [--reps 3] [--rows-series 100000] [out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

T0, ROWS, RPC, INTERVAL = 1_700_000_000_000, 480, 400, 15000


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:            # noqa: BLE001 -- reported, not fatal
        return "nvidia-smi unavailable: %s" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--rows-series", type=int, default=100_000)
    ap.add_argument("--groups", type=int, default=1000)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import filodb_b200.capi as capi
    info = card(); print(info, flush=True)
    nb = 20
    bdef, bfmt = capi.custom_bucket_def([2.0 * 3 ** i for i in range(nb - 1)] + [float("inf")])
    ctx = capi.Context(0)
    q = (T0, 15000, T0 + 7200000, 300000)
    res = {"card": info, "reps": a.reps}

    def timed(label, fn):
        out = {}
        for v in ("1", "0"):                      # warm-up of both kernels at this shape
            os.environ["FILO_HIST_V2"] = v; fn()
        for r in range(a.reps):
            for v in (("1", "0") if r % 2 == 0 else ("0", "1")):
                os.environ["FILO_HIST_V2"] = v; fn()
                out.setdefault("v2" if v == "1" else "v1", []).append(ctx.last_stats["kernel_ns"] / 1e6)
        os.environ.pop("FILO_HIST_V2", None)
        res[label] = out
        print("%-44s v2 %s ms   v1 %s ms" % (label, " ".join("%.2f" % x for x in out["v2"]), " ".join("%.2f" % x for x in out["v1"])), flush=True)

    tab = ctx.synth_hist_table(a.series, ROWS, bdef, bfmt, nb, rows_per_chunk=RPC, t0_ms=T0, interval_ms=INTERVAL, reset_period=97, seed=42, n_groups=a.groups)
    timed("quantile(0.99, rate[5m]) per series, %d" % a.series,
          lambda: ctx.query_hist(tab, capi.FN_RATE, *q, quantile=0.99, want_values=False))
    timed("quantile(0.99, sum(last) by g), %d / %d g" % (a.series, a.groups),
          lambda: ctx.query_hist(tab, capi.FN_LAST, *q, aggr=capi.AGG_SUM, quantile=0.99, want_values=False))
    tab.free()
    small = ctx.synth_hist_table(a.rows_series, ROWS, bdef, bfmt, nb, rows_per_chunk=RPC, t0_ms=T0, interval_ms=INTERVAL, reset_period=97, seed=42)
    timed("rate[5m] bucket rows per series, %d" % a.rows_series, lambda: ctx.query_hist(small, capi.FN_RATE, *q))
    timed("last bucket rows per series, %d" % a.rows_series, lambda: ctx.query_hist(small, capi.FN_LAST, *q))
    small.free()
    ctx.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
