"""stddev / stdvar across series against the matching sum, timed with CUDA events on one card in one call.

    python scratch/agg_moments_bench.py [series] [iters] [out.json]      # on an H100; the full record also goes to out.json if given

Two tables of `series` (default 5 M) series x 2 h at 15 s (480 rows, chunks 400 + 80), 100 groups, T = 481:
  * the C5 counter table: stddev(rate[5m]) by (cluster) against sum(rate[5m]) by (cluster)  (v4 counter kernel);
  * a C2-shaped XOR gauge table: stdvar(sum_over_time[5m]) by (g) against sum(sum_over_time[5m]) by (g)  (tile kernel).
Each pair is warmed up, then timed alternately three times (`iters` device-side queries per timing, results left on the device), with
the card's name, power limit and SM clock read in the same call."""
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import torch
import filodb_b200.capi as capi

S = int(sys.argv[1]) if len(sys.argv) > 1 else 5_000_000
ITERS = int(sys.argv[2]) if len(sys.argv) > 2 else 10
OUT = sys.argv[3] if len(sys.argv) > 3 else None
T0, STEP, ROWS, G = 1_700_000_000_000, 15000, 480, 100
Q = (T0, STEP, T0 + ROWS * 15000, 300000)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
    except Exception as e:                      # noqa: BLE001
        out = "nvidia-smi unavailable: %r" % e
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": out}


def timed(ctx, tab, fn, aggr, iters):
    T = capi.num_windows(*Q[:3])
    n = G * T
    vals = torch.empty(2 * n, dtype=torch.float64, device="cuda"); cnts = torch.empty(n, dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()                      # the queries and both events on one stream of its own (handle != 0)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(iters):
        ctx.query_device(tab, fn, *Q, vals.data_ptr(), cnts.data_ptr(), aggr=aggr, stream=s.cuda_stream, want_stats=False)
    e1.record(s)
    torch.cuda.synchronize()
    ctx.check()
    return e0.elapsed_time(e1) / iters


def main():
    ctx = capi.Context(0)
    res = {"card_before": card(), "series": S, "groups": G, "windows": capi.num_windows(*Q[:3]), "iters": ITERS, "pairs": []}
    cases = [("C5 counters: stddev(rate[5m]) by (cluster) vs sum", dict(value_kind=1, value_enc=1, reset_period=1000, schema_flags=1),
              capi.FN_RATE, capi.AGG_STDDEV),
             ("C2-shaped gauges: stdvar(sum_over_time[5m]) by (g) vs sum", dict(value_kind=0, value_enc=1, nan_per_million=1000),
              capi.FN_SUM_OVER_TIME, capi.AGG_STDVAR)]
    for label, kw, fn, mom in cases:
        tab = ctx.synth_table(S, ROWS, 400, T0, STEP, n_groups=G, seed=42, **kw)
        for a in (capi.AGG_SUM, mom):
            timed(ctx, tab, fn, a, 3)                            # warm-up: module loads, pool allocations
        runs = []
        for _ in range(3):
            runs.append({"sum_ms": timed(ctx, tab, fn, capi.AGG_SUM, ITERS), "moments_ms": timed(ctx, tab, fn, mom, ITERS)})
        r = {"query": label, "runs": runs,
             "ratio_median": sorted(x["moments_ms"] / x["sum_ms"] for x in runs)[1]}
        res["pairs"].append(r)
        print(json.dumps(r), flush=True)
        tab.free()
    res["card_after"] = card()
    ctx.close()
    if OUT:
        os.makedirs(os.path.dirname(os.path.abspath(OUT)), exist_ok=True)
        with open(OUT, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps({k: res[k] for k in ("card_before", "card_after")}))


if __name__ == "__main__":
    main()
