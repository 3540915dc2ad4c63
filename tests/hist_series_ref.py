"""CPU restatement (test infrastructure) of the two histogram query shapes that return per-series rows:

    LastSampleChunkedFunction.addChunks / LastSampleChunkedFunctionH.updateValue
        query/src/main/scala/filodb/query/exec/rangefn/RangeFunction.scala:599-614, 630-640
    InstantVectorFunctionMapper(HistogramQuantile) per range vector: HistogramQuantileImpl -> Histogram.quantile
        query/src/main/scala/filodb/query/exec/rangefn/InstantFunction.scala:362-368, vectors/Histogram.scala:53-108

Built on the oracle's reader (oracle.hist.Reader: RowHistogramReader / SectDeltaHistogramReader.apply, the raw value) and its
Histogram.quantile (oracle.hist.Buckets.quantile); the chunk set of a window is WindowedChunkIterator's (ChunkSetInfo.scala:481-510)."""
import numpy as np

DEFAULT_LOOKBACK_MS = 5 * 60 * 1000 + 1            # window <= 0 for last: the default staleness lookback + 1 ms (as filo_query)


def num_windows(start, step, end):
    adj = step if step > 0 else step + 1
    return (end - start) // adj + 1


class SeriesChunks:
    """One series as the oracle store holds it: per chunk the ChunkSetInfo end time (the last appended timestamp), a reader over the
    timestamp vector (encoded as the store encodes it: near-regular timestamps become an approximate const DeltaDeltaVector) and a
    reader over the histogram vector, and the ChunkSetInfo's numRows."""

    def __init__(self, store, series, ts, chunk_rows):
        from oracle import hist as H
        from oracle import oracle as o
        self.chunks, off = [], 0
        for c, n in enumerate(chunk_rows):
            t = np.asarray(ts[off:off + n], np.int64)
            self.chunks.append((int(t[-1]), o.Vec(o.encode_timestamps(t)), H.Reader(store.vector_bytes(series, c)), n))
            off += n


def last_series(sc, nb, start, step, end, window, inclusive=True):
    """-> values [T, nb] (NaN buckets: Histogram.empty), empty [T]."""
    if window <= 0:
        window = DEFAULT_LOOKBACK_MS
    adj = step if step > 0 else step + 1
    T = num_windows(start, step, end)
    win = window if inclusive else window - 1
    out = np.full((T, nb), np.nan); empty = np.ones(T, bool)
    for k in range(T):
        w_end = start + k * adj; w_start = w_end - max(win, 0)
        timestamp, value = -1, None                                            # LastSampleChunkedFunction(timestamp = -1L)
        for c, (end_time, tv, rd, num_rows) in enumerate(sc.chunks):
            if end_time < w_start:                                             # chunk set of the window (time-ordered chunks)
                continue
            if c > 0 and not (sc.chunks[c - 1][0] < w_end):
                continue
            end_row = min(tv.ceiling_index(w_end), num_rows - 1)               # min(ceilingIndex(endTime), info.numRows - 1)
            if end_row >= 0:
                t = tv.long_apply(end_row)
                if t >= w_start and t > timestamp:                             # addChunks, :607-613
                    timestamp, value = t, rd(end_row)                          # updateValue: asHistReader(endRowNum), no correction
        if value is not None:
            out[k] = value.astype(np.float64); empty[k] = False
    return out, empty


def last_store(store, ts_list, chunk_list, nb, start, step, end, window, inclusive=True):
    """last over every series of an oracle.hist.HistStore -> values [S, T, nb], empty [S, T]."""
    res = [last_series(SeriesChunks(store, s, ts_list[s], chunk_list[s]), nb, start, step, end, window, inclusive) for s in range(len(ts_list))]
    return np.stack([r[0] for r in res]), np.stack([r[1] for r in res])


def quantiles(buckets, values, empty, q):
    """Histogram.quantile(q) of every (row, window) histogram [rows, T, nb]; NaN for Histogram.empty (no makeMonotonic)."""
    rows, T = empty.shape
    out = np.full((rows, T), np.nan)
    for i in range(rows):
        for k in range(T):
            if not empty[i, k]:
                out[i, k] = buckets.quantile(values[i, k], q)
    return out


def hist_sum(buckets_n, values, empty, group_ids, n_groups):
    """HistSumRowAggregator.reduceAggregate in series order: the first histogram is copied, every further one added + makeMonotonic."""
    from oracle import hist as H
    S, T, nb = values.shape
    acc = np.full((n_groups, T, nb), np.nan); aempty = np.ones((n_groups, T), bool)
    for s in range(S):
        g = int(group_ids[s])
        for k in range(T):
            if empty[s, k]:
                continue
            if aempty[g, k]:
                acc[g, k] = values[s, k]; aempty[g, k] = False
            else:
                acc[g, k] = H.make_monotonic(acc[g, k] + values[s, k])
    return acc, aempty


def scan_counters(store, ts_list, chunk_list, start, step, end, window, inclusive=True):
    """(samples, bytes) scanned: CountingChunkInfoIterator under WindowedChunkIterator (ChunkSetInfo.scala:336-380, 445-529; the oracle's
    WindowedChunkIterator in oracle/filo_query.hpp) over the chunks that intersect [start - window, end] (TimeSeriesPartition.scala:365-366).
    A chunk counts once it is pulled: numRows, and the total bytes of its timestamp and histogram vectors."""
    from oracle import oracle as o
    if window <= 0:
        window = DEFAULT_LOOKBACK_MS
    adj = step if step > 0 else step + 1
    win = window if inclusive else window - 1
    samples = nbytes = 0
    for s in range(len(ts_list)):
        infos, off = [], 0
        for c, n in enumerate(chunk_list[s]):
            t = np.asarray(ts_list[s][off:off + n], np.int64); off += n
            if int(t[0]) <= end and int(t[-1]) >= start - window:             # csi::intersects(info, start - window, end)
                hv = store.vector_bytes(s, c)                                   # BinaryVector.totalBytes = numBytes + 4 of both vectors
                infos.append((int(t[-1]), n, o.Vec(o.encode_timestamps(t)).total_bytes() + int(np.frombuffer(hv[:4].tobytes(), np.int32)[0]) + 4))
        w_end, w_start, pos, window_infos = None, None, 0, []
        while w_end is None or w_end + adj <= end:
            if w_end is None:
                w_end = start; w_start = start - max(win, 0)
            else:
                w_end += adj; w_start += adj
            while window_infos and window_infos[0][0] < w_start:
                window_infos.pop(0)
            last_end = window_infos[-1][0] if window_infos else -1
            while w_end > last_end and pos < len(infos):
                info = infos[pos]; pos += 1
                samples += info[1]; nbytes += info[2]
                if w_start <= info[0] and info[1] > 0:
                    window_infos.append(info); last_end = max(info[0], last_end)
    return samples, nbytes
