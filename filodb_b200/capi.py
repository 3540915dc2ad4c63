"""ctypes binding of include/filo_b200.h.  Fails loudly when the CUDA library is missing (no fallback)."""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("FILO_LIB_PATH") or os.path.join(_HERE, "libfilo_b200.so")      # FILO_LIB_PATH: A/B runs of a variant build (developer switch)

FN_LAST, FN_RATE, FN_INCREASE, FN_DELTA, FN_SUM_OVER_TIME, FN_AVG_OVER_TIME, FN_COUNT_OVER_TIME, \
    FN_MIN_OVER_TIME, FN_MAX_OVER_TIME, FN_TIMESTAMP, FN_STDDEV_OVER_TIME, FN_STDVAR_OVER_TIME, FN_CHANGES, FN_QUANTILE_OVER_TIME, \
    FN_ZSCORE, FN_HOLT_WINTERS, FN_PREDICT_LINEAR, FN_MAD_OVER_TIME, FN_PRESENT_OVER_TIME = range(19)
AGG_NONE, AGG_SUM, AGG_AVG, AGG_MIN, AGG_MAX, AGG_COUNT, AGG_TOPK, AGG_BOTTOMK, AGG_STDDEV, AGG_STDVAR, AGG_GROUP = range(11)
AGG_MOMENTS = (AGG_STDDEV, AGG_STDVAR)          # partial form: values [2, G, T] = (Σv, Σv²)
SCHEMA_CUMULATIVE = 1
SCHEMA_LONG_VALUES = 2
Q_PARTIAL = 1
OK, ERR_INVALID_ARG, ERR_CUDA, ERR_CORRUPT_VECTOR, ERR_UNSUPPORTED, ERR_QUERY_LIMIT, ERR_BAD_QUERY, ERR_OOM = 0, -1, -2, -3, -4, -5, -6, -7

EXPORTS = ["filo_ctx_create", "filo_ctx_destroy", "filo_ctx_set_fn_args", "filo_ctx_check", "filo_last_error", "filo_load_series", "filo_table_append", "filo_synth_table", "filo_encode_table", "filo_encode_hist_table", "filo_synth_hist_table",
           "filo_table_set_groups", "filo_table_get_info", "filo_table_read_record", "filo_table_read_arena", "filo_table_free",
           "filo_num_windows", "filo_query", "filo_query_device", "filo_scan_series", "filo_query_hist", "filo_query_hist_device", "filo_merge_hist_partials", "filo_merge_topk_partials", "filo_query_avg_sum_count", "filo_host_register", "filo_host_unregister", "filo_present_partials",
           "filo_result_max_containers", "filo_encode_result_device", "filo_encode_result"]


class Cfg(C.Structure):
    _fields_ = [("inclusive_range", C.c_int32), ("group_by_cardinality_limit", C.c_int32),
                ("min_step_ms", C.c_int64), ("max_data_per_shard_query", C.c_int64)]


class Stats(C.Structure):
    _fields_ = [("bytes_scanned", C.c_int64), ("samples_scanned", C.c_int64), ("kernel_ns", C.c_int64),
                ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64), ("kernel_launches", C.c_int64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class TableInfo(C.Structure):
    _fields_ = [("n_series", C.c_int64), ("n_chunks", C.c_int64), ("n_samples", C.c_int64), ("arena_bytes", C.c_int64),
                ("algorithmic_bytes", C.c_int64), ("max_rows_per_series", C.c_int32), ("max_chunks_per_series", C.c_int32),
                ("n_groups", C.c_int32), ("schema_flags", C.c_int32), ("hist_buckets", C.c_int32), ("reserved", C.c_int32)]


class SynthSpec(C.Structure):
    _fields_ = [("n_series", C.c_int64), ("rows_per_series", C.c_int32), ("rows_per_chunk", C.c_int32),
                ("t0_ms", C.c_int64), ("interval_ms", C.c_int32), ("ts_jitter_ms", C.c_int32),
                ("value_kind", C.c_int32), ("value_enc", C.c_int32), ("reset_period", C.c_int32),
                ("nan_per_million", C.c_int32), ("n_groups", C.c_int32), ("schema_flags", C.c_int32),
                ("seed", C.c_uint64), ("series_id_base", C.c_int64), ("sin_table", C.c_void_p)]


class FiloError(RuntimeError):
    """Mirrors how the JNI shim surfaces a non-zero status: RuntimeException(message)."""

    def __init__(self, code, msg):
        super().__init__("filo_b200 error %d: %s" % (code, msg))
        self.code = code


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError("libfilo_b200.so is not built (%s). Run `python -m filodb_b200.build`; there is no CPU fallback." % LIB_PATH)
        _lib = C.CDLL(LIB_PATH)
        _sig(_lib)
    return _lib


def _sig(L):
    i32, i64, vp = C.c_int32, C.c_int64, C.c_void_p
    L.filo_ctx_create.restype = i32; L.filo_ctx_create.argtypes = [i32, C.POINTER(Cfg), C.POINTER(vp)]
    L.filo_ctx_destroy.restype = None; L.filo_ctx_destroy.argtypes = [vp]
    L.filo_ctx_check.restype = i32; L.filo_ctx_check.argtypes = [vp]
    L.filo_encode_table.restype = i32; L.filo_encode_table.argtypes = [vp, vp, vp, i64, i32, i32, i32, i32, vp, i32, C.POINTER(vp)]
    L.filo_encode_hist_table.restype = i32; L.filo_encode_hist_table.argtypes = [vp, vp, vp, i64, i32, i32, i32, i32, vp, i32, i32, vp, i32, C.POINTER(vp)]
    L.filo_synth_hist_table.restype = i32; L.filo_synth_hist_table.argtypes = [vp, i64, i32, i32, i64, i32, i32, i32, vp, i32, i32, i32, C.c_uint64, i64, C.POINTER(vp)]
    L.filo_table_append.restype = i32; L.filo_table_append.argtypes = [vp, vp, vp, vp, i32, i32]
    L.filo_result_max_containers.restype = i64; L.filo_result_max_containers.argtypes = [i64, i32]
    L.filo_encode_result.restype = i32; L.filo_encode_result.argtypes = [vp, vp, i64, i64, i64, i64, i64, vp, i64, vp, vp, vp, C.POINTER(i64), C.POINTER(i64)]
    L.filo_encode_result_device.restype = i32
    L.filo_encode_result_device.argtypes = [vp, vp, i64, i64, i64, i64, i64, vp, i64, vp, vp, vp, C.POINTER(i64), C.POINTER(i64), vp]
    L.filo_ctx_set_fn_args.restype = i32; L.filo_ctx_set_fn_args.argtypes = [vp, C.c_double, C.c_double]
    L.filo_last_error.restype = i32; L.filo_last_error.argtypes = [vp, C.c_char_p, i32]
    L.filo_load_series.restype = i32
    L.filo_load_series.argtypes = [vp, i64, vp, vp, i32, i32, vp, i32, i32, C.POINTER(vp)]
    L.filo_synth_table.restype = i32; L.filo_synth_table.argtypes = [vp, C.POINTER(SynthSpec), C.POINTER(vp)]
    L.filo_table_set_groups.restype = i32; L.filo_table_set_groups.argtypes = [vp, vp, vp, i32]
    L.filo_table_get_info.restype = i32; L.filo_table_get_info.argtypes = [vp, C.POINTER(TableInfo)]
    L.filo_table_read_record.restype = i64; L.filo_table_read_record.argtypes = [vp, vp, i64, vp, i64]
    L.filo_table_read_arena.restype = i64; L.filo_table_read_arena.argtypes = [vp, vp, i64, i64, vp, i64, vp]
    L.filo_table_free.restype = None; L.filo_table_free.argtypes = [vp, vp]
    L.filo_num_windows.restype = i32; L.filo_num_windows.argtypes = [i64, i64, i64]
    L.filo_query.restype = i32
    L.filo_query.argtypes = [vp, vp, i32, i64, i64, i64, i64, i32, i32, i32, vp, vp, C.POINTER(Stats)]
    L.filo_query_device.restype = i32
    L.filo_query_device.argtypes = [vp, vp, i32, i64, i64, i64, i64, i32, i32, i32, vp, vp, vp, C.POINTER(Stats)]
    L.filo_scan_series.restype = i32
    L.filo_scan_series.argtypes = [vp, i64, vp, vp, i32, i32, i32, i32, i64, i64, i64, i64, vp, C.POINTER(Stats)]
    L.filo_query_hist.restype = i32
    L.filo_query_hist.argtypes = [vp, vp, i32, i64, i64, i64, i64, i32, C.c_double, vp, vp, C.POINTER(Stats)]
    L.filo_query_hist_device.restype = i32
    L.filo_query_hist_device.argtypes = [vp, vp, i32, i64, i64, i64, i64, i32, C.c_double, vp, vp, vp, C.POINTER(Stats)]
    L.filo_merge_hist_partials.restype = i32
    L.filo_merge_hist_partials.argtypes = [vp, vp, i32, i32, C.c_double, vp, vp, vp, vp]
    L.filo_merge_topk_partials.restype = i32
    L.filo_merge_topk_partials.argtypes = [vp, i32, i32, i32, i32, i32, vp, vp, vp, vp, vp]
    L.filo_query_avg_sum_count.restype = i32; L.filo_query_avg_sum_count.argtypes = [vp, vp, vp, i64, i64, i64, i64, vp, C.POINTER(Stats)]
    L.filo_host_register.restype = i32; L.filo_host_register.argtypes = [vp, vp, i64]
    L.filo_host_unregister.restype = i32; L.filo_host_unregister.argtypes = [vp, vp]
    L.filo_present_partials.restype = i32; L.filo_present_partials.argtypes = [vp, i32, i64, vp, vp, vp, vp]


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def num_windows(start, step, end):
    return lib().filo_num_windows(start, step, end)


def geometric_bucket_def(first, mult, n):
    """GeometricBuckets.serialize (Histogram.scala:609-617): u16 length, i16 numBuckets, f64 firstBucket, f64 multiplier; format code 0x03."""
    import struct
    return np.frombuffer(struct.pack("<Hhdd", 18, n, float(first), float(mult)), np.uint8).copy(), 3


def exp_bucket_def(scale, start_index, num_positive):
    """Base2ExpHistogramBuckets.serialize (Histogram.scala:729-752): u16 length 16, u16 numBuckets (= num_positive + 1, the zero bucket first),
    i16 scale, i32 startIndexPositiveBuckets, u16 numPositiveBuckets, i32 / u16 of the unused negative range; format code 0x09."""
    import struct
    return np.frombuffer(struct.pack("<HHhiHiH", 16, num_positive + 1, scale, start_index, num_positive, 0, 0), np.uint8).copy(), 9


def _pack8(vals8):
    """NibblePack.pack8 (NibblePack.scala:108-183) of eight u64: bitmask byte, then for a non-zero mask the nibble-count byte and the
    set values as little-endian bit-packed fields of numNibbles * 4 bits each."""
    mask = 0; orv = 0; mintz = 64
    for i, v in enumerate(vals8):
        if v:
            mask |= 1 << i; orv |= v
            mintz = min(mintz, (v & -v).bit_length() - 1)
    out = bytearray([mask])
    if not mask:
        return bytes(out)
    lz = 64 - orv.bit_length()
    trailing = mintz // 4; nnib = 16 - lz // 4 - trailing; nbits = nnib * 4
    out.append(((nnib - 1) << 4) | trailing)
    acc = 0; pos = 0
    for v in vals8:
        if v:
            acc |= ((v >> (trailing * 4)) & ((1 << nbits) - 1)) << pos; pos += nbits
    out += acc.to_bytes((pos + 7) // 8, "little")
    return bytes(out)


def custom_bucket_def(les):
    """CustomBuckets.serialize (Histogram.scala:878-884): u16 length, u16 numBuckets, NibblePack.packDoubles(les) = the first value's bits
    followed by groups of eight XOR-with-previous values; format code 0x05."""
    import struct
    bits = [struct.unpack("<Q", struct.pack("<d", float(x)))[0] for x in les]
    body = bytearray(struct.pack("<Q", bits[0]))
    xs = [bits[i + 1] ^ bits[i] for i in range(len(bits) - 1)]
    for g in range(0, len(xs), 8):
        grp = xs[g:g + 8]; grp += [0] * (8 - len(grp))
        body += _pack8(grp)
    d = struct.pack("<HH", 2 + len(body), len(les)) + bytes(body)
    return np.frombuffer(d, np.uint8).copy(), 5


def sin_table(rows):
    return np.sin(np.arange(1, rows + 1, dtype=np.float64))


class Table:
    def __init__(self, ctx, handle):
        self.ctx, self.h = ctx, handle

    def info(self):
        ti = TableInfo()
        self.ctx._check(lib().filo_table_get_info(self.h, C.byref(ti)))
        return ti

    def append(self, n_chunks, info_addrs, ts_col=0, val_col=1):
        """filo_table_append: new chunks of the table's series (n_chunks[i] may be 0); only they cross PCIe."""
        nch = np.ascontiguousarray(n_chunks, np.int32)
        addrs = np.ascontiguousarray(info_addrs, np.uint64)
        if addrs.size == 0: addrs = np.zeros(1, np.uint64)
        self.ctx._check(lib().filo_table_append(self.ctx.h, self.h, _p(nch), _p(addrs), ts_col, val_col))

    def set_groups(self, group_ids, n_groups):
        g = np.ascontiguousarray(group_ids, np.int32) if group_ids is not None else None
        self.ctx._check(lib().filo_table_set_groups(self.ctx.h, self.h, _p(g), n_groups))

    def read_record(self, series):
        buf = np.zeros(1 << 16, np.uint8)
        n = lib().filo_table_read_record(self.ctx.h, self.h, series, _p(buf), buf.size)
        if n < 0 and -n > buf.size:
            buf = np.zeros(-n, np.uint8)
            n = lib().filo_table_read_record(self.ctx.h, self.h, series, _p(buf), buf.size)
        if n < 0:
            self.ctx._check(int(n))
        return buf[:n].copy()

    def read_arena(self, first, n, out=None):
        """Host copy of the records of series [first, first+n): (bytes uint8[], rec_off int64[n+1] relative to bytes[0])."""
        off = np.zeros(n + 1, np.int64)
        need = lib().filo_table_read_arena(self.ctx.h, self.h, first, n, None, 0, _p(off))
        if need > 0 or need < -(1 << 62):
            self.ctx._check(int(need))
        nbytes = -need
        buf = out if out is not None else np.empty(max(nbytes, 1), np.uint8)
        assert buf.size >= nbytes
        got = lib().filo_table_read_arena(self.ctx.h, self.h, first, n, _p(buf), buf.size, _p(off))
        if got < 0:
            self.ctx._check(int(got))
        return buf[:got], off

    def free(self):
        if self.h:
            lib().filo_table_free(self.ctx.h, self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Context:
    def __init__(self, device=0, inclusive_range=True, group_by_cardinality_limit=0, min_step_ms=0, max_data_per_shard_query=0):
        cfg = Cfg(int(inclusive_range), group_by_cardinality_limit, min_step_ms, max_data_per_shard_query)
        h = C.c_void_p()
        rc = lib().filo_ctx_create(device, C.byref(cfg), C.byref(h))
        if rc != 0:
            buf = C.create_string_buffer(512)
            lib().filo_last_error(None, buf, 512)
            raise FiloError(rc, buf.value.decode())
        self.h = h
        self.last_stats = None

    def close(self):
        if self.h:
            lib().filo_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            buf = C.create_string_buffer(1024)
            lib().filo_last_error(self.h, buf, 1024)
            raise FiloError(rc, buf.value.decode())

    def check(self):
        """filo_ctx_check: waits for the stats-less device queries of this ctx and raises their first device-side error."""
        self._check(lib().filo_ctx_check(self.h))

    def encode_result(self, values, start, step, end, container_ts_ms=0):
        """filo_encode_result: rows of `values` [n_rows, T] -> (containers uint8[n, 4096], rows_serialized, start_record_no, first_container)."""
        v = np.ascontiguousarray(values, np.float64)
        n, T = v.shape
        cap = int(lib().filo_result_max_containers(n, T))
        out = np.zeros((max(cap, 1), 4096), np.uint8)
        rs = np.zeros(n, np.int32); sr = np.zeros(n, np.int32); fc = np.zeros(n, np.int64)
        nc = C.c_int64(); nr = C.c_int64()
        self._check(lib().filo_encode_result(self.h, _p(v), n, start, step, end, container_ts_ms, _p(out), out.size, _p(rs), _p(sr), _p(fc), C.byref(nc), C.byref(nr)))
        return out[:nc.value].copy(), rs, sr, fc

    def set_fn_args(self, arg0=0.0, arg1=0.0):
        """funcParams of the following queries (quantile; sf, tf; duration)."""
        self._check(lib().filo_ctx_set_fn_args(self.h, float(arg0), float(arg1)))

    def load_series(self, n_chunks, info_addrs, ts_col=0, val_col=1, group_ids=None, n_groups=0, schema_flags=0):
        nch = np.ascontiguousarray(n_chunks, np.int32)
        addrs = np.ascontiguousarray(info_addrs, np.uint64)
        g = np.ascontiguousarray(group_ids, np.int32) if group_ids is not None else None
        h = C.c_void_p()
        self._check(lib().filo_load_series(self.h, nch.size, _p(nch), _p(addrs), ts_col, val_col, _p(g), n_groups, schema_flags, C.byref(h)))
        return Table(self, h)

    def encode_table(self, timestamps, values, rows_per_chunk=400, value_enc=1, schema_flags=0, group_ids=None, n_groups=0):
        """filo_encode_table: raw samples [n_series, rows] -> chunks encoded on the device -> resident table."""
        ts = np.ascontiguousarray(timestamps, np.int64); v = np.ascontiguousarray(values, np.float64)
        assert ts.shape == v.shape and ts.ndim == 2
        g = np.ascontiguousarray(group_ids, np.int32) if group_ids is not None else None
        h = C.c_void_p()
        self._check(lib().filo_encode_table(self.h, _p(ts), _p(v), ts.shape[0], ts.shape[1], rows_per_chunk, value_enc, schema_flags, _p(g), n_groups, C.byref(h)))
        return Table(self, h)

    def encode_hist_table(self, timestamps, bucket_counts, bucket_def, format_code, rows_per_chunk=400, schema_flags=SCHEMA_CUMULATIVE, group_ids=None, n_groups=0):
        """filo_encode_hist_table: cumulative bucket counts [n_series, rows, nb] -> SectDelta HistogramVectors encoded on the device."""
        ts = np.ascontiguousarray(timestamps, np.int64); b = np.ascontiguousarray(bucket_counts, np.int64)
        assert b.ndim == 3 and ts.shape == b.shape[:2]
        d = np.ascontiguousarray(bucket_def, np.uint8)
        g = np.ascontiguousarray(group_ids, np.int32) if group_ids is not None else None
        h = C.c_void_p()
        self._check(lib().filo_encode_hist_table(self.h, _p(ts), _p(b), b.shape[0], b.shape[1], rows_per_chunk, b.shape[2], format_code, _p(d), d.size,
                                                 schema_flags, _p(g), n_groups, C.byref(h)))
        return Table(self, h)

    def synth_hist_table(self, n_series, rows_per_series, bucket_def, format_code, n_buckets, rows_per_chunk=400, t0_ms=1_700_000_000_000, interval_ms=15000,
                         reset_period=0, n_groups=0, seed=42, series_id_base=0):
        d = np.ascontiguousarray(bucket_def, np.uint8)
        h = C.c_void_p()
        self._check(lib().filo_synth_hist_table(self.h, n_series, rows_per_series, rows_per_chunk, t0_ms, interval_ms, n_buckets, format_code, _p(d), d.size,
                                                reset_period, n_groups, seed, series_id_base, C.byref(h)))
        return Table(self, h)

    def synth_table(self, n_series, rows_per_series, rows_per_chunk=400, t0_ms=1_700_000_000_000, interval_ms=15000,
                    ts_jitter_ms=0, value_kind=0, value_enc=0, reset_period=0, nan_per_million=0, n_groups=0,
                    schema_flags=0, seed=42, series_id_base=0):
        st = sin_table(rows_per_series)
        spec = SynthSpec(n_series, rows_per_series, rows_per_chunk, t0_ms, interval_ms, ts_jitter_ms, value_kind, value_enc,
                         reset_period, nan_per_million, n_groups, schema_flags, seed, series_id_base, st.ctypes.data)
        h = C.c_void_p()
        self._check(lib().filo_synth_table(self.h, C.byref(spec), C.byref(h)))
        return Table(self, h)

    def out_shapes(self, table, start, step, end, aggr, k, flags=0):
        ti = table.info()
        T = num_windows(start, step if step > 0 else 1, end)
        if aggr == AGG_NONE:
            return (ti.n_series, T), None
        if aggr in (AGG_TOPK, AGG_BOTTOMK):
            return (ti.n_groups, T, k), (ti.n_groups, T, k)
        if aggr in AGG_MOMENTS and flags & Q_PARTIAL:
            return (2, ti.n_groups, T), (ti.n_groups, T)
        return (ti.n_groups, T), (ti.n_groups, T)

    def query(self, table, fn, start, step, end, window, aggr=AGG_NONE, k=0, flags=0):
        """PeriodicSamplesMapper(+AggregateMapReduce) -> host numpy arrays (values[, aux])."""
        vs, as_ = self.out_shapes(table, start, step, end, aggr, k, flags)
        out = np.zeros(vs, np.float64)
        aux = np.zeros(as_, np.int64) if as_ is not None else None
        st = Stats()
        self._check(lib().filo_query(self.h, table.h, fn, start, step, end, window, aggr, k, flags, _p(out), _p(aux), C.byref(st)))
        self.last_stats = st.as_dict()
        if aggr in (AGG_AVG, AGG_TOPK, AGG_BOTTOMK, AGG_STDDEV, AGG_STDVAR, AGG_GROUP) or (flags & Q_PARTIAL and aggr != AGG_NONE):
            return out, aux
        return out

    def query_hist(self, table, fn, start, step, end, window, aggr=AGG_NONE, quantile=None, want_values=True):
        """filo_query_hist -> values [rows, T, buckets] (NaN buckets = empty histogram)[, quantile [rows, T]]; rows = series or groups."""
        ti = table.info(); T = num_windows(start, step, end)
        rows = ti.n_series if aggr == AGG_NONE else ti.n_groups
        vals = np.zeros((rows, T, ti.hist_buckets), np.float64) if want_values else None
        qs = np.zeros((rows, T), np.float64) if quantile is not None else None
        st = Stats()
        self._check(lib().filo_query_hist(self.h, table.h, fn, start, step, end, window, aggr, float("nan") if quantile is None else float(quantile),
                                          _p(vals), _p(qs), C.byref(st)))
        self.last_stats = st.as_dict()
        if quantile is None: return vals
        return (vals, qs) if want_values else qs

    def host_register(self, arr):
        """filo_host_register over a numpy array's buffer (chunk vectors inside it are then gathered by the GPU directly)."""
        self._check(lib().filo_host_register(self.h, arr.ctypes.data, arr.nbytes))

    def host_unregister(self, arr):
        self._check(lib().filo_host_unregister(self.h, arr.ctypes.data))

    def query_avg_sum_count(self, t_sum, t_count, start, step, end, window):
        """filo_query_avg_sum_count: avg_over_time over downsampled data (AvgWithSumAndCountOverTimeFuncD / FuncL) -> [n_series, T]."""
        T = num_windows(start, step, end)
        out = np.zeros((t_sum.info().n_series, T), np.float64)
        st = Stats()
        self._check(lib().filo_query_avg_sum_count(self.h, t_sum.h, t_count.h, start, step, end, window, _p(out), C.byref(st)))
        self.last_stats = st.as_dict()
        return out

    def scan_series(self, n_chunks, info_addrs, fn, start, step, end, window, ts_col=0, val_col=1, schema_flags=0, out=None):
        """filo_scan_series: ingest + query + read-back of host-resident chunks in one pipelined call -> [n_series, T].
        `out` may be a preallocated (ideally pinned) float64 array of n_series * T elements."""
        nch = np.ascontiguousarray(n_chunks, np.int32)
        addrs = np.ascontiguousarray(info_addrs, np.uint64)
        T = num_windows(start, step, end)
        if out is None:
            out = np.zeros((nch.size, T), np.float64)
        assert out.size == nch.size * T and out.dtype == np.float64 and out.flags["C_CONTIGUOUS"]
        st = Stats()
        self._check(lib().filo_scan_series(self.h, nch.size, _p(nch), _p(addrs), ts_col, val_col, schema_flags, fn, start, step, end, window,
                                           out.ctypes.data, C.byref(st)))
        self.last_stats = st.as_dict()
        return out

    def query_device(self, table, fn, start, step, end, window, d_out, d_aux=0, aggr=AGG_NONE, k=0, flags=0, stream=0, want_stats=True):
        st = Stats()
        self._check(lib().filo_query_device(self.h, table.h, fn, start, step, end, window, aggr, k, flags,
                                            C.c_void_p(d_out), C.c_void_p(d_aux) if d_aux else None,
                                            C.c_void_p(stream) if stream else None, C.byref(st) if want_stats else None))
        if want_stats:
            self.last_stats = st.as_dict()
        return self.last_stats

    def query_hist_device(self, table, fn, start, step, end, window, d_values=0, d_quantile=0, aggr=AGG_NONE, quantile=None, stream=0, want_stats=True):
        """filo_query_hist_device: results into device buffers (raw addresses; 0 = not wanted) on `stream`; without want_stats the call
        does not synchronise and its device-side errors surface at the next call on this ctx or at check()."""
        st = Stats()
        self._check(lib().filo_query_hist_device(self.h, table.h, fn, start, step, end, window, aggr, float("nan") if quantile is None else float(quantile),
                                                 C.c_void_p(d_values) if d_values else None, C.c_void_p(d_quantile) if d_quantile else None,
                                                 C.c_void_p(stream) if stream else None, C.byref(st) if want_stats else None))
        if want_stats:
            self.last_stats = st.as_dict()
        return self.last_stats

    def merge_hist_partials(self, table, n_parts, n_windows, d_parts, d_out_values=0, d_out_quantile=0, quantile=None, stream=0):
        """filo_merge_hist_partials: rank-order fold of n_parts histogram SUM partials [n_parts, G, T, nb] (device address) into
        values [G, T, nb] and / or histogram_quantile [G, T]; `table` supplies G, the buckets and their tops."""
        self._check(lib().filo_merge_hist_partials(self.h, table.h, n_parts, n_windows, float("nan") if quantile is None else float(quantile),
                                                   C.c_void_p(d_parts) if d_parts else None, C.c_void_p(d_out_values) if d_out_values else None,
                                                   C.c_void_p(d_out_quantile) if d_out_quantile else None, C.c_void_p(stream) if stream else None))

    def merge_topk_partials(self, aggr, k, n_parts, n_groups, n_windows, d_part_values, d_part_ids, d_out_values, d_out_ids, stream=0):
        """filo_merge_topk_partials: the k best candidates per (group, window) of n_parts topk / bottomk outputs [n_parts, G, T, k] (device
        addresses, ids global series ordinals) into values / ids [G, T, k], in the form filo_query_device writes them."""
        ptr = lambda a: C.c_void_p(a) if a else None
        self._check(lib().filo_merge_topk_partials(self.h, aggr, k, n_parts, n_groups, n_windows, ptr(d_part_values), ptr(d_part_ids),
                                                   ptr(d_out_values), ptr(d_out_ids), ptr(stream)))

    def present_partials(self, aggr, n, d_values, d_counts, d_out, stream=0):
        self._check(lib().filo_present_partials(self.h, aggr, n, C.c_void_p(d_values), C.c_void_p(d_counts), C.c_void_p(d_out),
                                                C.c_void_p(stream) if stream else None))
