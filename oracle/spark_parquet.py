"""oracle/spark_parquet.py — Parquet read oracle: pyarrow (an independent Apache Parquet reader).

TEST INFRASTRUCTURE ONLY.  The reference decodes Parquet with libcudf through Table.readParquet
(GpuParquetScan.scala:3322-3503), absent from /root/reference; the format is the Apache Parquet
spec, whose reference implementation (parquet-cpp via pyarrow 24) serves as the oracle.  PINNED by
the parquet-testing corpus the reference vendors (tests/golden/parquet_testing.json; the reference's
own integration test over that corpus is parquet_testing_test.py).
Type mapping follows GpuColumnVector.java:417-453: date -> int32 days, timestamp -> int64 micros
(GpuParquetScan delivers micros), decimal -> unscaled integer in DECIMAL32/64/128 by precision.
"""
import decimal
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

from . import spark_cpu as O


def arrow_to_ocol(col):
    typ = col.type
    n = len(col)
    valid = np.array([v is not None for v in col.to_pylist()], dtype=bool) if col.null_count else np.ones(n, bool)
    if pa.types.is_decimal(typ):
        dt = O.decimal_dtype_for(typ.precision)
        # exact: the default decimal context keeps 28 digits and would round DECIMAL(29..38) values
        exact = decimal.Context(prec=80)
        vals = np.array([0 if v is None else int(decimal.Decimal(v).scaleb(typ.scale, exact)) for v in col.to_pylist()], dtype=object)
        return O.OCol(vals, valid, (dt, typ.precision, typ.scale))
    if pa.types.is_string(typ) or pa.types.is_binary(typ) or pa.types.is_large_string(typ):
        vals = np.array([b"" if v is None else (v if isinstance(v, bytes) else v.encode()) for v in col.to_pylist()], dtype=object)
        return O.OCol(vals, valid, (O.STRING, 0, 0))
    m = {pa.int8(): O.INT8, pa.int16(): O.INT16, pa.int32(): O.INT32, pa.int64(): O.INT64, pa.float32(): O.FLOAT32, pa.float64(): O.FLOAT64,
         pa.bool_(): O.BOOL8}
    if pa.types.is_date32(typ):
        dt, col = O.DATE32, col.cast(pa.int32())
    elif pa.types.is_timestamp(typ):
        dt, col = O.TIMESTAMP_US, col.cast(pa.timestamp("us")).cast(pa.int64())
    elif pa.types.is_unsigned_integer(typ):   # cudf UINT* columns keep the stored bits; this library exposes the signed view of the same width
        dt = {1: O.INT8, 2: O.INT16, 4: O.INT32, 8: O.INT64}[typ.bit_width // 8]
        arr = col.combine_chunks() if isinstance(col, pa.ChunkedArray) else col
        raw = np.array([0 if v is None else int(v) for v in arr.to_pylist()], dtype=np.uint64).astype({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[typ.bit_width // 8])
        return O.OCol(raw.view(O._NP[dt]), valid, (dt, 0, 0))
    else:
        dt = m[typ]
    arr = col.combine_chunks() if isinstance(col, pa.ChunkedArray) else col
    vals = np.array([0 if v is None else v for v in arr.to_pylist()]).astype(O._NP[dt]) if arr.null_count else arr.to_numpy(zero_copy_only=False).astype(O._NP[dt])
    return O.OCol(vals, valid, (dt, 0, 0))


def read_parquet(buf, columns):
    tbl = pq.read_table(io.BytesIO(bytes(buf)), columns=list(columns))
    return [arrow_to_ocol(tbl.column(c)) for c in columns]
