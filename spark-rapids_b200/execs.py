"""Python face of the C++ operator layer (csrc/exec.cu): same node names as the reference's GpuExec
classes, same pull-iterator-of-batches contract (GpuExec.internalDoExecuteColumnar)."""
import ctypes

from ._lib import lib, check
from . import _init as m


class GpuExec:
    def __init__(self, handle, keep=()):
        self.h = ctypes.c_int64(handle)
        self._keep = list(keep)  # programs / children / host buffers that must outlive the node

    def __del__(self):
        if getattr(self, "h", None) is not None and self.h.value and lib is not None:   # lib is None during interpreter shutdown
            lib.b2_exec_close(self.h)
            self.h = ctypes.c_int64(0)

    def next(self):
        out = ctypes.c_int64()
        check(lib.b2_exec_next(self.h, ctypes.byref(out)))
        return m.Table(out.value) if out.value else None

    def __iter__(self):
        while True:
            t = self.next()
            if t is None:
                return
            yield t

    def collect(self):
        """all output batches concatenated (like executeCollect on the columnar side)"""
        batches = list(self)
        if not batches:
            return None
        return batches[0] if len(batches) == 1 else m.concat(batches)

    @property
    def metrics(self):
        out = (ctypes.c_int64 * 3)()
        check(lib.b2_exec_metrics(self.h, out))
        return {"numOutputRows": out[0], "numOutputBatches": out[1], "opTime": out[2]}

    def device_time(self):
        """(self ms, total ms) of this node on the device while profiling was enabled"""
        out = (ctypes.c_double * 2)()
        check(lib.b2_exec_device_time(self.h, out))
        return out[0], out[1]


class HashJoinExec(GpuExec):
    @property
    def sub_partition_stats(self):
        """GpuSubPartitionHashJoin: first-level buckets (0 = not sub-partitioned), buckets repartitioned, bytes split per side"""
        out = (ctypes.c_int64 * 4)()
        check(lib.b2_exec_join_sub_partition_stats(self.h, out))
        return {"buckets": out[0], "repartitioned": out[1], "build_bytes": out[2], "stream_bytes": out[3]}

    @property
    def emit_stats(self):
        """stream batches whose output rows the filter-probe kernel wrote, batches joined through gather maps, and
        overflow reruns (emitted batches whose matches passed the estimated output size, joined again through the maps)"""
        out = (ctypes.c_int64 * 3)()
        check(lib.b2_exec_join_emit_stats(self.h, out))
        return {"emitted": out[0], "maps": out[1], "overflows": out[2]}


def _new(fn, *args, keep=(), cls=GpuExec):
    out = ctypes.c_int64()
    check(fn(*args, ctypes.byref(out)))
    return cls(out.value, keep)


def GpuBatchSource(tables=()):
    e = _new(lib.b2_exec_source)
    for t in tables:
        check(lib.b2_exec_source_push(e.h, t.h))
    return e


def GpuParquetScanExec(buffers, columns):
    import numpy as np
    names = (ctypes.c_char_p * len(columns))(*[c.encode() for c in columns])
    e = _new(lib.b2_exec_parquet_scan, names, len(columns))
    for b in buffers:
        arr = np.frombuffer(b, dtype=np.uint8) if not isinstance(b, np.ndarray) else b
        e._keep.append(arr)
        check(lib.b2_exec_parquet_scan_add(e.h, m._ptr(arr), arr.nbytes))
    return e


def GpuFilterExec(condition, child, output=None):
    """output: column indexes a pruning GpuProjectExec above the filter keeps (fused: only those are compacted)"""
    prog = condition if isinstance(condition, m.Program) else m.Program([condition])   # a Program: bound + compiled once per plan
    if output is not None:
        return _new(lib.b2_exec_filter_select, child.h, prog.h, m._i32s(output), len(output), keep=[prog, child])
    return _new(lib.b2_exec_filter, child.h, prog.h, keep=[prog, child])


def host_columns(arrays):
    """[(dtype, scale, numpy values | (chars, offsets), validity bits or None)] -> (ctypes array, keepalive)"""
    arr = (m.B2HostColumn * len(arrays))()
    keep = []
    for i, (dtype, scale, data, valid) in enumerate(arrays):
        arr[i].dtype, arr[i].scale = dtype, scale
        if dtype == m.STRING:
            chars, offsets = data
            arr[i].rows = len(offsets) - 1
            arr[i].data, arr[i].offsets = chars.ctypes.data, offsets.ctypes.data
            keep += [chars, offsets]
        else:
            arr[i].rows = len(data) if dtype != m.DECIMAL128 else len(data)
            arr[i].data = data.ctypes.data
            keep.append(data)
        if valid is not None:
            arr[i].validity_bits = valid.ctypes.data
            keep.append(valid)
    return arr, keep


def GpuHostBatchSource(batches):
    """HostColumnarToGpu: batches = list of host column lists (see host_columns); buffers should be pinned"""
    e = _new(lib.b2_exec_host_source)
    for b in batches:
        arr, keep = host_columns(b)
        e._keep += keep
        check(lib.b2_exec_host_source_push(e.h, arr, len(b)))
    return e


def GpuProjectExec(project_list, child):
    prog = m.Program(project_list)
    return _new(lib.b2_exec_project, child.h, prog.h, keep=[prog, child])


def GpuExpandExec(projections, child):
    """projections: list of expression lists (same output types); output = every batch projected by each, stacked"""
    progs = [p if isinstance(p, m.Program) else m.Program(p) for p in projections]
    arr = (ctypes.c_int64 * len(progs))(*[p.h.value for p in progs])
    return _new(lib.b2_exec_expand, child.h, arr, len(progs), keep=progs + [child])


class HashAggregateExec(GpuExec):
    @property
    def repartition_stats(self):
        """GpuMergeAggregateIterator: first-level buckets (0 = never bucketed), buckets split again, bytes split over all
        levels, deepest level reached"""
        out = (ctypes.c_int64 * 4)()
        check(lib.b2_exec_aggregate_repartition_stats(self.h, out))
        return {"buckets": out[0], "resplit": out[1], "bytes_split": out[2], "depth": out[3]}


def GpuHashAggregateExec(child, grouping, aggregates, pre_project=None, condition=None, mode="partial", target_bytes=None, num_buckets=16):
    """mode 'partial'/'complete': update aggregates over `pre_project` expressions (with `condition`
    fused in as the child filter); 'final': merge aggregation buffers whose keys lead the input.
    A 'partial' output (a 'final' input) is the keys, one column per aggregate, then one INT64 count of
    valid inputs per decimal SUM (Spark's isEmpty), so that a partial sum that overflowed stays NULL.
    target_bytes given: once the held partials pass target_bytes they are split into num_buckets spillable hash buckets
    and merged bucket by bucket, one output batch per group of buckets (the partials need not fit on the device)"""
    code = {"partial": 0, "final": 1, "complete": 2}[mode]
    if mode == "final":
        e = _new(lib.b2_exec_hash_aggregate, child.h, ctypes.c_int64(0), 0, code, m._i32s(grouping), len(grouping), m._agg_specs(aggregates),
                 len(aggregates), keep=[child], cls=HashAggregateExec)
    else:
        if isinstance(pre_project, m.Program):    # compiled once per plan (output 0 is the fused condition when `condition` is truthy)
            prog = pre_project
        else:
            prog = m.Program(([condition] if condition is not None else []) + list(pre_project))
        e = _new(lib.b2_exec_hash_aggregate, child.h, prog.h, int(condition is not None), code, m._i32s(grouping), len(grouping),
                 m._agg_specs(aggregates), len(aggregates), keep=[prog, child], cls=HashAggregateExec)
    if target_bytes is not None:
        check(lib.b2_exec_aggregate_set_repartitioning(e.h, int(target_bytes), int(num_buckets)))
    return e


def GpuShuffledHashJoinExec(stream_keys, build_keys, join_type, stream, build, nulls_equal=False, stream_out=None, build_out=None, condition=None,
                            target_bytes=None, num_sub_partitions=16):
    """join_type JOIN_RIGHT_OUTER keeps every build row (stream columns NULL where no stream row matched): Spark's RightOuter
    with BuildRight, or LeftOuter with BuildLeft with the children swapped;
    stream_out / build_out: columns a pruning GpuProjectExec above the join keeps (fused into the gathers);
    condition: non-equi join condition (Expr / Program) bound over [stream columns ++ build columns] (mixed join);
    target_bytes given: GpuSubPartitionHashJoin, a build side larger than target_bytes is split into num_sub_partitions
    spillable buckets with the stream side and joined bucket by bucket (the build side need not fit on the device)"""
    e = _hash_join(stream_keys, build_keys, join_type, stream, build, nulls_equal, stream_out, build_out)
    if condition is not None:
        prog = condition if isinstance(condition, m.Program) else m.Program([condition])
        check(lib.b2_exec_join_set_condition(e.h, prog.h))
        e._keep.append(prog)
    if target_bytes is not None:
        check(lib.b2_exec_join_set_sub_partitioning(e.h, int(target_bytes), int(num_sub_partitions)))
    return e


def _hash_join(stream_keys, build_keys, join_type, stream, build, nulls_equal, stream_out, build_out):
    if stream_out is not None or build_out is not None:
        so, bo = list(stream_out or []), list(build_out or [])
        return _new(lib.b2_exec_shuffled_hash_join_select, stream.h, build.h, m._i32s(stream_keys), m._i32s(build_keys), len(stream_keys), join_type,
                    int(nulls_equal), m._i32s(so), len(so), m._i32s(bo), len(bo), keep=[stream, build], cls=HashJoinExec)
    return _new(lib.b2_exec_shuffled_hash_join, stream.h, build.h, m._i32s(stream_keys), m._i32s(build_keys), len(stream_keys), join_type,
                int(nulls_equal), keep=[stream, build], cls=HashJoinExec)


def GpuSortExec(sort_order, child, global_sort=True, target_bytes=None):
    """target_bytes given: the out-of-core full sort (GpuOutOfCoreSortIterator) emitting stable sorted batches of at most
    target_bytes each (at least 16 KiB) whose input need not fit on the device; otherwise the partition is sorted as one
    batch (global_sort) or each batch on its own"""
    if target_bytes is not None:
        if not global_sort:
            raise ValueError("target_bytes needs global_sort=True")
        return _new(lib.b2_exec_sort_out_of_core, child.h, m._order_args(sort_order), len(sort_order), int(target_bytes), keep=[child])
    return _new(lib.b2_exec_sort, child.h, m._order_args(sort_order), len(sort_order), int(global_sort), -1, keep=[child])


def GpuTopN(limit, sort_order, child):
    return _new(lib.b2_exec_sort, child.h, m._order_args(sort_order), len(sort_order), 1, limit, keep=[child])


def GpuCoalesceBatches(child, target_rows):
    return _new(lib.b2_exec_coalesce, child.h, target_rows, keep=[child])


def GpuShuffleExchangeExec(child, key_cols, comm=None, world=1):
    return _new(lib.b2_exec_shuffle_exchange, child.h, m._i32s(key_cols), len(key_cols), comm.h if comm else ctypes.c_int64(0), world,
                keep=[child, comm])


def GpuBroadcastExchangeExec(child, comm=None, rank=0, world=1):
    """every rank gets the whole child relation (one batch); as the build child of a join: GpuBroadcastHashJoinExec"""
    return _new(lib.b2_exec_broadcast_exchange, child.h, comm.h if comm else ctypes.c_int64(0), rank, world, keep=[child, comm])


def GpuBroadcastHashJoinExec(stream_keys, build_keys, join_type, stream, build, comm=None, rank=0, world=1, **kw):
    """GpuBroadcastHashJoinExecBase.scala: the build side is broadcast, the stream side stays where it is (no shuffle).
    JOIN_RIGHT_OUTER is refused: every rank would emit the unmatched build rows (Spark never broadcasts the preserved side)"""
    if join_type == m.JOIN_RIGHT_OUTER:
        raise ValueError("a broadcast hash join cannot preserve its build side (JOIN_RIGHT_OUTER)")
    return GpuShuffledHashJoinExec(stream_keys, build_keys, join_type, stream, GpuBroadcastExchangeExec(build, comm, rank, world), **kw)
