"""Host-side mirror of the reference's operator interface for this path, over the C ABI (``libb2q.so``).

    Executor.executeWorkUnit(max_groups_buffer_entry_guess, is_agg, query_infos, ra_exe_unit, co, eo,
                             has_cardinality_estimation)  ->  ResultSet

has the parameter order and meaning of ``Executor::executeWorkUnit`` (QueryEngine/Execute.h:719-727); ``ResultSet``
exposes ``rowCount/colCount/getColType/getNextRow/entryCount/isEmpty/getStorageBuffer`` like
QueryEngine/ResultSet.h:183-330.  Errors that cross the reference's boundary as C++ exceptions are raised as the
Python exceptions below (same names).

This module only marshals arguments: all computation happens in the CUDA library.  If the library is missing the
import of this module's ``lib()`` fails loudly — there is no Python or CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence

import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb2q.so")
_lib = None


class QueryExecutionError(RuntimeError):
    """QueryExecutionError(ErrorCode) — QueryEngine/ExecutionKernel.cpp:133-160."""

    def __init__(self, code: int, msg: str):
        super().__init__(f"[{code}] {msg}")
        self.code = code


class CardinalityEstimationRequired(QueryExecutionError):
    """NativeCodegen.cpp:2972-2979: baseline hash without a cardinality estimate."""


class UnsupportedOnThisPath(QueryExecutionError):
    pass


class NoDeviceError(QueryExecutionError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -m heavydb_b200.build` (there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        L.b2q_abi_version.restype = C.c_int32
        L.b2q_error_string.restype = C.c_char_p
        L.b2q_error_string.argtypes = [C.c_int32]
        L.b2q_last_error_message.restype = C.c_char_p
        L.b2q_device_count.restype = C.c_int32
        L.b2q_rs_create_from_storage.restype = C.c_int32
        L.b2q_rs_create_from_storage.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]
        L.b2q_plan.restype = C.c_int32
        L.b2q_plan.argtypes = [C.POINTER(abi.ExecUnit), C.POINTER(abi.TableInfo), C.POINTER(abi.CompilationOptions),
                               C.POINTER(abi.ExecutionOptions), C.c_size_t, C.c_int32, C.POINTER(C.c_void_p)]
        L.b2q_query_plan.restype = C.POINTER(abi.Plan)
        L.b2q_query_plan.argtypes = [C.c_void_p]
        L.b2q_query_free.argtypes = [C.c_void_p]
        ewu = [C.POINTER(C.c_size_t), C.c_int32, C.POINTER(abi.TableInfo), C.POINTER(abi.ExecUnit),
               C.POINTER(abi.CompilationOptions), C.POINTER(abi.ExecutionOptions), C.c_int32]
        L.b2q_execute_work_unit.restype = C.c_int32
        L.b2q_execute_work_unit.argtypes = ewu + [C.POINTER(C.c_void_p)]
        L.b2q_execute_partial.restype = C.c_int32
        L.b2q_execute_partial.argtypes = ewu + [C.c_void_p, C.POINTER(C.c_void_p)]
        L.b2q_partial_num_arrays.restype = C.c_int32
        L.b2q_partial_num_arrays.argtypes = [C.c_void_p]
        L.b2q_partial_array.restype = C.c_int32
        L.b2q_partial_array.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_int64),
                                        C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
        L.b2q_partial_is_mergeable.restype = C.c_int32
        L.b2q_partial_is_mergeable.argtypes = [C.c_void_p]
        L.b2q_partial_plan.restype = C.POINTER(abi.Plan)
        L.b2q_partial_plan.argtypes = [C.c_void_p]
        L.b2q_partial_kernel_ms.restype = C.c_double
        L.b2q_partial_kernel_ms.argtypes = [C.c_void_p]
        L.b2q_partial_finalize.restype = C.c_int32
        L.b2q_partial_finalize.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
        L.b2q_partial_free.argtypes = [C.c_void_p]
        L.b2q_launch.restype = C.c_int32
        L.b2q_launch.argtypes = [C.c_void_p, C.POINTER(abi.Params), C.c_void_p]
        for n in ("b2q_rs_row_count", "b2q_rs_col_count", "b2q_rs_entry_count"):
            getattr(L, n).restype = C.c_size_t
            getattr(L, n).argtypes = [C.c_void_p]
        L.b2q_rs_is_empty.restype = C.c_int32
        L.b2q_rs_is_empty.argtypes = [C.c_void_p]
        L.b2q_rs_get_col_type.restype = abi.TypeInfo
        L.b2q_rs_get_col_type.argtypes = [C.c_void_p, C.c_size_t]
        L.b2q_rs_get_next_row.restype = C.c_int32
        L.b2q_rs_get_next_row.argtypes = [C.c_void_p, C.POINTER(abi.TargetValue), C.c_int32, C.c_int32]
        L.b2q_rs_get_row_at.restype = C.c_int32
        L.b2q_rs_get_row_at.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(abi.TargetValue), C.c_int32, C.c_int32]
        L.b2q_rs_move_to_begin.argtypes = [C.c_void_p]
        L.b2q_rs_is_row_at_empty.restype = C.c_int32
        L.b2q_rs_is_row_at_empty.argtypes = [C.c_void_p, C.c_size_t]
        L.b2q_rs_storage_buffer.restype = C.c_void_p
        L.b2q_rs_storage_buffer.argtypes = [C.c_void_p, C.POINTER(C.c_size_t)]
        L.b2q_rs_query_mem_desc.restype = C.POINTER(abi.Plan)
        L.b2q_rs_query_mem_desc.argtypes = [C.c_void_p]
        L.b2q_rs_kernel_ms.restype = C.c_double
        L.b2q_rs_kernel_ms.argtypes = [C.c_void_p]
        L.b2q_rs_free.argtypes = [C.c_void_p]
        L.b2q_rs_stat.restype = C.c_int64
        L.b2q_rs_stat.argtypes = [C.c_void_p, C.c_int32]
        L.b2q_last_launch_stat.restype = C.c_int64
        L.b2q_last_launch_stat.argtypes = [C.c_int32]
        L.b2q_rs_get_ndv_estimator.restype = C.c_size_t
        L.b2q_rs_get_ndv_estimator.argtypes = [C.c_void_p]
        L.b2q_rs_estimator_buffer.restype = C.c_void_p
        L.b2q_rs_estimator_buffer.argtypes = [C.c_void_p, C.POINTER(C.c_size_t)]
        L.b2q_rs_sort.restype = C.c_int32
        L.b2q_rs_sort.argtypes = [C.c_void_p, C.POINTER(abi.OrderEntry), C.c_int32, C.c_size_t]
        L.b2q_columnar_results_create.restype = C.c_int32
        L.b2q_columnar_results_create.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]
        L.b2q_columnar_results_size.restype = C.c_size_t
        L.b2q_columnar_results_size.argtypes = [C.c_void_p]
        L.b2q_columnar_results_num_columns.restype = C.c_size_t
        L.b2q_columnar_results_num_columns.argtypes = [C.c_void_p]
        L.b2q_columnar_results_column.restype = C.c_void_p
        L.b2q_columnar_results_column.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(abi.TypeInfo)]
        L.b2q_columnar_results_free.argtypes = [C.c_void_p]
        L.b2q_rs_drop_first_n.argtypes = [C.c_void_p, C.c_size_t]
        L.b2q_rs_keep_first_n.argtypes = [C.c_void_p, C.c_size_t]
        L.b2q_gen_column.restype = C.c_int32
        L.b2q_gen_column.argtypes = [C.c_void_p, C.c_int32, C.c_uint64, C.c_uint32, C.c_int64, C.c_int64, C.c_int64,
                                     C.c_int64, C.c_void_p]
        L.b2q_gen_column_strided.restype = C.c_int32
        L.b2q_gen_column_strided.argtypes = [C.c_void_p, C.c_int32, C.c_uint64, C.c_uint32, C.c_int64, C.c_int64, C.c_int64,
                                             C.c_int64, C.c_int64, C.c_void_p]
        L.b2q_comm_unique_id.restype = C.c_int32
        L.b2q_comm_unique_id.argtypes = [C.c_void_p]
        L.b2q_comm_init_rank.restype = C.c_int32
        L.b2q_comm_init_rank.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
        L.b2q_comm_init_all.restype = C.c_int32
        L.b2q_comm_init_all.argtypes = [C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_void_p)]
        L.b2q_comm_destroy.argtypes = [C.c_void_p]
        L.b2q_comm_rank.restype = C.c_int32
        L.b2q_comm_rank.argtypes = [C.c_void_p]
        L.b2q_comm_size.restype = C.c_int32
        L.b2q_comm_size.argtypes = [C.c_void_p]
        L.b2q_execute_work_unit_dist.restype = C.c_int32
        L.b2q_execute_work_unit_dist.argtypes = [C.c_void_p] + ewu + [C.c_void_p, C.POINTER(C.c_void_p)]
        L.b2q_execute_work_unit_multi.restype = C.c_int32
        L.b2q_execute_work_unit_multi.argtypes = [C.POINTER(C.c_void_p), C.c_int32, C.POINTER(C.c_size_t), C.c_int32,
                                                  C.POINTER(C.POINTER(abi.TableInfo)), C.POINTER(abi.ExecUnit),
                                                  C.POINTER(abi.CompilationOptions), C.POINTER(abi.ExecutionOptions), C.c_int32,
                                                  C.POINTER(C.c_void_p)]
        L.b2q_rs_device_columns.restype = C.c_int32
        L.b2q_rs_device_columns.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
        for n in ("b2q_device_columns_size", "b2q_device_columns_num_columns"):
            getattr(L, n).restype = C.c_size_t
            getattr(L, n).argtypes = [C.c_void_p]
        L.b2q_device_columns_device.restype = C.c_int32
        L.b2q_device_columns_device.argtypes = [C.c_void_p]
        L.b2q_device_columns_convert_ms.restype = C.c_double
        L.b2q_device_columns_convert_ms.argtypes = [C.c_void_p]
        L.b2q_device_columns_column.restype = C.c_void_p
        L.b2q_device_columns_column.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(abi.TypeInfo), C.POINTER(C.c_void_p),
                                                C.POINTER(C.c_int64)]
        L.b2q_device_columns_export_arrow.restype = C.c_int32
        L.b2q_device_columns_export_arrow.argtypes = [C.c_void_p, C.POINTER(C.c_char_p), C.POINTER(abi.ArrowSchema),
                                                      C.POINTER(abi.ArrowDeviceArray)]
        L.b2q_device_columns_free.argtypes = [C.c_void_p, C.c_void_p]
        if L.b2q_abi_version() != abi.ABI_VERSION:
            raise ImportError("libb2q.so ABI version mismatch")
        _lib = L
    return _lib


def _raise(code: int):
    msg = lib().b2q_last_error_message().decode() or lib().b2q_error_string(code).decode()
    if code == abi.ERR_CARDINALITY_ESTIMATION_REQUIRED:
        raise CardinalityEstimationRequired(code, msg)
    if code == abi.ERR_UNSUPPORTED:
        raise UnsupportedOnThisPath(code, msg)
    if code == abi.ERR_NO_DEVICE:
        raise NoDeviceError(code, msg)
    raise QueryExecutionError(code, msg)


def compilation_options(device_type: int = abi.DEVICE_GPU, hoist_literals: bool = True,
                        filter_on_deleted_column: bool = True) -> abi.CompilationOptions:
    """CompilationOptions::defaults(ExecutorDeviceType::GPU) — QueryEngine/CompilationOptions.h:52-65."""
    return abi.CompilationOptions(device_type, int(hoist_literals), int(not filter_on_deleted_column), 0)


def execution_options(allow_multifrag=True, output_columnar_hint=False, bigint_count=False, force_kernel=0,
                      device_ordinal=-1, result_on_device=False) -> abi.ExecutionOptions:
    eo = abi.ExecutionOptions()
    eo.result_on_device = int(result_on_device)
    eo.allow_multifrag = int(allow_multifrag)
    eo.output_columnar_hint = int(output_columnar_hint)
    eo.bigint_count = int(bigint_count)
    eo.force_kernel = force_kernel
    eo.device_ordinal = device_ordinal
    return eo


class ResultSet:
    """Output surface of QueryEngine/ResultSet.h for the numeric subset."""

    def __init__(self, handle):
        self._h = handle

    def __del__(self):
        if getattr(self, "_h", None):
            lib().b2q_rs_free(self._h)
            self._h = None

    def rowCount(self) -> int:
        return lib().b2q_rs_row_count(self._h)

    def colCount(self) -> int:
        return lib().b2q_rs_col_count(self._h)

    def entryCount(self) -> int:
        return lib().b2q_rs_entry_count(self._h)

    def isEmpty(self) -> bool:
        return bool(lib().b2q_rs_is_empty(self._h))

    def getColType(self, i: int):
        t = lib().b2q_rs_get_col_type(self._h, i)
        return (t.type, t.notnull, t.scale)

    def moveToBegin(self):
        lib().b2q_rs_move_to_begin(self._h)

    def getNextRow(self, translate_strings: bool = True, decimal_to_double: bool = True):
        nc = self.colCount()
        row = (abi.TargetValue * nc)()
        if not lib().b2q_rs_get_next_row(self._h, row, int(translate_strings), int(decimal_to_double)):
            return []
        return [v.py() for v in row]

    def rows(self, decimal_to_double: bool = True) -> List[tuple]:
        self.moveToBegin()
        L = lib()
        nc = self.colCount()
        row = (abi.TargetValue * nc)()
        out = []
        while L.b2q_rs_get_next_row(self._h, row, 0, int(decimal_to_double)):
            out.append(tuple(v.py() for v in row))
        return out

    def getRowAt(self, logical_index: int, translate_strings: bool = False, decimal_to_double: bool = True):
        """ResultSet::getRowAt / getRowAtNoTranslations (ResultSetIteration.cpp:266-284): the row of one entry (through the
        permutation when sorted) as a tuple, or () for an empty entry / an index past entryCount()."""
        row = (abi.TargetValue * self.colCount())()
        if not lib().b2q_rs_get_row_at(self._h, logical_index, row, int(translate_strings), int(decimal_to_double)):
            return ()
        return tuple(v.py() for v in row)

    def isRowAtEmpty(self, i: int) -> bool:
        return bool(lib().b2q_rs_is_row_at_empty(self._h, i))

    def getQueryMemDesc(self) -> abi.Plan:
        plan = abi.Plan()   # a copy: stays valid after the result set is freed
        C.memmove(C.byref(plan), lib().b2q_rs_query_mem_desc(self._h), C.sizeof(abi.Plan))
        return plan

    def getStorageBuffer(self) -> np.ndarray:
        """getStorage()->getUnderlyingBuffer() as bytes in the reference's row-wise layout."""
        n = C.c_size_t()
        p = lib().b2q_rs_storage_buffer(self._h, C.byref(n))
        if not n.value:
            return np.zeros(0, dtype=np.int8)
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_int8)), shape=(n.value,)).copy()

    def kernel_ms(self) -> float:
        return lib().b2q_rs_kernel_ms(self._h)

    def stats(self) -> dict:
        L = lib()
        return {"fragments_scanned": L.b2q_rs_stat(self._h, 0), "fragments_skipped": L.b2q_rs_stat(self._h, 1),
                "kernel_launches": L.b2q_rs_stat(self._h, 2), "h2d_bytes": L.b2q_rs_stat(self._h, 3),
                "sort_us": L.b2q_rs_stat(self._h, 4), "host_setup_us": L.b2q_rs_stat(self._h, 5),
                "host_stream_us": L.b2q_rs_stat(self._h, 6), "host_teardown_us": L.b2q_rs_stat(self._h, 7),
                "result_d2h_bytes": L.b2q_rs_stat(self._h, abi.STAT_RESULT_D2H_BYTES),
                "rows_scanned": L.b2q_rs_stat(self._h, abi.STAT_ROWS_SCANNED),
                "join_table": L.b2q_rs_stat(self._h, abi.STAT_JOIN_TABLE)}

    def columnarResults(self, num_threads: int = 8, with_scale: bool = False):
        """ColumnarResults(rows, num_columns, target_types) (QueryEngine/ColumnarResults.cpp:256-392): one numpy array per
        target in the target type's own dtype, rows in iteration order, NULLs as the type's inline sentinel.
        Returns [(sql_type, notnull, array), ...]."""
        L = lib()
        h = C.c_void_p()
        rc = L.b2q_columnar_results_create(self._h, int(num_threads), C.byref(h))
        if rc:
            _raise(rc)
        try:
            n = L.b2q_columnar_results_size(h)
            out = []
            for c in range(L.b2q_columnar_results_num_columns(h)):
                ti = abi.TypeInfo()
                ptr = L.b2q_columnar_results_column(h, c, C.byref(ti))
                dt = np.dtype(abi.NUMPY_OF[ti.type])
                arr = np.frombuffer(C.string_at(ptr, n * dt.itemsize), dtype=dt).copy() if n else np.empty(0, dtype=dt)
                out.append((ti.type, bool(ti.notnull), arr, ti.scale) if with_scale else (ti.type, bool(ti.notnull), arr))
            return out
        finally:
            L.b2q_columnar_results_free(h)

    def toArrow(self, names=None, num_threads: int = 8):
        """ArrowResultSetConverter::convertToArrow (QueryEngine/ArrowResultSetConverter.cpp): a pyarrow RecordBatch
        over the columnar results; the validity bitmap marks the inline NULL sentinels (dictionary-encoded strings
        travel as their int32 ids, as with translate_strings = false)."""
        import pyarrow as pa
        cols = self.columnarResults(num_threads, with_scale=True)
        arrays = []
        for ty, _nn, a, scale in cols:
            null = abi.NULL_OF[ty]
            mask = (a == null) if a.size else None
            if ty in abi.DECIMAL_TYPES:
                # arrow::decimal128(precision, scale) fed from the scaled int64 (ArrowResultSetConverter.cpp:1141, :1425-1440);
                # the precision is not carried across the C ABI: 19 digits hold every int64
                words = np.empty((a.size, 2), dtype=np.int64)
                words[:, 0] = a
                words[:, 1] = a >> 63                      # sign extension to 128 bits, little endian
                nulls = int(mask.sum()) if mask is not None else 0
                validity = pa.py_buffer(np.packbits(~mask, bitorder="little").tobytes()) if nulls else None
                arrays.append(pa.Array.from_buffers(pa.decimal128(19, scale), a.size, [validity, pa.py_buffer(words.tobytes())], nulls))
                continue
            arrays.append(pa.array(a, mask=mask if mask is not None and mask.any() else None))
        names = list(names) if names is not None else [f"col{i}" for i in range(len(arrays))]
        return pa.RecordBatch.from_arrays(arrays, names=names)

    def deviceColumns(self, stream: Optional[int] = None) -> "DeviceColumns":
        """The same columns as columnarResults(), made on the result's GPU (b2q_rs_device_columns): a result_on_device set is
        read where it lies, without a device-to-host copy.  `stream`: the CUDA stream (handle as an int) the conversion is
        ordered on; None = torch's current stream when torch is loaded, else the default stream."""
        if stream is None:
            stream = _current_torch_stream()
        h = C.c_void_p()
        rc = lib().b2q_rs_device_columns(self._h, C.c_void_p(stream), C.byref(h))
        if rc:
            _raise(rc)
        return DeviceColumns(h, stream)

    def getNDVEstimator(self) -> int:
        """ResultSet::getNDVEstimator (CardinalityEstimator.cpp:33-52) of an estimator query."""
        return lib().b2q_rs_get_ndv_estimator(self._h)

    def getHostEstimatorBuffer(self) -> np.ndarray:
        n = C.c_size_t()
        p = lib().b2q_rs_estimator_buffer(self._h, C.byref(n))
        if not p or n.value == 0:
            return np.zeros(0, dtype=np.uint8)
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(n.value,)).copy()

    def sort(self, order_entries, top_n: int = 0):
        """ResultSet::sort(order_entries, top_n) (ResultSet.h:279): order_entries = [(tle_no, is_desc, nulls_first)]."""
        arr = (abi.OrderEntry * max(len(order_entries), 1))()
        for i, (tle, desc, nf) in enumerate(order_entries):
            arr[i].tle_no, arr[i].is_desc, arr[i].nulls_first = tle, int(desc), int(nf)
        rc = lib().b2q_rs_sort(self._h, arr, len(order_entries), top_n)
        if rc:
            _raise(rc)

    def dropFirstN(self, n: int):
        lib().b2q_rs_drop_first_n(self._h, n)

    def keepFirstN(self, n: int):
        lib().b2q_rs_keep_first_n(self._h, n)


def _current_torch_stream() -> int:
    import sys
    torch = sys.modules.get("torch")
    if torch is None or not torch.cuda.is_initialized():
        return 0
    return int(torch.cuda.current_stream().cuda_stream)


class _CudaArray:
    """__cuda_array_interface__ (v3) over device memory a DeviceColumns owns; keeps that owner alive."""

    def __init__(self, owner, ptr: int, n: int, typestr: str):
        self._owner = owner
        # "stream": None: b2q_rs_device_columns has completed the columns before it returned
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr or 0, False), "version": 3,
                                         "strides": None, "stream": None}


class ArrowExport:
    """An exported Arrow C Device record batch (ArrowSchema + ArrowDeviceArray): the ctypes structs, owned here until
    release() (or garbage collection) calls their release callbacks."""

    def __init__(self):
        self.schema = abi.ArrowSchema()
        self.array = abi.ArrowDeviceArray()

    def release(self):
        for obj in (self.array.array, self.schema):
            if obj.release:
                obj.release(C.byref(obj))

    def __del__(self):
        self.release()


class DeviceColumns:
    """ColumnarResults in device memory (b2q_rs_device_columns / b2q_device_columns_*): per target the values in the target
    type's width (NULLs as the inline sentinel), an Arrow validity bitmap (None when the column has no NULL) and the NULL
    count."""

    def __init__(self, handle, stream: int = 0):
        self._h = handle
        self._stream = stream

    def __del__(self):
        if getattr(self, "_h", None):
            lib().b2q_device_columns_free(self._h, C.c_void_p(self._stream))
            self._h = None

    def size(self) -> int:
        return lib().b2q_device_columns_size(self._h)

    def num_columns(self) -> int:
        return lib().b2q_device_columns_num_columns(self._h)

    def device(self) -> int:
        return lib().b2q_device_columns_device(self._h)

    def convert_ms(self) -> float:
        """CUDA-event time of the conversion kernel."""
        return lib().b2q_device_columns_convert_ms(self._h)

    def column(self, i: int):
        """(values device pointer, (sql_type, notnull, scale), validity device pointer or None, null_count)"""
        ti, valid, nulls = abi.TypeInfo(), C.c_void_p(), C.c_int64()
        ptr = lib().b2q_device_columns_column(self._h, i, C.byref(ti), C.byref(valid), C.byref(nulls))
        if ptr is None and i >= self.num_columns():
            raise IndexError(i)
        return ptr or 0, (ti.type, bool(ti.notnull), ti.scale), valid.value, nulls.value

    def tensors(self):
        """[(values, validity)] as zero-copy CUDA torch tensors (validity: uint8 bitmap bytes, or None); they keep this
        object — and so the device memory — alive."""
        import torch
        n = self.size()
        out = []
        for i in range(self.num_columns()):
            ptr, (ty, _nn, _sc), valid, _nulls = self.column(i)
            dev = torch.device("cuda", self.device())
            vals = torch.as_tensor(_CudaArray(self, ptr, n, np.dtype(abi.NUMPY_OF[ty]).str), device=dev)
            mask = torch.as_tensor(_CudaArray(self, valid, (n + 7) // 8, "|u1"), device=dev) if valid else None
            out.append((vals, mask))
        return out

    def to_host(self):
        """[(sql_type, notnull, values ndarray, validity bytes ndarray or None, null_count)] copied back to the host."""
        out = []
        for i, (vals, mask) in enumerate(self.tensors()):
            _p, (ty, nn, _sc), _v, nulls = self.column(i)
            out.append((ty, nn, vals.cpu().numpy(), None if mask is None else mask.cpu().numpy(), nulls))
        return out

    def export_arrow(self, names=None) -> ArrowExport:
        """b2q_device_columns_export_arrow: the columns as an Arrow C Device record batch (a "+s" struct of one child per
        target; device_type ARROW_DEVICE_CUDA).  The buffers stay alive until both this object and the export are released."""
        ex = ArrowExport()
        c_names = None
        if names is not None:
            ex._names = [str(x).encode() for x in names]
            c_names = (C.c_char_p * len(ex._names))(*ex._names)
        rc = lib().b2q_device_columns_export_arrow(self._h, c_names, C.byref(ex.schema), C.byref(ex.array))
        if rc:
            _raise(rc)
        return ex


class Partial:
    """Per-device dense partial-aggregate table (between the scan and the cross-device merge)."""

    def __init__(self, handle):
        self._h = handle

    def __del__(self):
        if getattr(self, "_h", None):
            lib().b2q_partial_free(self._h)
            self._h = None

    def arrays(self):
        """[(device_ptr, count, dtype, redop)] — what the caller all-reduces (one collective per array)."""
        L = lib()
        out = []
        for i in range(L.b2q_partial_num_arrays(self._h)):
            p, n, dt, op = C.c_void_p(), C.c_int64(), C.c_int32(), C.c_int32()
            rc = L.b2q_partial_array(self._h, i, C.byref(p), C.byref(n), C.byref(dt), C.byref(op))
            if rc:
                _raise(rc)
            out.append((p.value, n.value, dt.value, op.value))
        return out

    def is_mergeable(self) -> bool:
        return bool(lib().b2q_partial_is_mergeable(self._h))

    def plan(self) -> abi.Plan:
        plan = abi.Plan()
        C.memmove(C.byref(plan), lib().b2q_partial_plan(self._h), C.sizeof(abi.Plan))
        return plan

    def kernel_ms(self) -> float:
        return lib().b2q_partial_kernel_ms(self._h)

    def finalize(self, stream: int = 0) -> ResultSet:
        h = C.c_void_p()
        rc = lib().b2q_partial_finalize(self._h, C.c_void_p(stream), C.byref(h))
        if rc:
            _raise(rc)
        return ResultSet(h)


class Executor:
    """Executor::executeWorkUnit for the scan/filter/group-by/aggregate path."""

    def __init__(self, device_ordinal: int = -1):
        self.device_ordinal = device_ordinal
        lib()

    @staticmethod
    def _built_table(query_infos, memory_level):
        if isinstance(query_infos, abi.BuiltTable):
            return query_infos
        return query_infos.build(memory_level)

    def plan(self, ra_exe_unit: abi.BuiltUnit, query_infos, co=None, eo=None, max_groups_buffer_entry_guess: int = 0,
             has_cardinality_estimation: bool = False, memory_level: int = abi.CPU_LEVEL) -> abi.Plan:
        """Planning only (host; works without a GPU)."""
        co = co or compilation_options()
        eo = eo or execution_options(device_ordinal=self.device_ordinal)
        bt = self._built_table(query_infos, memory_level)
        h = C.c_void_p()
        rc = lib().b2q_plan(C.byref(ra_exe_unit.unit), C.byref(bt.info), C.byref(co), C.byref(eo),
                            max_groups_buffer_entry_guess, int(has_cardinality_estimation), C.byref(h))
        if rc:
            _raise(rc)
        plan = abi.Plan()
        C.memmove(C.byref(plan), lib().b2q_query_plan(h), C.sizeof(abi.Plan))
        lib().b2q_query_free(h)
        return plan

    def resultSetFromStorage(self, storage: np.ndarray, ra_exe_unit: abi.BuiltUnit, query_infos, co=None, eo=None,
                             max_groups_buffer_entry_guess: int = 0, has_cardinality_estimation: bool = False,
                             memory_level: int = abi.CPU_LEVEL) -> ResultSet:
        """ResultSet(targets, device_type, query_mem_desc, ...) + allocateStorage(buffer) (ResultSet.h:183-217): the read-out
        surface over a group-by buffer the caller already holds, laid out as this unit's descriptor says.  Host only."""
        co = co or compilation_options()
        eo = eo or execution_options(device_ordinal=self.device_ordinal)
        bt = self._built_table(query_infos, memory_level)
        q = C.c_void_p()
        rc = lib().b2q_plan(C.byref(ra_exe_unit.unit), C.byref(bt.info), C.byref(co), C.byref(eo),
                            max_groups_buffer_entry_guess, int(has_cardinality_estimation), C.byref(q))
        if rc:
            _raise(rc)
        try:
            buf = np.ascontiguousarray(storage).view(np.uint8)
            h = C.c_void_p()
            rc = lib().b2q_rs_create_from_storage(q, buf.ctypes.data if buf.size else None, buf.size, C.byref(h))
            if rc:
                _raise(rc)
        finally:
            lib().b2q_query_free(q)
        return ResultSet(h)

    def executeWorkUnit(self, max_groups_buffer_entry_guess: int, is_agg: bool, query_infos, ra_exe_unit: abi.BuiltUnit,
                        co: Optional[abi.CompilationOptions] = None, eo: Optional[abi.ExecutionOptions] = None,
                        has_cardinality_estimation: bool = False, memory_level: int = abi.CPU_LEVEL,
                        result_on_device: Optional[bool] = None) -> ResultSet:
        """result_on_device=True: the result stays in GPU memory (ResultSet.deviceColumns() reads it there; the first host
        accessor copies it back once).  None keeps what `eo` says."""
        co = co or compilation_options()
        eo = eo or execution_options(device_ordinal=self.device_ordinal)
        if result_on_device is not None:
            eo = abi.ExecutionOptions.from_buffer_copy(eo)
            eo.result_on_device = int(result_on_device)
        bt = self._built_table(query_infos, memory_level)
        guess = C.c_size_t(max_groups_buffer_entry_guess)
        h = C.c_void_p()
        rc = lib().b2q_execute_work_unit(C.byref(guess), int(is_agg), C.byref(bt.info), C.byref(ra_exe_unit.unit),
                                         C.byref(co), C.byref(eo), int(has_cardinality_estimation), C.byref(h))
        if rc:
            _raise(rc)
        return ResultSet(h)

    def executePartial(self, max_groups_buffer_entry_guess: int, is_agg: bool, query_infos, ra_exe_unit: abi.BuiltUnit,
                       co=None, eo=None, has_cardinality_estimation: bool = False,
                       memory_level: int = abi.CPU_LEVEL, stream: int = 0) -> Partial:
        co = co or compilation_options()
        eo = eo or execution_options(device_ordinal=self.device_ordinal)
        bt = self._built_table(query_infos, memory_level)
        guess = C.c_size_t(max_groups_buffer_entry_guess)
        h = C.c_void_p()
        rc = lib().b2q_execute_partial(C.byref(guess), int(is_agg), C.byref(bt.info), C.byref(ra_exe_unit.unit),
                                       C.byref(co), C.byref(eo), int(has_cardinality_estimation), C.c_void_p(stream),
                                       C.byref(h))
        if rc:
            _raise(rc)
        return Partial(h)


class Comm:
    """One rank of a multi-GPU communicator inside libb2q (NCCL).  `Comm.init_rank` for one process per GPU (the 128-byte id
    is made by rank 0 with `Comm.unique_id()` and broadcast by the caller's own plumbing, e.g. torch.distributed);
    `Comm.init_all` for one process driving several devices."""

    def __init__(self, handle):
        self.h = handle

    @staticmethod
    def _host_nccl_first():
        """libb2q binds whatever libnccl.so.2 the process holds.  torch ships its own and breaks if another copy with the same
        SONAME got there first, so a Python host that has torch loads it before libb2q touches NCCL."""
        try:
            import torch  # noqa: F401  (plumbing: makes torch's bundled libnccl the process's NCCL)
            import torch.cuda.nccl as _n
            _n.version()
        except Exception:
            pass

    @staticmethod
    def unique_id() -> bytes:
        Comm._host_nccl_first()
        buf = C.create_string_buffer(abi.COMM_ID_BYTES)
        rc = lib().b2q_comm_unique_id(buf)
        if rc:
            _raise(rc)
        return buf.raw

    @classmethod
    def init_rank(cls, unique_id: bytes, nranks: int, rank: int, device: int = -1) -> "Comm":
        cls._host_nccl_first()
        h = C.c_void_p()
        rc = lib().b2q_comm_init_rank(C.c_char_p(unique_id), nranks, rank, device, C.byref(h))
        if rc:
            _raise(rc)
        return cls(h)

    @classmethod
    def init_all(cls, devices: Sequence[int]):
        cls._host_nccl_first()
        arr = (C.c_int32 * len(devices))(*devices)
        out = (C.c_void_p * len(devices))()
        rc = lib().b2q_comm_init_all(arr, len(devices), out)
        if rc:
            _raise(rc)
        return [cls(C.c_void_p(h)) for h in out]

    def rank(self):
        return lib().b2q_comm_rank(self.h)

    def size(self):
        return lib().b2q_comm_size(self.h)

    def destroy(self):
        if getattr(self, "h", None):
            lib().b2q_comm_destroy(self.h)
            self.h = None


def execute_work_unit_dist(comm: Comm, executor: "Executor", max_groups_buffer_entry_guess: int, is_agg: bool, query_infos,
                           ra_exe_unit: abi.BuiltUnit, co=None, eo=None, has_cardinality_estimation: bool = False,
                           memory_level: int = abi.GPU_LEVEL, stream: int = 0) -> ResultSet:
    """This rank's share of a multi-GPU work unit: scan -> NCCL merge inside libb2q -> materialise.  `query_infos` holds this
    rank's fragments plus the other ranks' fragments as chunk stats (abi.Table.add_remote_fragment)."""
    co = co or compilation_options()
    eo = eo or execution_options(device_ordinal=executor.device_ordinal)
    bt = executor._built_table(query_infos, memory_level)
    guess = C.c_size_t(max_groups_buffer_entry_guess)
    h = C.c_void_p()
    rc = lib().b2q_execute_work_unit_dist(comm.h, C.byref(guess), int(is_agg), C.byref(bt.info), C.byref(ra_exe_unit.unit), C.byref(co),
                                          C.byref(eo), int(has_cardinality_estimation), C.c_void_p(stream), C.byref(h))
    if rc:
        _raise(rc)
    return ResultSet(h)


def execute_work_unit_multi(comms: Sequence[Comm], executor: "Executor", max_groups_buffer_entry_guess: int, is_agg: bool,
                            tables_per_device, ra_exe_unit: abi.BuiltUnit, co=None, eo=None,
                            has_cardinality_estimation: bool = False, memory_level: int = abi.GPU_LEVEL) -> ResultSet:
    """One call, one host thread per device inside libb2q (Execute.cpp:3055-3101): tables_per_device[i] is what device i scans."""
    co = co or compilation_options()
    eo = eo or execution_options()
    bts = [executor._built_table(t, memory_level) for t in tables_per_device]
    infos = (C.POINTER(abi.TableInfo) * len(bts))(*[C.pointer(bt.info) for bt in bts])
    hs = (C.c_void_p * len(comms))(*[c.h for c in comms])
    guess = C.c_size_t(max_groups_buffer_entry_guess)
    h = C.c_void_p()
    rc = lib().b2q_execute_work_unit_multi(hs, len(comms), C.byref(guess), int(is_agg), infos, C.byref(ra_exe_unit.unit), C.byref(co),
                                           C.byref(eo), int(has_cardinality_estimation), C.byref(h))
    if rc:
        _raise(rc)
    return ResultSet(h)


def gen_column_device(dst_ptr: int, sql_type: int, seed: int, col_tag: int, row0: int, count: int, lo: int = 0,
                      span: int = 1, stream: int = 0, stride: int = 1):
    rc = lib().b2q_gen_column_strided(C.c_void_p(dst_ptr), sql_type, seed, col_tag, row0, count, lo, span, stride,
                                      C.c_void_p(stream))
    if rc:
        _raise(rc)
