"""ctypes mirror of include/b2q.h (the C ABI of the path) plus small builders for its POD inputs.

The structs here are field-for-field the ones declared in ``include/b2q.h``; the enum values are the reference's
own (Shared/sqltypes.h:65-99, Shared/sqldefs.h:31-40,76-90, QueryEngine/enums.h:54-60).  ``tests/test_abi.py``
checks sizes/offsets against the C compiler's view of the header.

Nothing in this module touches a GPU; it is shared by the product host wrapper (``executor.py``) and by the test
oracle's loader (``tests/oracle_lib.py``).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

# ---- SQLTypes subset -------------------------------------------------------------------------------------
kINT, kSMALLINT, kFLOAT, kDOUBLE, kBIGINT, kTINYINT = 6, 7, 8, 9, 12, 22
kBOOLEAN = 1  # only as the type of the deleted-rows column
kCHAR, kVARCHAR, kTEXT = 2, 3, 13   # dictionary-encoded strings: int32 ids (uint8 / uint16 under DICT(8) / DICT(16))
kTIME, kTIMESTAMP, kDATE = 10, 11, 14   # int64
kNUMERIC, kDECIMAL = 4, 5               # value * 10**scale as int64 (int32 / int16 under the DDL's ENCODING FIXED)
DECIMAL_TYPES = (kNUMERIC, kDECIMAL)
STRING_TYPES = (kCHAR, kVARCHAR, kTEXT)
TIME_TYPES = (kTIME, kTIMESTAMP, kDATE)
# ---- SQLOps subset ---------------------------------------------------------------------------------------
kEQ, kNE, kLT, kGT, kLE, kGE, kAND, kOR = 0, 2, 3, 4, 5, 6, 7, 8
kNOT, kISNULL = 9, 16   # Analyzer::UOper
# ---- SQLAgg subset ---------------------------------------------------------------------------------------
kAVG, kMIN, kMAX, kSUM, kCOUNT = 0, 1, 2, 3, 4
# ---- QueryDescriptionType --------------------------------------------------------------------------------
GroupByPerfectHash, GroupByBaselineHash, Projection, TableFunction, NonGroupedAggregate, Estimator = range(6)

# ---- error codes -----------------------------------------------------------------------------------------
OK = 0
ERR_OUT_OF_SLOTS = 3
ERR_UNSUPPORTED = 1000
ERR_CARDINALITY_ESTIMATION_REQUIRED = 1001
ERR_INVALID_ARGUMENT = 1002
ERR_NO_DEVICE = 1003
ERR_CUDA = 1004
ERR_KEY_OUT_OF_RANGE = 1005

COMM_ID_BYTES = 128
ABI_VERSION = 8   # B2Q_ABI_VERSION of include/b2q.h this mirror was written against
EXPR_COLUMN_VAR, EXPR_CONSTANT, EXPR_BIN_OPER, EXPR_AGG, EXPR_UOPER = 1, 2, 3, 4, 5
CPU_LEVEL, GPU_LEVEL = 1, 2
DEVICE_CPU, DEVICE_GPU = 0, 1
KERNEL_AUTO, KERNEL_NON_GROUPED, KERNEL_PERFECT_SMEM, KERNEL_PERFECT_GLOBAL, KERNEL_BASELINE_GLOBAL, KERNEL_BASELINE_PROBE = range(6)
DT_INT64, DT_FLOAT64, DT_UINT8 = 0, 1, 2
RED_SUM, RED_MIN, RED_MAX, RED_BOR = 0, 1, 2, 3
# b2q_rs_stat
(STAT_FRAGMENTS_SCANNED, STAT_FRAGMENTS_SKIPPED, STAT_KERNEL_LAUNCHES, STAT_H2D_BYTES, STAT_SORT_US, STAT_HOST_SETUP_US,
 STAT_HOST_STREAM_US, STAT_HOST_TEARDOWN_US, STAT_RESULT_D2H_BYTES, STAT_ROWS_SCANNED, STAT_JOIN_TABLE) = range(11)
# values of STAT_JOIN_TABLE: the join table the scan probed (b2q.h B2Q_JOIN_TABLE_*)
(JOIN_TABLE_NONE, JOIN_TABLE_CALLER, JOIN_TABLE_INT32_HBM, JOIN_TABLE_INT2_HBM, JOIN_TABLE_INT32_SMEM, JOIN_TABLE_INT2_SMEM,
 JOIN_TABLE_UINT16_SMEM) = range(7)

MAX_SLOTS = 16
MAX_TARGETS = 16
MAX_GROUP_COLS = 4

# Shared/InlineNullValues.h:30-36
NULL_TINYINT = -(2**7)
NULL_SMALLINT = -(2**15)
NULL_INT = -(2**31)
NULL_BIGINT = -(2**63)
NULL_DOUBLE = float(np.finfo(np.float64).tiny)  # DBL_MIN: smallest NORMAL double
NULL_FLOAT = np.float32(np.finfo(np.float32).tiny)  # FLT_MIN
EMPTY_KEY_64 = 2**63 - 1
EMPTY_KEY_32 = 2**31 - 1

NUMPY_OF = {kBOOLEAN: np.int8, kTINYINT: np.int8, kSMALLINT: np.int16, kINT: np.int32, kBIGINT: np.int64, kDOUBLE: np.float64, kFLOAT: np.float32,
            kCHAR: np.int32, kVARCHAR: np.int32, kTEXT: np.int32, kTIME: np.int64, kTIMESTAMP: np.int64, kDATE: np.int64,
            kNUMERIC: np.int64, kDECIMAL: np.int64}
SIZE_OF = {kBOOLEAN: 1, kTINYINT: 1, kSMALLINT: 2, kINT: 4, kBIGINT: 8, kDOUBLE: 8, kFLOAT: 4, kCHAR: 4, kVARCHAR: 4, kTEXT: 4, kTIME: 8, kTIMESTAMP: 8, kDATE: 8,
           kNUMERIC: 8, kDECIMAL: 8}
NULL_OF = {kBOOLEAN: NULL_TINYINT, kTINYINT: NULL_TINYINT, kSMALLINT: NULL_SMALLINT, kINT: NULL_INT, kBIGINT: NULL_BIGINT, kDOUBLE: NULL_DOUBLE, kFLOAT: NULL_FLOAT,
           kCHAR: NULL_INT, kVARCHAR: NULL_INT, kTEXT: NULL_INT, kTIME: NULL_BIGINT, kTIMESTAMP: NULL_BIGINT, kDATE: NULL_BIGINT,
           kNUMERIC: NULL_BIGINT, kDECIMAL: NULL_BIGINT}


class TypeInfo(C.Structure):
    _fields_ = [("type", C.c_int32), ("notnull", C.c_int32), ("scale", C.c_int32)]


class Expr(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("ti", TypeInfo),
        ("col_id", C.c_int32),
        ("op", C.c_int32),
        ("left", C.c_int32),
        ("right", C.c_int32),
        ("ival", C.c_int64),
        ("dval", C.c_double),
        ("is_null", C.c_int32),
        ("rte_idx", C.c_int32),
    ]


class OrderEntry(C.Structure):
    """Analyzer::OrderEntry (Analyzer/Analyzer.h:2960-2968)."""
    _fields_ = [("tle_no", C.c_int32), ("is_desc", C.c_int8), ("nulls_first", C.c_int8), ("pad_", C.c_int8 * 2)]


class ExecUnit(C.Structure):
    _fields_ = [
        ("exprs", C.POINTER(Expr)),
        ("num_exprs", C.c_int32),
        ("simple_quals", C.POINTER(C.c_int32)),
        ("num_simple_quals", C.c_int32),
        ("quals", C.POINTER(C.c_int32)),
        ("num_quals", C.c_int32),
        ("groupby_exprs", C.POINTER(C.c_int32)),
        ("num_groupby_exprs", C.c_int32),
        ("target_exprs", C.POINTER(C.c_int32)),
        ("num_target_exprs", C.c_int32),
        ("scan_limit", C.c_int64),
        ("num_join_quals", C.c_int32),
        ("has_estimator", C.c_int32),
        ("has_union_all", C.c_int32),
        ("has_window_function", C.c_int32),
        ("order_entries", C.POINTER(OrderEntry)),
        ("num_order_entries", C.c_int32),
        ("has_limit", C.c_int32),
        ("limit", C.c_int64),
        ("offset", C.c_int64),
        ("join_qual", C.c_int32),
        ("join_type", C.c_int32),
        ("inner_table", C.c_void_p),   # const B2QTableInfo*
        ("estimator_args", C.POINTER(C.c_int32)),
        ("num_estimator_args", C.c_int32),
        ("pad_", C.c_int32),
    ]


class ChunkStats(C.Structure):
    _fields_ = [
        ("int_min", C.c_int64),
        ("int_max", C.c_int64),
        ("fp_min", C.c_double),
        ("fp_max", C.c_double),
        ("has_nulls", C.c_int32),
        ("pad_", C.c_int32),
    ]


class FragmentInfo(C.Structure):
    _fields_ = [
        ("fragment_id", C.c_int32),
        ("device_id", C.c_int32),
        ("num_tuples", C.c_int64),
        ("col_buffers", C.POINTER(C.c_void_p)),
        ("col_stats", C.POINTER(ChunkStats)),
    ]


class TableInfo(C.Structure):
    _fields_ = [
        ("num_cols", C.c_int32),
        ("col_types", C.POINTER(TypeInfo)),
        ("num_fragments", C.c_int32),
        ("fragments", C.POINTER(FragmentInfo)),
        ("memory_level", C.c_int32),
        ("deleted_column_plus1", C.c_int32),
        ("col_encoded_sizes", C.POINTER(C.c_int8)),
    ]


class CompilationOptions(C.Structure):
    _fields_ = [("device_type", C.c_int32), ("hoist_literals", C.c_int32), ("ignore_deleted_column", C.c_int32),
                ("pad_", C.c_int32)]


class ExecutionOptions(C.Structure):
    _fields_ = [
        ("allow_multifrag", C.c_int32),
        ("output_columnar_hint", C.c_int32),
        ("bigint_count", C.c_int32),
        ("force_kernel", C.c_int32),
        ("device_ordinal", C.c_int32),
        ("result_on_device", C.c_int32),   # 1: the result stays in device memory until a host accessor needs it
    ]


class TargetInfo(C.Structure):
    _fields_ = [
        ("is_agg", C.c_int32),
        ("agg_kind", C.c_int32),
        ("sql_type", TypeInfo),
        ("agg_arg_type", TypeInfo),
        ("skip_null_val", C.c_int32),
        ("is_distinct", C.c_int32),
        ("arg_col_id", C.c_int32),
        ("first_slot", C.c_int32),
    ]


class Plan(C.Structure):
    _fields_ = [
        ("query_desc_type", C.c_int32),
        ("keyless_hash", C.c_int32),
        ("idx_target_as_key", C.c_int32),
        ("output_columnar", C.c_int32),
        ("interleaved_bins_on_gpu", C.c_int32),
        ("group_col_width", C.c_int32),
        ("effective_key_width", C.c_int32),
        ("num_targets", C.c_int32),
        ("num_slots", C.c_int32),
        ("key_col_id", C.c_int32),
        ("entry_count", C.c_int64),
        ("min_val", C.c_int64),
        ("max_val", C.c_int64),
        ("bucket", C.c_int64),
        ("has_nulls", C.c_int32),
        ("kernel", C.c_int32),
        ("row_size", C.c_int64),
        ("buffer_size", C.c_int64),
        ("num_group_cols", C.c_int32),
        ("group_col_ids", C.c_int32 * MAX_GROUP_COLS),
        ("group_col_widths", C.c_int8 * MAX_GROUP_COLS),
        ("pad2_", C.c_int32),
        ("slot_padded_width", C.c_int8 * MAX_SLOTS),
        ("slot_logical_width", C.c_int8 * MAX_SLOTS),
        ("slot_offset", C.c_int64 * MAX_SLOTS),
        ("init_vals", C.c_int64 * MAX_SLOTS),
        ("targets", TargetInfo * MAX_TARGETS),
        ("join_min_key", C.c_int64),
        ("join_max_key", C.c_int64),
        ("join_entry_count", C.c_int64),
        ("join_outer_col", C.c_int32),
        ("join_inner_col", C.c_int32),
        ("count_distinct_min", C.c_int64 * MAX_TARGETS),
        ("count_distinct_bits", C.c_int64 * MAX_TARGETS),
    ]

    #: fields that must agree between the product planner and the oracle planner
    PARITY_FIELDS = (
        "query_desc_type", "keyless_hash", "idx_target_as_key", "output_columnar", "group_col_width",
        "effective_key_width", "num_targets", "num_slots", "key_col_id", "entry_count", "min_val", "max_val",
        "bucket", "has_nulls", "row_size", "buffer_size", "num_group_cols",
        "join_min_key", "join_max_key", "join_entry_count", "join_outer_col", "join_inner_col",
    )

    def as_dict(self) -> dict:
        d = {k: getattr(self, k) for k in self.PARITY_FIELDS}
        n = self.num_slots
        d["slot_padded_width"] = list(self.slot_padded_width[:n])
        d["slot_logical_width"] = list(self.slot_logical_width[:n])
        d["slot_offset"] = list(self.slot_offset[:n])
        d["init_vals"] = list(self.init_vals[:n])
        d["group_col_ids"] = list(self.group_col_ids[: self.num_group_cols])
        d["group_col_widths"] = list(self.group_col_widths[: self.num_group_cols])
        d["targets"] = [
            (t.is_agg, t.agg_kind, t.sql_type.type, t.sql_type.notnull, t.agg_arg_type.type,
             t.agg_arg_type.notnull, t.skip_null_val, t.arg_col_id, t.first_slot, t.sql_type.scale, t.agg_arg_type.scale, t.is_distinct)
            for t in self.targets[: self.num_targets]
        ]
        d["count_distinct"] = [(self.count_distinct_min[i], self.count_distinct_bits[i]) for i in range(self.num_targets)]
        return d


class TargetValue(C.Structure):
    _fields_ = [("is_fp", C.c_int32), ("is_null", C.c_int32), ("ival", C.c_int64), ("dval", C.c_double)]

    def py(self):
        """Python value: None for NULL, float for fp targets, int otherwise."""
        if self.is_null:
            return None
        return self.dval if self.is_fp else self.ival


# ---- Arrow C Data / C Device Data Interface (include/b2q_arrow.h) -----------------------------------------------------
ARROW_FLAG_NULLABLE = 2
ARROW_DEVICE_CPU, ARROW_DEVICE_CUDA = 1, 2


class ArrowSchema(C.Structure):
    pass


ArrowSchema._fields_ = [
    ("format", C.c_char_p),
    ("name", C.c_char_p),
    ("metadata", C.c_char_p),
    ("flags", C.c_int64),
    ("n_children", C.c_int64),
    ("children", C.POINTER(C.POINTER(ArrowSchema))),
    ("dictionary", C.POINTER(ArrowSchema)),
    ("release", C.CFUNCTYPE(None, C.POINTER(ArrowSchema))),
    ("private_data", C.c_void_p),
]


class ArrowArray(C.Structure):
    pass


ArrowArray._fields_ = [
    ("length", C.c_int64),
    ("null_count", C.c_int64),
    ("offset", C.c_int64),
    ("n_buffers", C.c_int64),
    ("n_children", C.c_int64),
    ("buffers", C.POINTER(C.c_void_p)),
    ("children", C.POINTER(C.POINTER(ArrowArray))),
    ("dictionary", C.POINTER(ArrowArray)),
    ("release", C.CFUNCTYPE(None, C.POINTER(ArrowArray))),
    ("private_data", C.c_void_p),
]


class ArrowDeviceArray(C.Structure):
    _fields_ = [
        ("array", ArrowArray),
        ("device_id", C.c_int64),
        ("device_type", C.c_int32),
        ("sync_event", C.c_void_p),   # ARROW_DEVICE_CUDA: a cudaEvent_t*
        ("reserved", C.c_int64 * 3),
    ]


class Params(C.Structure):
    _fields_ = [
        ("error_codes", C.c_void_p),
        ("total_matched", C.c_void_p),
        ("group_by_buffers", C.c_void_p),
        ("num_fragments", C.POINTER(C.c_uint32)),
        ("num_tables", C.POINTER(C.c_uint32)),
        ("row_index_resume", C.c_void_p),
        ("col_buffers", C.POINTER(C.POINTER(C.c_void_p))),
        ("literals", C.c_void_p),
        ("num_rows", C.POINTER(C.c_int64)),
        ("frag_row_offsets", C.c_void_p),
        ("frag_ids", C.c_void_p),
        ("max_matched", C.c_void_p),
        ("init_agg_value", C.POINTER(C.c_int64)),
        ("join_hash_tables", C.c_void_p),
        ("row_func_mgr", C.c_void_p),
    ]


# =========================================================================================================
# Builders (host-side conveniences; they only assemble the POD structs above)
# =========================================================================================================
@dataclass
class _Node:
    kind: int
    type: int = 0
    notnull: bool = False
    col_id: int = -1
    op: int = 0
    left: int = -1
    right: int = -1
    ival: int = 0
    dval: float = 0.0
    is_null: bool = False
    rte_idx: int = 0
    scale: int = 0      # SQLTypeInfo::get_scale() of a DECIMAL / NUMERIC


class UnitBuilder:
    """Assembles a RelAlgExecutionUnit mirror.  Mirrors how Tests/GroupByTest.cpp:121-130 builds one by hand:
    ColumnVar / Constant / BinOper / AggExpr nodes, then quals / groupby_exprs / target_exprs lists."""

    def __init__(self, table: "Table"):
        self.table = table
        self.nodes: List[_Node] = []
        self.simple_quals: List[int] = []
        self.quals: List[int] = []
        self.groupby: List[int] = []
        self.targets: List[int] = []
        self.scan_limit = 0
        self.unsupported: Dict[str, int] = {}
        self.inner: Optional["Table"] = None            # input_descs[1] of a one-level INNER / LEFT hash join
        self.join_type = 0                              # JoinType: INNER = 0, LEFT = 1
        self.join_qual: int = -1
        self.estimator_kind = 0                         # 1 = NDVEstimator, 2 = LargeNDVEstimator
        self.estimator_args: List[int] = []
        self.order: List[Tuple[int, bool, bool]] = []   # sort_info.order_entries: (tle_no 1-based, is_desc, nulls_first)
        self.limit: Optional[int] = None
        self.offset = 0

    # -- expression nodes ---------------------------------------------------------------------------------
    def col(self, col_id: int, rte_idx: int = 0) -> int:
        """ColumnVar; rte_idx 1 = a column of the joined inner table (set with join())."""
        t, nn = (self.inner if rte_idx else self.table).col_types[col_id]
        if rte_idx and self.join_type == 1:
            nn = False      # the inner side of a LEFT join is nullable (RelAlgTranslator marks it so)
        self.nodes.append(_Node(EXPR_COLUMN_VAR, t, nn, col_id=col_id, rte_idx=rte_idx,
                                scale=(self.inner if rte_idx else self.table).col_scales.get(col_id, 0)))
        return len(self.nodes) - 1

    def join(self, inner: "Table", outer_col: int, inner_col: int, join_type: int = 0):
        """join_quals[0] = {outer.col = inner.col}, JoinType INNER (0) or LEFT (1); the inner table is passed as one
        concatenated fragment, the way the hash-join column fetch sees it."""
        self.inner = inner
        self.join_type = join_type
        self.join_qual = self.binop(kEQ, self.col(outer_col, 0), self.col(inner_col, 1))
        return self

    def const(self, value, sql_type: Optional[int] = None, is_null: bool = False, scale: int = 0) -> int:
        """Constant.  A DECIMAL constant carries its Datum the way the analyzer folds it: bigintval = value * 10**scale
        (pass the already scaled integer)."""
        if sql_type is None:
            sql_type = kDOUBLE if isinstance(value, float) else kBIGINT
        n = _Node(EXPR_CONSTANT, sql_type, True, is_null=is_null, scale=scale)
        if sql_type == kDOUBLE:
            n.dval = float(value)
        elif sql_type == kFLOAT:   # a FLOAT Datum: the literal rounded to float precision (Datum.floatval)
            n.dval = float(np.float32(value))
        else:
            n.ival = int(value)
        self.nodes.append(n)
        return len(self.nodes) - 1

    def binop(self, op: int, left: int, right: int) -> int:
        self.nodes.append(_Node(EXPR_BIN_OPER, kTINYINT, False, op=op, left=left, right=right))
        return len(self.nodes) - 1

    def uoper(self, op: int, operand: int) -> int:
        """Analyzer::UOper: kNOT over a boolean expression, kISNULL over a ColumnVar (IS NOT NULL = NOT(ISNULL))."""
        self.nodes.append(_Node(EXPR_UOPER, kBOOLEAN, op == kISNULL, op=op, left=operand))
        return len(self.nodes) - 1

    def cmp(self, col_id: int, op: int, value, const_type: Optional[int] = None, rte_idx: int = 0, scale: int = 0) -> int:
        return self.binop(op, self.col(col_id, rte_idx), self.const(value, const_type, scale=scale))

    def agg(self, kind: int, col_id: Optional[int] = None, bigint_count: bool = False, rte_idx: int = 0,
            is_distinct: bool = False) -> int:
        """AggExpr.  Result type as RelAlgTranslator assigns it: COUNT -> INT/BIGINT notnull... SUM(int) -> BIGINT,
        MIN/MAX -> arg type, AVG -> DOUBLE."""
        arg = -1
        scale = 0
        if col_id is None:
            assert kind == kCOUNT
            ti = (kBIGINT if bigint_count else kINT, False)
        else:
            arg = self.col(col_id, rte_idx)
            at, ann = (self.inner if rte_idx else self.table).col_types[col_id]
            if rte_idx and self.join_type == 1:
                ann = False
            if kind == kCOUNT:
                ti = (kBIGINT if bigint_count else kINT, False)
            elif kind == kSUM:
                ti = (at if at in DECIMAL_TYPES or at in (kDOUBLE, kFLOAT) else kBIGINT, ann)   # SUM(DECIMAL) keeps type and scale; SUM(FLOAT) is FLOAT
                scale = self.nodes[arg].scale
            elif kind == kAVG:
                ti = (kDOUBLE, ann)
            else:
                ti = (at, ann)
                scale = self.nodes[arg].scale
        self.nodes.append(_Node(EXPR_AGG, ti[0], ti[1], op=kind, left=arg, ival=int(is_distinct), scale=scale))   # ival: AggExpr::get_is_distinct()
        return len(self.nodes) - 1

    # -- unit lists ---------------------------------------------------------------------------------------
    def add_qual(self, e: int, simple: bool = False):
        (self.simple_quals if simple else self.quals).append(e)
        return self

    def group_by(self, col_id: int, rte_idx: int = 0):
        self.groupby.append(self.col(col_id, rte_idx))
        return self

    def target(self, e: int):
        self.targets.append(e)
        return self

    def target_col(self, col_id: int, rte_idx: int = 0):
        return self.target(self.col(col_id, rte_idx))

    def estimator(self, cols: Sequence, large: bool = False):
        """RelAlgExecutionUnit::createNdvExecutionUnit: estimator = [Large]NDVEstimator over the GROUP BY tuple; the unit
        keeps its quals (and join level) but has no groupby_exprs and no targets.  cols: column ids or (id, rte_idx)."""
        self.estimator_kind = 2 if large else 1
        self.estimator_args = [self.col(*c) if isinstance(c, tuple) else self.col(c) for c in cols]
        return self

    def order_by(self, tle_no: int, is_desc: bool = False, nulls_first: Optional[bool] = None):
        """sort_info.order_entries.  Default NULL placement is the reference's (NULLs are the largest values:
        last when ascending, first when descending — RelAlgTranslator / Calcite's default collation)."""
        self.order.append((tle_no, bool(is_desc), bool(is_desc) if nulls_first is None else bool(nulls_first)))
        return self

    def build(self) -> "BuiltUnit":
        return BuiltUnit(self)


class BuiltUnit:
    """Owns the ctypes arrays an ExecUnit points into."""

    def __init__(self, b: UnitBuilder):
        n = len(b.nodes)
        self.exprs = (Expr * max(n, 1))()
        for i, nd in enumerate(b.nodes):
            e = self.exprs[i]
            e.kind = nd.kind
            e.ti = TypeInfo(nd.type, int(nd.notnull), nd.scale)
            e.col_id, e.op, e.left, e.right = nd.col_id, nd.op, nd.left, nd.right
            e.ival, e.dval, e.is_null, e.rte_idx = nd.ival, nd.dval, int(nd.is_null), nd.rte_idx

        def arr(xs):
            return (C.c_int32 * max(len(xs), 1))(*xs)

        self._sq, self._q, self._g, self._t = arr(b.simple_quals), arr(b.quals), arr(b.groupby), arr(b.targets)
        u = ExecUnit()
        u.exprs, u.num_exprs = self.exprs, n
        u.simple_quals, u.num_simple_quals = self._sq, len(b.simple_quals)
        u.quals, u.num_quals = self._q, len(b.quals)
        u.groupby_exprs, u.num_groupby_exprs = self._g, len(b.groupby)
        u.target_exprs, u.num_target_exprs = self._t, len(b.targets)
        u.scan_limit = b.scan_limit
        self._order = (OrderEntry * max(len(b.order), 1))()
        for i, (tle, desc, nf) in enumerate(b.order):
            self._order[i].tle_no, self._order[i].is_desc, self._order[i].nulls_first = tle, int(desc), int(nf)
        u.order_entries, u.num_order_entries = self._order, len(b.order)
        u.has_limit, u.limit, u.offset = int(b.limit is not None), int(b.limit or 0), int(b.offset)
        self._est = arr(b.estimator_args)
        u.has_estimator, u.estimator_args, u.num_estimator_args = b.estimator_kind, self._est, len(b.estimator_args)
        u.join_qual = -1
        self.inner = b.inner
        if b.inner is not None:
            assert len(b.inner.fragments) <= 1, "the inner table must be one concatenated fragment"
            self._inner_built = b.inner.build(CPU_LEVEL)     # host chunks; the library copies what it needs
            u.num_join_quals, u.join_qual, u.join_type = 1, b.join_qual, b.join_type
            u.inner_table = C.cast(C.pointer(self._inner_built.info), C.c_void_p)
        for k, v in b.unsupported.items():
            setattr(u, k, v)
        self.unit = u


def chunk_stats(arr: np.ndarray, sql_type: int, notnull: bool, null=None) -> ChunkStats:
    """ChunkMetadata::chunkStats as the reference's encoders maintain them: min/max over NON-NULL values (NaN ignored),
    has_nulls when a NULL sentinel is present (DataMgr/Encoder.h; FixedLengthEncoder::updateStats)."""
    st = ChunkStats()
    null = NULL_OF[sql_type] if null is None else null
    if arr.size == 0:
        st.int_min, st.int_max = 2**63 - 1, -(2**63)
        st.fp_min, st.fp_max = float(np.finfo(np.float64).max), float(np.finfo(np.float64).min)
        return st
    if notnull:
        vals = arr
        st.has_nulls = 0
    else:
        mask = arr != null
        vals = arr[mask]
        st.has_nulls = int(vals.size != arr.size)
    if sql_type in (kDOUBLE, kFLOAT):
        vals = vals[~np.isnan(vals)]   # std::min(dataMin, NaN) keeps dataMin: the encoder never records a NaN
        if vals.size:
            st.fp_min, st.fp_max = float(vals.min()), float(vals.max())
        else:
            st.fp_min, st.fp_max = float(np.finfo(np.float64).max), float(np.finfo(np.float64).min)
    else:
        if vals.size:
            st.int_min, st.int_max = int(vals.min()), int(vals.max())
        else:
            st.int_min, st.int_max = 2**63 - 1, -(2**63)
    return st


@dataclass
class Fragment:
    """One fragment: per-column either a host ndarray or a raw device pointer (int) + explicit stats."""
    num_tuples: int
    host_cols: List[Optional[np.ndarray]] = field(default_factory=list)
    dev_ptrs: List[int] = field(default_factory=list)
    stats: List[ChunkStats] = field(default_factory=list)
    fragment_id: int = 0
    device_id: int = 0
    remote: bool = False   # lives on another device / rank: only its chunk stats are passed (col_buffers = NULL)


class Table:
    """InputTableInfo mirror: column types + fragments (Fragmenter::FragmentInfo + chunk pointers + chunk stats)."""

    def __init__(self, col_types: Sequence[tuple], encoded_sizes: Optional[Sequence[int]] = None,
                 deleted_column: Optional[int] = None, col_scales: Optional[Dict[int, int]] = None):
        # col_types: [(sql_type, notnull), ...]; encoded_sizes[c] = physical bytes of an `ENCODING FIXED` column (0 = none),
        # or -4 / -2 for a DATE column under `ENCODING DAYS(32|16)` (kENCODING_DATE_IN_DAYS: the chunk holds days)
        self.col_types = [(int(t), bool(nn)) for t, nn in col_types]
        self.encoded_sizes = [int(x) for x in encoded_sizes] if encoded_sizes is not None else [0] * len(self.col_types)
        self.deleted_column = deleted_column
        self.col_scales: Dict[int, int] = dict(col_scales or {})   # DECIMAL / NUMERIC columns: column index -> scale
        self.fragments: List[Fragment] = []

    def physical_dtype(self, c: int):
        """numpy dtype of the chunk elements of column c (narrower than the logical type under ENCODING FIXED)."""
        enc = self.encoded_sizes[c]
        if enc < 0:                                        # DATE ENCODING DAYS(32|16)
            return {4: np.int32, 2: np.int16}[-enc]
        if enc and self.col_types[c][0] in STRING_TYPES:   # DICT(8) / DICT(16): unsigned ids (ColumnIR.cpp:59-67)
            return {1: np.uint8, 2: np.uint16, 4: np.int32}[enc]
        if enc:
            return {1: np.int8, 2: np.int16, 4: np.int32}[enc]
        return NUMPY_OF[self.col_types[c][0]]

    def physical_null(self, c: int):
        enc = self.encoded_sizes[c]
        if enc < 0:
            return -(2 ** (8 * -enc - 1))
        if enc in (1, 2) and self.col_types[c][0] in STRING_TYPES:   # inline_fixed_encoding_null_val: the unsigned maximum
            return 2 ** (8 * enc) - 1
        if enc:
            return -(2 ** (8 * enc - 1))
        return NULL_OF[self.col_types[c][0]]

    @property
    def num_cols(self):
        return len(self.col_types)

    def add_host_fragment(self, cols: Sequence[Optional[np.ndarray]], fragment_id: Optional[int] = None):
        n = None
        fixed = []
        stats = []
        for c, ((t, nn), a) in enumerate(zip(self.col_types, cols)):
            if a is None:
                fixed.append(None)
                stats.append(ChunkStats())
                continue
            a = np.ascontiguousarray(a, dtype=self.physical_dtype(c))
            n = a.size if n is None else n
            assert a.size == n, "ragged fragment"
            fixed.append(a)
            if self.encoded_sizes[c] < 0:
                # DateDaysEncoder (DataMgr/DateDaysEncoder.h:246-254): the physical minimum is NULL whatever the column's
                # nullability, min / max are kept in epoch SECONDS
                st = chunk_stats(a, t, False, null=self.physical_null(c))
                if st.int_min <= st.int_max:
                    st.int_min, st.int_max = st.int_min * 86400, st.int_max * 86400
                stats.append(st)
                continue
            stats.append(chunk_stats(a, t, nn, null=self.physical_null(c)))
        fid = len(self.fragments) if fragment_id is None else fragment_id
        self.fragments.append(Fragment(n or 0, host_cols=fixed, stats=stats, fragment_id=fid))
        return self

    def add_device_fragment(self, num_tuples: int, dev_ptrs: Sequence[int], stats: Sequence[ChunkStats],
                            fragment_id: Optional[int] = None, device_id: int = 0):
        fid = len(self.fragments) if fragment_id is None else fragment_id
        self.fragments.append(Fragment(int(num_tuples), dev_ptrs=[int(p) for p in dev_ptrs], stats=list(stats),
                                       fragment_id=fid, device_id=device_id))
        return self

    def add_remote_fragment(self, num_tuples: int, stats: Sequence[ChunkStats], fragment_id: int, device_id: int = 0):
        """A fragment that another device / rank scans: it contributes its chunk statistics to planning (so that every
        device derives the same key ranges and the partial tables are position-aligned) and nothing else."""
        self.fragments.append(Fragment(int(num_tuples), stats=list(stats), fragment_id=fragment_id, device_id=device_id,
                                       remote=True))
        return self

    def total_tuples(self):
        return sum(f.num_tuples for f in self.fragments)

    def build(self, memory_level: int) -> "BuiltTable":
        return BuiltTable(self, memory_level)


class BuiltTable:
    """Owns the ctypes arrays a TableInfo points into."""

    def __init__(self, t: Table, memory_level: int):
        self.src = t
        nc = t.num_cols
        self.col_types = (TypeInfo * nc)(*[TypeInfo(ty, int(nn), t.col_scales.get(c, 0)) for c, (ty, nn) in enumerate(t.col_types)])
        nf = len(t.fragments)
        self.frags = (FragmentInfo * max(nf, 1))()
        self._keep = []
        for i, f in enumerate(t.fragments):
            bufs = (C.c_void_p * nc)()
            for c in range(nc):
                if memory_level == CPU_LEVEL:
                    a = f.host_cols[c] if f.host_cols else None
                    bufs[c] = a.ctypes.data if a is not None and a.size else None
                else:
                    bufs[c] = f.dev_ptrs[c] if f.dev_ptrs and f.dev_ptrs[c] else None
            stats = (ChunkStats * nc)(*f.stats)
            self._keep += [bufs, stats]
            fi = self.frags[i]
            fi.fragment_id, fi.device_id, fi.num_tuples = f.fragment_id, f.device_id, f.num_tuples
            fi.col_buffers, fi.col_stats = (None if f.remote else bufs), stats
        ti = TableInfo()
        ti.num_cols, ti.col_types = nc, self.col_types
        ti.num_fragments, ti.fragments = nf, self.frags
        ti.memory_level = memory_level
        ti.deleted_column_plus1 = 0 if t.deleted_column is None else t.deleted_column + 1
        if any(t.encoded_sizes):
            self.enc = (C.c_int8 * nc)(*t.encoded_sizes)
            ti.col_encoded_sizes = self.enc
        self.info = ti
