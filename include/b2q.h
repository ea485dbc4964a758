/*
 * b2q.h — C ABI of the H100-native scan -> filter -> hash-group-by/aggregate path.
 *
 * This is the drop-in boundary for ONE path of a HeavyDB-style engine: everything that runs below
 *     ResultSetPtr Executor::executeWorkUnit(size_t& max_groups_buffer_entry_guess, const bool is_agg,
 *         const std::vector<InputTableInfo>&, const RelAlgExecutionUnit&, const CompilationOptions&,
 *         const ExecutionOptions&, RenderInfo*, const bool has_cardinality_estimation, ColumnCacheMap&)
 *     (reference: QueryEngine/Execute.h:719-727, QueryEngine/Execute.cpp:2144)
 * for single-table filter + optional GROUP BY + COUNT/SUM/MIN/MAX/AVG.
 *
 * Two levels, both plain C (pointers + sizes, no C++/torch types):
 *
 *   outer  b2q_execute_work_unit()   — POD mirror of executeWorkUnit(); plans, launches, merges, materialises.
 *          b2q_execute_partial() / b2q_partial_*() / b2q_partial_finalize() — the same, split at the point
 *          where the reference merges per-device results on the host (Execute.cpp:1696,1772-1792) so the
 *          caller can run the NCCL all-reduce of the dense partial tables between the two halves.
 *          b2q_rs_*()                — the ResultSet output surface (QueryEngine/ResultSet.h:183-330).
 *
 *   inner  b2q_launch()              — the static-kernel replacement of the JIT'd
 *          multifrag_query_hoisted_literals(...) entry (QueryEngine/RuntimeFunctions.cpp:2434-2449); takes the
 *          same 15-slot parameter block (enum KernelParam, QueryEngine/enums.h:64-79) plus the restated
 *          QueryMemoryDescriptor (B2QPlan) that the JIT would have baked into the code.
 *
 * Enum VALUES below are the reference's own (Shared/sqltypes.h:65-99, Shared/sqldefs.h:31-40,76-90,
 * QueryEngine/enums.h:27-60) so that a reference-side binding is a cast, not a translation table.
 *
 * Everything outside the supported subset is REJECTED with B2Q_ERR_UNSUPPORTED — never silently ignored,
 * and there is no CPU fallback: without a CUDA device every compute entry returns B2Q_ERR_NO_DEVICE.
 */
#ifndef B2Q_H
#define B2Q_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2Q_ABI_VERSION 8 /* 2: sort_info, join level, rte_idx, columnar, dictionary / time types, B2QPlan join fields;
                            3: DATE_IN_DAYS chunks (negative col_encoded_sizes), column-vs-column quals, 16 filter leaves,
                               operands-before-node rule, b2q_columnar_results_*, host-phase stats;
                            4: DECIMAL / NUMERIC columns (B2QTypeInfo.scale), decimal_to_double of b2q_rs_get_next_row;
                            5: b2q_comm_* / b2q_execute_work_unit_dist / _multi (merge of the per-device tables inside the
                               library, NCCL), B2Q_KERNEL_BASELINE_PROBE, LIMIT 0 = empty result, COUNT(DISTINCT) on bitmaps
                               (B2QPlan.count_distinct_*);
                            6: B2QExecutionOptions.result_on_device (was pad_), B2QDeviceColumns / b2q_rs_device_columns /
                               b2q_device_columns_* (ColumnarResults in device memory, Arrow C Device export, b2q_arrow.h),
                               B2Q_STAT_RESULT_D2H_BYTES;
                            7: projection units (B2Q_Projection: column targets, no GROUP BY, B2QExecUnit.scan_limit),
                               B2Q_STAT_ROWS_SCANNED, TOTAL_MATCHED / MAX_MATCHED of b2q_launch;
                            8: B2Q_STAT_JOIN_TABLE (B2Q_JOIN_TABLE_*), b2q_last_launch_stat */

/* ---- SQLTypes subset (Shared/sqltypes.h:65-99) -------------------------------------------------------- */
enum {
  B2Q_kBOOLEAN = 1, /* only as the type of the deleted-rows column (B2QTableInfo.deleted_column_plus1) */
  /* dictionary-encoded strings (kENCODING_DICT only): the chunk holds int32 ids, or uint8 / uint16 ids for
   * `TEXT ENCODING DICT(8|16)` (col_encoded_sizes = 1 | 2, FixedWidthUnsigned decode, NULL = 255 / 65535,
   * ColumnIR.cpp:59-67, InlineNullValues.h:173-182).  Usable as GROUP BY keys, projected keys, COUNT arguments and
   * in `=` / `<>` against an id constant; results carry ids (getNextRow with translate_strings = false). */
  B2Q_kCHAR = 2,
  B2Q_kVARCHAR = 3,
  /* NUMERIC / DECIMAL(p, s): the chunk holds value x 10^s as int64, or int32 / int16 under the ENCODING FIXED the DDL
   * picks for p <= 9 / p <= 4 (col_encoded_sizes = 4 | 2); an integer to everything on the path (keys, quals against a
   * constant / column of the SAME scale, COUNT / SUM / MIN / MAX / AVG); the scale is applied at read-out only
   * (makeTargetValue ResultSetIteration.cpp:2193-2210, pair_to_double ResultSetBufferAccessors.h:222-225) */
  B2Q_kNUMERIC = 4,
  B2Q_kDECIMAL = 5,
  B2Q_kINT = 6,
  B2Q_kSMALLINT = 7,
  B2Q_kFLOAT = 8,
  B2Q_kDOUBLE = 9,
  /* TIME / TIMESTAMP / DATE: int64 (optionally ENCODING FIXED(32)); keys, COUNT / MIN / MAX arguments, comparisons */
  B2Q_kTIME = 10,
  B2Q_kTIMESTAMP = 11,
  B2Q_kBIGINT = 12,
  B2Q_kTEXT = 13,
  B2Q_kDATE = 14,
  B2Q_kTINYINT = 22
};

/* ---- SQLOps subset (Shared/sqldefs.h:31-40) ----------------------------------------------------------- */
enum { B2Q_kEQ = 0, B2Q_kNE = 2, B2Q_kLT = 3, B2Q_kGT = 4, B2Q_kLE = 5, B2Q_kGE = 6, B2Q_kAND = 7, B2Q_kOR = 8,
       B2Q_kNOT = 9, B2Q_kISNULL = 16 /* Analyzer::UOper: NOT <bool expr>, <ColumnVar> IS NULL; IS NOT NULL = NOT(ISNULL) */ };

/* ---- SQLAgg subset (Shared/sqldefs.h:76-90) ----------------------------------------------------------- */
enum { B2Q_kAVG = 0, B2Q_kMIN = 1, B2Q_kMAX = 2, B2Q_kSUM = 3, B2Q_kCOUNT = 4 };

/* ---- QueryDescriptionType (QueryEngine/enums.h:54-60) ------------------------------------------------- */
enum {
  B2Q_GroupByPerfectHash = 0,
  B2Q_GroupByBaselineHash = 1,
  B2Q_Projection = 2,
  B2Q_TableFunction = 3,
  B2Q_NonGroupedAggregate = 4,
  B2Q_Estimator = 5
};

/* ---- error codes ----------------------------------------------------------------------------------------
 * 0..18 are heavyai::ErrorCode (QueryEngine/enums.h:27-47); a NEGATIVE return from the inner entry is the
 * reference's "-pos" out-of-slots convention (GroupByAndAggregate.cpp:1149-1154).  Codes >= 1000 mirror the
 * C++ exceptions that cross the reference's outer boundary (SURVEY §8b "errors"). */
enum {
  B2Q_OK = 0,
  B2Q_ERR_DIV_BY_ZERO = 1,
  B2Q_ERR_OUT_OF_GPU_MEM = 2,
  B2Q_ERR_OUT_OF_SLOTS = 3,
  B2Q_ERR_OVERFLOW_OR_UNDERFLOW = 7,
  B2Q_ERR_OUT_OF_TIME = 8,
  B2Q_ERR_INTERRUPTED = 9,
  B2Q_ERR_UNSUPPORTED = 1000,                      /* feature outside the path (joins, sort, window, ...) */
  B2Q_ERR_CARDINALITY_ESTIMATION_REQUIRED = 1001,  /* CardinalityEstimationRequired (NativeCodegen.cpp:2972-2979) */
  B2Q_ERR_INVALID_ARGUMENT = 1002,
  B2Q_ERR_NO_DEVICE = 1003,                        /* no CUDA device: there is no CPU fallback */
  B2Q_ERR_CUDA = 1004,
  B2Q_ERR_KEY_OUT_OF_RANGE = 1005                  /* a key outside the chunk-stats range (stale metadata) */
};

/* ---- SQLTypeInfo subset -------------------------------------------------------------------------------- */
typedef struct B2QTypeInfo {
  int32_t type;    /* B2Q_k* SQLTypes value */
  int32_t notnull; /* SQLTypeInfo::get_notnull() */
  int32_t scale;   /* SQLTypeInfo::get_scale(): digits after the point of a DECIMAL / NUMERIC (0 for every other type).  The dimension of a
                      TIMESTAMP is NOT carried: only TIMESTAMP(0) columns belong on this path (the reference plans high-precision
                      timestamp keys differently, GroupByAndAggregate.cpp:288-298) */
} B2QTypeInfo;

/* ---- Analyzer::Expr subset (Analyzer/Analyzer.h:193 ColumnVar, :319 Constant, :434 BinOper, :1381 AggExpr)
 * Nodes live in one flat array in construction order; children are indices of EARLIER nodes (-1 = none) — anything
 * else is B2Q_ERR_INVALID_ARGUMENT. */
enum { B2Q_EXPR_COLUMN_VAR = 1, B2Q_EXPR_CONSTANT = 2, B2Q_EXPR_BIN_OPER = 3, B2Q_EXPR_AGG = 4,
       B2Q_EXPR_UOPER = 5 /* Analyzer::UOper with op in {kNOT, kISNULL}; operand = left */ };

typedef struct B2QExpr {
  int32_t kind;   /* B2Q_EXPR_* */
  B2QTypeInfo ti; /* Expr::get_type_info() */
  int32_t col_id; /* ColumnVar: column index in B2QTableInfo */
  int32_t op;     /* BinOper: SQLOps; AggExpr: SQLAgg */
  int32_t left;   /* BinOper: left operand; AggExpr: argument (-1 = COUNT(*)) */
  int32_t right;  /* BinOper: right operand */
  int64_t ival;   /* Constant: Datum for integer types (a string literal against a dictionary column: its id in THAT column's
                     dictionary, StringDictionaryProxy::getIdOfString; -1 = not in the dictionary); AggExpr: get_is_distinct() */
  double dval;    /* Constant: Datum for fp types */
  int32_t is_null;/* Constant::get_is_null() */
  int32_t rte_idx;/* ColumnVar::get_rte_idx(): 0 = the scanned (outer) table, 1 = the joined inner table */
} B2QExpr;
/* Dictionary-encoded strings are compared BY ID (= and <> only).  B2QTypeInfo does not carry the dictionary key, so a
 * `ColumnVar OP ColumnVar` over two string columns is the caller's promise that both use ONE dictionary
 * (SQLTypeInfo::getStringDictKey() equal — the id-compare branch of CodeGenerator::codegenCmp); columns of different dictionaries
 * need the reference's string comparison and must not be routed here. */

/* ---- Analyzer::OrderEntry (Analyzer/Analyzer.h:2960-2968) ------------------------------------------------ */
typedef struct B2QOrderEntry {
  int32_t tle_no;      /* target list entry number, 1-based */
  int8_t is_desc;
  int8_t nulls_first;
  int8_t pad_[2];
} B2QOrderEntry;

/* ---- RelAlgExecutionUnit subset (QueryEngine/RelAlgExecutionUnit.h:166-216) ---------------------------- */
struct B2QTableInfo;
typedef struct B2QExecUnit {
  const B2QExpr* exprs;
  int32_t num_exprs;
  const int32_t* simple_quals; /* expr indices; "col OP const" comparisons (narrow the key range, a21) */
  int32_t num_simple_quals;
  const int32_t* quals;        /* expr indices; AND-ed together */
  int32_t num_quals;
  const int32_t* groupby_exprs;/* expr indices; num_groupby_exprs == 0 <=> reference's {nullptr} */
  int32_t num_groupby_exprs;
  const int32_t* target_exprs; /* expr indices */
  int32_t num_target_exprs;
  /* Projection units (no groupby_exprs, every target a ColumnVar, no aggregate): the output holds at most scan_limit rows,
   * the first passing rows in (fragment, row) order — what RelAlgExecutor sets for LIMIT without ORDER BY (limit + offset,
   * get_scan_limit, RelAlgExecutor.cpp:3442-3449).  0 = no limit: the library counts the passing rows first (the non-grouped
   * COUNT(*) scan over the same quals) and sizes the output from that count. */
  int64_t scan_limit;
  /* join_quals (JoinQualsPerNestingLevel, RelAlgExecutionUnit.h:166-216): at most ONE nesting level, INNER or LEFT,
   * whose only qual is `ColumnVar(rte 0) = ColumnVar(rte 1)` over integer columns and for which the reference would
   * build a one-to-one PerfectJoinHashTable (JoinHashTable/PerfectJoinHashTable.cpp:168-300; probe
   * hash_join_idx[_nullable], GroupByRuntime.cpp:283-311).  LEFT: an outer row without a match continues with every
   * inner column NULL (codegenOuterJoinNullPlaceholder, ColumnIR.cpp:504-560); the unit's inner ColumnVars must then
   * be nullable, as RelAlgTranslator makes them.  Anything else (one-to-many, baseline join tables, more levels) is
   * rejected. */
  int32_t num_join_quals;      /* 0 or 1 */
  /* estimator (RelAlgExecutionUnit::createNdvExecutionUnit, CardinalityEstimator.cpp:94-116): 0 = none, 1 =
   * Analyzer::NDVEstimator (1 MiB bitmap), 2 = LargeNDVEstimator (256 MiB).  The unit then has no groupby_exprs and
   * no target_exprs; every row that passes the quals hashes the tuple `estimator_args` (each widened to int64, NULLs
   * as their sentinel) with MurmurHash3 and sets one bit (linear_probabilistic_count, RuntimeFunctions.cpp:2399-2408,
   * codegenEstimator GroupByAndAggregate.cpp:1825-1864).  b2q_rs_get_ndv_estimator() is ResultSet::getNDVEstimator. */
  int32_t has_estimator;
  int32_t has_union_all;
  int32_t has_window_function;
  /* sort_info (SortInfo, RelAlgExecutionUnit.h:117-156).  When any of it is set the returned ResultSet is what
   * RelAlgExecutor::executeSort makes of executeWorkUnit's result (RelAlgExecutor.cpp:3586-3610):
   * rs->sort(order_entries, limit + offset); rs->dropFirstN(offset); rs->keepFirstN(limit) — done on the device
   * over the aggregated table (compaction of non-empty entries, radix sort, gather), so only the kept rows are
   * copied back.  Ties keep ascending entry order (the reference's std::sort leaves them unspecified). */
  const B2QOrderEntry* order_entries;
  int32_t num_order_entries;
  int32_t has_limit;           /* std::optional<size_t> limit */
  int64_t limit;
  int64_t offset;
  /* the join level (used when num_join_quals == 1) */
  int32_t join_qual;           /* expr index of the equi-join BinOper(kEQ, ColumnVar, ColumnVar) */
  int32_t join_type;           /* JoinType (Shared/sqldefs.h:252): INNER = 0 or LEFT = 1 */
  /* input_descs[1]: the inner table the way the hash-join column fetch sees it — every column as ONE buffer over all
   * fragments (ColumnFetcher::getAllTableColumnFragments, ColumnFetcher.cpp:290-360), i.e. exactly one fragment whose
   * chunk stats cover the table; memory_level CPU (copied to the device per query) or GPU */
  const struct B2QTableInfo* inner_table;
  const int32_t* estimator_args; /* expr indices of the estimator's argument tuple (ColumnVars) */
  int32_t num_estimator_args;
  int32_t pad_;
} B2QExecUnit;

/* ---- ChunkMetadata::chunkStats per (fragment, column)  (Fragmenter/Fragmenter.h:73-146) ---------------- */
typedef struct B2QChunkStats {
  int64_t int_min, int_max; /* integer columns */
  double fp_min, fp_max;    /* fp columns */
  int32_t has_nulls;
  int32_t pad_;
} B2QChunkStats;

/* ---- Fragmenter::FragmentInfo + the column pointers ColumnFetcher would return (ColumnFetcher.cpp:214) - */
typedef struct B2QFragmentInfo {
  int32_t fragment_id;
  int32_t device_id;                /* reference rule: fragment_id % num_devices (InsertOrderFragmenter.cpp:435) */
  int64_t num_tuples;
  const void* const* col_buffers;   /* [num_cols]; flat fixed-width arrays; NULL for unreferenced columns.  The whole
                                       pointer may be NULL for a fragment that ANOTHER device scans: it then only
                                       contributes its chunk stats to planning, so that every device of a multi-GPU
                                       query derives the same key ranges (the reference plans once for all devices) */
  const B2QChunkStats* col_stats;   /* [num_cols] */
} B2QFragmentInfo;

/* ---- InputTableInfo (QueryEngine/InputMetadata.h:32-35) ------------------------------------------------ */
enum { B2Q_CPU_LEVEL = 1, B2Q_GPU_LEVEL = 2 }; /* Data_Namespace::MemoryLevel values */
typedef struct B2QTableInfo {
  int32_t num_cols;
  const B2QTypeInfo* col_types;     /* [num_cols] */
  int32_t num_fragments;
  const B2QFragmentInfo* fragments; /* [num_fragments] */
  int32_t memory_level;             /* where col_buffers live: B2Q_GPU_LEVEL (HBM resident) or B2Q_CPU_LEVEL
                                       (host; copied H2D inside the call, chunk by chunk) */
  int32_t deleted_column_plus1;     /* 1 + id of the table's BOOLEAN $deleted$ column, 0 = none.  Rows whose flag is
                                       true are skipped before any qual (Executor::addDeletedColumn Execute.cpp:4593,
                                       codegenSkipDeletedOuterTableRow NativeCodegen.cpp:3419-3451) */
  const int8_t* col_encoded_sizes;  /* [num_cols] or NULL.  Byte width of the PHYSICAL chunk element when the column is
                                       declared `ENCODING FIXED(bits)` (kENCODING_FIXED): 1, 2 or 4 for an integer
                                       column of a wider logical type; 0 = not encoded.  NULL is stored as the minimum
                                       of the physical width and decodes to the logical type's sentinel
                                       (CodeGenerator::codgenAdjustFixedEncNull, ColumnIR.cpp:456-500).
                                       NEGATIVE = kENCODING_DATE_IN_DAYS (the default encoding of DATE columns): -4 / -2
                                       for `DATE ENCODING DAYS(32|16)`; the chunk holds int32 / int16 days since the
                                       epoch, the physical minimum is NULL, values decode as days * 86400
                                       (FixedWidthSmallDate, ColumnIR.cpp:73-81, DecodersImpl.h:138-146) and the chunk
                                       stats are in epoch seconds (DateDaysEncoder.h:246-254) */
} B2QTableInfo;

/* ---- CompilationOptions / ExecutionOptions subsets (QueryEngine/CompilationOptions.h:31-66,70-122) ----- */
enum { B2Q_DEVICE_CPU = 0, B2Q_DEVICE_GPU = 1 }; /* ExecutorDeviceType */
typedef struct B2QCompilationOptions {
  int32_t device_type;    /* must be B2Q_DEVICE_GPU: no CPU fallback */
  int32_t hoist_literals; /* accepted, meaningless for static kernels */
  int32_t ignore_deleted_column; /* == !CompilationOptions::filter_on_deleted_column (default 0: deleted rows are skipped) */
  int32_t pad_;
} B2QCompilationOptions;

typedef struct B2QExecutionOptions {
  int32_t allow_multifrag;       /* one launch over all fragments of this device (Execute.cpp:3075-3101) */
  int32_t output_columnar_hint;  /* --enable-columnar-output */
  int32_t bigint_count;          /* g_bigint_count (--bigint-count) */
  int32_t force_kernel;          /* 0 = planner's choice; else B2Q_KERNEL_* (for tests / benchmarks) */
  int32_t device_ordinal;        /* CUDA device to run on (-1 = current); the calling thread's current device is restored on return */
  /* 1: the materialised result stays in device memory (no device-to-host copy inside the call); the host copy is made on the
   * first host accessor of the result set (row_count, get_next_row, storage_buffer, columnar_results_create, ...), and
   * b2q_rs_device_columns reads the device copy directly.  0 = copy the result to the host before returning.  Planning is
   * the same either way; estimator results always come back to the host. */
  int32_t result_on_device;
} B2QExecutionOptions;

/* static kernel families (one per C symbol b2q_k_*) */
enum {
  B2Q_KERNEL_AUTO = 0,
  B2Q_KERNEL_NON_GROUPED = 1,     /* register accumulators + warp/block reduce            */
  B2Q_KERNEL_PERFECT_SMEM = 2,    /* per-CTA private table in shared memory               */
  B2Q_KERNEL_PERFECT_GLOBAL = 3,  /* one dense table in HBM/L2, global reductions          */
  B2Q_KERNEL_BASELINE_GLOBAL = 4, /* open-addressing table in HBM (MurmurHash3, linear probe): built by the radix-partitioned
                                     aggregation (partition by home-slot range, aggregate each slice in shared memory) when the
                                     query's shape allows, else row by row with the reference's probe */
  B2Q_KERNEL_BASELINE_PROBE = 5   /* force_kernel only: baseline hash with the per-row probe kernel (plan.kernel stays 4) */
};

/* =========================================================================================================
 * Restated QueryMemoryDescriptor (QueryEngine/Descriptors/QueryMemoryDescriptor.h:69) — what the planner
 * decided.  Filled by b2q_plan(); consumed by b2q_launch() and by the result-set accessors.
 * ======================================================================================================= */
#define B2Q_MAX_SLOTS 16
#define B2Q_MAX_TARGETS 16
#define B2Q_MAX_FILTER_TERMS 16 /* comparison / IS NULL leaves of all quals together (an IN list is one leaf per value) */
#define B2Q_MAX_GROUP_COLS 4

typedef struct B2QTargetInfo { /* Shared/TargetInfo.h:49-78 */
  int32_t is_agg;
  int32_t agg_kind;        /* SQLAgg */
  B2QTypeInfo sql_type;
  B2QTypeInfo agg_arg_type;/* type = 0 (kNULLT) when there is no argument */
  int32_t skip_null_val;
  int32_t is_distinct;     /* always 0 here */
  int32_t arg_col_id;      /* -1 when no argument */
  int32_t first_slot;      /* slot index of this target (AVG owns first_slot and first_slot+1) */
} B2QTargetInfo;

typedef struct B2QPlan {
  int32_t query_desc_type;   /* QueryDescriptionType */
  int32_t keyless_hash;
  int32_t idx_target_as_key; /* slot index whose value != init marks a non-empty keyless entry */
  int32_t output_columnar;
  int32_t interleaved_bins_on_gpu; /* reported for parity; our kernels never interleave */
  int32_t group_col_width;   /* byte width of the GROUP BY column */
  int32_t effective_key_width;/* 8 for perfect hash; 4 or 8 for baseline */
  int32_t num_targets;
  int32_t num_slots;
  int32_t key_col_id;
  int64_t entry_count;
  int64_t min_val, max_val, bucket;
  int32_t has_nulls;
  int32_t kernel;            /* B2Q_KERNEL_* chosen */
  int64_t row_size;          /* bytes, row-wise */
  int64_t buffer_size;       /* bytes of the whole result buffer */
  /* multi-column perfect hash (GroupByAndAggregate.cpp:232-280, codegenPerfectHashFunction :1549-1597):
   * entry = sum_i (key_i - min_i) * prod_{j<i} cardinality_j; min_val = 0, max_val = the cardinality product */
  int32_t num_group_cols;
  int32_t group_col_ids[B2Q_MAX_GROUP_COLS];
  int8_t group_col_widths[B2Q_MAX_GROUP_COLS];
  int32_t pad2_;
  int8_t slot_padded_width[B2Q_MAX_SLOTS];
  int8_t slot_logical_width[B2Q_MAX_SLOTS];
  int64_t slot_offset[B2Q_MAX_SLOTS]; /* row-wise: byte offset inside the row; columnar: offset of the column */
  int64_t init_vals[B2Q_MAX_SLOTS];   /* init_agg_val_vec (OutputBufferInitialization.cpp:26-86) */
  B2QTargetInfo targets[B2Q_MAX_TARGETS];
  /* the join level, if any: a one-to-one perfect hash table over [join_min_key, join_max_key] of the inner key
   * (PerfectJoinHashTable: hash_entry_count = max - min + 1, slots = inner row index or -1).  With a join, column ids
   * in this descriptor (key_col_id, group_col_ids, targets[].arg_col_id) >= the outer table's num_cols denote inner
   * table column (id - num_cols). */
  int64_t join_min_key, join_max_key, join_entry_count;
  int32_t join_outer_col, join_inner_col; /* -1 without a join */
  /* COUNT(DISTINCT c) targets — CountDistinctDescriptor with CountDistinctImplType::Bitmap (init_count_distinct_descriptors,
   * GroupByAndAggregate.cpp:650-855): one bitmap of count_distinct_bits[t] bits per group, bit 0 = count_distinct_min[t];
   * 0 bits = target t is not a distinct aggregate.  The reference keeps a POINTER to the group's bitmap in the target's slot
   * and counts its bits when the value is read (count_distinct_set_size, ResultSetIteration.cpp:2178); here the bitmaps stay
   * in HBM and the slot of the returned buffer holds the set size itself.  Descriptors the reference would serve with a
   * std::set (fp argument, range too wide) cannot run on its GPU either (QueryMustRunOnCpu): B2Q_ERR_UNSUPPORTED. */
  int64_t count_distinct_min[B2Q_MAX_TARGETS];
  int64_t count_distinct_bits[B2Q_MAX_TARGETS];
} B2QPlan;

/* The 15-slot kernel parameter block of the reference's JIT entry (enums.h:64-79), device pointers. */
typedef struct B2QParams {
  int32_t* error_codes;            /* ERROR_CODE      */
  int32_t* total_matched;          /* TOTAL_MATCHED   projection: receives the rows written (may be NULL) */
  int64_t** group_by_buffers;      /* GROUPBY_BUF     — [0] = the output buffer in reference layout */
  const uint32_t* num_fragments;   /* NUM_FRAGMENTS   (host pointer, read on the host)   */
  const uint32_t* num_tables;      /* NUM_TABLES      (must point at 1) */
  const uint32_t* row_index_resume;/* ROW_INDEX_RESUME (unused) */
  const int8_t*** col_buffers;     /* COL_BUFFERS     host array [frag][col] of DEVICE pointers */
  const int8_t* literals;          /* LITERALS        (unused: literals live in the plan) */
  const int64_t* num_rows;         /* NUM_ROWS        host array [frag] */
  const uint64_t* frag_row_offsets;/* FRAG_ROW_OFFSETS (unused) */
  const int32_t* frag_ids;         /* FRAG_IDS        (unused) */
  const int32_t* max_matched;      /* MAX_MATCHED     (host pointer; projection: the output's capacity in rows, NULL = the plan's
                                      entry_count; unused otherwise) */
  const int64_t* init_agg_value;   /* INIT_AGG_VALS   host array [num_slots]; NULL = plan->init_vals */
  const int64_t* join_hash_tables; /* JOIN_HASH_TABLES NULL, or [0] = device address of the int32 one-to-one table
                                      (what HashJoin::getJoinHashBuffer returns) when the plan has a join level */
  const int8_t* row_func_mgr;      /* ROW_FUNC_MGR    must be NULL */
} B2QParams;

typedef struct B2QQuery B2QQuery;         /* plan + compiled filter/aggregate program (opaque) */
typedef struct B2QPartial B2QPartial;     /* per-device dense partial-aggregate table in HBM (opaque) */
typedef struct B2QResultSet B2QResultSet; /* ResultSet output surface (opaque) */

/* ---- library ------------------------------------------------------------------------------------------- */
int32_t b2q_abi_version(void);
const char* b2q_error_string(int32_t code);
const char* b2q_last_error_message(void); /* thread-local detail for the last failing call */
int32_t b2q_device_count(void);           /* 0 when no CUDA device is visible */

/* ---- planning (host only; usable without a GPU) --------------------------------------------------------- */
/* Restates GroupByAndAggregate::initQueryMemoryDescriptor + QueryMemoryDescriptor::init.
 * max_groups_buffer_entry_guess / has_cardinality_estimation have executeWorkUnit()'s meaning. */
int32_t b2q_plan(const B2QExecUnit* ra_exe_unit, const B2QTableInfo* query_info,
                 const B2QCompilationOptions* co, const B2QExecutionOptions* eo,
                 size_t max_groups_buffer_entry_guess, int32_t has_cardinality_estimation, B2QQuery** out);
const B2QPlan* b2q_query_plan(const B2QQuery* q);
void b2q_query_free(B2QQuery* q);

/* ---- outer entry: Executor::executeWorkUnit --------------------------------------------------------------
 * Same parameter order as the reference (RenderInfo* and ColumnCacheMap& have no meaning here and are
 * dropped).  *max_groups_buffer_entry_guess is in/out like the reference's size_t&. */
int32_t b2q_execute_work_unit(size_t* max_groups_buffer_entry_guess, int32_t is_agg,
                              const B2QTableInfo* query_infos, const B2QExecUnit* ra_exe_unit,
                              const B2QCompilationOptions* co, const B2QExecutionOptions* eo,
                              int32_t has_cardinality_estimation, B2QResultSet** out);

/* ---- split form for multi-GPU: [scan+aggregate] -> (caller's NCCL all-reduce) -> [materialise] ----------- */
int32_t b2q_execute_partial(size_t* max_groups_buffer_entry_guess, int32_t is_agg,
                            const B2QTableInfo* query_infos, const B2QExecUnit* ra_exe_unit,
                            const B2QCompilationOptions* co, const B2QExecutionOptions* eo,
                            int32_t has_cardinality_estimation, void* cuda_stream, B2QPartial** out);
/* Dense per-slot arrays of the partial table.  Every array is position-aligned across devices (perfect-hash /
 * non-grouped layouts), initialised to the identity of its reduction, so the merge of N devices is exactly
 * one all-reduce per array — the device-side replacement of ResultSetStorage::reduce
 * (ResultSetReduction.cpp:203-396, slot op :1496-1566). */
enum { B2Q_DT_INT64 = 0, B2Q_DT_FLOAT64 = 1, B2Q_DT_UINT8 = 2 /* "group touched" flags, merged with MAX */ };
enum { B2Q_RED_SUM = 0, B2Q_RED_MIN = 1, B2Q_RED_MAX = 2,
       B2Q_RED_BOR = 3 /* bitwise OR: the estimator bitmap (reduce_estimator_results, CardinalityEstimator.cpp:142-161);
                          NCCL has no OR — all-gather + OR, see heavydb_b200/multigpu.py */ };
int32_t b2q_partial_num_arrays(const B2QPartial* p);
int32_t b2q_partial_array(const B2QPartial* p, int32_t i, void** device_ptr, int64_t* count, int32_t* dtype,
                          int32_t* redop);
int32_t b2q_partial_is_mergeable(const B2QPartial* p); /* 0 for baseline-hash (not position aligned) */
const B2QPlan* b2q_partial_plan(const B2QPartial* p);
double b2q_partial_kernel_ms(const B2QPartial* p);     /* CUDA-event time of the scan kernel(s) */
int32_t b2q_partial_finalize(B2QPartial* p, void* cuda_stream, B2QResultSet** out);
void b2q_partial_free(B2QPartial* p);

/* ---- multi-GPU with the merge inside the library ---------------------------------------------------------
 * The reference runs ONE process with one host thread per device (Executor::launchKernelsViaResourceMgr,
 * Execute.cpp:3055-3101; ExecutionKernel::run, ExecutionKernel.cpp:215-218) and reduces the per-device result sets on the
 * HOST (Executor::reduceMultiDeviceResults, Execute.cpp:1696,1772-1792 -> ResultSetStorage::reduce).  Here each device's
 * scan is followed, on the same CUDA stream and without a host synchronisation, by NCCL collectives over NVLink that
 * merge the tables in HBM: dense (perfect-hash / non-grouped) tables by ONE all-reduce per reduction class — COUNT and
 * integer SUM arrays are adjacent, so configs[1] is a single 160 KB all-reduce —, baseline-hash tables by an all-gather of
 * the peers' key / accumulator arrays and a device-side re-probe (ResultSetReduction.cpp:698-828), estimator bitmaps by
 * all-gather + OR.  libnccl.so.2 is bound at run time; without it these entries return B2Q_ERR_UNSUPPORTED.
 *
 *   b2q_comm_init_all     ncclCommInitAll: all devices driven by this process (b2q_execute_work_unit_multi)
 *   b2q_comm_init_rank    ncclCommInitRank: one process per device (torchrun & co.); the 128-byte id comes from
 *                         b2q_comm_unique_id on rank 0 and travels by whatever the host already has
 *   ..._dist              this rank's share: `query_infos` = its own fragments plus the other ranks' fragments as chunk
 *                         stats only (col_buffers == NULL), so that every rank plans the same layout; every rank gets the
 *                         merged ResultSet
 *   ..._multi             one call, one host thread per device, tables[i] = what device comms[i] scans; the ResultSet
 *                         is materialised by comms[0]'s device */
#define B2Q_COMM_ID_BYTES 128
typedef struct B2QComm B2QComm;
int32_t b2q_comm_unique_id(void* id128);
int32_t b2q_comm_init_rank(const void* id128, int32_t nranks, int32_t rank, int32_t device_ordinal, B2QComm** out);
int32_t b2q_comm_init_all(const int32_t* devices, int32_t ndev, B2QComm** out /* [ndev] */);
void b2q_comm_destroy(B2QComm* comm);
int32_t b2q_comm_rank(const B2QComm* comm);
int32_t b2q_comm_size(const B2QComm* comm);
int32_t b2q_execute_work_unit_dist(B2QComm* comm, size_t* max_groups_buffer_entry_guess, int32_t is_agg,
                                   const B2QTableInfo* query_infos, const B2QExecUnit* ra_exe_unit,
                                   const B2QCompilationOptions* co, const B2QExecutionOptions* eo,
                                   int32_t has_cardinality_estimation, void* cuda_stream, B2QResultSet** out);
int32_t b2q_execute_work_unit_multi(B2QComm* const* comms, int32_t ndev, size_t* max_groups_buffer_entry_guess, int32_t is_agg,
                                    const B2QTableInfo* const* query_infos_per_device, const B2QExecUnit* ra_exe_unit,
                                    const B2QCompilationOptions* co, const B2QExecutionOptions* eo,
                                    int32_t has_cardinality_estimation, B2QResultSet** out);

/* ---- inner entry: the static-kernel replacement of multifrag_query_hoisted_literals ---------------------- */
int32_t b2q_launch(const B2QQuery* query, const B2QParams* params, void* cuda_stream);

/* ---- ResultSet surface (QueryEngine/ResultSet.h) --------------------------------------------------------- */
typedef struct B2QTargetValue { /* ScalarTargetValue for the numeric subset (QueryEngine/TargetValue.h) */
  int32_t is_fp;   /* 0: ival holds int64_t, 1: dval holds double (FLOAT targets are widened like getNextRow) */
  int32_t is_null; /* value equals the type's NULL sentinel (Shared/InlineNullValues.h:30-36) */
  int64_t ival;
  double dval;
} B2QTargetValue;

size_t b2q_rs_row_count(const B2QResultSet* rs);   /* ResultSet::rowCount()  :306 */
size_t b2q_rs_col_count(const B2QResultSet* rs);   /* ResultSet::colCount() */
size_t b2q_rs_entry_count(const B2QResultSet* rs); /* ResultSet::entryCount() */
int32_t b2q_rs_is_empty(const B2QResultSet* rs);   /* ResultSet::isEmpty() */
B2QTypeInfo b2q_rs_get_col_type(const B2QResultSet* rs, size_t col_idx); /* ResultSet::getColType() */
/* ResultSet::getNextRow(translate_strings, decimal_to_double) :259 — returns 1 and fills row[colCount()],
 * or 0 at the end.  Dictionary strings always come back as ids (translate_strings is accepted and ignored); a DECIMAL
 * target is a double (value / 10^scale, NULL_DOUBLE for NULL) under decimal_to_double, else the scaled int64.
 * b2q_rs_move_to_begin() == ResultSet::moveToBegin(). */
int32_t b2q_rs_get_next_row(B2QResultSet* rs, B2QTargetValue* row, int32_t translate_strings, int32_t decimal_to_double);
/* ResultSet::getRowAt(logical_index) / getRowAtNoTranslations(logical_index) (ResultSet.h:259-270, ResultSetIteration.cpp:266-284):
 * random access by entry (through the permutation of a sorted set); returns 1 and fills `row`, 0 for an empty entry or an index
 * past b2q_rs_entry_count().  Independent of the getNextRow cursor. */
int32_t b2q_rs_get_row_at(const B2QResultSet* rs, size_t logical_index, B2QTargetValue* row, int32_t translate_strings,
                          int32_t decimal_to_double);

/* ColumnarResults (QueryEngine/ColumnarResults.h:60-232, .cpp:256-392): the rows of a result set, in iteration order
 * (ResultSet::sort permutation, OFFSET, LIMIT applied), as one contiguous array per target in the target type's own
 * width (COUNT int32 / int64, SUM(int) int64, AVG double, keys at their column type); NULLs keep the type's inline
 * sentinel.  This is what ColumnFetcher hands to the next step and what ArrowResultSetConverter reads; host code in
 * the reference too.  `num_threads` conversion threads (is_parallel_execution_enforced). */
typedef struct B2QColumnarResults B2QColumnarResults;
int32_t b2q_columnar_results_create(const B2QResultSet* rs, int32_t num_threads, B2QColumnarResults** out);
size_t b2q_columnar_results_size(const B2QColumnarResults* cr);                                  /* ColumnarResults::size() */
size_t b2q_columnar_results_num_columns(const B2QColumnarResults* cr);
const int8_t* b2q_columnar_results_column(const B2QColumnarResults* cr, size_t col, B2QTypeInfo* ti); /* getColumnBuffers()[col], getColumnType(col) */
void b2q_columnar_results_free(B2QColumnarResults* cr);
void b2q_rs_move_to_begin(B2QResultSet* rs);
int32_t b2q_rs_is_row_at_empty(const B2QResultSet* rs, size_t entry_idx); /* ResultSet::isRowAtEmpty() */
/* getStorage()->getUnderlyingBuffer(): host copy of the output buffer in the reference's own row-wise /
 * columnar layout (ResultSet.h:55-84, QueryMemoryDescriptor.cpp:848-955). */
const int8_t* b2q_rs_storage_buffer(const B2QResultSet* rs, size_t* size_bytes);
const B2QPlan* b2q_rs_query_mem_desc(const B2QResultSet* rs); /* getQueryMemDesc() */
double b2q_rs_kernel_ms(const B2QResultSet* rs);
/* ResultSet::sort(order_entries, top_n) (ResultSet.h:279, ResultSet.cpp:781-849) followed by iteration in sorted
 * order; top_n == 0 sorts everything.  dropFirstN / keepFirstN are SQL OFFSET / LIMIT (ResultSet.cpp:58-66).
 * The sort runs on the device (sort.cu); ties keep ascending entry order.  FLOAT targets order by the float's value,
 * AVG as pair_to_double (DECIMAL scale included); a dictionary-encoded string target is refused with B2Q_ERR_UNSUPPORTED
 * (the reference orders it by string, through the dictionary). */
/* ResultSet::getNDVEstimator (CardinalityEstimator.cpp:33-52) of an estimator query: -total_bits * ln(unset/total),
 * 1 for an empty bitmap, 0 when every bit is set; b2q_rs_estimator_buffer = getHostEstimatorBuffer(). */
size_t b2q_rs_get_ndv_estimator(const B2QResultSet* rs);
const int8_t* b2q_rs_estimator_buffer(const B2QResultSet* rs, size_t* size_bytes);
int32_t b2q_rs_sort(B2QResultSet* rs, const B2QOrderEntry* order_entries, int32_t num_order_entries, size_t top_n);
void b2q_rs_drop_first_n(B2QResultSet* rs, size_t n);
void b2q_rs_keep_first_n(B2QResultSet* rs, size_t n);
/* execution statistics of the call that produced the result set */
enum { B2Q_STAT_FRAGMENTS_SCANNED = 0, B2Q_STAT_FRAGMENTS_SKIPPED = 1 /* Executor::skipFragment, Execute.cpp:4776 */,
       B2Q_STAT_KERNEL_LAUNCHES = 2, B2Q_STAT_H2D_BYTES = 3, B2Q_STAT_SORT_US = 4 /* device time of compaction + sort + gather */,
       /* host wall-clock of the CPU_LEVEL streaming scan: staging setup, copy+scan pipeline, teardown */
       B2Q_STAT_HOST_SETUP_US = 5, B2Q_STAT_HOST_STREAM_US = 6, B2Q_STAT_HOST_TEARDOWN_US = 7,
       B2Q_STAT_RESULT_D2H_BYTES = 8 /* result-storage bytes copied device -> host so far (0 for a result_on_device set no host
                                        accessor has read yet) */,
       B2Q_STAT_ROWS_SCANNED = 9 /* projection: rows of the chunks the projection kernel loaded (a scan limit stops it early);
                                    0 for every other query */,
       B2Q_STAT_JOIN_TABLE = 10 /* the one-to-one join table the scan probed: a B2Q_JOIN_TABLE_* value */ };
/* Layouts of the join table.  The planner picks one from the inner key's range E = join_entry_count and the inner columns
 * the query reads: staged into shared memory when it fits beside the group table (the group table's replicas give way
 * first), else probed in HBM / L2.  {row, value} slots carry the first 1/2/4-byte integer inner column the query reads;
 * uint16 slots hold only that column's value - its chunk-stats minimum (0xFFFE = NULL, 0xFFFF = no row) and are chosen
 * when it is the only inner column read, its chunk-stats span is below 65534 and the {row, value} table does not fit.
 * The uint16 layout trusts the inner column's chunk stats: a value outside them fails the query with
 * B2Q_ERR_KEY_OUT_OF_RANGE, where the other layouts would have read it. */
enum { B2Q_JOIN_TABLE_NONE = 0, B2Q_JOIN_TABLE_CALLER = 1 /* b2q_launch: the caller's int32 table, read in place */,
       B2Q_JOIN_TABLE_INT32_HBM = 2, B2Q_JOIN_TABLE_INT2_HBM = 3, B2Q_JOIN_TABLE_INT32_SMEM = 4, B2Q_JOIN_TABLE_INT2_SMEM = 5,
       B2Q_JOIN_TABLE_UINT16_SMEM = 6 };
int64_t b2q_rs_stat(const B2QResultSet* rs, int32_t which);
/* statistics of the calling thread's last successful b2q_launch (it returns no result set): B2Q_STAT_JOIN_TABLE; -1 for
 * every other statistic */
int64_t b2q_last_launch_stat(int32_t which);
void b2q_rs_free(B2QResultSet* rs);
/* ResultSet(targets, device_type, query_mem_desc, ...) + allocateStorage(buffer) (ResultSet.h:183-217): a result set over a
 * group-by buffer the caller already holds, laid out as the planned query's descriptor says (b2q_plan); the bytes are
 * copied.  Read-out only (rowCount / getNextRow / isRowAtEmpty / ColumnarResults) — nothing is computed and no device is
 * needed, the way ResultSetTest wraps hand-filled storage. */
int32_t b2q_rs_create_from_storage(const B2QQuery* q, const int8_t* storage, size_t size_bytes, B2QResultSet** out);

/* ---- ColumnarResults in device memory ------------------------------------------------------------------------
 * b2q_rs_device_columns converts a result set, on `cuda_stream` of the result's device, into exactly what
 * b2q_columnar_results_create produces on the host: the same rows in iteration order (permutation, OFFSET, LIMIT applied),
 * one array per target in the target type's width, NULLs as the inline sentinel.  A result_on_device set is read where it
 * lies (no device-to-host copy); a host-resident one is uploaded first.  Each column also gets an Arrow validity bitmap
 * (bit set = valid, LSB first, one bit per row) and its NULL count; a column without NULLs reports validity = NULL and
 * null_count = 0.  Returns once the columns are complete.  Without a CUDA device: B2Q_ERR_NO_DEVICE.
 *
 * b2q_device_columns_export_arrow fills an Arrow C Device Data Interface record batch (b2q_arrow.h): a "+s" struct with
 * one child per target, formats c/s/i/l/f/g (dictionary ids i, TIME-family l) and d:19,<scale> for DECIMAL (a decimal128
 * buffer made on the device), device_type ARROW_DEVICE_CUDA, device_id = the result's device, sync_event -> a cudaEvent_t
 * recorded after the conversion.  `names` may be NULL ("col<i>").  The buffers stay alive until both
 * b2q_device_columns_free and the exported array's release have run; whichever runs last frees them stream-ordered
 * (b2q_device_columns_free on its `cuda_stream`; release on the legacy default stream after the conversion's event, i.e.
 * after work the consumer enqueued on any blocking stream of that device). */
typedef struct B2QDeviceColumns B2QDeviceColumns;
struct ArrowSchema;
struct ArrowDeviceArray;
int32_t b2q_rs_device_columns(const B2QResultSet* rs, void* cuda_stream, B2QDeviceColumns** out);
size_t b2q_device_columns_size(const B2QDeviceColumns* dc);        /* rows */
size_t b2q_device_columns_num_columns(const B2QDeviceColumns* dc);
int32_t b2q_device_columns_device(const B2QDeviceColumns* dc);     /* CUDA device ordinal of the buffers */
double b2q_device_columns_convert_ms(const B2QDeviceColumns* dc);  /* CUDA-event time of the conversion kernel */
/* device pointer of column `col`'s values (NULL for an index out of range); *validity = its bitmap or NULL */
const void* b2q_device_columns_column(const B2QDeviceColumns* dc, size_t col, B2QTypeInfo* type_info, const uint32_t** validity,
                                      int64_t* null_count);
int32_t b2q_device_columns_export_arrow(B2QDeviceColumns* dc, const char* const* names, struct ArrowSchema* schema,
                                        struct ArrowDeviceArray* array);
void b2q_device_columns_free(B2QDeviceColumns* dc, void* cuda_stream);

/* ---- synthetic data (bench / tests): counter-based generator, identical to oracle/oracle_gen.h ----------
 * value(row) = lo + splitmix64(seed ^ (col_tag << 56) ^ row) % span   (integers)
 *            = (splitmix64(...) >> 11) * 2^-53                        (doubles in [0,1))
 * Writes `count` elements of `width` bytes starting at global row `row0` into a DEVICE buffer. */
int32_t b2q_gen_column(void* device_dst, int32_t sql_type, uint64_t seed, uint32_t col_tag, int64_t row0,
                       int64_t count, int64_t lo, int64_t span, void* cuda_stream);
/* BIGINT only: value = lo + (u % span) * stride — sparse keys (range too wide for a perfect hash => baseline hash) */
int32_t b2q_gen_column_strided(void* device_dst, int32_t sql_type, uint64_t seed, uint32_t col_tag, int64_t row0,
                               int64_t count, int64_t lo, int64_t span, int64_t stride, void* cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* B2Q_H */
