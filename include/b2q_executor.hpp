/*
 * b2q_executor.hpp — C++ host-side mirror of the reference's operator interface for this path, header-only, over the
 * C ABI of b2q.h.  Names, argument order and error behaviour follow the reference so that a test written against
 * it reads like Tests/GroupByTest.cpp:73-152 (which builds a RelAlgExecutionUnit by hand and calls
 * executor->executeWorkUnit(...) directly):
 *
 *   Executor::executeWorkUnit(size_t& max_groups_buffer_entry_guess, const bool is_agg,
 *                             const std::vector<InputTableInfo>&, const RelAlgExecutionUnit&,
 *                             const CompilationOptions&, const ExecutionOptions&, RenderInfo*,
 *                             const bool has_cardinality_estimation, ColumnCacheMap&)      (Execute.h:719-727)
 *   ResultSet::rowCount / colCount / getColType / getNextRow / isEmpty / entryCount       (ResultSet.h:183-330)
 *   exceptions: QueryExecutionError(code), CardinalityEstimationRequired, QueryNotSupported
 *
 * Only marshalling happens here; all computation is in libb2q (CUDA).  Link with -lb2q.
 */
#pragma once
#include <cstdint>
#include <list>
#include <map>
#include <mutex>
#include <optional>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "b2q.h"
#include "b2q_arrow.h"

namespace b2q {

/* ---- SQLTypeInfo / enums: the reference's own values ---- */
enum SQLTypes { kBOOLEAN = B2Q_kBOOLEAN /* the $deleted$ column only */, kCHAR = B2Q_kCHAR, kVARCHAR = B2Q_kVARCHAR, kNUMERIC = B2Q_kNUMERIC, kDECIMAL = B2Q_kDECIMAL, kINT = B2Q_kINT, kSMALLINT = B2Q_kSMALLINT, kDOUBLE = B2Q_kDOUBLE,
                kTIME = B2Q_kTIME, kTIMESTAMP = B2Q_kTIMESTAMP, kBIGINT = B2Q_kBIGINT, kTEXT = B2Q_kTEXT /* dictionary-encoded */,
                kDATE = B2Q_kDATE, kTINYINT = B2Q_kTINYINT };
enum SQLOps { kEQ = B2Q_kEQ, kNE = B2Q_kNE, kLT = B2Q_kLT, kGT = B2Q_kGT, kLE = B2Q_kLE, kGE = B2Q_kGE, kAND = B2Q_kAND, kOR = B2Q_kOR,
              kNOT = B2Q_kNOT, kISNULL = B2Q_kISNULL };
enum SQLAgg { kAVG = B2Q_kAVG, kMIN = B2Q_kMIN, kMAX = B2Q_kMAX, kSUM = B2Q_kSUM, kCOUNT = B2Q_kCOUNT };
enum class ExecutorDeviceType { CPU = B2Q_DEVICE_CPU, GPU = B2Q_DEVICE_GPU };

/* EncodingType (Shared/sqltypes.h:261-273), the values this path can read */
enum EncodingType { kENCODING_NONE = 0, kENCODING_FIXED = 1, kENCODING_DICT = 4, kENCODING_DATE_IN_DAYS = 7 };

struct SQLTypeInfo {
  SQLTypes type{kBIGINT};
  bool notnull{false};
  EncodingType compression{kENCODING_NONE};
  int comp_param{0}; /* bits for kENCODING_FIXED / kENCODING_DATE_IN_DAYS / DICT(8|16); the dictionary id otherwise */
  int dimension{0};  /* precision of a DECIMAL / NUMERIC (informational on this path) */
  int scale{0};      /* digits after the point of a DECIMAL / NUMERIC */
  SQLTypeInfo() = default;
  SQLTypeInfo(SQLTypes t, int d, int s, bool nn) : type(t), notnull(nn), dimension(d), scale(s) {} /* SQLTypeInfo(kDECIMAL, 10, 4, false) */
  SQLTypeInfo(SQLTypes t, bool nn) : type(t), notnull(nn) {}
  SQLTypeInfo(SQLTypes t, bool nn, EncodingType c, int p) : type(t), notnull(nn), compression(c), comp_param(p) {}
  SQLTypes get_type() const { return type; }
  bool get_notnull() const { return notnull; }
  int get_dimension() const { return dimension; }
  int get_scale() const { return scale; }
  bool is_decimal() const { return type == kDECIMAL || type == kNUMERIC; }
  B2QTypeInfo pod() const { return B2QTypeInfo{type, notnull ? 1 : 0, scale}; }
  EncodingType get_compression() const { return compression; }
  int get_comp_param() const { return comp_param; }
  /* B2QTableInfo.col_encoded_sizes entry: physical bytes under FIXED / DICT(8|16), minus the bytes under
   * DATE_IN_DAYS (comp_param 0 means 32 there, as in SQLTypeInfo::get_size), 0 when the chunk has the logical width */
  int8_t encoded_size() const {
    if (compression == kENCODING_FIXED) return static_cast<int8_t>(comp_param / 8);
    if (compression == kENCODING_DATE_IN_DAYS) return static_cast<int8_t>(comp_param == 16 ? -2 : -4);
    if (compression == kENCODING_DICT && (comp_param == 8 || comp_param == 16)) return static_cast<int8_t>(comp_param / 8);
    return 0;
  }
};

/* ---- exceptions that cross the reference's boundary ---- */
struct QueryExecutionError : std::runtime_error { /* ExecutionKernel.cpp:133-160 */
  int32_t code;
  QueryExecutionError(int32_t c, const std::string& m) : std::runtime_error(m), code(c) {}
  int32_t getErrorCode() const { return code; }
};
struct CardinalityEstimationRequired : QueryExecutionError { using QueryExecutionError::QueryExecutionError; };
struct QueryNotSupported : QueryExecutionError { using QueryExecutionError::QueryExecutionError; };

/* ---- Analyzer:: expression subset; nodes are owned by the RelAlgExecutionUnit they are built into ---- */
using ExprRef = int32_t;

struct RelAlgExecutionUnit { /* RelAlgExecutionUnit.h:166-216 */
  std::vector<B2QExpr> exprs;
  std::list<ExprRef> simple_quals;
  std::list<ExprRef> quals;
  std::list<ExprRef> groupby_exprs; /* empty == the reference's {nullptr} (non-grouped) */
  std::vector<ExprRef> target_exprs;
  size_t scan_limit{0};
  /* join_quals (JoinQualsPerNestingLevel): at most one INNER level whose only qual is outer.col = inner.col */
  enum class JoinType { INNER = 0, LEFT = 1 };
  struct JoinCondition { std::list<ExprRef> quals; JoinType type{JoinType::INNER}; };
  std::vector<JoinCondition> join_quals;
  /* ra_exe_unit.estimator (Analyzer::NDVEstimator / LargeNDVEstimator over the GROUP BY tuple,
   * RelAlgExecutionUnit::createNdvExecutionUnit, CardinalityEstimator.cpp:94-116): such a unit has no groupby_exprs,
   * no targets and no sort_info; the result answers ResultSet::getNDVEstimator() */
  struct NDVEstimator { std::list<ExprRef> expr_tuple; bool large{false}; };
  std::optional<NDVEstimator> estimator;
  /* features outside this path: anything non-zero is rejected by the library */
  int32_t has_union_all{0}, has_window_function{0};
  /* SortInfo (RelAlgExecutionUnit.h:117-156); Analyzer::OrderEntry == B2QOrderEntry{tle_no, is_desc, nulls_first} */
  struct SortInfo {
    std::list<B2QOrderEntry> order_entries;
    std::optional<size_t> limit;
    size_t offset{0};
  } sort_info;

  ExprRef makeColumnVar(const SQLTypeInfo& ti, int32_t column_id, int32_t rte_idx = 0) { /* Analyzer::ColumnVar(ti, column_key, rte_idx) */
    B2QExpr e{};
    e.kind = B2Q_EXPR_COLUMN_VAR; e.ti = ti.pod(); e.col_id = column_id; e.left = e.right = -1; e.rte_idx = rte_idx;
    exprs.push_back(e);
    return static_cast<ExprRef>(exprs.size() - 1);
  }
  ExprRef makeConstant(int64_t v) {
    B2QExpr e{};
    e.kind = B2Q_EXPR_CONSTANT; e.ti = {B2Q_kBIGINT, 1}; e.ival = v; e.left = e.right = -1;
    exprs.push_back(e);
    return static_cast<ExprRef>(exprs.size() - 1);
  }
  ExprRef makeConstant(const SQLTypeInfo& ti, int64_t v) { /* Analyzer::Constant(ti, false, Datum) of an integer / time type */
    B2QExpr e{};
    e.kind = B2Q_EXPR_CONSTANT; e.ti = ti.pod(); e.ival = v; /* DECIMAL: Datum.bigintval = value x 10^scale */ e.left = e.right = -1;
    exprs.push_back(e);
    return static_cast<ExprRef>(exprs.size() - 1);
  }
  ExprRef makeUOper(SQLOps op, ExprRef operand) { /* Analyzer::UOper(kBOOLEAN, kNOT | kISNULL, operand) */
    B2QExpr e{};
    e.kind = B2Q_EXPR_UOPER; e.ti = {B2Q_kBOOLEAN, 0}; e.op = op; e.left = operand; e.right = -1;
    exprs.push_back(e);
    return static_cast<ExprRef>(exprs.size() - 1);
  }
  ExprRef makeConstant(double v) {
    B2QExpr e{};
    e.kind = B2Q_EXPR_CONSTANT; e.ti = {B2Q_kDOUBLE, 1}; e.dval = v; e.left = e.right = -1;
    exprs.push_back(e);
    return static_cast<ExprRef>(exprs.size() - 1);
  }
  ExprRef makeBinOper(SQLOps op, ExprRef l, ExprRef r) { /* Analyzer::BinOper(kBOOLEAN, op, kONE, l, r) */
    B2QExpr e{};
    e.kind = B2Q_EXPR_BIN_OPER; e.ti = {B2Q_kTINYINT, 0}; e.op = op; e.left = l; e.right = r;
    exprs.push_back(e);
    return static_cast<ExprRef>(exprs.size() - 1);
  }
  ExprRef makeAggExpr(const SQLTypeInfo& ti, SQLAgg agg, ExprRef arg /* -1 = COUNT(*) */, bool is_distinct = false) { /* Analyzer::AggExpr(ti, agg, arg, is_distinct, ...) */
    B2QExpr e{};
    e.kind = B2Q_EXPR_AGG; e.ti = ti.pod(); e.op = agg; e.left = arg; e.right = -1; e.ival = is_distinct ? 1 : 0;
    exprs.push_back(e);
    return static_cast<ExprRef>(exprs.size() - 1);
  }
};

/* ---- InputTableInfo: Fragmenter::FragmentInfo + chunk stats + the column pointers ColumnFetcher returns ---- */
struct ChunkStats { int64_t int_min{0}, int_max{-1}; double fp_min{0}, fp_max{-1}; bool has_nulls{false}; };
struct FragmentInfo {
  int fragmentId{0};
  int deviceId{0};
  size_t numTuples{0};
  std::vector<const void*> col_buffers; /* [num_cols] */
  std::vector<ChunkStats> chunkStats;   /* [num_cols] */
};
enum class MemoryLevel { CPU_LEVEL = B2Q_CPU_LEVEL, GPU_LEVEL = B2Q_GPU_LEVEL };
struct InputTableInfo {
  std::vector<SQLTypeInfo> col_types;
  std::vector<FragmentInfo> fragments;
  MemoryLevel memory_level{MemoryLevel::GPU_LEVEL};
  int deleted_column{-1}; /* id of the BOOLEAN $deleted$ column (Executor::addDeletedColumn, Execute.cpp:4593), -1 = none */
};

struct CompilationOptions { /* CompilationOptions.h:31-66 */
  ExecutorDeviceType device_type{ExecutorDeviceType::GPU};
  bool hoist_literals{true};
  bool filter_on_deleted_column{true}; /* false: rows flagged in the $deleted$ column are scanned like any other */
  static CompilationOptions defaults(ExecutorDeviceType dt = ExecutorDeviceType::GPU) { return CompilationOptions{dt, true}; }
};
struct ExecutionOptions { /* CompilationOptions.h:70-122 */
  bool allow_multifrag{true};
  bool output_columnar_hint{false};
  bool bigint_count{false}; /* g_bigint_count */
  bool result_on_device{false}; /* keep the result in device memory (B2QExecutionOptions::result_on_device) */
  bool with_dynamic_watchdog{false};
  unsigned dynamic_watchdog_time_limit{10000}; /* ms (Execute.cpp:87) */
  bool allow_runtime_query_interrupt{false};
  /* the session's token (Executor::interruptToken): what Executor::interrupt(query_session, ...) sets */
  const B2QInterruptToken* interrupt_token{nullptr};
  static ExecutionOptions defaults() { return ExecutionOptions{}; }
};
struct RenderInfo;              /* unused on this path */
struct ColumnCacheMap {};       /* unused on this path */

using TargetValue = B2QTargetValue; /* ScalarTargetValue for the numeric subset */

class ResultSet {
 public:
  explicit ResultSet(B2QResultSet* h) : h_(h) {}
  ~ResultSet() { b2q_rs_free(h_); }
  ResultSet(const ResultSet&) = delete;
  ResultSet& operator=(const ResultSet&) = delete;
  size_t rowCount() const { return b2q_rs_row_count(h_); }
  size_t colCount() const { return b2q_rs_col_count(h_); }
  size_t entryCount() const { return b2q_rs_entry_count(h_); }
  bool isEmpty() const { return b2q_rs_is_empty(h_) != 0; }
  bool definitelyHasNoRows() const { return isEmpty(); }
  SQLTypeInfo getColType(size_t i) const { auto t = b2q_rs_get_col_type(h_, i); SQLTypeInfo r(static_cast<SQLTypes>(t.type), t.notnull != 0); r.scale = t.scale; return r; }
  void moveToBegin() const { b2q_rs_move_to_begin(h_); }
  std::vector<TargetValue> getNextRow(const bool translate_strings, const bool decimal_to_double) const {
    std::vector<TargetValue> row(colCount());
    if (!b2q_rs_get_next_row(h_, row.data(), translate_strings, decimal_to_double)) row.clear();
    return row;
  }
  /* ResultSet::getRowAt(logical_index) / getRowAtNoTranslations (ResultSet.h:259-270): empty vector for an empty entry */
  std::vector<TargetValue> getRowAt(const size_t logical_index) const {
    std::vector<TargetValue> row(colCount());
    if (!b2q_rs_get_row_at(h_, logical_index, row.data(), 1, 0)) row.clear();
    return row;
  }
  std::vector<TargetValue> getRowAtNoTranslations(const size_t logical_index) const {
    std::vector<TargetValue> row(colCount());
    if (!b2q_rs_get_row_at(h_, logical_index, row.data(), 0, 0)) row.clear();
    return row;
  }
  bool isRowAtEmpty(size_t i) const { return b2q_rs_is_row_at_empty(h_, i) != 0; }
  const int8_t* getUnderlyingBuffer(size_t* size_bytes) const { return b2q_rs_storage_buffer(h_, size_bytes); }
  const B2QPlan& getQueryMemDesc() const { return *b2q_rs_query_mem_desc(h_); }
  /* ResultSet::sort(order_entries, top_n, ...) ResultSet.h:279; dropFirstN / keepFirstN ResultSet.cpp:58-66 */
  void sort(const std::list<B2QOrderEntry>& order_entries, size_t top_n) {
    std::vector<B2QOrderEntry> oes(order_entries.begin(), order_entries.end());
    const int32_t rc = b2q_rs_sort(h_, oes.data(), static_cast<int32_t>(oes.size()), top_n);
    if (rc != B2Q_OK) throw QueryExecutionError(rc, b2q_last_error_message());
  }
  size_t getNDVEstimator() const { return b2q_rs_get_ndv_estimator(h_); } /* CardinalityEstimator.cpp:33-52 */
  void dropFirstN(size_t n) { b2q_rs_drop_first_n(h_, n); }
  void keepFirstN(size_t n) { b2q_rs_keep_first_n(h_, n); }
  const B2QResultSet* handle() const { return h_; }
 private:
  B2QResultSet* h_;
};
using ResultSetPtr = std::shared_ptr<ResultSet>;

/* ColumnarResults (QueryEngine/ColumnarResults.h:60-232): ColumnarResults(row_set_mem_owner, rows, num_columns,
 * target_types, executor_id, thread_idx, is_parallel_execution_enforced) — the memory owner, executor id and thread
 * index have no counterpart here; the buffers live as long as this object. */
class ColumnarResults {
 public:
  ColumnarResults(const ResultSet& rows, const size_t num_columns, const std::vector<SQLTypeInfo>& /*target_types*/,
                  const bool is_parallel_execution_enforced = false) {
    const int32_t rc = b2q_columnar_results_create(rows.handle(), is_parallel_execution_enforced ? 8 : 1, &h_);
    if (rc != B2Q_OK) throw QueryExecutionError(rc, b2q_last_error_message());
    if (num_columns != b2q_columnar_results_num_columns(h_)) { b2q_columnar_results_free(h_); throw QueryExecutionError(B2Q_ERR_INVALID_ARGUMENT, "num_columns"); }
    for (size_t c = 0; c < num_columns; ++c) {
      B2QTypeInfo ti;
      column_buffers_.push_back(b2q_columnar_results_column(h_, c, &ti));
      target_types_.emplace_back(static_cast<SQLTypes>(ti.type), ti.notnull != 0);
      target_types_.back().scale = ti.scale;
    }
  }
  ~ColumnarResults() { b2q_columnar_results_free(h_); }
  ColumnarResults(const ColumnarResults&) = delete;
  ColumnarResults& operator=(const ColumnarResults&) = delete;
  const std::vector<const int8_t*>& getColumnBuffers() const { return column_buffers_; }
  size_t size() const { return b2q_columnar_results_size(h_); }
  const SQLTypeInfo& getColumnType(const int col_id) const { return target_types_[col_id]; }
 private:
  B2QColumnarResults* h_{nullptr};
  std::vector<const int8_t*> column_buffers_;
  std::vector<SQLTypeInfo> target_types_;
};

/* The same columns in device memory (b2q_rs_device_columns): what the GPU branch of ArrowResultSetConverter hands over.
 * Column buffers, validity bitmaps (nullptr for a column without NULLs) and NULL counts live as long as this object, or as
 * long as an Arrow export of it that has not been released, whichever is longer. */
class DeviceColumnarResults {
 public:
  explicit DeviceColumnarResults(const ResultSet& rows, void* cuda_stream = nullptr) : stream_(cuda_stream) {
    const int32_t rc = b2q_rs_device_columns(rows.handle(), cuda_stream, &h_);
    if (rc != B2Q_OK) throw QueryExecutionError(rc, b2q_last_error_message());
    const size_t nc = b2q_device_columns_num_columns(h_);
    for (size_t c = 0; c < nc; ++c) {
      B2QTypeInfo ti;
      const uint32_t* valid = nullptr;
      int64_t nulls = 0;
      column_buffers_.push_back(static_cast<const int8_t*>(b2q_device_columns_column(h_, c, &ti, &valid, &nulls)));
      validity_.push_back(valid);
      null_counts_.push_back(nulls);
      target_types_.emplace_back(static_cast<SQLTypes>(ti.type), ti.notnull != 0);
      target_types_.back().scale = ti.scale;
    }
  }
  ~DeviceColumnarResults() { b2q_device_columns_free(h_, stream_); }
  DeviceColumnarResults(const DeviceColumnarResults&) = delete;
  DeviceColumnarResults& operator=(const DeviceColumnarResults&) = delete;
  const std::vector<const int8_t*>& getColumnBuffers() const { return column_buffers_; } /* device pointers */
  const std::vector<const uint32_t*>& getValidityBitmaps() const { return validity_; }
  int64_t nullCount(const int col_id) const { return null_counts_[col_id]; }
  size_t size() const { return b2q_device_columns_size(h_); }
  int deviceId() const { return b2q_device_columns_device(h_); }
  const SQLTypeInfo& getColumnType(const int col_id) const { return target_types_[col_id]; }
  /* synthesize_metadata (InputMetadata.cpp:381-470) of one column, computed by the conversion (b2q_device_columns_chunk_stats) */
  ChunkStats chunkStats(const int col_id) const {
    B2QChunkStats s;
    const int32_t rc = b2q_device_columns_chunk_stats(h_, static_cast<size_t>(col_id), &s);
    if (rc != B2Q_OK) throw QueryExecutionError(rc, b2q_last_error_message());
    return ChunkStats{s.int_min, s.int_max, s.fp_min, s.fp_max, s.has_nulls != 0};
  }
  /* the temporary table the next step reads (getResultSetColumn + synthesize_metadata): one GPU_LEVEL fragment, id 0, on
   * deviceId(), over these columns and their stats.  This object must outlive every call that reads the table. */
  InputTableInfo asTable() const {
    InputTableInfo t;
    t.col_types = target_types_;
    t.memory_level = MemoryLevel::GPU_LEVEL;
    FragmentInfo f;
    f.fragmentId = 0;
    f.deviceId = deviceId();
    f.numTuples = size();
    for (size_t c = 0; c < column_buffers_.size(); ++c) {
      f.col_buffers.push_back(column_buffers_[c]);
      f.chunkStats.push_back(chunkStats(static_cast<int>(c)));
    }
    t.fragments.push_back(std::move(f));
    return t;
  }
  /* Arrow C Device Data Interface record batch; the caller owns both structs and calls their release */
  void exportArrow(const std::vector<std::string>& names, ArrowSchema* schema, ArrowDeviceArray* array) const {
    std::vector<const char*> cn;
    for (const auto& n : names) cn.push_back(n.c_str());
    const int32_t rc = b2q_device_columns_export_arrow(h_, cn.empty() ? nullptr : cn.data(), schema, array);
    if (rc != B2Q_OK) throw QueryExecutionError(rc, b2q_last_error_message());
  }
 private:
  void* stream_;
  B2QDeviceColumns* h_{nullptr};
  std::vector<const int8_t*> column_buffers_;
  std::vector<const uint32_t*> validity_;
  std::vector<int64_t> null_counts_;
  std::vector<SQLTypeInfo> target_types_;
};

class Executor {
 public:
  Executor() = default;
  Executor(const Executor&) = delete;
  Executor& operator=(const Executor&) = delete;
  ~Executor() { for (auto& kv : tokens_) b2q_interrupt_token_destroy(kv.second); }

  /* the runtime-interrupt token of a session (made on first use); a query of the session passes it in
   * ExecutionOptions::interrupt_token together with allow_runtime_query_interrupt */
  const B2QInterruptToken* interruptToken(const std::string& query_session) { return token(query_session); }
  /* Executor::interrupt(query_session, interrupt_session) (GpuInterrupt.cpp:33-160): the session's running (or next) call
   * fails with B2Q_ERR_INTERRUPTED.  A plain store: safe from any thread while the call runs. */
  void interrupt(const std::string& query_session, const std::string& /*interrupt_session*/) { b2q_interrupt(token(query_session)); }
  /* Executor::resetInterrupt (GpuInterrupt.cpp:292-300) */
  void resetInterrupt(const std::string& query_session) { b2q_interrupt_reset(token(query_session)); }

  ResultSetPtr executeWorkUnit(size_t& max_groups_buffer_entry_guess, const bool is_agg,
                               const std::vector<InputTableInfo>& query_infos, const RelAlgExecutionUnit& ra_exe_unit,
                               const CompilationOptions& co, const ExecutionOptions& options, RenderInfo* /*render_info*/,
                               const bool has_cardinality_estimation, ColumnCacheMap& /*column_cache*/) {
    return dispatch(max_groups_buffer_entry_guess, is_agg, query_infos, ra_exe_unit, co, options, has_cardinality_estimation, nullptr, 0);
  }

  /* ResultSet(targets, device_type, query_mem_desc, row_set_mem_owner, ...) + allocateStorage(buffer) (ResultSet.h:183-217):
   * the read-out surface over a group-by buffer the caller already holds, laid out as this unit's descriptor says (the bytes
   * are copied; host only, nothing is computed) */
  ResultSetPtr resultSetFromStorage(const int8_t* storage, const size_t size_bytes, size_t max_groups_buffer_entry_guess,
                                    const std::vector<InputTableInfo>& query_infos, const RelAlgExecutionUnit& ra_exe_unit,
                                    const CompilationOptions& co, const ExecutionOptions& options,
                                    const bool has_cardinality_estimation = false) {
    static const int8_t empty = 0;
    return dispatch(max_groups_buffer_entry_guess, true, query_infos, ra_exe_unit, co, options, has_cardinality_estimation,
                    storage ? storage : &empty, size_bytes);
  }

 private:
  ResultSetPtr dispatch(size_t& max_groups_buffer_entry_guess, const bool is_agg, const std::vector<InputTableInfo>& query_infos,
                        const RelAlgExecutionUnit& ra_exe_unit, const CompilationOptions& co, const ExecutionOptions& options,
                        const bool has_cardinality_estimation, const int8_t* storage, const size_t storage_bytes) {
    const size_t n_tables = 1 + ra_exe_unit.join_quals.size();
    if (query_infos.size() != n_tables || n_tables > 2) throw QueryNotSupported(B2Q_ERR_UNSUPPORTED, "one input table, or two with one join level, on this path");
    /* flatten to the POD structs of the C ABI */
    struct Flat {
      std::vector<B2QTypeInfo> col_types;
      std::vector<int8_t> enc;
      std::vector<std::vector<B2QChunkStats>> stats;
      std::vector<B2QFragmentInfo> frags;
      B2QTableInfo tbl{};
      void fill(const InputTableInfo& ti) {
        bool any_enc = false;
        for (const auto& t : ti.col_types) {
          col_types.push_back(t.pod());
          enc.push_back(t.encoded_size());
          any_enc |= enc.back() != 0;
        }
        const int nc = static_cast<int>(col_types.size());
        stats.resize(ti.fragments.size());
        frags.resize(ti.fragments.size());
        for (size_t f = 0; f < ti.fragments.size(); ++f) {
          const FragmentInfo& fi = ti.fragments[f];
          stats[f].resize(nc);
          for (int c = 0; c < nc; ++c) {
            const ChunkStats& s = fi.chunkStats[c];
            stats[f][c] = B2QChunkStats{s.int_min, s.int_max, s.fp_min, s.fp_max, s.has_nulls ? 1 : 0, 0};
          }
          frags[f] = B2QFragmentInfo{fi.fragmentId, fi.deviceId, static_cast<int64_t>(fi.numTuples), fi.col_buffers.data(), stats[f].data()};
        }
        tbl = B2QTableInfo{nc, col_types.data(), static_cast<int32_t>(frags.size()), frags.data(), static_cast<int32_t>(ti.memory_level), ti.deleted_column + 1, any_enc ? enc.data() : nullptr};
      }
    } outer, inner;
    outer.fill(query_infos.front());
    if (n_tables == 2) inner.fill(query_infos[1]);
    const B2QTableInfo& tbl = outer.tbl;
    std::vector<int32_t> sq(ra_exe_unit.simple_quals.begin(), ra_exe_unit.simple_quals.end());
    std::vector<int32_t> q(ra_exe_unit.quals.begin(), ra_exe_unit.quals.end());
    std::vector<int32_t> g(ra_exe_unit.groupby_exprs.begin(), ra_exe_unit.groupby_exprs.end());
    B2QExecUnit u{};
    u.exprs = ra_exe_unit.exprs.data(); u.num_exprs = static_cast<int32_t>(ra_exe_unit.exprs.size());
    u.simple_quals = sq.data(); u.num_simple_quals = static_cast<int32_t>(sq.size());
    u.quals = q.data(); u.num_quals = static_cast<int32_t>(q.size());
    u.groupby_exprs = g.data(); u.num_groupby_exprs = static_cast<int32_t>(g.size());
    u.target_exprs = ra_exe_unit.target_exprs.data(); u.num_target_exprs = static_cast<int32_t>(ra_exe_unit.target_exprs.size());
    u.scan_limit = static_cast<int64_t>(ra_exe_unit.scan_limit);
    std::vector<int32_t> est;
    if (ra_exe_unit.estimator) {
      est.assign(ra_exe_unit.estimator->expr_tuple.begin(), ra_exe_unit.estimator->expr_tuple.end());
      u.has_estimator = ra_exe_unit.estimator->large ? 2 : 1;
      u.estimator_args = est.data();
      u.num_estimator_args = static_cast<int32_t>(est.size());
    }
    u.num_join_quals = static_cast<int32_t>(ra_exe_unit.join_quals.size());
    u.join_qual = -1;
    if (u.num_join_quals == 1) {
      const auto& jc = ra_exe_unit.join_quals.front();
      if (jc.quals.size() != 1) throw QueryNotSupported(B2Q_ERR_UNSUPPORTED, "exactly one equi-join qual per level on this path");
      u.join_qual = jc.quals.front();
      u.join_type = static_cast<int32_t>(jc.type);
      u.inner_table = &inner.tbl;
    }
    u.has_union_all = ra_exe_unit.has_union_all;
    std::vector<B2QOrderEntry> oes(ra_exe_unit.sort_info.order_entries.begin(), ra_exe_unit.sort_info.order_entries.end());
    u.order_entries = oes.data(); u.num_order_entries = static_cast<int32_t>(oes.size());
    u.has_limit = ra_exe_unit.sort_info.limit.has_value() ? 1 : 0;
    u.limit = static_cast<int64_t>(ra_exe_unit.sort_info.limit.value_or(0));
    u.offset = static_cast<int64_t>(ra_exe_unit.sort_info.offset);
    u.has_window_function = ra_exe_unit.has_window_function;
    B2QCompilationOptions cco{static_cast<int32_t>(co.device_type), co.hoist_literals ? 1 : 0, co.filter_on_deleted_column ? 0 : 1, 0};
    B2QExecutionOptions ceo{options.allow_multifrag ? 1 : 0, options.output_columnar_hint ? 1 : 0, options.bigint_count ? 1 : 0, 0, -1,
                            options.result_on_device ? 1 : 0, options.with_dynamic_watchdog ? 1 : 0, options.dynamic_watchdog_time_limit,
                            options.allow_runtime_query_interrupt ? 1 : 0, 0, options.interrupt_token};
    B2QResultSet* rs = nullptr;
    int32_t rc;
    if (storage) {
      B2QQuery* planned = nullptr;
      rc = b2q_plan(&u, &tbl, &cco, &ceo, max_groups_buffer_entry_guess, has_cardinality_estimation ? 1 : 0, &planned);
      if (rc == B2Q_OK) rc = b2q_rs_create_from_storage(planned, storage, storage_bytes, &rs);
      b2q_query_free(planned);
    } else {
      rc = b2q_execute_work_unit(&max_groups_buffer_entry_guess, is_agg ? 1 : 0, &tbl, &u, &cco, &ceo, has_cardinality_estimation ? 1 : 0, &rs);
    }
    if (rc != B2Q_OK) {
      const std::string msg = std::string(b2q_error_string(rc)) + ": " + b2q_last_error_message();
      if (rc == B2Q_ERR_CARDINALITY_ESTIMATION_REQUIRED) throw CardinalityEstimationRequired(rc, msg);
      if (rc == B2Q_ERR_UNSUPPORTED) throw QueryNotSupported(rc, msg);
      throw QueryExecutionError(rc, msg);
    }
    return std::make_shared<ResultSet>(rs);
  }

  B2QInterruptToken* token(const std::string& session) {
    std::lock_guard<std::mutex> g(tokens_mu_);
    auto it = tokens_.find(session);
    if (it != tokens_.end()) return it->second;
    B2QInterruptToken* t = nullptr;
    const int32_t rc = b2q_interrupt_token_create(&t);
    if (rc != B2Q_OK) throw QueryExecutionError(rc, b2q_last_error_message());
    tokens_.emplace(session, t);
    return t;
  }
  std::mutex tokens_mu_;
  std::map<std::string, B2QInterruptToken*> tokens_;
};

}  // namespace b2q
