/*
 * b2q_internal.h — structures shared by the host planner (planner.cpp), the executor (executor.cpp) and the
 * sm_90a kernels (kernels.cu).  Not part of the ABI.
 *
 * The reference JIT-compiles one row function per query (QueryEngine/NativeCodegen.cpp:2917 compileWorkUnit).
 * Here the query is lowered to a tiny *device program* (DevProgram) that static kernels interpret in a
 * vector-at-a-time fashion: every switch on an operator / width is executed once per R rows per thread and is
 * warp-uniform, so the interpretation overhead is amortised and never diverges.
 */
#pragma once
#include <float.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../include/b2q.h"

#define B2Q_MAX_COLS 16   /* distinct columns a query may reference */
#define B2Q_MAX_TERMS B2Q_MAX_FILTER_TERMS
#define B2Q_MAX_FILTER_OPS 34 /* 16 leaves + 15 connectives (+ the deleted-rows term and its AND) */
#define B2Q_MAX_ACCS 24   /* internal accumulators */
#define B2Q_MAX_FRAGS_INLINE 0

/* ---- filter ---------------------------------------------------------------------------------------------
 * A comparison `col OP literal` is normalised on the host to a closed range test plus flags:
 *     pass = !is_null(v) && (negate ^ (lo <= v && v <= hi))
 * (restates DEF_CMP_NULLABLE, RuntimeFunctions.cpp:73-107: NULL compares to null_bool_val which toBool()
 * (LogicalIR.cpp:344-352) turns into "row fails").  AND/OR trees are evaluated in postfix order on "is TRUE"
 * bits, which is exact for Kleene logic without NOT (logical_and/logical_or, RuntimeFunctions.cpp:320-357). */
struct DevTerm {
  int64_t lo;           /* integer domain: in_range = (unsigned)(v - lo) <= span  (32-bit columns: low words used) */
  uint64_t span;
  double flo, fhi;      /* fp domain, inclusive */
  int64_t null_bits;    /* column NULL sentinel: int value (sign-extended) or double bits */
  int32_t col;          /* index into the launch's column table */
  int8_t width;         /* 1,2,4,8 */
  int8_t col_is_fp;     /* column holds doubles */
  int8_t cmp_fp;        /* compare in the double domain (column or literal is fp) */
  int8_t negate;        /* result = in_range XOR negate */
  int8_t null_check;    /* explicit `v != NULL` needed (the host folds it into the range whenever it can) */
  /* column OP column (col2 >= 0): both sides loaded, compared as int64 or — if either side is fp — as double;
   * TRUE only when neither side is NULL (DEF_CMP_NULLABLE, RuntimeFunctions.cpp:73-107) */
  int8_t width2;
  int8_t col2_is_fp;
  int8_t op2;           /* B2Q_kEQ .. B2Q_kGE */
  int32_t col2;         /* -1: comparison with a constant */
  int8_t nullable1, nullable2;
  /* set term (an IN / NOT IN list past the leaf program): in_range = v in [lo, lo + span] and bit v - lo of set_bits is set,
   * tested on the register-class value like the range test; negate and null_check as above (a NULL row is never TRUE) */
  int8_t is_set;
  int8_t pad_;
  int64_t null_bits2;
  const uint32_t* set_bits; /* device bitmap over [lo, lo + span], built per call from B2QQuery::set_values (executor.cpp) */
};

enum { FOP_TERM = 0, FOP_AND = 1, FOP_OR = 2 };
struct DevFilter {
  int32_t n_terms;
  int32_t n_ops;                 /* 0 => no filter */
  uint8_t ops[B2Q_MAX_FILTER_OPS]; /* (kind << 4) | term index */
  DevTerm terms[B2Q_MAX_TERMS];
};

/* ---- accumulators ---------------------------------------------------------------------------------------
 * Internal dense arrays, one per accumulator, `entry_count` elements of 8 bytes in HBM, initialised to the
 * identity of their reduction so partial tables of several GPUs merge with one all-reduce per array.  The
 * reference's slot layout (NULL-sentinel init values, AVG pairs, key slots) is produced afterwards by the
 * materialise kernel. */
enum {
  ACC_COUNT = 0,   /* rows (COUNT(*)) or non-skipped values of `col` (col >= 0) */
  ACC_SUM_I64 = 1, /* wrap-around int64 sum (agg_sum, RuntimeFunctions.cpp:1151-1155) */
  ACC_SUM_F64 = 2,
  ACC_MIN_I64 = 3,
  ACC_MAX_I64 = 4,
  ACC_MIN_F64 = 5, /* stored as order-preserving int64 */
  ACC_MAX_F64 = 6,
  ACC_TOUCH = 7,   /* "some row reached this group": ONE BYTE per entry (the array holds uint8), merged with MAX */
  ACC_BITMAP = 9,  /* COUNT(DISTINCT c): the array holds one bitmap of bm_words 32-bit words per entry; a value sets bit
                      (v - bm_min) / bucket (agg_count_distinct_bitmap[_skip_val], RuntimeFunctions.cpp:366-376,1201-1210); merged with OR */
  ACC_NDV = 8      /* estimator query: the array is the linear-counting bitmap (plan.buffer_size bytes), one bit set per row
                      at MurmurHash3(tuple of DevProgram::keys) % bits (linear_probabilistic_count), merged with OR */
};

struct DevAcc {
  int64_t skip1_val;   /* skip the value when v == skip1_val (argument's own NULL sentinel) */
  int64_t skip2_val;   /* ... or when (skip2_trunc32 ? (int32)v : v) == skip2_val (aggregate type's sentinel) */
  int32_t col;         /* -1: no argument (COUNT(*)) */
  int8_t op;           /* ACC_* */
  int8_t width;        /* argument byte width */
  int8_t is_fp;        /* argument holds doubles: skip test is an fp compare against skip1 (as double) */
  int8_t skip1_en;
  int8_t skip2_en;
  int8_t skip2_trunc32;
  int8_t pad_[2];
  /* ACC_BITMAP */
  int64_t bm_min;      /* value of bit 0 */
  int64_t bm_bits;     /* bits per entry */
  int32_t bm_words;    /* 32-bit words per entry = align8(ceil(bits / 8)) / 4 (bitmapPaddedSizeBytes on the GPU) */
  int32_t bm_bucket;   /* > 1: bit = (v - bm_min) / bucket */
};

/* ---- group key ------------------------------------------------------------------------------------------ */
struct DevKey {
  int64_t min_val;     /* perfect hash: idx = key - min_val (bucket == 0 in this path) */
  int64_t null_val;    /* key column NULL sentinel as stored in the chunk (physical width, sign-extended) */
  int64_t null_logical;/* the logical type's sentinel (differs from null_val under ENCODING FIXED) */
  int64_t null_idx;    /* perfect hash: entry index of the NULL group (= max - min + 1), -1 if none */
  int64_t entry_count;
  uint64_t hash_magic; /* baseline: 2^64 / entry_count + 1 — h % entry_count by two multiplies (Lemire fastmod, exact for 32-bit h) */
  int32_t col;         /* -1: non-grouped */
  int8_t width;
  int8_t translate_null; /* has_nulls && column nullable (GroupByAndAggregate.cpp:1337-1350) */
  int8_t hash_key_width; /* baseline: bytes hashed by MurmurHash3 (4 or 8) */
  int8_t div_day;        /* 8-byte DATE key: idx = (key - min_val) / 86400 (the day bucket of DATE ranges, ExpressionRange.cpp:622) */
};

/* one GROUP BY column of a multi-column perfect hash (codegenPerfectHashFunction, GroupByAndAggregate.cpp:1549-1597):
 * entry = sum_c d_c * mult_c with d_c = key_c - min_c (NULL -> card_c - 1, i.e. max_c + 1 - min_c) */
struct DevKeyComp {
  int64_t min_val;
  int64_t null_val;     /* sentinel as stored in the chunk (sign-extended) */
  int64_t null_logical; /* sentinel of the logical type (what a projected NULL key reads as) */
  uint32_t card;        /* max - min + 1 (+1 when the column has NULLs) */
  uint32_t mult;        /* product of the cardinalities of the preceding columns */
  int32_t col;
  int8_t width;
  int8_t translate_null;
  int8_t div_day;       /* scan: 8-byte DATE component, d = (key - min_val) / 86400 */
  int8_t pad_;
  /* materialise only (DevLayout.keys): key of component index d = min_val + d * step, the NULL group stores null_stored */
  int64_t step;
  int64_t null_stored;
};

/* ---- one INNER hash-join level (PerfectJoinHashTable one-to-one: int32 slots, -1 = no row) ------------------ */
struct DevJoin {
  int64_t min_key;      /* slot = key - min_key */
  int64_t entry_count;  /* max_key - min_key + 1 */
  int64_t null_val;     /* outer key's NULL as stored in the chunk */
  int32_t fk_col;       /* launch column of the outer key, -1: no join */
  int8_t fk_width;      /* width code of the outer key column */
  int8_t nullable;      /* hash_join_idx_nullable: a NULL outer key never matches */
  int8_t packed_col;    /* >= 0: the table is {int32 row, int32 value-of-this-inner-launch-column} per slot, so the probe
                           and the gather of that column are ONE 8-byte load (random 4-byte gathers are bound by L1 tag
                           throughput, ~1 sector/clk/SM: two dependent gathers per row cost twice the scan itself) */
  int8_t packed_width;  /* width code of that column in the inner table */
  int8_t probe_cg;  /* experiment knob (B2Q_JOIN_CG): probe with ld.global.cg (L2 only) instead of the L1 path */
  int8_t left;          /* LEFT join: a row without a match stays, its inner columns read col_null[] */
  int8_t slot16;        /* the table is ONE uint16 per slot, staged in shared memory: value - slot16_min of packed_col
                           (the only inner column the query reads), 0xFFFE = that column is NULL, 0xFFFF = no row.
                           A 1e5-row dimension is then 200 KB and fits next to the group table. */
  int8_t pad_[5];
  int64_t slot16_min;
};

struct DevProgram {
  DevJoin join;
  int8_t col_inner[B2Q_MAX_COLS];    /* launch column belongs to the joined inner table: read at the matching inner row */
  int64_t col_null[B2Q_MAX_COLS];    /* inner columns: the NULL a LEFT join's unmatched row reads (chunk sentinel / NULL_DOUBLE bits) */
  DevFilter filter;
  DevKey key;
  int32_t n_keys;       /* > 1: multi-column perfect hash, `keys` below; the single-column paths use `key` */
  int32_t pad_keys_;
  DevKeyComp keys[B2Q_MAX_GROUP_COLS];
  int32_t n_accs;
  int32_t n_cols;
  float est_selectivity; /* planner's estimate from chunk stats (uniformity assumption) */
  int8_t eager_key;      /* load the key column for every row, overlapped with the filter columns */
  int8_t eager_args;     /* load aggregate arguments for every row instead of only the passing ones */
  int8_t col_width[B2Q_MAX_COLS];    /* byte width of launch column c */
  int8_t fused;          /* shared-memory-table fast path: the program is {COUNT(*)} and/or {one integer SUM without a
                            NULL test}: both updates of a row happen under ONE predicate region */
  int8_t fused_cnt;      /* accumulator index of the COUNT(*), or -1 */
  int8_t fused_sum;      /* accumulator index of the SUM_I64, or -1 */
  int8_t touch_acc;      /* index of the ACC_TOUCH accumulator, or -1 */
  int8_t touch_piggyback;/* global-table kernels: accumulator (COUNT / SUM_I64 without a skip test) whose returning
                            atomic also maintains the touched flag, or -1 (explicit flag check per row) */
  DevAcc accs[B2Q_MAX_ACCS];
};

/* ---- how a reference slot is produced from the accumulators (materialise kernel) ------------------------- */
enum {
  SLOT_KEY = 0,        /* projected group key (agg_id) */
  SLOT_COUNT = 1,      /* accs[a] as integer */
  SLOT_VALUE = 2,      /* accs[a] (int64 bits or double bits) ; if nn >= 0 and accs[nn] == 0 -> init (NULL sentinel) */
  SLOT_VALUE_ORD = 3,  /* like SLOT_VALUE but accs[a] holds an order-preserving int64 image of a double */
  SLOT_NONE = 4,       /* zero-width slot (baseline key reference) */
  SLOT_BITCOUNT = 5    /* COUNT(DISTINCT): number of bits set in the entry's bitmap of accs[a] (count_distinct_set_size) */
};
struct DevSlot {
  int64_t init_val;
  int64_t offset;      /* byte offset inside the row (row-wise) or of the slot column (columnar) */
  int64_t identity;    /* identity of accs[acc] (used when nn == -2) */
  int32_t acc;         /* accumulator index */
  int32_t nn;          /* >= 0: accumulator whose value 0 means "no value seen" -> init_val;
                          -2: "no value seen" <=> accs[acc] still holds its identity; -1: always valid */
  int8_t kind;         /* SLOT_* */
  int8_t width;        /* padded slot width: 0, 4 or 8 */
  int8_t key_comp;     /* SLOT_KEY of a multi-column key: which GROUP BY column */
  int8_t scale_day;    /* MIN / MAX over a days-encoded DATE chunk: the accumulator holds days, the slot seconds */
  int8_t as_float;     /* FLOAT argument (takes_float_argument, TargetInfo.h:106-110): the accumulator is a double; the slot gets
                          its float image in the low 4 bytes, the high 4 bytes keep the init pattern's (agg_*_float write 32 bits) */
  int8_t clamp_init;   /* SLOT_VALUE_ORD over a NOT NULL argument: the reference starts from +-DBL_MAX (+-FLT_MAX), which neither
                          +-inf nor a NaN can beat; the accumulator is clamped to that init value at materialise (b2q_clamp_ord) */
  int8_t pad_[2];
  int32_t bm_words;    /* SLOT_BITCOUNT: 32-bit words per entry */
  int32_t pad2_;
};
struct DevLayout {
  int64_t row_size;
  int64_t entry_count;
  int64_t key_min;       /* perfect: key = key_min + idx * key_step */
  int64_t key_step;      /* 1, or 86400 for a DATE key (bucketed range / days-encoded chunk) */
  int64_t key_null_stored; /* perfect hash stores the TRANSLATED NULL key: max + (bucket ? bucket : 1) */
  int64_t key_null_val;  /* value projected for the NULL group */
  int64_t null_idx;
  int32_t n_slots;
  int32_t touched_acc;   /* accumulator whose value != 0 marks a non-empty entry (non-keyless layouts) */
  int32_t keyless_marker;/* keyless: slot index whose init value marks an empty entry (idx_target_as_key), else -1 */
  int32_t n_keys;        /* > 1: multi-column perfect hash */
  int32_t touch_via_acc; /* accumulator (COUNT / integer SUM updated by every passing row) whose non-zero value also marks the entry, or -1 */
  DevKeyComp keys[B2Q_MAX_GROUP_COLS];
  int8_t has_key_col;    /* row starts with the group key(s) (non-keyless) */
  int8_t key_width;      /* 4 or 8 */
  int8_t baseline;       /* key comes from the keys[] array */
  int8_t columnar;       /* ResultSet.h:72-84 layout: slot offsets are column offsets, keys are int64 columns */
  int64_t key_col_stride;/* columnar: bytes per key column = align8(8 * entry_count) */
  DevSlot slots[B2Q_MAX_SLOTS];
};

/* identities ------------------------------------------------------------------------------------------------ */
#define B2Q_I64_MAX 0x7FFFFFFFFFFFFFFFLL
#define B2Q_I64_MIN (-B2Q_I64_MAX - 1)

/* order-preserving map double -> int64 (NaNs excluded by the caller) and back */
#if defined(__CUDACC__)
#define B2Q_HD __host__ __device__ __forceinline__
#else
#define B2Q_HD inline
#endif
B2Q_HD int64_t b2q_f64_to_ord(int64_t bits) { return bits ^ ((bits >> 63) & B2Q_I64_MAX); }
B2Q_HD int64_t b2q_ord_to_f64(int64_t ord) { return ord ^ ((ord >> 63) & B2Q_I64_MAX); }
/* MIN / MAX of doubles: std::min(old, NaN) keeps old, so a NaN never beats a number (RuntimeFunctions.cpp:1458-1468), yet a
 * group whose values are ALL NaN does not end "empty": the nullable form assigns its first value and ends at NaN
 * (DEF_SKIP_AGG, :1558-1569), the NOT NULL form keeps its init value (std::min(DBL_MAX, NaN)).  So a NaN enters the
 * order-preserving accumulator as the image next to the identity (a NaN bit pattern itself): it loses to every number and is
 * still told apart from "no value seen" at materialise. */
B2Q_HD bool b2q_bits_is_nan(int64_t bits) { return (bits & B2Q_I64_MAX) > 0x7FF0000000000000LL; }
B2Q_HD int64_t b2q_f64_min_ord(int64_t bits) { return b2q_bits_is_nan(bits) ? B2Q_I64_MAX - 1 : b2q_f64_to_ord(bits); }
B2Q_HD int64_t b2q_f64_max_ord(int64_t bits) { return b2q_bits_is_nan(bits) ? B2Q_I64_MIN + 1 : b2q_f64_to_ord(bits); }
/* NOT NULL MIN / MAX of a double start from the init value DBL_MAX / -DBL_MAX (FLT_MAX / -FLT_MAX for a FLOAT argument) instead
 * of an identity: agg_min_double(DBL_MAX, +inf) stays DBL_MAX.  This clamps the order-preserving accumulator `raw` of a MIN
 * (identity I64_MAX) or MAX (identity I64_MIN) the same way; the result is the init value exactly when the clamp bites. */
B2Q_HD int64_t b2q_clamp_ord(int64_t raw, int64_t identity, bool as_float) {
  const double lim = as_float ? (double)FLT_MAX : DBL_MAX;
  int64_t b;
  if (identity == B2Q_I64_MAX) { memcpy(&b, &lim, 8); const int64_t o = b2q_f64_to_ord(b); return raw < o ? raw : o; }
  const double neg = -lim;
  memcpy(&b, &neg, 8);
  const int64_t o = b2q_f64_to_ord(b);
  return raw > o ? raw : o;
}

B2Q_HD int64_t b2q_acc_identity(int op) {
  switch (op) {
    case ACC_MIN_I64: case ACC_MIN_F64: return B2Q_I64_MAX; /* ord(+inf) < I64_MAX: fine as identity */
    case ACC_MAX_I64: case ACC_MAX_F64: return B2Q_I64_MIN;
    default: return 0; /* COUNT, SUM_I64; SUM_F64: +0.0 */
  }
}

/* ---- read-out of a reference-layout result buffer ------------------------------------------------------------
 * One definition for the host reader (getNextRow / getRowAt / ColumnarResults in executor.cpp) and the device
 * conversion (columnar.cu), so that the two cannot drift.  Slots are aligned to their padded width, so the device loads
 * are plain typed loads; the host goes through memcpy. */
#define B2Q_NULL_DOUBLE DBL_MIN
#define B2Q_NULL_FLOAT FLT_MIN

B2Q_HD int64_t b2q_ld(const int8_t* p, int w) {
  if (w == 1) return *p; /* projection: logical-sized TINYINT / SMALLINT columns of a columnar buffer */
#if defined(__CUDA_ARCH__)
  if (w == 2) return *reinterpret_cast<const int16_t*>(p);
  return w == 4 ? (int64_t)*reinterpret_cast<const int32_t*>(p) : *reinterpret_cast<const int64_t*>(p);
#else
  if (w == 2) { int16_t x; memcpy(&x, p, 2); return x; }
  if (w == 4) { int32_t x; memcpy(&x, p, 4); return x; }
  int64_t x;
  memcpy(&x, p, 8);
  return x;
#endif
}
B2Q_HD float b2q_ld_f32(const int8_t* p) {
#if defined(__CUDA_ARCH__)
  return *reinterpret_cast<const float*>(p);
#else
  float f;
  memcpy(&f, p, 4);
  return f;
#endif
}
B2Q_HD double b2q_bits_f64(int64_t bits) {
#if defined(__CUDA_ARCH__)
  return __longlong_as_double(bits);
#else
  double d;
  memcpy(&d, &bits, 8);
  return d;
#endif
}

/* logical size / NULL sentinel (dictionary-encoded strings are int32 ids, TIME-family types int64) */
B2Q_HD bool b2q_is_dict_string(int t) { return t == B2Q_kTEXT || t == B2Q_kVARCHAR || t == B2Q_kCHAR; }
B2Q_HD bool b2q_is_decimal(int t) { return t == B2Q_kDECIMAL || t == B2Q_kNUMERIC; }
B2Q_HD int b2q_type_size(int t) {
  return t == B2Q_kTINYINT ? 1 : t == B2Q_kSMALLINT ? 2 : (t == B2Q_kINT || t == B2Q_kFLOAT || b2q_is_dict_string(t)) ? 4 : 8;
}
B2Q_HD int64_t b2q_int_null(int t) {
  return t == B2Q_kTINYINT ? INT8_MIN : t == B2Q_kSMALLINT ? INT16_MIN : (t == B2Q_kINT || b2q_is_dict_string(t)) ? INT32_MIN : INT64_MIN;
}
B2Q_HD double b2q_exp_to_scale(int scale) { double d = 1; for (int i = 0; i < scale; ++i) d *= 10; return d; }

/* where entry `e` keeps slot `s` / its first key: row-wise (ResultSet.h:55-70) or columnar (:72-84) */
B2Q_HD const int8_t* b2q_slot_ptr(const B2QPlan& p, const int8_t* buf, int64_t e, int s) {
  return p.output_columnar ? buf + p.slot_offset[s] + e * p.slot_padded_width[s] : buf + e * p.row_size + p.slot_offset[s];
}
B2Q_HD const int8_t* b2q_key_ptr(const B2QPlan& p, const int8_t* buf, int64_t e) {
  return p.output_columnar ? buf + e * 8 : buf + e * p.row_size;
}

/* ResultSet::getColType: AVG reads as DOUBLE, every other target as its own type */
B2Q_HD B2QTypeInfo b2q_target_col_type(const B2QTargetInfo& t) {
  if (t.is_agg && t.agg_kind == B2Q_kAVG) { B2QTypeInfo d; d.type = B2Q_kDOUBLE; d.notnull = 0; d.scale = 0; return d; }
  return t.sql_type;
}

/* getRowAt / getTargetValueFromBufferRowwise|Colwise (ResultSetIteration.cpp:820-1000) for target `i` of entry `entry` */
B2Q_HD void b2q_read_target(const B2QPlan& p, const int8_t* buf, int64_t entry, int i, bool decimal_to_double, B2QTargetValue* out) {
  const B2QTargetInfo& t = p.targets[i];
  const int s = t.first_slot;
  int w = p.slot_padded_width[s];
  const int8_t* ptr = b2q_slot_ptr(p, buf, entry, s);
  if (w == 0) { ptr = b2q_key_ptr(p, buf, entry); w = p.effective_key_width; } /* baseline: the key column is the target */
  const int64_t ival = b2q_ld(ptr, w);
  B2QTargetValue o;
  o.is_fp = 0; o.is_null = 0; o.ival = 0; o.dval = 0;
  /* compact type (get_compact_type): MIN/MAX -> argument type, otherwise the target type */
  const bool has_arg = t.agg_arg_type.type != 0;
  const int compact_type = (t.is_agg && has_arg && (t.agg_kind == B2Q_kMIN || t.agg_kind == B2Q_kMAX)) ? t.agg_arg_type.type : t.sql_type.type;
  if (t.is_agg && t.agg_kind == B2Q_kAVG) { /* pair_to_double, ResultSetBufferAccessors.h:197-227 */
    const int64_t cnt = b2q_ld(b2q_slot_ptr(p, buf, entry, s + 1), 8);
    o.is_fp = 1;
    if (cnt == 0) { o.dval = B2Q_NULL_DOUBLE; o.is_null = 1; }
    else {
      double dividend;
      if (t.sql_type.type == B2Q_kDOUBLE) dividend = b2q_bits_f64(ival);
      else if (t.sql_type.type == B2Q_kFLOAT) dividend = b2q_ld_f32(ptr); /* float_argument_input: pair_to_double reads the sum as a float */
      else dividend = static_cast<double>(ival);
      /* DECIMAL: one division by count x 10^scale, ResultSetBufferAccessors.h:222-225 */
      o.dval = b2q_is_decimal(t.sql_type.type) && t.sql_type.scale ? dividend / (static_cast<double>(cnt) * b2q_exp_to_scale(t.sql_type.scale))
                                                                   : dividend / static_cast<double>(cnt);
      o.is_null = o.dval == B2Q_NULL_DOUBLE;
    }
  } else if (compact_type == B2Q_kDOUBLE) {
    o.is_fp = 1;
    o.dval = b2q_bits_f64(ival);
    o.is_null = o.dval == B2Q_NULL_DOUBLE;
  } else if (compact_type == B2Q_kFLOAT) { /* make_target_value: a float read from the slot's low 4 bytes (ResultSetIteration.cpp:2140-2160) */
    const float f = b2q_ld_f32(ptr);
    o.is_fp = 1;
    o.dval = f;
    o.is_null = f == B2Q_NULL_FLOAT;
  } else if (b2q_is_decimal(compact_type)) { /* makeTargetValue, ResultSetIteration.cpp:2193-2210 */
    const B2QTypeInfo& ct = compact_type == t.sql_type.type ? t.sql_type : t.agg_arg_type;
    const bool agg_null = t.is_agg && (t.agg_kind == B2Q_kSUM || t.agg_kind == B2Q_kMIN || t.agg_kind == B2Q_kMAX);
    o.is_null = ival == INT64_MIN && (agg_null || !ct.notnull);
    if (decimal_to_double) {
      o.is_fp = 1;
      o.dval = o.is_null ? B2Q_NULL_DOUBLE : static_cast<double>(ival) / b2q_exp_to_scale(ct.scale);
    } else o.ival = ival;
  } else {
    int64_t resized = ival;
    switch (b2q_type_size(compact_type)) {
      case 1: resized = static_cast<int8_t>(ival); break;
      case 2: resized = static_cast<int16_t>(ival); break;
      case 4: resized = static_cast<int32_t>(ival); break;
      default: break;
    }
    if (resized == b2q_int_null(compact_type)) { o.ival = b2q_int_null(t.sql_type.type); o.is_null = 1; }
    else o.ival = ival;
  }
  *out = o;
}

/* one value of a ColumnarResults column of byte width `width` (toBuffer, ColumnarResults.cpp:42-90); returns the
 * stored bits widened to int64 (doubles / floats as their bit pattern) so that the caller can test them against the
 * column's NULL sentinel */
B2Q_HD int64_t b2q_store_target(const B2QTargetValue& v, int width, int8_t* dst) {
  if (v.is_fp && width == 4) {
    const float f = v.is_null ? B2Q_NULL_FLOAT : static_cast<float>(v.dval);
    int32_t bits;
    memcpy(&bits, &f, 4);
    *reinterpret_cast<int32_t*>(dst) = bits;
    return bits;
  }
  int64_t x = v.ival;
  if (v.is_fp) memcpy(&x, &v.dval, 8);
  switch (width) {
    case 1: x = static_cast<int8_t>(x); *dst = static_cast<int8_t>(x); break;
    case 2: x = static_cast<int16_t>(x); *reinterpret_cast<int16_t*>(dst) = static_cast<int16_t>(x); break;
    case 4: x = static_cast<int32_t>(x); *reinterpret_cast<int32_t*>(dst) = static_cast<int32_t>(x); break;
    default: *reinterpret_cast<int64_t*>(dst) = x;
  }
  return x;
}

/* the NULL sentinel of a ColumnarResults column as b2q_store_target returns its bits */
B2Q_HD int64_t b2q_null_bits(int type) {
  if (type == B2Q_kDOUBLE) { const double d = B2Q_NULL_DOUBLE; int64_t b; memcpy(&b, &d, 8); return b; }
  if (type == B2Q_kFLOAT) { const float f = B2Q_NULL_FLOAT; int32_t b; memcpy(&b, &f, 4); return b; }
  return b2q_int_null(type);
}

/* ---- stopping a running call (B2QExecutionOptions: runtime interrupt, dynamic watchdog) --------------------------------
 * Both pointers NULL = nothing is checked (the kernels test that once, warp-uniformly, per chunk). */
struct DevInterrupt {
  const volatile uint32_t* flag; /* device view of the interrupt token's flag (mapped host memory), or NULL */
  const uint64_t* t0;            /* watchdog: %globaltimer when the call's first kernel ran (device memory), or NULL */
  uint64_t budget_ns;            /* watchdog budget */
};
#define B2Q_INTERRUPT_POLL_NS 100000ull /* a CTA reads the mapped flag at most once per 100 us */

/* ---- launch description handed to the kernels ----------------------------------------------------------- */
struct DevLaunch {
  /* column table: col_ptrs[frag * n_cols + c] — device pointers (device array) */
  const int8_t* const* col_ptrs;
  const int64_t* frag_rows;        /* [n_frags] device */
  const int64_t* frag_chunk_start; /* [n_frags + 1] device: prefix sum of chunks per fragment */
  int32_t n_frags;
  int32_t split;                   /* HBM-table kernels: COUNT / integer SUM arrays are (lo[n] | hi[n]) 32-bit halves (1) or plain int64[] (0) */
  int64_t total_chunks;
  int64_t* accs[B2Q_MAX_ACCS];     /* dense accumulator arrays in HBM */
  int64_t* keys;                   /* baseline: open-addressing key array (EMPTY_KEY_64 initialised) */
  int32_t* error;                  /* device int: first error code */
  const int32_t* join_buff;        /* one-to-one join table (HashJoin::getJoinHashBuffer), or nullptr */
  DevInterrupt intr;               /* what stops the launch early (error word <- B2Q_ERR_INTERRUPTED / OUT_OF_TIME) */
};

/* chosen at plan time, needed at launch */
struct SmemPlan {
  int32_t use_smem;       /* per-CTA private table */
  int32_t replicas;       /* power of two, >= 1 */
  int32_t acc_bytes[B2Q_MAX_ACCS]; /* bytes per entry in shared memory (4 or 8) */
  int32_t acc_off[B2Q_MAX_ACCS];   /* byte offset of the accumulator's array inside ONE replica */
  int32_t replica_bytes;
  int32_t total_bytes;
  int32_t join_off;       /* >= 0: the join table is TMA-staged into shared memory at this byte offset (dimension-sized tables) */
  int32_t join_bytes;     /* bytes staged (multiple of 16) */
};

/* ---- ORDER BY / LIMIT over the materialised table (sort.cu) ------------------------------------------------ */
#define B2Q_MAX_ORDER_ENTRIES 8
/* F32 / AVG_F32: float_argument_input, the float's 4 bytes in the slot's low word */
enum { SORTKEY_I64 = 0, SORTKEY_F64 = 1, SORTKEY_AVG_I64 = 2, SORTKEY_AVG_F64 = 3, SORTKEY_F32 = 4, SORTKEY_AVG_F32 = 5 };
struct DevSortKey {        /* one Analyzer::OrderEntry resolved against the output layout */
  int64_t off1, off2;      /* slot offsets (row-wise: inside the row; columnar: of the column); off2 = AVG's count slot */
  int64_t null_pattern;    /* null_val_bit_pattern of the compact type (ResultSet::isNull, ResultSetIteration.cpp:2601-2618) */
  int8_t w1;               /* 4 or 8 */
  int8_t kind;             /* SORTKEY_* */
  int8_t nullable;         /* !get_compact_type(target).get_notnull() */
  int8_t is_desc, nulls_first;
  int8_t scale;            /* AVG of a DECIMAL: pair_to_double divides by count x 10^scale */
  int8_t pad_[2];
};
struct DevSortLayout {     /* what the kernels need to address an entry of a reference-layout buffer */
  int64_t row_size, entry_count;
  int64_t marker_off, marker_init; /* keyless: the idx_target_as_key slot and its init value */
  int8_t columnar, grouped, keyless, marker_w, key_w;
  int8_t pad_[3];
};
struct DevGatherCols {     /* columnar gather: every key / slot column, offsets for the source and the compact buffer */
  int32_t n;
  int32_t pad_;
  int64_t in_off[B2Q_MAX_SLOTS + B2Q_MAX_GROUP_COLS], out_off[B2Q_MAX_SLOTS + B2Q_MAX_GROUP_COLS];
  int8_t width[B2Q_MAX_SLOTS + B2Q_MAX_GROUP_COLS];
};

/* ---- device ColumnarResults (columnar.cu) over a result set of executor.cpp ----------------------------------- */
namespace b2q {
struct RsSource {
  const B2QPlan* plan;
  const int8_t* d_buf;  /* device copy of the storage (result_on_device), else nullptr */
  const int8_t* h_buf;  /* host copy, else nullptr */
  size_t buf_size;
  int device;           /* device of d_buf, -1 without one */
  const uint32_t* perm; /* ResultSet::permutation_ (host), n_perm entries; n_perm == 0: not sorted */
  size_t n_perm;
  size_t drop_first, keep_first;
};
bool rs_source(const B2QResultSet* rs, RsSource* out);
DevSortLayout sort_layout_for(const B2QPlan& p);
}  // namespace b2q

/* ---- projection (project.cu): one projected column, decoded the way the chunk decoders hand it to agg_id ----------- */
enum { PROJ_INT = 0, PROJ_F64 = 1, PROJ_F32 = 2 };
struct DevProjCol {
  int64_t null_phys;    /* the chunk's NULL as loaded (sign-extended; 255 / 65535 for DICT(8|16)) */
  int64_t null_logical; /* what a NULL row stores: the logical type's sentinel */
  int64_t out_off;      /* row-wise: byte offset inside the row; columnar: offset of the column */
  int32_t col;          /* launch column */
  int8_t width;         /* physical width code of the chunk (load32 / load64) */
  int8_t out_w;         /* slot width: 8 row-wise, the logical size columnar */
  int8_t kind;          /* PROJ_* */
  int8_t days;          /* DATE ENCODING DAYS: value * 86400 */
  int8_t translate_null;/* the physical NULL differs from the logical one (ENCODING FIXED, DICT(8|16), DAYS) */
  int8_t pad_[7];
};
struct DevProject {
  int32_t n;
  int32_t pad_;
  int64_t scan_limit;   /* B2QExecUnit::scan_limit (0 = none) */
  DevProjCol cols[B2Q_MAX_TARGETS];
};

/* host-side query object behind B2QQuery */
struct B2QQuery {
  B2QPlan plan;
  DevProgram prog;
  DevLayout layout;
  SmemPlan smem;
  int32_t col_ids[B2Q_MAX_COLS]; /* launch column index -> table column id (>= n_outer_cols: inner column id + n_outer_cols) */
  int32_t bigint_count;
  int32_t n_outer_cols;          /* columns of the scanned table; 0 < join_inner_key_col + 1 only with a join */
  int32_t join_inner_key_col;    /* inner table column of the join key, -1 without a join */
  /* sort_info of the execution unit (copied: the partial / finalize split outlives the caller's unit) */
  int32_t n_order;
  B2QOrderEntry order[B2Q_MAX_ORDER_ENTRIES];
  int32_t has_limit;
  int64_t limit, offset;
  int64_t total_tuples;          /* rows of all fragments of the table (every device's) */
  DevProject proj;               /* plan.query_desc_type == B2Q_Projection */
  /* the values of set term t (prog.filter.terms[t].is_set): sorted, unique, in the column's register class (days for a
   * days-encoded DATE); empty for every other term */
  std::vector<int64_t> set_values[B2Q_MAX_TERMS];
};
