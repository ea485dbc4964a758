/* TEST INFRASTRUCTURE — never linked into the product.
 *
 * A host-side reading of the FILTER part of the device program the planner emits (heavydb_b200/csrc/b2q_internal.h:
 * DevFilter / DevTerm), one row at a time, following the semantics the scan kernel implements
 * (kernels.cu: eval_term, eval_term2, eval_filter).  tests/test_filter_lowering.py uses it to check the planner's
 * lowering — range encoding of comparisons, NULL folding, De Morgan push-down, operand ordering on the 4-deep mask stack,
 * constants of days-encoded DATE columns — against the oracle on the CPU, where no kernel can run. */
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../../heavydb_b200/csrc/b2q_internal.h"

namespace {
int64_t load_int(const int8_t* base, int width, int64_t row) {
  switch (width) {
    case 8: { int64_t v; memcpy(&v, base + row * 8, 8); return v; }
    case 4: { int32_t v; memcpy(&v, base + row * 4, 4); return v; }
    case 2: { int16_t v; memcpy(&v, base + row * 2, 2); return v; }
    case -2: { uint16_t v; memcpy(&v, base + row * 2, 2); return v; }
    case -1: return static_cast<uint8_t>(base[row]);
    default: return base[row];
  }
}
double as_double(int64_t bits) { double d; memcpy(&d, &bits, 8); return d; }
/* an fp column: double bits; a FLOAT chunk (width 4) widened exactly, as the kernels do on every load */
int64_t load_fp_bits(const int8_t* base, int width, int64_t row) {
  if (width == 4) { float f; memcpy(&f, base + row * 4, 4); const double d = f; int64_t b; memcpy(&b, &d, 8); return b; }
  int64_t b; memcpy(&b, base + row * 8, 8); return b;
}

bool eval_term(const DevTerm& t, const int8_t* col, int64_t row) {
  const bool neg = t.negate;
  if (!t.cmp_fp) {
    const int64_t v = load_int(col, t.width, row);
    bool r;
    if (t.width == 8) r = (static_cast<uint64_t>(v) - static_cast<uint64_t>(t.lo) <= t.span) != neg;
    else r = (static_cast<uint32_t>(static_cast<int32_t>(v)) - static_cast<uint32_t>(t.lo) <= static_cast<uint32_t>(t.span)) != neg;
    if (t.null_check) {
      const int64_t nullv = t.width == 8 ? t.null_bits : static_cast<int64_t>(static_cast<int32_t>(t.null_bits));
      if (v == nullv) r = false;
    }
    return r;
  }
  double d;
  bool isnull;
  if (t.col_is_fp) { d = as_double(load_fp_bits(col, t.width, row)); isnull = d == as_double(t.null_bits); }
  else {
    const int64_t v = load_int(col, t.width, row);
    d = static_cast<double>(v);
    isnull = v == (t.width == 8 ? t.null_bits : static_cast<int64_t>(static_cast<int32_t>(t.null_bits)));
  }
  bool r = ((d >= t.flo) & (d <= t.fhi)) != neg;
  if (t.null_check && isnull) r = false;
  return r;
}

bool eval_term2(const DevTerm& t, const int8_t* c1, const int8_t* c2, int64_t row) {
  const int64_t a = t.col_is_fp ? load_fp_bits(c1, t.width, row) : load_int(c1, t.width, row);
  const int64_t b = t.col2_is_fp ? load_fp_bits(c2, t.width2, row) : load_int(c2, t.width2, row);
  bool isnull, r;
  const int op = t.op2;
  if (t.cmp_fp) {
    double x, y;
    isnull = false;
    if (t.col_is_fp) { x = as_double(a); isnull |= t.nullable1 && x == as_double(t.null_bits); } else { x = static_cast<double>(a); isnull |= t.nullable1 && a == t.null_bits; }
    if (t.col2_is_fp) { y = as_double(b); isnull |= t.nullable2 && y == as_double(t.null_bits2); } else { y = static_cast<double>(b); isnull |= t.nullable2 && b == t.null_bits2; }
    r = op == B2Q_kEQ ? x == y : op == B2Q_kNE ? x != y : op == B2Q_kLT ? x < y : op == B2Q_kGT ? x > y : op == B2Q_kLE ? x <= y : x >= y;
  } else {
    isnull = (t.nullable1 && a == t.null_bits) || (t.nullable2 && b == t.null_bits2);
    r = op == B2Q_kEQ ? a == b : op == B2Q_kNE ? a != b : op == B2Q_kLT ? a < b : op == B2Q_kGT ? a > b : op == B2Q_kLE ? a <= b : a >= b;
  }
  return r && !isnull;
}
}  // namespace

/* 1 / 0 = the row passes / fails the lowered filter; -1 = the program is not one this emulator reads (join level,
 * stack deeper than the device's).  table_cols[c] = chunk of table column c for the fragment, `row` inside it. */
static int32_t eval_filter_impl(const B2QQuery* q, const void* const* table_cols, int64_t row);
extern "C" int32_t b2q_test_eval_filter(const B2QQuery* q, const void* const* table_cols, int64_t row) {
  if (!q || q->prog.join.fk_col >= 0) return -1;
  return eval_filter_impl(q, table_cols, row);
}
/* Join programs: the caller has already done the probe — table_cols[n_outer + c] is inner column c GATHERED at the matching
 * inner row for every outer row (the chunk's NULL sentinel where a LEFT join found no match), so the filter reads one
 * denormalised row exactly as the kernel reads it through the join index. */
extern "C" int32_t b2q_test_eval_filter_joined(const B2QQuery* q, const void* const* table_cols, int64_t row) {
  if (!q || q->prog.join.fk_col < 0) return -1;
  return eval_filter_impl(q, table_cols, row);
}
static int32_t eval_filter_impl(const B2QQuery* q, const void* const* table_cols, int64_t row) {
  const DevFilter& f = q->prog.filter;
  if (f.n_ops == 0) return 1;
  bool st[4];
  int sp = 0;
  for (int i = 0; i < f.n_ops; ++i) {
    const uint32_t op = f.ops[i], kind = op >> 4;
    if (kind == FOP_TERM) {
      if (sp >= 4) return -1;
      const DevTerm& t = f.terms[op & 15];
      const int8_t* c1 = static_cast<const int8_t*>(table_cols[q->col_ids[t.col]]);
      st[sp++] = t.col2 >= 0 ? eval_term2(t, c1, static_cast<const int8_t*>(table_cols[q->col_ids[t.col2]]), row) : eval_term(t, c1, row);
    } else {
      if (sp < 2) return -1;
      const bool b = st[--sp], a = st[--sp];
      st[sp++] = kind == FOP_AND ? (a && b) : (a || b);
    }
  }
  return sp == 1 ? (st[0] ? 1 : 0) : -1;
}
extern "C" int32_t b2q_test_filter_terms(const B2QQuery* q) { return q ? q->prog.filter.n_terms : -1; }

/* The entry a passing row aggregates into under PERFECT hash, read from the lowered key mapping (DevKey / DevKeyComp) with
 * the semantics of process_chunk's "group index" block: idx = key - min (raw chunk value: days for a days-encoded DATE),
 * `/ 86400` for an 8-byte DATE, NULL -> the translated NULL entry; several GROUP BY columns: mixed radix.
 * -1 = out of range (the kernel raises KEY_OUT_OF_RANGE), -2 = not a perfect-hash program. */
extern "C" int64_t b2q_test_group_index(const B2QQuery* q, const void* const* table_cols, int64_t row) {
  if (!q || q->plan.query_desc_type != B2Q_GroupByPerfectHash) return -2;
  const DevProgram& P = q->prog;
  if (P.n_keys > 1) {
    int64_t e = 0;
    for (int c = 0; c < P.n_keys; ++c) {
      const DevKeyComp& kc = P.keys[c];
      const int64_t k = load_int(static_cast<const int8_t*>(table_cols[q->col_ids[kc.col]]), kc.width, row);
      int64_t d = k - kc.min_val;
      if (kc.div_day) { d = d / 86400; if (k % 86400 != 0 && !(kc.translate_null && k == kc.null_val)) d = -1; }
      if (kc.translate_null && k == kc.null_val) d = static_cast<int64_t>(kc.card) - 1;
      if (static_cast<uint64_t>(d) >= kc.card) return -1;
      e += d * static_cast<int64_t>(kc.mult);
    }
    return e;
  }
  const DevKey& K = P.key;
  if (K.col < 0) return -2;
  const int64_t k = load_int(static_cast<const int8_t*>(table_cols[q->col_ids[K.col]]), K.width, row);
  int64_t idx;
  if (K.width != 8) { /* the 32-bit key path: unsigned difference of the low words */
    idx = static_cast<uint32_t>(static_cast<uint32_t>(static_cast<int32_t>(k)) - static_cast<uint32_t>(K.min_val));
    if (K.translate_null && static_cast<int32_t>(k) == static_cast<int32_t>(K.null_val)) idx = K.null_idx;
  } else {
    idx = k - K.min_val;
    if (K.div_day) { idx = idx / 86400; if (k % 86400 != 0 && !(K.translate_null && k == K.null_val)) idx = -1; }
    if (K.translate_null && k == K.null_val) idx = K.null_idx;
  }
  return static_cast<uint64_t>(idx) < static_cast<uint64_t>(K.entry_count) ? idx : -1;
}

/* ---------------------------------------------------------------------------------------------------------------------
 * The whole lowered program on the host: filter -> entry -> accumulators (DevAcc skip rules) -> materialise (DevLayout),
 * for non-grouped and perfect-hash programs without a join.  Accumulator semantics follow process_chunk /
 * not_skipped64 (kernels.cu); materialise is the host reading of b2q_k_materialize.  DOUBLE sums are accumulated per
 * fragment and folded in fragment order, the order of the oracle's host reduce.
 * Returns 0, or a B2Q error code (KEY_OUT_OF_RANGE), or -2 for programs outside this emulator.
 * ------------------------------------------------------------------------------------------------------------------- */
namespace {
bool skipped(const DevAcc& a, int64_t v) {
  if (!a.skip1_en && !a.skip2_en) return false;
  if (a.is_fp) return as_double(v) == as_double(a.skip1_val);
  const int64_t w = a.skip2_trunc32 ? static_cast<int64_t>(static_cast<int32_t>(v)) : v;
  return (a.skip1_en && v == a.skip1_val) || (a.skip2_en && w == a.skip2_val);
}
}  // namespace

static int32_t run_program_impl(const B2QQuery* q, int32_t n_frags, const void* const* const* frag_cols,
                                const int64_t* frag_rows, const uint8_t* const* frag_valid, int8_t* out);
extern "C" int32_t b2q_test_run_program(const B2QQuery* q, int32_t n_frags, const void* const* const* frag_cols,
                                        const int64_t* frag_rows, int8_t* out) {
  if (!q || q->prog.join.fk_col >= 0) return -2;
  return run_program_impl(q, n_frags, frag_cols, frag_rows, nullptr, out);
}
/* Join programs on denormalised rows (see b2q_test_eval_filter_joined); frag_valid[f][row] == 0: an INNER join found no
 * match for the row, which then does not exist. */
extern "C" int32_t b2q_test_run_program_joined(const B2QQuery* q, int32_t n_frags, const void* const* const* frag_cols,
                                               const int64_t* frag_rows, const uint8_t* const* frag_valid, int8_t* out) {
  if (!q || q->prog.join.fk_col < 0) return -2;
  return run_program_impl(q, n_frags, frag_cols, frag_rows, frag_valid, out);
}
static int32_t run_program_impl(const B2QQuery* q, int32_t n_frags, const void* const* const* frag_cols,
                                const int64_t* frag_rows, const uint8_t* const* frag_valid, int8_t* out) {
  const B2QPlan& plan = q->plan;
  if (plan.query_desc_type != B2Q_GroupByPerfectHash && plan.query_desc_type != B2Q_NonGroupedAggregate) return -2;
  const DevProgram& P = q->prog;
  const int64_t n = plan.entry_count;
  std::vector<std::vector<int64_t>> accs(P.n_accs, std::vector<int64_t>(static_cast<size_t>(n)));
  std::vector<uint8_t> touch(static_cast<size_t>(n), 0);
  for (int a = 0; a < P.n_accs; ++a) for (int64_t i = 0; i < n; ++i) accs[a][i] = b2q_acc_identity(P.accs[a].op);
  std::vector<std::vector<double>> fsum(P.n_accs);
  std::vector<std::vector<uint32_t>> bitmaps(P.n_accs); /* ACC_BITMAP: bm_words 32-bit words per entry */
  for (int a = 0; a < P.n_accs; ++a) if (P.accs[a].op == ACC_BITMAP) bitmaps[a].assign(static_cast<size_t>(n) * P.accs[a].bm_words, 0u);
  for (int f = 0; f < n_frags; ++f) {
    for (int a = 0; a < P.n_accs; ++a) if (P.accs[a].op == ACC_SUM_F64) fsum[a].assign(static_cast<size_t>(n), 0.0);
    std::vector<uint8_t> ftouch(static_cast<size_t>(n), 0);
    for (int64_t row = 0; row < frag_rows[f]; ++row) {
      if (frag_valid && !frag_valid[f][row]) continue;
      const int32_t pass = eval_filter_impl(q, frag_cols[f], row);
      if (pass < 0) return -2;
      if (!pass) continue;
      int64_t e = 0;
      if (plan.query_desc_type == B2Q_GroupByPerfectHash) {
        e = b2q_test_group_index(q, frag_cols[f], row);
        if (e == -1) return B2Q_ERR_KEY_OUT_OF_RANGE;
        if (e < 0) return -2;
      }
      ftouch[e] = 1;
      for (int a = 0; a < P.n_accs; ++a) {
        const DevAcc& A = P.accs[a];
        if (A.op == ACC_TOUCH) { touch[e] = 1; continue; }
        int64_t v = 0;
        if (A.col >= 0) {
          const int8_t* col = static_cast<const int8_t*>(frag_cols[f][q->col_ids[A.col]]);
          v = A.is_fp ? load_fp_bits(col, A.width, row) : load_int(col, A.width, row);
          if (skipped(A, v)) continue;
        }
        if (A.op == ACC_BITMAP) { /* as process_chunk: bit (v - min) / bucket of the entry's bitmap */
          uint64_t idx = static_cast<uint64_t>(v - A.bm_min);
          if (A.bm_bucket > 1) idx /= static_cast<uint64_t>(A.bm_bucket);
          if (idx >= static_cast<uint64_t>(A.bm_bits)) return B2Q_ERR_KEY_OUT_OF_RANGE;
          bitmaps[a][static_cast<size_t>(e) * A.bm_words + (idx >> 5)] |= 1u << (idx & 31);
          continue;
        }
        int64_t& acc = accs[a][e];
        switch (A.op) {
          case ACC_COUNT: acc += 1; break;
          case ACC_SUM_I64: acc = static_cast<int64_t>(static_cast<uint64_t>(acc) + static_cast<uint64_t>(v)); break;
          case ACC_SUM_F64: fsum[a][e] += as_double(v); break;
          case ACC_MIN_I64: acc = v < acc ? v : acc; break;
          case ACC_MAX_I64: acc = v > acc ? v : acc; break;
          case ACC_MIN_F64: { const int64_t o = b2q_f64_min_ord(v); acc = o < acc ? o : acc; break; }
          case ACC_MAX_F64: { const int64_t o = b2q_f64_max_ord(v); acc = o > acc ? o : acc; break; }
          default: return -2;
        }
      }
    }
    for (int a = 0; a < P.n_accs; ++a)
      if (P.accs[a].op == ACC_SUM_F64)
        for (int64_t i = 0; i < n; ++i)
          if (ftouch[i]) { const double s = as_double(accs[a][i]) + fsum[a][i]; memcpy(&accs[a][i], &s, 8); }
  }
  /* ---- materialise (b2q_k_materialize) ---- */
  const DevLayout& L = q->layout;
  if (L.baseline) return -2;
  for (int64_t i = 0; i < L.entry_count; ++i) {
    int8_t* row = out + i * L.row_size;
    bool touched = true;
    int64_t key = 0, mkey_stored[B2Q_MAX_GROUP_COLS], mkey_proj[B2Q_MAX_GROUP_COLS];
    if (L.n_keys > 1) {
      for (int c = 0; c < L.n_keys; ++c) {
        const DevKeyComp& kc = L.keys[c];
        const int64_t comp = (i / kc.mult) % kc.card;
        const bool is_null_comp = kc.translate_null && comp == static_cast<int64_t>(kc.card) - 1;
        mkey_stored[c] = is_null_comp ? kc.null_stored : kc.min_val + comp * kc.step;
        mkey_proj[c] = is_null_comp ? kc.null_logical : kc.min_val + comp * kc.step;
      }
      if (L.touched_acc >= 0) touched = touch[i] != 0 || (L.touch_via_acc >= 0 && accs[L.touch_via_acc][i] != 0);
    } else {
      key = (i == L.null_idx) ? L.key_null_val : L.key_min + i * L.key_step;
      if (L.touched_acc >= 0) touched = touch[i] != 0 || (L.touch_via_acc >= 0 && accs[L.touch_via_acc][i] != 0);
    }
    auto put64 = [](int8_t* p, int64_t v) { memcpy(p, &v, 8); };
    auto put32 = [](int8_t* p, int32_t v) { memcpy(p, &v, 4); };
    if (L.has_key_col && L.columnar) {
      if (L.n_keys > 1) for (int c = 0; c < L.n_keys; ++c) put64(out + c * L.key_col_stride + i * 8, touched ? mkey_stored[c] : B2Q_I64_MAX);
      else put64(out + i * 8, touched ? ((i == L.null_idx) ? L.key_null_stored : key) : B2Q_I64_MAX);
    } else if (L.has_key_col && L.n_keys > 1) {
      for (int c = 0; c < L.n_keys; ++c) put64(row + c * 8, touched ? mkey_stored[c] : B2Q_I64_MAX);
    } else if (L.has_key_col) {
      if (L.key_width == 4) { put32(row, touched ? static_cast<int32_t>(key) : 0x7FFFFFFF); put32(row + 4, 0); }
      else put64(row, touched ? ((i == L.null_idx) ? L.key_null_stored : key) : B2Q_I64_MAX);
    }
    int64_t vals[B2Q_MAX_SLOTS];
    for (int s = 0; s < L.n_slots; ++s) {
      const DevSlot& sl = L.slots[s];
      int64_t val = sl.init_val;
      if (touched && sl.kind != SLOT_NONE && sl.width != 0) {
        switch (sl.kind) {
          case SLOT_KEY: val = L.n_keys > 1 ? mkey_proj[sl.key_comp] : key; break;
          case SLOT_COUNT: val = accs[sl.acc][i]; break;
          case SLOT_BITCOUNT: {
            int64_t nbits = 0;
            for (int k = 0; k < sl.bm_words; ++k) nbits += __builtin_popcount(bitmaps[sl.acc][static_cast<size_t>(i) * sl.bm_words + k]);
            val = nbits;
            break;
          }
          default: {
            const int64_t raw = accs[sl.acc][i];
            bool is_null = false;
            if (sl.nn >= 0) is_null = accs[sl.nn][i] == 0;
            else if (sl.nn == -2) is_null = raw == sl.identity || (sl.clamp_init && b2q_clamp_ord(raw, sl.identity, sl.as_float) != raw);
            val = is_null ? sl.init_val : (sl.kind == SLOT_VALUE_ORD ? b2q_ord_to_f64(raw) : (sl.scale_day ? raw * 86400 : raw));
            if (sl.as_float && !is_null) { /* as b2q_k_materialize: float image in the low word, init pattern's high word */
              const float f = static_cast<float>(as_double(val));
              uint32_t fb; memcpy(&fb, &f, 4);
              val = (sl.init_val & static_cast<int64_t>(0xFFFFFFFF00000000ll)) | static_cast<int64_t>(fb);
            }
          }
        }
      }
      vals[s] = val;
    }
    if (L.keyless_marker >= 0 && vals[L.keyless_marker] == L.slots[L.keyless_marker].init_val)
      for (int s = 0; s < L.n_slots; ++s) vals[s] = L.slots[s].init_val;
    if (L.columnar) {
      for (int s = 0; s < L.n_slots; ++s) {
        const DevSlot& sl = L.slots[s];
        if (sl.kind == SLOT_NONE || sl.width == 0) continue;
        if (sl.width == 4) put32(out + sl.offset + i * 4, static_cast<int32_t>(vals[s])); else put64(out + sl.offset + i * 8, vals[s]);
      }
      continue;
    }
    int end = 0;
    for (int s = 0; s < L.n_slots; ++s) {
      const DevSlot& sl = L.slots[s];
      if (sl.kind == SLOT_NONE || sl.width == 0) continue;
      if (sl.width == 4) put32(row + sl.offset, static_cast<int32_t>(vals[s])); else put64(row + sl.offset, vals[s]);
      end = std::max(end, static_cast<int>(sl.offset) + sl.width);
    }
    if (end) for (; end + 4 <= L.row_size; end += 4) put32(row + end, 0);
  }
  return 0;
}

/* The join table layout the planner chose for a query, with the shared-memory sizes its choice rests on:
 * out = {B2Q_JOIN_TABLE_* value, smem.use_smem, smem.replica_bytes, smem.replicas, smem.join_bytes}.  The value is derived
 * from the program and the shared-memory plan the way executor.cpp's join_table_kind does. */
extern "C" int32_t b2q_test_join_layout(const B2QQuery* q, int64_t* out) {
  if (!q || !out) return -1;
  const DevJoin& j = q->prog.join;
  int64_t kind = B2Q_JOIN_TABLE_NONE;
  if (j.fk_col >= 0) {
    if (q->smem.join_off < 0) kind = j.packed_col >= 0 ? B2Q_JOIN_TABLE_INT2_HBM : B2Q_JOIN_TABLE_INT32_HBM;
    else kind = j.slot16 ? B2Q_JOIN_TABLE_UINT16_SMEM : j.packed_col >= 0 ? B2Q_JOIN_TABLE_INT2_SMEM : B2Q_JOIN_TABLE_INT32_SMEM;
  }
  out[0] = kind;
  out[1] = q->smem.use_smem;
  out[2] = q->smem.replica_bytes;
  out[3] = q->smem.replicas;
  out[4] = q->smem.join_bytes;
  return 0;
}
