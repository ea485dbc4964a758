/* TEST INFRASTRUCTURE — never linked into the product.
 *
 * The host reading of the lowered program (filter_emulator.cpp, included unchanged) extended by the set term that the planner
 * emits for an IN / NOT IN list past the leaf program (DevTerm::is_set, B2QQuery::set_values).  The set term is read as a
 * search in the term's value list, independently of the device's bitmap.  tests/test_in_list_cpu.py uses it.
 *
 * The whole-program entry points filter every row here, then hand filter_emulator.cpp's run_program_impl a copy of the query
 * whose filter is one term over an extra column holding that result, so that the accumulate / materialise reading is the
 * existing one. */
#include <cstddef>

#include "filter_emulator.cpp"

namespace {
/* membership in the sorted value list, inside [lo, lo + span] in the register class as the device tests it; a NULL row is never
 * TRUE when null_check */
bool eval_set_term(const DevTerm& t, const std::vector<int64_t>& values, const int8_t* col, int64_t row) {
  const int64_t v = load_int(col, t.width, row);
  bool in;
  if (t.width == 8) in = static_cast<uint64_t>(v) - static_cast<uint64_t>(t.lo) <= t.span;
  else in = static_cast<uint32_t>(static_cast<int32_t>(v)) - static_cast<uint32_t>(t.lo) <= static_cast<uint32_t>(t.span);
  in = in && std::binary_search(values.begin(), values.end(), v);
  bool r = in != static_cast<bool>(t.negate);
  if (t.null_check && v == (t.width == 8 ? t.null_bits : static_cast<int64_t>(static_cast<int32_t>(t.null_bits)))) r = false;
  return r;
}

/* eval_filter_impl with set terms: 1 / 0 = passes / fails, -1 = a program this reading does not take */
int32_t eval_filter_sets(const B2QQuery* q, const void* const* table_cols, int64_t row) {
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
      if (t.is_set) st[sp++] = eval_set_term(t, q->set_values[op & 15], c1, row);
      else st[sp++] = t.col2 >= 0 ? eval_term2(t, c1, static_cast<const int8_t*>(table_cols[q->col_ids[t.col2]]), row) : eval_term(t, c1, row);
    } else {
      if (sp < 2) return -1;
      const bool b = st[--sp], a = st[--sp];
      st[sp++] = kind == FOP_AND ? (a && b) : (a || b);
    }
  }
  return sp == 1 ? (st[0] ? 1 : 0) : -1;
}

/* the whole program with set terms: the filter's result per row becomes an int8 column after every column the query reads,
 * and a copy of the query filters on it with one range term [1, 1] */
int32_t run_program_sets(const B2QQuery* q, int32_t n_frags, const void* const* const* frag_cols, const int64_t* frag_rows,
                         const uint8_t* const* frag_valid, int8_t* out) {
  if (q->prog.n_cols >= B2Q_MAX_COLS) return -2;
  int n_table = 0;
  for (int c = 0; c < q->prog.n_cols; ++c) n_table = std::max(n_table, q->col_ids[c] + 1);
  std::vector<std::vector<int8_t>> pass(static_cast<size_t>(n_frags));
  std::vector<std::vector<const void*>> cols(static_cast<size_t>(n_frags));
  std::vector<const void* const*> frag_ptrs(static_cast<size_t>(n_frags));
  for (int f = 0; f < n_frags; ++f) {
    pass[f].resize(static_cast<size_t>(std::max<int64_t>(frag_rows[f], 1)));
    for (int64_t row = 0; row < frag_rows[f]; ++row) {
      const int32_t r = eval_filter_sets(q, frag_cols[f], row);
      if (r < 0) return -2;
      pass[f][static_cast<size_t>(row)] = static_cast<int8_t>(r);
    }
    cols[f].assign(frag_cols[f], frag_cols[f] + n_table);
    cols[f].push_back(pass[f].data());
    frag_ptrs[f] = cols[f].data();
  }
  B2QQuery Q = *q;
  DevFilter& fl = Q.prog.filter;
  memset(&fl, 0, sizeof(fl));
  DevTerm& t = fl.terms[0];
  t.col = Q.prog.n_cols;
  t.col2 = -1;
  t.width = 1;
  t.lo = 1;
  t.span = 0;
  Q.col_ids[Q.prog.n_cols++] = n_table;
  fl.n_terms = 1;
  fl.n_ops = 1;
  fl.ops[0] = static_cast<uint8_t>(FOP_TERM << 4);
  return run_program_impl(&Q, n_frags, frag_ptrs.data(), frag_rows, frag_valid, out);
}
}  // namespace

/* b2q_test_eval_filter / _joined with set terms (the same row semantics, join programs on denormalised rows) */
extern "C" int32_t b2q_test_eval_filter_sets(const B2QQuery* q, const void* const* table_cols, int64_t row) {
  return q ? eval_filter_sets(q, table_cols, row) : -1;
}

/* b2q_test_run_program / _joined with set terms (same arguments and results) */
extern "C" int32_t b2q_test_run_program_sets(const B2QQuery* q, int32_t n_frags, const void* const* const* frag_cols,
                                             const int64_t* frag_rows, int8_t* out) {
  if (!q || q->prog.join.fk_col >= 0) return -2;
  return run_program_sets(q, n_frags, frag_cols, frag_rows, nullptr, out);
}
extern "C" int32_t b2q_test_run_program_joined_sets(const B2QQuery* q, int32_t n_frags, const void* const* const* frag_cols,
                                                    const int64_t* frag_rows, const uint8_t* const* frag_valid, int8_t* out) {
  if (!q || q->prog.join.fk_col < 0) return -2;
  return run_program_sets(q, n_frags, frag_cols, frag_rows, frag_valid, out);
}

/* set terms of the lowered filter, and the values of set term number `k` (in term order): returns the count, copies at most
 * `cap` values to `out` */
extern "C" int32_t b2q_test_set_terms(const B2QQuery* q) {
  if (!q) return -1;
  int32_t n = 0;
  for (int t = 0; t < q->prog.filter.n_terms; ++t) n += q->prog.filter.terms[t].is_set ? 1 : 0;
  return n;
}
extern "C" int64_t b2q_test_set_values(const B2QQuery* q, int32_t k, int64_t* out, int64_t cap) {
  if (!q) return -1;
  for (int t = 0; t < q->prog.filter.n_terms; ++t) {
    if (!q->prog.filter.terms[t].is_set || k-- != 0) continue;
    const std::vector<int64_t>& v = q->set_values[t];
    for (int64_t i = 0; i < cap && i < static_cast<int64_t>(v.size()); ++i) out[i] = v[static_cast<size_t>(i)];
    return static_cast<int64_t>(v.size());
  }
  return -1;
}

/* The filter program's bytes as they were before set terms existed: term count, op count, the ops, and every term up to
 * (not including) DevTerm::set_bits.  `out` receives at most `cap` bytes; returns the length. */
extern "C" int64_t b2q_test_filter_bytes(const B2QQuery* q, uint8_t* out, int64_t cap) {
  if (!q) return -1;
  const DevFilter& f = q->prog.filter;
  std::vector<uint8_t> b;
  auto put = [&](const void* p, size_t n) { b.insert(b.end(), static_cast<const uint8_t*>(p), static_cast<const uint8_t*>(p) + n); };
  put(&f.n_terms, 4);
  put(&f.n_ops, 4);
  put(f.ops, static_cast<size_t>(f.n_ops));
  for (int t = 0; t < f.n_terms; ++t) put(&f.terms[t], offsetof(DevTerm, set_bits));
  for (size_t i = 0; i < b.size() && static_cast<int64_t>(i) < cap; ++i) out[i] = b[i];
  return static_cast<int64_t>(b.size());
}
