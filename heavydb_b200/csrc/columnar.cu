/*
 * columnar.cu — ColumnarResults in device memory (b2q_rs_device_columns) and its Arrow C Device Data Interface export.
 *
 * The reference hands a result to the next step or to a client as ColumnarResults (QueryEngine/ColumnarResults.cpp:256-392)
 * and, for sql_execute_gdf, as Arrow buffers in device memory (the GPU branch of ArrowResultSetConverter,
 * ArrowResultSetConverter.cpp:595, device-specific types :1147).  Here the same columns are made on the device from the
 * reference-layout buffer the materialise kernel wrote, without a round trip over PCIe:
 *   1. the entries the iteration visits: the ordered compaction of non-empty entries of sort.cu (compact_entries), or
 *      the result set's permutation when it is sorted; then the dropFirstN / keepFirstN window
 *   2. one conversion kernel: thread r decodes row r with the host reader's own per-slot code (b2q_read_target,
 *      b2q_internal.h), writes every target at its width, an Arrow validity word per 32 rows (__ballot_sync) and, for
 *      DECIMAL targets, the decimal128 image Arrow wants.  The buffer is read once and every column written once.
 *      The same pass keeps each column's chunk stats (synthesize_metadata, InputMetadata.cpp:381-470): every value is
 *      mapped to an order-preserving unsigned key, a warp takes the min / max key with __reduce_max_sync, a CTA with a
 *      shared-memory atomic and the grid with one global atomic per column; the keys ride the NULL-count copy back.
 */
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cfloat>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/b2q_arrow.h"
#include "b2q_internal.h"

namespace b2q {
int sm_count();
size_t compact_scratch_bytes(int64_t entries);
cudaError_t compact_entries(const DevSortLayout& L, const int8_t* buf, uint32_t* block_counts, uint32_t* perm, uint32_t* d_total,
                            cudaStream_t st, int64_t* n_out);
int32_t report_error(int32_t code, const std::string& msg); /* executor.cpp: sets the thread's last error message */
bool device_present();
}  // namespace b2q

using namespace b2q;

namespace {

struct DevColumnsOut {
  int8_t* values[B2Q_MAX_TARGETS];
  uint32_t* validity[B2Q_MAX_TARGETS];
  int8_t* dec128[B2Q_MAX_TARGETS]; /* DECIMAL targets: 16 bytes per row, the int64 sign-extended; else nullptr */
  int64_t null_bits[B2Q_MAX_TARGETS];
  int8_t width[B2Q_MAX_TARGETS];
  int8_t is_fp[B2Q_MAX_TARGETS];
  int32_t n_cols;
};

constexpr int COL_BLOCK = 256;
constexpr uint64_t SIGN64 = 0x8000000000000000ull;

/* Order-preserving keys of a stored value (bits as b2q_store_target returns them): signed integers with the sign bit
 * flipped, IEEE floats with every bit flipped when negative and the sign bit flipped otherwise (-0 sorts below +0).
 * Columns of 4 bytes or less use 32-bit keys, 8-byte columns 64-bit ones. */
__host__ __device__ inline uint32_t key32(int64_t bits, bool fp) {
  const uint32_t b = static_cast<uint32_t>(bits);
  return fp && (b >> 31) ? ~b : b ^ 0x80000000u;
}
__host__ __device__ inline uint64_t key64(int64_t bits, bool fp) {
  const uint64_t b = static_cast<uint64_t>(bits);
  return fp && (b >> 63) ? ~b : b ^ SIGN64;
}

/* the largest key of the warp; the 64-bit one as its high word, then the low word among the lanes that hold that high word */
__device__ inline uint64_t warp_max_key(uint64_t k, bool wide) {
  if (!wide) return __reduce_max_sync(~0u, static_cast<uint32_t>(k));
  const uint32_t hi = __reduce_max_sync(~0u, static_cast<uint32_t>(k >> 32));
  const uint32_t lo = __reduce_max_sync(~0u, static_cast<uint32_t>(k >> 32) == hi ? static_cast<uint32_t>(k) : 0u);
  return (static_cast<uint64_t>(hi) << 32) | lo;
}

/* row r of the output = entry entries[first + r] (or first + r when every entry is visited in order) */
__global__ void __launch_bounds__(COL_BLOCK) b2q_k_device_columns(const __grid_constant__ B2QPlan p, const int8_t* __restrict__ buf,
                                                                 const uint32_t* __restrict__ entries, int64_t first, int64_t n,
                                                                 const __grid_constant__ DevColumnsOut o,
                                                                 unsigned long long* __restrict__ null_counts) {
  /* null_counts[c]; then per column the complement of its smallest key and its largest key, both 0 when no value
   * entered the range (a NULL or a NaN never does) */
  unsigned long long* const neg_min_keys = null_counts + B2Q_MAX_TARGETS;
  unsigned long long* const max_keys = null_counts + 2 * B2Q_MAX_TARGETS;
  __shared__ unsigned int s_nulls[B2Q_MAX_TARGETS];
  __shared__ unsigned long long s_neg_min[B2Q_MAX_TARGETS], s_max[B2Q_MAX_TARGETS];
  if (threadIdx.x < B2Q_MAX_TARGETS) {
    s_nulls[threadIdx.x] = 0;
    s_neg_min[threadIdx.x] = 0;
    s_max[threadIdx.x] = 0;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t n_round = (n + 31) & ~int64_t(31); /* whole warps stay in the loop for the ballots */
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_round; r += stride) {
    const bool in = r < n;
    const int64_t e = in ? (entries ? (int64_t)entries[first + r] : first + r) : 0;
    const unsigned in_mask = __ballot_sync(~0u, in);
    for (int c = 0; c < o.n_cols; ++c) {
      bool valid = false;
      const bool wide = o.width[c] == 8;
      uint64_t neg_min = 0, mx = 0;
      if (in) {
        B2QTargetValue v;
        b2q_read_target(p, buf, e, c, false, &v); /* decimals stay scaled int64, as in ColumnarResults */
        const int w = o.width[c];
        const int64_t bits = b2q_store_target(v, w, o.values[c] + r * w);
        valid = bits != o.null_bits[c];
        if (o.dec128[c]) {
          int64_t* d = reinterpret_cast<int64_t*>(o.dec128[c] + r * 16);
          d[0] = bits;
          d[1] = bits >> 63;
        }
        /* NoneEncoder::updateStats: std::min / std::max never take a NaN */
        const bool nan = o.is_fp[c] && (wide ? (static_cast<uint64_t>(bits) << 1) > (0x7FF0000000000000ull << 1)
                                             : (static_cast<uint32_t>(bits) << 1) > (0x7F800000u << 1));
        if (valid && !nan) {
          mx = wide ? key64(bits, o.is_fp[c]) : key32(bits, o.is_fp[c]);
          neg_min = wide ? ~mx : ~static_cast<uint32_t>(mx);
        }
      }
      const unsigned vm = __ballot_sync(~0u, valid);
      neg_min = warp_max_key(neg_min, wide);
      mx = warp_max_key(mx, wide);
      if (lane == 0) {
        o.validity[c][r >> 5] = vm;
        const unsigned nulls = __popc(in_mask & ~vm);
        if (nulls) atomicAdd(&s_nulls[c], nulls);
        if (neg_min) atomicMax(&s_neg_min[c], (unsigned long long)neg_min);
        if (mx) atomicMax(&s_max[c], (unsigned long long)mx);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x < o.n_cols) {
    const int c = threadIdx.x;
    if (s_nulls[c]) atomicAdd(&null_counts[c], (unsigned long long)s_nulls[c]);
    if (s_neg_min[c]) atomicMax(&neg_min_keys[c], s_neg_min[c]);
    if (s_max[c]) atomicMax(&max_keys[c], s_max[c]);
  }
}

/* synthesize_metadata of one column from its reduced keys: a fresh NoneEncoder<T>'s stats (min = numeric_limits<T>::max(),
 * max = lowest()) where no value entered the range.  A key of 0 never belongs to a value except the smallest key's
 * complement of INT32_MAX / INT64_MAX, which then decodes to that same limit. */
B2QChunkStats chunk_stats_from_keys(const B2QTypeInfo& ti, uint64_t neg_min, uint64_t max_key, int64_t null_count) {
  B2QChunkStats s;
  memset(&s, 0, sizeof(s));
  s.has_nulls = null_count > 0;
  const int t = ti.type;
  if (t == B2Q_kDOUBLE || t == B2Q_kFLOAT) {
    auto fp = [&](uint64_t k) {
      if (t == B2Q_kDOUBLE) { const uint64_t b = (k >> 63) ? k ^ SIGN64 : ~k; double d; memcpy(&d, &b, 8); return d; }
      const uint32_t k32 = static_cast<uint32_t>(k), b = (k32 >> 31) ? k32 ^ 0x80000000u : ~k32;
      float f; memcpy(&f, &b, 4);
      return static_cast<double>(f);
    };
    const double lim = t == B2Q_kDOUBLE ? DBL_MAX : static_cast<double>(FLT_MAX);
    s.fp_min = neg_min ? fp(t == B2Q_kDOUBLE ? ~neg_min : static_cast<uint32_t>(~neg_min)) : lim;
    s.fp_max = max_key ? fp(max_key) : -lim;
    return s;
  }
  const int w = b2q_type_size(t);
  const int64_t hi = w == 1 ? INT8_MAX : w == 2 ? INT16_MAX : w == 4 ? INT32_MAX : INT64_MAX;
  auto val = [&](uint64_t k) {
    return w == 8 ? static_cast<int64_t>(k ^ SIGN64) : static_cast<int64_t>(static_cast<int32_t>(static_cast<uint32_t>(k) ^ 0x80000000u));
  };
  s.int_min = neg_min ? val(w == 8 ? ~neg_min : static_cast<uint32_t>(~neg_min)) : hi;
  s.int_max = max_key ? val(max_key) : -hi - 1;
  return s;
}

size_t pad256(size_t n) { return (n + 255) & ~size_t(255); }

/* The device memory of one conversion.  Owned jointly by the B2QDeviceColumns handle and every node of an exported Arrow
 * array; the last owner frees it. */
struct DcShared {
  std::atomic<int> refs{1};
  int device = 0;
  int8_t* base = nullptr;       /* one stream-ordered allocation: every column, bitmap, decimal128 buffer */
  cudaEvent_t done = nullptr;   /* recorded after the conversion (ArrowDeviceArray::sync_event points here) */
};

/* on_release: the owner is an Arrow array whose consumer gave no stream — free after the conversion and after whatever
 * the legacy default stream is ordered behind (every blocking stream of the device) */
void dc_unref(DcShared* s, cudaStream_t st, bool on_release) {
  if (--s->refs > 0) return;
  int cur = -1;
  cudaGetDevice(&cur);
  if (cur != s->device) cudaSetDevice(s->device);
  if (on_release) {
    st = cudaStreamLegacy;
    if (s->done) cudaStreamWaitEvent(st, s->done, 0);
  }
  if (s->base) cudaFreeAsync(s->base, st);
  if (s->done) cudaEventDestroy(s->done);
  if (cur >= 0 && cur != s->device) cudaSetDevice(cur);
  cudaGetLastError();
  delete s;
}

}  // namespace

struct B2QDeviceColumns {
  DcShared* sh = nullptr;
  size_t n = 0;
  int nt = 0;
  double convert_ms = 0;
  B2QTypeInfo types[B2Q_MAX_TARGETS];
  int width[B2Q_MAX_TARGETS];
  int8_t* values[B2Q_MAX_TARGETS];
  uint32_t* validity[B2Q_MAX_TARGETS];
  int8_t* dec128[B2Q_MAX_TARGETS];
  int64_t null_count[B2Q_MAX_TARGETS];
  B2QChunkStats stats[B2Q_MAX_TARGETS];
};

namespace {

/* ---- Arrow export ------------------------------------------------------------------------------------------------ */
struct SchemaPriv {
  std::string format, name;
  std::vector<ArrowSchema> child_storage;
  std::vector<ArrowSchema*> child_ptrs;
};
void schema_release(ArrowSchema* s) {
  if (!s || !s->release) return;
  for (int64_t i = 0; i < s->n_children; ++i)
    if (s->children[i] && s->children[i]->release) s->children[i]->release(s->children[i]);
  delete static_cast<SchemaPriv*>(s->private_data);
  s->release = nullptr;
}

struct ArrayPriv {
  DcShared* sh = nullptr;
  const void* buffers[2] = {nullptr, nullptr};
  std::vector<ArrowArray> child_storage;
  std::vector<ArrowArray*> child_ptrs;
};
void array_release(ArrowArray* a) {
  if (!a || !a->release) return;
  for (int64_t i = 0; i < a->n_children; ++i) /* children not moved out by the consumer */
    if (a->children[i] && a->children[i]->release) a->children[i]->release(a->children[i]);
  ArrayPriv* pr = static_cast<ArrayPriv*>(a->private_data);
  DcShared* sh = pr->sh;
  delete pr;
  a->release = nullptr;
  dc_unref(sh, nullptr, true);
}

/* the format ResultSet.toArrow() / ArrowResultSetConverter gives a column of this type */
std::string arrow_format(const B2QTypeInfo& t) {
  switch (t.type) {
    case B2Q_kTINYINT: return "c";
    case B2Q_kSMALLINT: return "s";
    case B2Q_kFLOAT: return "f";
    case B2Q_kDOUBLE: return "g";
    case B2Q_kDECIMAL: case B2Q_kNUMERIC: return "d:19," + std::to_string(t.scale); /* the precision is not carried: 19 digits hold every int64 */
    default: return b2q_type_size(t.type) == 4 ? "i" : "l"; /* INT, dictionary ids; BIGINT and the TIME family */
  }
}

}  // namespace

extern "C" {

int32_t b2q_rs_device_columns(const B2QResultSet* rs, void* stream, B2QDeviceColumns** out) {
  RsSource src;
  if (!out || !rs_source(rs, &src)) return report_error(B2Q_ERR_INVALID_ARGUMENT, "null argument");
  const B2QPlan& p = *src.plan;
  if (p.query_desc_type == B2Q_Estimator) return report_error(B2Q_ERR_UNSUPPORTED, "an estimator result has no rows");
  if (!device_present()) return report_error(B2Q_ERR_NO_DEVICE, "no CUDA device visible; this path has no CPU fallback");
  const int nt = p.num_targets;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int caller = -1;
  cudaGetDevice(&caller);
  int device = src.device >= 0 ? src.device : caller;
  if (device < 0) device = 0;
  if (device != caller && cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return report_error(B2Q_ERR_CUDA, "cudaSetDevice"); }
  std::vector<void*> temps; /* freed stream-ordered after the conversion */
  DcShared* sh = new DcShared();
  sh->device = device;
  B2QDeviceColumns* dc = new B2QDeviceColumns();
  dc->sh = sh;
  dc->nt = nt;
  cudaEvent_t ev0 = nullptr;
  cudaError_t e = cudaSuccess;
  auto fail = [&](int32_t code, const std::string& m) {
    cudaGetLastError();
    if (st) cudaStreamSynchronize(st); else cudaDeviceSynchronize();
    for (void* t : temps) cudaFreeAsync(t, st);
    if (ev0) cudaEventDestroy(ev0);
    b2q_device_columns_free(dc, stream);
    if (caller >= 0 && caller != device) cudaSetDevice(caller);
    cudaGetLastError();
    return report_error(code, m);
  };
  auto tmp = [&](size_t bytes, void** ptr) {
    e = cudaMallocAsync(ptr, std::max<size_t>(bytes, 16), st);
    if (e == cudaSuccess) temps.push_back(*ptr);
    return e == cudaSuccess;
  };
  /* the storage on the device: the result's own copy, or the host copy uploaded */
  const int8_t* d_buf = src.d_buf;
  if (!d_buf && src.buf_size) {
    void* up = nullptr;
    if (!tmp(src.buf_size, &up)) return fail(B2Q_ERR_OUT_OF_GPU_MEM, "device copy of the storage buffer");
    e = cudaMemcpyAsync(up, src.h_buf, src.buf_size, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return fail(B2Q_ERR_CUDA, std::string("storage upload: ") + cudaGetErrorString(e));
    d_buf = static_cast<const int8_t*>(up);
  }
  /* 1. the entries the iteration visits */
  const uint32_t* entries = nullptr;
  int64_t n_entries = 0;
  if (src.n_perm) {
    void* d_perm = nullptr;
    if (!tmp(src.n_perm * 4, &d_perm)) return fail(B2Q_ERR_OUT_OF_GPU_MEM, "permutation");
    e = cudaMemcpyAsync(d_perm, src.perm, src.n_perm * 4, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return fail(B2Q_ERR_CUDA, std::string("permutation upload: ") + cudaGetErrorString(e));
    entries = static_cast<const uint32_t*>(d_perm);
    n_entries = static_cast<int64_t>(src.n_perm); /* the sort's compaction already dropped the empty entries */
  } else if (src.buf_size && p.entry_count > 0) {
    void* scratch = nullptr;
    if (!tmp(compact_scratch_bytes(p.entry_count), &scratch)) return fail(B2Q_ERR_OUT_OF_GPU_MEM, "compaction scratch");
    const size_t nb = pad256((static_cast<size_t>(p.entry_count) + 2047) / 2048 * 4);
    uint32_t* block_counts = static_cast<uint32_t*>(scratch);
    uint32_t* perm = reinterpret_cast<uint32_t*>(static_cast<int8_t*>(scratch) + nb);
    uint32_t* d_total = reinterpret_cast<uint32_t*>(static_cast<int8_t*>(scratch) + nb + pad256(static_cast<size_t>(p.entry_count) * 4));
    e = compact_entries(sort_layout_for(p), d_buf, block_counts, perm, d_total, st, &n_entries);
    if (e != cudaSuccess) return fail(B2Q_ERR_CUDA, std::string("compaction: ") + cudaGetErrorString(e));
    entries = n_entries == p.entry_count ? nullptr : perm; /* every entry visited: row r is entry first + r */
  }
  const size_t total = static_cast<size_t>(n_entries);
  const size_t first = std::min(total, src.drop_first);
  size_t n = total - first;
  if (src.keep_first) n = std::min(n, src.keep_first);
  dc->n = n;
  /* 2. one allocation for every output buffer */
  const size_t words = (std::max<size_t>(n, 1) + 31) / 32;
  const size_t counters = static_cast<size_t>(B2Q_MAX_TARGETS) * 3 * 8; /* NULL counts, smallest-key complements, largest keys */
  size_t bytes = pad256(counters);
  for (int c = 0; c < nt; ++c) {
    dc->types[c] = b2q_target_col_type(p.targets[c]);
    dc->width[c] = b2q_type_size(dc->types[c].type);
    bytes += pad256(std::max<size_t>(n, 1) * dc->width[c]) + pad256(words * 4);
    if (b2q_is_decimal(dc->types[c].type)) bytes += pad256(std::max<size_t>(n, 1) * 16);
  }
  e = cudaMallocAsync(reinterpret_cast<void**>(&sh->base), bytes, st);
  if (e != cudaSuccess) { sh->base = nullptr; return fail(B2Q_ERR_OUT_OF_GPU_MEM, "device columns"); }
  int8_t* q = sh->base;
  unsigned long long* d_nulls = reinterpret_cast<unsigned long long*>(q);
  q += pad256(counters);
  DevColumnsOut o;
  memset(&o, 0, sizeof(o));
  o.n_cols = nt;
  for (int c = 0; c < nt; ++c) {
    dc->values[c] = q; q += pad256(std::max<size_t>(n, 1) * dc->width[c]);
    dc->validity[c] = reinterpret_cast<uint32_t*>(q); q += pad256(words * 4);
    dc->dec128[c] = nullptr;
    if (b2q_is_decimal(dc->types[c].type)) { dc->dec128[c] = q; q += pad256(std::max<size_t>(n, 1) * 16); }
    o.values[c] = dc->values[c];
    o.validity[c] = dc->validity[c];
    o.dec128[c] = dc->dec128[c];
    o.width[c] = static_cast<int8_t>(dc->width[c]);
    o.null_bits[c] = b2q_null_bits(dc->types[c].type);
    o.is_fp[c] = dc->types[c].type == B2Q_kDOUBLE || dc->types[c].type == B2Q_kFLOAT;
  }
  if (cudaEventCreate(&ev0) != cudaSuccess || cudaEventCreate(&sh->done) != cudaSuccess) return fail(B2Q_ERR_CUDA, "cudaEventCreate");
  e = cudaMemsetAsync(d_nulls, 0, counters, st);
  if (e == cudaSuccess) e = cudaEventRecord(ev0, st);
  if (e == cudaSuccess && n > 0 && nt > 0) {
    const int64_t blocks = std::min<int64_t>((static_cast<int64_t>(n) + COL_BLOCK - 1) / COL_BLOCK, static_cast<int64_t>(sm_count()) * 16);
    b2q_k_device_columns<<<static_cast<int>(std::max<int64_t>(blocks, 1)), COL_BLOCK, 0, st>>>(p, d_buf, entries, static_cast<int64_t>(first),
                                                                                               static_cast<int64_t>(n), o, d_nulls);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaEventRecord(sh->done, st);
  unsigned long long h_nulls[3 * B2Q_MAX_TARGETS] = {};
  if (e == cudaSuccess) e = cudaMemcpyAsync(h_nulls, d_nulls, counters, cudaMemcpyDeviceToHost, st);
  for (void* t : temps) cudaFreeAsync(t, st);
  temps.clear();
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(B2Q_ERR_CUDA, std::string("device columns: ") + cudaGetErrorString(e));
  float ms = 0;
  if (cudaEventElapsedTime(&ms, ev0, sh->done) == cudaSuccess) dc->convert_ms = ms;
  cudaEventDestroy(ev0);
  for (int c = 0; c < nt; ++c) {
    dc->null_count[c] = static_cast<int64_t>(h_nulls[c]);
    dc->stats[c] = chunk_stats_from_keys(dc->types[c], h_nulls[B2Q_MAX_TARGETS + c], h_nulls[2 * B2Q_MAX_TARGETS + c], dc->null_count[c]);
  }
  if (caller >= 0 && caller != device) cudaSetDevice(caller);
  cudaGetLastError();
  *out = dc;
  return B2Q_OK;
}

size_t b2q_device_columns_size(const B2QDeviceColumns* dc) { return dc ? dc->n : 0; }
size_t b2q_device_columns_num_columns(const B2QDeviceColumns* dc) { return dc ? static_cast<size_t>(dc->nt) : 0; }
int32_t b2q_device_columns_device(const B2QDeviceColumns* dc) { return dc ? dc->sh->device : -1; }
double b2q_device_columns_convert_ms(const B2QDeviceColumns* dc) { return dc ? dc->convert_ms : 0; }

const void* b2q_device_columns_column(const B2QDeviceColumns* dc, size_t col, B2QTypeInfo* ti, const uint32_t** validity, int64_t* null_count) {
  if (!dc || col >= static_cast<size_t>(dc->nt)) return nullptr;
  if (ti) *ti = dc->types[col];
  if (validity) *validity = dc->null_count[col] ? dc->validity[col] : nullptr;
  if (null_count) *null_count = dc->null_count[col];
  return dc->values[col];
}

int32_t b2q_device_columns_chunk_stats(const B2QDeviceColumns* dc, size_t col, B2QChunkStats* out) {
  if (!dc || !out || col >= static_cast<size_t>(dc->nt)) return report_error(B2Q_ERR_INVALID_ARGUMENT, "no such device column");
  *out = dc->stats[col];
  return B2Q_OK;
}

int32_t b2q_device_columns_export_arrow(B2QDeviceColumns* dc, const char* const* names, ArrowSchema* schema, ArrowDeviceArray* array) {
  if (!dc || !schema || !array) return report_error(B2Q_ERR_INVALID_ARGUMENT, "null argument");
  const int nt = dc->nt;
  SchemaPriv* sp = new SchemaPriv();
  sp->format = "+s";
  sp->child_storage.resize(nt);
  for (int c = 0; c < nt; ++c) {
    SchemaPriv* cp = new SchemaPriv();
    cp->format = arrow_format(dc->types[c]);
    cp->name = names && names[c] ? names[c] : "col" + std::to_string(c);
    ArrowSchema& s = sp->child_storage[c];
    s = ArrowSchema{cp->format.c_str(), cp->name.c_str(), nullptr, ARROW_FLAG_NULLABLE, 0, nullptr, nullptr, schema_release, cp};
    sp->child_ptrs.push_back(&s);
  }
  *schema = ArrowSchema{sp->format.c_str(), sp->name.c_str(), nullptr, 0, nt, nt ? sp->child_ptrs.data() : nullptr, nullptr, schema_release, sp};

  ArrayPriv* ap = new ArrayPriv();
  ap->sh = dc->sh;
  ap->child_storage.resize(nt);
  for (int c = 0; c < nt; ++c) {
    ArrayPriv* cp = new ArrayPriv();
    cp->sh = dc->sh;
    cp->buffers[0] = dc->null_count[c] ? dc->validity[c] : nullptr;
    cp->buffers[1] = dc->dec128[c] ? dc->dec128[c] : dc->values[c];
    ArrowArray& a = ap->child_storage[c];
    a = ArrowArray{static_cast<int64_t>(dc->n), dc->null_count[c], 0, 2, 0, cp->buffers, nullptr, nullptr, array_release, cp};
    ap->child_ptrs.push_back(&a);
  }
  dc->sh->refs += nt + 1;
  array->array = ArrowArray{static_cast<int64_t>(dc->n), 0, 0, 1, nt, ap->buffers, nt ? ap->child_ptrs.data() : nullptr, nullptr, array_release, ap};
  array->device_id = dc->sh->device;
  array->device_type = ARROW_DEVICE_CUDA;
  array->sync_event = &dc->sh->done;
  array->reserved[0] = array->reserved[1] = array->reserved[2] = 0;
  return B2Q_OK;
}

void b2q_device_columns_free(B2QDeviceColumns* dc, void* stream) {
  if (!dc) return;
  dc_unref(dc->sh, static_cast<cudaStream_t>(stream), false);
  delete dc;
}

}  // extern "C"
