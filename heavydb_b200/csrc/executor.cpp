/*
 * executor.cpp — host side of the path and the C ABI of include/b2q.h.
 *
 * Mirrors, for the one path in scope, what sits between Executor::executeWorkUnit and the result set in the
 * reference:
 *   executeWorkUnitImpl / createKernels / launchKernels      QueryEngine/Execute.cpp:2213-2399,3028,3158
 *   fetchChunks (column pointers; H2D when not resident)      QueryEngine/Execute.cpp:3581, ColumnFetcher.cpp:214-288
 *   launchGpuCode (param block, init, launch, copy back)      QueryEngine/QueryExecutionContext.cpp:211-582
 *   per-block / per-device reduction                          Execute.cpp:1696,1772; ResultSetReduction.cpp:203-396
 *     -> here: CTA tables are merged on the device into one dense table; devices merge by all-reduce of that table
 *   ResultSet iteration                                       QueryEngine/ResultSetIteration.cpp:2086-2220,2457-2492
 *
 * There is no CPU execution path in this file: every compute entry needs a CUDA device.
 */
#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <mutex>
#include <numeric>
#include <string>
#include <thread>
#include <vector>

#include "b2q_internal.h"
#include "multi.h"
#include "radix_agg.h"

namespace b2q {
int32_t make_query(const B2QExecUnit* u, const B2QTableInfo* t, const B2QExecutionOptions* eo, size_t guess,
                   bool has_card, bool filter_deleted, B2QQuery* out, std::string* err);
int scan_rows_per_chunk(int block);
void scan_config(const B2QQuery& q, int* block, int* ctas_per_sm);
cudaError_t launch_scan(const B2QQuery& q, const DevLaunch& launch, const int8_t* smem_image, int block, int ctas_per_sm,
                        cudaStream_t st);
cudaError_t launch_init(const B2QQuery& q, int64_t* const* accs, int64_t* keys, int8_t* smem_image, cudaStream_t st);
cudaError_t launch_join_build(const int8_t* keys, int width, int64_t n_rows, int64_t min_key, int64_t entry_count, int nullable,
                              int64_t null_val, int32_t* buff, int32_t* error, const int8_t* packed_vals, int packed_width,
                              cudaStream_t st);
cudaError_t launch_materialize(const B2QQuery& q, const int64_t* const* accs, const int64_t* keys, int8_t* out,
                               cudaStream_t st);
cudaError_t launch_join_split(const int64_t* split, int64_t* out, int64_t n, cudaStream_t st);
cudaError_t launch_gen(void* dst, int sql_type, uint64_t seed, uint32_t col_tag, int64_t row0, int64_t count, int64_t lo,
                       int64_t span, int64_t stride, cudaStream_t st);
cudaError_t launch_join_slot16(const int32_t* rows, int64_t entry_count, const int8_t* vals, int width, int64_t null_val, int64_t vmin,
                               uint16_t* out, int32_t* error, cudaStream_t st);
cudaError_t launch_bitmap_or(uint64_t* dst, const uint64_t* gathered, int64_t words, int copies, cudaStream_t st);
size_t sort_scratch_bytes(int64_t entries);
cudaError_t sort_device(const DevSortLayout& L, const DevSortKey* keys, int n_keys, const int8_t* buf, int8_t* scratch,
                        cudaStream_t st, const uint32_t** perm_out, int64_t* n_out, int* launches, int64_t top_n,
                        const volatile uint32_t* stop, bool* stopped);
cudaError_t sort_gather(const DevSortLayout& Lin, const DevGatherCols& G, const int8_t* in, int8_t* out, const uint32_t* perm,
                        int64_t first, int64_t n_out, cudaStream_t st);
int project_rows_per_chunk();
cudaError_t launch_project(const B2QQuery& q, const int8_t* const* col_ptrs, const int64_t* frag_rows, const int64_t* frag_chunk_start,
                           const int64_t* frag_row_base, int n_frags, int64_t total_chunks, int64_t chunk_base, int8_t* out,
                           int64_t row_size, int64_t cap, unsigned long long* status, unsigned long long* ticket,
                           unsigned long long* counters, int32_t* error, const DevInterrupt& intr, cudaStream_t st);
cudaError_t launch_watchdog_start(uint64_t* t0, cudaStream_t st);
cudaError_t launch_set_error(int32_t* error, int32_t code, cudaStream_t st);
size_t set_bytes(const B2QQuery& q);
cudaError_t build_sets(B2QQuery& q, int8_t* blk, int* launches, cudaStream_t st);
}  // namespace b2q

using namespace b2q;

static thread_local std::string g_err;

static int32_t set_err(int32_t code, const std::string& m) {
  g_err = m;
  return code;
}
#define CU(call)                                                                                               \
  do {                                                                                                         \
    cudaError_t e__ = (call);                                                                                  \
    if (e__ != cudaSuccess) {                                                                                  \
      cudaGetLastError();                                                                                      \
      return set_err(e__ == cudaErrorMemoryAllocation ? B2Q_ERR_OUT_OF_GPU_MEM : B2Q_ERR_CUDA,                 \
                     std::string(#call) + ": " + cudaGetErrorString(e__));                                     \
    }                                                                                                          \
  } while (0)

static bool have_device() {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return false; }
  return n > 0;
}

/* B2Q_TRACE=1: wall-clock marks of one b2q_execute_work_unit call on stderr (where the host side of a step goes) */
struct CallTrace {
  bool on = false;
  std::chrono::steady_clock::time_point last;
  std::string line;
  void begin() {
    static const bool knob = []() { const char* e = getenv("B2Q_TRACE"); return e && atoi(e) != 0; }();
    on = knob;
    line.clear();
    last = std::chrono::steady_clock::now();
  }
  void mark(const char* what) {
    if (!on) return;
    const auto now = std::chrono::steady_clock::now();
    char buf[96];
    snprintf(buf, sizeof(buf), " %s %.0f us |", what, std::chrono::duration<double, std::micro>(now - last).count());
    line += buf;
    last = now;
  }
  void end() { if (on) fprintf(stderr, "[b2q]%s\n", line.c_str()); on = false; }
};
static thread_local CallTrace g_trace;

/* ---------------------------------------------------------------------------------------------------------- */
/* All device memory of one query comes from the CUDA stream-ordered pool in ONE allocation (the pool keeps freed
 * memory, so steady-state calls do not touch the driver's allocator — the reference re-uses its CudaMgr slabs
 * the same way, DataMgr/BufferMgr/GpuCudaBufferMgr). */
static void configure_pool_once(int device) {
  static std::mutex mu;
  static bool done[64] = {};
  std::lock_guard<std::mutex> g(mu);
  if (device < 0 || device >= 64 || done[device]) return;
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    unsigned long long thr = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  cudaGetLastError();
  done[device] = true;
}

struct DeviceBlock {
  int8_t* base = nullptr;
  size_t size = 0;
  size_t used = 0;
  cudaError_t alloc(size_t n, cudaStream_t st) {
    size = n;
    used = 0;
    return cudaMallocAsync(reinterpret_cast<void**>(&base), n, st);
  }
  static size_t pad(size_t n) { return (n + 255) & ~size_t(255); }
  int8_t* take(size_t n) {
    int8_t* p = base + used;
    used += pad(n);
    return p;
  }
  void release(cudaStream_t st) {
    if (base) cudaFreeAsync(base, st);
    base = nullptr;
  }
};

/* ---- stopping a running call: interrupt token and dynamic watchdog (B2QExecutionOptions) ------------------------------
 * The token's flag is pinned host memory, mapped into every device's address space (portable): the host stores into it, the
 * kernels read it with a relaxed system-scope load (interrupt_poll, scan_kernel.cuh). */
struct B2QInterruptToken {
  uint32_t* flag = nullptr;        /* host pointer == device pointer (unified addressing) */
};

/* What one call checks, made from its B2QExecutionOptions once the call's device and stream are known.  The watchdog's start
 * time lives in one device word written by the call's first kernel (b2q_k_watchdog_start); every checking kernel of the call
 * compares %globaltimer with it, so the budget covers the call's device work as a whole.  Shared by the partial(s) of the call
 * (a radix retry, a projection's pre-flight count) so that the budget does not restart. */
struct CallInterrupt {
  DevInterrupt dev = {};                        /* what the kernels check */
  const volatile uint32_t* host_flag = nullptr; /* the token as the host reads it between steps */
  bool watchdog = false;
  uint64_t* d_t0 = nullptr;
  int device = -1;
  cudaStream_t stream = nullptr;
  bool enabled() const { return dev.flag != nullptr || watchdog; }
  bool interrupted() const { return host_flag && *host_flag; }
  static std::shared_ptr<CallInterrupt> from(const B2QExecutionOptions* eo) {
    auto c = std::make_shared<CallInterrupt>();
    if (eo && eo->allow_runtime_query_interrupt && eo->interrupt_token && eo->interrupt_token->flag) {
      c->host_flag = eo->interrupt_token->flag;
      c->dev.flag = eo->interrupt_token->flag;
    }
    if (eo && eo->with_dynamic_watchdog) {
      c->watchdog = true;
      c->dev.budget_ns = static_cast<uint64_t>(eo->dynamic_watchdog_time_limit) * 1000000ull;
    }
    return c;
  }
  /* on the call's device, before its first kernel: the watchdog's start word (once per call) */
  cudaError_t start(int dev_id, cudaStream_t st) {
    if (!watchdog || d_t0) return cudaSuccess;
    device = dev_id;
    stream = st;
    cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&d_t0), sizeof(uint64_t), st);
    if (e != cudaSuccess) { d_t0 = nullptr; return e; }
    dev.t0 = d_t0;
    return launch_watchdog_start(d_t0, st);
  }
  /* Execute.cpp:2319-2324: a query that was interrupted and also ran out of time reports INTERRUPTED */
  int32_t resolve(int32_t rc) const {
    if (rc == B2Q_ERR_OUT_OF_TIME && watchdog && interrupted()) return B2Q_ERR_INTERRUPTED;
    return rc;
  }
  ~CallInterrupt() {
    if (!d_t0) return;
    int cur = -1;
    cudaGetDevice(&cur);
    if (cur != device) cudaSetDevice(device);
    cudaFreeAsync(d_t0, stream);
    if (cur >= 0 && cur != device) cudaSetDevice(cur);
    cudaGetLastError();
  }
};
static const DevInterrupt kNoInterrupt = {nullptr, nullptr, 0};

/* wall-clock phases of a host-resident stream (stream_host_table) */
struct HostPhases {
  double setup_us = 0, stream_us = 0, teardown_us = 0;
};

struct B2QPartial {
  B2QQuery q;
  int device = 0;
  std::shared_ptr<CallInterrupt> intr; /* never null for a partial of b2q_execute_*; null for b2q_launch */
  DeviceBlock blk;
  int64_t* accs[B2Q_MAX_ACCS] = {};
  int64_t* keys = nullptr;
  int8_t* smem_image = nullptr;
  int32_t* d_error = nullptr;
  std::vector<void*> extra;  /* stream-ordered allocations made after the main block */
  /* join level: the one-to-one table and, per launch column, the device copy of an inner-table column (else nullptr) */
  const int32_t* join_buff = nullptr;
  const int8_t* inner_cols[B2Q_MAX_COLS] = {};
  bool split = false;        /* COUNT / SUM_I64 arrays are in the (lo[n] | hi[n]) layout of the global-table kernels */
  bool result_on_device = false; /* B2QExecutionOptions::result_on_device: finalize keeps the result in device memory */
  /* baseline hash as a two-pass radix-partitioned aggregation (radix_agg.cu); buffers sized for `radix_batch_chunks` chunks a launch */
  bool radix = false;
  RadixPlan rp;
  RadixBuffers rb = {};
  int64_t radix_batch_chunks = 0;
  int radix_n_cta1 = 0;
  uint32_t radix_cap = 0;
  cudaStream_t stream = nullptr; /* the stream the work was enqueued on: frees are ordered after it */
  /* deferred completion (single-sync calls): the device error word is copied into this pinned word on the stream and read
   * after the call's one synchronize at the end of finalize */
  bool deferred = false;
  int32_t* h_err = nullptr;
  size_t h_err_cap = 0;
  cudaEvent_t ev[4] = {}; /* init begin/end, scan begin/end */
  bool scan_timed = false;
  double scan_ms = 0, init_ms = 0, h2d_bytes = 0;
  HostPhases host;
  int64_t launches = 0, frags_scanned = 0, frags_skipped = 0;
  ~B2QPartial() {
    /* Kernels may still be running on `stream` (error paths return before the synchronize), and the caller's current
     * device may be another one: free on the owning device, in the order of the stream the work was enqueued on. */
    int cur = -1;
    cudaGetDevice(&cur);
    if (cur != device) cudaSetDevice(device);
    for (void* x : extra) cudaFreeAsync(x, stream);
    blk.release(stream);
    for (auto& e : ev) if (e) cudaEventDestroy(e);
    if (cur >= 0 && cur != device) cudaSetDevice(cur);
    cudaGetLastError();
    release_h_err();
  }
  void release_h_err();
  bool stream_busy() const { return cudaStreamQuery(stream) == cudaErrorNotReady; }
};

/* Result buffers are page-locked host memory so the copy-back is one asynchronous DMA at PCIe rate straight into
 * the buffer the ResultSet owns.  Page-locking is expensive, so released buffers are kept in a small
 * cache and handed to the next result of a similar size. */
struct PinnedCache {
  struct Item { int8_t* p; size_t cap; };
  std::mutex mu;
  std::vector<Item> free_list;
  size_t cached_bytes = 0;
  static constexpr size_t kMaxCached = size_t(2) << 30;
  int8_t* get(size_t n, size_t* cap_out) {
    {
      std::lock_guard<std::mutex> g(mu);
      int best = -1;
      for (size_t i = 0; i < free_list.size(); ++i)
        if (free_list[i].cap >= n && free_list[i].cap <= 2 * n + (1 << 20) && (best < 0 || free_list[i].cap < free_list[best].cap)) best = static_cast<int>(i);
      if (best >= 0) {
        Item it = free_list[best];
        free_list.erase(free_list.begin() + best);
        cached_bytes -= it.cap;
        *cap_out = it.cap;
        return it.p;
      }
    }
    int8_t* p = nullptr;
    const size_t cap = std::max<size_t>(n, 4096);
    if (cudaHostAlloc(reinterpret_cast<void**>(&p), cap, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    *cap_out = cap;
    return p;
  }
  void put(int8_t* p, size_t cap) {
    if (!p) return;
    std::lock_guard<std::mutex> g(mu);
    if (cached_bytes + cap > kMaxCached) { cudaFreeHost(p); return; }
    free_list.push_back({p, cap});
    cached_bytes += cap;
  }
};
static PinnedCache& pinned_cache() { static PinnedCache* c = new PinnedCache(); return *c; }
void B2QPartial::release_h_err() {
  if (h_err) {
    if (stream_busy()) cudaStreamSynchronize(stream); /* the async copy into the word must have landed before it is recycled */
    pinned_cache().put(reinterpret_cast<int8_t*>(h_err), h_err_cap);
  }
  h_err = nullptr;
}

struct B2QResultSet {
  B2QQuery q;
  int8_t* buf = nullptr;   /* pinned; every byte is written by the D2H copy */
  size_t buf_size = 0, buf_cap = 0;
  /* result_on_device: the materialised buffer stays in device memory (d_buf, buf_size bytes on `device`); `buf` is filled by
   * ONE device-to-host copy on the first host accessor (ensure_host) and from then on the set reads like any other */
  int8_t* d_buf = nullptr;
  int device = -1;
  std::once_flag host_once;
  int32_t host_rc = B2Q_OK;
  std::string host_err;
  int64_t d2h_bytes = 0;   /* B2Q_STAT_RESULT_D2H_BYTES */
  int64_t cursor = 0;
  int64_t cached_rows = -1;
  /* ResultSet::sort / dropFirstN / keepFirstN state (ResultSet.h: permutation_, drop_first_, keep_first_) */
  std::vector<uint32_t> perm;
  bool sorted = false;
  size_t drop_first = 0, keep_first = 0, fetched = 0;
  double sort_ms = 0;
  double scan_ms = 0, init_ms = 0, mat_ms = 0, h2d_bytes = 0;
  HostPhases host;
  int64_t launches = 0, frags_scanned = 0, frags_skipped = 0;
  int64_t rows_scanned = 0; /* B2Q_STAT_ROWS_SCANNED */
  int32_t join_table = B2Q_JOIN_TABLE_NONE; /* B2Q_STAT_JOIN_TABLE */
  bool heap_buf = false; /* b2q_rs_create_from_storage: a plain heap copy of the caller's buffer (no device involved) */
  ~B2QResultSet() {
    if (heap_buf) free(buf); else pinned_cache().put(buf, buf_cap);
    if (d_buf) { /* every reader of d_buf synchronised before returning: the free is ordered on the default stream */
      int cur = -1;
      cudaGetDevice(&cur);
      if (cur != device) cudaSetDevice(device);
      cudaFreeAsync(d_buf, nullptr);
      if (cur >= 0 && cur != device) cudaSetDevice(cur);
      cudaGetLastError();
    }
  }
};

/* the host copy of a result_on_device set, made once (thread-safe); false when it could not be made (g_err is set) */
static bool ensure_host(const B2QResultSet* crs) {
  B2QResultSet* rs = const_cast<B2QResultSet*>(crs);
  if (!rs->d_buf) return true;
  std::call_once(rs->host_once, [rs]() {
    rs->buf = pinned_cache().get(rs->buf_size, &rs->buf_cap);
    if (!rs->buf) { rs->host_rc = B2Q_ERR_INVALID_ARGUMENT; rs->host_err = "out of (pinned) host memory for the result buffer"; return; }
    int cur = -1;
    cudaGetDevice(&cur);
    if (cur != rs->device) cudaSetDevice(rs->device);
    const cudaError_t e = cudaMemcpy(rs->buf, rs->d_buf, rs->buf_size, cudaMemcpyDeviceToHost);
    if (cur >= 0 && cur != rs->device) cudaSetDevice(cur);
    if (e != cudaSuccess) {
      cudaGetLastError();
      pinned_cache().put(rs->buf, rs->buf_cap);
      rs->buf = nullptr;
      rs->host_rc = B2Q_ERR_CUDA;
      rs->host_err = std::string("result buffer to the host: ") + cudaGetErrorString(e);
      return;
    }
    rs->d2h_bytes += static_cast<int64_t>(rs->buf_size);
  });
  if (rs->host_rc != B2Q_OK) { set_err(rs->host_rc, rs->host_err); return false; }
  return true;
}

/* reduction class of an accumulator across devices (ResultSetStorage::reduceOneSlot's algebra on the internal arrays) */
enum { MERGE_SUM_I64 = 0, MERGE_SUM_F64 = 1, MERGE_MIN = 2, MERGE_MAX = 3, MERGE_FLAG = 4, MERGE_BOR = 5, kMergeClasses = 6 };
static int merge_class(int op) {
  switch (op) {
    case ACC_COUNT: case ACC_SUM_I64: return MERGE_SUM_I64;
    case ACC_SUM_F64: return MERGE_SUM_F64;
    case ACC_MIN_I64: case ACC_MIN_F64: return MERGE_MIN;
    case ACC_MAX_I64: case ACC_MAX_F64: return MERGE_MAX;
    case ACC_TOUCH: return MERGE_FLAG;
    default: return MERGE_BOR;
  }
}

/* bytes of accumulator array a: entry_count x 8, except the estimator's bitmap */
static size_t acc_array_bytes(const B2QQuery& q, int a) {
  if (q.prog.accs[a].op == ACC_NDV) return static_cast<size_t>(q.plan.buffer_size);
  if (q.prog.accs[a].op == ACC_BITMAP) return std::max<size_t>(static_cast<size_t>(q.plan.entry_count), 1) * static_cast<size_t>(q.prog.accs[a].bm_words) * 4;
  return std::max<size_t>(static_cast<size_t>(q.plan.entry_count), 1) * 8;
}

static size_t table_bytes(const B2QQuery& q) {
  const size_t n = std::max<size_t>(static_cast<size_t>(q.plan.entry_count), 1);
  size_t total = 0;
  for (int a = 0; a < q.prog.n_accs; ++a) total += DeviceBlock::pad(acc_array_bytes(q, a));
  if (q.plan.kernel == B2Q_KERNEL_BASELINE_GLOBAL) total += DeviceBlock::pad(n * 8);
  if (q.smem.use_smem) total += DeviceBlock::pad(std::max<int>(q.smem.replica_bytes, 16));
  total += 256; /* error word */
  return total;
}

static bool split_layout(const B2QQuery& q, bool radix);
static int32_t alloc_partial(B2QPartial& p, size_t extra_bytes, cudaStream_t st) {
  const B2QQuery& q = p.q;
  configure_pool_once(p.device);
  p.stream = st;
  const size_t n = std::max<size_t>(static_cast<size_t>(q.plan.entry_count), 1);
  CU(p.blk.alloc(table_bytes(q) + DeviceBlock::pad(extra_bytes) + DeviceBlock::pad(set_bytes(q)) + 4096, st));
  /* arrays of one reduction class (int64 SUM: COUNT / SUM_I64; f64 SUM; MIN; MAX; flags; bitmap) sit next to each other, so
   * that the cross-GPU merge is ONE collective per class over a contiguous range (C2: COUNT + SUM = one all-reduce) */
  for (int cls = 0; cls < kMergeClasses; ++cls)
    for (int a = 0; a < q.prog.n_accs; ++a)
      if (merge_class(q.prog.accs[a].op) == cls) p.accs[a] = reinterpret_cast<int64_t*>(p.blk.take(acc_array_bytes(q, a)));
  if (q.plan.kernel == B2Q_KERNEL_BASELINE_GLOBAL) p.keys = reinterpret_cast<int64_t*>(p.blk.take(n * 8));
  if (q.smem.use_smem) p.smem_image = p.blk.take(std::max<int>(q.smem.replica_bytes, 16));
  p.d_error = reinterpret_cast<int32_t*>(p.blk.take(256));
  p.split = split_layout(q, p.radix);
  if (const size_t sb = set_bytes(q)) { /* set terms: this device's own bitmaps, in the block, before the first scan */
    int n = 0;
    CU(build_sets(p.q, p.blk.take(sb), &n, st));
    p.launches += n;
  }
  for (auto& e : p.ev) CU(cudaEventCreate(&e));
  CU(cudaMemsetAsync(p.d_error, 0, sizeof(int32_t), st));
  CU(cudaEventRecord(p.ev[0], st));
  CU(launch_init(q, p.accs, p.keys, p.smem_image, st));
  for (int a = 0; a < q.prog.n_accs; ++a) /* the estimator's bitmap and the COUNT(DISTINCT) bitmaps start all-zero */
    if (q.prog.accs[a].op == ACC_NDV || q.prog.accs[a].op == ACC_BITMAP) CU(cudaMemsetAsync(p.accs[a], 0, acc_array_bytes(q, a), st));
  CU(cudaEventRecord(p.ev[1], st));
  return B2Q_OK;
}

/* ---- baseline hash through the radix-partitioned aggregation ------------------------------------------------------
 * B2Q_BASELINE_RADIX=0 keeps the per-row probe kernel (experiments / the fallback's own tests). */
static bool radix_enabled() {
  static const bool on = []() { const char* e = getenv("B2Q_BASELINE_RADIX"); return !e || atoi(e) != 0; }();
  return on;
}

/* memory a new stream-ordered allocation can count on: free device memory + what the pool holds but does not use */
static size_t pool_headroom(int device) {
  size_t free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) { cudaGetLastError(); return size_t(1) << 30; }
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    unsigned long long reserved = 0, used = 0;
    if (cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReservedMemCurrent, &reserved) == cudaSuccess &&
        cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemCurrent, &used) == cudaSuccess && reserved > used)
      free_b += static_cast<size_t>(reserved - used);
  }
  cudaGetLastError();
  return free_b;
}

/* buffers for launches of up to `max_chunks` chunks; larger launches run in batches over the same buffers */
static int32_t radix_prepare(B2QPartial& p, int64_t max_chunks, cudaStream_t st) {
  const B2QQuery& q = p.q;
  const size_t budget = std::max<size_t>(pool_headroom(p.device) / 2, size_t(256) << 20);
  int64_t batch = std::max<int64_t>(max_chunks, 1);
  int n_cta1 = 0;
  uint32_t cap = 0;
  size_t tuples = 0;
  for (;;) {
    radix_geometry(q, p.rp, batch, &n_cta1, &cap);
    tuples = static_cast<size_t>(p.rp.n_parts) * n_cta1 * cap;
    if ((tuples < (size_t(1) << 32) - 2 && tuples * p.rp.tuple_words * 8 <= budget) || batch <= n_cta1) break;
    batch = (batch + 1) / 2;
  }
  if (tuples >= (size_t(1) << 32) - 2) return set_err(B2Q_ERR_OUT_OF_GPU_MEM, "radix scratch does not fit");
  const size_t b_scratch = DeviceBlock::pad(tuples * p.rp.tuple_words * 8);
  const size_t b_counts = DeviceBlock::pad(static_cast<size_t>(p.rp.n_parts) * n_cta1 * 4);
  int8_t* base = nullptr;
  CU(cudaMallocAsync(reinterpret_cast<void**>(&base), b_scratch + b_counts + 256, st));
  p.extra.push_back(base);
  p.rb.scratch = reinterpret_cast<int64_t*>(base);
  p.rb.counts = reinterpret_cast<uint32_t*>(base + b_scratch);
  p.rb.work_counter = reinterpret_cast<uint32_t*>(base + b_scratch + b_counts);
  p.radix_batch_chunks = batch;
  p.radix_n_cta1 = n_cta1;
  p.radix_cap = cap;
  return B2Q_OK;
}

static int32_t radix_launch(B2QPartial& p, const DevLaunch& L, cudaStream_t st) {
  for (int64_t c0 = 0; c0 < L.total_chunks; c0 += p.radix_batch_chunks) {
    const int64_t c1 = std::min(L.total_chunks, c0 + p.radix_batch_chunks);
    int n_cta1 = p.radix_n_cta1;
    uint32_t cap = p.radix_cap;
    if (c1 - c0 < p.radix_batch_chunks) { /* a short (last) batch: fewer CTAs / smaller regions inside the same buffers */
      radix_geometry(p.q, p.rp, c1 - c0, &n_cta1, &cap);
      if (static_cast<size_t>(n_cta1) * cap > static_cast<size_t>(p.radix_n_cta1) * p.radix_cap) { n_cta1 = p.radix_n_cta1; cap = p.radix_cap; }
    }
    CU(launch_radix(p.q, p.rp, L, p.rb, c0, c1, n_cta1, cap, st));
    p.launches += 2;
  }
  return B2Q_OK;
}

/* Launch tables of one launch over fragments whose referenced columns are in device memory, as host words:
 * [column pointers nf x n_cols | rows nf | chunk prefix sums nf + 1].  They travel to the device in ONE H2D copy. */
static size_t launch_table_bytes(int nf, int nc) { return (static_cast<size_t>(nf) * nc + nf + nf + 1) * 8 + 64; }

static std::vector<int64_t> launch_tables(const std::vector<const int8_t*>& cols, const std::vector<int64_t>& rows, int64_t chunk_rows) {
  const size_t nf = rows.size();
  std::vector<int64_t> host(cols.size() + nf + nf + 1);
  memcpy(host.data(), cols.data(), cols.size() * 8);
  memcpy(host.data() + cols.size(), rows.data(), nf * 8);
  int64_t* cs = host.data() + cols.size() + nf;
  cs[0] = 0;
  for (size_t f = 0; f < nf; ++f) cs[f + 1] = cs[f] + (rows[f] + chunk_rows - 1) / chunk_rows;
  return host;
}

static int64_t scan_chunk_rows(const B2QPartial& p) {
  int block, ctas;
  scan_config(p.q, &block, &ctas);
  return p.radix ? radix_chunk_rows() : scan_rows_per_chunk(block);
}

/* one scan of the partial over launch tables in device memory: b2q_k_scan, or the radix pair in batches */
static int32_t scan_launch(B2QPartial& p, const int8_t* const* cols, const int64_t* rows, const int64_t* chunk_start, int nf,
                           int64_t chunks, cudaStream_t st) {
  DevLaunch L;
  memset(&L, 0, sizeof(L));
  L.col_ptrs = cols;
  L.frag_rows = rows;
  L.frag_chunk_start = chunk_start;
  L.n_frags = nf;
  L.total_chunks = chunks;
  for (int a = 0; a < p.q.prog.n_accs; ++a) L.accs[a] = p.accs[a];
  L.keys = p.keys;
  L.error = p.d_error;
  L.join_buff = p.join_buff;
  L.split = p.split ? 1 : 0;
  L.intr = p.intr ? p.intr->dev : kNoInterrupt;
  if (p.radix) return radix_launch(p, L, st);
  int block, ctas;
  scan_config(p.q, &block, &ctas);
  CU(launch_scan(p.q, L, p.smem_image, block, ctas, st));
  p.launches += 1;
  return B2Q_OK;
}

/* one scan launch over every fragment of `cols` / `rows`, device-resident; the launch tables go into the partial's block */
static int32_t scan_device_fragments(B2QPartial& p, const std::vector<const int8_t*>& cols, const std::vector<int64_t>& rows,
                                     cudaStream_t st, bool time_it) {
  const std::vector<int64_t> host = launch_tables(cols, rows, scan_chunk_rows(p));
  const int64_t chunks = host.back();
  if (chunks == 0) return B2Q_OK;
  int8_t* d_tab = p.blk.take(host.size() * 8);
  if (p.blk.used > p.blk.size) return set_err(B2Q_ERR_CUDA, "internal: launch tables exceed the device block");
  CU(cudaMemcpyAsync(d_tab, host.data(), host.size() * 8, cudaMemcpyHostToDevice, st));
  if (p.radix) {
    const int32_t rc = radix_prepare(p, chunks, st);
    if (rc != B2Q_OK) return rc;
  }
  if (time_it) CU(cudaEventRecord(p.ev[2], st));
  const int64_t* tab = reinterpret_cast<const int64_t*>(d_tab);
  const int32_t rc = scan_launch(p, reinterpret_cast<const int8_t* const*>(d_tab), tab + cols.size(), tab + cols.size() + rows.size(),
                                 static_cast<int>(rows.size()), chunks, st);
  if (rc != B2Q_OK) return rc;
  if (time_it) { CU(cudaEventRecord(p.ev[3], st)); p.scan_timed = true; }
  /* `host` is pageable: the copy above was staged by the runtime before cudaMemcpyAsync returned */
  return B2Q_OK;
}

/* HBM-table kernels: COUNT / integer SUM as (lo[n] | hi[n]) halves of which only the low words are hot (a returning 32-bit
 * atomic + the rare carry), so that a 1e7-group table is 40 MB of L2 next to the column stream.  The alternative — plain int64
 * words updated with RED.ADD.64, no return trip — is faster in isolation (tools/atom_bench.cu) but not inside the scan kernel,
 * where 80 MB of words do not stay resident in L2 next to the column stream.  B2Q_GLOBAL_SPLIT=0 keeps that layout selectable
 * for tables the cache does hold. */
static bool split_layout(const B2QQuery& q, bool radix) {
  if (!(q.plan.kernel == B2Q_KERNEL_PERFECT_GLOBAL || (q.plan.kernel == B2Q_KERNEL_BASELINE_GLOBAL && !radix))) return false;
  static const int knob = []() { const char* e = getenv("B2Q_GLOBAL_SPLIT"); return e ? atoi(e) : 1; }();
  if (knob != 0) return true;
  /* without the returning atomic the touched flag rests on "a value in [1, 2^31) cannot sum to zero": fewer than 2^32 rows */
  if (q.prog.touch_piggyback >= 0 && q.total_tuples >= (int64_t(1) << 32)) return true;
  return false;
}

/* the split layout is folded to plain int64 before anything downstream (NCCL merge,
 * materialise) wants plain int64 */
static int32_t normalize_partial(B2QPartial& p, cudaStream_t st) {
  if (!p.split) return B2Q_OK;
  const int64_t n = p.q.plan.entry_count;
  for (int a = 0; a < p.q.prog.n_accs; ++a) {
    const int op = p.q.prog.accs[a].op;
    if (op != ACC_COUNT && op != ACC_SUM_I64) continue;
    int64_t* out = nullptr;
    CU(cudaMallocAsync(reinterpret_cast<void**>(&out), std::max<int64_t>(n, 1) * 8, st));
    p.extra.push_back(out);
    CU(launch_join_split(p.accs[a], out, n, st));
    p.accs[a] = out;
  }
  p.split = false;
  return B2Q_OK;
}

static void collect_timings(B2QPartial& p) {
  float ms = 0;
  if (p.ev[0] && p.ev[1] && cudaEventElapsedTime(&ms, p.ev[0], p.ev[1]) == cudaSuccess) p.init_ms = ms;
  if (p.scan_timed && cudaEventElapsedTime(&ms, p.ev[2], p.ev[3]) == cudaSuccess) p.scan_ms = ms;
  cudaGetLastError();
}

/* Executor::skipFragment (QueryEngine/Execute.cpp:4776-4935): a fragment whose chunk min/max cannot satisfy one of
 * the simple quals (`col OP const`, AND-ed) is never scanned — and, for host-resident tables, never copied. */
static bool skip_fragment(const B2QExecUnit& u, const B2QTableInfo& tbl, const B2QFragmentInfo& fr, bool filter_deleted) {
  if (fr.num_tuples == 0) return true;
  if (!fr.col_buffers) return true; /* a fragment of another device: passed for its chunk stats only (see b2q.h) */
  /* isFragmentFullyDeleted (Execute.cpp:4740-4774): the $deleted$ chunk holds only `true` */
  if (filter_deleted && tbl.deleted_column_plus1 > 0 && fr.col_stats[tbl.deleted_column_plus1 - 1].int_min >= 1 &&
      fr.col_stats[tbl.deleted_column_plus1 - 1].int_max >= fr.col_stats[tbl.deleted_column_plus1 - 1].int_min) return true;
  for (int i = 0; i < u.num_simple_quals; ++i) {
    const int qi = u.simple_quals[i];
    if (qi < 0 || qi >= u.num_exprs) return false;
    const B2QExpr& q = u.exprs[qi];
    if (q.kind != B2Q_EXPR_BIN_OPER) return false;
    if (q.left < 0 || q.left >= u.num_exprs || q.right < 0 || q.right >= u.num_exprs) return false;
    const B2QExpr& l = u.exprs[q.left];
    const B2QExpr& c = u.exprs[q.right];
    if (l.kind != B2Q_EXPR_COLUMN_VAR || l.rte_idx != 0 || c.kind != B2Q_EXPR_CONSTANT) continue; /* chunk stats of the scanned table only */
    if (c.kind != B2Q_EXPR_CONSTANT) return false;
    if (c.is_null || l.col_id < 0 || l.col_id >= tbl.num_cols) continue;
    const B2QChunkStats& st = fr.col_stats[l.col_id];
    const bool col_fp = tbl.col_types[l.col_id].type == B2Q_kDOUBLE || tbl.col_types[l.col_id].type == B2Q_kFLOAT;
    const bool const_fp = c.ti.type == B2Q_kDOUBLE || c.ti.type == B2Q_kFLOAT; /* either carries its value in dval here */
    if (col_fp) { /* canSkipFragmentForFpQual (Execute.cpp:4700-4774): FLOAT and DOUBLE chunks both keep fp min / max */
      const double mn = st.fp_min, mx = st.fp_max, v = const_fp ? c.dval : static_cast<double>(c.ival);
      if (mn > mx) return false;
      switch (q.op) {
        case B2Q_kGE: if (mx < v) return true; break;
        case B2Q_kGT: if (mx <= v) return true; break;
        case B2Q_kLE: if (mn > v) return true; break;
        case B2Q_kLT: if (mn >= v) return true; break;
        case B2Q_kEQ: if (mn > v || mx < v) return true; break;
        default: break;
      }
      continue;
    }
    if (const_fp) continue; /* integer column against an fp literal: not considered */
    const int64_t mn = st.int_min, mx = st.int_max, v = c.ival;
    if (mn > mx) return false;
    switch (q.op) {
      case B2Q_kGE: if (mx < v) return true; break;
      case B2Q_kGT: if (mx <= v) return true; break;
      case B2Q_kLE: if (mn > v) return true; break;
      case B2Q_kLT: if (mn >= v) return true; break;
      case B2Q_kEQ: if (mn > v || mx < v) return true; break;
      default: break;
    }
  }
  return false;
}

/* the fragments a scan reads, in the order given (skip_fragment leaves the others out), counted into `scanned` / `skipped` */
static std::vector<int> scanned_fragments(const B2QExecUnit& u, const B2QTableInfo& tbl, bool filter_deleted, int64_t* scanned,
                                          int64_t* skipped) {
  std::vector<int> frags;
  for (int f = 0; f < tbl.num_fragments; ++f)
    if (!skip_fragment(u, tbl, tbl.fragments[f], filter_deleted)) frags.push_back(f);
  *scanned += static_cast<int64_t>(frags.size());
  *skipped += tbl.num_fragments - static_cast<int64_t>(frags.size());
  return frags;
}

/* per fragment of `frags`: its rows and the launch's column pointers, a joined inner table's columns (col_inner) from `inner` */
static int32_t fragment_columns(const B2QQuery& q, const B2QTableInfo& tbl, const std::vector<int>& frags, const int8_t* const* inner,
                                std::vector<const int8_t*>* cols, std::vector<int64_t>* rows) {
  for (int f : frags) {
    rows->push_back(tbl.fragments[f].num_tuples);
    for (int c = 0; c < q.prog.n_cols; ++c) {
      const bool in = q.prog.col_inner[c] != 0;
      const int8_t* ptr = in ? inner[c] : static_cast<const int8_t*>(tbl.fragments[f].col_buffers[q.col_ids[c]]);
      /* an empty device-resident inner table has no buffers; a host-resident scan never reads them except through a join match */
      if (!ptr && !(in && tbl.memory_level == B2Q_CPU_LEVEL)) return set_err(B2Q_ERR_INVALID_ARGUMENT, "referenced column has a NULL buffer");
      cols->push_back(ptr);
    }
  }
  return B2Q_OK;
}

/* ---- host-resident tables ------------------------------------------------------------------------------------------------
 * stream_host_table runs the scan of every host-resident table, aggregate and projection alike.  The fragments are cut into
 * slices of at most kHostSliceRows rows, one launch per slice.  The referenced columns of a slice are copied on a copy stream
 * into one of two staging sets, so that the copy of slice k+1 overlaps the scan of slice k (the reference does the H2D in
 * fetchChunks, unpipelined).  The caller's `launch` enqueues a slice's scan over that slice's launch tables, which are written
 * once up front.  Columns of a joined inner table (col_inner) are resident for the whole query and are not staged.
 * With `paced`, the host waits for the scan that last used a staging set before it refills it (the stream still holds the other
 * set's copy and scan, so the pipeline keeps its depth) and reads `watch`, device words copied after every scan.  A non-zero
 * first int32 there stops the stream: an error word, or a projection's done flag (0 or 1, so its low word says the same).  So
 * does the interrupt token; a stop seen only on the host goes into `error` (launch_set_error), the way every other stop travels. */
constexpr int64_t kHostSliceRows = int64_t(1) << 24; /* 16 Mi rows: a multiple of every kernel's chunk */

struct HostSlice {
  size_t index;
  const int8_t* const* cols;  /* device launch tables of the slice: [n_cols] */
  const int64_t* rows;        /* [1] */
  const int64_t* chunk_start; /* [2] = {0, chunks} */
  const int64_t* row_base;    /* [1]: the slice's first row in its fragment */
  int64_t chunks, chunk_base; /* chunks of this slice, and of the slices before it */
};

struct HostStream {
  bool paced = false;
  const void* watch = nullptr;
  size_t watch_bytes = 0;       /* at most 64 */
  void* watch_out = nullptr;    /* when set: `watch` as of the end of the stream, read once more after the last slice */
  int32_t* error = nullptr;
  const CallInterrupt* intr = nullptr;
  double* device_ms = nullptr;  /* when set: device time from the first copy to the last scan */
  std::function<int32_t(const HostSlice&)> launch;
};

static int32_t stream_host_table(const B2QQuery& q, const std::vector<const int8_t*>& cols, const std::vector<int64_t>& rows,
                                 int64_t chunk_rows, const HostStream& hs, cudaStream_t st, double* h2d_bytes, HostPhases* phases) {
  using clock = std::chrono::steady_clock;
  auto us_since = [](clock::time_point t0) { return std::chrono::duration<double, std::micro>(clock::now() - t0).count(); };
  const auto t_begin = clock::now();
  const int nc = q.prog.n_cols;
  struct Slice { size_t frag; int64_t row0, rows; };
  std::vector<Slice> sl;
  int64_t max_rows = 0;
  for (size_t f = 0; f < rows.size(); ++f)
    for (int64_t r = 0; r < rows[f]; r += kHostSliceRows) {
      sl.push_back({f, r, std::min(kHostSliceRows, rows[f] - r)});
      max_rows = std::max(max_rows, sl.back().rows);
    }
  const size_t ns = sl.size();
  if (ns == 0) return B2Q_OK;
  /* one device block: per-slice launch tables [cols ns x nc | rows ns | chunk_start 2 ns | row_base ns] | two staging sets */
  size_t set_bytes = 0, col_off[B2Q_MAX_COLS] = {};
  for (int c = 0; c < nc; ++c)
    if (!q.prog.col_inner[c]) { col_off[c] = set_bytes; set_bytes += DeviceBlock::pad(static_cast<size_t>(max_rows) * q.prog.col_width[c] + 16); }
  std::vector<int64_t> tab(ns * nc + 4 * ns);
  const size_t tab_bytes = DeviceBlock::pad(tab.size() * 8);
  int8_t* blk = nullptr;
  CU(cudaMallocAsync(reinterpret_cast<void**>(&blk), tab_bytes + 2 * set_bytes, st));
  int64_t* t_rows = tab.data() + ns * nc;
  int64_t* t_cs = t_rows + ns;
  int64_t* t_base = t_cs + 2 * ns;
  int64_t chunk_base = 0;
  for (size_t i = 0; i < ns; ++i) {
    int8_t* set = blk + tab_bytes + (i & 1) * set_bytes;
    for (int c = 0; c < nc; ++c)
      tab[i * nc + c] = reinterpret_cast<int64_t>(q.prog.col_inner[c] ? cols[sl[i].frag * nc + c] : set + col_off[c]);
    t_rows[i] = sl[i].rows;
    t_cs[2 * i] = 0;
    t_cs[2 * i + 1] = (sl[i].rows + chunk_rows - 1) / chunk_rows;
    t_base[i] = sl[i].row0;
  }
  const int64_t* d_tab = reinterpret_cast<const int64_t*>(blk);
  size_t pin_cap = 0;
  int8_t* h_watch = hs.paced ? pinned_cache().get(64, &pin_cap) : nullptr;
  if (hs.paced && !h_watch) { cudaFreeAsync(blk, st); cudaGetLastError(); return set_err(B2Q_ERR_INVALID_ARGUMENT, "out of (pinned) host memory"); }
  if (h_watch) memset(h_watch, 0, 64);
  cudaStream_t copy_st = nullptr;
  cudaEvent_t ready = nullptr, t0 = nullptr, t1 = nullptr, copied[2] = {}, scanned[2] = {};
  bool busy[2] = {false, false};
  cudaError_t e = cudaMemcpyAsync(blk, tab.data(), tab.size() * 8, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&copy_st, cudaStreamNonBlocking);
  for (cudaEvent_t* x : {&ready, &copied[0], &copied[1], &scanned[0], &scanned[1]})
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(x, cudaEventDisableTiming);
  if (e == cudaSuccess && hs.device_ms) e = cudaEventCreate(&t0);
  if (e == cudaSuccess && hs.device_ms) e = cudaEventCreate(&t1);
  /* the block was allocated in st's order: the copy stream may write into it only after that point */
  if (e == cudaSuccess) e = cudaEventRecord(ready, st);
  if (e == cudaSuccess) e = cudaStreamWaitEvent(copy_st, ready, 0);
  if (e == cudaSuccess && t0) e = cudaEventRecord(t0, st);
  phases->setup_us += us_since(t_begin);
  const auto t_stream = clock::now();
  int32_t rc = B2Q_OK;
  for (size_t i = 0; i < ns && e == cudaSuccess; ++i) {
    const int k = static_cast<int>(i & 1);
    if (busy[k]) {
      if (hs.paced) {
        e = cudaEventSynchronize(scanned[k]); /* the scan that used this set, and the read of `watch` after it */
        int32_t stop = 0;
        memcpy(&stop, h_watch, sizeof(stop));
        if (e != cudaSuccess || stop) break;
        if (hs.intr && hs.intr->interrupted()) { e = launch_set_error(hs.error, B2Q_ERR_INTERRUPTED, st); break; }
      }
      e = cudaStreamWaitEvent(copy_st, scanned[k], 0);
    }
    const Slice& x = sl[i];
    for (int c = 0; c < nc && e == cudaSuccess; ++c) {
      if (q.prog.col_inner[c]) continue;
      const size_t w = static_cast<size_t>(q.prog.col_width[c]), nbytes = static_cast<size_t>(x.rows) * w;
      e = cudaMemcpyAsync(reinterpret_cast<int8_t*>(tab[i * nc + c]), cols[x.frag * nc + c] + static_cast<size_t>(x.row0) * w, nbytes,
                          cudaMemcpyHostToDevice, copy_st);
      if (e == cudaSuccess) *h2d_bytes += static_cast<double>(nbytes);
    }
    if (e == cudaSuccess) e = cudaEventRecord(copied[k], copy_st);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(st, copied[k], 0);
    if (e != cudaSuccess) break;
    rc = hs.launch(HostSlice{i, reinterpret_cast<const int8_t* const*>(d_tab + i * nc), d_tab + ns * nc + i, d_tab + ns * nc + ns + 2 * i,
                             d_tab + ns * nc + 3 * ns + i, t_cs[2 * i + 1], chunk_base});
    if (rc != B2Q_OK) break;
    chunk_base += t_cs[2 * i + 1];
    if (h_watch) e = cudaMemcpyAsync(h_watch, hs.watch, hs.watch_bytes, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaEventRecord(scanned[k], st);
    busy[k] = true;
  }
  if (e == cudaSuccess && rc == B2Q_OK && t1) e = cudaEventRecord(t1, st);
  if (e == cudaSuccess && rc == B2Q_OK && hs.watch_out) e = cudaMemcpyAsync(h_watch, hs.watch, hs.watch_bytes, cudaMemcpyDeviceToHost, st);
  cudaError_t e_sync = copy_st ? cudaStreamSynchronize(copy_st) : cudaSuccess;
  if (e == cudaSuccess) e = e_sync;
  e_sync = cudaStreamSynchronize(st);
  if (e == cudaSuccess) e = e_sync;
  phases->stream_us += us_since(t_stream);
  const auto t_down = clock::now();
  float ms = 0;
  if (e == cudaSuccess && rc == B2Q_OK && t0 && cudaEventElapsedTime(&ms, t0, t1) == cudaSuccess) *hs.device_ms = ms;
  if (e == cudaSuccess && rc == B2Q_OK && hs.watch_out) memcpy(hs.watch_out, h_watch, hs.watch_bytes);
  cudaFreeAsync(blk, st); /* back to the stream-ordered pool, which keeps it: cudaFree of staging buffers this size is slow */
  if (copy_st) cudaStreamDestroy(copy_st);
  for (cudaEvent_t x : {ready, t0, t1, copied[0], copied[1], scanned[0], scanned[1]}) if (x) cudaEventDestroy(x);
  if (h_watch) pinned_cache().put(h_watch, pin_cap);
  phases->teardown_us += us_since(t_down);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return set_err(e == cudaErrorMemoryAllocation ? B2Q_ERR_OUT_OF_GPU_MEM : B2Q_ERR_CUDA, std::string("host-resident scan: ") + cudaGetErrorString(e));
  }
  return rc;
}

/* An aggregate over a host-resident table: stream_host_table, one scan launch per slice.  The host waits between slices only
 * with an interrupt token or a watchdog, and then reads the call's error word. */
static int32_t scan_host_table(B2QPartial& p, const std::vector<const int8_t*>& cols, const std::vector<int64_t>& rows, cudaStream_t st) {
  const int64_t chunk_rows = scan_chunk_rows(p);
  if (p.radix) {
    int64_t max_rows = 0;
    for (int64_t r : rows) max_rows = std::max(max_rows, std::min(r, kHostSliceRows));
    const int32_t rc = radix_prepare(p, (max_rows + chunk_rows - 1) / chunk_rows, st);
    if (rc != B2Q_OK) return rc;
  }
  HostStream hs;
  hs.paced = p.intr && p.intr->enabled();
  hs.watch = hs.error = p.d_error;
  hs.watch_bytes = sizeof(int32_t);
  hs.intr = p.intr.get();
  hs.launch = [&](const HostSlice& s) { return scan_launch(p, s.cols, s.rows, s.chunk_start, 1, s.chunks, st); };
  return stream_host_table(p.q, cols, rows, chunk_rows, hs, st, &p.h2d_bytes, &p.host);
}

/* B2Q_STAT_JOIN_TABLE of a query as prepared for its scan (prepare_join / choose_kernel) */
static int32_t join_table_kind(const B2QQuery& q) {
  if (q.prog.join.fk_col < 0) return B2Q_JOIN_TABLE_NONE;
  const bool packed = q.prog.join.packed_col >= 0;
  if (q.smem.join_off < 0) return packed ? B2Q_JOIN_TABLE_INT2_HBM : B2Q_JOIN_TABLE_INT32_HBM;
  return q.prog.join.slot16 ? B2Q_JOIN_TABLE_UINT16_SMEM : packed ? B2Q_JOIN_TABLE_INT2_SMEM : B2Q_JOIN_TABLE_INT32_SMEM;
}
static thread_local int32_t g_launch_join_table = B2Q_JOIN_TABLE_NONE; /* b2q_last_launch_stat */

/* The join level: inner-table columns to the device (they are small: dimension tables) and the one-to-one table
 * built there (PerfectJoinHashTable::reify -> initHashTableOnGpu / fill_hash_join_buff on the device). */
static int32_t prepare_join(B2QPartial& p, const B2QExecUnit& u, cudaStream_t st) {
  const B2QQuery& q = p.q;
  if (q.prog.join.fk_col < 0) return B2Q_OK;
  const B2QTableInfo& inner = *u.inner_table;
  const int64_t rows = inner.num_fragments ? inner.fragments[0].num_tuples : 0;
  auto phys_bytes = [&](int c) -> int {
    if (inner.col_encoded_sizes && inner.col_encoded_sizes[c] > 0) return inner.col_encoded_sizes[c];
    if (inner.col_encoded_sizes && inner.col_encoded_sizes[c] < 0) return -inner.col_encoded_sizes[c]; /* DATE ENCODING DAYS */
    switch (inner.col_types[c].type) {
      case B2Q_kTINYINT: case B2Q_kBOOLEAN: return 1;
      case B2Q_kSMALLINT: return 2;
      case B2Q_kINT: case B2Q_kFLOAT: case B2Q_kTEXT: case B2Q_kVARCHAR: case B2Q_kCHAR: return 4;
      default: return 8;
    }
  };
  std::vector<const int8_t*> dev(static_cast<size_t>(inner.num_cols), nullptr);
  auto device_col = [&](int c, const int8_t** out) -> int32_t {
    if (dev[c]) { *out = dev[c]; return B2Q_OK; }
    const void* src = rows ? inner.fragments[0].col_buffers[c] : nullptr;
    if (rows && !src) return set_err(B2Q_ERR_INVALID_ARGUMENT, "referenced inner column has a NULL buffer");
    if (inner.memory_level == B2Q_GPU_LEVEL) { dev[c] = static_cast<const int8_t*>(src); *out = dev[c]; return B2Q_OK; }
    if (inner.memory_level != B2Q_CPU_LEVEL) return set_err(B2Q_ERR_INVALID_ARGUMENT, "inner table memory_level must be B2Q_CPU_LEVEL or B2Q_GPU_LEVEL");
    int8_t* d = nullptr;
    const size_t nbytes = static_cast<size_t>(std::max<int64_t>(rows, 1)) * phys_bytes(c);
    CU(cudaMallocAsync(reinterpret_cast<void**>(&d), nbytes, st));
    p.extra.push_back(d);
    if (rows) { CU(cudaMemcpyAsync(d, src, static_cast<size_t>(rows) * phys_bytes(c), cudaMemcpyHostToDevice, st)); p.h2d_bytes += static_cast<double>(rows) * phys_bytes(c); }
    dev[c] = d;
    *out = d;
    return B2Q_OK;
  };
  for (int c = 0; c < q.prog.n_cols; ++c) {
    if (!q.prog.col_inner[c]) continue;
    const int32_t rc = device_col(q.col_ids[c] - q.n_outer_cols, &p.inner_cols[c]);
    if (rc != B2Q_OK) return rc;
  }
  const int8_t* d_key = nullptr;
  int32_t rc = device_col(q.join_inner_key_col, &d_key);
  if (rc != B2Q_OK) return rc;
  int32_t* buff = nullptr;
  const bool slot16 = q.prog.join.slot16 != 0;
  const int pc = slot16 ? -1 : q.prog.join.packed_col; /* slots {row, value of that inner column}: see DevJoin */
  /* + 16: the shared-memory staging copies whole 16-byte units (SmemPlan::join_bytes) */
  CU(cudaMallocAsync(reinterpret_cast<void**>(&buff), static_cast<size_t>(std::max<int64_t>(q.plan.join_entry_count, 1)) * (pc >= 0 ? 8 : 4) + 16, st));
  p.extra.push_back(buff);
  const B2QTypeInfo kt = inner.col_types[q.join_inner_key_col];
  const int kw = phys_bytes(q.join_inner_key_col);
  const int64_t knull = kw == 1 ? INT8_MIN : kw == 2 ? INT16_MIN : kw == 4 ? INT32_MIN : INT64_MIN;
  CU(launch_join_build(d_key, kw, rows, q.plan.join_min_key, q.plan.join_entry_count, kt.notnull ? 0 : 1, knull, buff, p.d_error,
                       pc >= 0 ? p.inner_cols[pc] : nullptr, q.prog.join.packed_width, st));
  p.launches += 1;
  p.join_buff = buff;
  if (slot16) { /* the row table only served to detect duplicates; the kernels probe the value-only 16-bit table */
    uint16_t* t16 = nullptr;
    CU(cudaMallocAsync(reinterpret_cast<void**>(&t16), static_cast<size_t>(std::max<int64_t>(q.plan.join_entry_count, 1)) * 2 + 16, st));
    p.extra.push_back(t16);
    const int c = q.prog.join.packed_col;
    CU(launch_join_slot16(buff, q.plan.join_entry_count, p.inner_cols[c], q.prog.join.packed_width, q.prog.col_null[c], q.prog.join.slot16_min, t16, p.d_error, st));
    p.launches += 1;
    p.join_buff = reinterpret_cast<const int32_t*>(t16);
  }
  return B2Q_OK;
}

static int32_t execute_partial_attempt(size_t* guess, const B2QTableInfo* tbl, const B2QExecUnit* u,
                                       const B2QCompilationOptions* co, const B2QExecutionOptions* eo, int32_t has_card,
                                       cudaStream_t st, bool allow_radix, bool defer, const std::shared_ptr<CallInterrupt>& intr,
                                       B2QPartial** out);

static int32_t execute_partial_impl(size_t* guess, const B2QTableInfo* tbl, const B2QExecUnit* u,
                                    const B2QCompilationOptions* co, const B2QExecutionOptions* eo, int32_t has_card,
                                    cudaStream_t st, B2QPartial** out) {
  const auto intr = CallInterrupt::from(eo);
  int32_t rc = execute_partial_attempt(guess, tbl, u, co, eo, has_card, st, radix_enabled(), false, intr, out);
  /* a structure of the radix path was too small for this input (hash clusters longer than its overflow areas): the
   * per-row probe kernel handles anything */
  if (rc == B2Q_RADIX_RETRY) rc = execute_partial_attempt(guess, tbl, u, co, eo, has_card, st, false, false, intr, out);
  return intr->resolve(rc);
}

/* what a non-zero device error word means at the boundary */
static int32_t device_error(int32_t dev_err) {
  if (dev_err == B2Q_RADIX_RETRY) return set_err(dev_err, "radix path: retry with the probe kernel");
  if (dev_err == B2Q_ERR_UNSUPPORTED) return set_err(dev_err, "join is not one-to-one (the reference rebuilds a one-to-many table): outside this path");
  if (dev_err == B2Q_ERR_INTERRUPTED) return set_err(dev_err, "the query was interrupted (b2q_interrupt on its token)");
  if (dev_err == B2Q_ERR_OUT_OF_TIME) return set_err(dev_err, "the query's device work exceeded dynamic_watchdog_time_limit");
  if (dev_err) return set_err(dev_err, dev_err == B2Q_ERR_OUT_OF_SLOTS ? "group-by table is full (OUT_OF_SLOTS)" : "group or join key outside the chunk-stats range");
  return B2Q_OK;
}

/* defer = true: nothing is synchronised here — the error word travels to the pinned p->h_err on the stream and the
 * caller checks it (partial_complete) after its own synchronize: scan -> merge -> materialise -> D2H is then ONE stream
 * of work with one host wait at the end. */
static int32_t execute_partial_attempt(size_t* guess, const B2QTableInfo* tbl, const B2QExecUnit* u,
                                       const B2QCompilationOptions* co, const B2QExecutionOptions* eo, int32_t has_card,
                                       cudaStream_t st, bool allow_radix, bool defer, const std::shared_ptr<CallInterrupt>& intr,
                                       B2QPartial** out) {
  if (!tbl || !u || !co || !eo || !out) return set_err(B2Q_ERR_INVALID_ARGUMENT, "null argument");
  if (co->device_type != B2Q_DEVICE_GPU) return set_err(B2Q_ERR_UNSUPPORTED, "device_type must be GPU: this path has no CPU execution");
  std::unique_ptr<B2QPartial> p(new B2QPartial());
  std::string err;
  const size_t g = guess ? *guess : 0;
  int32_t rc = make_query(u, tbl, eo, g, has_card != 0, !co->ignore_deleted_column, &p->q, &err);
  if (rc != B2Q_OK) return set_err(rc, err);
  if (p->q.plan.query_desc_type == B2Q_Projection)
    return set_err(B2Q_ERR_UNSUPPORTED, "projection units run through b2q_execute_work_unit (one device); the split and multi-device forms are outside this path");
  g_trace.mark("plan");
  if (!have_device()) return set_err(B2Q_ERR_NO_DEVICE, "no CUDA device visible; this path has no CPU fallback");
  if (eo->device_ordinal >= 0) CU(cudaSetDevice(eo->device_ordinal));
  CU(cudaGetDevice(&p->device));
  p->intr = intr;
  CU(p->intr->start(p->device, st));
  p->radix = allow_radix && eo->force_kernel != B2Q_KERNEL_BASELINE_PROBE && radix_plan(p->q, &p->rp);
  p->result_on_device = eo->result_on_device != 0 && p->q.plan.query_desc_type != B2Q_Estimator; /* the bitmap is tiny and read on the host */
  const size_t extra = tbl->memory_level == B2Q_GPU_LEVEL ? launch_table_bytes(tbl->num_fragments, p->q.prog.n_cols) : 0;
  rc = alloc_partial(*p, extra, st);
  if (rc != B2Q_OK) return rc;
  g_trace.mark("alloc+init");
  rc = prepare_join(*p, *u, st);
  if (rc != B2Q_OK) return rc;
  const std::vector<int> frags = scanned_fragments(*u, *tbl, !co->ignore_deleted_column, &p->frags_scanned, &p->frags_skipped);
  if (tbl->memory_level != B2Q_GPU_LEVEL && tbl->memory_level != B2Q_CPU_LEVEL)
    return set_err(B2Q_ERR_INVALID_ARGUMENT, "memory_level must be B2Q_CPU_LEVEL or B2Q_GPU_LEVEL");
  std::vector<const int8_t*> cols;
  std::vector<int64_t> rows;
  rc = fragment_columns(p->q, *tbl, frags, p->inner_cols, &cols, &rows);
  if (rc != B2Q_OK) return rc;
  if (!frags.empty()) {
    /* device-resident: one kernel over every fragment handed to this device (Execute.cpp:3075-3101) */
    rc = tbl->memory_level == B2Q_GPU_LEVEL ? scan_device_fragments(*p, cols, rows, st, true) : scan_host_table(*p, cols, rows, st);
    if (rc != B2Q_OK) return rc;
  }
  rc = normalize_partial(*p, st);
  if (rc != B2Q_OK) return rc;
  g_trace.mark("scan enqueued");
  /* with an interrupt or a watchdog a host-resident scan defers too: a stop must reach every rank of a multi-device call
   * through the merged error word, never as an early return that leaves the peers in a collective */
  if (defer && (tbl->memory_level == B2Q_GPU_LEVEL || p->intr->enabled())) {
    p->h_err = reinterpret_cast<int32_t*>(pinned_cache().get(64, &p->h_err_cap));
    if (!p->h_err) return set_err(B2Q_ERR_INVALID_ARGUMENT, "out of (pinned) host memory");
    *p->h_err = 0;
    p->deferred = true;
    *out = p.release();
    return B2Q_OK;
  }
  int32_t dev_err = 0;
  CU(cudaMemcpyAsync(&dev_err, p->d_error, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  collect_timings(*p);
  rc = device_error(dev_err);
  if (rc != B2Q_OK) return rc;
  *out = p.release();
  return B2Q_OK;
}

/* deferred partial: enqueue the copy of the error word (after whatever merged it across devices) */
static int32_t partial_enqueue_error_copy(B2QPartial& p, cudaStream_t st) {
  if (p.deferred) CU(cudaMemcpyAsync(p.h_err, p.d_error, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  return B2Q_OK;
}

/* ---- ORDER BY / LIMIT on the device (sort.cu) ---------------------------------------------------------------- */
static DevSortLayout sort_layout_of(const B2QPlan& p) {
  DevSortLayout L;
  memset(&L, 0, sizeof(L));
  L.row_size = p.row_size;
  L.entry_count = p.entry_count;
  L.columnar = static_cast<int8_t>(p.output_columnar);
  L.grouped = p.query_desc_type != B2Q_NonGroupedAggregate;
  L.keyless = static_cast<int8_t>(p.keyless_hash);
  if (p.keyless_hash) {
    L.marker_off = p.slot_offset[p.idx_target_as_key];
    L.marker_w = p.slot_padded_width[p.idx_target_as_key];
    L.marker_init = p.init_vals[p.idx_target_as_key];
  }
  L.key_w = static_cast<int8_t>(p.output_columnar ? 8 : p.effective_key_width);
  return L;
}

/* one Analyzer::OrderEntry against the output layout; the value is read the way ResultSetComparator reads it
 * (getColumnInternal at the padded slot width, AVG as a (sum, count) pair, baseline key targets from the key) */
static DevSortKey sort_key_of(const B2QPlan& p, const B2QOrderEntry& oe) {
  DevSortKey k;
  memset(&k, 0, sizeof(k));
  const B2QTargetInfo& t = p.targets[oe.tle_no - 1];
  const int s = t.first_slot;
  k.off1 = p.slot_offset[s];
  k.w1 = p.slot_padded_width[s];
  if (k.w1 == 0) { k.off1 = 0; k.w1 = static_cast<int8_t>(p.output_columnar ? 8 : p.effective_key_width); } /* baseline: the key is the target */
  const bool has_arg = t.agg_arg_type.type != 0;
  const bool minmax = t.is_agg && has_arg && (t.agg_kind == B2Q_kMIN || t.agg_kind == B2Q_kMAX);
  const B2QTypeInfo compact = minmax ? t.agg_arg_type : t.sql_type; /* get_compact_type */
  k.nullable = !compact.notnull;
  k.is_desc = oe.is_desc;
  k.nulls_first = oe.nulls_first;
  if (t.is_agg && t.agg_kind == B2Q_kAVG) {
    k.kind = t.sql_type.type == B2Q_kDOUBLE ? SORTKEY_AVG_F64 : t.sql_type.type == B2Q_kFLOAT ? SORTKEY_AVG_F32 : SORTKEY_AVG_I64;
    k.scale = static_cast<int8_t>(b2q_is_decimal(t.sql_type.type) ? t.sql_type.scale : 0);
    k.off2 = p.slot_offset[s + 1];
  } else if (compact.type == B2Q_kDOUBLE) {
    k.kind = SORTKEY_F64;
    const double nd = DBL_MIN;
    memcpy(&k.null_pattern, &nd, 8);
  } else if (compact.type == B2Q_kFLOAT) {
    k.kind = SORTKEY_F32;
    k.null_pattern = b2q_null_bits(B2Q_kFLOAT);
  } else {
    k.kind = SORTKEY_I64;
    k.null_pattern = b2q_int_null(compact.type);
  }
  return k;
}

/* the same descriptor for a buffer of `n` entries (compacted result): row-wise only the sizes change, columnar
 * every column moves (getColOffInBytes, QueryMemoryDescriptor.cpp:918-955) */
static void relayout_entries(B2QPlan& p, int64_t n) {
  p.entry_count = n;
  if (!p.output_columnar) { p.buffer_size = p.row_size * n; return; }
  const bool keyed = p.query_desc_type != B2Q_NonGroupedAggregate && !p.keyless_hash;
  int64_t off = keyed ? static_cast<int64_t>(std::max(p.num_group_cols, 1)) * ((8 * n + 7) & ~int64_t(7)) : 0;
  for (int s = 0; s < p.num_slots; ++s) {
    p.slot_offset[s] = off;
    off += (static_cast<int64_t>(p.slot_padded_width[s]) * n + 7) & ~int64_t(7);
  }
  p.buffer_size = off;
}

static DevGatherCols gather_cols_of(const B2QPlan& in, const B2QPlan& out) {
  DevGatherCols g;
  memset(&g, 0, sizeof(g));
  if (!in.output_columnar) return g;
  const bool keyed = in.query_desc_type != B2Q_NonGroupedAggregate && !in.keyless_hash;
  if (keyed)
    for (int c = 0; c < std::max(in.num_group_cols, 1); ++c) {
      g.in_off[g.n] = c * ((8 * in.entry_count + 7) & ~int64_t(7));
      g.out_off[g.n] = c * ((8 * out.entry_count + 7) & ~int64_t(7));
      g.width[g.n++] = 8;
    }
  for (int s = 0; s < in.num_slots; ++s) {
    if (!in.slot_padded_width[s]) continue;
    g.in_off[g.n] = in.slot_offset[s];
    g.out_off[g.n] = out.slot_offset[s];
    g.width[g.n++] = in.slot_padded_width[s];
  }
  return g;
}

/* get_truncated_row_count-style window over `n` sorted rows: [first, first + count) */
static void limit_window(const B2QQuery& q, int64_t n, int64_t* first, int64_t* count) {
  /* LIMIT 0: RelSort::isEmptyResult() (RelAlgDag.h:2557) turns the step into just_validate and an empty result
   * (RelAlgExecutor.cpp:1277, :3559); a unit that still carries it gets exactly that */
  if (q.has_limit && q.limit == 0) { *first = 0; *count = 0; return; }
  const int64_t top_n = (q.has_limit ? q.limit : 0) + q.offset; /* rs->sort(order_entries, limit + offset) */
  int64_t kept = (q.n_order && top_n) ? std::min(top_n, n) : n;  /* topPermutation resizes to top_n */
  *first = std::min<int64_t>(q.offset, kept);                   /* dropFirstN(offset) */
  int64_t c = kept - *first;
  if (q.has_limit && q.limit) c = std::min(c, q.limit);          /* keepFirstN(limit); keep_first_ == 0 means "no limit" */
  *count = c;
}

/* ORDER BY / LIMIT / OFFSET over a materialised device buffer laid out as rs->q.plan says: compaction of the non-empty
 * entries, sort, and a gather of the kept rows into a compact buffer, which becomes the result (rs->d_buf when on_device,
 * else copied into rs->buf).  Frees d_in (stream-ordered) and returns after the stream's work is complete. */
static int32_t sort_keep_rows(B2QResultSet* rs, int8_t* d_in, bool on_device, int device, cudaStream_t st, const CallInterrupt* intr) {
  const B2QPlan plan = rs->q.plan;
  const B2QQuery& q = rs->q;
  int8_t* d_scratch = nullptr;
  int8_t* d_compact = nullptr;
  cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&d_scratch), sort_scratch_bytes(plan.entry_count), st);
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaEventCreate(&ev0); cudaEventCreate(&ev1);
  const DevSortLayout L = sort_layout_of(plan);
  DevSortKey keys[B2Q_MAX_ORDER_ENTRIES];
  for (int i = 0; i < q.n_order; ++i) keys[i] = sort_key_of(plan, q.order[i]);
  const uint32_t* d_perm = nullptr;
  int64_t n = 0, first = 0, count = 0;
  int sort_launches = 0;
  bool stopped = false;
  if (e == cudaSuccess) e = cudaEventRecord(ev0, st);
  if (e == cudaSuccess) e = sort_device(L, keys, q.n_order, d_in, d_scratch, st, &d_perm, &n, &sort_launches,
                                        (q.has_limit ? q.limit : 0) + q.offset, intr ? intr->host_flag : nullptr, &stopped);
  if (e == cudaSuccess && !stopped) {
    limit_window(q, n, &first, &count);
    relayout_entries(rs->q.plan, count);
    rs->buf_size = static_cast<size_t>(rs->q.plan.buffer_size);
    if (rs->buf_size) {
      if (!on_device) {
        rs->buf = pinned_cache().get(rs->buf_size, &rs->buf_cap);
        if (!rs->buf) e = cudaErrorMemoryAllocation;
      }
      if (e == cudaSuccess) e = cudaMallocAsync(reinterpret_cast<void**>(&d_compact), rs->buf_size, st);
      const DevGatherCols G = gather_cols_of(plan, rs->q.plan);
      if (e == cudaSuccess) e = sort_gather(L, G, d_in, d_compact, d_perm, first, count, st);
      if (e == cudaSuccess) e = cudaEventRecord(ev1, st);
      if (on_device) { /* the compact buffer IS the result */
        if (e == cudaSuccess) { rs->d_buf = d_compact; rs->device = device; d_compact = nullptr; }
      } else if (e == cudaSuccess) {
        e = cudaMemcpyAsync(rs->buf, d_compact, rs->buf_size, cudaMemcpyDeviceToHost, st);
        rs->d2h_bytes = static_cast<int64_t>(rs->buf_size);
      }
      sort_launches += 1;
    } else if (e == cudaSuccess) {
      e = cudaEventRecord(ev1, st);
    }
  }
  if (d_compact) cudaFreeAsync(d_compact, st);
  if (d_scratch) cudaFreeAsync(d_scratch, st);
  cudaFreeAsync(d_in, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e == cudaSuccess) { float ms = 0; if (cudaEventElapsedTime(&ms, ev0, ev1) == cudaSuccess) rs->sort_ms = ms; }
  cudaEventDestroy(ev0); cudaEventDestroy(ev1);
  if (e != cudaSuccess) { cudaGetLastError(); return set_err(B2Q_ERR_CUDA, std::string("sort/materialise: ") + cudaGetErrorString(e)); }
  if (stopped) return set_err(B2Q_ERR_INTERRUPTED, "the query was interrupted (b2q_interrupt on its token) during ORDER BY");
  rs->sorted = true;
  rs->launches += sort_launches;
  return B2Q_OK;
}

static int32_t finalize_core(B2QPartial* p, cudaStream_t st, B2QResultSet** out);

static int32_t finalize_impl(B2QPartial* p, cudaStream_t st, B2QResultSet** out) {
  if (!p || !out) return set_err(B2Q_ERR_INVALID_ARGUMENT, "null argument");
  if (p->deferred) {
    const int32_t rc0 = partial_enqueue_error_copy(*p, st);
    if (rc0 != B2Q_OK) return rc0;
    if (p->intr && p->intr->enabled()) {
      /* a call that can be stopped waits for its scan here: a stopped one neither materialises nor copies back its partial table
       * (for 1e7 groups that copy alone is several ms of the time from the interrupt to the return) */
      if (cudaStreamSynchronize(st) != cudaSuccess) { cudaGetLastError(); return set_err(B2Q_ERR_CUDA, "stream synchronize"); }
      if (*p->h_err) {
        collect_timings(*p);
        p->deferred = false;
        return device_error(*p->h_err);
      }
    }
  }
  int32_t rc = finalize_core(p, st, out);
  if (!p->deferred) return rc;
  /* the call's one host wait has happened inside finalize_core (or happens here when nothing was copied back) */
  if (cudaStreamSynchronize(st) != cudaSuccess) { cudaGetLastError(); if (rc == B2Q_OK) { delete *out; *out = nullptr; } return set_err(B2Q_ERR_CUDA, "stream synchronize"); }
  collect_timings(*p);
  p->deferred = false;
  const int32_t dev_err = *p->h_err;
  if (rc == B2Q_OK && dev_err) { delete *out; *out = nullptr; }
  if (dev_err) return device_error(dev_err);
  if (rc == B2Q_OK) { (*out)->scan_ms = p->scan_ms; (*out)->init_ms = p->init_ms; }
  return rc;
}

static int32_t finalize_core(B2QPartial* p, cudaStream_t st, B2QResultSet** out) {
  CU(cudaSetDevice(p->device));
  std::unique_ptr<B2QResultSet> rs(new B2QResultSet());
  rs->q = p->q;
  rs->scan_ms = p->scan_ms;
  rs->init_ms = p->init_ms;
  rs->h2d_bytes = p->h2d_bytes;
  rs->host = p->host;
  rs->launches = p->launches + 2; /* + b2q_k_init + b2q_k_materialize */
  rs->frags_scanned = p->frags_scanned;
  rs->frags_skipped = p->frags_skipped;
  rs->join_table = join_table_kind(p->q);
  const size_t nbytes = static_cast<size_t>(p->q.plan.buffer_size);
  if (p->q.plan.query_desc_type == B2Q_Estimator) { /* the result is the bitmap itself (ResultSet::getHostEstimatorBuffer) */
    rs->launches = p->launches + 1; /* + b2q_k_init */
    rs->buf_size = nbytes;
    rs->buf = pinned_cache().get(nbytes, &rs->buf_cap);
    if (!rs->buf) return set_err(B2Q_ERR_INVALID_ARGUMENT, "out of (pinned) host memory for the estimator buffer");
    cudaError_t e = cudaMemcpyAsync(rs->buf, p->accs[0], nbytes, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { cudaGetLastError(); return set_err(B2Q_ERR_CUDA, std::string("estimator buffer: ") + cudaGetErrorString(e)); }
    rs->d2h_bytes = static_cast<int64_t>(nbytes);
    *out = rs.release();
    return B2Q_OK;
  }
  const bool want_sort = p->q.n_order > 0 || p->q.has_limit || p->q.offset > 0;
  if (nbytes && want_sort) {
    /* materialise on the device, sort / truncate there, copy back only the kept rows */
    int8_t* d_out = nullptr;
    CU(cudaMallocAsync(reinterpret_cast<void**>(&d_out), nbytes, st));
    cudaError_t e = launch_materialize(p->q, p->accs, p->keys, d_out, st);
    if (e != cudaSuccess) { cudaFreeAsync(d_out, st); cudaGetLastError(); return set_err(B2Q_ERR_CUDA, std::string("materialise: ") + cudaGetErrorString(e)); }
    const int32_t rc = sort_keep_rows(rs.get(), d_out, p->result_on_device, p->device, st, p->intr.get());
    if (rc != B2Q_OK) return rc;
    *out = rs.release();
    return B2Q_OK;
  }
  rs->buf_size = nbytes;
  if (nbytes) {
    if (!p->result_on_device) {
      rs->buf = pinned_cache().get(nbytes, &rs->buf_cap);
      if (!rs->buf) return set_err(B2Q_ERR_INVALID_ARGUMENT, "out of (pinned) host memory for the result buffer");
      g_trace.mark("pinned buffer");
    }
    int8_t* d_out = nullptr;
    CU(cudaMallocAsync(reinterpret_cast<void**>(&d_out), nbytes, st));
    cudaError_t e = launch_materialize(p->q, p->accs, p->keys, d_out, st);
    if (p->result_on_device) { /* kept: the result set owns it (freed with the set, on its device) */
      rs->d_buf = d_out;
      rs->device = p->device;
    } else {
      if (e == cudaSuccess) e = cudaMemcpyAsync(rs->buf, d_out, nbytes, cudaMemcpyDeviceToHost, st);
      rs->d2h_bytes = static_cast<int64_t>(nbytes);
      cudaFreeAsync(d_out, st);
    }
    g_trace.mark("materialise + D2H enqueued");
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    g_trace.mark("stream synchronize");
    if (e != cudaSuccess) { cudaGetLastError(); return set_err(B2Q_ERR_CUDA, std::string("materialise: ") + cudaGetErrorString(e)); }
  }
  *out = rs.release();
  return B2Q_OK;
}

/* ---- result-set iteration ------------------------------------------------------------------------------- */
static const int8_t* rs_slot_ptr(const B2QResultSet* rs, int64_t e, int s) { return b2q_slot_ptr(rs->q.plan, rs->buf, e, s); }
static const int8_t* rs_key_ptr(const B2QResultSet* rs, int64_t e) { return b2q_key_ptr(rs->q.plan, rs->buf, e); }

/* ResultSetStorage::isEmptyEntry / isEmptyEntryColumnar (ResultSetIteration.cpp:2457-2545) */
static bool rs_is_empty_entry(const B2QResultSet* rs, int64_t e) {
  const B2QPlan& p = rs->q.plan;
  if (p.query_desc_type == B2Q_Estimator) return true; /* an estimator result set has no storage, only the bitmap */
  if (p.query_desc_type == B2Q_NonGroupedAggregate) return false;
  if (p.keyless_hash) {
    const int s = p.idx_target_as_key;
    int64_t v;
    if (p.slot_padded_width[s] == 4) { int32_t x; memcpy(&x, rs_slot_ptr(rs, e, s), 4); v = x; }
    else memcpy(&v, rs_slot_ptr(rs, e, s), 8);
    return v == p.init_vals[s];
  }
  if (!p.output_columnar && p.effective_key_width == 4) { int32_t k; memcpy(&k, rs_key_ptr(rs, e), 4); return k == 0x7FFFFFFF; }
  int64_t k;
  memcpy(&k, rs_key_ptr(rs, e), 8);
  return k == B2Q_I64_MAX;
}


/* ---- cross-GPU merge of a partial (NCCL, on the stream that produced it) -------------------------------------------
 * Dense tables are position-aligned on every device (all devices plan over the same key ranges) and initialised to the
 * identity of their reduction: the merge is one in-place all-reduce per reduction class, grouped into one NCCL launch,
 * with the device error word riding along (MAX) so that every rank reports the same outcome.  No host synchronisation
 * between scan, merge and materialise. */
#define NC(call)                                                                                                      \
  do {                                                                                                                \
    ncclResult_t r__ = (call);                                                                                        \
    if (r__ != ncclSuccess) return set_err(B2Q_ERR_CUDA, std::string(#call) + ": " + api->GetErrorString(r__));       \
  } while (0)

/* Baseline-hash tables are not position-aligned across devices (each device claimed its slots in its own order): every rank
 * gathers the peers' key / accumulator arrays and re-probes their entries into its own table — ResultSetStorage::reduce for
 * baseline layouts (ResultSetReduction.cpp:698-828) on the device.  Afterwards every rank holds the same set of rows. */
static int32_t b2q_baseline_merge(B2QPartial& p, const B2QComm* comm, const NcclApi* api, cudaStream_t st) {
  const B2QQuery& q = p.q;
  if (p.split) return set_err(B2Q_ERR_CUDA, "internal: split accumulators reached the baseline merge");
  const int64_t E = q.plan.entry_count;
  const int na = q.prog.n_accs;
  const size_t arr = static_cast<size_t>(E) * 8;
  /* per-rank bytes of every gathered array: int64[E], except the COUNT(DISTINCT) bitmaps ([E][bm_words] 32-bit words) */
  size_t bytes_of[B2Q_MAX_ACCS], total = arr;
  for (int a = 0; a < na; ++a) { bytes_of[a] = DeviceBlock::pad(acc_array_bytes(q, a)); total += bytes_of[a]; }
  int8_t* stage = nullptr;
  CU(cudaMallocAsync(reinterpret_cast<void**>(&stage), total * comm->nranks + 256, st));
  p.extra.push_back(stage);
  const int64_t* g_keys = reinterpret_cast<const int64_t*>(stage);
  const int64_t* g_accs[B2Q_MAX_ACCS];
  NC(api->GroupStart());
  NC(api->AllGather(p.keys, stage, static_cast<size_t>(E), ncclInt64, comm->comm, st));
  int8_t* dst = stage + arr * comm->nranks;
  for (int a = 0; a < na; ++a) {
    g_accs[a] = reinterpret_cast<const int64_t*>(dst);
    const size_t own = acc_array_bytes(q, a); /* the gathered blocks are packed at the array's own size: entry i of rank r sits at (r E + i) */
    NC(api->AllGather(p.accs[a], dst, own, ncclUint8, comm->comm, st));
    dst += bytes_of[a] * comm->nranks;
  }
  NC(api->AllReduce(p.d_error, p.d_error, 1, ncclInt32, ncclMax, comm->comm, st));
  NC(api->GroupEnd());
  CU(launch_baseline_merge(q, g_keys, g_accs, E * comm->nranks, E * comm->rank, E * (comm->rank + 1), p.keys, p.accs, p.d_error, st));
  p.launches += 1;
  /* a rank whose merged table ran out of slots must not be the only one to say so */
  NC(api->AllReduce(p.d_error, p.d_error, 1, ncclInt32, ncclMax, comm->comm, st));
  return B2Q_OK;
}

static int32_t merge_partial(B2QPartial& p, const B2QComm* comm, cudaStream_t st) {
  if (!comm || comm->nranks <= 1) return B2Q_OK;
  std::string why;
  const NcclApi* api = nccl_api(&why);
  if (!api) return set_err(B2Q_ERR_UNSUPPORTED, why);
  const B2QQuery& q = p.q;
  if (q.plan.kernel == B2Q_KERNEL_BASELINE_GLOBAL) return b2q_baseline_merge(p, comm, api, st);
  struct Span { int8_t* lo; int8_t* hi; int cls; };
  std::vector<Span> spans;
  for (int cls = 0; cls < kMergeClasses; ++cls)
    for (int a = 0; a < q.prog.n_accs; ++a) {
      if (merge_class(q.prog.accs[a].op) != cls) continue;
      int8_t* lo = reinterpret_cast<int8_t*>(p.accs[a]);
      int8_t* hi = lo + DeviceBlock::pad(acc_array_bytes(q, a));
      if (q.prog.accs[a].op == ACC_TOUCH) hi = lo + DeviceBlock::pad(std::max<size_t>(static_cast<size_t>(q.plan.entry_count), 1));
      if (!spans.empty() && spans.back().cls == cls && spans.back().hi == lo) spans.back().hi = hi; /* contiguous: one collective */
      else spans.push_back({lo, hi, cls});
    }
  int8_t* gathered = nullptr; /* estimator bitmaps: NCCL has no OR — all-gather, then OR on the device */
  NC(api->GroupStart());
  for (const Span& sp : spans) {
    const size_t bytes = static_cast<size_t>(sp.hi - sp.lo);
    switch (sp.cls) {
      case MERGE_SUM_I64: NC(api->AllReduce(sp.lo, sp.lo, bytes / 8, ncclInt64, ncclSum, comm->comm, st)); break;
      case MERGE_SUM_F64: NC(api->AllReduce(sp.lo, sp.lo, bytes / 8, ncclFloat64, ncclSum, comm->comm, st)); break;
      case MERGE_MIN: NC(api->AllReduce(sp.lo, sp.lo, bytes / 8, ncclInt64, ncclMin, comm->comm, st)); break;
      case MERGE_MAX: NC(api->AllReduce(sp.lo, sp.lo, bytes / 8, ncclInt64, ncclMax, comm->comm, st)); break;
      case MERGE_FLAG: NC(api->AllReduce(sp.lo, sp.lo, bytes, ncclUint8, ncclMax, comm->comm, st)); break;
      default: {
        if (cudaMallocAsync(reinterpret_cast<void**>(&gathered), bytes * comm->nranks, st) != cudaSuccess) { cudaGetLastError(); api->GroupEnd(); return set_err(B2Q_ERR_OUT_OF_GPU_MEM, "estimator merge buffer"); }
        p.extra.push_back(gathered);
        NC(api->AllGather(sp.lo, gathered, bytes, ncclUint8, comm->comm, st));
        break;
      }
    }
  }
  NC(api->AllReduce(p.d_error, p.d_error, 1, ncclInt32, ncclMax, comm->comm, st));
  NC(api->GroupEnd());
  if (gathered)
    for (const Span& sp : spans)
      if (sp.cls == MERGE_BOR) CU(launch_bitmap_or(reinterpret_cast<uint64_t*>(sp.lo), reinterpret_cast<const uint64_t*>(gathered), static_cast<int64_t>(sp.hi - sp.lo) / 8, comm->nranks, st));
  return B2Q_OK;
}

/* one rank's share of a multi-device work unit: scan -> merge -> materialise -> D2H, one host wait at the end */
static int32_t execute_work_unit_rank(const B2QComm* comm, size_t* guess, const B2QTableInfo* tbl, const B2QExecUnit* u,
                                      const B2QCompilationOptions* co, const B2QExecutionOptions* eo, int32_t has_card,
                                      cudaStream_t st, bool finalize, B2QResultSet** out, double* kernel_ms) {
  B2QExecutionOptions eo_dev = *eo;
  if (comm) eo_dev.device_ordinal = comm->device;
  const auto intr = CallInterrupt::from(eo);
  for (int attempt = 0; attempt < 2; ++attempt) {
    B2QPartial* p = nullptr;
    int32_t rc = execute_partial_attempt(guess, tbl, u, co, &eo_dev, has_card, st, attempt == 0 && radix_enabled(),
                                         tbl->memory_level == B2Q_GPU_LEVEL || intr->enabled(), intr, &p);
    if (rc != B2Q_OK) return rc; /* planning errors are the same on every rank: nobody reaches the collective */
    rc = merge_partial(*p, comm, st);
    if (rc == B2Q_OK && finalize) rc = finalize_impl(p, st, out);
    else if (rc == B2Q_OK) { /* a device that only contributes: wait for its part, report its error word */
      if (p->deferred) rc = partial_enqueue_error_copy(*p, st);
      if (rc == B2Q_OK && cudaStreamSynchronize(st) != cudaSuccess) { cudaGetLastError(); rc = set_err(B2Q_ERR_CUDA, "stream synchronize"); }
      if (rc == B2Q_OK) { collect_timings(*p); if (p->deferred) { p->deferred = false; rc = device_error(*p->h_err); } }
    }
    if (kernel_ms) *kernel_ms = p->scan_ms;
    delete p;
    if (rc != B2Q_RADIX_RETRY) return intr->resolve(rc); /* the error word was MAX-merged: every rank retries together */
  }
  return set_err(B2Q_ERR_CUDA, "internal: radix retry did not converge");
}

/* ---- projection (project.cu) ---------------------------------------------------------------------------------------
 * One launch of b2q_k_project over `nf` fragments whose referenced columns are in device memory, writing at most `cap` rows
 * into `d_out` (laid out for `cap` entries).  Returns the rows written and the rows of the chunks the kernel loaded after
 * the call's host wait. */
struct ProjectRun {
  int64_t written = 0, scanned = 0;
  double kernel_ms = 0;
  int32_t error = 0; /* the launch's error word: B2Q_ERR_INTERRUPTED / OUT_OF_TIME when it was stopped */
};
static int32_t project_scan(const B2QQuery& q, const std::vector<const int8_t*>& cols, const std::vector<int64_t>& rows,
                            int8_t* d_out, int64_t cap, cudaStream_t st, const DevInterrupt& intr, ProjectRun* run) {
  const std::vector<int64_t> host = launch_tables(cols, rows, project_rows_per_chunk());
  const int nf = static_cast<int>(rows.size());
  const int64_t chunks = host.back();
  run->written = run->scanned = 0;
  if (chunks == 0 || cap == 0) return B2Q_OK;
  const size_t tab_bytes = DeviceBlock::pad(host.size() * 8), status_bytes = DeviceBlock::pad(static_cast<size_t>(chunks) * 8);
  int8_t* blk = nullptr;
  CU(cudaMallocAsync(reinterpret_cast<void**>(&blk), tab_bytes + status_bytes + 256, st));
  unsigned long long* status = reinterpret_cast<unsigned long long*>(blk + tab_bytes);
  unsigned long long* counters = reinterpret_cast<unsigned long long*>(blk + tab_bytes + status_bytes); /* ticket, done, written, scanned, error */
  unsigned long long h_counters[5] = {};
  cudaEvent_t ev[2] = {};
  cudaError_t e = cudaMemcpyAsync(blk, host.data(), host.size() * 8, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(status, 0, status_bytes + 256, st);
  if (e == cudaSuccess) e = cudaEventCreate(&ev[0]);
  if (e == cudaSuccess) e = cudaEventCreate(&ev[1]);
  if (e == cudaSuccess) e = cudaEventRecord(ev[0], st);
  if (e == cudaSuccess) {
    const int8_t* const* d_cols = reinterpret_cast<const int8_t* const*>(blk);
    const int64_t* d_rows = reinterpret_cast<const int64_t*>(blk) + cols.size();
    const int64_t row_size = q.plan.output_columnar ? 0 : q.plan.row_size;
    e = launch_project(q, d_cols, d_rows, d_rows + nf, nullptr, nf, chunks, 0, d_out, row_size, cap, status, counters, counters + 1,
                       reinterpret_cast<int32_t*>(counters + 4), intr, st);
  }
  if (e == cudaSuccess) e = cudaEventRecord(ev[1], st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(h_counters, counters, sizeof(h_counters), cudaMemcpyDeviceToHost, st);
  cudaFreeAsync(blk, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  float ms = 0;
  if (e == cudaSuccess && cudaEventElapsedTime(&ms, ev[0], ev[1]) == cudaSuccess) run->kernel_ms = ms;
  for (cudaEvent_t x : ev) if (x) cudaEventDestroy(x);
  if (e != cudaSuccess) { cudaGetLastError(); return set_err(e == cudaErrorMemoryAllocation ? B2Q_ERR_OUT_OF_GPU_MEM : B2Q_ERR_CUDA, std::string("projection: ") + cudaGetErrorString(e)); }
  run->written = static_cast<int64_t>(h_counters[2]);
  run->scanned = static_cast<int64_t>(h_counters[3]);
  run->error = static_cast<int32_t>(h_counters[4]);
  return B2Q_OK;
}

/* The same over a host-resident table, through stream_host_table: one launch per slice.  The launches continue one order: the
 * status words are indexed by a chunk number that runs on across slices (chunk_base), every slice has its own ticket, the done
 * flag and the row counters are shared, and each slice's offset words start at its first row in the fragment.  The host reads
 * the done flag after every slice, so a scan limit also stops the copies. */
static int32_t project_scan_host(const B2QQuery& q, const std::vector<const int8_t*>& cols, const std::vector<int64_t>& rows, int8_t* d_out,
                                 int64_t cap, cudaStream_t st, const CallInterrupt* intr, ProjectRun* run, double* h2d_bytes, HostPhases* phases) {
  const int64_t chunk_rows = project_rows_per_chunk();
  int64_t chunks = 0, ns = 0;
  for (int64_t n : rows)
    for (int64_t r = 0; r < n; r += kHostSliceRows, ++ns) chunks += (std::min(kHostSliceRows, n - r) + chunk_rows - 1) / chunk_rows;
  run->written = run->scanned = 0;
  if (!ns || cap == 0) return B2Q_OK;
  /* status words | done, written, scanned, error word, tickets[ns] */
  const size_t status_bytes = DeviceBlock::pad(static_cast<size_t>(chunks) * 8), ctr_bytes = DeviceBlock::pad((4 + ns) * 8);
  int8_t* blk = nullptr;
  CU(cudaMallocAsync(reinterpret_cast<void**>(&blk), status_bytes + ctr_bytes, st));
  unsigned long long* status = reinterpret_cast<unsigned long long*>(blk);
  unsigned long long* counters = reinterpret_cast<unsigned long long*>(blk + status_bytes);
  int32_t* d_error = reinterpret_cast<int32_t*>(counters + 3);
  unsigned long long last[4] = {}; /* done, written, scanned, error word */
  const int64_t row_size = q.plan.output_columnar ? 0 : q.plan.row_size;
  const DevInterrupt dint = intr ? intr->dev : kNoInterrupt;
  HostStream hs;
  hs.paced = true;
  hs.watch = counters;
  hs.watch_bytes = sizeof(last);
  hs.watch_out = last;
  hs.error = d_error;
  hs.intr = intr;
  hs.device_ms = &run->kernel_ms;
  hs.launch = [&](const HostSlice& s) -> int32_t {
    const cudaError_t e = launch_project(q, s.cols, s.rows, s.chunk_start, s.row_base, 1, s.chunks, s.chunk_base, d_out, row_size, cap,
                                         status, counters + 4 + s.index, counters, d_error, dint, st);
    if (e != cudaSuccess) { cudaGetLastError(); return set_err(B2Q_ERR_CUDA, std::string("projection (host table): ") + cudaGetErrorString(e)); }
    return B2Q_OK;
  };
  const cudaError_t e = cudaMemsetAsync(blk, 0, status_bytes + ctr_bytes, st);
  const int32_t rc = e == cudaSuccess ? stream_host_table(q, cols, rows, chunk_rows, hs, st, h2d_bytes, phases)
                                      : set_err(B2Q_ERR_CUDA, std::string("projection (host table): ") + cudaGetErrorString(e));
  cudaFreeAsync(blk, st);
  if (rc != B2Q_OK) return rc;
  run->written = static_cast<int64_t>(last[1]);
  run->scanned = static_cast<int64_t>(last[2]);
  run->error = static_cast<int32_t>(last[3]);
  return B2Q_OK;
}

/* the layout of a projection buffer for `n` entries: row-wise the prefix of a longer buffer, columnar every column moves */
static void projection_relayout(B2QQuery& q, int64_t n) {
  relayout_entries(q.plan, n);
  for (int s = 0; s < q.proj.n; ++s) q.proj.cols[s].out_off = q.plan.slot_offset[s];
}

/* a columnar buffer written for `cap` entries holding `n`: the same columns at stride n, padding zeroed (the bytes the
 * reference's descriptor would have for an n-entry buffer) */
static cudaError_t projection_compact(const B2QPlan& at_cap, const B2QPlan& at_n, const int8_t* d_in, int8_t* d_out, cudaStream_t st) {
  const int64_t n = at_n.entry_count;
  auto one = [&](int64_t in_off, int64_t out_off, int w) -> cudaError_t {
    const int64_t bytes = w * n, padded = (bytes + 7) & ~int64_t(7);
    cudaError_t e = cudaSuccess;
    if (d_in + in_off != d_out + out_off && bytes) e = cudaMemcpyAsync(d_out + out_off, d_in + in_off, bytes, cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess && padded > bytes) e = cudaMemsetAsync(d_out + out_off + bytes, 0, padded - bytes, st);
    return e;
  };
  cudaError_t e = one(0, 0, 8);
  for (int s = 0; s < at_n.num_slots && e == cudaSuccess; ++s) e = one(at_cap.slot_offset[s], at_n.slot_offset[s], at_n.slot_padded_width[s]);
  return e;
}

/* COUNT(*) over the quals of a projection unit: the pre-flight that sizes a projection without a scan limit */
static int32_t projection_count(const B2QTableInfo* tbl, const B2QExecUnit* u, const B2QCompilationOptions* co,
                                const B2QExecutionOptions* eo, cudaStream_t st, const std::shared_ptr<CallInterrupt>& intr,
                                int64_t* count, double* h2d_bytes) {
  std::vector<B2QExpr> exprs(u->exprs, u->exprs + u->num_exprs);
  B2QExpr cnt;
  memset(&cnt, 0, sizeof(cnt));
  cnt.kind = B2Q_EXPR_AGG;
  cnt.ti.type = B2Q_kBIGINT;
  cnt.op = B2Q_kCOUNT;
  cnt.left = cnt.right = -1;
  exprs.push_back(cnt);
  const int32_t target = static_cast<int32_t>(exprs.size()) - 1;
  B2QExecUnit cu = *u;
  cu.exprs = exprs.data();
  cu.num_exprs = static_cast<int32_t>(exprs.size());
  cu.target_exprs = &target;
  cu.num_target_exprs = 1;
  cu.num_order_entries = 0;
  cu.has_limit = 0;
  cu.limit = cu.offset = 0;
  cu.scan_limit = 0;
  B2QExecutionOptions ceo = *eo;
  ceo.bigint_count = 1;
  ceo.result_on_device = 0;
  ceo.output_columnar_hint = 0;
  ceo.force_kernel = 0;
  B2QPartial* p = nullptr;
  int32_t rc = execute_partial_attempt(nullptr, tbl, &cu, co, &ceo, 0, st, false, false, intr, &p);
  if (rc != B2Q_OK) return rc;
  std::unique_ptr<B2QPartial> own(p);
  B2QResultSet* crs = nullptr;
  rc = finalize_impl(p, st, &crs);
  if (rc != B2Q_OK) return rc;
  std::unique_ptr<B2QResultSet> rs(crs);
  B2QTargetValue v;
  b2q_read_target(rs->q.plan, rs->buf, 0, 0, false, &v);
  *count = v.is_null ? 0 : v.ival;
  *h2d_bytes += rs->h2d_bytes;
  return B2Q_OK;
}

/* Executor::executeWorkUnit for a projection unit (QueryDescriptionType::Projection, is_agg = false) */
static int32_t execute_projection_impl(const B2QTableInfo* tbl, const B2QExecUnit* u, const B2QCompilationOptions* co,
                                       const B2QExecutionOptions* eo, const std::shared_ptr<CallInterrupt>& intr, B2QResultSet** out);
static int32_t execute_projection(const B2QTableInfo* tbl, const B2QExecUnit* u, const B2QCompilationOptions* co,
                                  const B2QExecutionOptions* eo, B2QResultSet** out) {
  const auto intr = CallInterrupt::from(eo);
  return intr->resolve(execute_projection_impl(tbl, u, co, eo, intr, out));
}
static int32_t execute_projection_impl(const B2QTableInfo* tbl, const B2QExecUnit* u, const B2QCompilationOptions* co,
                                       const B2QExecutionOptions* eo, const std::shared_ptr<CallInterrupt>& intr, B2QResultSet** out) {
  if (!tbl || !u || !co || !eo || !out) return set_err(B2Q_ERR_INVALID_ARGUMENT, "null argument");
  if (co->device_type != B2Q_DEVICE_GPU) return set_err(B2Q_ERR_UNSUPPORTED, "device_type must be GPU: this path has no CPU execution");
  std::unique_ptr<B2QResultSet> rs(new B2QResultSet());
  std::string err;
  int32_t rc = make_query(u, tbl, eo, 0, false, !co->ignore_deleted_column, &rs->q, &err);
  if (rc != B2Q_OK) return set_err(rc, err);
  if (!have_device()) return set_err(B2Q_ERR_NO_DEVICE, "no CUDA device visible; this path has no CPU fallback");
  if (tbl->memory_level != B2Q_GPU_LEVEL && tbl->memory_level != B2Q_CPU_LEVEL)
    return set_err(B2Q_ERR_INVALID_ARGUMENT, "memory_level must be B2Q_CPU_LEVEL or B2Q_GPU_LEVEL");
  if (eo->device_ordinal >= 0) CU(cudaSetDevice(eo->device_ordinal));
  int device = 0;
  CU(cudaGetDevice(&device));
  configure_pool_once(device);
  cudaStream_t st = nullptr;
  CU(intr->start(device, st));
  const bool filter_deleted = !co->ignore_deleted_column;
  B2QQuery& q = rs->q;
  /* fragments in fragment-id order (the order resultsUnion gives per-fragment results), skipped ones left out */
  std::vector<int> frags = scanned_fragments(*u, *tbl, filter_deleted, &rs->frags_scanned, &rs->frags_skipped);
  std::stable_sort(frags.begin(), frags.end(), [&](int a, int b) { return tbl->fragments[a].fragment_id < tbl->fragments[b].fragment_id; });
  std::vector<const int8_t*> cols;
  std::vector<int64_t> rows;
  rc = fragment_columns(q, *tbl, frags, nullptr, &cols, &rows); /* a projection unit has no join level */
  if (rc != B2Q_OK) return rc;
  const int64_t tuples = std::accumulate(rows.begin(), rows.end(), int64_t(0));
  /* capacity: LIMIT 0 is an empty result (RelSort::isEmptyResult); else the scan limit, never more than the rows scanned; else
   * the exact number of passing rows (the pre-flight: one more scan and one more host wait) */
  int64_t cap = std::min<int64_t>(u->scan_limit, tuples);
  if (q.has_limit && q.limit == 0) {
    cap = 0;
  } else if (u->scan_limit == 0) {
    rc = projection_count(tbl, u, co, eo, st, intr, &cap, &rs->h2d_bytes);
    if (rc != B2Q_OK) return rc;
    rs->launches += set_bytes(q) ? 3 : 2; /* its b2q_k_init and scan, and its own set build */
    if (intr->interrupted()) return set_err(B2Q_ERR_INTERRUPTED, "the query was interrupted (b2q_interrupt on its token) after its row count");
  }
  projection_relayout(q, cap);
  const B2QPlan at_cap = q.plan;
  int8_t* d_out = nullptr;
  /* the output buffer, followed by the bitmaps of the set terms */
  const size_t out_bytes = DeviceBlock::pad(static_cast<size_t>(std::max<int64_t>(at_cap.buffer_size, 8)));
  CU(cudaMallocAsync(reinterpret_cast<void**>(&d_out), out_bytes + set_bytes(q), st));
  if (set_bytes(q) && !rows.empty() && cap) {
    int n = 0;
    const cudaError_t e = build_sets(q, d_out + out_bytes, &n, st);
    if (e != cudaSuccess) { cudaGetLastError(); cudaFreeAsync(d_out, st); return set_err(B2Q_ERR_CUDA, std::string("IN-list bitmaps: ") + cudaGetErrorString(e)); }
    rs->launches += n;
  }
  ProjectRun run;
  if (tbl->memory_level == B2Q_CPU_LEVEL) rc = project_scan_host(q, cols, rows, d_out, cap, st, intr.get(), &run, &rs->h2d_bytes, &rs->host);
  else rc = project_scan(q, cols, rows, d_out, cap, st, intr->dev, &run);
  if (rc == B2Q_OK && run.error) rc = device_error(run.error);
  if (rc != B2Q_OK) { cudaFreeAsync(d_out, st); return rc; }
  rs->launches += rows.empty() ? 0 : 1;
  rs->scan_ms = run.kernel_ms;
  rs->rows_scanned = run.scanned;
  /* the result holds exactly the rows written (compactProjectionBuffersGpu, QueryMemoryInitializer.cpp:1408-1431) */
  projection_relayout(q, run.written);
  int8_t* d_res = d_out;
  cudaError_t e = cudaSuccess;
  if (q.plan.output_columnar) {
    if (run.written < cap) {
      d_res = nullptr;
      e = cudaMallocAsync(reinterpret_cast<void**>(&d_res), std::max<int64_t>(q.plan.buffer_size, 8), st);
      if (e == cudaSuccess) e = projection_compact(at_cap, q.plan, d_out, d_res, st);
      cudaFreeAsync(d_out, st);
    } else {
      e = projection_compact(at_cap, q.plan, d_out, d_out, st); /* zero the column padding only */
    }
  }
  if (e != cudaSuccess) { if (d_res) cudaFreeAsync(d_res, st); cudaGetLastError(); return set_err(B2Q_ERR_CUDA, std::string("projection compaction: ") + cudaGetErrorString(e)); }
  const bool want_sort = q.n_order > 0 || q.has_limit || q.offset > 0;
  if (q.plan.buffer_size && want_sort) {
    rc = sort_keep_rows(rs.get(), d_res, eo->result_on_device != 0, device, st, intr.get());
    if (rc != B2Q_OK) return rc;
    *out = rs.release();
    return B2Q_OK;
  }
  rs->buf_size = static_cast<size_t>(q.plan.buffer_size);
  if (!rs->buf_size) {
    cudaFreeAsync(d_res, st);
  } else if (eo->result_on_device) {
    rs->d_buf = d_res;
    rs->device = device;
  } else {
    rs->buf = pinned_cache().get(rs->buf_size, &rs->buf_cap);
    if (!rs->buf) { cudaFreeAsync(d_res, st); return set_err(B2Q_ERR_INVALID_ARGUMENT, "out of (pinned) host memory for the result buffer"); }
    e = cudaMemcpyAsync(rs->buf, d_res, rs->buf_size, cudaMemcpyDeviceToHost, st);
    rs->d2h_bytes = static_cast<int64_t>(rs->buf_size);
    cudaFreeAsync(d_res, st);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { cudaGetLastError(); return set_err(B2Q_ERR_CUDA, std::string("projection result: ") + cudaGetErrorString(e)); }
  *out = rs.release();
  return B2Q_OK;
}

static bool is_projection_unit(const B2QExecUnit* u) {
  if (!u || u->has_estimator || u->num_groupby_exprs != 0 || u->num_target_exprs <= 0 || !u->target_exprs || !u->exprs) return false;
  for (int i = 0; i < u->num_target_exprs; ++i) {
    const int t = u->target_exprs[i];
    if (t < 0 || t >= u->num_exprs || u->exprs[t].kind != B2Q_EXPR_COLUMN_VAR) return false;
  }
  return true;
}

/* The entry points select eo->device_ordinal / the partial's / the communicator's device; the caller gets its own current
 * device back when they return (the work they enqueued stays bound to its stream). */
struct CallerDevice {
  int dev = -1;
  CallerDevice() { if (cudaGetDevice(&dev) != cudaSuccess) { dev = -1; cudaGetLastError(); } }
  ~CallerDevice() {
    int now = -1;
    if (dev >= 0 && cudaGetDevice(&now) == cudaSuccess && now != dev) cudaSetDevice(dev);
  }
};

/* what columnar.cu (b2q_rs_device_columns) reads of a result set */
namespace b2q {
bool rs_source(const B2QResultSet* rs, RsSource* out) {
  if (!rs) return false;
  *out = RsSource{&rs->q.plan, rs->d_buf, rs->buf, rs->buf_size, rs->d_buf ? rs->device : -1, rs->perm.data(), rs->perm.size(),
                  rs->drop_first, rs->keep_first};
  return true;
}
DevSortLayout sort_layout_for(const B2QPlan& p) { return sort_layout_of(p); }
int32_t report_error(int32_t code, const std::string& msg) { return set_err(code, msg); }
bool device_present() { return have_device(); }
}  // namespace b2q

extern "C" {

int32_t b2q_abi_version(void) { return B2Q_ABI_VERSION; }
const char* b2q_last_error_message(void) { return g_err.c_str(); }
const char* b2q_error_string(int32_t code) {
  switch (code) {
    case B2Q_OK: return "No Error";
    case B2Q_ERR_DIV_BY_ZERO: return "Division by zero";
    case B2Q_ERR_OUT_OF_GPU_MEM: return "Query couldn't keep the entire working set of columns in GPU memory";
    case B2Q_ERR_OUT_OF_SLOTS: return "Out of Slots";
    case B2Q_ERR_OVERFLOW_OR_UNDERFLOW: return "Overflow or underflow";
    case B2Q_ERR_OUT_OF_TIME: return "Query execution has exceeded the time limit";
    case B2Q_ERR_INTERRUPTED: return "Query execution has been interrupted";
    case B2Q_ERR_UNSUPPORTED: return "Feature outside the scan/filter/group-by/aggregate path";
    case B2Q_ERR_CARDINALITY_ESTIMATION_REQUIRED: return "CardinalityEstimationRequired";
    case B2Q_ERR_INVALID_ARGUMENT: return "Invalid argument";
    case B2Q_ERR_NO_DEVICE: return "No CUDA device (no CPU fallback on this path)";
    case B2Q_ERR_CUDA: return "CUDA error";
    case B2Q_ERR_KEY_OUT_OF_RANGE: return "Group key outside the chunk-stats range";
    default: return code < 0 ? "Out of Slots (-pos)" : "Unknown error";
  }
}
int32_t b2q_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int32_t b2q_plan(const B2QExecUnit* u, const B2QTableInfo* t, const B2QCompilationOptions* co, const B2QExecutionOptions* eo,
                 size_t guess, int32_t has_card, B2QQuery** out) {
  if (!out || !co) return set_err(B2Q_ERR_INVALID_ARGUMENT, "null argument");
  if (co->device_type != B2Q_DEVICE_GPU) return set_err(B2Q_ERR_UNSUPPORTED, "device_type must be GPU: this path has no CPU execution");
  std::unique_ptr<B2QQuery> q(new B2QQuery());
  std::string err;
  const int32_t rc = make_query(u, t, eo, guess, has_card != 0, !co->ignore_deleted_column, q.get(), &err);
  if (rc != B2Q_OK) return set_err(rc, err);
  *out = q.release();
  return B2Q_OK;
}
const B2QPlan* b2q_query_plan(const B2QQuery* q) { return q ? &q->plan : nullptr; }
void b2q_query_free(B2QQuery* q) { delete q; }

int32_t b2q_execute_partial(size_t* guess, int32_t /*is_agg*/, const B2QTableInfo* tbl, const B2QExecUnit* u,
                            const B2QCompilationOptions* co, const B2QExecutionOptions* eo, int32_t has_card,
                            void* stream, B2QPartial** out) {
  CallerDevice restore;
  return execute_partial_impl(guess, tbl, u, co, eo, has_card, static_cast<cudaStream_t>(stream), out);
}

int32_t b2q_execute_work_unit(size_t* guess, int32_t is_agg, const B2QTableInfo* tbl, const B2QExecUnit* u,
                              const B2QCompilationOptions* co, const B2QExecutionOptions* eo, int32_t has_card,
                              B2QResultSet** out) {
  (void)is_agg;
  CallerDevice restore;
  if (is_projection_unit(u) && !u->num_join_quals) return execute_projection(tbl, u, co, eo, out);
  g_trace.begin();
  const auto intr = CallInterrupt::from(eo);
  for (int attempt = 0; attempt < 2; ++attempt) {
    B2QPartial* p = nullptr;
    int32_t rc = execute_partial_attempt(guess, tbl, u, co, eo, has_card, nullptr, attempt == 0 && radix_enabled(), true, intr, &p);
    if (rc == B2Q_OK) {
      rc = finalize_impl(p, nullptr, out);
      g_trace.mark("finalize");
      delete p;
      g_trace.mark("release");
    }
    if (rc != B2Q_RADIX_RETRY) { g_trace.end(); return intr->resolve(rc); }
  }
  return set_err(B2Q_ERR_CUDA, "internal: radix retry did not converge");
}

int32_t b2q_partial_num_arrays(const B2QPartial* p) { return p ? p->q.prog.n_accs : 0; }
int32_t b2q_partial_array(const B2QPartial* p, int32_t i, void** ptr, int64_t* count, int32_t* dtype, int32_t* redop) {
  if (!p || i < 0 || i >= p->q.prog.n_accs) return set_err(B2Q_ERR_INVALID_ARGUMENT, "array index");
  const int op = p->q.prog.accs[i].op;
  if (ptr) *ptr = p->accs[i];
  if (count) *count = op == ACC_NDV ? p->q.plan.buffer_size : op == ACC_BITMAP ? static_cast<int64_t>(acc_array_bytes(p->q, i)) : p->q.plan.entry_count;
  if (dtype) *dtype = op == ACC_SUM_F64 ? B2Q_DT_FLOAT64 : (op == ACC_TOUCH || op == ACC_NDV || op == ACC_BITMAP) ? B2Q_DT_UINT8 : B2Q_DT_INT64;
  if (redop) *redop = (op == ACC_NDV || op == ACC_BITMAP) ? B2Q_RED_BOR : (op == ACC_MIN_I64 || op == ACC_MIN_F64) ? B2Q_RED_MIN : (op == ACC_MAX_I64 || op == ACC_MAX_F64 || op == ACC_TOUCH) ? B2Q_RED_MAX : B2Q_RED_SUM;
  return B2Q_OK;
}
int32_t b2q_partial_is_mergeable(const B2QPartial* p) { return p && p->q.plan.kernel != B2Q_KERNEL_BASELINE_GLOBAL; }
const B2QPlan* b2q_partial_plan(const B2QPartial* p) { return p ? &p->q.plan : nullptr; }
double b2q_partial_kernel_ms(const B2QPartial* p) { return p ? p->scan_ms : 0; }
int32_t b2q_partial_finalize(B2QPartial* p, void* stream, B2QResultSet** out) {
  CallerDevice restore;
  return finalize_impl(p, static_cast<cudaStream_t>(stream), out);
}
void b2q_partial_free(B2QPartial* p) { delete p; }

/* Inner entry: same parameter block as the reference's JIT kernel; writes the reference-layout buffer on the
 * device (params->group_by_buffers[0]) instead of returning a host ResultSet. */
int32_t b2q_launch(const B2QQuery* query, const B2QParams* prm, void* stream) {
  if (!query || !prm) return set_err(B2Q_ERR_INVALID_ARGUMENT, "null argument");
  if (set_bytes(*query))
    return set_err(B2Q_ERR_UNSUPPORTED, "the filter holds an IN list planned as a value set, whose bitmap is built in memory of the call; "
                                        "b2q_launch runs on caller memory only: use b2q_execute_work_unit / b2q_execute_partial");
  if (!have_device()) return set_err(B2Q_ERR_NO_DEVICE, "no CUDA device visible; this path has no CPU fallback");
  if (prm->row_func_mgr) return set_err(B2Q_ERR_UNSUPPORTED, "row function manager");
  if (query->plan.query_desc_type == B2Q_Estimator) return set_err(B2Q_ERR_UNSUPPORTED, "estimator queries run through b2q_execute_work_unit / b2q_execute_partial");
  const bool has_join = query->prog.join.fk_col >= 0;
  if (has_join != (prm->join_hash_tables != nullptr)) return set_err(B2Q_ERR_INVALID_ARGUMENT, "JOIN_HASH_TABLES must be given exactly when the plan has a join level");
  if (!prm->num_fragments || !prm->col_buffers || !prm->num_rows || !prm->group_by_buffers)
    return set_err(B2Q_ERR_INVALID_ARGUMENT, "missing kernel parameter");
  if (prm->num_tables && *prm->num_tables != (has_join ? 2u : 1u)) return set_err(B2Q_ERR_UNSUPPORTED, "number of input tables does not match the plan");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  /* with a join level col_buffers[frag] holds the scanned table's columns followed by the inner table's (the same
   * device pointers in every fragment) */
  const int nf = static_cast<int>(*prm->num_fragments);
  const int nc = query->prog.n_cols;
  std::vector<const int8_t*> cols(static_cast<size_t>(nf) * nc);
  std::vector<int64_t> rows(nf);
  for (int f = 0; f < nf; ++f) {
    rows[f] = prm->num_rows[f];
    for (int c = 0; c < nc; ++c) cols[static_cast<size_t>(f) * nc + c] = prm->col_buffers[f][query->col_ids[c]];
  }
  if (query->plan.query_desc_type == B2Q_Projection) { /* rows at TOTAL_MATCHED++ up to MAX_MATCHED, in (fragment, row) order */
    B2QQuery q = *query;
    const int64_t cap = prm->max_matched ? *prm->max_matched : q.plan.entry_count;
    if (cap < 0) return set_err(B2Q_ERR_INVALID_ARGUMENT, "MAX_MATCHED is negative");
    projection_relayout(q, cap);
    int64_t* d_out = nullptr;
    CU(cudaMemcpyAsync(&d_out, prm->group_by_buffers, sizeof(int64_t*), cudaMemcpyDefault, st));
    CU(cudaStreamSynchronize(st));
    ProjectRun run;
    const int32_t rc = project_scan(q, cols, rows, reinterpret_cast<int8_t*>(d_out), cap, st, kNoInterrupt, &run);
    if (rc != B2Q_OK) return rc;
    const int32_t matched = static_cast<int32_t>(std::min<int64_t>(run.written, INT32_MAX));
    if (prm->total_matched) CU(cudaMemcpy(prm->total_matched, &matched, sizeof(int32_t), cudaMemcpyDefault));
    const int32_t ok = 0;
    if (prm->error_codes) CU(cudaMemcpy(prm->error_codes, &ok, sizeof(int32_t), cudaMemcpyDefault));
    g_launch_join_table = B2Q_JOIN_TABLE_NONE; /* projections have no join level */
    return B2Q_OK;
  }
  B2QPartial p;
  p.q = *query;
  if (prm->init_agg_value) {
    for (int s = 0; s < p.q.plan.num_slots; ++s) { p.q.plan.init_vals[s] = prm->init_agg_value[s]; p.q.layout.slots[s].init_val = prm->init_agg_value[s]; }
  }
  CU(cudaGetDevice(&p.device));
  int32_t rc = alloc_partial(p, launch_table_bytes(nf, nc), st);
  if (rc != B2Q_OK) return rc;
  /* with a join level JOIN_HASH_TABLES[0] is the built one-to-one table */
  if (has_join) {
    p.join_buff = reinterpret_cast<const int32_t*>(static_cast<intptr_t>(prm->join_hash_tables[0]));
    p.q.prog.join.packed_col = -1; /* the caller's table is the reference's plain int32 layout */
    p.q.prog.join.slot16 = 0;
    if (p.q.smem.join_off >= 0) { p.q.smem.total_bytes = p.q.smem.join_off; p.q.smem.join_off = -1; p.q.smem.join_bytes = 0; } /* ... and is read in place */
  }
  if (nf > 0) {
    rc = scan_device_fragments(p, cols, rows, st, false);
    if (rc != B2Q_OK) return rc;
  }
  int64_t* d_out = nullptr;
  CU(cudaMemcpyAsync(&d_out, prm->group_by_buffers, sizeof(int64_t*), cudaMemcpyDefault, st));
  CU(cudaStreamSynchronize(st));
  rc = normalize_partial(p, st);
  if (rc != B2Q_OK) return rc;
  CU(launch_materialize(p.q, p.accs, p.keys, reinterpret_cast<int8_t*>(d_out), st));
  int32_t dev_err = 0;
  CU(cudaMemcpyAsync(&dev_err, p.d_error, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (prm->error_codes) cudaMemcpy(prm->error_codes, &dev_err, sizeof(int32_t), cudaMemcpyDefault);
  if (!dev_err) g_launch_join_table = has_join ? B2Q_JOIN_TABLE_CALLER : B2Q_JOIN_TABLE_NONE;
  return dev_err;
}

/* ---- ResultSet surface ---------------------------------------------------------------------------------- */
/* ResultSet::entryCount(): permutation_.size() once sorted, else the descriptor's entry count (ResultSetIteration.cpp:752-754) */
size_t b2q_rs_entry_count(const B2QResultSet* rs) {
  if (!rs) return 0;
  return rs->perm.empty() ? static_cast<size_t>(rs->q.plan.entry_count) : rs->perm.size();
}
size_t b2q_rs_col_count(const B2QResultSet* rs) { return rs ? static_cast<size_t>(rs->q.plan.num_targets) : 0; }
int32_t b2q_rs_is_row_at_empty(const B2QResultSet* rs, size_t e) { /* ResultSet::isRowAtEmpty; an index past the storage is empty */
  if (!rs || e >= static_cast<size_t>(rs->q.plan.entry_count) || !ensure_host(rs)) return 1;
  return rs_is_empty_entry(rs, static_cast<int64_t>(e));
}
static size_t truncated_row_count(size_t total, size_t keep_first, size_t drop_first) { /* get_truncated_row_count, ResultSet.cpp */
  if (total <= drop_first) return 0;
  const size_t rest = total - drop_first;
  return keep_first ? std::min(rest, keep_first) : rest;
}
size_t b2q_rs_row_count(const B2QResultSet* rs) { /* ResultSet::rowCountImpl (ResultSet.cpp:565-600) */
  if (!rs || !ensure_host(rs)) return 0;
  if (!rs->perm.empty()) return truncated_row_count(rs->perm.size(), rs->keep_first, rs->drop_first);
  if (rs->cached_rows < 0) {
    int64_t n = 0;
    for (int64_t e = 0; e < rs->q.plan.entry_count; ++e) n += !rs_is_empty_entry(rs, e);
    const_cast<B2QResultSet*>(rs)->cached_rows = n;
  }
  return truncated_row_count(static_cast<size_t>(rs->cached_rows), rs->keep_first, rs->drop_first);
}
int32_t b2q_rs_is_empty(const B2QResultSet* rs) { return b2q_rs_row_count(rs) == 0; }
B2QTypeInfo b2q_rs_get_col_type(const B2QResultSet* rs, size_t col) {
  if (!rs || col >= static_cast<size_t>(rs->q.plan.num_targets)) return B2QTypeInfo{0, 0, 0}; /* kNULLT */
  return b2q_target_col_type(rs->q.plan.targets[col]);
}
void b2q_rs_move_to_begin(B2QResultSet* rs) { if (rs) { rs->cursor = 0; rs->fetched = 0; } }

static void read_entry(const B2QResultSet* rs, int64_t entry, B2QTargetValue* row, bool decimal_to_double);

int32_t b2q_rs_get_next_row(B2QResultSet* rs, B2QTargetValue* row, int32_t /*translate_strings: results carry ids*/, int32_t decimal_to_double) {
  if (!rs || !row || rs->q.plan.query_desc_type == B2Q_Estimator || !ensure_host(rs)) return 0;
  /* getNextRowImpl + advanceCursorToNextEntry (ResultSetIteration.cpp:320-340, :731-750) */
  const int64_t n_entries = static_cast<int64_t>(b2q_rs_entry_count(rs));
  int64_t entry = 0;
  do {
    if (rs->keep_first && rs->fetched >= rs->drop_first + rs->keep_first) return 0;
    while (rs->cursor < n_entries && rs_is_empty_entry(rs, rs->perm.empty() ? rs->cursor : rs->perm[rs->cursor])) ++rs->cursor;
    if (rs->cursor >= n_entries) return 0;
    entry = rs->perm.empty() ? rs->cursor : rs->perm[rs->cursor];
    ++rs->cursor;
    ++rs->fetched;
  } while (rs->drop_first && rs->fetched <= rs->drop_first);
  read_entry(rs, entry, row, decimal_to_double != 0);
  return 1;
}

/* ResultSet::getRowAt(logical_index) / getRowAtNoTranslations (ResultSetIteration.cpp:266-284): the row of entry
 * permutation_[logical_index] (or logical_index itself when the set is not sorted); 0 = past entryCount() or an empty entry.
 * Random access: it neither moves the getNextRow cursor nor looks at dropFirstN / keepFirstN (as in the reference). */
int32_t b2q_rs_get_row_at(const B2QResultSet* rs, size_t logical_index, B2QTargetValue* row, int32_t /*translate_strings*/, int32_t decimal_to_double) {
  if (!rs || !row || rs->q.plan.query_desc_type == B2Q_Estimator || !ensure_host(rs)) return 0;
  if (logical_index >= b2q_rs_entry_count(rs)) return 0;
  const int64_t entry = rs->perm.empty() ? static_cast<int64_t>(logical_index) : static_cast<int64_t>(rs->perm[logical_index]);
  if (rs_is_empty_entry(rs, entry)) return 0;
  read_entry(rs, entry, row, decimal_to_double != 0);
  return 1;
}

/* getRowAt / getTargetValueFromBufferRowwise|Colwise (ResultSetIteration.cpp:820-1000) for one storage entry; the per-slot
 * decode is b2q_read_target (b2q_internal.h), which the device conversion (columnar.cu) runs too */
static void read_entry(const B2QResultSet* rs, int64_t entry, B2QTargetValue* row, bool decimal_to_double) {
  for (int i = 0; i < rs->q.plan.num_targets; ++i) b2q_read_target(rs->q.plan, rs->buf, entry, i, decimal_to_double, &row[i]);
}

/* ---- ColumnarResults (QueryEngine/ColumnarResults.cpp:256-392, materializeAllColumnsThroughIteration :1043-1140):
 * the rows of a result set, in iteration order (permutation, OFFSET and LIMIT applied), as one contiguous array per
 * target in the target type's own width; NULLs stay the type's inline sentinel (toBuffer, ColumnarResults.cpp:42-90).
 * Host code in the reference as well; rows are converted by blocks on `num_threads` threads. */
struct B2QColumnarResults {
  size_t num_rows = 0;
  std::vector<B2QTypeInfo> types;
  std::vector<std::vector<int8_t>> cols;
};

int32_t b2q_columnar_results_create(const B2QResultSet* rs, int32_t num_threads, B2QColumnarResults** out) {
  if (!rs || !out) return set_err(B2Q_ERR_INVALID_ARGUMENT, "null argument");
  if (rs->q.plan.query_desc_type == B2Q_Estimator) return set_err(B2Q_ERR_UNSUPPORTED, "an estimator result has no rows");
  if (!ensure_host(rs)) return rs->host_rc;
  const B2QPlan& p = rs->q.plan;
  /* the storage entries the cursor would visit */
  std::vector<int64_t> entries;
  const int64_t n_entries = static_cast<int64_t>(b2q_rs_entry_count(rs));
  for (int64_t i = 0; i < n_entries; ++i) {
    const int64_t e = rs->perm.empty() ? i : rs->perm[i];
    if (!rs_is_empty_entry(rs, e)) entries.push_back(e);
  }
  const size_t first = std::min(entries.size(), rs->drop_first);
  const size_t n = truncated_row_count(entries.size(), rs->keep_first, rs->drop_first);
  std::unique_ptr<B2QColumnarResults> cr(new B2QColumnarResults);
  cr->num_rows = n;
  const int nt = p.num_targets;
  cr->types.resize(nt);
  cr->cols.resize(nt);
  std::vector<int> width(nt);
  for (int c = 0; c < nt; ++c) {
    cr->types[c] = b2q_rs_get_col_type(rs, c);
    width[c] = b2q_type_size(cr->types[c].type);
    if (width[c] <= 0) return set_err(B2Q_ERR_UNSUPPORTED, "target type has no fixed width");
    cr->cols[c].resize(std::max<size_t>(n, 1) * width[c]);
  }
  auto convert = [&](size_t lo, size_t hi) {
    B2QTargetValue row[B2Q_MAX_TARGETS];
    for (size_t r = lo; r < hi; ++r) {
      read_entry(rs, entries[first + r], row, false); /* decimals stay scaled int64 (ColumnarResults.cpp:155,550 getRowAtNoTranslations / getNextRow(false, false)) */
      for (int c = 0; c < nt; ++c) b2q_store_target(row[c], width[c], cr->cols[c].data() + r * width[c]);
    }
  };
  const size_t threads = std::max<size_t>(1, std::min<size_t>(num_threads > 0 ? num_threads : 1, n / 65536 + 1));
  if (threads == 1) convert(0, n);
  else {
    std::vector<std::thread> pool;
    const size_t step = (n + threads - 1) / threads;
    for (size_t t = 0; t < threads; ++t) pool.emplace_back(convert, std::min(n, t * step), std::min(n, (t + 1) * step));
    for (auto& th : pool) th.join();
  }
  *out = cr.release();
  return B2Q_OK;
}
size_t b2q_columnar_results_size(const B2QColumnarResults* cr) { return cr ? cr->num_rows : 0; }
size_t b2q_columnar_results_num_columns(const B2QColumnarResults* cr) { return cr ? cr->cols.size() : 0; }
const int8_t* b2q_columnar_results_column(const B2QColumnarResults* cr, size_t col, B2QTypeInfo* ti) {
  if (!cr || col >= cr->cols.size()) return nullptr;
  if (ti) *ti = cr->types[col];
  return cr->cols[col].data();
}
void b2q_columnar_results_free(B2QColumnarResults* cr) { delete cr; }

const int8_t* b2q_rs_storage_buffer(const B2QResultSet* rs, size_t* size_bytes) {
  const bool ok = rs && ensure_host(rs);
  if (size_bytes) *size_bytes = ok ? rs->buf_size : 0;
  return ok ? rs->buf : nullptr;
}
const B2QPlan* b2q_rs_query_mem_desc(const B2QResultSet* rs) { return rs ? &rs->q.plan : nullptr; }
double b2q_rs_kernel_ms(const B2QResultSet* rs) { return rs ? rs->scan_ms : 0; }

/* ResultSet::getNDVEstimator (CardinalityEstimator.cpp:33-52) */
size_t b2q_rs_get_ndv_estimator(const B2QResultSet* rs) {
  if (!rs || rs->q.plan.query_desc_type != B2Q_Estimator || !rs->buf) return 0;
  size_t bits_set = 0;
  const uint64_t* w = reinterpret_cast<const uint64_t*>(rs->buf);
  for (size_t i = 0; i < rs->buf_size / 8; ++i) bits_set += static_cast<size_t>(__builtin_popcountll(w[i]));
  if (bits_set == 0) return 1; /* empty result: one slot is enough */
  const size_t total_bits = rs->buf_size * 8;
  const double ratio = static_cast<double>(total_bits - bits_set) / static_cast<double>(total_bits);
  if (ratio == 0.) return 0;   /* saturated: no usable estimate */
  return static_cast<size_t>(-static_cast<double>(total_bits) * log(ratio));
}
const int8_t* b2q_rs_estimator_buffer(const B2QResultSet* rs, size_t* size_bytes) {
  const bool ok = rs && rs->q.plan.query_desc_type == B2Q_Estimator;
  if (size_bytes) *size_bytes = ok ? rs->buf_size : 0;
  return ok ? rs->buf : nullptr;
}

/* ResultSet::sort (ResultSet.cpp:781-849) on an existing result set: the storage buffer goes to the device (a result_on_device
 * set is sorted where it lies), the kernels of sort.cu order the non-empty entries, the permutation comes back (the buffer
 * itself is not moved). */
int32_t b2q_rs_sort(B2QResultSet* rs, const B2QOrderEntry* order_entries, int32_t n_entries, size_t top_n) {
  if (!rs || (n_entries && !order_entries)) return set_err(B2Q_ERR_INVALID_ARGUMENT, "null argument");
  if (n_entries < 0 || n_entries > B2Q_MAX_ORDER_ENTRIES) return set_err(B2Q_ERR_UNSUPPORTED, "more ORDER BY entries than the path carries");
  const B2QPlan& plan = rs->q.plan;
  for (int i = 0; i < n_entries; ++i) {
    if (order_entries[i].tle_no < 1 || order_entries[i].tle_no > plan.num_targets) return set_err(B2Q_ERR_INVALID_ARGUMENT, "order entry refers to a target that does not exist");
    /* ResultSet::sort orders dictionary strings through the dictionary (ResultSet.cpp:1424-1436), which this path does not hold */
    const B2QTargetInfo& t = plan.targets[order_entries[i].tle_no - 1];
    const bool minmax = t.is_agg && t.agg_arg_type.type != 0 && (t.agg_kind == B2Q_kMIN || t.agg_kind == B2Q_kMAX);
    if (b2q_is_dict_string(minmax ? t.agg_arg_type.type : t.sql_type.type))
      return set_err(B2Q_ERR_UNSUPPORTED, "ORDER BY a dictionary-encoded string needs the dictionary");
  }
  if (!have_device()) return set_err(B2Q_ERR_NO_DEVICE, "no CUDA device visible; this path has no CPU fallback");
  rs->perm.clear();
  rs->cursor = 0; rs->fetched = 0;
  if (!rs->buf_size || plan.entry_count <= 0) return B2Q_OK;
  cudaStream_t st = nullptr;
  CallerDevice restore;
  if (rs->d_buf) CU(cudaSetDevice(rs->device));
  int8_t* d_buf = nullptr;
  int8_t* d_scratch = nullptr;
  cudaError_t e = cudaSuccess;
  if (!rs->d_buf) {
    CU(cudaMallocAsync(reinterpret_cast<void**>(&d_buf), rs->buf_size, st));
    e = cudaMemcpyAsync(d_buf, rs->buf, rs->buf_size, cudaMemcpyHostToDevice, st);
  }
  if (e == cudaSuccess) e = cudaMallocAsync(reinterpret_cast<void**>(&d_scratch), sort_scratch_bytes(plan.entry_count), st);
  const DevSortLayout L = sort_layout_of(plan);
  DevSortKey keys[B2Q_MAX_ORDER_ENTRIES];
  for (int i = 0; i < n_entries; ++i) keys[i] = sort_key_of(plan, order_entries[i]);
  const uint32_t* d_perm = nullptr;
  int64_t n = 0;
  int launches = 0;
  bool stopped = false; /* ResultSet::sort takes no interrupt token */
  if (e == cudaSuccess) e = sort_device(L, keys, n_entries, rs->d_buf ? rs->d_buf : d_buf, d_scratch, st, &d_perm, &n, &launches, static_cast<int64_t>(top_n),
                                        nullptr, &stopped);
  if (e == cudaSuccess) {
    const int64_t keep = top_n && static_cast<int64_t>(top_n) < n ? static_cast<int64_t>(top_n) : n;
    rs->perm.resize(static_cast<size_t>(keep));
    if (keep) e = cudaMemcpyAsync(rs->perm.data(), d_perm, static_cast<size_t>(keep) * 4, cudaMemcpyDeviceToHost, st);
  }
  if (d_scratch) cudaFreeAsync(d_scratch, st);
  if (d_buf) cudaFreeAsync(d_buf, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { cudaGetLastError(); rs->perm.clear(); return set_err(B2Q_ERR_CUDA, std::string("sort: ") + cudaGetErrorString(e)); }
  rs->launches += launches;
  rs->sorted = true;
  return B2Q_OK;
}
void b2q_rs_drop_first_n(B2QResultSet* rs, size_t n) { if (rs) { rs->drop_first = n; rs->cursor = 0; rs->fetched = 0; } }   /* ResultSet::dropFirstN :63-66 */
void b2q_rs_keep_first_n(B2QResultSet* rs, size_t n) { if (rs) { rs->keep_first = n; rs->cursor = 0; rs->fetched = 0; } }   /* ResultSet::keepFirstN :58-61 */
int64_t b2q_rs_stat(const B2QResultSet* rs, int32_t which) {
  if (!rs) return -1;
  switch (which) {
    case B2Q_STAT_FRAGMENTS_SCANNED: return rs->frags_scanned;
    case B2Q_STAT_FRAGMENTS_SKIPPED: return rs->frags_skipped;
    case B2Q_STAT_KERNEL_LAUNCHES: return rs->launches;
    case B2Q_STAT_H2D_BYTES: return static_cast<int64_t>(rs->h2d_bytes);
    case B2Q_STAT_SORT_US: return static_cast<int64_t>(rs->sort_ms * 1000.0);
    case B2Q_STAT_HOST_SETUP_US: return static_cast<int64_t>(rs->host.setup_us);
    case B2Q_STAT_HOST_STREAM_US: return static_cast<int64_t>(rs->host.stream_us);
    case B2Q_STAT_HOST_TEARDOWN_US: return static_cast<int64_t>(rs->host.teardown_us);
    case B2Q_STAT_RESULT_D2H_BYTES: return rs->d2h_bytes;
    case B2Q_STAT_ROWS_SCANNED: return rs->rows_scanned;
    case B2Q_STAT_JOIN_TABLE: return rs->join_table;
    default: return -1;
  }
}
int64_t b2q_last_launch_stat(int32_t which) { return which == B2Q_STAT_JOIN_TABLE ? g_launch_join_table : -1; }
void b2q_rs_free(B2QResultSet* rs) { delete rs; }

/* A ResultSet over storage the caller already holds: ResultSet(targets, device_type, query_mem_desc, row_set_mem_owner, ...)
 * followed by allocateStorage(buffer, ...) (ResultSet.h:183-217, ResultSet.cpp allocateStorage) — how ResultSetTest and the
 * reduction code wrap a filled group-by buffer.  The descriptor is the planned query's; the bytes are copied.  Nothing
 * is computed here: it is the read-out half (rowCount / getNextRow / isRowAtEmpty / ColumnarResults) on its own. */
int32_t b2q_rs_create_from_storage(const B2QQuery* q, const int8_t* storage, size_t size_bytes, B2QResultSet** out) {
  if (!q || !out || (!storage && size_bytes)) return set_err(B2Q_ERR_INVALID_ARGUMENT, "null argument");
  if (q->plan.query_desc_type == B2Q_Estimator) return set_err(B2Q_ERR_UNSUPPORTED, "an estimator result is a bitmap, not a group-by buffer");
  if (size_bytes != static_cast<size_t>(q->plan.buffer_size)) return set_err(B2Q_ERR_INVALID_ARGUMENT, "storage size differs from the descriptor's buffer size");
  std::unique_ptr<B2QResultSet> rs(new B2QResultSet());
  rs->q = *q;
  rs->heap_buf = true;
  rs->buf_cap = std::max<size_t>(size_bytes, 8);
  rs->buf = static_cast<int8_t*>(malloc(rs->buf_cap));
  if (!rs->buf) return set_err(B2Q_ERR_INVALID_ARGUMENT, "out of host memory");
  if (size_bytes) memcpy(rs->buf, storage, size_bytes);
  rs->buf_size = size_bytes;
  *out = rs.release();
  return B2Q_OK;
}

/* ---- multi-GPU entry points ------------------------------------------------------------------------------------ */
int32_t b2q_comm_unique_id(void* id128) {
  std::string why;
  const NcclApi* api = nccl_api(&why);
  if (!api) return set_err(B2Q_ERR_UNSUPPORTED, why);
  if (!id128) return set_err(B2Q_ERR_INVALID_ARGUMENT, "null argument");
  static_assert(sizeof(ncclUniqueId) == B2Q_COMM_ID_BYTES, "ncclUniqueId size");
  ncclUniqueId id;
  const ncclResult_t r = api->GetUniqueId(&id);
  if (r != ncclSuccess) return set_err(B2Q_ERR_CUDA, std::string("ncclGetUniqueId: ") + api->GetErrorString(r));
  memcpy(id128, &id, sizeof(id));
  return B2Q_OK;
}

int32_t b2q_comm_init_rank(const void* id128, int32_t nranks, int32_t rank, int32_t device, B2QComm** out) {
  std::string why;
  const NcclApi* api = nccl_api(&why);
  if (!api) return set_err(B2Q_ERR_UNSUPPORTED, why);
  if (!id128 || !out || nranks < 1 || rank < 0 || rank >= nranks) return set_err(B2Q_ERR_INVALID_ARGUMENT, "communicator arguments");
  if (!have_device()) return set_err(B2Q_ERR_NO_DEVICE, "no CUDA device visible");
  CallerDevice restore;
  if (device >= 0) CU(cudaSetDevice(device));
  std::unique_ptr<B2QComm> c(new B2QComm());
  CU(cudaGetDevice(&c->device));
  c->rank = rank;
  c->nranks = nranks;
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  const ncclResult_t r = api->CommInitRank(&c->comm, nranks, id, rank);
  if (r != ncclSuccess) return set_err(B2Q_ERR_CUDA, std::string("ncclCommInitRank: ") + api->GetErrorString(r));
  *out = c.release();
  return B2Q_OK;
}

int32_t b2q_comm_init_all(const int32_t* devices, int32_t ndev, B2QComm** out) {
  std::string why;
  const NcclApi* api = nccl_api(&why);
  if (!api) return set_err(B2Q_ERR_UNSUPPORTED, why);
  if (!devices || !out || ndev < 1 || ndev > 64) return set_err(B2Q_ERR_INVALID_ARGUMENT, "communicator arguments");
  if (!have_device()) return set_err(B2Q_ERR_NO_DEVICE, "no CUDA device visible");
  std::vector<ncclComm_t> comms(ndev);
  std::vector<int> devs(devices, devices + ndev);
  const ncclResult_t r = api->CommInitAll(comms.data(), ndev, devs.data());
  if (r != ncclSuccess) return set_err(B2Q_ERR_CUDA, std::string("ncclCommInitAll: ") + api->GetErrorString(r));
  for (int i = 0; i < ndev; ++i) {
    out[i] = new B2QComm();
    out[i]->comm = comms[i];
    out[i]->rank = i;
    out[i]->nranks = ndev;
    out[i]->device = devs[i];
  }
  return B2Q_OK;
}

void b2q_comm_destroy(B2QComm* c) {
  if (!c) return;
  const NcclApi* api = nccl_api(nullptr);
  if (api && c->comm) api->CommDestroy(c->comm);
  delete c;
}
int32_t b2q_comm_rank(const B2QComm* c) { return c ? c->rank : -1; }
int32_t b2q_comm_size(const B2QComm* c) { return c ? c->nranks : 0; }

int32_t b2q_execute_work_unit_dist(B2QComm* comm, size_t* guess, int32_t /*is_agg*/, const B2QTableInfo* tbl, const B2QExecUnit* u,
                                   const B2QCompilationOptions* co, const B2QExecutionOptions* eo, int32_t has_card, void* stream,
                                   B2QResultSet** out) {
  if (!comm || !eo) return set_err(B2Q_ERR_INVALID_ARGUMENT, "null argument");
  CallerDevice restore;
  return execute_work_unit_rank(comm, guess, tbl, u, co, eo, has_card, static_cast<cudaStream_t>(stream), true, out, nullptr);
}

int32_t b2q_execute_work_unit_multi(B2QComm* const* comms, int32_t ndev, size_t* guess, int32_t /*is_agg*/, const B2QTableInfo* const* tbls,
                                    const B2QExecUnit* u, const B2QCompilationOptions* co, const B2QExecutionOptions* eo, int32_t has_card,
                                    B2QResultSet** out) {
  if (!comms || !tbls || !eo || !out || ndev < 1) return set_err(B2Q_ERR_INVALID_ARGUMENT, "null argument");
  /* one host thread per device (Executor::launchKernelsViaResourceMgr -> ExecutionKernel::run, Execute.cpp:3055-3101,
   * ExecutionKernel.cpp:215-218); device 0 of the list materialises the merged table */
  std::vector<int32_t> rcs(ndev, B2Q_OK);
  std::vector<std::string> msgs(ndev);
  std::vector<std::thread> ths;
  const size_t g = guess ? *guess : 0;
  for (int i = 0; i < ndev; ++i)
    ths.emplace_back([&, i]() {
      size_t gi = g;
      cudaStream_t st = nullptr;
      if (cudaSetDevice(comms[i]->device) != cudaSuccess || cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) {
        cudaGetLastError();
        rcs[i] = B2Q_ERR_CUDA;
        msgs[i] = "device / stream setup";
        return;
      }
      rcs[i] = execute_work_unit_rank(comms[i], &gi, tbls[i], u, co, eo, has_card, st, i == 0, i == 0 ? out : nullptr, nullptr);
      if (rcs[i] != B2Q_OK) msgs[i] = g_err;
      cudaStreamDestroy(st);
    });
  for (auto& t : ths) t.join();
  for (int i = 0; i < ndev; ++i)
    if (rcs[i] != B2Q_OK) {
      if (i != 0 && rcs[0] == B2Q_OK && out && *out) { delete *out; *out = nullptr; }
      return set_err(rcs[i], msgs[i]);
    }
  return B2Q_OK;
}

/* ---- runtime query interrupt ------------------------------------------------------------------------------------------ */
int32_t b2q_interrupt_token_create(B2QInterruptToken** out) {
  if (!out) return set_err(B2Q_ERR_INVALID_ARGUMENT, "null argument");
  *out = nullptr;
  if (!have_device()) return set_err(B2Q_ERR_NO_DEVICE, "no CUDA device visible: an interrupt token is device-mapped host memory");
  std::unique_ptr<B2QInterruptToken> t(new B2QInterruptToken());
  void* p = nullptr;
  /* mapped: the kernels read it where it lies; portable: every device of a multi-device call reads the same word */
  CU(cudaHostAlloc(&p, 64, cudaHostAllocMapped | cudaHostAllocPortable));
  t->flag = static_cast<uint32_t*>(p);
  __atomic_store_n(t->flag, 0u, __ATOMIC_RELEASE);
  *out = t.release();
  return B2Q_OK;
}
void b2q_interrupt_token_destroy(B2QInterruptToken* t) {
  if (!t) return;
  if (t->flag) { cudaFreeHost(t->flag); cudaGetLastError(); }
  delete t;
}
/* Executor::interrupt (GpuInterrupt.cpp:33-160) sets the flag of the running query's session; this is that store */
void b2q_interrupt(B2QInterruptToken* t) { if (t && t->flag) __atomic_store_n(t->flag, 1u, __ATOMIC_RELEASE); }
/* Executor::resetInterrupt (GpuInterrupt.cpp:292-300) */
void b2q_interrupt_reset(B2QInterruptToken* t) { if (t && t->flag) __atomic_store_n(t->flag, 0u, __ATOMIC_RELEASE); }
int32_t b2q_interrupt_is_set(const B2QInterruptToken* t) { return t && t->flag && __atomic_load_n(t->flag, __ATOMIC_ACQUIRE) ? 1 : 0; }

int32_t b2q_gen_column(void* dst, int32_t sql_type, uint64_t seed, uint32_t col_tag, int64_t row0, int64_t count,
                       int64_t lo, int64_t span, void* stream) {
  if (!have_device()) return set_err(B2Q_ERR_NO_DEVICE, "no CUDA device visible");
  CU(launch_gen(dst, sql_type, seed, col_tag, row0, count, lo, span, 1, static_cast<cudaStream_t>(stream)));
  return B2Q_OK;
}

int32_t b2q_gen_column_strided(void* dst, int32_t sql_type, uint64_t seed, uint32_t col_tag, int64_t row0, int64_t count,
                               int64_t lo, int64_t span, int64_t stride, void* stream) {
  if (!have_device()) return set_err(B2Q_ERR_NO_DEVICE, "no CUDA device visible");
  CU(launch_gen(dst, sql_type, seed, col_tag, row0, count, lo, span, stride, static_cast<cudaStream_t>(stream)));
  return B2Q_OK;
}

} /* extern "C" */
