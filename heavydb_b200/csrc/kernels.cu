/*
 * kernels.cu — the small kernels around the scan (join-table build, table init, split-accumulator join, materialise,
 * synthetic columns) and the host-side launch wrappers called from executor.cpp.  The scan kernel itself is
 * scan_kernel.cuh, instantiated in scan_inst.cu.
 */
#include "scan_kernel.cuh"

namespace b2q {

/* ---------------------------------------------------------------------------------------------------------
 * one-to-one perfect join table (fill_hash_join_buff, JoinHashTable/Runtime/HashJoinRuntime.cpp:120-216, and its
 * init_hash_join_buff): slot[key - min] = inner row index, NULL keys skipped; a slot claimed twice means the join is
 * not one-to-one (the reference then rebuilds a one-to-many table — outside this path)
 * ------------------------------------------------------------------------------------------------------- */
__global__ void b2q_k_join_build(const int8_t* __restrict__ keys, int width, int64_t n_rows, int64_t min_key, int64_t entry_count,
                                 int nullable, int64_t null_val, int32_t* __restrict__ buff, int32_t* __restrict__ error,
                                 const int8_t* __restrict__ packed_vals, int packed_width) {
  /* packed_vals != nullptr: slots are {int32 row, int32 value}; the value of the winning row is written by the thread
   * that claimed the slot (one winner per slot, so no race) */
  const int slot_words = packed_vals ? 2 : 1;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n_rows; row += stride) {
    int64_t k;
    switch (width) {
      case 8: k = reinterpret_cast<const int64_t*>(keys)[row]; break;
      case 4: k = reinterpret_cast<const int32_t*>(keys)[row]; break;
      case 2: k = reinterpret_cast<const int16_t*>(keys)[row]; break;
      default: k = reinterpret_cast<const signed char*>(keys)[row]; break;
    }
    if (nullable && k == null_val) continue;
    const uint64_t d = (uint64_t)(k - min_key);
    if (d >= (uint64_t)entry_count) { atomicCAS(error, 0, B2Q_ERR_KEY_OUT_OF_RANGE); continue; }
    if (atomicCAS(buff + d * slot_words, -1, (int32_t)row) != -1) { atomicCAS(error, 0, B2Q_ERR_UNSUPPORTED); continue; }
    if (packed_vals) {
      int32_t v;
      switch (packed_width) {
        case 4: v = reinterpret_cast<const int32_t*>(packed_vals)[row]; break;
        case 2: v = reinterpret_cast<const int16_t*>(packed_vals)[row]; break;
        case -2: v = reinterpret_cast<const uint16_t*>(packed_vals)[row]; break;
        case -1: v = reinterpret_cast<const uint8_t*>(packed_vals)[row]; break;
        default: v = reinterpret_cast<const signed char*>(packed_vals)[row]; break;
      }
      buff[d * 2 + 1] = v;
    }
  }
}

/* one-to-one row table -> value-only uint16 slots (DevJoin::slot16): value - vmin, 0xFFFE = NULL, 0xFFFF = no row */
__global__ void b2q_k_join_slot16(const int32_t* __restrict__ rows, int64_t entry_count, const int8_t* __restrict__ vals, int width,
                                  int64_t null_val, int64_t vmin, uint16_t* __restrict__ out, int32_t* __restrict__ error) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; d < entry_count; d += stride) {
    const int32_t row = rows[d];
    uint32_t code = 0xFFFFu;
    if (row >= 0) {
      int64_t v;
      switch (width) {
        case 4: v = reinterpret_cast<const int32_t*>(vals)[row]; break;
        case 2: v = reinterpret_cast<const int16_t*>(vals)[row]; break;
        case -2: v = reinterpret_cast<const uint16_t*>(vals)[row]; break;
        case -1: v = reinterpret_cast<const uint8_t*>(vals)[row]; break;
        default: v = reinterpret_cast<const signed char*>(vals)[row]; break;
      }
      if (v == null_val) code = 0xFFFEu;
      else if ((uint64_t)(v - vmin) < 0xFFFEull) code = (uint32_t)(v - vmin);
      else atomicCAS(error, 0, B2Q_ERR_KEY_OUT_OF_RANGE); /* a value outside its chunk-stats range (stale metadata) */
    }
    out[d] = (uint16_t)code;
  }
}

/* ---------------------------------------------------------------------------------------------------------
 * table initialisation (replaces init_group_by_buffer_gpu, GpuInitGroups.cu:124-171): accumulators to the
 * identity of their reduction, baseline keys to EMPTY_KEY_64, plus the one-replica shared-memory image.
 * ------------------------------------------------------------------------------------------------------- */
struct InitArgs {
  int64_t* accs[B2Q_MAX_ACCS];
  int8_t ops[B2Q_MAX_ACCS];
  int32_t n_accs;
  int64_t entry_count;
  int64_t* keys;      /* or nullptr */
  int8_t* smem_image; /* or nullptr */
  SmemPlan smem;
};

__global__ void b2q_k_init(const __grid_constant__ InitArgs A) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < A.entry_count; i += stride) {
    for (int a = 0; a < A.n_accs; ++a) {
      const int64_t id = b2q_acc_identity(A.ops[a]);
      if (A.ops[a] == ACC_TOUCH) reinterpret_cast<uint8_t*>(A.accs[a])[i] = 0;
      else if (A.ops[a] != ACC_BITMAP && A.ops[a] != ACC_NDV) A.accs[a][i] = id; /* the bitmaps are zeroed with a memset */
      if (A.smem_image && A.smem.acc_bytes[a] > 0) {
        int8_t* p = A.smem_image + A.smem.acc_off[a];
        if (A.smem.acc_bytes[a] == 1) reinterpret_cast<uint8_t*>(p)[i] = 0;
        else if (A.smem.acc_bytes[a] == 4) reinterpret_cast<uint32_t*>(p)[i] = 0u;
        else reinterpret_cast<int64_t*>(p)[i] = id;
      }
    }
    if (A.keys) A.keys[i] = B2Q_I64_MAX;
  }
}

/* split (lo[n] | hi[n]) accumulator -> plain int64[n] (needed before the NCCL merge and by materialise) */
__global__ void b2q_k_join_split(const int64_t* __restrict__ split, int64_t* __restrict__ out, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const uint32_t* lo = reinterpret_cast<const uint32_t*>(split);
  const int32_t* hi = reinterpret_cast<const int32_t*>(split) + n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    out[i] = (int64_t)(((uint64_t)(uint32_t)hi[i] << 32) + lo[i]);
}

/* estimator bitmaps of several devices (reduce_estimator_results, CardinalityEstimator.cpp:142-161): dst |= every gathered copy */
__global__ void b2q_k_bitmap_or(uint64_t* __restrict__ dst, const uint64_t* __restrict__ gathered, int64_t words, int copies) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += stride) {
    uint64_t v = dst[i];
    for (int c = 0; c < copies; ++c) v |= gathered[(size_t)c * words + i];
    dst[i] = v;
  }
}

/* the bitmaps of a query's set terms (DevTerm::set_bits), zeroed beforehand: one atomicOr per value (InValuesBitmap's
 * constructor, InValuesBitmap.cpp:40-95, done on the device).  values[i] belongs to the first set s with i < end[s]. */
struct SetBuildArgs {
  const int64_t* values;         /* every set's values, set after set */
  uint32_t* bits[B2Q_MAX_TERMS];
  int64_t end[B2Q_MAX_TERMS];    /* exclusive prefix ends into values */
  int64_t min[B2Q_MAX_TERMS];
  int32_t n_sets;
};
__global__ void b2q_k_set_build(const SetBuildArgs a) {
  const int64_t n = a.end[a.n_sets - 1];
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    int s = 0;
    while (i >= a.end[s]) ++s;
    const uint64_t d = (uint64_t)a.values[i] - (uint64_t)a.min[s];
    atomicOr(a.bits[s] + (d >> 5), 1u << (uint32_t)(d & 31));
  }
}

/* ---------------------------------------------------------------------------------------------------------
 * materialise: dense accumulators -> the reference's row-wise output buffer
 * (layout: QueryMemoryDescriptor.cpp:848-955; empty-entry conventions: ResultSetIteration.cpp:2457-2492)
 * ------------------------------------------------------------------------------------------------------- */
struct MatArgs {
  DevLayout layout;
  const int64_t* accs[B2Q_MAX_ACCS];
  const int64_t* keys;
  int8_t* out;
};

__global__ void b2q_k_materialize(const __grid_constant__ MatArgs A) {
  const DevLayout& L = A.layout;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < L.entry_count; i += stride) {
    int8_t* row = A.out + i * L.row_size;
    bool touched = true;
    int64_t key = 0;
    int64_t mkey_stored[B2Q_MAX_GROUP_COLS], mkey_proj[B2Q_MAX_GROUP_COLS];
    if (L.n_keys > 1) { /* mixed-radix decomposition of the entry index */
      for (int c = 0; c < L.n_keys; ++c) {
        const DevKeyComp& kc = L.keys[c];
        const int64_t comp = (i / kc.mult) % kc.card;
        const bool is_null_comp = kc.translate_null && comp == (int64_t)kc.card - 1;
        mkey_stored[c] = is_null_comp ? kc.null_stored : kc.min_val + comp * kc.step; /* a NULL key is stored translated: max + (bucket ? bucket : 1) */
        mkey_proj[c] = is_null_comp ? kc.null_logical : kc.min_val + comp * kc.step;
      }
      if (L.touched_acc >= 0) touched = reinterpret_cast<const uint8_t*>(A.accs[L.touched_acc])[i] != 0 || (L.touch_via_acc >= 0 && A.accs[L.touch_via_acc][i] != 0);
    } else if (L.baseline) {
      key = A.keys[i];
      touched = key != B2Q_I64_MAX;
      if (touched && L.key_width == 4) key = (int64_t)(int32_t)key;
    } else {
      key = (i == L.null_idx) ? L.key_null_val : L.key_min + i * L.key_step;
      if (L.touched_acc >= 0) touched = reinterpret_cast<const uint8_t*>(A.accs[L.touched_acc])[i] != 0 || (L.touch_via_acc >= 0 && A.accs[L.touch_via_acc][i] != 0);
    }
    if (L.has_key_col && L.columnar) {
      /* int64 key columns (initColumnarGroups, QueryMemoryInitializer.cpp:729-735; keys written by
       * get_columnar_group_bin_offset / set_matching_group_value_perfect_hash_columnar / get_group_value_columnar) */
      if (L.n_keys > 1) {
        for (int c = 0; c < L.n_keys; ++c) reinterpret_cast<int64_t*>(A.out + c * L.key_col_stride)[i] = touched ? mkey_stored[c] : B2Q_I64_MAX;
      } else {
        const int64_t stored = (!L.baseline && i == L.null_idx) ? L.key_null_stored : key;
        reinterpret_cast<int64_t*>(A.out)[i] = touched ? stored : B2Q_I64_MAX;
      }
    } else if (L.has_key_col && L.n_keys > 1) {
      for (int c = 0; c < L.n_keys; ++c) reinterpret_cast<int64_t*>(row)[c] = touched ? mkey_stored[c] : B2Q_I64_MAX;
    } else if (L.has_key_col) {
      if (L.key_width == 4) {
        *reinterpret_cast<int32_t*>(row) = touched ? (int32_t)key : 0x7FFFFFFF;
        *reinterpret_cast<int32_t*>(row + 4) = 0;
      } else {
        /* perfect hash stores the TRANSLATED key (NULL -> max+1), GroupByRuntime.cpp:194-209 */
        const int64_t stored = (!L.baseline && i == L.null_idx) ? L.key_null_stored : key;
        *reinterpret_cast<int64_t*>(row) = touched ? stored : B2Q_I64_MAX;
      }
    }
    int64_t vals[B2Q_MAX_SLOTS];
    for (int s = 0; s < L.n_slots; ++s) {
      const DevSlot& sl = L.slots[s];
      int64_t val = sl.init_val;
      if (touched && sl.kind != SLOT_NONE && sl.width != 0) {
        switch (sl.kind) {
          case SLOT_KEY: val = L.n_keys > 1 ? mkey_proj[sl.key_comp] : key; break;
          case SLOT_COUNT: val = A.accs[sl.acc][i]; break;
          case SLOT_BITCOUNT: { /* count_distinct_set_size over the entry's bitmap (CountDistinct.h:54-70) */
            const uint32_t* w = reinterpret_cast<const uint32_t*>(A.accs[sl.acc]) + (size_t)i * (size_t)sl.bm_words;
            int64_t n = 0;
            for (int k = 0; k < sl.bm_words; ++k) n += __popc(w[k]);
            val = n;
            break;
          }
          default: {
            const int64_t raw = A.accs[sl.acc][i];
            bool is_null = false;
            if (sl.nn >= 0) is_null = A.accs[sl.nn][i] == 0;
            else if (sl.nn == -2) is_null = raw == sl.identity || (sl.clamp_init && b2q_clamp_ord(raw, sl.identity, sl.as_float) != raw);
            val = is_null ? sl.init_val : (sl.kind == SLOT_VALUE_ORD ? b2q_ord_to_f64(raw) : (sl.scale_day ? raw * 86400 : raw));
            if (sl.as_float && !is_null) /* agg_*_float: 32 bits written, the slot's high word still holds the init pattern's */
              val = (sl.init_val & (int64_t)0xFFFFFFFF00000000ll) | (int64_t)(uint32_t)__float_as_int((float)__longlong_as_double(val));
            break;
          }
        }
      }
      vals[s] = val;
    }
    /* keyless layouts: an entry whose marker slot still holds its init value IS empty for every reader
     * (ResultSetIteration.cpp:2457-2476); leave it entirely at the init pattern */
    if (L.keyless_marker >= 0 && vals[L.keyless_marker] == L.slots[L.keyless_marker].init_val) {
      for (int s = 0; s < L.n_slots; ++s) vals[s] = L.slots[s].init_val;
    }
    if (L.columnar) {
      for (int s = 0; s < L.n_slots; ++s) {
        const DevSlot& sl = L.slots[s];
        if (sl.kind == SLOT_NONE || sl.width == 0) continue;
        if (sl.width == 4) reinterpret_cast<int32_t*>(A.out + sl.offset)[i] = (int32_t)vals[s];
        else reinterpret_cast<int64_t*>(A.out + sl.offset)[i] = vals[s];
      }
      /* an odd number of 4-byte entries leaves 4 bytes of column padding; the pool buffer is recycled */
      if (i == L.entry_count - 1 && (L.entry_count & 1))
        for (int s = 0; s < L.n_slots; ++s)
          if (L.slots[s].width == 4 && L.slots[s].kind != SLOT_NONE) reinterpret_cast<int32_t*>(A.out + L.slots[s].offset)[L.entry_count] = 0;
      continue;
    }
    int end = 0;
    for (int s = 0; s < L.n_slots; ++s) {
      const DevSlot& sl = L.slots[s];
      if (sl.kind == SLOT_NONE || sl.width == 0) continue;
      if (sl.width == 4) *reinterpret_cast<int32_t*>(row + sl.offset) = (int32_t)vals[s];
      else *reinterpret_cast<int64_t*>(row + sl.offset) = vals[s];
      end = max(end, (int)sl.offset + sl.width);
    }
    /* an odd number of 4-byte slots leaves alignment padding (QueryMemoryDescriptor.cpp:848-860); the buffer comes from
     * a recycled pool, so write the zeros the reference's freshly allocated buffer would hold */
    if (end) for (; end + 4 <= L.row_size; end += 4) *reinterpret_cast<int32_t*>(row + end) = 0;
  }
}

/* ---------------------------------------------------------------------------------------------------------
 * synthetic columns: same counter-based generator as oracle/oracle_gen.h
 * ------------------------------------------------------------------------------------------------------- */
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

__global__ void b2q_k_gen(void* dst, int sql_type, uint64_t seed, uint32_t col_tag, int64_t row0, int64_t count,
                          int64_t lo, uint64_t span, int64_t key_stride) {
  const int64_t step = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += step) {
    const uint64_t u = splitmix64(seed ^ ((uint64_t)col_tag << 56) ^ (uint64_t)(row0 + i));
    switch (sql_type) {
      case B2Q_kDOUBLE: static_cast<double*>(dst)[i] = (double)(u >> 11) * (1.0 / 9007199254740992.0); break;
      case B2Q_kBIGINT: static_cast<int64_t*>(dst)[i] = lo + (int64_t)(u % span) * key_stride; break;
      case B2Q_kINT: static_cast<int32_t*>(dst)[i] = (int32_t)(lo + (int64_t)(u % span)); break;
      case B2Q_kSMALLINT: static_cast<int16_t*>(dst)[i] = (int16_t)(lo + (int64_t)(u % span)); break;
      default: static_cast<int8_t*>(dst)[i] = (int8_t)(lo + (int64_t)(u % span)); break;
    }
  }
}

/* =========================================================================================================
 * host-side launch wrappers (called from executor.cpp)
 * ======================================================================================================= */
int sm_count() {
  static std::atomic<int> cached[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return 132;
  int n = cached[dev].load(std::memory_order_relaxed);
  if (!n) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    n = n > 0 ? n : 132;
    cached[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

int scan_rows_per_chunk(int block) { return block * R; }

/* block/grid policy: one CTA per SM with 1024 threads when the table needs more than half of the shared memory,
 * otherwise two CTAs of 512 threads per SM (better tail behaviour, same number of resident threads). */
void scan_config(const B2QQuery& q, int* block, int* ctas_per_sm) {
  const bool big_table = q.smem.total_bytes > 100 * 1024; /* group-table replicas and/or a staged join table */
  *block = big_table ? 1024 : 512;
  *ctas_per_sm = big_table ? 1 : 2;
}

cudaError_t launch_scan(const B2QQuery& q, const DevLaunch& launch, const int8_t* smem_image, int block, int ctas_per_sm,
                        cudaStream_t st) {
  ScanArgs a;
  a.prog = q.prog;
  a.launch = launch;
  a.smem = q.smem;
  a.smem_image = smem_image;
  a.ndv_bitmap_bytes = q.plan.query_desc_type == B2Q_Estimator ? q.plan.buffer_size : 0;
  ScanConfig c;
  c.block = block;
  const int64_t max_ctas = (int64_t)sm_count() * ctas_per_sm;
  c.grid = (int)(launch.total_chunks < max_ctas ? (launch.total_chunks > 0 ? launch.total_chunks : 1) : max_ctas);
  c.smem_bytes = (size_t)q.smem.total_bytes; /* 0 for the HBM-table kernels unless a join table is staged */
  const int kernel = q.plan.kernel;
  const bool key32 = q.prog.n_keys <= 1 && q.prog.key.col >= 0 && q.prog.key.width <= 4;
  /* one hash-join level: separate instantiations (0 none, 1 INNER, 2 LEFT), the plain scan stays as it was */
  const int j = a.prog.join.fk_col < 0 ? 0 : (a.prog.join.left ? 2 : 1);
  const int g = (kernel == B2Q_KERNEL_NON_GROUPED || kernel == B2Q_KERNEL_PERFECT_SMEM) ? 0 : kernel == B2Q_KERNEL_PERFECT_GLOBAL ? 1 : 2;
  const bool wagg = kernel == B2Q_KERNEL_NON_GROUPED;
  typedef cudaError_t (*Entry)(const ScanArgs&, const ScanConfig&, bool, bool, cudaStream_t);
  static const Entry table[3][3] = {{launch_scan_j0_g0, launch_scan_j0_g1, launch_scan_j0_g2},
                                    {launch_scan_j1_g0, launch_scan_j1_g1, launch_scan_j1_g2},
                                    {launch_scan_j2_g0, launch_scan_j2_g1, launch_scan_j2_g2}};
  return table[j][g](a, c, wagg, key32, st);
}

cudaError_t launch_join_build(const int8_t* keys, int width, int64_t n_rows, int64_t min_key, int64_t entry_count, int nullable,
                              int64_t null_val, int32_t* buff, int32_t* error, const int8_t* packed_vals, int packed_width,
                              cudaStream_t st) {
  if (entry_count > 0) {
    cudaError_t e = cudaMemsetAsync(buff, 0xFF, (size_t)entry_count * (packed_vals ? 8 : 4), st); /* init_hash_join_buff: every slot -1 */
    if (e != cudaSuccess) return e;
  }
  if (n_rows <= 0 || entry_count <= 0) return cudaSuccess;
  const int block = 256;
  int64_t blocks = (n_rows + block - 1) / block;
  const int64_t cap = (int64_t)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  b2q_k_join_build<<<(int)blocks, block, 0, st>>>(keys, width, n_rows, min_key, entry_count, nullable, null_val, buff, error, packed_vals, packed_width);
  return cudaGetLastError();
}

cudaError_t launch_join_slot16(const int32_t* rows, int64_t entry_count, const int8_t* vals, int width, int64_t null_val, int64_t vmin,
                               uint16_t* out, int32_t* error, cudaStream_t st) {
  if (entry_count <= 0) return cudaSuccess;
  const int block = 256;
  int64_t blocks = (entry_count + block - 1) / block;
  const int64_t cap = (int64_t)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  b2q_k_join_slot16<<<(int)blocks, block, 0, st>>>(rows, entry_count, vals, width, null_val, vmin, out, error);
  return cudaGetLastError();
}

cudaError_t launch_init(const B2QQuery& q, int64_t* const* accs, int64_t* keys, int8_t* smem_image, cudaStream_t st) {
  InitArgs a;
  a.n_accs = q.prog.n_accs;
  for (int i = 0; i < q.prog.n_accs; ++i) { a.accs[i] = accs[i]; a.ops[i] = q.prog.accs[i].op; }
  a.entry_count = q.plan.entry_count;
  a.keys = keys;
  a.smem_image = smem_image;
  a.smem = q.smem;
  const int block = 256;
  int64_t blocks = (q.plan.entry_count + block - 1) / block;
  const int64_t cap = (int64_t)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  b2q_k_init<<<(int)blocks, block, 0, st>>>(a);
  return cudaGetLastError();
}

/* dynamic watchdog: the call's first kernel records the start of its device work (dynamic_watchdog_init, cuda_mapd_rt.cu:140-164,
 * here %globaltimer for the whole call instead of per-SM cycle counters per launch) */
__global__ void b2q_k_watchdog_start(uint64_t* t0) {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  *t0 = t;
}
cudaError_t launch_watchdog_start(uint64_t* t0, cudaStream_t st) {
  b2q_k_watchdog_start<<<1, 1, 0, st>>>(t0);
  return cudaGetLastError();
}

/* the host saw the interrupt between two steps: the code goes into the call's error word like a kernel's would (first error
 * wins), so that it travels the same way, through the cross-device MAX all-reduce included */
__global__ void b2q_k_set_error(int32_t* error, int32_t code) { atomicCAS(error, 0, code); }
cudaError_t launch_set_error(int32_t* error, int32_t code, cudaStream_t st) {
  b2q_k_set_error<<<1, 1, 0, st>>>(error, code);
  return cudaGetLastError();
}

cudaError_t launch_bitmap_or(uint64_t* dst, const uint64_t* gathered, int64_t words, int copies, cudaStream_t st) {
  if (words <= 0) return cudaSuccess;
  const int64_t cap = (int64_t)sm_count() * 8;
  int64_t blocks = (words + 255) / 256;
  if (blocks > cap) blocks = cap;
  b2q_k_bitmap_or<<<(int)blocks, 256, 0, st>>>(dst, gathered, words, copies);
  return cudaGetLastError();
}

/* The set terms of `q` get their bitmaps in `blk` (set_bytes(q) bytes, device memory): the value lists are copied in after
 * the bitmaps, the bitmaps zeroed and built by one kernel, and each term's set_bits points at its bitmap.  Returns the kernels
 * launched (0 without a set term). */
size_t set_bytes(const B2QQuery& q) {
  size_t bytes = 0;
  for (int t = 0; t < q.prog.filter.n_terms; ++t)
    if (q.prog.filter.terms[t].is_set) bytes += ((q.prog.filter.terms[t].span >> 5) + 1) * 4 + q.set_values[t].size() * 8 + 16;
  return bytes;
}
cudaError_t build_sets(B2QQuery& q, int8_t* blk, int* launches, cudaStream_t st) {
  *launches = 0;
  SetBuildArgs a;
  memset(&a, 0, sizeof(a));
  std::vector<int64_t> values;
  size_t bits_bytes = 0;
  for (int t = 0; t < q.prog.filter.n_terms; ++t) {
    DevTerm& term = q.prog.filter.terms[t];
    if (!term.is_set) continue;
    const size_t words = (term.span >> 5) + 1;
    term.set_bits = reinterpret_cast<const uint32_t*>(blk + bits_bytes);
    a.bits[a.n_sets] = reinterpret_cast<uint32_t*>(blk + bits_bytes);
    a.min[a.n_sets] = term.lo;
    values.insert(values.end(), q.set_values[t].begin(), q.set_values[t].end());
    a.end[a.n_sets++] = static_cast<int64_t>(values.size());
    bits_bytes += (words * 4 + 15) & ~size_t(15);
  }
  if (!a.n_sets) return cudaSuccess;
  int64_t* d_values = reinterpret_cast<int64_t*>(blk + bits_bytes);
  a.values = d_values;
  /* pageable source: the runtime has staged it when cudaMemcpyAsync returns */
  cudaError_t e = cudaMemcpyAsync(d_values, values.data(), values.size() * 8, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(blk, 0, bits_bytes, st);
  if (e != cudaSuccess) return e;
  const int block = 256;
  int64_t blocks = (static_cast<int64_t>(values.size()) + block - 1) / block;
  const int64_t cap = (int64_t)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  b2q_k_set_build<<<(int)blocks, block, 0, st>>>(a);
  *launches = 1;
  return cudaGetLastError();
}

cudaError_t launch_join_split(const int64_t* split, int64_t* out, int64_t n, cudaStream_t st) {
  const int block = 256;
  int64_t blocks = (n + block - 1) / block;
  const int64_t cap = (int64_t)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  b2q_k_join_split<<<(int)blocks, block, 0, st>>>(split, out, n);
  return cudaGetLastError();
}

cudaError_t launch_materialize(const B2QQuery& q, const int64_t* const* accs, const int64_t* keys, int8_t* out,
                               cudaStream_t st) {
  MatArgs a;
  a.layout = q.layout;
  for (int i = 0; i < q.prog.n_accs; ++i) a.accs[i] = accs[i];
  a.keys = keys;
  a.out = out;
  const int block = 256;
  int64_t blocks = (q.plan.entry_count + block - 1) / block;
  const int64_t cap = (int64_t)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  b2q_k_materialize<<<(int)blocks, block, 0, st>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_gen(void* dst, int sql_type, uint64_t seed, uint32_t col_tag, int64_t row0, int64_t count, int64_t lo,
                       int64_t span, int64_t stride, cudaStream_t st) {
  if (count <= 0) return cudaSuccess;
  const int block = 256;
  int64_t blocks = (count + block - 1) / block;
  const int64_t cap = (int64_t)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  b2q_k_gen<<<(int)blocks, block, 0, st>>>(dst, sql_type, seed, col_tag, row0, count, lo, (uint64_t)(span > 0 ? span : 1), stride ? stride : 1);
  return cudaGetLastError();
}

}  // namespace b2q
