/*
 * radix_agg.cu — baseline-hash GROUP BY (sparse / high-cardinality keys) as a two-pass radix-partitioned aggregation.
 *
 * Replaces, for the sparse-key case, what the reference does per row with get_group_value + get_matching_group_value
 * (GroupByRuntime.cpp:25-48, cuda_mapd_rt.cu:180-216: MurmurHash3 home slot, linear probe, CAS claim on a table in
 * global memory) followed by agg_*_shared atomics on the claimed row.  The table that comes out is the same kind of
 * table — open addressing, h = MurmurHash3(key) % entry_count, every key reachable from its home slot by a linear probe
 * over occupied slots — but no row ever touches it in HBM:
 *
 *   pass 1  b2q_k_radix_partition[_tile]   streams the fragments once (same coalesced column loads and filter program as
 *           b2q_k_scan), hashes the key and appends the tuple {key, argument values} of every passing row to the region
 *           of (partition = home slot / S, this CTA).  Regions are private to a CTA, so the append cursor is a shared-
 *           memory counter.  Tuples of one or two words are first bucketed by partition in shared memory, a chunk of
 *           8192 rows at a time, and leave in runs of consecutive tuples (tools/scatter_bench.cu: one 16-byte store per
 *           tuple straight to its place is slow whatever the number of partitions; runs of ~9 tuples are about twice as
 *           fast).
 *   pass 2  b2q_k_radix_aggregate   one CTA per partition: the partition's tuples are streamed through a private
 *           shared-memory table — lookup, claim and update are shared-memory operations — whose occupied slots are then
 *           merged into the table in HBM with the reference's probe, once per key instead of once per row.
 *
 * Algorithmic traffic: read columns + write tuples + read tuples ~ 3x the column bytes, sequential, instead of two
 * random 32-byte sectors per row.
 * Rows a region has no room for (skewed keys) and keys the private table has no room for are inserted straight into the
 * HBM table with the probe of the row-by-row kernel — any input is handled, uniform ones fast.
 */
#include "scan_kernel.cuh"
#include "radix_agg.h"

namespace b2q {

constexpr int kRadixBlock = 1024;  /* pass 1 and pass 2: one CTA per SM */
constexpr int kTupleBlock = 128;   /* pass 2: tuples a warp takes at a time (4 per lane) */

/* ---- table in HBM: the reference's probe (get_group_value, GroupByRuntime.cpp:25-48) with plain 64-bit accumulators ---- */
__device__ __forceinline__ uint32_t home_slot(int64_t key, int hw, uint64_t magic, uint32_t n) {
  return (uint32_t)__umul64hi(magic * (uint64_t)murmur3_key(key, hw), (uint64_t)n); /* == MurmurHash3(key) % n */
}

/* The partition of a key and its bucket in pass 2's private table do NOT follow the reference's hash: MurmurHash3 + a 64-bit
 * fast-mod is ~45 instructions, needed once per KEY when the private table is merged into the HBM table, not once per ROW.
 * A 32-bit multiply-xorshift mix of the key picks the partition (its high bits, by multiply-shift) and the bucket (its
 * re-multiplied low bits). */
__device__ __forceinline__ uint32_t mix_key(int64_t key) {
  uint32_t x = (uint32_t)key ^ ((uint32_t)((uint64_t)key >> 32) * 0x85ebca6bu);
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}
__device__ __forceinline__ uint32_t part_of_mix(uint32_t mix, uint32_t n_parts) { return __umulhi(mix, n_parts); }
__device__ __forceinline__ uint32_t bucket_of_mix(uint32_t mix, uint32_t nb_mask) { return ((mix * 0x9E3779B1u) >> 9) & nb_mask; }

__device__ __forceinline__ int64_t global_probe(unsigned long long* keys, uint32_t n, uint32_t h, int64_t key) {
  const unsigned long long want = (unsigned long long)key;
  uint32_t p = h;
  for (;;) {
    unsigned long long cur = __ldcg(keys + p);
    if (cur == (unsigned long long)B2Q_I64_MAX) cur = atomicCAS(keys + p, (unsigned long long)B2Q_I64_MAX, want);
    if (cur == (unsigned long long)B2Q_I64_MAX || cur == want) return p;
    p = p + 1 == n ? 0 : p + 1;
    if (p == h) return -1;
  }
}

/* raw value -> accumulator, HBM table */
__device__ __forceinline__ void global_acc_raw(int op, int64_t* slot, int64_t v) {
  switch (op) {
    case ACC_COUNT: atomicAdd(reinterpret_cast<unsigned long long*>(slot), 1ull); break;
    case ACC_SUM_I64: atomicAdd(reinterpret_cast<unsigned long long*>(slot), (unsigned long long)v); break;
    case ACC_SUM_F64: red_add_f64(slot, __longlong_as_double(v)); break;
    case ACC_MIN_I64: red_min_s64(slot, v); break;
    case ACC_MAX_I64: red_max_s64(slot, v); break;
    case ACC_MIN_F64: red_min_s64(slot, b2q_f64_min_ord(v)); break;
    case ACC_MAX_F64: red_max_s64(slot, b2q_f64_max_ord(v)); break;
    default: break;
  }
}
/* partial accumulator -> accumulator (ResultSetStorage::reduceOneSlot's algebra on the internal arrays) */
__device__ __forceinline__ void global_acc_merge(int op, int64_t* slot, int64_t v) {
  switch (op) {
    case ACC_COUNT: case ACC_SUM_I64: if (v) atomicAdd(reinterpret_cast<unsigned long long*>(slot), (unsigned long long)v); break;
    case ACC_SUM_F64: if (__longlong_as_double(v) != 0.0) red_add_f64(slot, __longlong_as_double(v)); break;
    case ACC_MIN_I64: case ACC_MIN_F64: if (v != B2Q_I64_MAX) red_min_s64(slot, v); break;
    case ACC_MAX_I64: case ACC_MAX_F64: if (v != B2Q_I64_MIN) red_max_s64(slot, v); break;
    default: break;
  }
}

__device__ __forceinline__ bool value_skipped(const DevAcc& a, int64_t v) {
  if (a.is_fp) return a.skip1_en && __longlong_as_double(v) == __longlong_as_double(a.skip1_val);
  const int64_t w = a.skip2_trunc32 ? (int64_t)(int32_t)v : v;
  return (a.skip1_en && v == a.skip1_val) || (a.skip2_en && w == a.skip2_val);
}

/* one raw tuple {key, vals[]} into the HBM table */
__device__ __noinline__ void global_insert_raw(const RadixArgs& A, int64_t key, const int64_t* vals) { /* rare (skewed keys, a full private table): kept out of line so that the row loops stay small */
  const DevProgram& P = A.prog;
  const uint32_t n = (uint32_t)P.key.entry_count;
  const int64_t e = global_probe(reinterpret_cast<unsigned long long*>(A.launch.keys), n, home_slot(key, P.key.hash_key_width, P.key.hash_magic, n), key);
  if (e < 0) { atomicCAS(A.launch.error, 0, B2Q_ERR_OUT_OF_SLOTS); return; }
  for (int a = 0; a < P.n_accs; ++a) {
    const DevAcc& acc = P.accs[a];
    const int vi = A.acc_val[a];
    const int64_t v = vi >= 0 ? vals[vi] : 0;
    if (vi >= 0 && value_skipped(acc, v)) continue;
    global_acc_raw(acc.op, A.launch.accs[a] + e, v);
  }
}

/* the high-word delta of a COUNT / integer SUM whose low word lives in shared memory: straight to the key's entry in HBM */
__device__ __noinline__ void global_add_hi(const RadixArgs& A, int64_t key, int a, int32_t hi) { /* rare: a carry out of a 32-bit low word, or a value wider than 32 bits */
  const DevProgram& P = A.prog;
  const uint32_t n = (uint32_t)P.key.entry_count;
  const int64_t e = global_probe(reinterpret_cast<unsigned long long*>(A.launch.keys), n, home_slot(key, P.key.hash_key_width, P.key.hash_magic, n), key);
  if (e < 0) { atomicCAS(A.launch.error, 0, B2Q_ERR_OUT_OF_SLOTS); return; }
  red_add_u64(A.launch.accs[a] + e, (uint64_t)(int64_t)hi << 32);
}

/* ---- private shared-memory table (pass 2): 64-bit slots, 32-bit native atomics ---- */
__device__ __forceinline__ void smem_add64(int64_t* slot, int64_t v) {
  uint32_t* w = reinterpret_cast<uint32_t*>(slot);
  const uint32_t vl = (uint32_t)v;
  const uint32_t old = atomicAdd(w, vl);
  const int32_t hi = (int32_t)(v >> 32) + (int32_t)((uint32_t)(old + vl) < old);
  if (hi != 0) atomicAdd(w + 1, (uint32_t)hi);
}
__device__ __forceinline__ void smem_acc_raw(int op, int64_t* slot, int64_t v) {
  switch (op) {
    case ACC_COUNT: smem_add64(slot, 1); break;
    case ACC_SUM_I64: smem_add64(slot, v); break;
    case ACC_SUM_F64: atomicAdd(reinterpret_cast<double*>(slot), __longlong_as_double(v)); break;
    case ACC_MIN_I64: if (v < *reinterpret_cast<volatile long long*>(slot)) atomicMin(reinterpret_cast<long long*>(slot), (long long)v); break;
    case ACC_MAX_I64: if (v > *reinterpret_cast<volatile long long*>(slot)) atomicMax(reinterpret_cast<long long*>(slot), (long long)v); break;
    case ACC_MIN_F64: { const long long o = b2q_f64_min_ord(v); if (o < *reinterpret_cast<volatile long long*>(slot)) atomicMin(reinterpret_cast<long long*>(slot), o); break; }
    case ACC_MAX_F64: { const long long o = b2q_f64_max_ord(v); if (o > *reinterpret_cast<volatile long long*>(slot)) atomicMax(reinterpret_cast<long long*>(slot), o); break; }
    default: break;
  }
}

/* ==========================================================================================================
 * pass 1: partition
 * ======================================================================================================== */
template <bool KEY32, bool FULL>
__device__ __forceinline__ void partition_chunk(const RadixArgs& A, const int8_t* const* __restrict__ cols, int64_t row0, int64_t frag_rows,
                                                uint32_t* s_cnt, uint64_t pol) {
  constexpr int nthr = kRadixBlock;
  const DevProgram& P = A.prog;
  uint32_t valid = (1u << R) - 1u;
  if (!FULL) {
    valid = 0;
#pragma unroll
    for (int j = 0; j < R; ++j) valid |= (uint32_t)(row0 + (int64_t)j * nthr < frag_rows) << j;
  }
  int32_t k32[KEY32 ? R : 1];
  int64_t k64[KEY32 ? 1 : R];
  const bool eager_key = P.eager_key;
  if (eager_key) {
    if (KEY32) load32<true>(reinterpret_cast<int32_t(&)[R]>(k32), cols[P.key.col], P.key.width, row0, nthr, valid, pol);
    else load64<true>(reinterpret_cast<int64_t(&)[R]>(k64), cols[P.key.col], row0, nthr, valid, pol);
  }
  const uint32_t pass = eval_filter<FULL, 0>(P.filter, cols, row0, nthr, valid, pol, P.col_inner, nullptr, -1, nullptr, P.col_null);
  if (!eager_key) {
    if (KEY32) load32<true>(reinterpret_cast<int32_t(&)[R]>(k32), cols[P.key.col], P.key.width, row0, nthr, pass, pol);
    else load64<true>(reinterpret_cast<int64_t(&)[R]>(k64), cols[P.key.col], row0, nthr, pass, pol);
  }
  const int tw = A.tuple_words;
  const uint32_t region0 = blockIdx.x * A.cap;          /* this CTA's region inside a partition's block of regions */
  const uint32_t part_stride = gridDim.x * A.cap;
#define B2Q_KEY_OF(j) (KEY32 ? (int64_t)k32[KEY32 ? (j) : 0] : k64[KEY32 ? 0 : (j)])
  /* The append cursor of (partition, this CTA) is a shared-memory counter; the tuple goes to the region's next free place.
   * Register budget (64 at 1024 threads): keys and ONE value vector stay live, places are computed row by row. */
  if (tw == 2) { /* {key, one value}: one 16-byte store per row */
    int64_t v[R];
    if (A.val_width[0] == 8) load64<true>(v, cols[A.val_col[0]], row0, nthr, pass, pol);
    else {
      int32_t t32[R];
      load32<true>(t32, cols[A.val_col[0]], A.val_width[0], row0, nthr, pass, pol);
#pragma unroll
      for (int j = 0; j < R; ++j) v[j] = t32[j];
    }
#pragma unroll
    for (int j = 0; j < R; ++j) {
      if (!(pass >> j & 1)) continue;
      int64_t key = B2Q_KEY_OF(j);
      if (key == P.key.null_val) key = P.key.null_logical; /* ENCODING FIXED: physical NULL -> logical NULL */
      const uint32_t part = part_of_mix(mix_key(key), (uint32_t)A.n_parts);
      const uint32_t pos = atomicAdd(s_cnt + part, 1u);
      if (pos < A.cap) {
        int64_t* dst = A.scratch + ((uint64_t)part * part_stride + region0 + pos) * 2u;
        asm volatile("st.global.v2.b64 [%0], {%1, %2};" ::"l"(dst), "l"(key), "l"(v[j]) : "memory");
      } else {
        global_insert_raw(A, key, &v[j]); /* no room (skewed keys): the reference's probe on the table in HBM */
      }
    }
    return;
  }
  uint32_t place[R]; /* tuple index inside the scratch area; ~0u: no room */
  uint32_t direct = 0;
#pragma unroll
  for (int j = 0; j < R; ++j) {
    place[j] = ~0u;
    if (!(pass >> j & 1)) continue;
    int64_t key = B2Q_KEY_OF(j);
    if (key == P.key.null_val) key = P.key.null_logical;
    const uint32_t part = part_of_mix(mix_key(key), (uint32_t)A.n_parts);
    const uint32_t pos = atomicAdd(s_cnt + part, 1u);
    if (pos < A.cap) {
      place[j] = part * part_stride + region0 + pos;
      A.scratch[(uint64_t)place[j] * (uint64_t)tw] = key;
    } else direct |= 1u << j;
  }
  for (int c = 0; c < A.n_vals; ++c) {
    int64_t v[R];
    if (A.val_width[c] == 8) load64<true>(v, cols[A.val_col[c]], row0, nthr, pass, pol);
    else {
      int32_t t32[R];
      load32<true>(t32, cols[A.val_col[c]], A.val_width[c], row0, nthr, pass, pol);
#pragma unroll
      for (int j = 0; j < R; ++j) v[j] = t32[j];
    }
#pragma unroll
    for (int j = 0; j < R; ++j) if (place[j] != ~0u) A.scratch[(uint64_t)place[j] * (uint64_t)tw + 1 + c] = v[j];
  }
  if (direct) { /* rare: re-read the row's values one by one */
#pragma unroll 1
    for (int j = 0; j < R; ++j) {
      if (!(direct >> j & 1)) continue;
      int64_t key = B2Q_KEY_OF(j);
      if (key == P.key.null_val) key = P.key.null_logical;
      int64_t vals[B2Q_RADIX_MAX_VALS];
      const int64_t row = row0 + (int64_t)j * nthr;
      for (int c = 0; c < A.n_vals; ++c) {
        const int8_t* b = cols[A.val_col[c]];
        switch (A.val_width[c]) {
          case 8: vals[c] = reinterpret_cast<const int64_t*>(b)[row]; break;
          case 4: vals[c] = reinterpret_cast<const int32_t*>(b)[row]; break;
          case 2: vals[c] = reinterpret_cast<const int16_t*>(b)[row]; break;
          case -2: vals[c] = reinterpret_cast<const uint16_t*>(b)[row]; break;
          case -1: vals[c] = reinterpret_cast<const uint8_t*>(b)[row]; break;
          default: vals[c] = reinterpret_cast<const signed char*>(b)[row]; break;
        }
      }
      global_insert_raw(A, key, vals);
    }
  }
#undef B2Q_KEY_OF
}

/* direct variant (tuples of three words and more): every tuple goes straight to its place — 32 different lines per warp store.
 * tools/scatter_bench.cu measures it against the tile variant. */
template <bool KEY32>
__global__ void __launch_bounds__(kRadixBlock, 1) b2q_k_radix_partition(const __grid_constant__ RadixArgs A) {
  extern __shared__ __align__(16) uint32_t s_cnt[]; /* [n_parts] */
  const DevProgram& P = A.prog;
  const DevLaunch& Lh = A.launch;
  const int tid = threadIdx.x;
  constexpr int nthr = kRadixBlock;
  const int64_t chunk_rows = (int64_t)nthr * R;
  for (int i = tid; i < A.n_parts; i += nthr) s_cnt[i] = 0;
  __syncthreads();
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  int frag = 0;
  int64_t frag_first = 0;
  int64_t next_first = __ldg(Lh.frag_chunk_start + 1);
  for (int64_t chunk = A.chunk_begin + blockIdx.x; chunk < A.chunk_end; chunk += gridDim.x) {
    while (chunk >= next_first) {
      ++frag;
      frag_first = next_first;
      next_first = __ldg(Lh.frag_chunk_start + frag + 1);
    }
    const int64_t frag_rows = __ldg(Lh.frag_rows + frag);
    const int64_t base_row = (chunk - frag_first) * chunk_rows;
    const int8_t* const* __restrict__ cols = Lh.col_ptrs + (size_t)frag * P.n_cols;
    if (base_row + chunk_rows <= frag_rows) partition_chunk<KEY32, true>(A, cols, base_row + tid, frag_rows, s_cnt, pol);
    else partition_chunk<KEY32, false>(A, cols, base_row + tid, frag_rows, s_cnt, pol);
    __syncwarp(); /* the (rare) probe of a row without room diverges per lane */
  }
  __syncthreads();
  /* how many tuples each region holds: counts[part * n_cta + cta] */
  for (int i = tid; i < A.n_parts; i += nthr) A.counts[(size_t)i * gridDim.x + blockIdx.x] = min(s_cnt[i], A.cap);
}

/* tile variant (tuples of one or two words): the passing rows of a chunk (BLOCK x R = 8192 rows) are bucketed by partition in
 * shared memory — count with a shared atomic (which also ranks the row inside its bucket), scan, place — and written out
 * with consecutive lanes on consecutive tuples of a region, i.e. in runs of chunk / n_parts tuples instead of one tuple per
 * line (tools/scatter_bench.cu: the fewer the partitions, the longer the runs and the faster). */
template <bool KEY32, int TW>
__global__ void __launch_bounds__(kRadixBlock, 1) b2q_k_radix_partition_tile(const __grid_constant__ RadixArgs A) {
  extern __shared__ __align__(16) int8_t s_tile_raw[];
  constexpr int nthr = kRadixBlock;
  constexpr int TILE = nthr * R;
  const DevProgram& P = A.prog;
  const DevLaunch& Lh = A.launch;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int NP = A.n_parts;
  int64_t* tile = reinterpret_cast<int64_t*>(s_tile_raw);                 /* [TILE][TW] tuples in partition order */
  uint32_t* s_cur = reinterpret_cast<uint32_t*>(tile + (size_t)TILE * TW);  /* [NP] tuples of the region so far */
  uint32_t* s_cnt = s_cur + NP;                                           /* [NP] tuples of this chunk */
  uint32_t* s_off = s_cnt + NP;                                           /* [NP + 1] exclusive scan of s_cnt */
  uint16_t* s_pid = reinterpret_cast<uint16_t*>(s_off + NP + 1);          /* [TILE] partition of a tile slot */
  __shared__ uint32_t s_warp[32];
  const int64_t chunk_rows = (int64_t)TILE;
  for (int i = tid; i < NP; i += nthr) { s_cur[i] = 0; s_cnt[i] = 0; }
  __syncthreads();
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  const uint32_t region0 = blockIdx.x * A.cap;
  const uint32_t part_stride = gridDim.x * A.cap;
  const int per = (NP + nthr - 1) / nthr; /* scan: partitions per thread */
  int frag = 0;
  int64_t frag_first = 0;
  int64_t next_first = __ldg(Lh.frag_chunk_start + 1);
  for (int64_t chunk = A.chunk_begin + blockIdx.x; chunk < A.chunk_end; chunk += gridDim.x) {
    while (chunk >= next_first) {
      ++frag;
      frag_first = next_first;
      next_first = __ldg(Lh.frag_chunk_start + frag + 1);
    }
    const int64_t frag_rows = __ldg(Lh.frag_rows + frag);
    const int64_t row0 = (chunk - frag_first) * chunk_rows + tid;
    const int8_t* const* __restrict__ cols = Lh.col_ptrs + (size_t)frag * P.n_cols;
    const bool full = (chunk - frag_first + 1) * chunk_rows <= frag_rows;
    uint32_t valid = (1u << R) - 1u;
    if (!full) {
      valid = 0;
#pragma unroll
      for (int j = 0; j < R; ++j) valid |= (uint32_t)(row0 + (int64_t)j * nthr < frag_rows) << j;
    }
    /* ---- rows in: key, filter, value (all loads predicated, so the ragged last chunk of a fragment takes the same path) ---- */
    int32_t k32[KEY32 ? R : 1];
    int64_t k64[KEY32 ? 1 : R];
    const bool eager_key = P.eager_key;
    if (eager_key) {
      if (KEY32) load32<true>(reinterpret_cast<int32_t(&)[R]>(k32), cols[P.key.col], P.key.width, row0, nthr, valid, pol);
      else load64<true>(reinterpret_cast<int64_t(&)[R]>(k64), cols[P.key.col], row0, nthr, valid, pol);
    }
    const uint32_t pass = eval_filter<false, 0>(P.filter, cols, row0, nthr, valid, pol, P.col_inner, nullptr, -1, nullptr, P.col_null);
    if (!eager_key) {
      if (KEY32) load32<true>(reinterpret_cast<int32_t(&)[R]>(k32), cols[P.key.col], P.key.width, row0, nthr, pass, pol);
      else load64<true>(reinterpret_cast<int64_t(&)[R]>(k64), cols[P.key.col], row0, nthr, pass, pol);
    }
    int64_t v[TW == 2 ? R : 1];
    if (TW == 2) {
      if (A.val_width[0] == 8) load64<true>(reinterpret_cast<int64_t(&)[R]>(v), cols[A.val_col[0]], row0, nthr, pass, pol);
      else {
        int32_t t32[R];
        load32<true>(t32, cols[A.val_col[0]], A.val_width[0], row0, nthr, pass, pol);
#pragma unroll
        for (int j = 0; j < R; ++j) v[TW == 2 ? j : 0] = t32[j];
      }
    }
    /* ---- count + rank: (partition << 16 | rank inside the chunk's bucket); TILE <= 65536 ---- */
    uint32_t pr[R];
#pragma unroll
    for (int j = 0; j < R; ++j) {
      pr[j] = ~0u;
      if (!(pass >> j & 1)) continue;
      int64_t key = KEY32 ? (int64_t)k32[KEY32 ? j : 0] : k64[KEY32 ? 0 : j];
      if (key == P.key.null_val) key = P.key.null_logical; /* ENCODING FIXED: physical NULL -> logical NULL */
      if (KEY32) k32[KEY32 ? j : 0] = (int32_t)key; else k64[KEY32 ? 0 : j] = key;
      const uint32_t part = part_of_mix(mix_key(key), (uint32_t)NP);
      pr[j] = part << 16 | atomicAdd(s_cnt + part, 1u);
    }
    __syncthreads();
    /* ---- exclusive scan of the bucket sizes ---- */
    uint32_t loc = 0;
    for (int q = 0; q < per; ++q) { const int i = tid * per + q; if (i < NP) loc += s_cnt[i]; }
    uint32_t inc = loc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
      uint32_t w = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += t; }
      s_warp[lane] = w;
    }
    __syncthreads();
    uint32_t run = inc - loc + (warp ? s_warp[warp - 1] : 0u);
    for (int q = 0; q < per; ++q) { const int i = tid * per + q; if (i < NP) { s_off[i] = run; run += s_cnt[i]; } }
    if (tid == nthr - 1) s_off[NP] = run;
    __syncthreads();
    /* ---- place ---- */
#pragma unroll
    for (int j = 0; j < R; ++j) {
      if (pr[j] == ~0u) continue;
      const uint32_t part = pr[j] >> 16, slot = s_off[part] + (pr[j] & 0xFFFFu);
      const int64_t key = KEY32 ? (int64_t)k32[KEY32 ? j : 0] : k64[KEY32 ? 0 : j];
      if (TW == 2) { tile[(size_t)slot * 2] = key; tile[(size_t)slot * 2 + 1] = v[TW == 2 ? j : 0]; }
      else tile[slot] = key;
      s_pid[slot] = (uint16_t)part;
    }
    __syncthreads();
    /* ---- runs out: lane i takes tile slot i ---- */
    const uint32_t total = s_off[NP];
    for (uint32_t slot = tid; slot < total; slot += nthr) {
      const uint32_t part = s_pid[slot];
      const uint32_t pos = s_cur[part] + (slot - s_off[part]);
      if (pos < A.cap) {
        int64_t* dst = A.scratch + ((uint64_t)part * part_stride + region0 + pos) * (uint64_t)TW;
        if (TW == 2) {
          const longlong2 t = *reinterpret_cast<const longlong2*>(tile + (size_t)slot * 2);
          asm volatile("st.global.v2.b64 [%0], {%1, %2};" ::"l"(dst), "l"(t.x), "l"(t.y) : "memory");
        } else *dst = tile[slot];
      } else { /* no room in the region (skewed keys): the reference's probe on the table in HBM */
        global_insert_raw(A, tile[(size_t)slot * TW], tile + (size_t)slot * TW + 1);
      }
    }
    __syncthreads();
    for (int i = tid; i < NP; i += nthr) { s_cur[i] += s_cnt[i]; s_cnt[i] = 0; }
    __syncthreads();
  }
  for (int i = tid; i < NP; i += nthr) A.counts[(size_t)i * gridDim.x + blockIdx.x] = min(s_cur[i], A.cap);
}

/* ==========================================================================================================
 * pass 2: aggregate one partition at a time in a private shared-memory table, then merge it into the table in HBM
 * ======================================================================================================== */
/* The private table is NOT a slice of the reference's table: it is a bucketed table (4 slots per bucket, bucket = the key's
 * home slot / 4 inside the partition's range, overflow into the following buckets) because probe LENGTHS decide the cost
 * on a SIMT machine — ncu on the first version, which probed a slice of the reference's linear-probing layout in shared
 * memory: mean probe length 2 at load 0.67, but the tail decays like 0.93^k, the longest of a warp's 32 probes was ~25
 * steps, and most of the warp instructions per tuple went into waiting for it.  A lookup
 * here reads one 32-byte bucket (two LDS.128) and nearly always ends there.  When the partition's tuples are through, every
 * occupied slot is merged into the table in HBM with the reference's own probe (get_group_value, GroupByRuntime.cpp:25-48):
 * ~1e7 probes per 1e9 rows.  A key that finds no room within kMaxBuckets buckets (more distinct keys in the range than the
 * estimate behind entry_count promised) goes to the HBM table directly, row by row.
 * Accumulators: COUNT / integer SUM as 32-bit low words (native ATOMS.ADD; a carry or a value wider than 32 bits is sent to
 * the HBM entry at once, RED.ADD.64 of hi << 32), the others as 64-bit slots at their identity. */
constexpr int kBucket = 4, kMaxBuckets = 8;
constexpr int kQueue = 64; /* pass 2: parked tuples per warp */

__device__ __forceinline__ void lds128(const int64_t* p, int64_t& a, int64_t& b) {
  asm volatile("ld.shared.v2.b64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "r"(smem_u32(p)) : "memory");
}

/* slot of `want` in the private table (claimed if new), or -1 when its buckets are full; starts at bucket b */
__device__ __noinline__ int bucket_find(int64_t* s_keys, uint32_t nb_mask, uint32_t b, int64_t want) {
  for (int step = 0; step < kMaxBuckets; ++step, b = (b + 1) & nb_mask) {
    int64_t* bk = s_keys + (size_t)b * kBucket;
    for (;;) {
      int64_t k0, k1, k2, k3;
      lds128(bk, k0, k1);
      lds128(bk + 2, k2, k3);
      const uint32_t hit = (uint32_t)(k0 == want) | (uint32_t)(k1 == want) << 1 | (uint32_t)(k2 == want) << 2 | (uint32_t)(k3 == want) << 3;
      if (hit) return (int)(b * kBucket + (__ffs(hit) - 1));
      const uint32_t empty = (uint32_t)(k0 == B2Q_I64_MAX) | (uint32_t)(k1 == B2Q_I64_MAX) << 1 | (uint32_t)(k2 == B2Q_I64_MAX) << 2 | (uint32_t)(k3 == B2Q_I64_MAX) << 3;
      if (!empty) break; /* full bucket without the key: next bucket */
      const int j = __ffs(empty) - 1;
      const unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(bk + j), (unsigned long long)B2Q_I64_MAX, (unsigned long long)want);
      if (old == (unsigned long long)B2Q_I64_MAX || old == (unsigned long long)want) return (int)(b * kBucket + j);
      /* lost the slot to another key: look at the bucket again */
    }
  }
  return -1;
}

/* TWT: tuple words known at compile time (1 or 2), 0 = read from the arguments; FUSED: the program is {one COUNT(*) or integer SUM
 * without a NULL test} — one predicated ATOMS per tuple, no accumulator loop.  (In the one generic kernel, a large share of the
 * warp instructions were selects between the two tuple formats and re-reads of these loop invariants.) */
template <int TWT, bool FUSED>
__global__ void __launch_bounds__(kRadixBlock, 1) b2q_k_radix_aggregate(const __grid_constant__ RadixArgs A) {
  extern __shared__ __align__(128) int8_t s_raw[];
  const DevProgram& P = A.prog;
  const DevLaunch& Lh = A.launch;
  const int tid = threadIdx.x, lane = tid & 31;
  constexpr int nthr = kRadixBlock;
  const uint32_t S = 1u << A.log_s;                 /* slots of the private table == home slots per partition */
  const int n_accs = P.n_accs;
  int64_t* s_keys = reinterpret_cast<int64_t*>(s_raw);
  int8_t* s_acc = s_raw + (size_t)S * 8;            /* accumulator a: s_acc + acc_off[a] * S, 4 or 8 bytes per slot */
  uint32_t* s_blk = reinterpret_cast<uint32_t*>(s_acc + (size_t)A.acc_bytes_total * S); /* [n_cta1 + 1] block prefix of the partition's regions */
  /* per warp: 64 parked tuples {key, value or tuple address} (at most 31 left over + 32 new before a drain) */
  int64_t* q_key = reinterpret_cast<int64_t*>(s_raw + A.queue_off) + (size_t)(tid >> 5) * 2 * kQueue;
  int64_t* q_aux = q_key + kQueue;
  const uint32_t lt = (1u << lane) - 1u;
  __shared__ uint32_t s_part;
  const uint32_t n = (uint32_t)P.key.entry_count;
  const uint64_t magic = P.key.hash_magic;
  const int hw = P.key.hash_key_width;
  const int tw = TWT ? TWT : A.tuple_words;
  const int n_cta1 = A.n_cta1;
  const uint32_t nb_mask = S / kBucket - 1;
  constexpr bool fused = FUSED;
  const bool fused_count = fused && P.accs[0].op == ACC_COUNT;
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  for (;;) {
    __syncthreads();
    if (tid == 0) s_part = atomicAdd(A.work_counter, 1u);
    __syncthreads();
    const uint32_t part = s_part;
    if (part >= (uint32_t)A.n_parts) break;
    /* ---- empty table ---- */
    for (uint32_t i = tid; i < S; i += nthr) s_keys[i] = B2Q_I64_MAX;
    for (int a = 0; a < n_accs; ++a) {
      int8_t* base = s_acc + (size_t)A.acc_off[a] * S;
      if (A.acc_bytes[a] == 4) for (uint32_t i = tid; i < S; i += nthr) reinterpret_cast<uint32_t*>(base)[i] = 0u;
      else { const int64_t id = b2q_acc_identity(P.accs[a].op); for (uint32_t i = tid; i < S; i += nthr) reinterpret_cast<int64_t*>(base)[i] = id; }
    }
    if (tid < 32) { /* warp 0: inclusive scan of ceil(count / kTupleBlock) over the n_cta1 regions */
      uint32_t run = 0;
      for (int base = 0; base < n_cta1; base += 32) {
        const int c = base + lane;
        uint32_t b = c < n_cta1 ? (__ldg(A.counts + (size_t)part * n_cta1 + c) + kTupleBlock - 1) / kTupleBlock : 0u;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, b, o); if (lane >= o) b += t; }
        if (c < n_cta1) s_blk[c + 1] = run + b;
        run += __shfl_sync(0xffffffffu, b, 31);
      }
      if (lane == 0) s_blk[0] = 0;
    }
    __syncthreads();
    /* ---- stream the partition's tuples through the table ---- */
    const uint32_t total_blocks = s_blk[n_cta1];
    uint32_t qn = 0; /* tuples parked in this warp's queue (warp-uniform) */
    /* one tuple into the private table.  e >= 0: its slot is known; e == -2: find / claim it first (all lanes of the warp
     * arrive together: the queue is drained 32 at a time); e == -3: nothing to do for this lane */
    auto update = [&](int64_t k, int64_t aux, int e, bool find) {
      if (find) {
        if (e == -2) e = bucket_find(s_keys, nb_mask, bucket_of_mix(mix_key(k), nb_mask), k);
        __syncwarp(); /* a few lanes visit a second bucket or retry a claim: reconverge before the updates */
        if (e == -3) return;
      }
      const int64_t* vals = tw <= 2 ? nullptr : reinterpret_cast<const int64_t*>(aux) + 1;
      if (e < 0) { /* no room in the private table: the row goes to the table in HBM */
        int64_t rv[B2Q_RADIX_MAX_VALS];
        for (int cidx = 0; cidx < A.n_vals; ++cidx) rv[cidx] = tw <= 2 ? aux : __ldcg(vals + cidx);
        global_insert_raw(A, k, rv);
      } else if (fused) {
        const int64_t add = fused_count ? 1 : aux;
        const uint32_t vl = (uint32_t)add;
        const uint32_t old = atomicAdd(reinterpret_cast<uint32_t*>(s_acc) + e, vl);
        const int32_t hi32 = (int32_t)(add >> 32) + (int32_t)((uint32_t)(old + vl) < old);
        if (hi32 != 0) global_add_hi(A, k, 0, hi32);
      } else {
        for (int a = 0; a < n_accs; ++a) {
          const DevAcc& acc = P.accs[a];
          const int vi = A.acc_val[a];
          const int64_t v = vi < 0 ? 0 : (tw <= 2 ? aux : __ldcg(vals + vi));
          if (vi >= 0 && value_skipped(acc, v)) continue;
          int8_t* base = s_acc + (size_t)A.acc_off[a] * S;
          if (A.acc_bytes[a] == 4) {
            const int64_t add = acc.op == ACC_COUNT ? 1 : v;
            const uint32_t vl = (uint32_t)add;
            const uint32_t old = atomicAdd(reinterpret_cast<uint32_t*>(base) + e, vl);
            const int32_t hi32 = (int32_t)(add >> 32) + (int32_t)((uint32_t)(old + vl) < old);
            if (hi32 != 0) global_add_hi(A, k, a, hi32);
          } else smem_acc_raw(acc.op, reinterpret_cast<int64_t*>(base) + e, v);
        }
      }
    };
    int c = 0; /* region of block b: blocks are taken in increasing order, so the region is a moving cursor */
    for (uint32_t b = tid >> 5; b < total_blocks; b += nthr / 32) {
      while (s_blk[c + 1] <= b) ++c;
      const uint32_t cnt = __ldg(A.counts + (size_t)part * n_cta1 + c);
      const uint32_t off = (b - s_blk[c]) * kTupleBlock;
      const int64_t* tp = A.scratch + (((uint64_t)part * n_cta1 + c) * A.cap + off) * (uint64_t)tw;
      const uint32_t m = min((uint32_t)kTupleBlock, cnt - off);
      constexpr int U = kTupleBlock / 32;
      int64_t key[U], v0[U];
      uint32_t pos[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint32_t i = lane + 32u * u;
        key[u] = B2Q_I64_MAX; v0[u] = 0;
        if (i < m) {
          if (tw == 2) asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%0, %1}, [%2], %3;" : "=l"(key[u]), "=l"(v0[u]) : "l"(tp + (size_t)i * 2), "l"(pol));
          else key[u] = __ldcg(tp + (size_t)i * tw);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) pos[u] = bucket_of_mix(mix_key(key[u]), nb_mask);
      /* the common case — the key sits in its first bucket — for all U tuples at once: 2 U independent 16-byte loads in
       * flight, no claim, no second bucket, no divergence.  Whatever is left (a key's first appearance in the partition, a
       * full first bucket: ~6 % of the tuples, but at least one lane of 5 warps out of 6) is NOT resolved here — ncu on the
       * version that called bucket_find for the odd lanes right away: nearly half of the kernel's warp instructions were that
       * call, executed for one or two active lanes.  Those tuples are parked in a queue of the
       * warp in shared memory and resolved 32 at a time, one per lane. */
      int e[U];
      uint32_t hits = 0;
#pragma unroll
      for (int u = 0; u < U; ++u) { /* (checking the following bucket here as well was measured slower) */
        const int64_t* bk = s_keys + (size_t)pos[u] * kBucket;
        const longlong2 ka = *reinterpret_cast<const longlong2*>(bk);
        const longlong2 kb = *reinterpret_cast<const longlong2*>(bk + 2);
        const uint32_t hit = (uint32_t)(ka.x == key[u]) | (uint32_t)(ka.y == key[u]) << 1 | (uint32_t)(kb.x == key[u]) << 2 | (uint32_t)(kb.y == key[u]) << 3;
        e[u] = (int)(pos[u] * kBucket) + __ffs(hit) - 1;
        hits |= (uint32_t)(hit != 0) << u;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint32_t i = lane + 32u * u;
        const bool live = i < m, hit = hits >> u & 1;
        const int64_t aux = tw <= 2 ? v0[u] : (int64_t)(tp + (size_t)i * tw); /* the value itself, or where the tuple lies */
        const bool park = live && !hit;
        const uint32_t pm = __ballot_sync(0xffffffffu, park);
        if (pm) {
          if (park) {
            const uint32_t at = qn + __popc(pm & lt);
            q_key[at] = key[u];
            q_aux[at] = aux;
          }
          qn += __popc(pm);
          __syncwarp();
          if (qn >= 32) { qn -= 32; update(q_key[qn + lane], q_aux[qn + lane], -2, true); __syncwarp(); }
        }
        if (live && hit) update(key[u], aux, e[u], false);
      }
    }
    if (qn) { /* what is left in the warp's queue */
      update(lane < qn ? q_key[lane] : 0, lane < qn ? q_aux[lane] : 0, lane < qn ? -2 : -3, true);
      qn = 0;
      __syncwarp();
    }
    __syncthreads();
    /* ---- merge the private table into the table in HBM: the reference's probe, once per key ---- */
    for (uint32_t i = tid; i < S; i += nthr) {
      const int64_t key = s_keys[i];
      if (key == B2Q_I64_MAX) continue;
      const int64_t e = global_probe(reinterpret_cast<unsigned long long*>(Lh.keys), n, home_slot(key, hw, magic, n), key);
      if (e < 0) { atomicCAS(Lh.error, 0, B2Q_ERR_OUT_OF_SLOTS); continue; }
      for (int a = 0; a < n_accs; ++a) {
        const int8_t* base = s_acc + (size_t)A.acc_off[a] * S;
        if (A.acc_bytes[a] == 4) { const uint32_t x = reinterpret_cast<const uint32_t*>(base)[i]; if (x) red_add_u64(Lh.accs[a] + e, (uint64_t)x); }
        else global_acc_merge(P.accs[a].op, Lh.accs[a] + e, reinterpret_cast<const int64_t*>(base)[i]);
      }
    }
  }
}

/* ==========================================================================================================
 * cross-device merge of baseline-hash tables: ResultSetStorage::reduce's re-probe (ResultSetReduction.cpp:698-828 — every
 * non-empty entry of `that` is looked up / claimed in `this` with the group-by probe and its slots are reduced one by one)
 * run by a grid over the peers' tables instead of a host loop
 * ======================================================================================================== */
struct MergeArgs {
  const int64_t* src_keys;             /* [n_src] entries of the peers' key arrays, EMPTY_KEY_64 = no entry */
  const int64_t* src_accs[B2Q_MAX_ACCS];
  int64_t n_src;
  int64_t skip_begin, skip_end;        /* entries of this rank's own block inside the gathered arrays */
  int64_t* keys;
  int64_t* accs[B2Q_MAX_ACCS];
  int32_t* error;
  int8_t ops[B2Q_MAX_ACCS];
  int32_t bm_words[B2Q_MAX_ACCS];      /* ACC_BITMAP: 32-bit words per entry of the COUNT(DISTINCT) bitmaps (the arrays are [entries][bm_words]) */
  int32_t n_accs, hash_key_width;
  uint32_t entry_count;
  uint64_t hash_magic;
};

__global__ void b2q_k_baseline_merge(const __grid_constant__ MergeArgs A) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < A.n_src; i += stride) {
    if (i >= A.skip_begin && i < A.skip_end) continue;
    const int64_t key = A.src_keys[i];
    if (key == B2Q_I64_MAX) continue;
    const int64_t e = global_probe(reinterpret_cast<unsigned long long*>(A.keys), A.entry_count, home_slot(key, A.hash_key_width, A.hash_magic, A.entry_count), key);
    if (e < 0) { atomicCAS(A.error, 0, B2Q_ERR_OUT_OF_SLOTS); continue; }
    for (int a = 0; a < A.n_accs; ++a) {
      if (A.ops[a] == ACC_BITMAP) { /* count_distinct_set_union (CountDistinct.h:89-140): OR the peer's bitmap of this group into ours */
        const int w = A.bm_words[a];
        const uint32_t* src = reinterpret_cast<const uint32_t*>(A.src_accs[a]) + (size_t)i * w;
        uint32_t* dst = reinterpret_cast<uint32_t*>(A.accs[a]) + (size_t)e * w;
        for (int k = 0; k < w; ++k) { const uint32_t bits = src[k]; if (bits) atomicOr(dst + k, bits); }
      } else global_acc_merge(A.ops[a], A.accs[a] + e, A.src_accs[a][i]);
    }
  }
}

/* ==========================================================================================================
 * host side
 * ======================================================================================================== */
int sm_count();
static size_t radix_tile_smem(const RadixPlan& rp);

cudaError_t launch_baseline_merge(const B2QQuery& q, const int64_t* src_keys, const int64_t* const* src_accs, int64_t n_src, int64_t skip_begin,
                                  int64_t skip_end, int64_t* keys, int64_t* const* accs, int32_t* error, cudaStream_t st) {
  MergeArgs a;
  memset(&a, 0, sizeof(a));
  a.src_keys = src_keys;
  a.n_src = n_src;
  a.skip_begin = skip_begin;
  a.skip_end = skip_end;
  a.keys = keys;
  a.error = error;
  a.n_accs = q.prog.n_accs;
  for (int i = 0; i < q.prog.n_accs; ++i) { a.src_accs[i] = src_accs[i]; a.accs[i] = accs[i]; a.ops[i] = q.prog.accs[i].op; a.bm_words[i] = q.prog.accs[i].bm_words; }
  a.hash_key_width = q.prog.key.hash_key_width;
  a.entry_count = static_cast<uint32_t>(q.prog.key.entry_count);
  a.hash_magic = q.prog.key.hash_magic;
  if (n_src <= 0) return cudaSuccess;
  const int grid = static_cast<int>(std::max<int64_t>(1, std::min<int64_t>((n_src + 255) / 256, sm_count() * 8)));
  b2q_k_baseline_merge<<<grid, 256, 0, st>>>(a);
  return cudaGetLastError();
}

bool radix_plan(const B2QQuery& q, RadixPlan* rp) {
  const DevProgram& P = q.prog;
  memset(rp, 0, sizeof(*rp));
  if (q.plan.kernel != B2Q_KERNEL_BASELINE_GLOBAL || P.join.fk_col >= 0 || P.n_keys > 1 || P.key.col < 0) return false;
  if (q.plan.entry_count < 1 || q.plan.entry_count > (int64_t(1) << 31)) return false;
  /* tuple = {key, one word per distinct aggregate argument column} */
  int n_vals = 0;
  for (int a = 0; a < P.n_accs; ++a) {
    const DevAcc& acc = P.accs[a];
    if (acc.op == ACC_TOUCH || acc.op == ACC_NDV || acc.op == ACC_BITMAP) return false;
    if (acc.is_fp && acc.width != 8) return false; /* FLOAT arguments: tuples carry integer-widened words */
    rp->acc_val[a] = -1;
    if (acc.col < 0) continue;
    int vi = -1;
    for (int c = 0; c < n_vals; ++c) if (rp->val_col[c] == acc.col) vi = c;
    if (vi < 0) {
      if (n_vals == B2Q_RADIX_MAX_VALS) return false;
      rp->val_col[n_vals] = static_cast<int8_t>(acc.col);
      rp->val_width[n_vals] = acc.width;
      vi = n_vals++;
    }
    rp->acc_val[a] = static_cast<int8_t>(vi);
  }
  rp->n_vals = n_vals;
  rp->tuple_words = 1 + n_vals;
  /* pass 2, shared-memory bytes per entry: key + 4 (COUNT / integer SUM) or 8 per accumulator, 8-byte arrays first */
  int off = 0;
  for (int pass = 0; pass < 2; ++pass)
    for (int a = 0; a < P.n_accs; ++a) {
      const int bytes = (P.accs[a].op == ACC_COUNT || P.accs[a].op == ACC_SUM_I64) ? 4 : 8;
      if ((pass == 0) != (bytes == 8)) continue;
      rp->acc_bytes[a] = static_cast<int8_t>(bytes);
      rp->acc_off[a] = static_cast<int16_t>(off);
      off += bytes;
    }
  rp->acc_bytes_total = off;
  /* slice: the largest power of two of entries whose keys + accumulators (+ overflow area) fit the shared memory of a CTA */
  const int64_t entry_bytes = 8 + off;
  const int64_t budget = 193 * 1024; /* of the 227 KB a CTA may opt in to: 32 KB are the warps' queues, ~1 KB the block prefix */
  int log_s = 4;
  while (log_s < 20 && (int64_t(2) << log_s) * entry_bytes <= budget) ++log_s;
  if ((int64_t(1) << log_s) * entry_bytes > budget) return false;
  rp->log_s = log_s;
  const int64_t S = int64_t(1) << log_s;
  rp->n_parts = static_cast<int32_t>((q.plan.entry_count + S - 1) / S);
  if (rp->n_parts > 8192) return false; /* per-CTA counters / the open lines of #SM x n_parts regions */
  /* pass 1 buckets a chunk in shared memory when the tile (8192 tuples), its partition ids and three counters per partition fit */
  rp->tile = rp->tuple_words <= 2 && radix_tile_smem(*rp) <= 220 * 1024;
  return true;
}

static size_t radix_tile_smem(const RadixPlan& rp) {
  const size_t tile = static_cast<size_t>(kRadixBlock) * R;
  return tile * rp.tuple_words * 8 + (static_cast<size_t>(rp.n_parts) * 3 + 1) * 4 + tile * 2 + 16;
}
size_t radix_smem_pass1(const RadixPlan& rp) { return rp.tile ? radix_tile_smem(rp) : static_cast<size_t>(rp.n_parts) * 4; }

/* pass 2: [keys S x 8][accumulators][block prefix n_cta1 + 1][per-warp queues of parked tuples] */
static size_t radix_queue_off(const RadixPlan& rp, int n_cta1) {
  const size_t S = size_t(1) << rp.log_s;
  return (S * (8 + rp.acc_bytes_total) + (static_cast<size_t>(n_cta1) + 1) * 4 + 15) / 16 * 16;
}
size_t radix_smem_pass2(const B2QQuery&, const RadixPlan& rp, int n_cta1) {
  const size_t S = size_t(1) << rp.log_s;
  return radix_queue_off(rp, n_cta1) + static_cast<size_t>(kRadixBlock / 32) * 2 * kQueue * 8;
}

/* grid of pass 1 and the region capacity for a batch of `chunks` scan chunks */
void radix_geometry(const B2QQuery& q, const RadixPlan& rp, int64_t chunks, int* n_cta1, uint32_t* cap) {
  const int64_t ctas = std::max<int64_t>(1, std::min<int64_t>(sm_count(), chunks));
  const double rows_per_cta = static_cast<double>((chunks + ctas - 1) / ctas) * kRadixBlock * R;
  const double S = static_cast<double>(int64_t(1) << rp.log_s);
  const double mean = rows_per_cta * std::min(1.0, S / static_cast<double>(q.plan.entry_count));
  const double c = mean + 6.0 * sqrt(mean) + 16.0;
  *n_cta1 = static_cast<int>(ctas);
  *cap = static_cast<uint32_t>(std::min<double>(c, rows_per_cta + 1)) + 1u;
}

int radix_chunk_rows() { return kRadixBlock * R; }

cudaError_t launch_radix(const B2QQuery& q, const RadixPlan& rp, const DevLaunch& launch, const RadixBuffers& buf, int64_t chunk_begin,
                         int64_t chunk_end, int n_cta1, uint32_t cap, cudaStream_t st) {
  static std::atomic<unsigned long long> attr_mask{0};
  int dev = 0;
  cudaGetDevice(&dev);
  RadixArgs a;
  a.prog = q.prog;
  a.launch = launch;
  a.scratch = buf.scratch;
  a.counts = buf.counts;
  a.work_counter = buf.work_counter;
  a.n_parts = rp.n_parts;
  a.log_s = rp.log_s;
  a.n_cta1 = n_cta1;
  a.cap = cap;
  a.n_vals = rp.n_vals;
  a.tuple_words = rp.tuple_words;
  memcpy(a.val_col, rp.val_col, sizeof(a.val_col));
  memcpy(a.val_width, rp.val_width, sizeof(a.val_width));
  memcpy(a.acc_val, rp.acc_val, sizeof(a.acc_val));
  memcpy(a.acc_bytes, rp.acc_bytes, sizeof(a.acc_bytes));
  memcpy(a.acc_off, rp.acc_off, sizeof(a.acc_off));
  a.acc_bytes_total = rp.acc_bytes_total;
  a.queue_off = static_cast<int32_t>(radix_queue_off(rp, n_cta1));
  a.chunk_begin = chunk_begin;
  a.chunk_end = chunk_end;
  const size_t smem2 = radix_smem_pass2(q, rp, n_cta1);
  if (dev < 64 && !(attr_mask.load(std::memory_order_acquire) >> dev & 1ull)) {
    int optin = 0;
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    cudaFuncAttributes fa;
    const void* fns2[3] = {reinterpret_cast<const void*>(b2q_k_radix_aggregate<0, false>), reinterpret_cast<const void*>(b2q_k_radix_aggregate<1, true>),
                           reinterpret_cast<const void*>(b2q_k_radix_aggregate<2, true>)};
    for (const void* f : fns2) {
      cudaError_t e = cudaFuncGetAttributes(&fa, f);
      if (e != cudaSuccess) return e;
      e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes);
      if (e != cudaSuccess) return e;
    }
    attr_mask.fetch_or(1ull << dev, std::memory_order_release);
  }
  cudaError_t e = cudaMemsetAsync(buf.work_counter, 0, 8, st);
  if (e != cudaSuccess) return e;
  const bool key32 = q.prog.key.width != 8;
  const size_t smem1 = radix_smem_pass1(rp);
  if (rp.tile) {
    /* the four tile instantiations need the opt-in shared-memory limit, once per device */
    static std::atomic<unsigned long long> tile_mask{0};
    if (dev < 64 && !(tile_mask.load(std::memory_order_acquire) >> dev & 1ull)) {
      int optin = 0;
      cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
      const void* fns[4] = {reinterpret_cast<const void*>(b2q_k_radix_partition_tile<false, 1>), reinterpret_cast<const void*>(b2q_k_radix_partition_tile<false, 2>),
                            reinterpret_cast<const void*>(b2q_k_radix_partition_tile<true, 1>), reinterpret_cast<const void*>(b2q_k_radix_partition_tile<true, 2>)};
      for (const void* f : fns) {
        cudaFuncAttributes fa;
        e = cudaFuncGetAttributes(&fa, f);
        if (e != cudaSuccess) return e;
        e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes);
        if (e != cudaSuccess) return e;
      }
      tile_mask.fetch_or(1ull << dev, std::memory_order_release);
    }
    if (key32 && rp.tuple_words == 1) b2q_k_radix_partition_tile<true, 1><<<n_cta1, kRadixBlock, smem1, st>>>(a);
    else if (key32) b2q_k_radix_partition_tile<true, 2><<<n_cta1, kRadixBlock, smem1, st>>>(a);
    else if (rp.tuple_words == 1) b2q_k_radix_partition_tile<false, 1><<<n_cta1, kRadixBlock, smem1, st>>>(a);
    else b2q_k_radix_partition_tile<false, 2><<<n_cta1, kRadixBlock, smem1, st>>>(a);
  } else if (key32) b2q_k_radix_partition<true><<<n_cta1, kRadixBlock, smem1, st>>>(a);
  else b2q_k_radix_partition<false><<<n_cta1, kRadixBlock, smem1, st>>>(a);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const int grid2 = std::max(1, std::min(sm_count(), rp.n_parts));
  const DevProgram& P = q.prog;
  const bool fused = P.n_accs == 1 && rp.acc_bytes[0] == 4 && !P.accs[0].skip1_en && !P.accs[0].skip2_en && rp.tuple_words <= 2;
  if (fused && rp.tuple_words == 2) b2q_k_radix_aggregate<2, true><<<grid2, kRadixBlock, smem2, st>>>(a);
  else if (fused) b2q_k_radix_aggregate<1, true><<<grid2, kRadixBlock, smem2, st>>>(a);
  else b2q_k_radix_aggregate<0, false><<<grid2, kRadixBlock, smem2, st>>>(a);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  return cudaGetLastError();
}

}  // namespace b2q
