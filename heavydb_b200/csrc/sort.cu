/*
 * sort.cu — ORDER BY / LIMIT over the aggregated table, on the device (SURVEY §8f-1).
 *
 * Replaces, for the output of this path, what the reference does on the host after executeWorkUnit returns
 * (RelAlgExecutor::executeSort, RelAlgExecutor.cpp:3586-3610):
 *     ResultSet::sort(order_entries, limit + offset)     ResultSet.cpp:781-849
 *       initPermutationBuffer  — indices of the non-empty entries            :870-885
 *       ResultSetComparator    — per order entry: NULLs first/last, then int / double / AVG-pair compare   :1310-1478
 *       topPermutation         — std::partial_sort / std::sort               :1501-1527
 *     dropFirstN(offset), keepFirstN(limit)                                  :58-66
 * and, on the reference's GPU path, the thrust sort of InPlaceSortImpl.cu:25-60 / TopKSort.cu.
 *
 * Device algorithm (all kernels hand-written, no thrust/cub):
 *   1. ordered stream compaction of the non-empty entries -> perm[] (ascending entry index)
 *   2. for every order entry, LAST to FIRST (LSD over the composite key): build an order-preserving 64-bit image of
 *      the entry's value (DESC = complemented), stable 8-bit radix sort passes (passes whose digit is uniform
 *      degenerate to a copy), then one stable pass on the NULL rank (nulls_first ? 0 : 2, value 1)
 *   3. gather the first top_n rows into a compact buffer in the same row-wise / columnar layout, so only the rows
 *      that are kept cross PCIe.
 * Ties keep ascending entry order (every pass is stable); the reference's std::sort leaves ties unspecified.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <utility>
#include <vector>

#include "b2q_internal.h"

namespace {

constexpr int SORT_BLOCK = 256;
constexpr int SORT_WARPS = SORT_BLOCK / 32;
constexpr int SORT_ITEMS = 8;
constexpr int SORT_TILE = SORT_BLOCK * SORT_ITEMS;

__device__ __forceinline__ const int8_t* slot_addr(const DevSortLayout& L, const int8_t* buf, int64_t e, int64_t off, int w) {
  return L.columnar ? buf + off + e * w : buf + e * L.row_size + off;
}
__device__ __forceinline__ int64_t read_slot(const DevSortLayout& L, const int8_t* buf, int64_t e, int64_t off, int w) {
  const int8_t* p = slot_addr(L, buf, e, off, w);
  if (w == 1) return *p; /* logical-sized columns of a columnar projection */
  if (w == 2) return *reinterpret_cast<const int16_t*>(p);
  return w == 4 ? (int64_t) * reinterpret_cast<const int32_t*>(p) : *reinterpret_cast<const int64_t*>(p);
}
/* ResultSetStorage::isEmptyEntry / isEmptyEntryColumnar (ResultSetIteration.cpp:2457-2545) */
__device__ __forceinline__ bool entry_empty(const DevSortLayout& L, const int8_t* buf, int64_t e) {
  if (!L.grouped) return false;
  if (L.keyless) return read_slot(L, buf, e, L.marker_off, L.marker_w) == L.marker_init;
  if (L.key_w == 4) return *reinterpret_cast<const int32_t*>(slot_addr(L, buf, e, 0, 4)) == 0x7FFFFFFF;
  return *reinterpret_cast<const int64_t*>(slot_addr(L, buf, e, 0, 8)) == B2Q_I64_MAX;
}

/* ---- 1. ordered compaction ---------------------------------------------------------------------------------- */
__global__ void b2q_k_sort_count(const DevSortLayout L, const int8_t* __restrict__ buf, uint32_t* __restrict__ block_counts) {
  const int64_t base = (int64_t)blockIdx.x * SORT_TILE;
  int c = 0;
  for (int k = 0; k < SORT_ITEMS; ++k) {
    const int64_t e = base + (int64_t)k * SORT_BLOCK + threadIdx.x;
    c += (e < L.entry_count && !entry_empty(L, buf, e)) ? 1 : 0;
  }
  __shared__ int s_sum[SORT_WARPS];
  for (int o = 16; o; o >>= 1) c += __shfl_down_sync(~0u, c, o);
  if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < SORT_WARPS; ++w) t += s_sum[w];
    block_counts[blockIdx.x] = (uint32_t)t;
  }
}

/* single-block exclusive scan of `n` uint32 (in place); writes the grand total to *total */
__global__ void b2q_k_sort_scan(uint32_t* __restrict__ a, int64_t n, uint32_t* __restrict__ total) {
  __shared__ uint32_t s_part[1024];
  const int t = threadIdx.x, T = blockDim.x;
  const int64_t per = (n + T - 1) / T;
  const int64_t lo = (int64_t)t * per, hi = lo + per < n ? lo + per : n;
  uint32_t sum = 0;
  for (int64_t i = lo; i < hi; ++i) sum += a[i];
  s_part[t] = sum;
  __syncthreads();
  for (int o = 1; o < T; o <<= 1) { /* Hillis-Steele inclusive scan of the per-thread sums */
    const uint32_t v = t >= o ? s_part[t - o] : 0;
    __syncthreads();
    s_part[t] += v;
    __syncthreads();
  }
  uint32_t run = t ? s_part[t - 1] : 0;
  for (int64_t i = lo; i < hi; ++i) {
    const uint32_t v = a[i];
    a[i] = run;
    run += v;
  }
  if (t == T - 1 && total) *total = s_part[T - 1];
}

__global__ void b2q_k_sort_compact(const DevSortLayout L, const int8_t* __restrict__ buf, const uint32_t* __restrict__ block_offsets,
                                   uint32_t* __restrict__ perm) {
  __shared__ uint32_t s_warp[SORT_WARPS];
  __shared__ uint32_t s_run;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_run = block_offsets[blockIdx.x];
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * SORT_TILE;
  for (int k = 0; k < SORT_ITEMS; ++k) {
    const int64_t e = base + (int64_t)k * SORT_BLOCK + threadIdx.x;
    const bool keep = e < L.entry_count && !entry_empty(L, buf, e);
    const uint32_t m = __ballot_sync(~0u, keep);
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    uint32_t before = s_run;
    for (int w = 0; w < warp; ++w) before += s_warp[w];
    if (keep) perm[before + __popc(m & ((1u << lane) - 1u))] = (uint32_t)e;
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t t = 0;
      for (int w = 0; w < SORT_WARPS; ++w) t += s_warp[w];
      s_run += t;
    }
    __syncthreads();
  }
}

/* ---- 2. sort keys ------------------------------------------------------------------------------------------- */
__device__ __forceinline__ double avg_of(const DevSortKey& K, int64_t sum, int64_t cnt) { /* pair_to_double, ResultSetBufferAccessors.h:197-227 */
  const double dividend = K.kind == SORTKEY_AVG_F64   ? __longlong_as_double(sum)
                          : K.kind == SORTKEY_AVG_F32 ? (double)__int_as_float((int32_t)sum)
                                                      : (double)sum;
  return K.scale ? dividend / ((double)cnt * b2q_exp_to_scale(K.scale)) : dividend / (double)cnt;
}
__device__ __forceinline__ uint64_t f64_key(double d) {
  if (d == 0.0) d = 0.0; /* -0.0 and +0.0 compare equal in the reference's `<` */
  const uint64_t b = (uint64_t)__double_as_longlong(d);
  return (b >> 63) ? ~b : b | 0x8000000000000000ull;
}

/* mode 0: order-preserving value image (0 for NULLs so they tie); mode 1: the NULL rank */
__global__ void b2q_k_sort_make_keys(const DevSortLayout L, const DevSortKey K, const int8_t* __restrict__ buf,
                                     const uint32_t* __restrict__ perm, int64_t n, uint64_t* __restrict__ keys, int mode) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    const int64_t e = perm[j];
    const int64_t v = read_slot(L, buf, e, K.off1, K.w1);
    bool is_null = false;
    uint64_t key;
    if (K.kind == SORTKEY_AVG_I64 || K.kind == SORTKEY_AVG_F64 || K.kind == SORTKEY_AVG_F32) {
      const int64_t cnt = read_slot(L, buf, e, K.off2, 8);
      is_null = K.nullable && cnt == 0; /* ResultSet::isNull for a pair: !val.i2 */
      key = f64_key(cnt == 0 ? 2.2250738585072014e-308 /* NULL_DOUBLE */ : avg_of(K, v, cnt));
    } else if (K.kind == SORTKEY_F64) {
      is_null = K.nullable && v == K.null_pattern;
      key = f64_key(__longlong_as_double(v));
    } else if (K.kind == SORTKEY_F32) { /* the slot's high word is not part of the value */
      const int32_t b = (int32_t)v;
      is_null = K.nullable && b == (int32_t)K.null_pattern;
      key = f64_key((double)__int_as_float(b)); /* widened exactly: the order of the floats */
    } else {
      is_null = K.nullable && v == K.null_pattern;
      key = (uint64_t)v ^ 0x8000000000000000ull;
    }
    if (mode == 0) keys[j] = is_null ? 0ull : (K.is_desc ? ~key : key);
    else keys[j] = is_null ? (K.nulls_first ? 0ull : 2ull) : 1ull;
  }
}

/* OR / AND of all keys: a digit position whose bits are equal in both is uniform and its pass can be skipped */
__global__ void b2q_k_sort_bits(const uint64_t* __restrict__ keys, int64_t n, unsigned long long* __restrict__ or_and) {
  unsigned long long o = 0, a = ~0ull;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) { o |= keys[j]; a &= keys[j]; }
  for (int s = 16; s; s >>= 1) { o |= __shfl_down_sync(~0u, o, s); a &= __shfl_down_sync(~0u, a, s); }
  if ((threadIdx.x & 31) == 0) { atomicOr(or_and, o); atomicAnd(or_and + 1, a); }
}

/* ---- top-k pre-filter: with LIMIT << groups, only entries whose PRIMARY sort key falls into the leading 16-bit buckets
 * that hold the first top_n entries can reach the output (the primary key dominates the order; ties and the further
 * order entries are settled by the full sort of the survivors).  bucket = NULL rank (2 bits) | top 14 bits of the key. */
/* `shift` drops the low bits so that the 14 bits kept are the highest ones in which the keys differ at all (bits above
 * them are equal for every key and do not order anything) */
__device__ __forceinline__ uint32_t topk_bucket(uint64_t key, uint64_t rank, int shift) {
  return (uint32_t)(rank << 14) | (uint32_t)((key >> shift) & 0x3FFFull);
}

__global__ void b2q_k_sort_bucket_hist(const uint64_t* __restrict__ keys, const uint64_t* __restrict__ ranks, int64_t n, int shift,
                                       uint32_t* __restrict__ hist16) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t n_round = (n + 31) & ~int64_t(31); /* whole warps stay in the loop for the match */
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n_round; j += stride) {
    const uint32_t b = j < n ? topk_bucket(keys[j], ranks ? ranks[j] : 1ull, shift) : 0xFFFFFFFFu;
    /* clustered keys would hammer one L2 address: lanes with the same bucket send one atomic */
    const uint32_t m = __match_any_sync(~0u, b);
    if (j < n && (m & ((1u << (threadIdx.x & 31)) - 1u)) == 0) atomicAdd(&hist16[b], (uint32_t)__popc(m));
  }
}

__global__ void b2q_k_sort_bucket_count(const uint64_t* __restrict__ keys, const uint64_t* __restrict__ ranks, int64_t n, int shift, uint32_t max_bucket,
                                        uint32_t* __restrict__ block_counts) {
  const int64_t base = (int64_t)blockIdx.x * SORT_TILE;
  int c = 0;
  for (int k = 0; k < SORT_ITEMS; ++k) {
    const int64_t j = base + (int64_t)k * SORT_BLOCK + threadIdx.x;
    c += (j < n && topk_bucket(keys[j], ranks ? ranks[j] : 1ull, shift) <= max_bucket) ? 1 : 0;
  }
  __shared__ int s_sum[SORT_WARPS];
  for (int o = 16; o; o >>= 1) c += __shfl_down_sync(~0u, c, o);
  if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < SORT_WARPS; ++w) t += s_sum[w];
    block_counts[blockIdx.x] = (uint32_t)t;
  }
}

__global__ void b2q_k_sort_bucket_compact(const uint64_t* __restrict__ keys, const uint64_t* __restrict__ ranks, int64_t n, int shift, uint32_t max_bucket,
                                          const uint32_t* __restrict__ block_offsets, const uint32_t* __restrict__ perm_in,
                                          uint32_t* __restrict__ perm_out) {
  __shared__ uint32_t s_warp[SORT_WARPS];
  __shared__ uint32_t s_run;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_run = block_offsets[blockIdx.x];
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * SORT_TILE;
  for (int k = 0; k < SORT_ITEMS; ++k) { /* ordered: the survivors keep ascending entry order (tie rule) */
    const int64_t j = base + (int64_t)k * SORT_BLOCK + threadIdx.x;
    const bool keep = j < n && topk_bucket(keys[j], ranks ? ranks[j] : 1ull, shift) <= max_bucket;
    const uint32_t m = __ballot_sync(~0u, keep);
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    uint32_t before = s_run;
    for (int w = 0; w < warp; ++w) before += s_warp[w];
    if (keep) perm_out[before + __popc(m & ((1u << lane) - 1u))] = perm_in[j];
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t t = 0;
      for (int w = 0; w < SORT_WARPS; ++w) t += s_warp[w];
      s_run += t;
    }
    __syncthreads();
  }
}

/* ---- stable LSD radix pass (8-bit digit) -------------------------------------------------------------------- */
__global__ void b2q_k_sort_hist(const uint64_t* __restrict__ keys, int64_t n, int shift, uint32_t* __restrict__ hist /* [256][nblocks] */,
                                uint32_t* __restrict__ bin_total /* [256] */) {
  __shared__ uint32_t s_h[256];
  s_h[threadIdx.x] = 0;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * SORT_TILE;
  for (int k = 0; k < SORT_ITEMS; ++k) {
    const int64_t j = base + (int64_t)k * SORT_BLOCK + threadIdx.x;
    if (j < n) atomicAdd(&s_h[(keys[j] >> shift) & 255u], 1u);
  }
  __syncthreads();
  const uint32_t c = s_h[threadIdx.x];
  hist[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = c;
  if (c) atomicAdd(&bin_total[threadIdx.x], c);
}

/* exclusive scan of the [256][nblocks] histogram in digit-major order, one CTA per digit: the digit's base is the
 * sum of the totals of the smaller digits (bin_total, accumulated by the histogram kernel), then a tiled block scan
 * along the row with a running carry — coalesced, 256 CTAs instead of one */
__global__ void b2q_k_sort_scan_rows(uint32_t* __restrict__ hist, int nblocks, const uint32_t* __restrict__ bin_total) {
  __shared__ uint32_t s_warp[32];
  __shared__ uint32_t s_carry;
  const int d = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  if (t < 32) { /* base = sum of bin_total[0..d) */
    uint32_t v = 0;
    for (int i = t; i < d; i += 32) v += bin_total[i];
    for (int o = 16; o; o >>= 1) v += __shfl_down_sync(~0u, v, o);
    if (t == 0) s_carry = v;
  }
  __syncthreads();
  uint32_t* row = hist + (size_t)d * nblocks;
  for (int base = 0; base < nblocks; base += blockDim.x) {
    const int i = base + t;
    const uint32_t v = i < nblocks ? row[i] : 0;
    uint32_t inc = v; /* inclusive warp scan */
    for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(~0u, inc, o); if (lane >= o) inc += u; }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
      uint32_t w = lane < (blockDim.x >> 5) ? s_warp[lane] : 0;
      for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(~0u, w, o); if (lane >= o) w += u; }
      s_warp[lane] = w; /* inclusive scan of the warp totals */
    }
    __syncthreads();
    const uint32_t carry = s_carry;
    const uint32_t before = carry + (warp ? s_warp[warp - 1] : 0) + inc - v;
    if (i < nblocks) row[i] = before;
    __syncthreads();
    if (t == blockDim.x - 1) s_carry = carry + s_warp[(blockDim.x >> 5) - 1];
    __syncthreads();
  }
}

/* uniform[0] = 1 when every key has the same digit: the scatter then degenerates to a copy */
__global__ void b2q_k_sort_uniform(const uint32_t* __restrict__ bin_total, int64_t n, uint32_t* __restrict__ uniform) {
  const bool u = bin_total[threadIdx.x] == (uint32_t)n;
  const int any = __syncthreads_or(u);
  if (threadIdx.x == 0) uniform[0] = any ? 1u : 0u;
}

__global__ void b2q_k_sort_scatter(const uint64_t* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
                                   uint64_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out, int64_t n, int shift,
                                   const uint32_t* __restrict__ hist_scanned, const uint32_t* __restrict__ uniform) {
  const int64_t base = (int64_t)blockIdx.x * SORT_TILE;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  /* element order inside the tile = (warp, k, lane): each warp owns a contiguous run, so ranks are stable */
  const int64_t wbase = base + (int64_t)warp * (SORT_ITEMS * 32);
  if (uniform[0]) {
    for (int k = 0; k < SORT_ITEMS; ++k) {
      const int64_t j = wbase + k * 32 + lane;
      if (j < n) { keys_out[j] = keys_in[j]; vals_out[j] = vals_in[j]; }
    }
    return;
  }
  __shared__ uint32_t s_cnt[SORT_WARPS][256];
  for (int i = threadIdx.x; i < SORT_WARPS * 256; i += SORT_BLOCK) (&s_cnt[0][0])[i] = 0;
  __syncthreads();
  uint64_t key[SORT_ITEMS];
  uint32_t rank[SORT_ITEMS];
  for (int k = 0; k < SORT_ITEMS; ++k) {
    const int64_t j = wbase + k * 32 + lane;
    const bool valid = j < n;
    key[k] = valid ? keys_in[j] : 0;
    const uint32_t d = valid ? (uint32_t)((key[k] >> shift) & 255u) : 256u; /* 256: matches only other invalid lanes */
    const uint32_t m = __match_any_sync(~0u, d);
    const uint32_t before = __popc(m & ((1u << lane) - 1u));
    uint32_t old = 0;
    if (valid && before == 0) { old = s_cnt[warp][d]; s_cnt[warp][d] = old + __popc(m); } /* one leader per digit, warp-private row */
    old = __shfl_sync(~0u, old, __ffs(m) - 1);
    rank[k] = old + before;
    __syncwarp();
  }
  __syncthreads();
  /* exclusive prefix over the warps per digit + the tile's global base */
  {
    const int d = threadIdx.x; /* 256 threads == 256 digits */
    uint32_t run = hist_scanned[(size_t)d * gridDim.x + blockIdx.x];
    for (int w = 0; w < SORT_WARPS; ++w) {
      const uint32_t c = s_cnt[w][d];
      s_cnt[w][d] = run;
      run += c;
    }
  }
  __syncthreads();
  for (int k = 0; k < SORT_ITEMS; ++k) {
    const int64_t j = wbase + k * 32 + lane;
    if (j < n) {
      const uint32_t d = (uint32_t)((key[k] >> shift) & 255u);
      const uint32_t pos = s_cnt[warp][d] + rank[k];
      keys_out[pos] = key[k];
      vals_out[pos] = vals_in[j];
    }
  }
}

/* ---- 3. gather the kept rows into a compact buffer of the same layout ---------------------------------------- */
__global__ void b2q_k_sort_gather(const DevSortLayout Lin, const int8_t* __restrict__ in, int8_t* __restrict__ out,
                                  const uint32_t* __restrict__ perm, int64_t first, int64_t n_out, const DevGatherCols G) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  if (!Lin.columnar) {
    const int64_t words = Lin.row_size / 8;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_out * words; i += stride) {
      const int64_t r = i / words, w = i - r * words;
      reinterpret_cast<int64_t*>(out)[r * words + w] = reinterpret_cast<const int64_t*>(in)[(int64_t)perm[first + r] * words + w];
    }
    return;
  }
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_out; r += stride) {
    const int64_t e = perm[first + r];
    for (int c = 0; c < G.n; ++c) {
      switch (G.width[c]) {
        case 1: (out + G.out_off[c])[r] = (in + G.in_off[c])[e]; break;
        case 2: reinterpret_cast<int16_t*>(out + G.out_off[c])[r] = reinterpret_cast<const int16_t*>(in + G.in_off[c])[e]; break;
        case 4: reinterpret_cast<int32_t*>(out + G.out_off[c])[r] = reinterpret_cast<const int32_t*>(in + G.in_off[c])[e]; break;
        default: reinterpret_cast<int64_t*>(out + G.out_off[c])[r] = reinterpret_cast<const int64_t*>(in + G.in_off[c])[e];
      }
    }
    if (r == n_out - 1) /* column padding of narrow columns up to 8 bytes (recycled buffer) */
      for (int c = 0; c < G.n; ++c)
        for (int64_t b = n_out * G.width[c]; b & 7; ++b) (out + G.out_off[c])[b] = 0;
  }
}

int grid_for(int64_t n, int block, int cap) {
  int64_t b = (n + block - 1) / block;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace

namespace b2q {

int sm_count();

/* Step 1 on its own: the non-empty entries of `buf` in ascending order -> perm[0, *n_out).  block_counts holds
 * ceil(entry_count / SORT_TILE) words, perm entry_count words; d_total is one device word.  One stream synchronisation
 * (the count decides the caller's next allocation). */
size_t compact_scratch_bytes(int64_t entries) {
  const size_t n = (size_t)(entries > 0 ? entries : 1);
  auto pad = [](size_t x) { return (x + 255) & ~size_t(255); };
  return pad((n + SORT_TILE - 1) / SORT_TILE * 4) + pad(n * 4) + 256;
}

cudaError_t compact_entries(const DevSortLayout& L, const int8_t* buf, uint32_t* block_counts, uint32_t* perm, uint32_t* d_total,
                            cudaStream_t st, int64_t* n_out) {
  *n_out = 0;
  if (L.entry_count <= 0) return cudaSuccess;
  const int nblocks = (int)((L.entry_count + SORT_TILE - 1) / SORT_TILE);
  b2q_k_sort_count<<<nblocks, SORT_BLOCK, 0, st>>>(L, buf, block_counts);
  b2q_k_sort_scan<<<1, 1024, 0, st>>>(block_counts, (int64_t)nblocks, d_total);
  b2q_k_sort_compact<<<nblocks, SORT_BLOCK, 0, st>>>(L, buf, block_counts, perm);
  uint32_t h_total = 0;
  cudaError_t e = cudaMemcpyAsync(&h_total, d_total, 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return e;
  *n_out = h_total;
  return cudaSuccess;
}

/* Bytes of device scratch sort_device() needs for a table of `entries` entries. */
size_t sort_scratch_bytes(int64_t entries) {
  const size_t n = (size_t)(entries > 0 ? entries : 1);
  const size_t nblocks = (n + SORT_TILE - 1) / SORT_TILE;
  auto pad = [](size_t x) { return (x + 255) & ~size_t(255); };
  return pad(nblocks * 4) + 2 * pad(n * 4) + 2 * pad(n * 8) + pad(256 * nblocks * 4) + pad(256 * 4) + 1024 + pad(65536 * 4);
}

/* Sorts the non-empty entries of the device buffer `buf` (layout L) by `keys` (n_keys order entries).
 * Returns in *perm_out a pointer (inside `scratch`) to the sorted entry indices and in *n_out their count.
 * One stream synchronisation (the count of non-empty entries decides every later grid). */
/* `stop` (the call's interrupt token, or NULL) is read after each of those host waits; once it is set nothing more is enqueued
 * and *stopped says so (the permutation is then incomplete). */
cudaError_t sort_device(const DevSortLayout& L, const DevSortKey* keys, int n_keys, const int8_t* buf, int8_t* scratch,
                        cudaStream_t st, const uint32_t** perm_out, int64_t* n_out, int* launches, int64_t top_n,
                        const volatile uint32_t* stop, bool* stopped) {
  *stopped = false;
  auto interrupted = [&]() { if (stop && *stop) *stopped = true; return *stopped; };
  const int64_t n_entries = L.entry_count;
  const size_t nblocks_c = (size_t)((n_entries + SORT_TILE - 1) / SORT_TILE);
  auto pad = [](size_t x) { return (x + 255) & ~size_t(255); };
  int8_t* p = scratch;
  uint32_t* block_counts = reinterpret_cast<uint32_t*>(p); p += pad(std::max<size_t>(nblocks_c, 1) * 4);
  uint32_t* perm_a = reinterpret_cast<uint32_t*>(p); p += pad((size_t)std::max<int64_t>(n_entries, 1) * 4);
  uint32_t* perm_b = reinterpret_cast<uint32_t*>(p); p += pad((size_t)std::max<int64_t>(n_entries, 1) * 4);
  uint64_t* keys_a = reinterpret_cast<uint64_t*>(p); p += pad((size_t)std::max<int64_t>(n_entries, 1) * 8);
  uint64_t* keys_b = reinterpret_cast<uint64_t*>(p); p += pad((size_t)std::max<int64_t>(n_entries, 1) * 8);
  uint32_t* hist = reinterpret_cast<uint32_t*>(p); p += pad(256 * std::max<size_t>(nblocks_c, 1) * 4);
  uint32_t* bin_total = reinterpret_cast<uint32_t*>(p); p += pad(256 * 4);
  uint32_t* d_total = reinterpret_cast<uint32_t*>(p);
  uint32_t* d_uniform = d_total + 1;
  unsigned long long* d_bits = reinterpret_cast<unsigned long long*>(p + 64);
  uint32_t* hist16 = reinterpret_cast<uint32_t*>(p + 1024);
  *launches = 0;
  *perm_out = perm_a;
  *n_out = 0;
  if (n_entries <= 0) return cudaSuccess;

  cudaError_t e = compact_entries(L, buf, block_counts, perm_a, d_total, st, n_out);
  *launches += 3;
  if (e != cudaSuccess || interrupted()) return e;
  uint32_t h_total = 0;
  int64_t n = *n_out; /* the number of non-empty entries, whatever is sorted below */
  if (n <= 1 || n_keys == 0) return cudaGetLastError();

  uint32_t* pin = perm_a;
  uint32_t* pout = perm_b;
  if (top_n > 0 && n >= 65536 && top_n * 8 <= n) {
    /* top-k pre-filter on the primary order entry (see topk_bucket) */
    const int g0 = grid_for(n, 256, sm_count() * 8);
    const int nb0 = (int)((n + SORT_TILE - 1) / SORT_TILE);
    b2q_k_sort_make_keys<<<g0, 256, 0, st>>>(L, keys[0], buf, pin, n, keys_a, 0);
    const uint64_t* ranks = nullptr;
    if (keys[0].nullable) { b2q_k_sort_make_keys<<<g0, 256, 0, st>>>(L, keys[0], buf, pin, n, keys_b, 1); ranks = keys_b; *launches += 1; }
    unsigned long long hb[2] = {0ull, ~0ull};
    cudaMemcpyAsync(d_bits, hb, 16, cudaMemcpyHostToDevice, st);
    b2q_k_sort_bits<<<g0, 256, 0, st>>>(keys_a, n, d_bits);
    e = cudaMemcpyAsync(hb, d_bits, 16, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess || interrupted()) return e;
    const unsigned long long kdiff = hb[0] ^ hb[1];
    const int msb = kdiff ? 63 - __builtin_clzll(kdiff) : 0;
    const int shift = msb > 13 ? msb - 13 : 0;
    cudaMemsetAsync(hist16, 0, 65536 * 4, st);
    b2q_k_sort_bucket_hist<<<g0, 256, 0, st>>>(keys_a, ranks, n, shift, hist16);
    *launches += 3;
    std::vector<uint32_t> h16(65536);
    e = cudaMemcpyAsync(h16.data(), hist16, 65536 * 4, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess || interrupted()) return e;
    uint32_t max_bucket = 65535;
    int64_t cum = 0;
    for (uint32_t b = 0; b < 65536; ++b) { cum += h16[b]; if (cum >= top_n) { max_bucket = b; break; } }
    if (cum < n) { /* worth it: fewer survivors than entries */
      b2q_k_sort_bucket_count<<<nb0, SORT_BLOCK, 0, st>>>(keys_a, ranks, n, shift, max_bucket, block_counts);
      b2q_k_sort_scan<<<1, 1024, 0, st>>>(block_counts, (int64_t)nb0, d_total);
      b2q_k_sort_bucket_compact<<<nb0, SORT_BLOCK, 0, st>>>(keys_a, ranks, n, shift, max_bucket, block_counts, pin, pout);
      *launches += 3;
      e = cudaMemcpyAsync(&h_total, d_total, 4, cudaMemcpyDeviceToHost, st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(st);
      if (e != cudaSuccess || interrupted()) return e;
      std::swap(pin, pout);
      n = h_total; /* >= top_n survivors, in ascending entry order */
    }
  }

  const int nblocks = (int)((n + SORT_TILE - 1) / SORT_TILE);
  const int kgrid = grid_for(n, 256, sm_count() * 8);
  auto radix_pass = [&](int shift) {
    cudaMemsetAsync(bin_total, 0, 256 * 4, st);
    b2q_k_sort_hist<<<nblocks, SORT_BLOCK, 0, st>>>(keys_a, n, shift, hist, bin_total);
    b2q_k_sort_uniform<<<1, 256, 0, st>>>(bin_total, n, d_uniform);
    b2q_k_sort_scan_rows<<<256, 1024, 0, st>>>(hist, nblocks, bin_total);
    b2q_k_sort_scatter<<<nblocks, SORT_BLOCK, 0, st>>>(keys_a, pin, keys_b, pout, n, shift, hist, d_uniform);
    *launches += 4;
    std::swap(keys_a, keys_b);
    std::swap(pin, pout);
  };
  for (int k = n_keys - 1; k >= 0; --k) {
    b2q_k_sort_make_keys<<<kgrid, 256, 0, st>>>(L, keys[k], buf, pin, n, keys_a, 0);
    *launches += 1;
    /* which digit positions actually differ: one tiny reduction + an 16-byte copy-back instead of up to 8 passes */
    unsigned long long h_bits[2] = {0ull, ~0ull};
    cudaMemcpyAsync(d_bits, h_bits, 16, cudaMemcpyHostToDevice, st);
    b2q_k_sort_bits<<<kgrid, 256, 0, st>>>(keys_a, n, d_bits);
    *launches += 1;
    e = cudaMemcpyAsync(h_bits, d_bits, 16, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess || interrupted()) return e;
    const unsigned long long diff = h_bits[0] ^ h_bits[1];
    for (int shift = 0; shift < 64; shift += 8) if ((diff >> shift) & 255ull) radix_pass(shift);
    if (keys[k].nullable) {
      b2q_k_sort_make_keys<<<kgrid, 256, 0, st>>>(L, keys[k], buf, pin, n, keys_a, 1);
      *launches += 1;
      radix_pass(0);
    }
  }
  *perm_out = pin;
  return cudaGetLastError();
}

cudaError_t sort_gather(const DevSortLayout& Lin, const DevGatherCols& G, const int8_t* in, int8_t* out,
                        const uint32_t* perm, int64_t first, int64_t n_out, cudaStream_t st) {
  if (n_out <= 0) return cudaSuccess;
  const int64_t work = Lin.columnar ? n_out : n_out * (Lin.row_size / 8);
  b2q_k_sort_gather<<<grid_for(work, 256, sm_count() * 16), 256, 0, st>>>(Lin, in, out, perm, first, n_out, G);
  return cudaGetLastError();
}

}  // namespace b2q
