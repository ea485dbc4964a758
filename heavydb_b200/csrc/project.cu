/*
 * project.cu — the projection kernel (b2q_k_project): scan -> filter -> ordered stream compaction of the passing rows into the
 * reference's projection buffer, stopping at the scan limit.
 *
 * The reference's GPU kernel claims each output row with an atomic add on TOTAL_MATCHED (GroupByAndAggregate.cpp:1080-1101),
 * so its row order is arbitrary and, under a scan limit, so is WHICH rows survive.  This kernel writes the one deterministic
 * admissible answer: rows in (fragment, row) order, what resultsUnion makes of per-fragment results; under a scan limit the
 * first scan_limit passing rows in that order.
 *
 *   - chunk geometry, column loads, filter evaluation and the evict-first policy are b2q_k_scan's (scan_kernel.cuh);
 *   - chunks are claimed with a ticket (atomic counter), so they are claimed in order: a chunk only waits on chunks that
 *     running CTAs have already claimed, and forward progress does not depend on which CTAs are co-resident;
 *   - output offsets: pass bits -> __ballot_sync / __popc per (row slot, warp) -> CTA exclusive scan -> decoupled look-back
 *     over one 64-bit status word per chunk (2-bit flag + count, release / acquire at GPU scope).  No atomics on output
 *     positions;
 *   - the chunk whose inclusive prefix reaches the scan limit raises a done flag; a CTA checks it before it claims a chunk
 *     and before it loads any column, so LIMIT n reads a few chunks, not the table;
 *   - projected columns are loaded predicated on the rows that are written (a 32-byte sector without such a row is never
 *     fetched), decoded the way the chunk decoders hand them to agg_id (ENCODING FIXED / DICT(8|16) NULLs to the logical
 *     NULL, DAYS * 86400), staged compacted in shared memory and written by consecutive threads.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "scan_kernel.cuh"

namespace b2q {

constexpr int kProjBlock = 256;
constexpr int kProjWarps = kProjBlock / 32;
constexpr int64_t kProjChunk = (int64_t)kProjBlock * R;

/* status word of a chunk: flag in the top two bits, row count below */
constexpr unsigned long long kFlagAgg = 1ull << 62, kFlagInc = 2ull << 62, kCountMask = (1ull << 62) - 1;

struct ProjArgs {
  DevFilter filter;
  DevProject proj;
  const int8_t* const* col_ptrs;   /* [frag * n_cols + c] */
  const int64_t* frag_rows;        /* [n_frags] */
  const int64_t* frag_chunk_start; /* [n_frags + 1] */
  const int64_t* frag_row_base;    /* [n_frags]: added to the offset word (a host slice's first row), or nullptr */
  int32_t n_frags, n_cols;
  int64_t total_chunks;            /* chunks of this launch */
  int64_t chunk_base;              /* status index of this launch's chunk 0 (launches over host slices continue the order) */
  int8_t* out;
  int64_t row_size;                /* row-wise bytes per row */
  int64_t cap;                     /* rows the buffer holds: columnar column stride, and the write limit */
  int32_t columnar;
  int32_t pad_;
  unsigned long long* status;      /* [all chunks of all launches] zero-initialised */
  unsigned long long* ticket;      /* this launch's chunk counter, zero-initialised */
  unsigned long long* counters;    /* [0] done flag, [1] rows written, [2] rows of the chunks loaded */
  int32_t* error;                  /* B2Q_ERR_INTERRUPTED / OUT_OF_TIME when the launch was stopped */
  DevInterrupt intr;
};

__device__ __forceinline__ void st_release(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ void store_w(int8_t* dst, int w, int64_t v) {
  switch (w) {
    case 1: *dst = (int8_t)v; break;
    case 2: *reinterpret_cast<int16_t*>(dst) = (int16_t)v; break;
    case 4: *reinterpret_cast<int32_t*>(dst) = (int32_t)v; break;
    default: *reinterpret_cast<int64_t*>(dst) = v;
  }
}

/* one chunk whose pass bits are known: stage each column compacted in shared memory, then write the run [excl, excl + n) */
template <bool FULL>
__device__ __forceinline__ uint32_t chunk_pass(const ProjArgs& A, const int8_t* const* cols, int64_t row0, int64_t frag_rows, uint64_t pol) {
  uint32_t valid = (1u << R) - 1u;
  if (!FULL) {
    valid = 0;
#pragma unroll
    for (int j = 0; j < R; ++j) valid |= (uint32_t)(row0 + (int64_t)j * kProjBlock < frag_rows) << j;
  }
  return eval_filter<FULL, 0>(A.filter, cols, row0, kProjBlock, valid, pol, nullptr, nullptr, -1, nullptr, nullptr);
}

__global__ void __launch_bounds__(kProjBlock) b2q_k_project(const __grid_constant__ ProjArgs A) {
  __shared__ int64_t s_stage[kProjChunk];
  __shared__ uint32_t s_off[R * kProjWarps]; /* per (row slot j, warp): count, then exclusive offset inside the chunk */
  __shared__ unsigned long long s_chunk;
  __shared__ long long s_excl, s_total;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  const int64_t limit = A.proj.scan_limit > 0 ? (A.proj.scan_limit < A.cap ? A.proj.scan_limit : A.cap) : A.cap;
  unsigned long long* done = A.counters;

  /* Interrupt / watchdog: the stop takes the scan limit's path.  Thread 0 polls before it claims a chunk; a stop records its
   * code and raises the done flag, and from then on every CTA claims nothing more.  Why no CTA can then wait forever in the
   * look-back below: a CTA only looks back over chunks with smaller tickets, i.e. chunks some CTA has already claimed, and
   * every claimed chunk publishes a status word with a flag its successors accept as final — a chunk claimed before the
   * done flag is processed to the end (its own look-back only waits on earlier claims, by induction), a chunk claimed after
   * it publishes an empty aggregate (kFlagAgg | 0) at once.  Chunks never claimed have no successor that waits on them. */
  const bool check = interrupt_enabled(A.intr);
  PollState poll = {0, 0};
  int frag = 0;
  int64_t frag_first = 0, next_first = __ldg(A.frag_chunk_start + 1);
  for (;;) {
    if (tid == 0) {
      unsigned long long c = ~0ull;
      if (check) {
        const int32_t code = interrupt_poll(A.intr, A.error, poll);
        if (code) { atomicCAS(A.error, 0, code); st_release(done, 1ull); }
      }
      if (!ld_acquire(done)) {
        c = atomicAdd(A.ticket, 1ull);
        if (c >= (unsigned long long)A.total_chunks) c = ~0ull;
        else if (ld_acquire(done)) { /* claimed after the limit was reached: publish an empty aggregate for the chunks behind */
          st_release(A.status + A.chunk_base + c, kFlagAgg);
          c = ~0ull;
        }
      }
      s_chunk = c;
    }
    __syncthreads();
    const unsigned long long chunk_u = s_chunk;
    if (chunk_u == ~0ull) break;
    const int64_t chunk = (int64_t)chunk_u;
    while (chunk >= next_first) { /* a CTA's tickets increase: the owning fragment is a moving cursor */
      ++frag;
      frag_first = next_first;
      next_first = __ldg(A.frag_chunk_start + frag + 1);
    }
    const int64_t frag_rows = __ldg(A.frag_rows + frag);
    const int64_t base_row = (chunk - frag_first) * kProjChunk;
    const int8_t* const* cols = A.col_ptrs + (size_t)frag * A.n_cols;
    const int64_t row0 = base_row + tid;
    const bool full = base_row + kProjChunk <= frag_rows;
    const uint32_t pass = full ? chunk_pass<true>(A, cols, row0, frag_rows, pol) : chunk_pass<false>(A, cols, row0, frag_rows, pol);

    /* ranks: row (j, tid) is at s_off[j][warp] + popc(ballot_j below this lane) inside the chunk */
    uint32_t rank[R];
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const uint32_t b = __ballot_sync(~0u, pass >> j & 1);
      rank[j] = __popc(b & ((1u << lane) - 1u));
      if (lane == 0) s_off[j * kProjWarps + warp] = __popc(b);
    }
    __syncthreads();
    if (warp == 0) {
      static_assert(R * kProjWarps == 64, "two counts per lane");
      const uint32_t v0 = s_off[2 * lane], v1 = s_off[2 * lane + 1];
      uint32_t incl = v0 + v1;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(~0u, incl, o);
        if (lane >= o) incl += y;
      }
      const uint32_t ex = incl - v0 - v1;
      s_off[2 * lane] = ex;
      s_off[2 * lane + 1] = ex + v0;
      const uint32_t total = __shfl_sync(~0u, incl, 31);
      if (lane == 0) {
        unsigned long long* my = A.status + A.chunk_base + chunk;
        const int64_t gidx = A.chunk_base + chunk;
        int64_t excl = 0;
        if (gidx == 0) st_release(my, kFlagInc | total);
        else {
          st_release(my, kFlagAgg | total);
          for (int64_t i = gidx - 1;; --i) { /* decoupled look-back */
            unsigned long long s;
            do { s = ld_acquire(A.status + i); } while (!(s >> 62));
            excl += (int64_t)(s & kCountMask);
            if ((s >> 62) == 2 || i == 0) break;
          }
          st_release(my, kFlagInc | (unsigned long long)(excl + total));
        }
        const int64_t incl_rows = excl + total;
        if (incl_rows >= limit) st_release(done, 1ull);
        atomicMax(A.counters + 1, (unsigned long long)(incl_rows < limit ? incl_rows : limit));
        const int64_t rows_here = frag_rows - base_row < kProjChunk ? frag_rows - base_row : kProjChunk;
        atomicAdd(A.counters + 2, (unsigned long long)rows_here);
        s_excl = excl;
        s_total = total;
      }
    }
    __syncthreads();
    const int64_t excl = s_excl;
    const int64_t keep = limit - excl; /* rows of this chunk that still fit */
    if (keep > 0) {
      const int64_t n = s_total < keep ? s_total : keep;
      uint32_t wmask = 0;
      int pos[R];
#pragma unroll
      for (int j = 0; j < R; ++j) {
        pos[j] = (int)s_off[j * kProjWarps + warp] + (int)rank[j];
        wmask |= (uint32_t)((pass >> j & 1) && pos[j] < keep) << j;
      }
      const int64_t frag_base = A.frag_row_base ? __ldg(A.frag_row_base + frag) : 0;
      /* column -1: the offset word (the row's index inside its fragment), then every projected column */
      for (int k = -1; k < A.proj.n; ++k) {
        int64_t v[R];
        int w;
        int64_t off;
        if (k < 0) {
#pragma unroll
          for (int j = 0; j < R; ++j) v[j] = frag_base + row0 + (int64_t)j * kProjBlock;
          w = 8;
          off = 0;
        } else {
          const DevProjCol& pc = A.proj.cols[k];
          w = pc.out_w;
          off = pc.out_off;
          if (pc.width == 8) {
            load64<true>(v, cols[pc.col], row0, kProjBlock, wmask, pol);
          } else {
            int32_t x[R];
            load32<true>(x, cols[pc.col], pc.width, row0, kProjBlock, wmask, pol);
#pragma unroll
            for (int j = 0; j < R; ++j) {
              int64_t y = pc.kind == PROJ_F32 ? (int64_t)(uint32_t)x[j] : (int64_t)x[j]; /* a FLOAT slot: the float's 4 bytes, upper word 0 */
              if (pc.translate_null && y == pc.null_phys) y = pc.null_logical;
              else if (pc.days) y *= 86400;
              v[j] = y;
            }
          }
        }
#pragma unroll
        for (int j = 0; j < R; ++j)
          if (wmask >> j & 1) s_stage[pos[j]] = v[j];
        __syncthreads();
        if (A.columnar) {
          int8_t* dst = A.out + off + excl * w;
          for (int64_t i = tid; i < n; i += kProjBlock) store_w(dst + i * w, w, s_stage[i]);
        } else {
          int8_t* dst = A.out + excl * A.row_size + off;
          for (int64_t i = tid; i < n; i += kProjBlock) *reinterpret_cast<int64_t*>(dst + i * A.row_size) = s_stage[i];
        }
        __syncthreads();
      }
    }
  }
}

/* the launch geometry of b2q_k_project: persistent CTAs, as many as are resident at once */
int project_rows_per_chunk() { return static_cast<int>(kProjChunk); }

cudaError_t launch_project(const B2QQuery& q, const int8_t* const* col_ptrs, const int64_t* frag_rows, const int64_t* frag_chunk_start,
                           const int64_t* frag_row_base, int n_frags, int64_t total_chunks, int64_t chunk_base, int8_t* out,
                           int64_t row_size, int64_t cap, unsigned long long* status, unsigned long long* ticket,
                           unsigned long long* counters, int32_t* error, const DevInterrupt& intr, cudaStream_t st) {
  ProjArgs a;
  memset(&a, 0, sizeof(a));
  a.error = error;
  a.intr = intr;
  a.filter = q.prog.filter;
  a.proj = q.proj;
  a.col_ptrs = col_ptrs;
  a.frag_rows = frag_rows;
  a.frag_chunk_start = frag_chunk_start;
  a.frag_row_base = frag_row_base;
  a.n_frags = n_frags;
  a.n_cols = q.prog.n_cols;
  a.total_chunks = total_chunks;
  a.chunk_base = chunk_base;
  a.out = out;
  a.row_size = row_size;
  a.cap = cap;
  a.columnar = q.plan.output_columnar;
  a.status = status;
  a.ticket = ticket;
  a.counters = counters;
  int dev = 0, sms = 132, per_sm = 1;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, b2q_k_project, kProjBlock, 0);
  int64_t grid = static_cast<int64_t>(sms) * (per_sm > 0 ? per_sm : 1);
  if (grid > total_chunks) grid = total_chunks;
  if (grid < 1) grid = 1;
  b2q_k_project<<<static_cast<int>(grid), kProjBlock, 0, st>>>(a);
  return cudaGetLastError();
}

}  // namespace b2q
