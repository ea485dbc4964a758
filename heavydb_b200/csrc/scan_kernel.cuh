/*
 * scan_kernel.cuh — the scan -> filter -> group-by/aggregate kernel (b2q_k_scan) as a template; instantiated per
 * (table mode, join level) in scan_inst.cu, which is compiled once per (join, group) so that the 42 instantiations
 * build in parallel.
 *
 * They replace what the reference JIT-compiles per query:
 *   row loop            query_group_by_template / query_template + multifrag_query_hoisted_literals
 *                       (QueryEngine/QueryTemplateGenerator.cpp:552-815,257-549; RuntimeFunctions.cpp:2434-2472)
 *   column decode       fixed_width_int_decode / fixed_width_double_decode (QueryEngine/DecodersImpl.h:30-61,112-136)
 *   filter              DEF_CMP_NULLABLE + toBool (RuntimeFunctions.cpp:73-107, LogicalIR.cpp:344-352)
 *   group lookup        get_group_value_fast[_keyless] (GroupByRuntime.cpp:194-209, RuntimeFunctions.cpp:2126-2152),
 *                       get_group_value + get_matching_group_value (GroupByRuntime.cpp:20-48, cuda_mapd_rt.cu:180-216)
 *   aggregate update    agg_*_shared / agg_*_skip_val_shared (cuda_mapd_rt.cu:437-1198)
 *   smem table          init_shared_mem + JIT'd reduce_from_smem_to_gmem (cuda_mapd_rt.cu:73-87,
 *                       GpuSharedMemoryUtils.cpp:96-383)
 *   buffer init         init_group_by_buffer_gpu (GpuInitGroups.cu:124-171)
 *
 * Design (DESIGN.md has the numbers):
 *   - persistent CTAs, grid = #SMs x CTAs/SM, static chunk striding over all fragments of the launch;
 *   - each thread owns R rows per chunk, lane-consecutive => every column load is a fully coalesced
 *     ld.global.nc.L1::no_allocate of the column's own width; R independent loads per column are in flight;
 *   - vector-at-a-time interpretation of the device program: all operator/width switches are warp-uniform and
 *     executed once per R rows;
 *   - group table private to the CTA in shared memory (TMA bulk copy of an identity image initialises it),
 *     warp-private replicas for small tables; 32-bit native shared atomics only: a 64-bit integer SUM keeps its low
 *     word in shared memory and sends the (rare) carries straight to the HBM table, because sm_90a has no native
 *     64-bit shared-memory atomic add (ATOMS.CAST.SPIN loops otherwise);
 *   - warp-aggregated update (shuffle reduction, one atomic per warp) for the non-grouped case;
 *   - tables too large for shared memory go to one dense table in HBM/L2 with RED.E.ADD/MIN/MAX;
 *   - sparse keys: open addressing in HBM, MurmurHash3 (same function and home slot as the reference), 64-bit CAS.
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

#include "b2q_internal.h"

namespace b2q {


constexpr int R = 8;                 /* rows per thread per chunk */
constexpr int kMaxBlock = 1024;

enum { MODE_SMEM = 0, MODE_GLOBAL = 1, MODE_BASELINE = 2 };

/* ---------------------------------------------------------------------------------------------------------
 * loads: streaming (read-only path, no L1 allocation), branch-free predication.
 * The asm is deliberately NOT volatile: the data is immutable for the kernel, so the compiler may hoist and batch
 * the loads of a vector, which is what puts R independent requests per column in flight.
 * ------------------------------------------------------------------------------------------------------- */
template <bool PRED>
__device__ __forceinline__ int64_t ldg_b64(const int8_t* p, uint32_t pred, uint64_t pol) {
  int64_t v;
  if (PRED)
    asm("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\tmov.b64 %0, 0;\n\t@p ld.global.nc.L1::no_allocate.L2::cache_hint.b64 %0, [%1], %3;\n\t}" : "=l"(v) : "l"(p), "r"(pred), "l"(pol));
  else
    asm("ld.global.nc.L1::no_allocate.L2::cache_hint.b64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol));
  return v;
}
template <bool PRED>
__device__ __forceinline__ int32_t ldg_s32(const int8_t* p, uint32_t pred, uint64_t pol) {
  int32_t v;
  if (PRED)
    asm("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\tmov.b32 %0, 0;\n\t@p ld.global.nc.L1::no_allocate.L2::cache_hint.s32 %0, [%1], %3;\n\t}" : "=r"(v) : "l"(p), "r"(pred), "l"(pol));
  else
    asm("ld.global.nc.L1::no_allocate.L2::cache_hint.s32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return v;
}
template <bool PRED>
__device__ __forceinline__ int32_t ldg_s16(const int8_t* p, uint32_t pred, uint64_t pol) {
  int32_t v;
  if (PRED)
    asm("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\tmov.b32 %0, 0;\n\t@p ld.global.nc.L1::no_allocate.L2::cache_hint.s16 %0, [%1], %3;\n\t}" : "=r"(v) : "l"(p), "r"(pred), "l"(pol));
  else
    asm("ld.global.nc.L1::no_allocate.L2::cache_hint.s16 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return (int32_t)(int16_t)v;
}
template <bool PRED>
__device__ __forceinline__ int32_t ldg_s8(const int8_t* p, uint32_t pred, uint64_t pol) {
  int32_t v;
  if (PRED)
    asm("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\tmov.b32 %0, 0;\n\t@p ld.global.nc.L1::no_allocate.L2::cache_hint.s8 %0, [%1], %3;\n\t}" : "=r"(v) : "l"(p), "r"(pred), "l"(pol));
  else
    asm("ld.global.nc.L1::no_allocate.L2::cache_hint.s8 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return (int32_t)(int8_t)v;
}

/* zero-extending variants: dictionary ids stored on 1 / 2 bytes are unsigned (FixedWidthUnsigned, ColumnIR.cpp:59-67) */
template <bool PRED>
__device__ __forceinline__ int32_t ldg_u16(const int8_t* p, uint32_t pred, uint64_t pol) {
  uint32_t v;
  if (PRED)
    asm("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\tmov.b32 %0, 0;\n\t@p ld.global.nc.L1::no_allocate.L2::cache_hint.u16 %0, [%1], %3;\n\t}" : "=r"(v) : "l"(p), "r"(pred), "l"(pol));
  else
    asm("ld.global.nc.L1::no_allocate.L2::cache_hint.u16 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return (int32_t)(v & 0xFFFFu);
}
template <bool PRED>
__device__ __forceinline__ int32_t ldg_u8(const int8_t* p, uint32_t pred, uint64_t pol) {
  uint32_t v;
  if (PRED)
    asm("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\tmov.b32 %0, 0;\n\t@p ld.global.nc.L1::no_allocate.L2::cache_hint.u8 %0, [%1], %3;\n\t}" : "=r"(v) : "l"(p), "r"(pred), "l"(pol));
  else
    asm("ld.global.nc.L1::no_allocate.L2::cache_hint.u8 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return (int32_t)(v & 0xFFu);
}

/* R rows of an 8-byte column: rows row0 + j*stride */
/* jidx != nullptr: the column belongs to the joined inner table and is read at the matching inner rows (a gather
 * through the normal cached path: dimension tables are small and re-read constantly).  Call sites pass a
 * compile-time nullptr in the kernels without a join level, so the branch disappears there. */
template <bool PRED>
__device__ __forceinline__ void load64(int64_t (&v)[R], const int8_t* __restrict__ base, int64_t row0, int stride, uint32_t mask, uint64_t pol,
                                       const int32_t* jidx = nullptr, const int32_t* /* jval: only 1/2/4-byte columns are packed */ = nullptr,
                                       const int64_t* nullp = nullptr) {
  if (jidx) { /* nullp (LEFT join kernels only): an unmatched row (idx < 0) reads NULL (codegenOuterJoinNullPlaceholder) */
#pragma unroll
    for (int j = 0; j < R; ++j) v[j] = (mask >> j & 1) ? ((nullp && jidx[j] < 0) ? *nullp : __ldg(reinterpret_cast<const long long*>(base) + jidx[j])) : 0;
    return;
  }
  const int8_t* p = base + row0 * 8;
  const int64_t step = (int64_t)stride * 8;
#pragma unroll
  for (int j = 0; j < R; ++j) v[j] = ldg_b64<PRED>(p + j * step, mask >> j & 1, pol);
}
/* R rows of a 1/2/4-byte integer column, sign-extended to 32 bits (width -1 / -2: zero-extended) */
template <bool PRED>
__device__ __forceinline__ void load32(int32_t (&v)[R], const int8_t* __restrict__ base, int width, int64_t row0, int stride, uint32_t mask, uint64_t pol,
                                       const int32_t* jidx = nullptr, const int32_t* jval = nullptr, const int64_t* nullp = nullptr) {
  if (jval) { /* the column that rides in the packed join table: already in registers since the probe */
#pragma unroll
    for (int j = 0; j < R; ++j) v[j] = (mask >> j & 1) ? jval[j] : 0;
    return;
  }
  if (jidx) {
#pragma unroll
    for (int j = 0; j < R; ++j) {
      int32_t x = 0;
      if (nullp && (mask >> j & 1) && jidx[j] < 0) x = (int32_t)*nullp;
      else if (mask >> j & 1) {
        const int64_t i = jidx[j];
        switch (width) {
          case 4: x = __ldg(reinterpret_cast<const int32_t*>(base) + i); break;
          case 2: x = __ldg(reinterpret_cast<const int16_t*>(base) + i); break;
          case -2: x = __ldg(reinterpret_cast<const uint16_t*>(base) + i); break;
          case -1: x = __ldg(reinterpret_cast<const uint8_t*>(base) + i); break;
          default: x = __ldg(reinterpret_cast<const signed char*>(base) + i); break;
        }
      }
      v[j] = x;
    }
    return;
  }
  if (width == 4) {
    const int8_t* p = base + row0 * 4;
    const int64_t step = (int64_t)stride * 4;
#pragma unroll
    for (int j = 0; j < R; ++j) v[j] = ldg_s32<PRED>(p + j * step, mask >> j & 1, pol);
  } else if (width == 2) {
    const int8_t* p = base + row0 * 2;
    const int64_t step = (int64_t)stride * 2;
#pragma unroll
    for (int j = 0; j < R; ++j) v[j] = ldg_s16<PRED>(p + j * step, mask >> j & 1, pol);
  } else if (width == -2) {
    const int8_t* p = base + row0 * 2;
    const int64_t step = (int64_t)stride * 2;
#pragma unroll
    for (int j = 0; j < R; ++j) v[j] = ldg_u16<PRED>(p + j * step, mask >> j & 1, pol);
  } else if (width == -1) {
    const int8_t* p = base + row0;
    const int64_t step = (int64_t)stride;
#pragma unroll
    for (int j = 0; j < R; ++j) v[j] = ldg_u8<PRED>(p + j * step, mask >> j & 1, pol);
  } else {
    const int8_t* p = base + row0;
    const int64_t step = (int64_t)stride;
#pragma unroll
    for (int j = 0; j < R; ++j) v[j] = ldg_s8<PRED>(p + j * step, mask >> j & 1, pol);
  }
}

/* ---------------------------------------------------------------------------------------------------------
 * filter: one comparison = one unsigned range test, (v - lo) <= span, in the column's register class
 * ------------------------------------------------------------------------------------------------------- */
template <bool FULL>
__device__ __forceinline__ uint32_t eval_term(const DevTerm& t, const int8_t* const* __restrict__ cols, int64_t row0,
                                              int stride, uint32_t valid, uint64_t pol, const int32_t* jidx = nullptr,
                                              const int32_t* jval = nullptr, const int64_t* jnull = nullptr) {
  uint32_t m = 0;
  const bool neg = t.negate;
  if (!t.cmp_fp) {
    if (t.width == 8) {
      int64_t v[R];
      load64<!FULL>(v, cols[t.col], row0, stride, valid, pol, jidx, nullptr, jnull);
      const uint64_t lo = (uint64_t)t.lo, span = t.span;
      if (lo == 0x8000000000000000ull) { /* only an upper bound (`<`, `<=`): one signed compare instead of subtract + compare */
        const int64_t hi = (int64_t)(lo + span);
#pragma unroll
        for (int j = 0; j < R; ++j) m |= (uint32_t)((v[j] <= hi) != neg) << j;
      } else {
#pragma unroll
        for (int j = 0; j < R; ++j) m |= (uint32_t)(((uint64_t)v[j] - lo <= span) != neg) << j;
      }
      if (t.null_check) {
        const int64_t nullv = t.null_bits;
#pragma unroll
        for (int j = 0; j < R; ++j) m &= ~((uint32_t)(v[j] == nullv) << j);
      }
    } else {
      int32_t v[R];
      load32<!FULL>(v, cols[t.col], t.width, row0, stride, valid, pol, jidx, jval, jnull);
      const uint32_t lo = (uint32_t)t.lo, span = (uint32_t)t.span;
#pragma unroll
      for (int j = 0; j < R; ++j) m |= (uint32_t)(((uint32_t)v[j] - lo <= span) != neg) << j;
      if (t.null_check) {
        const int32_t nullv = (int32_t)t.null_bits;
#pragma unroll
        for (int j = 0; j < R; ++j) m &= ~((uint32_t)(v[j] == nullv) << j);
      }
    }
  } else {
    const double lo = t.flo, hi = t.fhi;
    double d[R];
    uint32_t isnull = 0;
    if (t.col_is_fp && t.width == 4) { /* FLOAT chunk (fixed_width_float_decode, DecodersImpl.h:112-123): widened exactly */
      int32_t v[R];
      load32<!FULL>(v, cols[t.col], 4, row0, stride, valid, pol, jidx, jval, jnull);
      const double nullv = __longlong_as_double(t.null_bits);
#pragma unroll
      for (int j = 0; j < R; ++j) { d[j] = (double)__int_as_float(v[j]); isnull |= (uint32_t)(d[j] == nullv) << j; }
    } else if (t.col_is_fp) {
      int64_t v[R];
      load64<!FULL>(v, cols[t.col], row0, stride, valid, pol, jidx, nullptr, jnull);
      const double nullv = __longlong_as_double(t.null_bits);
#pragma unroll
      for (int j = 0; j < R; ++j) { d[j] = __longlong_as_double(v[j]); isnull |= (uint32_t)(d[j] == nullv) << j; }
    } else if (t.width == 8) {
      int64_t v[R];
      load64<!FULL>(v, cols[t.col], row0, stride, valid, pol, jidx, nullptr, jnull);
      const int64_t nullv = t.null_bits;
#pragma unroll
      for (int j = 0; j < R; ++j) { d[j] = (double)v[j]; isnull |= (uint32_t)(v[j] == nullv) << j; }
    } else {
      int32_t v[R];
      load32<!FULL>(v, cols[t.col], t.width, row0, stride, valid, pol, jidx, jval, jnull);
      const int32_t nullv = (int32_t)t.null_bits;
#pragma unroll
      for (int j = 0; j < R; ++j) { d[j] = (double)v[j]; isnull |= (uint32_t)(v[j] == nullv) << j; }
    }
#pragma unroll
    for (int j = 0; j < R; ++j) m |= (uint32_t)(((d[j] >= lo) & (d[j] <= hi)) != neg) << j;
    if (t.null_check) m &= ~isnull;
  }
  return m & valid;
}

/* column OP column */
template <bool FULL>
__device__ __forceinline__ uint32_t eval_term2(const DevTerm& t, const int8_t* const* __restrict__ cols, int64_t row0, int stride,
                                               uint32_t valid, uint64_t pol, const int32_t* jidx1, const int32_t* jval1,
                                               const int64_t* jnull1, const int32_t* jidx2, const int32_t* jval2, const int64_t* jnull2) {
  int64_t a[R], b[R];
  if (t.width == 8) load64<!FULL>(a, cols[t.col], row0, stride, valid, pol, jidx1, jval1, jnull1);
  else {
    int32_t x[R];
    load32<!FULL>(x, cols[t.col], t.width, row0, stride, valid, pol, jidx1, jval1, jnull1);
#pragma unroll
    for (int j = 0; j < R; ++j) a[j] = t.col_is_fp ? __double_as_longlong((double)__int_as_float(x[j])) : (int64_t)x[j];
  }
  if (t.width2 == 8) load64<!FULL>(b, cols[t.col2], row0, stride, valid, pol, jidx2, jval2, jnull2);
  else {
    int32_t x[R];
    load32<!FULL>(x, cols[t.col2], t.width2, row0, stride, valid, pol, jidx2, jval2, jnull2);
#pragma unroll
    for (int j = 0; j < R; ++j) b[j] = t.col2_is_fp ? __double_as_longlong((double)__int_as_float(x[j])) : (int64_t)x[j];
  }
  uint32_t isnull = 0, m = 0;
  const int op = t.op2;
  if (t.cmp_fp) {
    const double n1 = __longlong_as_double(t.null_bits), n2 = __longlong_as_double(t.null_bits2);
#pragma unroll
    for (int j = 0; j < R; ++j) {
      double x, y;
      if (t.col_is_fp) { x = __longlong_as_double(a[j]); isnull |= (uint32_t)(t.nullable1 && x == n1) << j; }
      else { x = (double)a[j]; isnull |= (uint32_t)(t.nullable1 && a[j] == t.null_bits) << j; }
      if (t.col2_is_fp) { y = __longlong_as_double(b[j]); isnull |= (uint32_t)(t.nullable2 && y == n2) << j; }
      else { y = (double)b[j]; isnull |= (uint32_t)(t.nullable2 && b[j] == t.null_bits2) << j; }
      const bool r = op == B2Q_kEQ ? x == y : op == B2Q_kNE ? x != y : op == B2Q_kLT ? x < y : op == B2Q_kGT ? x > y : op == B2Q_kLE ? x <= y : x >= y;
      m |= (uint32_t)r << j;
    }
  } else {
#pragma unroll
    for (int j = 0; j < R; ++j) {
      isnull |= (uint32_t)((t.nullable1 && a[j] == t.null_bits) || (t.nullable2 && b[j] == t.null_bits2)) << j;
      const bool r = op == B2Q_kEQ ? a[j] == b[j] : op == B2Q_kNE ? a[j] != b[j] : op == B2Q_kLT ? a[j] < b[j] : op == B2Q_kGT ? a[j] > b[j] : op == B2Q_kLE ? a[j] <= b[j] : a[j] >= b[j];
      m |= (uint32_t)r << j;
    }
  }
  return m & ~isnull & valid;
}

template <bool FULL, int JOIN>
__device__ __forceinline__ uint32_t eval_filter(const DevFilter& f, const int8_t* const* __restrict__ cols,
                                                int64_t row0, int stride, uint32_t valid, uint64_t pol,
                                                const int8_t* __restrict__ col_inner, const int32_t* jidx, int packed_col,
                                                const int32_t* jval, const int64_t* __restrict__ col_null) {
#define B2Q_TERM_JX(t) ((JOIN && col_inner[(t).col]) ? jidx : nullptr), ((JOIN && (t).col == packed_col) ? jval : nullptr), (JOIN == 2 ? col_null + (t).col : nullptr)
#define B2Q_TERM_JX2(t) ((JOIN && col_inner[(t).col2]) ? jidx : nullptr), ((JOIN && (t).col2 == packed_col) ? jval : nullptr), (JOIN == 2 ? col_null + (t).col2 : nullptr)
#define B2Q_EVAL_TERM(t) ((t).col2 >= 0 ? eval_term2<FULL>((t), cols, row0, stride, valid, pol, B2Q_TERM_JX(t), B2Q_TERM_JX2(t)) \
                                       : eval_term<FULL>((t), cols, row0, stride, valid, pol, B2Q_TERM_JX(t)))
  if (f.n_ops == 0) return valid;
  if (f.n_ops == 1) return B2Q_EVAL_TERM(f.terms[0]);
  uint32_t s0 = 0, s1 = 0, s2 = 0, s3 = 0;
  for (int i = 0; i < f.n_ops; ++i) {
    const uint32_t op = f.ops[i];
    const uint32_t kind = op >> 4;
    if (kind == FOP_TERM) {
      const uint32_t m = B2Q_EVAL_TERM(f.terms[op & 15]);
      s3 = s2; s2 = s1; s1 = s0; s0 = m;
    } else {
      s0 = (kind == FOP_AND) ? (s1 & s0) : (s1 | s0);
      s1 = s2; s2 = s3; s3 = 0;
    }
  }
  return s0 & valid;
#undef B2Q_EVAL_TERM
#undef B2Q_TERM_JX2
#undef B2Q_TERM_JX
}

/* ---------------------------------------------------------------------------------------------------------
 * skip test (NULL handling of aggregate arguments), see DevAcc
 * ------------------------------------------------------------------------------------------------------- */
__device__ __forceinline__ uint32_t not_skipped64(const DevAcc& a, const int64_t (&v)[R], uint32_t pass) {
  if (!a.skip1_en && !a.skip2_en) return pass;
  uint32_t m = 0;
  if (a.is_fp) {
    const double s = __longlong_as_double(a.skip1_val);
#pragma unroll
    for (int j = 0; j < R; ++j) m |= (uint32_t)(__longlong_as_double(v[j]) != s) << j;
  } else {
    const int64_t s1 = a.skip1_val, s2 = a.skip2_val;
    const bool e1 = a.skip1_en, e2 = a.skip2_en, tr = a.skip2_trunc32;
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const int64_t w = tr ? (int64_t)(int32_t)v[j] : v[j];
      const bool skip = (e1 & (v[j] == s1)) | (e2 & (w == s2));
      m |= (uint32_t)(!skip) << j;
    }
  }
  return m & pass;
}
__device__ __forceinline__ uint32_t not_skipped32(const DevAcc& a, const int32_t (&v)[R], uint32_t pass) {
  if (!a.skip1_en && !a.skip2_en) return pass;
  /* a sign-extended 32-bit value can only equal a skip value that itself fits in 32 bits */
  const bool e1 = a.skip1_en && a.skip1_val == (int64_t)(int32_t)a.skip1_val;
  const bool e2 = a.skip2_en && a.skip2_val == (int64_t)(int32_t)a.skip2_val;
  const int32_t s1 = (int32_t)a.skip1_val, s2 = (int32_t)a.skip2_val;
  uint32_t m = 0;
#pragma unroll
  for (int j = 0; j < R; ++j) {
    const bool skip = (e1 & (v[j] == s1)) | (e2 & (v[j] == s2));
    m |= (uint32_t)(!skip) << j;
  }
  return m & pass;
}

/* ---------------------------------------------------------------------------------------------------------
 * MurmurHash3 x86_32 for one 4- or 8-byte key, seed 0 (QueryEngine/MurmurHash3Inl.h:11-72)
 * ------------------------------------------------------------------------------------------------------- */
__device__ __forceinline__ uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
__device__ __forceinline__ uint32_t murmur_block(uint32_t h1, uint32_t k1) {
  k1 *= 0xcc9e2d51u; k1 = rotl32(k1, 15); k1 *= 0x1b873593u;
  h1 ^= k1; h1 = rotl32(h1, 13); h1 = h1 * 5 + 0xe6546b64u;
  return h1;
}
__device__ __forceinline__ uint32_t murmur3_key(int64_t key, int width) {
  uint32_t h1 = 0;
  h1 = murmur_block(h1, (uint32_t)key);
  if (width == 8) h1 = murmur_block(h1, (uint32_t)((uint64_t)key >> 32));
  h1 ^= (uint32_t)width;
  h1 ^= h1 >> 16; h1 *= 0x85ebca6bu; h1 ^= h1 >> 13; h1 *= 0xc2b2ae35u; h1 ^= h1 >> 16;
  return h1;
}

/* MurmurHash3_x86_32 finalisation for a key of `len` bytes whose 4-byte blocks were folded with murmur_block */
__device__ __forceinline__ uint32_t murmur3_fmix(uint32_t h1, uint32_t len) {
  h1 ^= len;
  h1 ^= h1 >> 16; h1 *= 0x85ebca6bu; h1 ^= h1 >> 13; h1 *= 0xc2b2ae35u; h1 ^= h1 >> 16;
  return h1;
}

/* ---------------------------------------------------------------------------------------------------------
 * global (HBM / L2) reductions without return value
 * ------------------------------------------------------------------------------------------------------- */
__device__ __forceinline__ void red_add_u64(int64_t* p, uint64_t v) { asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void red_add_f64(int64_t* p, double v) { asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory"); }
__device__ __forceinline__ void red_min_s64(int64_t* p, int64_t v) { asm volatile("red.global.min.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void red_max_s64(int64_t* p, int64_t v) { asm volatile("red.global.max.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }

/* HBM/L2-resident table (MODE_GLOBAL / MODE_BASELINE).  COUNT and integer SUM keep a SPLIT accumulator: the array's
 * first 4n bytes are the low words, the next 4n bytes the high words.  Only the low words are hot (native 32-bit
 * L2 atomics); the high word sees the rare carry / a value wider than 32 bits.  That halves the randomly accessed
 * footprint — 40 MB instead of 80 MB for 1e7 groups — which is what lets the table stay L2-resident while 16 GB of
 * column data streams through the same L2 (with 64-bit REDs on the 80 MB table, the table thrashes L2 and DRAM traffic
 * is a multiple of the algorithmic bytes).  Table accesses carry an evict_last L2 policy, the column stream evict_first. */
__device__ __forceinline__ uint32_t global_split_add(int64_t* arr, uint32_t e, int64_t n, uint32_t vl, int32_t vh, uint64_t pol_tab) {
  uint32_t* lo = reinterpret_cast<uint32_t*>(arr) + e;
  uint32_t old;
  asm volatile("atom.global.add.L2::cache_hint.u32 %0, [%1], %2, %3;" : "=r"(old) : "l"(lo), "r"(vl), "l"(pol_tab) : "memory");
  const int32_t hi = vh + (int32_t)((uint32_t)(old + vl) < old);
  if (hi != 0) atomicAdd(reinterpret_cast<int32_t*>(arr) + n + e, hi);
  return old;
}
/* "group touched" flag piggy-backed on an accumulator that every passing row updates: the FIRST atomic on an entry
 * always returns the initial 0, so storing the flag whenever 0 comes back marks every touched group and costs no
 * extra L2 request for the (overwhelmingly common) rows that see a non-zero running value. */
/* n < 0: the array is a plain int64[] (the table is small enough to stay L2-resident as 8-byte words): one RED.ADD.64 without a
 * return trip, cheaper than the returning 32-bit atomic on the split layout (tools/atom_bench.cu) — as long as no flag byte
 * is read per row, which would give that back. */
__device__ __forceinline__ void global_split_add_touch(int64_t* arr, uint8_t* flags, uint32_t e, int64_t n, uint32_t vl, int32_t vh, uint64_t pol_tab) {
  if (n < 0) {
    const uint64_t v = ((uint64_t)(uint32_t)vh << 32) + vl;
    /* evict_last on the table is what keeps its 8-byte words L2-resident next to the evict_first column stream: without the hint
     * the same kernel writes the table's sectors back to DRAM over and over */
    asm volatile("red.global.add.L2::cache_hint.u64 [%0], %1, %2;" ::"l"(arr + e), "l"(v), "l"(pol_tab) : "memory");
    /* touched = flag OR accumulator != 0 (b2q_k_materialize): a value in [1, 2^31) cannot leave the sum at zero while the launch
     * set holds fewer than 2^32 rows (the executor checks), so only the other rows keep the flag — for a COUNT, none */
    if (flags && v - 1 >= 0x7FFFFFFFull) {
      uint32_t w;
      asm volatile("ld.global.ca.u8 %0, [%1];" : "=r"(w) : "l"(flags + e));
      if (!w) flags[e] = 1;
    }
    return;
  }
  const uint32_t old = global_split_add(arr, e, n, vl, vh, pol_tab);
  if (flags && old == 0) flags[e] = 1;
}

__device__ __forceinline__ void global_update(int op, int64_t* arr, uint8_t* flags, uint32_t e, int64_t n, int64_t v, uint64_t pol_tab) {
  switch (op) {
    case ACC_COUNT: global_split_add_touch(arr, flags, e, n, 1u, 0, pol_tab); break;
    case ACC_SUM_I64: global_split_add_touch(arr, flags, e, n, (uint32_t)v, (int32_t)(v >> 32), pol_tab); break;
    case ACC_SUM_F64: red_add_f64(arr + e, __longlong_as_double(v)); break;
    case ACC_MIN_I64: red_min_s64(arr + e, v); break;
    case ACC_MAX_I64: red_max_s64(arr + e, v); break;
    case ACC_MIN_F64: red_min_s64(arr + e, b2q_f64_min_ord(v)); break;
    default: red_max_s64(arr + e, b2q_f64_max_ord(v)); break;
  }
}

/* ---------------------------------------------------------------------------------------------------------
 * shared-memory table updates.  `tab` points at the accumulator's array inside this warp's replica.
 * 64-bit integer SUM: (hi:lo) += v with lo in shared memory (native 32-bit ATOMS.ADD) and the rare hi deltas
 * (carry out of lo, or a value that does not fit 32 bits) sent to the HBM table with RED.ADD.64.
 * ------------------------------------------------------------------------------------------------------- */
/* branch-free predicated forms: the compiler wraps `if (p) atomicAdd(...)` in BSSY/BRA/BSYNC per row; a predicated
 * ATOMS needs none of that */
__device__ __forceinline__ void smem_inc_pred(uint32_t saddr, uint32_t pred) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0;\n\t@p red.shared.add.u32 [%0], 1;\n\t}" ::"r"(saddr), "r"(pred) : "memory");
}
__device__ __forceinline__ uint32_t smem_add_ret_pred(uint32_t saddr, uint32_t v, uint32_t pred) {
  uint32_t old = 0;
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %3, 0;\n\t@p atom.shared.add.u32 %0, [%1], %2;\n\t}" : "+r"(old) : "r"(saddr), "r"(v), "r"(pred) : "memory");
  return old;
}
__device__ __forceinline__ void smem_sum_i64_pred(uint32_t saddr, int64_t* gslot, uint32_t vl, int32_t vh, uint32_t pred) {
  const uint32_t old = smem_add_ret_pred(saddr, vl, pred);
  const int32_t hi = vh + (int32_t)((uint32_t)(old + vl) < old);
  if (pred && hi != 0) red_add_u64(gslot, (uint64_t)(int64_t)hi << 32);
}

__device__ __forceinline__ void smem_sum_i64(int8_t* tab, int64_t* garr, uint32_t e, uint32_t vl, int32_t vh) {
  const uint32_t old = atomicAdd(reinterpret_cast<uint32_t*>(tab) + e, vl);
  const int32_t hi = vh + (int32_t)((uint32_t)(old + vl) < old);
  if (hi != 0) red_add_u64(garr + e, (uint64_t)(int64_t)hi << 32);
}

__device__ __forceinline__ void smem_minmax(int op, int8_t* tab, uint32_t e, int64_t v) {
  const bool fp = (op == ACC_MIN_F64) | (op == ACC_MAX_F64);
  if (fp) v = op == ACC_MIN_F64 ? b2q_f64_min_ord(v) : b2q_f64_max_ord(v); /* a NaN loses to every number (b2q_f64_min_ord) */
  long long* p = reinterpret_cast<long long*>(tab) + e;
  const long long cur = *reinterpret_cast<volatile long long*>(p);
  if ((op == ACC_MIN_I64) | (op == ACC_MIN_F64)) { if (v < cur) atomicMin(p, (long long)v); }
  else { if (v > cur) atomicMax(p, (long long)v); }
}

/* warp-level reductions for the single-group (non-grouped) case */
__device__ __forceinline__ int64_t warp_sum_i64(int64_t v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int64_t warp_min_i64(int64_t v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) { const int64_t w = __shfl_xor_sync(0xffffffffu, v, o); v = w < v ? w : v; }
  return v;
}
__device__ __forceinline__ int64_t warp_max_i64(int64_t v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) { const int64_t w = __shfl_xor_sync(0xffffffffu, v, o); v = w > v ? w : v; }
  return v;
}

/* ---------------------------------------------------------------------------------------------------------
 * TMA bulk copy global -> shared (cp.async.bulk, SASS UBLKCP) with mbarrier completion
 * ------------------------------------------------------------------------------------------------------- */
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(phase)
        : "memory");
  }
}
__device__ __forceinline__ void tma_bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

/* ---------------------------------------------------------------------------------------------------------
 * the scan kernel
 * ------------------------------------------------------------------------------------------------------- */
struct ScanArgs {
  DevProgram prog;
  DevLaunch launch;
  SmemPlan smem;
  const int8_t* smem_image; /* identity image of ONE replica in HBM (MODE_SMEM) */
  int64_t ndv_bitmap_bytes;  /* estimator query: size of the ACC_NDV bitmap (a power of two) */
};

extern __shared__ __align__(128) int8_t b2q_smem[];

/* one chunk: R rows per thread.  FULL = every row of the chunk exists (no tail masking). */
/* JOIN: 0 = no join level, 1 = INNER, 2 = LEFT (separate instantiations: the plain scan and the INNER probe do not pay
 * for the NULL placeholders of the outer join) */
template <int MODE, bool WAGG, bool KEY32, bool FULL, int BLOCK, int JOIN>
__device__ __forceinline__ void process_chunk(const ScanArgs& A, const int8_t* const* __restrict__ cols, int64_t row0,
                                              int64_t frag_rows, int lane, int8_t* my_tab, uint64_t pol, uint64_t pol_tab) {
  /* BLOCK is a compile-time constant so that the R loads of a column are one base pointer + immediate offsets */
  constexpr int nthr = BLOCK;
  const DevProgram& P = A.prog;
  const DevLaunch& Lh = A.launch;
  uint32_t valid = (1u << R) - 1u;
  if (!FULL) {
    valid = 0;
#pragma unroll
    for (int j = 0; j < R; ++j) valid |= (uint32_t)(row0 + (int64_t)j * nthr < frag_rows) << j;
  }

  /* ---- join level: probe the one-to-one table with the outer key; rows without a match leave `valid`
   * (hash_join_idx[_nullable], GroupByRuntime.cpp:283-311; INNER join).  Columns of the inner table are then read at
   * jidx[] — see load32 / load64. ---- */
  int32_t jidx[JOIN ? R : 1];
  int32_t jval[JOIN ? R : 1]; /* value of the inner column that is packed into the join table (DevJoin::packed_col) */
#define JX(c) ((JOIN && P.col_inner[c]) ? jidx : nullptr), ((JOIN && (c) == P.join.packed_col) ? jval : nullptr), (JOIN == 2 ? P.col_null + (c) : nullptr)
  if (JOIN) {
    const DevJoin& J = P.join;
    const int32_t* __restrict__ buff = Lh.join_buff;
    const int32_t* jsm = A.smem.join_off >= 0 ? reinterpret_cast<const int32_t*>(b2q_smem + A.smem.join_off) : nullptr; /* staged copy */
    const bool packed = J.packed_col >= 0;
    const int32_t packed_null = (JOIN == 2 && packed) ? (int32_t)P.col_null[J.packed_col] : 0;
    const int32_t slot16_null = packed ? (int32_t)P.col_null[J.packed_col] : 0; /* a NULL attribute of a matched row */
    uint32_t matched = 0;
    if (J.fk_width == 8) {
      int64_t k[R];
      load64<!FULL>(k, cols[J.fk_col], row0, nthr, valid, pol);
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const uint64_t d = (uint64_t)(k[j] - J.min_key);
        const bool ok = (valid >> j & 1) && d < (uint64_t)J.entry_count && !(J.nullable && k[j] == J.null_val);
        int32_t idx = -1, val = packed_null;
        if (ok && J.slot16) { /* value-only 16-bit slot in shared memory (DevJoin::slot16) */
          const uint32_t s16 = reinterpret_cast<const uint16_t*>(jsm)[d];
          idx = s16 == 0xFFFFu ? -1 : 0;
          val = s16 >= 0xFFFEu ? slot16_null : (int32_t)(J.slot16_min + (int64_t)s16);
        } else if (ok) {
          if (packed) {
            const int2 e2 = jsm ? reinterpret_cast<const int2*>(jsm)[d]
                                : (J.probe_cg ? __ldcg(reinterpret_cast<const int2*>(buff) + d) : __ldg(reinterpret_cast<const int2*>(buff) + d));
            idx = e2.x;
            val = (JOIN == 2 && e2.x < 0) ? packed_null : e2.y;
          } else {
            idx = jsm ? jsm[d] : __ldg(buff + d);
          }
        }
        jidx[JOIN ? j : 0] = idx;
        jval[JOIN ? j : 0] = val;
        matched |= (uint32_t)(idx >= 0) << j;
      }
    } else {
      int32_t k[R];
      load32<!FULL>(k, cols[J.fk_col], J.fk_width, row0, nthr, valid, pol);
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const uint64_t d = (uint64_t)((int64_t)k[j] - J.min_key);
        const bool ok = (valid >> j & 1) && d < (uint64_t)J.entry_count && !(J.nullable && (int64_t)k[j] == J.null_val);
        int32_t idx = -1, val = packed_null;
        if (ok && J.slot16) { /* value-only 16-bit slot in shared memory (DevJoin::slot16) */
          const uint32_t s16 = reinterpret_cast<const uint16_t*>(jsm)[d];
          idx = s16 == 0xFFFFu ? -1 : 0;
          val = s16 >= 0xFFFEu ? slot16_null : (int32_t)(J.slot16_min + (int64_t)s16);
        } else if (ok) {
          if (packed) {
            const int2 e2 = jsm ? reinterpret_cast<const int2*>(jsm)[d]
                                : (J.probe_cg ? __ldcg(reinterpret_cast<const int2*>(buff) + d) : __ldg(reinterpret_cast<const int2*>(buff) + d));
            idx = e2.x;
            val = (JOIN == 2 && e2.x < 0) ? packed_null : e2.y;
          } else {
            idx = jsm ? jsm[d] : __ldg(buff + d);
          }
        }
        jidx[JOIN ? j : 0] = idx;
        jval[JOIN ? j : 0] = val;
        matched |= (uint32_t)(idx >= 0) << j;
      }
    }
    if (JOIN != 2) valid &= matched; /* INNER: no match, no row; LEFT: the row stays and its inner columns are NULL */
  }

  /* ---- key column: issued before the filter when the planner expects most sectors to be needed anyway ---- */
  int32_t k32[KEY32 ? R : 1];
  int64_t k64[KEY32 ? 1 : R];
  const bool has_key = !WAGG && P.key.col >= 0;
  const bool eager_key = P.eager_key;
  if (has_key && eager_key) {
    if (KEY32) load32<true>(reinterpret_cast<int32_t(&)[R]>(k32), cols[P.key.col], P.key.width, row0, nthr, valid, pol, JX(P.key.col));
    else load64<true>(reinterpret_cast<int64_t(&)[R]>(k64), cols[P.key.col], row0, nthr, valid, pol, JX(P.key.col));
  }

  uint32_t pass = eval_filter<FULL, JOIN>(P.filter, cols, row0, nthr, valid, pol, P.col_inner, jidx, P.join.packed_col, jval, P.col_null);

  if (has_key && !eager_key) {
    if (KEY32) load32<true>(reinterpret_cast<int32_t(&)[R]>(k32), cols[P.key.col], P.key.width, row0, nthr, pass, pol, JX(P.key.col));
    else load64<true>(reinterpret_cast<int64_t(&)[R]>(k64), cols[P.key.col], row0, nthr, pass, pol, JX(P.key.col));
  }

  /* ---- group index ---- */
  uint32_t e[R];
#pragma unroll
  for (int j = 0; j < R; ++j) e[j] = 0;
  if (!WAGG && !KEY32 && MODE != MODE_BASELINE && P.n_keys > 1) {
    /* multi-column perfect hash: perfect_key_hash (GroupByAndAggregate.cpp:1549-1597) — mixed-radix index over the
     * NULL-translated keys; one warp-uniform pass per GROUP BY column */
    uint32_t bad = 0;
    const uint32_t kmask = P.eager_key ? valid : pass;
    for (int c = 0; c < P.n_keys; ++c) {
      const DevKeyComp& kc = P.keys[c];
      const int64_t mn = kc.min_val, nullv = kc.null_val;
      const uint64_t card = kc.card;
      const uint32_t mult = kc.mult;
      const bool tr = kc.translate_null;
      if (kc.width == 8) {
        int64_t k[R];
        load64<true>(k, cols[kc.col], row0, nthr, kmask, pol, JX(kc.col));
#pragma unroll
        for (int j = 0; j < R; ++j) {
          int64_t d = k[j] - mn;
          if (kc.div_day) { /* DATE: bucketed by day; a value off the day grid has no reconstructible key */
            d = d / 86400;
            if (k[j] % 86400 != 0 && !(tr && k[j] == nullv)) d = -1;
          }
          if (tr) d = (k[j] == nullv) ? (int64_t)card - 1 : d;
          bad |= (uint32_t)((uint64_t)d >= card) << j;
          e[j] += (uint32_t)d * mult;
        }
      } else {
        int32_t k[R];
        load32<true>(k, cols[kc.col], kc.width, row0, nthr, kmask, pol, JX(kc.col));
#pragma unroll
        for (int j = 0; j < R; ++j) {
          int64_t d = (int64_t)k[j] - mn;
          if (tr) d = ((int64_t)k[j] == nullv) ? (int64_t)card - 1 : d;
          bad |= (uint32_t)((uint64_t)d >= card) << j;
          e[j] += (uint32_t)d * mult;
        }
      }
    }
    bad &= pass;
    if (bad) { atomicCAS(Lh.error, 0, B2Q_ERR_KEY_OUT_OF_RANGE); pass &= ~bad; }
  }
  if (has_key) {
    if (MODE != MODE_BASELINE) {
      uint32_t bad = 0;
      const bool tr = P.key.translate_null;
      if (KEY32) {
        const uint32_t mn = (uint32_t)P.key.min_val, n = (uint32_t)P.key.entry_count, nidx = (uint32_t)P.key.null_idx;
        const int32_t nullv = (int32_t)P.key.null_val;
        if (tr) {
#pragma unroll
          for (int j = 0; j < R; ++j) {
            uint32_t idx = (uint32_t)k32[KEY32 ? j : 0] - mn;
            idx = (k32[KEY32 ? j : 0] == nullv) ? nidx : idx;
            bad |= (uint32_t)(idx >= n) << j;
            e[j] = idx;
          }
        } else {
#pragma unroll
          for (int j = 0; j < R; ++j) {
            const uint32_t idx = (uint32_t)k32[KEY32 ? j : 0] - mn;
            bad |= (uint32_t)(idx >= n) << j;
            e[j] = idx;
          }
        }
      } else {
        const int64_t mn = P.key.min_val, nullv = P.key.null_val, nidx = P.key.null_idx;
        const uint64_t n = (uint64_t)P.key.entry_count;
#pragma unroll
        for (int j = 0; j < R; ++j) {
          int64_t idx = k64[KEY32 ? 0 : j] - mn;
          if (P.key.div_day) { /* DATE: (key - min) / bucket (get_group_value_fast, GroupByRuntime.cpp:194-209) */
            idx = idx / 86400;
            if (k64[KEY32 ? 0 : j] % 86400 != 0 && !(tr && k64[KEY32 ? 0 : j] == nullv)) idx = -1;
          }
          if (tr) idx = (k64[KEY32 ? 0 : j] == nullv) ? nidx : idx;
          bad |= (uint32_t)((uint64_t)idx >= n) << j;
          e[j] = (uint32_t)idx;
        }
      }
      bad &= pass;
      if (bad) { atomicCAS(Lh.error, 0, B2Q_ERR_KEY_OUT_OF_RANGE); pass &= ~bad; }
    } else {
      const uint32_t n = (uint32_t)P.key.entry_count;
      const uint64_t magic = P.key.hash_magic;
      const int hw = P.key.hash_key_width;
      unsigned long long* keys = reinterpret_cast<unsigned long long*>(Lh.keys);
      /* get_group_value (GroupByRuntime.cpp:25-48): h = MurmurHash3(key) % entry_count, linear probe.
       * Phase 1 puts the home-slot loads of all R rows in flight together (ld.global.cg: L2 is the coherence point,
       * so a concurrent claim by another SM is visible); phase 2 resolves each row, falling back to the probe loop. */
      int64_t key[R];
      uint32_t h[R];
      unsigned long long first[R];
#pragma unroll
      for (int j = 0; j < R; ++j) {
        key[j] = KEY32 ? (int64_t)k32[KEY32 ? j : 0] : k64[KEY32 ? 0 : j];
        if (key[j] == P.key.null_val) key[j] = P.key.null_logical; /* ENCODING FIXED: physical NULL -> logical NULL */
        h[j] = (uint32_t)__umul64hi(magic * (uint64_t)murmur3_key(key[j], hw), (uint64_t)n); /* == hash % n */
      }
#pragma unroll
      for (int j = 0; j < R; ++j) first[j] = (pass >> j & 1) ? __ldcg(keys + h[j]) : 0ull;
#pragma unroll
      for (int j = 0; j < R; ++j) {
        if (!(pass >> j & 1)) continue;
        const unsigned long long want = (unsigned long long)key[j];
        uint32_t p = h[j];
        unsigned long long cur = first[j];
        bool found = false;
        for (;;) { /* claim an EMPTY_KEY_64 slot with a 64-bit CAS; a lost race re-examines the same slot */
          if (cur == (unsigned long long)B2Q_I64_MAX) cur = atomicCAS(keys + p, (unsigned long long)B2Q_I64_MAX, want);
          if (cur == (unsigned long long)B2Q_I64_MAX || cur == want) { found = true; break; }
          p = p + 1 == n ? 0 : p + 1;
          if (p == h[j]) break;
          cur = __ldcg(keys + p);
        }
        if (!found) { atomicCAS(Lh.error, 0, B2Q_ERR_OUT_OF_SLOTS); pass &= ~(1u << j); }
        e[j] = p;
      }
      /* the probe loops diverge per lane; without an explicit reconvergence the warp stays split for the rest of the
       * kernel and every following column load is issued lane by lane (ncu: 3.8 active threads per LDG, one 32-B
       * sector per thread, 23x the algorithmic DRAM traffic) */
      __syncwarp();
    }
  }

  const uint32_t arg_mask = P.eager_args ? valid : pass;

  /* ---- fused fast path: COUNT(*) and/or one integer SUM, both updates of a row under one predicate region
   * (the per-accumulator loops spend a large share of their instructions per row on predicate extraction,
   * BSSY/BRA/BSYNC and address math; fusing them removes most of it) ---- */
  if (MODE == MODE_SMEM && !WAGG && P.fused) {
    const int ic = P.fused_cnt, is = P.fused_sum;
    const uint32_t cnt32 = ic >= 0 ? smem_u32(my_tab + A.smem.acc_off[ic]) : 0u;
    if (is < 0) {
#pragma unroll
      for (int j = 0; j < R; ++j) if (pass >> j & 1) atomicAdd(reinterpret_cast<uint32_t*>(my_tab + A.smem.acc_off[ic]) + e[j], 1u);
      return;
    }
    const DevAcc& sa = P.accs[is];
    uint32_t* sum_tab = reinterpret_cast<uint32_t*>(my_tab + A.smem.acc_off[is]);
    uint32_t* cnt_tab = reinterpret_cast<uint32_t*>(my_tab + A.smem.acc_off[ic >= 0 ? ic : is]);
    int64_t* gsum = Lh.accs[is];
    (void)cnt32;
    if (sa.op == ACC_SUM_F64) { /* AVG/SUM(double): CAS-loop add on the (warp-private) replica + the count */
      int64_t v[R];
      load64<true>(v, cols[sa.col], row0, nthr, arg_mask, pol, JX(sa.col));
      double* dsum = reinterpret_cast<double*>(sum_tab);
      /* (measured and dropped: plain LDS / DADD / STS on the warp-private replica, lanes of a row grouped by entry with
       * MATCH.ANY and serialised by rank — more than twice as slow as this CAS loop on C3: MATCH.ANY + REDUX per row costs
       * more than the ATOMS.CAST.SPIN it saves) */
#pragma unroll
      for (int j = 0; j < R; ++j)
        if (pass >> j & 1) {
          if (ic >= 0) atomicAdd(cnt_tab + e[j], 1u);
          atomicAdd(dsum + e[j], __longlong_as_double(v[j]));
        }
    } else if (sa.width == 8) {
      int64_t v[R];
      load64<true>(v, cols[sa.col], row0, nthr, arg_mask, pol, JX(sa.col));
      if (ic >= 0) {
#pragma unroll
        for (int j = 0; j < R; ++j)
          if (pass >> j & 1) {
            atomicAdd(cnt_tab + e[j], 1u);
            const uint32_t vl = (uint32_t)v[j];
            const uint32_t old = atomicAdd(sum_tab + e[j], vl);
            const int32_t hi = (int32_t)(v[j] >> 32) + (int32_t)((uint32_t)(old + vl) < old);
            if (hi != 0) red_add_u64(gsum + e[j], (uint64_t)(int64_t)hi << 32);
          }
      } else {
#pragma unroll
        for (int j = 0; j < R; ++j)
          if (pass >> j & 1) {
            const uint32_t vl = (uint32_t)v[j];
            const uint32_t old = atomicAdd(sum_tab + e[j], vl);
            const int32_t hi = (int32_t)(v[j] >> 32) + (int32_t)((uint32_t)(old + vl) < old);
            if (hi != 0) red_add_u64(gsum + e[j], (uint64_t)(int64_t)hi << 32);
          }
      }
    } else {
      int32_t v[R];
      load32<true>(v, cols[sa.col], sa.width, row0, nthr, arg_mask, pol, JX(sa.col));
#pragma unroll
      for (int j = 0; j < R; ++j)
        if (pass >> j & 1) {
          if (ic >= 0) atomicAdd(cnt_tab + e[j], 1u);
          const uint32_t vl = (uint32_t)v[j];
          const uint32_t old = atomicAdd(sum_tab + e[j], vl);
          const int32_t hi = (v[j] >> 31) + (int32_t)((uint32_t)(old + vl) < old);
          if (hi != 0) red_add_u64(gsum + e[j], (uint64_t)(int64_t)hi << 32);
        }
    }
    return;
  }

  /* ---- aggregate updates: one warp-uniform dispatch per accumulator per R rows ---- */
  for (int a = 0; a < P.n_accs; ++a) {
    const DevAcc& acc = P.accs[a];
    const int op = acc.op;
    int64_t* garr = Lh.accs[a];
    int8_t* tab = (MODE == MODE_SMEM) ? my_tab + A.smem.acc_off[a] : nullptr;
    /* flags array when THIS accumulator carries the touched flag for the global-table kernels */
    uint8_t* pig = (MODE != MODE_SMEM && P.touch_piggyback == a) ? reinterpret_cast<uint8_t*>(Lh.accs[P.touch_acc]) : nullptr;
    const int64_t n_split = Lh.split ? P.key.entry_count : int64_t(-1); /* (lo[n] | hi[n]) layout of COUNT / integer SUM, or plain int64[] */

    if (op == ACC_NDV) {
      /* estimator query: linear_probabilistic_count (RuntimeFunctions.cpp:2399-2408, cuda_mapd_rt.cu:1300-1308) over
       * the tuple of int64 sub-keys (codegenEstimator); the bitmap lives in HBM/L2 and saturates quickly, so a
       * plain load filters out the bits that are already set before the atomic OR */
      if (WAGG) {
        uint32_t h[R];
#pragma unroll
        for (int j = 0; j < R; ++j) h[j] = 0;
        for (int c = 0; c < P.n_keys; ++c) {
          const DevKeyComp& kc = P.keys[c];
          int64_t k[R];
          if (kc.width == 8) load64<true>(k, cols[kc.col], row0, nthr, pass, pol, JX(kc.col));
          else {
            int32_t t32[R];
            load32<true>(t32, cols[kc.col], kc.width, row0, nthr, pass, pol, JX(kc.col));
#pragma unroll
            for (int j = 0; j < R; ++j) k[j] = t32[j];
          }
#pragma unroll
          for (int j = 0; j < R; ++j) {
            const int64_t v = (kc.translate_null && k[j] == kc.null_val) ? kc.null_logical : k[j];
            h[j] = murmur_block(murmur_block(h[j], (uint32_t)v), (uint32_t)((uint64_t)v >> 32));
          }
        }
        uint32_t* bitmap = reinterpret_cast<uint32_t*>(garr);
        const uint32_t bits_mask = (uint32_t)(A.ndv_bitmap_bytes * 8ull - 1ull); /* the buffer sizes are powers of two */
#pragma unroll
        for (int j = 0; j < R; ++j) {
          if (!(pass >> j & 1)) continue;
          const uint32_t bit_pos = murmur3_fmix(h[j], (uint32_t)P.n_keys * 8u) & bits_mask;
          const uint32_t bit = 1u << (bit_pos & 31u);
          uint32_t* w = bitmap + (bit_pos >> 5);
          if (!(__ldcg(w) & bit)) atomicOr(w, bit);
        }
      }
      continue;
    }

    if (op == ACC_BITMAP) {
      /* COUNT(DISTINCT c): agg_count_distinct_bitmap[_skip_val] (RuntimeFunctions.cpp:366-376, :1201-1210) — bit
       * (v - min) / bucket of the group's bitmap; the bitmaps live in HBM / L2 and saturate quickly, so a plain load filters
       * out the bits that are already set before the atomic OR (as for the estimator's bitmap) */
      int64_t v[R];
      if (acc.width == 8) load64<true>(v, cols[acc.col], row0, nthr, arg_mask, pol, JX(acc.col));
      else {
        int32_t t32[R];
        load32<true>(t32, cols[acc.col], acc.width, row0, nthr, arg_mask, pol, JX(acc.col));
#pragma unroll
        for (int j = 0; j < R; ++j) v[j] = t32[j];
      }
      const uint32_t m = not_skipped64(acc, v, pass);
      uint32_t* bitmaps = reinterpret_cast<uint32_t*>(garr);
      uint32_t bad = 0;
#pragma unroll
      for (int j = 0; j < R; ++j) {
        if (!(m >> j & 1)) continue;
        uint64_t idx = (uint64_t)(v[j] - acc.bm_min);
        if (acc.bm_bucket > 1) idx /= (uint64_t)acc.bm_bucket;
        if (idx >= (uint64_t)acc.bm_bits) { bad |= 1u << j; continue; } /* outside the chunk-stats range: the reference would write out of bounds */
        uint32_t* w = bitmaps + (size_t)e[j] * (size_t)acc.bm_words + (size_t)(idx >> 5);
        const uint32_t bit = 1u << (idx & 31u);
        if (!(__ldcg(w) & bit)) atomicOr(w, bit);
      }
      if (bad) atomicCAS(Lh.error, 0, B2Q_ERR_KEY_OUT_OF_RANGE);
      continue;
    }

    if (op == ACC_COUNT && acc.col < 0) { /* COUNT(*) */
      if (WAGG) {
        const uint32_t c = __reduce_add_sync(0xffffffffu, (uint32_t)__popc(pass));
        if (lane == 0 && c) atomicAdd(reinterpret_cast<uint32_t*>(tab), c);
      } else if (MODE == MODE_SMEM) {
        const uint32_t tab32 = smem_u32(tab);
#pragma unroll
        for (int j = 0; j < R; ++j) smem_inc_pred(tab32 + e[j] * 4u, pass >> j & 1);
      } else {
#pragma unroll
        for (int j = 0; j < R; ++j) if (pass >> j & 1) global_split_add_touch(garr, pig, e[j], n_split, 1u, 0, pol_tab);
      }
      continue;
    }

    if (op == ACC_TOUCH) { /* "a row reached this group": a byte flag, set at most once per thread view */
      if (MODE == MODE_SMEM) {
#pragma unroll
        for (int j = 0; j < R; ++j) if (pass >> j & 1) reinterpret_cast<uint8_t*>(tab)[e[j]] = 1;
      } else if (P.touch_piggyback < 0) {
        uint8_t* flags = reinterpret_cast<uint8_t*>(garr);
#pragma unroll
        for (int j = 0; j < R; ++j) {
          if (!(pass >> j & 1)) continue;
          uint32_t w;
          asm volatile("ld.global.ca.L2::cache_hint.u8 %0, [%1], %2;" : "=r"(w) : "l"(flags + e[j]), "l"(pol_tab)); /* a stale 0 only costs a redundant store */
          if (!w) flags[e[j]] = 1;
        }
      }
      continue;
    }

    const bool narrow = acc.width <= 4 && !acc.is_fp && (op == ACC_COUNT || op == ACC_SUM_I64 || op == ACC_MIN_I64 || op == ACC_MAX_I64);
    if (narrow) {
      /* 1/2/4-byte integer argument: 32-bit registers */
      int32_t v[R];
      load32<true>(v, cols[acc.col], acc.width, row0, nthr, arg_mask, pol, JX(acc.col));
      const uint32_t m = not_skipped32(acc, v, pass);
      if (WAGG) {
        if (op == ACC_COUNT) {
          const uint32_t c = __reduce_add_sync(0xffffffffu, (uint32_t)__popc(m));
          if (lane == 0 && c) atomicAdd(reinterpret_cast<uint32_t*>(tab), c);
        } else if (op == ACC_SUM_I64) {
          int64_t s = 0;
#pragma unroll
          for (int j = 0; j < R; ++j) s += (m >> j & 1) ? (int64_t)v[j] : 0;
          s = warp_sum_i64(s);
          if (lane == 0 && s) smem_sum_i64(tab, garr, 0, (uint32_t)s, (int32_t)(s >> 32));
        } else {
          const bool is_min = op == ACC_MIN_I64;
          int64_t r = is_min ? B2Q_I64_MAX : B2Q_I64_MIN;
#pragma unroll
          for (int j = 0; j < R; ++j) if (m >> j & 1) r = is_min ? min(r, (int64_t)v[j]) : max(r, (int64_t)v[j]);
          r = is_min ? warp_min_i64(r) : warp_max_i64(r);
          if (lane == 0 && r != (is_min ? B2Q_I64_MAX : B2Q_I64_MIN)) smem_minmax(op, tab, 0, r);
        }
      } else if (MODE == MODE_SMEM) {
        const uint32_t tab32 = smem_u32(tab);
        if (op == ACC_COUNT) {
#pragma unroll
          for (int j = 0; j < R; ++j) smem_inc_pred(tab32 + e[j] * 4u, m >> j & 1);
        } else if (op == ACC_SUM_I64) {
#pragma unroll
          for (int j = 0; j < R; ++j) smem_sum_i64_pred(tab32 + e[j] * 4u, garr + e[j], (uint32_t)v[j], v[j] >> 31, m >> j & 1);
        } else {
#pragma unroll
          for (int j = 0; j < R; ++j) if (m >> j & 1) smem_minmax(op, tab, e[j], (int64_t)v[j]);
        }
      } else {
#pragma unroll
        for (int j = 0; j < R; ++j) if (m >> j & 1) global_update(op, garr, pig, e[j], n_split, (int64_t)v[j], pol_tab);
      }
      continue;
    }

    /* 8-byte argument (BIGINT or DOUBLE), or a FLOAT column: 4-byte chunk elements widened (exactly) to double */
    int64_t v[R];
    if (acc.width == 8) load64<true>(v, cols[acc.col], row0, nthr, arg_mask, pol, JX(acc.col));
    else {
      int32_t t32[R];
      load32<true>(t32, cols[acc.col], acc.width, row0, nthr, arg_mask, pol, JX(acc.col));
#pragma unroll
      for (int j = 0; j < R; ++j) v[j] = acc.is_fp ? __double_as_longlong((double)__int_as_float(t32[j])) : (int64_t)t32[j];
    }
    const uint32_t m = not_skipped64(acc, v, pass);
    if (WAGG) {
      switch (op) {
        case ACC_COUNT: {
          const uint32_t c = __reduce_add_sync(0xffffffffu, (uint32_t)__popc(m));
          if (lane == 0 && c) atomicAdd(reinterpret_cast<uint32_t*>(tab), c);
          break;
        }
        case ACC_SUM_I64: {
          int64_t s = 0;
#pragma unroll
          for (int j = 0; j < R; ++j) s += (m >> j & 1) ? v[j] : 0;
          s = warp_sum_i64(s);
          if (lane == 0 && s) smem_sum_i64(tab, garr, 0, (uint32_t)s, (int32_t)(s >> 32));
          break;
        }
        case ACC_SUM_F64: {
          double s = 0;
#pragma unroll
          for (int j = 0; j < R; ++j) s += (m >> j & 1) ? __longlong_as_double(v[j]) : 0.0;
          const uint32_t any = __ballot_sync(0xffffffffu, m != 0);
          s = warp_sum_f64(s);
          if (lane == 0 && any) atomicAdd(reinterpret_cast<double*>(tab), s);
          break;
        }
        default: {
          const bool is_min = (op == ACC_MIN_I64) | (op == ACC_MIN_F64);
          const bool fp = (op == ACC_MIN_F64) | (op == ACC_MAX_F64);
          int64_t r = is_min ? B2Q_I64_MAX : B2Q_I64_MIN;
#pragma unroll
          for (int j = 0; j < R; ++j) {
            if (!(m >> j & 1)) continue;
            int64_t x = v[j];
            if (fp) x = is_min ? b2q_f64_min_ord(x) : b2q_f64_max_ord(x);
            r = is_min ? min(r, x) : max(r, x);
          }
          r = is_min ? warp_min_i64(r) : warp_max_i64(r);
          if (lane == 0 && r != (is_min ? B2Q_I64_MAX : B2Q_I64_MIN)) {
            long long* p = reinterpret_cast<long long*>(tab);
            if (is_min) atomicMin(p, (long long)r); else atomicMax(p, (long long)r);
          }
          break;
        }
      }
    } else if (MODE == MODE_SMEM) {
      switch (op) { /* dispatch hoisted out of the row loop */
        case ACC_COUNT: {
          const uint32_t tab32 = smem_u32(tab);
#pragma unroll
          for (int j = 0; j < R; ++j) smem_inc_pred(tab32 + e[j] * 4u, m >> j & 1);
          break;
        }
        case ACC_SUM_I64: {
          const uint32_t tab32 = smem_u32(tab);
#pragma unroll
          for (int j = 0; j < R; ++j) smem_sum_i64_pred(tab32 + e[j] * 4u, garr + e[j], (uint32_t)v[j], (int32_t)(v[j] >> 32), m >> j & 1);
          break;
        }
        case ACC_SUM_F64:
#pragma unroll
          for (int j = 0; j < R; ++j) if (m >> j & 1) atomicAdd(reinterpret_cast<double*>(tab) + e[j], __longlong_as_double(v[j]));
          break;
        default:
#pragma unroll
          for (int j = 0; j < R; ++j) if (m >> j & 1) smem_minmax(op, tab, e[j], v[j]);
          break;
      }
    } else {
#pragma unroll
      for (int j = 0; j < R; ++j) if (m >> j & 1) global_update(op, garr, pig, e[j], n_split, v[j], pol_tab);
    }
  }
}
#undef JX

template <int MODE, bool WAGG, bool KEY32, int BLOCK, int JOIN>
__global__ void __launch_bounds__(BLOCK, 1024 / BLOCK) b2q_k_scan(const __grid_constant__ ScanArgs A) {
  const DevProgram& P = A.prog;
  const DevLaunch& Lh = A.launch;
  const int tid = threadIdx.x;
  constexpr int nthr = BLOCK;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  const int64_t chunk_rows = (int64_t)nthr * R;
  __shared__ uint64_t s_bar;
  int8_t* my_tab = nullptr;

  /* a dimension-sized join table is staged into shared memory next to the group table: the probe is then a shared-memory
   * load instead of one random L2 sector per row (the L2 sector rate is what bounds the join kernels) */
  const bool stage_join = JOIN && A.smem.join_off >= 0;
  if (MODE == MODE_SMEM || stage_join) {
    /* TMA-stage the identity image into every replica of the CTA-private table */
    const uint32_t rb = (uint32_t)A.smem.replica_bytes;
    const uint32_t nrep = MODE == MODE_SMEM ? (uint32_t)A.smem.replicas : 0u;
    if (tid == 0) {
      mbar_init(&s_bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0) {
      mbar_expect_tx(&s_bar, rb * nrep + (stage_join ? (uint32_t)A.smem.join_bytes : 0u));
      for (uint32_t r = 0; r < nrep; ++r) {
        uint32_t off = 0;
        while (off < rb) { /* bulk copies of <= 64 KB, 16-byte granularity (replica_bytes is a multiple of 16) */
          const uint32_t n = min(rb - off, 65536u);
          tma_bulk_g2s(b2q_smem + (size_t)r * rb + off, A.smem_image + off, n, &s_bar);
          off += n;
        }
      }
      if (stage_join) {
        const uint32_t jb = (uint32_t)A.smem.join_bytes;
        uint32_t off = 0;
        while (off < jb) {
          const uint32_t n = min(jb - off, 65536u);
          tma_bulk_g2s(b2q_smem + A.smem.join_off + off, reinterpret_cast<const int8_t*>(Lh.join_buff) + off, n, &s_bar);
          off += n;
        }
      }
    }
    mbar_wait(&s_bar, 0);
    /* (a replica per HALF-warp for C3-sized tables was measured: no change) */
    if (MODE == MODE_SMEM) my_tab = b2q_smem + (size_t)(warp & (A.smem.replicas - 1)) * rb;
  }

  /* L2 policy for the column stream: it is read exactly once, so mark it evict-first and keep L2 for what is
   * re-used (the HBM/L2-resident group table of the global-table kernels) */
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  uint64_t pol_tab;
  asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol_tab));

  /* chunks are visited in increasing order, so the owning fragment is a moving cursor, not a search */
  int frag = 0;
  int64_t frag_first = 0;                                   /* first chunk of `frag` */
  int64_t next_first = __ldg(Lh.frag_chunk_start + 1);      /* first chunk of frag + 1 */
  for (int64_t chunk = blockIdx.x; chunk < Lh.total_chunks; chunk += gridDim.x) {
    while (chunk >= next_first) {
      ++frag;
      frag_first = next_first;
      next_first = __ldg(Lh.frag_chunk_start + frag + 1);
    }
    const int64_t frag_rows = __ldg(Lh.frag_rows + frag);
    const int64_t base_row = (chunk - frag_first) * chunk_rows;
    const int8_t* const* __restrict__ cols = Lh.col_ptrs + (size_t)frag * P.n_cols;
    if (base_row + chunk_rows <= frag_rows)
      process_chunk<MODE, WAGG, KEY32, true, BLOCK, JOIN>(A, cols, base_row + tid, frag_rows, lane, my_tab, pol, pol_tab);
    else
      process_chunk<MODE, WAGG, KEY32, false, BLOCK, JOIN>(A, cols, base_row + tid, frag_rows, lane, my_tab, pol, pol_tab);
  }

  if (MODE == MODE_SMEM) {
    /* flush the CTA-private table into the dense HBM table: one RED per (entry, accumulator) that moved */
    __syncthreads();
    const uint32_t rb = (uint32_t)A.smem.replica_bytes;
    const int nrep = A.smem.replicas;
    const int64_t n = P.key.entry_count;
    for (int a = 0; a < P.n_accs; ++a) {
      const int op = P.accs[a].op;
      int64_t* garr = Lh.accs[a];
      const int8_t* base = b2q_smem + A.smem.acc_off[a];
      for (int64_t i = tid; i < n; i += nthr) {
        switch (op) {
          case ACC_NDV: case ACC_BITMAP: break; /* live in HBM only */
          case ACC_TOUCH: {
            uint32_t s = 0;
            for (int r = 0; r < nrep; ++r) s |= reinterpret_cast<const uint8_t*>(base + (size_t)r * rb)[i];
            if (s) reinterpret_cast<uint8_t*>(garr)[i] = 1;
            break;
          }
          case ACC_COUNT:
          case ACC_SUM_I64: {
            uint64_t s = 0;
            for (int r = 0; r < nrep; ++r) s += reinterpret_cast<const uint32_t*>(base + (size_t)r * rb)[i];
            if (s) red_add_u64(garr + i, s);
            break;
          }
          case ACC_SUM_F64: {
            double s = 0;
            bool any = false;
            for (int r = 0; r < nrep; ++r) { const double x = reinterpret_cast<const double*>(base + (size_t)r * rb)[i]; any |= (x != 0.0); s += x; }
            if (any) red_add_f64(garr + i, s);
            break;
          }
          case ACC_MIN_I64:
          case ACC_MIN_F64: {
            int64_t s = B2Q_I64_MAX;
            for (int r = 0; r < nrep; ++r) { const int64_t x = reinterpret_cast<const int64_t*>(base + (size_t)r * rb)[i]; s = x < s ? x : s; }
            if (s != B2Q_I64_MAX) red_min_s64(garr + i, s);
            break;
          }
          default: {
            int64_t s = B2Q_I64_MIN;
            for (int r = 0; r < nrep; ++r) { const int64_t x = reinterpret_cast<const int64_t*>(base + (size_t)r * rb)[i]; s = x > s ? x : s; }
            if (s != B2Q_I64_MIN) red_max_s64(garr + i, s);
            break;
          }
        }
      }
    }
  }
}

struct ScanConfig {
  int block;
  int grid;
  size_t smem_bytes;
};

template <int MODE, bool WAGG, bool KEY32, int BLOCK, int JOIN>
static cudaError_t launch_scan_tb(const ScanArgs& a, const ScanConfig& c, cudaStream_t st) {
  /* the opt-in shared-memory limit is a per-device function attribute: remember which devices have it (one atomic mask per
   * instantiation: b2q_execute_* may be called from one host thread per device) */
  static std::atomic<unsigned long long> attr_set_mask{0};
  int cur_dev = 0;
  cudaGetDevice(&cur_dev);
  const bool attr_set = cur_dev < 64 && (attr_set_mask.load(std::memory_order_acquire) >> cur_dev & 1ull);
  if (!attr_set) {
    int optin = 0;
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, cur_dev);
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, b2q_k_scan<MODE, WAGG, KEY32, BLOCK, JOIN>);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(b2q_k_scan<MODE, WAGG, KEY32, BLOCK, JOIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes);
    if (e != cudaSuccess) return e;
    if (cur_dev < 64) attr_set_mask.fetch_or(1ull << cur_dev, std::memory_order_release);
  }
  b2q_k_scan<MODE, WAGG, KEY32, BLOCK, JOIN><<<c.grid, c.block, c.smem_bytes, st>>>(a);
  return cudaGetLastError();
}

/* one entry per (join level, table-mode group); defined by scan_inst.cu compiled with -DB2Q_SCAN_JOIN=j -DB2Q_SCAN_GROUP=g
 * (group 0: shared-memory table incl. the non-grouped kernel, 1: HBM/L2 table, 2: baseline hash) */
#define B2Q_SCAN_ENTRY(j, g) cudaError_t launch_scan_j##j##_g##g(const ScanArgs& a, const ScanConfig& c, bool wagg, bool key32, cudaStream_t st)
B2Q_SCAN_ENTRY(0, 0); B2Q_SCAN_ENTRY(0, 1); B2Q_SCAN_ENTRY(0, 2);
B2Q_SCAN_ENTRY(1, 0); B2Q_SCAN_ENTRY(1, 1); B2Q_SCAN_ENTRY(1, 2);
B2Q_SCAN_ENTRY(2, 0); B2Q_SCAN_ENTRY(2, 1); B2Q_SCAN_ENTRY(2, 2);

}  // namespace b2q
