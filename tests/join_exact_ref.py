"""A plain reference of the one-level hash join, in numpy and Python ints: no oracle, no planner.

Build (PerfectJoinHashTable, one-to-one): the table spans [min, max] of the inner key's chunk stats, E = max - min + 1
entries, row_of[k - min] = the inner row holding key k.  NULL inner keys are skipped; a key that appears twice makes the
table not one-to-one (the reference then builds a one-to-many table, which this path refuses: NotOneToOne); a key outside
the chunk-stats range is KeyOutOfRange.

Probe (hash_join_idx[_nullable]): the outer key is decoded to its logical value at full 64-bit width (FIXED(8|16|32) chunks
sign-extended, their physical minimum is NULL); a NULL outer key misses, and so does a key outside [min, min + E).  INNER
drops the rows that miss; LEFT keeps them and every inner column reads NULL.

The joined columns come out as physical arrays with the column's NULL sentinel (unmatched LEFT rows included), which is
what int_exact_ref.groups_of and fp_exact_ref.groups_of take: the aggregate semantics live there, not here.

The uint16 join-table layout stores only one inner column, as value - vmin with 0xFFFE = NULL and 0xFFFF = no row
(DevJoin::slot16).  slot16_encode / slot16_decode restate that encoding; Joined.inner_via_slot16 reads an inner column
through it, which must give what the plain gather gives.

Mutations of the probe subclass Probe and override one method (test_join_exact_ref.py shows each changes a result).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

import int_exact_ref as ix
from heavydb_b200 import abi

SLOT16_NULL, SLOT16_EMPTY = 0xFFFE, 0xFFFF


class NotOneToOne(Exception):
    pass


class KeyOutOfRange(Exception):
    pass


def width_of(table: abi.Table, c: int) -> ix.Width:
    """The int_exact_ref width of column c of an abi.Table."""
    t, _nn = table.col_types[c]
    return ix.Width(f"col{c}", t, table.encoded_sizes[c], table.col_scales.get(c, 0))


def column(table: abi.Table, c: int) -> np.ndarray:
    """All fragments of column c, physical values."""
    return np.concatenate([f.host_cols[c] for f in table.fragments]) if table.fragments else np.zeros(0, table.physical_dtype(c))


def null_mask(table: abi.Table, c: int, phys: np.ndarray) -> np.ndarray:
    """Rows of column c that are NULL: a nullable column holding its physical sentinel."""
    if table.col_types[c][1]:
        return np.zeros(phys.size, bool)
    return phys == table.physical_null(c)


def stats_range(table: abi.Table, c: int):
    """[min, max] of column c's chunk stats (the inner table is one fragment); (0, -1) for an empty range."""
    st = table.fragments[0].stats[c]
    return (0, -1) if st.int_max < st.int_min else (int(st.int_min), int(st.int_max))


@dataclass
class JoinTable:
    min_key: int
    entry_count: int
    row_of: np.ndarray          # int64 [entry_count], -1 = no inner row
    null_rows: np.ndarray       # inner rows whose key is NULL (never matched, except by a mutation)


class Probe:
    """The reference build and probe; each method is one step a mutation may change."""

    def decode_outer(self, table: abi.Table, c: int):
        """(logical int64 keys, NULL mask) of the outer key column."""
        phys = column(table, c)
        return phys.astype(np.int64), null_mask(table, c, phys)

    def build(self, dim: abi.Table, c: int) -> JoinTable:
        lo, hi = stats_range(dim, c)
        e = hi - lo + 1
        keys = column(dim, c).astype(np.int64)
        nulls = null_mask(dim, c, keys)
        row_of = np.full(max(e, 0), -1, np.int64)
        rows = np.flatnonzero(~nulls)
        k = keys[rows]
        if rows.size and (k.min() < lo or k.max() > hi):
            raise KeyOutOfRange(f"inner key outside its chunk stats [{lo}, {hi}]")
        d = k - lo
        if np.unique(d).size != d.size:
            raise NotOneToOne("duplicate inner key")
        row_of[d] = rows
        return JoinTable(lo, e, row_of, np.flatnonzero(nulls))

    def slot(self, jt: JoinTable, k: np.ndarray, null: np.ndarray):
        """(hit mask, slot index) of every outer key: a non-NULL key inside [min, min + E)."""
        hit = ~null & (k >= jt.min_key) & (k <= jt.min_key + jt.entry_count - 1)
        return hit, np.where(hit, k - np.where(hit, jt.min_key, 0), 0)

    def probe(self, jt: JoinTable, k: np.ndarray, null: np.ndarray) -> np.ndarray:
        """The matching inner row of every outer row, -1 for none."""
        hit, d = self.slot(jt, k, null)
        idx = np.full(k.size, -1, np.int64)
        if jt.entry_count > 0:
            idx[hit] = jt.row_of[d[hit]]
        return idx

    def slot16_decode(self, codes: np.ndarray, vmin: int, null):
        """uint16 slots -> (matched, physical value, NULL where 0xFFFE)."""
        codes = codes.astype(np.int64)
        matched = codes != SLOT16_EMPTY
        vals = np.where(codes >= SLOT16_NULL, null, vmin + codes)
        return matched, vals


def slot16_encode(jt: JoinTable, vals: np.ndarray, null, vmin: int) -> np.ndarray:
    """The value-only table: one uint16 per slot.  A value outside [vmin, vmin + 0xFFFD] is KeyOutOfRange, as the device
    build reports it."""
    out = np.full(jt.entry_count, SLOT16_EMPTY, np.int64)
    has = jt.row_of >= 0
    v = vals[jt.row_of[has]].astype(np.int64)
    code = np.where(v == null, SLOT16_NULL, v - vmin)
    if np.any((v != null) & ((v - vmin < 0) | (v - vmin >= SLOT16_NULL))):
        raise KeyOutOfRange("packed value outside its chunk stats")
    out[has] = code
    return out.astype(np.uint16)


@dataclass
class Joined:
    """The rows a join keeps: outer row numbers, the matching inner row (-1 = none, LEFT only)."""
    fact: abi.Table
    dim: abi.Table
    rows: np.ndarray
    idx: np.ndarray
    left: bool
    jt: JoinTable
    probe: Probe
    outer_col: int

    def outer(self, c: int) -> np.ndarray:
        return column(self.fact, c)[self.rows]

    def inner(self, c: int) -> np.ndarray:
        """Inner column c at the matching rows, its physical NULL where there is no match."""
        col = column(self.dim, c)
        null = self.dim.physical_null(c)
        out = np.full(self.idx.size, null, dtype=col.dtype)
        m = self.idx >= 0
        out[m] = col[self.idx[m]]
        return out

    def inner_via_slot16(self, c: int, vmin: int) -> np.ndarray:
        """inner(c) read back through the uint16 table (the probe of DevJoin::slot16)."""
        col = column(self.dim, c)
        null = self.dim.physical_null(c)
        codes = slot16_encode(self.jt, col, null, vmin)
        k, nl = self.probe.decode_outer(self.fact, self.outer_col)
        hit, d = self.probe.slot(self.jt, k[self.rows], nl[self.rows])
        out = np.full(self.rows.size, null, dtype=np.int64)
        if self.jt.entry_count:
            matched, vals = self.probe.slot16_decode(codes[d[hit]], vmin, null)
            sub = np.full(hit.sum(), null, dtype=np.int64)
            sub[matched] = vals[matched]
            out[hit] = sub
        return out.astype(col.dtype)

    def width(self, c: int, inner: bool) -> ix.Width:
        return width_of(self.dim if inner else self.fact, c)


def join(fact: abi.Table, dim: abi.Table, outer_col: int, inner_col: int, left: bool, probe: Probe | None = None) -> Joined:
    """One join level: fact.outer_col = dim.inner_col, INNER or LEFT."""
    probe = probe or Probe()
    jt = probe.build(dim, inner_col)
    k, null = probe.decode_outer(fact, outer_col)
    idx = probe.probe(jt, k, null)
    rows = np.arange(k.size) if left else np.flatnonzero(idx >= 0)
    return Joined(fact, dim, rows, idx[rows], left, jt, probe, outer_col)


def int_groups(j: Joined, key, arg_col: int, arg_inner: bool, mask=None, frag_rows=None) -> dict:
    """int_exact_ref groups of an integer argument over the joined rows.  key: None (non-grouped), ("outer", c) or
    ("inner", c); a NULL group key (an unmatched LEFT row grouped by an inner column) is the group None."""
    w = j.width(arg_col, arg_inner)
    vals = j.inner(arg_col) if arg_inner else j.outer(arg_col)
    nullable = j.left or not (j.dim if arg_inner else j.fact).col_types[arg_col][1]
    keys, knull = _keys(j, key)
    groups = ix.groups_of(w, keys, vals, nullable, mask=mask, frag_rows=frag_rows)
    return _rename_null(groups, knull)


def fp_groups(j: Joined, key, arg_col: int, mask=None) -> dict:
    """fp_exact_ref groups of a DOUBLE / FLOAT inner argument over the joined rows."""
    import fp_exact_ref as fx
    vals = j.inner(arg_col)
    keys, knull = _keys(j, key)
    return _rename_null(fx.groups_of(keys, vals, null=j.dim.physical_null(arg_col), mask=mask), knull)


def _keys(j: Joined, key):
    if key is None:
        return None, None
    side, c = key
    if side == "outer":
        return j.outer(c).astype(np.int64), None
    vals = j.inner(c).astype(np.int64)
    null = int(j.dim.physical_null(c))
    return vals, null if (j.left or not j.dim.col_types[c][1]) else None


def _rename_null(groups: dict, knull):
    if knull is None or knull not in groups:
        return groups
    groups[None] = groups.pop(knull)
    return groups


# ---- mutations: each restates one plausible probe bug -----------------------------------------------------------------------
class Trunc32(Probe):
    """The outer key compared in 32 bits: k mod 2^32 read as an int32."""

    def decode_outer(self, table, c):
        k, null = super().decode_outer(table, c)
        return k.astype(np.int32).astype(np.int64), null


class MinOffByOne(Probe):
    """slot = k - (min + 1)."""

    def slot(self, jt, k, null):
        hit = ~null & (k >= jt.min_key + 1) & (k <= jt.min_key + jt.entry_count)
        return hit, np.where(hit, k - np.where(hit, jt.min_key + 1, 0), 0)


class NullInnerMatches(Probe):
    """A NULL outer key matches the first inner row whose key is NULL."""

    def probe(self, jt, k, null):
        idx = super().probe(jt, k, null)
        if jt.null_rows.size:
            idx[null] = jt.null_rows[0]
        return idx


class FixedNullUndecoded(Probe):
    """The physical NULL of a FIXED(8|16|32) outer key read as the plain value (the type's minimum)."""

    def decode_outer(self, table, c):
        k, null = super().decode_outer(table, c)
        if table.encoded_sizes[c] > 0:
            null = np.zeros_like(null)
        return k, null


class Slot16Shifted(Probe):
    """uint16 slots decoded with only 0xFFFF special: 0xFFFE (NULL) reads as vmin + 0xFFFE."""

    def slot16_decode(self, codes, vmin, null):
        codes = codes.astype(np.int64)
        matched = codes != SLOT16_EMPTY
        return matched, np.where(codes >= SLOT16_EMPTY, null, vmin + codes)


MUTATIONS = [Trunc32, MinOffByOne, NullInnerMatches, FixedNullUndecoded, Slot16Shifted]


# ---- the layout rule, restated (planner.cpp choose_kernel / the join lines of the program lowering) ---------------------------
SMEM_ROOM = 216 * 1024          # of the 227 KB a CTA may opt in to
SLOT16_SPAN_LIMIT = 65534       # the value span must be below this (0xFFFE, 0xFFFF are the two codes)


def slot16_eligible(packed: bool, inner_cols_read: int, span: int | None) -> bool:
    """uint16 slots are possible when the packed column is the only inner column read and its chunk-stats span < 65534."""
    return packed and inner_cols_read == 1 and span is not None and 0 <= span < SLOT16_SPAN_LIMIT


def layout(entries: int, packed: bool, slot16_ok: bool, use_smem: bool, replica_bytes: int, replicas: int,
           stage: bool = True) -> tuple:
    """(JOIN_TABLE_* value, replicas left, staged bytes) for a join table of `entries` slots next to a group table of
    `replicas` copies of `replica_bytes` (use_smem = the group table is in shared memory at all)."""
    def try_stage(slot_bytes):
        jb = (entries * slot_bytes + 15) // 16 * 16
        rep = replicas
        if use_smem:
            while rep > 1 and replica_bytes * rep + jb + 128 > SMEM_ROOM:
                rep //= 2
        base = replica_bytes * rep if use_smem else 0
        off = (base + 127) // 128 * 128
        return (rep, jb) if off + jb <= SMEM_ROOM else None

    if stage and entries > 0:
        got = try_stage(8 if packed else 4)
        if got:
            return (abi.JOIN_TABLE_INT2_SMEM if packed else abi.JOIN_TABLE_INT32_SMEM), got[0], got[1]
        if slot16_ok:
            got = try_stage(2)
            if got:
                return abi.JOIN_TABLE_UINT16_SMEM, got[0], got[1]
    return (abi.JOIN_TABLE_INT2_HBM if packed else abi.JOIN_TABLE_INT32_HBM), replicas, 0


# ---- edge tables ---------------------------------------------------------------------------------------------------------------
# t: one outer key column per physical width (nullable, plus NOT NULL INT and FIXED(16)), a small group key x, a 1024-value
# group key g and a BIGINT value v.
FACT_KEYS = [("k8", abi.kTINYINT, 0, False), ("k16", abi.kSMALLINT, 0, False), ("k32", abi.kINT, 0, False),
             ("k64", abi.kBIGINT, 0, False), ("f8", abi.kINT, 1, False), ("f16", abi.kBIGINT, 2, False),
             ("f32", abi.kBIGINT, 4, False), ("k32nn", abi.kINT, 0, True), ("f16nn", abi.kBIGINT, 2, True)]
FACT_NAMES = [k[0] for k in FACT_KEYS] + ["x", "g", "v"]
KEY_NAMES = [k[0] for k in FACT_KEYS]
DIM_NAMES = ["id", "a", "b", "w"]
INT32_MIN, INT32_MAX = -(2 ** 31), 2 ** 31 - 1


@dataclass(frozen=True)
class Case:
    """One dimension shape, built to reach one join-table layout."""
    name: str
    layout: int                 # JOIN_TABLE_* of the queries that read `reads` of the inner table
    key_type: int               # inner key: abi.kINT or abi.kBIGINT
    key_min: int                # least inner key (the chunk stats may start lower: stats_pad)
    entries: int                # E of the chunk stats, stats_pad included
    packed: str = "INT8"        # int_exact_ref width of the inner attribute a
    span: int = 0               # a's non-NULL values lie in [a_lo, a_lo + span] with both ends present (0: the width's pool)
    reads_a: bool = True        # the case's queries read a (the packed column); else only b / w
    reads_b: bool = False       # ... and also the BIGINT b (no uint16 slots then)
    key_nullable: bool = True   # NULL inner keys (never matched)
    stats_pad: int = 0          # inner key chunk stats wider than the values by this on both sides


CASES = [
    Case("int32_smem", abi.JOIN_TABLE_INT32_SMEM, abi.kINT, -100, 2000, reads_a=False, reads_b=True),
    Case("int32_smem_multi_copy", abi.JOIN_TABLE_INT32_SMEM, abi.kINT, -100, 30001, reads_a=False, reads_b=True, stats_pad=2),
    Case("int32_hbm", abi.JOIN_TABLE_INT32_HBM, abi.kINT, -100, 80000, reads_a=False, reads_b=True),
    Case("int32_smem_fixed_nulls", abi.JOIN_TABLE_INT32_SMEM, abi.kINT, -32800, 33000, reads_a=False, reads_b=True),
    Case("int32_smem_near_int32_min", abi.JOIN_TABLE_INT32_SMEM, abi.kINT, INT32_MIN + 1, 3000, reads_a=False, reads_b=True),
    Case("int2_smem", abi.JOIN_TABLE_INT2_SMEM, abi.kINT, -100, 2000, packed="INT8"),
    Case("int2_smem_multi_copy", abi.JOIN_TABLE_INT2_SMEM, abi.kBIGINT, -100, 20001, packed="INT16", reads_b=True),
    Case("int2_smem_fixed16", abi.JOIN_TABLE_INT2_SMEM, abi.kINT, -100, 3000, packed="INT_FIXED16"),
    Case("int2_smem_near_int32_max", abi.JOIN_TABLE_INT2_SMEM, abi.kBIGINT, INT32_MAX - 2999, 3000, packed="INT32"),
    Case("int2_hbm", abi.JOIN_TABLE_INT2_HBM, abi.kINT, -100, 40000, packed="INT16", reads_b=True),
    Case("int2_hbm_span_65534", abi.JOIN_TABLE_INT2_HBM, abi.kINT, -100, 40000, packed="INT16", span=65534),
    Case("uint16_span_65533", abi.JOIN_TABLE_UINT16_SMEM, abi.kINT, -100, 60000, packed="INT16", span=65533),
    Case("uint16_int8", abi.JOIN_TABLE_UINT16_SMEM, abi.kBIGINT, -100, 50000, packed="INT8", stats_pad=3),
    Case("uint16_dict8", abi.JOIN_TABLE_UINT16_SMEM, abi.kINT, -100, 40000, packed="DICT8"),
    Case("uint16_fixed16", abi.JOIN_TABLE_UINT16_SMEM, abi.kINT, -100, 100000, packed="INT_FIXED16", span=65000,
         key_nullable=False),
]
CASE = {c.name: c for c in CASES}


def attr_values(case: Case, rng, n: int) -> np.ndarray:
    """Physical values of the inner attribute a: the width's pool (the NULL sentinel's neighbours, the extremes), or both ends
    of [lo, lo + span]; 10 % NULL."""
    w = ix.WIDTH[case.packed]
    if case.span:
        lo = w.lo
        p = np.array([lo, lo + 1, lo + case.span - 1, lo + case.span, 0, -1, 1], dtype=np.int64)
        p = p[(p >= lo) & (p <= lo + case.span)]
    else:
        p = np.array(ix.pool(w), dtype=np.int64)
    v = p[rng.integers(0, p.size, n)]
    v[: p.size] = p                                     # every pool value is present
    v[rng.random(n) < 0.1] = w.null
    v[p.size] = w.null
    return v.astype(w.dtype)


def dim_table(case: Case, seed: int = 0) -> abi.Table:
    """d(id, a, b, w): unique keys over [key_min, key_min + E - 2 pad) with holes (one in ten keys missing, never the two
    ends), NULL keys when nullable, a from attr_values, b sparse BIGINT, w DOUBLE; one fragment."""
    rng = np.random.default_rng(seed)
    e = case.entries - 2 * case.stats_pad
    keys = case.key_min + np.arange(e, dtype=np.int64)
    keep = rng.random(e) >= 0.1
    keep[0] = keep[-1] = True
    keys = rng.permutation(keys[keep])
    if case.key_nullable:
        keys = np.concatenate([keys, np.full(7, ix.WIDTH["INT32" if case.key_type == abi.kINT else "INT64"].null)])
    n = keys.size
    a = attr_values(case, rng, n)
    b = rng.integers(-10 ** 6, 10 ** 6, n).astype(np.int64) * 1_000_003
    b[rng.random(n) < 0.1] = abi.NULL_BIGINT
    w = rng.normal(0, 100, n)
    w[rng.random(n) < 0.1] = abi.NULL_DOUBLE
    wa = ix.WIDTH[case.packed]
    t = abi.Table([(case.key_type, not case.key_nullable), (wa.sql_type, False), (abi.kBIGINT, False), (abi.kDOUBLE, False)],
                  encoded_sizes=[0, wa.enc, 0, 0])
    t.add_host_fragment([keys.astype(np.int32 if case.key_type == abi.kINT else np.int64), a, b, w])
    st = t.fragments[0].stats[0]
    st.int_min, st.int_max = case.key_min - case.stats_pad, case.key_min + e - 1 + case.stats_pad
    return t


def outer_keys(case: Case, rng, n: int) -> np.ndarray:
    """Logical outer keys (Python ints): min - 1, min, min + 1, max, max + 1 = min + E, keys in holes and in range, keys
    congruent mod 2^32 to in-range keys, INT32_MIN / INT32_MAX and their neighbours, the narrow types' extremes."""
    lo, hi = case.key_min - case.stats_pad, case.key_min + case.entries - 1 - case.stats_pad
    edge = [lo - 1, lo, lo + 1, hi - 1, hi, hi + 1, case.key_min, case.key_min - 1, lo + 2 ** 32, hi - 2 ** 32, lo + 5 + 2 ** 32,
            INT32_MIN, INT32_MIN + 1, INT32_MAX, INT32_MAX + 1, -128, -127, 127, -32768, -32767, 32767, 0, -1]
    ks = np.array(edge, dtype=np.int64)[rng.integers(0, len(edge), n)]
    inner = rng.random(n) < 0.6
    ks[inner] = rng.integers(lo, hi + 1, int(inner.sum()))
    return ks


def fact_table(case: Case, n: int, frag_rows: int, seed: int = 1) -> abi.Table:
    """t(k8, k16, k32, k64, f8, f16, f32, k32nn, f16nn, x, g, v): every key column holds the same logical key where its width
    can (a nullable column gets NULL where it cannot, a NOT NULL one the width's nearest end), plus 5 % NULLs."""
    rng = np.random.default_rng(seed)
    logical = outer_keys(case, rng, n)
    t = abi.Table([(ty, nn) for _n, ty, _e, nn in FACT_KEYS] + [(abi.kINT, True), (abi.kINT, True), (abi.kBIGINT, False)],
                  encoded_sizes=[e for _n, _t, e, _nn in FACT_KEYS] + [0, 0, 0])
    cols = []
    nulls = rng.random(n) < 0.05
    for c, (_name, _ty, _enc, nn) in enumerate(FACT_KEYS):
        dt = t.physical_dtype(c)
        info = np.iinfo(dt)
        null = t.physical_null(c)
        lo, hi = info.min + 1, info.max
        fits = (logical >= lo) & (logical <= hi)
        k = np.clip(logical, lo, hi)
        if not nn:
            k = np.where(fits & ~nulls, k, null)
        cols.append(k.astype(dt))
    x = rng.integers(0, 16, n).astype(np.int32)
    g = rng.integers(0, 1024, n).astype(np.int32)
    v = np.array(ix.pool(ix.WIDTH["INT64"]), dtype=np.int64)[rng.integers(0, 16, n)]
    v[rng.random(n) < 0.1] = abi.NULL_BIGINT
    cols += [x, g, v]
    for b in range(0, n, frag_rows):
        t.add_host_fragment([c[b:b + frag_rows] for c in cols])
    return t
