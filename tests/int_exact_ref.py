"""Exact per-group integer aggregates and predicates in plain Python ints, the integer counterpart of fp_exact_ref.

The product adds 64-bit integers as a 32-bit low word plus a carry / high-word delta, in an order that changes from run to
run; integer addition mod 2^64 does not care about the order, so the exact answer is unique:

- COUNT(*) counts the group's rows that pass the filter, COUNT(col) its non-NULL values;
- SUM is the exact sum reduced mod 2^64 to a signed int64 (the reference's int64 adds wrap);
- MIN / MAX are exact;
- AVG is pair_to_double of (wrapped sum, count): double(sum) / double(count), DECIMAL dividing by count x 10^scale
  (ResultSetBufferAccessors.h:197-227);
- COUNT(DISTINCT) is the size of a set.

Predicates follow the reference's semantics in exact arithmetic: an integer column against an integer literal compares
Python ints; against a floating-point literal the reference casts the column to DOUBLE, so float(v) is compared; NULL
makes a comparison unknown (three-valued AND / OR / NOT); a days-encoded DATE is days x 86400 seconds.

The nullable form of an aggregate is the one of a nullable argument, and of every aggregate of a non-grouped query.  Two
behaviours of that form:
- COUNT32 (modelled exactly, IntGroup.count32): a COUNT(col) in its nullable form counts into 32 bits.  convertNullIfAny
  casts a nullable argument to int32 (the COUNT's type) and compares it with NULL_INT; a NOT NULL argument is compared
  uncast.  A value that then equals INT32_MIN is not counted (a BIGINT 2^31 or -2^31 of a nullable column, -2^31 of a NOT
  NULL one).  The kernels do the same (DevAcc.skip2_trunc32).
- SENTINEL_SUM (excluded by name, never by a tolerance): a SUM whose running sum equals INT64_MIN.  The reference's
  agg_sum_skip_val then takes the next value as if the group were empty, so the result depends on the order of the adds;
  IntGroup.sentinel_sum names the groups where a sequential executor meets it.  The product decides NULL by the non-NULL
  count (DESIGN.md section 6), so its SUM is the wrapped sum whatever the order, read as NULL only when it IS INT64_MIN.
Other edges are left out of the data:
- A NOT NULL column never holds its sentinel here: the reference reads it as NULL (test_reference_quirks pins that).
- A group key equal to EMPTY_KEY (INT64_MAX, or INT32_MAX in a 4-byte key slot) is never generated: it marks an empty entry.
Nothing here calls the oracle or the planner.
"""
from __future__ import annotations

import itertools
from dataclasses import dataclass, field

import numpy as np

from heavydb_b200 import abi

INT64_MIN, INT64_MAX = -(2 ** 63), 2 ** 63 - 1
SECONDS_PER_DAY = 86400


def wrap64(x: int) -> int:
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >> 63 else x


def pair_to_double(s: int, count: int, scale: int = 0):
    """AVG as the reference reads it; None for an empty pair."""
    if count == 0:
        return None
    return float(s) / (float(count) * 10.0 ** scale) if scale else float(s) / float(count)


# ---- physical widths ---------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Width:
    """One physical storage of an integer-like column: the SQL type, the encoded size abi.Table takes (0: none, 1 / 2 / 4:
    FIXED or DICT, -2 / -4: DATE ENCODING DAYS), and the DECIMAL scale."""
    name: str
    sql_type: int
    enc: int = 0
    scale: int = 0

    @property
    def bits(self) -> int:
        return 8 * abs(self.enc) if self.enc else 8 * abi.SIZE_OF[self.sql_type]

    @property
    def is_dict(self) -> bool:
        return self.sql_type in abi.STRING_TYPES

    @property
    def is_days(self) -> bool:
        return self.enc < 0

    @property
    def dtype(self):
        if self.is_dict and self.enc in (1, 2):
            return {1: np.uint8, 2: np.uint16}[self.enc]
        return {8: np.int8, 16: np.int16, 32: np.int32, 64: np.int64}[self.bits]

    @property
    def null(self) -> int:
        """The physical NULL sentinel: the unsigned maximum of a DICT(8|16) id, else the signed minimum."""
        if self.is_dict and self.enc in (1, 2):
            return 2 ** self.bits - 1
        return -(2 ** (self.bits - 1))

    @property
    def lo(self) -> int:
        """The least physical value that is not NULL."""
        return 0 if self.is_dict and self.enc in (1, 2) else self.null + 1

    @property
    def hi(self) -> int:
        return self.null - 1 if self.is_dict and self.enc in (1, 2) else 2 ** (self.bits - 1) - 1

    def logical(self, phys: int) -> int:
        return phys * SECONDS_PER_DAY if self.is_days else phys

    @property
    def summable(self) -> bool:
        return not (self.is_dict or self.is_days)

    def table(self, notnull: bool) -> abi.Table:
        """t(k INT NOT NULL, v <this width>)."""
        return abi.Table([(abi.kINT, True), (self.sql_type, notnull)], encoded_sizes=[0, self.enc],
                         col_scales={1: self.scale} if self.scale else None)


WIDTHS = [
    Width("INT8", abi.kTINYINT), Width("INT16", abi.kSMALLINT), Width("INT32", abi.kINT), Width("INT64", abi.kBIGINT),
    Width("INT_FIXED8", abi.kINT, 1), Width("INT_FIXED16", abi.kINT, 2),
    Width("BIGINT_FIXED8", abi.kBIGINT, 1), Width("BIGINT_FIXED16", abi.kBIGINT, 2), Width("BIGINT_FIXED32", abi.kBIGINT, 4),
    Width("DICT8", abi.kTEXT, 1), Width("DICT16", abi.kTEXT, 2),
    Width("DAYS16", abi.kDATE, -2), Width("DAYS32", abi.kDATE, -4),
    Width("DECIMAL18_2", abi.kDECIMAL, 0, 2),
]
WIDTH = {w.name: w for w in WIDTHS}
DECIMAL18_MAX = 10 ** 18 - 1

# the edges every width is drawn from, where the width can hold them
EDGES = [-(2 ** 31), -(2 ** 31) + 1, -1, 0, 1, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1, 2 ** 32, 2 ** 53, 2 ** 53 + 1, 2 ** 62,
         INT64_MAX, -INT64_MAX, 254, 65534]


def pool(w: Width) -> list:
    """Physical non-NULL values: the type's min + 1 and min + 2 (the NULL sentinel's neighbours), max - 1 and max, and every
    edge the width can hold (DECIMAL(18, s): at most 18 digits)."""
    hi = min(w.hi, DECIMAL18_MAX) if w.sql_type == abi.kDECIMAL else w.hi
    lo = max(w.lo, -DECIMAL18_MAX) if w.sql_type == abi.kDECIMAL else w.lo
    vals = {lo, lo + 1, hi - 1, hi} | {e for e in EDGES if lo <= e <= hi}
    return sorted(vals)


def carry_value(w: Width) -> int:
    """The value whose low 32-bit word is largest: 2^32 - 1 where the width holds it, else -1 (sign-extended, 0xFFFFFFFF)."""
    return 2 ** 32 - 1 if w.lo <= 2 ** 32 - 1 <= w.hi else -1 if w.lo <= -1 else w.hi


# ---- datasets: (keys, physical values) with keys in [0, 64) ------------------------------------------------------------------
def _pool_rows(w, rng, rows):
    p = np.array(pool(w), dtype=object)
    return rng.integers(0, 64, rows), p[rng.integers(0, p.size, rows)]


def _carry_dense(w, rng, rows):
    return rng.integers(0, 64, rows), np.array([carry_value(w)] * rows, dtype=object)


def _wrap_to_zero(w, rng, rows):
    """Groups whose values sum to 0 mod 2^64 (exactly 0 where the width cannot reach 2^64): x, y and -(x + y) mod 2^64."""
    p = pool(w)
    keys, vals = [], []
    g = 0
    while len(vals) < rows:
        x, y = p[rng.integers(len(p))], p[rng.integers(len(p))]
        z = wrap64(-(x + y))
        if not (w.lo <= z <= w.hi) or (w.sql_type == abi.kDECIMAL and abs(z) > DECIMAL18_MAX) or x == y == 0:
            continue
        keys += [g % 64] * 3
        vals += [x, y, z]
        g += 1
    return np.array(keys[:rows - rows % 3]), np.array(vals[:rows - rows % 3], dtype=object)


def _cancelling(w, rng, rows):
    """+-m pairs, m the largest magnitude both signs hold (+-(2^63 - 1) for 64 bits), on both orders."""
    m = min(w.hi, -w.lo, DECIMAL18_MAX if w.sql_type == abi.kDECIMAL else w.hi)
    keys = rng.integers(0, 64, rows // 2)
    sign = rng.integers(0, 2, rows // 2) * 2 - 1
    vals = np.stack([sign * m, -sign * m], axis=1).reshape(-1).astype(object)
    return np.repeat(keys, 2), vals


DATASETS = {"pool": _pool_rows, "carry_dense": _carry_dense, "wrap_to_zero": _wrap_to_zero, "cancelling": _cancelling}


def dataset_names(w: Width) -> list:
    """Sums are only defined where SUM is: DICT ids and DAYS dates take the pool only."""
    return list(DATASETS) if w.summable else ["pool"]


def make_dataset(w: Width, name: str, rows: int, nullable: bool, seed: int = 0, p_null: float = 0.1):
    """(keys int32, physical values as w.dtype).  A nullable column gets NULLs with probability p_null and one group (key 63)
    of NULL only; a NOT NULL column never holds its sentinel."""
    rng = np.random.default_rng(seed)
    keys, vals = DATASETS[name](w, rng, rows)
    phys = np.array([int(v) for v in vals], dtype=w.dtype) if len(vals) else np.zeros(0, w.dtype)
    keys = np.asarray(keys, dtype=np.int32)
    if nullable:
        phys[rng.random(phys.size) < p_null] = w.null
        phys[keys == 63] = w.null
    return keys, phys


# ---- per-group reference ------------------------------------------------------------------------------------------------------
@dataclass
class IntGroup:
    values: list                    # logical non-NULL values, Python ints, in row order
    rows: int                       # COUNT(*)
    prefix_sums: set = field(default_factory=set)   # every running sum a sequential executor can meet (see sentinel_sum)
    skip_form: bool = False                          # the nullable form of the aggregates (module docstring)
    nullable: bool = False

    @property
    def count(self) -> int:
        return len(self.values)

    @property
    def sum(self):
        return wrap64(sum(self.values)) if self.values else None

    @property
    def min(self):
        return min(self.values) if self.values else None

    @property
    def max(self):
        return max(self.values) if self.values else None

    def avg(self, scale: int = 0):
        return pair_to_double(self.sum, self.count, scale) if self.values else None

    @property
    def count32(self) -> int:
        """COUNT(col) into a 32-bit count (the module docstring's COUNT32)."""
        if not self.skip_form:
            return self.count
        return sum(1 for v in self.values if (_int32(v) if self.nullable else v) != -(2 ** 31))

    @property
    def count_distinct(self) -> int:
        return len(set(self.values))

    @property
    def sentinel_sum(self) -> bool:
        """SENTINEL_SUM: the wrapped sum, or a running sum of a sequential executor, equals INT64_MIN."""
        return self.sum == INT64_MIN or INT64_MIN in self.prefix_sums


def _int32(x: int) -> int:
    x &= 0xFFFFFFFF
    return x - (1 << 32) if x >> 31 else x


def groups_of(w: Width, keys, phys, nullable: bool, mask=None, frag_rows=None) -> dict:
    """{key: IntGroup} over the rows where `mask` holds; keys None = one group (key None), whose aggregates take their
    nullable form.  frag_rows: the fragment size the table was cut into, so that the running sums of each fragment and of
    the fragments' reduction are recorded."""
    skip_form = nullable or keys is None
    phys = np.asarray(phys)
    n = phys.size
    mask = np.ones(n, bool) if mask is None else np.asarray(mask)
    ks = np.zeros(n, np.int64) if keys is None else np.asarray(keys).astype(np.int64)
    out = {}
    frag = np.arange(n) // (frag_rows or max(n, 1))
    sel = np.flatnonzero(mask)
    order = sel[np.argsort(ks[sel], kind="stable")]                   # grouped, each group in row order
    bounds = np.flatnonzero(np.diff(ks[order])) + 1
    for a, b in zip(np.r_[0, bounds], np.r_[bounds, order.size]) if order.size else []:
        idx = order[a:b]
        k = ks[idx[0]]
        vals = [int(v) for v in phys[idx]]
        nn = [(f, w.logical(v)) for f, v in zip(frag[idx], vals) if not (nullable and v == w.null)]
        g = IntGroup([v for _f, v in nn], int(idx.size), skip_form=skip_form, nullable=nullable)
        if skip_form and w.summable:
            for _f, part in itertools.groupby(nn, key=lambda t: t[0]):
                g.prefix_sums |= {wrap64(s) for s in itertools.accumulate(v for _f, v in part)}
            g.prefix_sums |= {wrap64(s) for s in itertools.accumulate(v for _f, v in nn)}
        out[None if keys is None else int(k)] = g
    if keys is None and not out:
        out[None] = IntGroup([], 0, skip_form=True, nullable=nullable)
    return out


# ---- predicates: three-valued, exact ------------------------------------------------------------------------------------------
# a predicate on the one column v: ("cmp", op, literal) | ("in", [literals]) | ("between", lo, hi) | ("isnull",)
# | ("not", p) | ("and", p, q) | ("or", p, q); literals are Python ints (exact) or floats (the column is cast to DOUBLE)
_CMP = {"=": lambda a, b: a == b, "<>": lambda a, b: a != b, "<": lambda a, b: a < b, ">": lambda a, b: a > b,
        "<=": lambda a, b: a <= b, ">=": lambda a, b: a >= b}


def _not(x):
    return None if x is None else not x


def _and(x, y):
    if x is False or y is False:
        return False
    return None if x is None or y is None else True


def _or(x, y):
    if x is True or y is True:
        return True
    return None if x is None or y is None else False


def evaluate(p, v):
    """True / False / None (unknown) for the logical value v (None = NULL)."""
    kind = p[0]
    if kind == "isnull":
        return v is None
    if kind == "not":
        return _not(evaluate(p[1], v))
    if kind in ("and", "or"):
        return (_and if kind == "and" else _or)(evaluate(p[1], v), evaluate(p[2], v))
    if kind == "in":
        r = False
        for lit in p[1]:
            r = _or(r, evaluate(("cmp", "=", lit), v))
        return r
    if kind == "between":
        return _and(evaluate(("cmp", ">=", p[1]), v), evaluate(("cmp", "<=", p[2]), v))
    op, lit = p[1], p[2]
    if v is None:
        return None
    return _CMP[op](float(v), lit) if isinstance(lit, float) else _CMP[op](v, lit)


def passing(w: Width, phys, nullable: bool, p) -> np.ndarray:
    """Rows where the predicate is TRUE (WHERE drops unknown)."""
    out = np.zeros(len(phys), bool)
    for i, x in enumerate(phys):
        x = int(x)
        out[i] = evaluate(p, None if nullable and x == w.null else w.logical(x)) is True
    return out


def literal_sql(w: Width, lit) -> str:
    """The SQL text of a literal compared with a column of width w: DECIMAL literals carry the scale's fraction digits,
    fp literals a decimal point."""
    if isinstance(lit, float):
        return repr(lit) if "e" not in repr(lit) else f"{lit:.1f}"
    if w.scale:
        s = str(abs(lit)).rjust(w.scale + 1, "0")
        return f"{'-' if lit < 0 else ''}{s[:-w.scale]}.{s[-w.scale:]}"
    return str(lit)


def predicate_sql(w: Width, p, col="v") -> str:
    kind = p[0]
    if kind == "isnull":
        return f"{col} IS NULL"
    if kind == "not":
        return f"NOT ({predicate_sql(w, p[1], col)})"
    if kind in ("and", "or"):
        return f"({predicate_sql(w, p[1], col)}) {kind.upper()} ({predicate_sql(w, p[2], col)})"
    if kind == "in":
        return f"{col} IN ({', '.join(literal_sql(w, x) for x in p[1])})"
    if kind == "between":
        return f"{col} BETWEEN {literal_sql(w, p[1])} AND {literal_sql(w, p[2])}"
    return f"{col} {p[1]} {literal_sql(w, p[2])}"


def edge_literals(w: Width) -> list:
    """Integer literals at the width's edges, in the column's logical unit (seconds for DAYS, scaled units for DECIMAL):
    type min - 1, min (the sentinel), sentinel + 1, max, max + 1, 2^31 +- 1, 2^32, 2^53 +- 1, INT64_MIN / INT64_MAX; DAYS
    also a second on either side of each day; then k + 0.5 and 2^53 + 1 as fp literals (not against DECIMAL, whose literals are
    scaled integers, nor against dictionary ids or days-encoded dates, which refuse them)."""
    unit = SECONDS_PER_DAY if w.is_days else 1
    phys = {w.lo - 2, w.lo - 1, w.null, w.null + 1, w.lo, w.lo + 1, w.hi, w.hi + 1, 0, 1, -1}
    ints = {x * unit for x in phys}
    if w.is_days:
        ints |= {x * unit + d for x in (w.lo, w.hi, -1, 0, 1) for d in (-1, 1)}
    ints |= {2 ** 31 - 1, 2 ** 31 + 1, -(2 ** 31) + 1, -(2 ** 31) - 1, 2 ** 32, 2 ** 53 - 1, 2 ** 53 + 1, INT64_MIN, INT64_MAX}
    if w.scale:   # the scaled literal must fit int64 and the column's 18 digits of precision are the interesting edge
        ints = {x for x in ints if abs(x) <= DECIMAL18_MAX} | {DECIMAL18_MAX, -DECIMAL18_MAX, DECIMAL18_MAX + 1}
    ints = sorted(x for x in ints if INT64_MIN <= x <= INT64_MAX)
    fps = [] if w.scale or w.is_dict or w.is_days else sorted({w.lo * unit - 0.5, w.hi * unit + 0.5, -0.5, 0.5, 1.5, float(2 ** 53 + 1), float(2 ** 31) - 0.5})
    return ints + fps
