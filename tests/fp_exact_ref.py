"""Exact per-group floating-point aggregates and the error each can carry after IEEE double summation in ANY order.

The product adds doubles with round-to-nearest f64 adds (`red/atom .add.f64`, shared-memory atomics, warp shuffles, NCCL sum)
in an order and a tree that change from run to run.  Whatever the order, with u = 2^-53 and g(k) = k u / (1 - k u), the
computed sum s^ of n values obeys |s^ - s| <= g(n - 1) * sum|x| (Higham, Accuracy and Stability of Numerical Algorithms,
eq. 4.4), where s is the exact sum.  The functions here compare a result with the exact value under that bound:

- DOUBLE SUM: |s^ - s| <= g(n-1) sum|x| + ulp(s)/2  (the extra half ulp: s itself is the correctly rounded math.fsum).
- DOUBLE AVG: the SUM bound / n + u |avg| (one division).
- FLOAT SUM: the DOUBLE SUM bound + ulp_f32(s^)/2 (the accumulator is a double of the exactly widened floats, narrowed once).
- FLOAT AVG: the FLOAT SUM read back as a float, divided by the integer count in double: the FLOAT SUM bound / n + u |avg|.

Special values follow the reference's agg_*_double / agg_*_float[_skip_val] (RuntimeFunctions.cpp:1444-1520, :1558-1593):
any NaN makes SUM / AVG NaN, +inf with -inf makes NaN; MIN / MAX never pick a NaN while a number is there, and a group of
NaN only ends at NaN (nullable: the first value is assigned) or at the slot's init value (NOT NULL: std::min(DBL_MAX, NaN),
which also keeps a NOT NULL MIN of +inf at DBL_MAX);
COUNT(col) counts NaN; the sign of a zero MIN / MAX depends on arrival order and either is accepted; a result equal to the
NULL sentinel (DBL_MIN, FLT_MIN) reads as NULL.  Nothing here calls the oracle.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from fractions import Fraction

import numpy as np

U = 2.0 ** -53
DBL_MAX = float(np.finfo(np.float64).max)
FLT_MAX = float(np.finfo(np.float32).max)
NULL_DOUBLE = float(np.finfo(np.float64).tiny)
NULL_FLOAT = float(np.finfo(np.float32).tiny)
# the least exact sum whose float rounding is +inf: FLT_MAX + ulp_f32(FLT_MAX) / 2
FLT_OVERFLOW = FLT_MAX + 2.0 ** 103


def gamma(k: int) -> float:
    k = max(k, 0)
    return k * U / (1.0 - k * U)


def ulp(x: float) -> float:
    return math.ulp(x)


def ulp32(x: float) -> float:
    """ulp of the float32 nearest x (its spacing; the largest finite float's for infinities)."""
    a = abs(float(np.float32(x))) if math.isfinite(x) else FLT_MAX
    return float(np.spacing(np.float32(min(a, FLT_MAX))))


@dataclass
class Group:
    """The non-NULL values one group aggregates (float64; FLOAT values widened exactly) and its row count."""
    values: np.ndarray
    rows: int                       # COUNT(*): rows of the group that pass the filter, NULL values included

    @property
    def n(self) -> int:             # COUNT(col): NaN is not NULL
        return int(self.values.size)

    @property
    def has_nan(self) -> bool:
        return bool(np.isnan(self.values).any())

    def _finite(self):
        v = self.values
        return v[np.isfinite(v)]

    @property
    def exact(self) -> Fraction:
        """The exact sum of the finite values."""
        return sum((Fraction(float(x)) for x in self._finite()), Fraction(0))

    @property
    def exact_sum(self) -> float:
        """The IEEE result an exact summation rounds to: NaN, +-inf, or the correctly rounded sum (+-inf past DBL_MAX)."""
        v = self.values
        if self.has_nan or ((v == np.inf).any() and (v == -np.inf).any()):
            return math.nan
        if (v == np.inf).any():
            return math.inf
        if (v == -np.inf).any():
            return -math.inf
        try:
            return math.fsum(self._finite())
        except OverflowError:
            return math.inf if self.exact > 0 else -math.inf

    @property
    def abs_sum(self) -> float:
        f = self._finite()
        try:
            return math.fsum(np.abs(f))
        except OverflowError:
            return math.inf

    @property
    def sum_bound(self) -> float:
        """Largest |s^ - s| any order of n - 1 double additions can give, s the rounded exact sum."""
        s = self.exact_sum
        return gamma(self.n - 1) * self.abs_sum + (0.5 * ulp(s) if math.isfinite(s) else 0.0)

    def minmax(self, is_min: bool, nullable: bool, as_float: bool = False):
        """MIN / MAX as the reference gives them when no NaN is the group's first value (see the module docstring)."""
        v = self.values
        if v.size == 0:
            return None
        num = v[~np.isnan(v)]
        big = FLT_MAX if as_float else DBL_MAX
        if num.size == 0:
            return math.nan if nullable else (big if is_min else -big)
        r = float(num.min() if is_min else num.max())
        if not nullable:                 # agg_min_double starts from DBL_MAX: +inf never beats it (MAX: -DBL_MAX, -inf)
            r = min(r, big) if is_min else max(r, -big)
        return None if r == (NULL_FLOAT if as_float else NULL_DOUBLE) else r


def groups_of(keys, values, null=None, mask=None) -> dict:
    """{key: Group} over the rows where `mask` holds; `keys` None = one group (non-grouped, key None).  Values equal to
    `null` (the column's NULL sentinel, compared as the reference does: `val != skip_val`) are not aggregated."""
    values = np.asarray(values)
    if mask is None:
        mask = np.ones(values.size, dtype=bool)
    vals = values[mask].astype(np.float64)
    ks = np.zeros(vals.size, dtype=np.int64) if keys is None else np.asarray(keys)[mask]
    out = {}
    if vals.size == 0:
        return out if keys is not None else {None: Group(np.zeros(0), 0)}
    order = np.argsort(ks, kind="stable")
    ks, vals = ks[order], vals[order]
    bounds = np.flatnonzero(np.diff(ks)) + 1
    for a, b in zip(np.r_[0, bounds], np.r_[bounds, ks.size]):
        g = vals[a:b]
        nn = g if null is None else g[g != float(null)]
        out[None if keys is None else int(ks[a])] = Group(nn, int(b - a))
    return out


# ---- checks: each returns None when `got` is acceptable, else a message ------------------------------------------------------
def _special(got, want):
    """NaN / inf / NULL agreement; returns (done, message)."""
    if want is None or got is None:
        return True, None if want is None and got is None else f"NULL mismatch: got {got!r}, want {want!r}"
    if math.isnan(want) or math.isnan(got):
        return True, None if math.isnan(want) and math.isnan(got) else f"NaN mismatch: got {got!r}, want {want!r}"
    return False, None


def check_double_sum(got, g: Group):
    s = g.exact_sum
    want = None if g.n == 0 else s
    done, msg = _special(got, want)
    if done:
        return msg
    if math.isinf(s):
        return None if got == s else f"got {got!r}, want {s!r}"
    b = g.sum_bound
    if math.isinf(got) and b != math.inf:
        return f"got {got!r}, want {s!r} +- {b:.3g}"
    if got == 0.0 and s == 0.0:          # either sign of zero (the nullable reference assigns its first value: -0.0 stays)
        return None
    if abs(got - s) <= b and not (got == NULL_DOUBLE):
        return None
    return f"got {got!r}, want {s!r} +- {b:.3g} (off by {abs(got - s):.3g})"


def check_double_avg(got, g: Group):
    if g.n == 0:
        return None if got is None else f"got {got!r}, want NULL"
    s = g.exact_sum
    avg = s / g.n if math.isfinite(s) else s
    done, msg = _special(got, None if avg == NULL_DOUBLE else avg)
    if done:
        return msg
    if math.isinf(avg):
        return None if got == avg else f"got {got!r}, want {avg!r}"
    b = g.sum_bound / g.n + U * abs(avg)
    if (got == 0.0 and avg == 0.0) or abs(got - avg) <= b:
        return None
    return f"AVG got {got!r}, want {avg!r} +- {b:.3g}"


def float_sum_interval(g: Group):
    """(exact double sum s, bound on |narrow(s^) - s|) of a FLOAT SUM, before the narrowing's own half ulp."""
    return g.exact_sum, g.sum_bound


def check_float_sum(got, g: Group):
    s, b = float_sum_interval(g)
    want = None if g.n == 0 else s
    done, msg = _special(got, want)
    if done:
        return msg
    if math.isinf(got) or math.isinf(s):
        # the double sum rounds to a float past FLT_MAX exactly when |s^| >= FLT_MAX + ulp/2
        can_overflow = abs(s) + b >= FLT_OVERFLOW
        must_overflow = abs(s) - b >= FLT_OVERFLOW
        if math.isinf(got):
            return None if can_overflow and math.copysign(1, got) == math.copysign(1, s) else f"got {got!r}, want {s!r} +- {b:.3g}"
        return None if not must_overflow and abs(got - s) <= b + 0.5 * ulp32(got) else f"got {got!r}, want {s!r} (overflow)"
    if got == 0.0 and s == 0.0:
        return None
    tol = b + 0.5 * ulp32(got)
    if abs(got - s) <= tol and got != NULL_FLOAT:
        return None
    return f"FLOAT SUM got {got!r}, want {s!r} +- {tol:.3g} (off by {abs(got - s):.3g})"


def check_float_avg(got, g: Group):
    """pair_to_double of a FLOAT AVG: the float sum read back as a float, divided by the count in double."""
    if g.n == 0:
        return None if got is None else f"got {got!r}, want NULL"
    s, b = float_sum_interval(g)
    done, msg = _special(got, s)
    if done:
        return msg
    if math.isinf(got) or math.isinf(s):
        return check_float_sum(got * g.n if math.isfinite(got) else got, g)
    avg = s / g.n
    tol = (b + 0.5 * ulp32(got * g.n)) / g.n + U * abs(avg)
    if (got == 0.0 and avg == 0.0) or abs(got - avg) <= tol:
        return None
    return f"FLOAT AVG got {got!r}, want {avg!r} +- {tol:.3g}"


def check_minmax(got, g: Group, is_min: bool, nullable: bool, as_float: bool = False):
    want = g.minmax(is_min, nullable, as_float)
    done, msg = _special(got, want)
    if done:
        return msg
    if got == want:                      # == : -0.0 == +0.0, either sign accepted
        return None
    return f"{'MIN' if is_min else 'MAX'} got {got!r}, want {want!r}"


def sensitive(g: Group, as_float: bool = False) -> bool:
    """True when one dropped, duplicated or sign-flipped value moves any acceptable result out of the bound: the bound (and,
    for FLOAT, the narrowing's half ulp) stays below half the smallest non-zero |x|."""
    v = np.abs(g.values[g.values != 0])
    if v.size == 0 or not math.isfinite(g.exact_sum):
        return False
    tol = g.sum_bound + (0.5 * ulp32(g.exact_sum + float(v.max())) if as_float else 0.0)
    return 2 * tol < float(v.min())


# ---- datasets shared by the CPU proofs of the bound and the GPU tests ----------------------------------------------------------
# name -> (rows, groups, builder(rng, rows) -> values, sql type, sensitive).  `sensitive`: every group must satisfy sensitive();
# the cancellation sets are bound-only.
def _pos12(rng, n):
    return 1.0 + rng.random(n)


def _pos2e20(rng, n):
    return (1.0 + rng.random(n)) * 2.0 ** 20


def _cancel(rng, n):
    v = rng.integers(-3, 4, n).astype(np.float64)
    big = rng.random(n) < 0.02
    v[big] = np.where(rng.random(int(big.sum())) < 0.5, -1e16, 1e16)
    return v


def _f32_pos(rng, n):
    return (1.0 + rng.random(n)).astype(np.float32)


def _f32_subnormal(rng, n):
    """subnormal floats (as little as 2^-149 apart) whose sums cross into the normal range at 2^-126"""
    return (rng.integers(2 ** 19, 2 ** 23, n).astype(np.float64) * 2.0 ** -149).astype(np.float32)


def _f32_mixed(rng, n):
    return (rng.random(n) * 8 - 1).astype(np.float32)


DATASETS = {
    "pos12": (1 << 20, 64, _pos12, "DOUBLE", True),
    "pos2e20": (1 << 20, 64, _pos2e20, "DOUBLE", True),
    "cancel": (1 << 18, 16, _cancel, "DOUBLE", False),
    "f32_pos": (1 << 18, 32, _f32_pos, "FLOAT", True),
    "f32_subnormal": (1 << 16, 64, _f32_subnormal, "FLOAT", True),
    "f32_mixed": (1 << 17, 8, _f32_mixed, "FLOAT", False),
}


def make_dataset(name, seed=0):
    """(keys int32 in [0, groups), values) of DATASETS[name]."""
    rows, groups, build, _ty, _sens = DATASETS[name]
    rng = np.random.default_rng(seed)
    return rng.integers(0, groups, rows).astype(np.int32), build(rng, rows)
