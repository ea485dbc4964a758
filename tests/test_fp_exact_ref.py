"""The exact floating-point reference (fp_exact_ref) on the CPU: its bound holds for every summation order the GPU can take,
it is tight enough that one dropped, duplicated or sign-flipped row fails it, and its special-value rules are the
reference's, as the oracle (the reference restated) executes them."""
import math

import numpy as np
import pytest

import fp_exact_ref as fx
import oracle_lib
import sqlmini
from heavydb_b200 import abi

NAN, INF = math.nan, math.inf


def warp_tree(lanes: np.ndarray) -> np.ndarray:
    """warp_sum_f64's butterfly: v += shfl_xor(v, o) for o = 16, 8, 4, 2, 1 over [..., 32] lane values."""
    v = lanes.copy()
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., idx ^ o]
    return v[..., 0]


def gpu_like_sum(x: np.ndarray, rng, replicas=4, ctas=7) -> float:
    """Rows dealt to CTAs, inside a CTA to warps of 32 lanes; every lane adds its rows in turn, a warp reduces with the
    butterfly, warps add into one of `replicas` shared-memory tables, replicas are flushed into the global slot, CTAs in a
    random order."""
    pad = (-x.size) % (32 * ctas)
    xs = np.concatenate([x, np.zeros(pad)]).reshape(ctas, -1, 32)          # [cta, row step, lane]
    total = 0.0
    for c in rng.permutation(ctas):
        lane_sums = np.cumsum(xs[c], axis=0)[-1] if xs.shape[1] else np.zeros(32)
        reps = np.zeros(replicas)
        steps = xs[c].shape[0]
        for w, chunk in enumerate(np.array_split(np.arange(steps), 3)):     # three warps take turns at the rows
            if chunk.size:
                reps[w % replicas] += warp_tree(np.cumsum(xs[c][chunk], axis=0)[-1])
        del lane_sums
        s = 0.0
        for r in reps:
            s += r
        total += s
    return total


def orders(x: np.ndarray, rng):
    yield "sequential", np.cumsum(x)[-1]
    yield "reversed", np.cumsum(x[::-1])[-1]
    for i in range(3):
        yield f"random{i}", np.cumsum(rng.permutation(x))[-1]
    yield "pairwise", np.add.reduce(x)
    yield "blocked", np.cumsum(np.add.reduce(x[: x.size // 256 * 256].reshape(-1, 256), axis=1))[-1] + np.sum(x[x.size // 256 * 256:])
    yield "gpu_like", gpu_like_sum(x, rng)


@pytest.mark.parametrize("name", sorted(fx.DATASETS))
def test_bound_holds_in_every_order(name):
    keys, vals = fx.make_dataset(name)
    is_float = fx.DATASETS[name][3] == "FLOAT"
    rng = np.random.default_rng(1)
    for k, g in fx.groups_of(keys, vals).items():
        for how, s in orders(g.values, rng):
            s = float(s)
            assert fx.check_double_sum(s, g) is None, (name, k, how, fx.check_double_sum(s, g))
            assert fx.check_double_avg(s / g.n, g) is None, (name, k, how)
            if is_float:
                f = float(np.float32(s))
                assert fx.check_float_sum(f, g) is None, (name, k, how, fx.check_float_sum(f, g))
                assert fx.check_float_avg(f / g.n, g) is None, (name, k, how)


def test_bound_holds_for_one_hot_group_of_16m_rows():
    """The largest GPU case: one group of 1.6e7 values in [1, 2) — the bound stays under half the smallest value."""
    rng = np.random.default_rng(2)
    x = 1.0 + rng.random(16_000_000)
    g = fx.Group(x, x.size)
    assert fx.sensitive(g)
    for how, s in [("sequential", np.cumsum(x)[-1]), ("pairwise", np.add.reduce(x)),
                   ("reversed", np.cumsum(x[::-1])[-1])]:
        assert fx.check_double_sum(float(s), g) is None, how
    assert fx.check_double_sum(float(np.add.reduce(x[1:])), g) is not None   # one row dropped
    assert fx.check_double_sum(float(np.add.reduce(x) + x[7]), g) is not None  # one row twice


@pytest.mark.parametrize("name", sorted(n for n, d in fx.DATASETS.items() if d[4]))
def test_bound_is_tight_enough_to_see_one_row(name):
    """Every group of the non-cancellation datasets: dropping, duplicating or sign-flipping any single value (the smallest
    one, the hardest to see) fails the check, whatever order the mutated values are added in."""
    keys, vals = fx.make_dataset(name)
    is_float = fx.DATASETS[name][3] == "FLOAT"
    rng = np.random.default_rng(3)
    check = fx.check_float_sum if is_float else fx.check_double_sum
    for k, g in fx.groups_of(keys, vals).items():
        assert fx.sensitive(g, as_float=is_float), (name, k)
        i = int(np.argmin(np.abs(g.values)))
        flipped = g.values.copy()
        flipped[i] = -flipped[i]
        for what, x in [("dropped", np.delete(g.values, i)), ("duplicated", np.append(g.values, g.values[i])), ("flipped", flipped)]:
            for how, s in orders(x, rng):
                s = float(np.float32(s)) if is_float else float(s)
                assert check(s, g) is not None, (name, k, what, how)


def test_cancellation_is_bound_only():
    keys, vals = fx.make_dataset("cancel")
    assert not all(fx.sensitive(g) for g in fx.groups_of(keys, vals).values())


def test_chunk_stats_ignore_nan():
    """FixedLengthEncoder / NoneEncoder keep std::min(dataMin, v): a NaN never becomes a chunk's min or max."""
    a = np.array([3.0, NAN, -2.0, abi.NULL_DOUBLE, NAN])
    st = abi.chunk_stats(a, abi.kDOUBLE, notnull=False)
    assert (st.fp_min, st.fp_max, st.has_nulls) == (-2.0, 3.0, 1)
    st = abi.chunk_stats(np.array([NAN, NAN]), abi.kDOUBLE, notnull=True)
    assert (st.fp_min, st.fp_max) == (fx.DBL_MAX, -fx.DBL_MAX)           # as if empty: the encoder's initial values
    st = abi.chunk_stats(np.array([NAN, 1.5, NAN], dtype=np.float32), abi.kFLOAT, notnull=True)
    assert (st.fp_min, st.fp_max) == (1.5, 1.5)


def test_chunk_stats_with_nan_keep_the_keyless_marker():
    """The planner picks MIN(v) as the keyless marker from the chunk's max; NaN stats made it fall back."""
    from heavydb_b200 import executor
    t = abi.Table([(abi.kINT, True), (abi.kDOUBLE, True)])
    t.add_host_fragment([np.array([0, 1, 1], dtype=np.int32), np.array([1.0, NAN, 2.0])])
    unit = sqlmini.parse("SELECT k, MIN(v) FROM t GROUP BY k;", t, ["k", "v"])
    p = executor.Executor().plan(unit, t)
    assert p.as_dict() == oracle_lib.plan(unit, t).as_dict()
    assert p.keyless_hash


# ---- special values: the module's rules against the oracle -------------------------------------------------------------------
NEXT_DN = float(np.nextafter(fx.NULL_DOUBLE, 0))
NEXT_UP = float(np.nextafter(fx.NULL_DOUBLE, 1))
NEXT_FDN = float(np.nextafter(np.float32(fx.NULL_FLOAT), np.float32(0)))
NEXT_FUP = float(np.nextafter(np.float32(fx.NULL_FLOAT), np.float32(1)))
QNAN, NEG_NAN = NAN, -NAN
PAYLOAD_NAN = float(np.array([0x7FF800000000BEEF], dtype=np.int64).view(np.float64)[0])

# group -> values in arrival order.  No group starts with a NaN followed by a number (see the leading-NaN test below).
SPECIAL_DOUBLE = {
    0: [QNAN, QNAN],                     # only NaN
    1: [3.0, NEG_NAN, 1.0],              # NaN among numbers: SUM NaN, MIN / MAX ignore it
    2: [2.0, PAYLOAD_NAN, -5.0],
    3: [-0.0, -0.0],                     # only -0.0
    4: [INF, -INF],                      # inf - inf
    5: [INF, 1.0, 2.0],
    6: [-INF, 7.0],
    7: [1e308, 1e308, 1e308],            # positive values past DBL_MAX
    8: [NEXT_DN, NEXT_UP, NEXT_UP],      # the NULL sentinel's neighbours are values
    9: [5e-324, 5e-324, 1e-320],         # subnormals
    10: [0.0, -0.0],
    11: [1.5, -1.5],
    12: [fx.NULL_DOUBLE, fx.NULL_DOUBLE],  # NULL only (the NOT NULL column holds 1.0 there instead)
    13: [INF, QNAN],
}


def _special_table(spec, sql_type, nullable, null_replacement):
    k, v = [], []
    for g, vals in spec.items():
        for x in vals:
            k.append(g)
            v.append(null_replacement if (not nullable and x == (fx.NULL_DOUBLE if sql_type == abi.kDOUBLE else fx.NULL_FLOAT)) else x)
    dt = abi.NUMPY_OF[sql_type]
    t = abi.Table([(abi.kINT, True), (sql_type, not nullable)])
    t.add_host_fragment([np.array(k, np.int32), np.array(v, dt)])
    return t, np.array(k, np.int32), np.array(v, dt)


SPECIAL_SQL = "SELECT k, SUM(v), MIN(v), MAX(v), AVG(v), COUNT(v), COUNT(*) FROM t GROUP BY k;"


def check_special_rows(rows, keys, vals, sql_type, nullable, skip=()):
    """Rows of SPECIAL_SQL against the module's rules; returns a list of mismatches."""
    is_float = sql_type == abi.kFLOAT
    null = (fx.NULL_FLOAT if is_float else fx.NULL_DOUBLE) if nullable else None
    groups = fx.groups_of(keys, vals, null=null)
    bad = []
    assert sorted(r[0] for r in rows) == sorted(groups)
    for r in rows:
        g = groups[r[0]]
        if r[0] in skip:
            continue
        for what, msg in [
                ("SUM", (fx.check_float_sum if is_float else fx.check_double_sum)(r[1], g)),
                ("MIN", fx.check_minmax(r[2], g, True, nullable, is_float)),
                ("MAX", fx.check_minmax(r[3], g, False, nullable, is_float)),
                ("AVG", (fx.check_float_avg if is_float else fx.check_double_avg)(r[4], g)),
                ("COUNT", None if r[5] == g.n else f"{r[5]} != {g.n}"),
                ("COUNT(*)", None if r[6] == g.rows else f"{r[6]} != {g.rows}")]:
            if msg:
                bad.append((r[0], what, msg))
    return bad


def special_float():
    f = {g: [float(np.float32(x)) if math.isfinite(x) and abs(x) < 1e38 else x for x in vals] for g, vals in SPECIAL_DOUBLE.items()}
    f[7] = [3e38, 3e38]                                        # past FLT_MAX: the double sum narrows to +inf
    f[8] = [NEXT_FDN, NEXT_FUP, NEXT_FUP]
    f[9] = [float(np.float32(2.0 ** -149)), float(np.float32(2.0 ** -140)), float(np.float32(2.0 ** -126)) * 0.75]
    f[12] = [fx.NULL_FLOAT, fx.NULL_FLOAT]
    f[14] = [float(np.float32(2.0 ** -127)), float(np.float32(2.0 ** -127))]   # two subnormals sum to FLT_MIN == NULL_FLOAT
    return f


@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("sql_type", [abi.kDOUBLE, abi.kFLOAT])
def test_oracle_agrees_with_the_special_value_rules(sql_type, nullable):
    spec = SPECIAL_DOUBLE if sql_type == abi.kDOUBLE else special_float()
    t, keys, vals = _special_table(spec, sql_type, nullable, 1.0)
    unit = sqlmini.parse(SPECIAL_SQL, t, ["k", "v"])
    rows = oracle_lib.execute(unit, t, entry_guess=32, has_card=True).rows()
    skip = ()
    if sql_type == abi.kFLOAT:
        skip = (14,)      # the reference adds in float: FLT_MIN reads as NULL there; checked on its own below
    assert check_special_rows(rows, keys, vals, sql_type, nullable, skip) == []
    by_key = {r[0]: r for r in rows}
    # pinned: the all-NaN group's MIN / MAX (NaN for the nullable form, the init value for NOT NULL)
    if nullable:
        assert math.isnan(by_key[0][2]) and math.isnan(by_key[0][3])
    else:
        big = fx.FLT_MAX if sql_type == abi.kFLOAT else fx.DBL_MAX
        assert by_key[0][2:4] == (big, -big)
    assert by_key[7][1] == INF


def test_oracle_float_sum_equal_to_the_null_sentinel_reads_as_null():
    t, _k, _v = _special_table(special_float(), abi.kFLOAT, True, 1.0)
    rows = {r[0]: r for r in oracle_lib.execute(sqlmini.parse(SPECIAL_SQL, t, ["k", "v"]), t, entry_guess=32, has_card=True).rows()}
    assert rows[14][1] is None and rows[14][5] == 2


def test_oracle_nullable_sum_of_negative_zeros_is_negative_zero():
    """agg_sum_double_skip_val ASSIGNS the first value: a nullable SUM over -0.0 only is -0.0 in the reference (the GPU's
    accumulator starts at +0.0 and gives +0.0; DESIGN.md, known deviations).  NOT NULL starts from +0.0 in both."""
    for nullable, sign in [(True, -1.0), (False, 1.0)]:
        t = abi.Table([(abi.kINT, True), (abi.kDOUBLE, not nullable)])
        t.add_host_fragment([np.zeros(3, np.int32), np.array([-0.0, -0.0, -0.0])])
        rows = oracle_lib.execute(sqlmini.parse("SELECT k, SUM(v) FROM t GROUP BY k;", t, ["k", "v"]), t, entry_guess=4, has_card=True).rows()
        assert rows[0][1] == 0.0 and math.copysign(1.0, rows[0][1]) == sign


def test_oracle_nullable_min_takes_a_leading_nan():
    """The arrival-order dependence the exact reference leaves out: the nullable MIN / MAX assigns its FIRST value, and
    std::min(NaN, x) keeps the NaN, so a group whose first row is NaN ends at NaN; the same values in another order do not.
    The GPU never lets a NaN beat a number (DESIGN.md, known deviations)."""
    t = abi.Table([(abi.kINT, True), (abi.kDOUBLE, False)])
    t.add_host_fragment([np.array([0, 0, 0, 1, 1, 1], np.int32), np.array([NAN, 3.0, 1.0, 3.0, NAN, 1.0])])
    rows = {r[0]: r for r in oracle_lib.execute(sqlmini.parse("SELECT k, MIN(v), MAX(v) FROM t GROUP BY k;", t, ["k", "v"]),
                                                 t, entry_guess=4, has_card=True).rows()}
    assert math.isnan(rows[0][1]) and math.isnan(rows[0][2])
    assert rows[1][1:] == (1.0, 3.0)


def test_module_rejects_wrong_special_values():
    """The checks themselves: NaN vs number, NULL vs value, inf vs finite, a finite overflow."""
    g = fx.Group(np.array([1.0, NAN]), 2)
    assert fx.check_double_sum(1.0, g) and fx.check_double_sum(NAN, g) is None
    g = fx.Group(np.array([NAN, NAN]), 2)
    assert fx.check_minmax(None, g, True, True) and fx.check_minmax(NAN, g, True, True) is None
    assert fx.check_minmax(fx.DBL_MAX, g, True, False) is None and fx.check_minmax(NAN, g, True, False)
    g = fx.Group(np.array([1e308, 1e308]), 2)
    assert fx.check_double_sum(INF, g) is None and fx.check_double_sum(1e308, g)
    g = fx.Group(np.array([3e38, 3e38]), 2)
    assert fx.check_float_sum(INF, g) is None and fx.check_float_sum(3.4e38, g)
    g = fx.Group(np.array([-0.0, 0.0]), 2)
    assert fx.check_minmax(0.0, g, True, True) is None and fx.check_minmax(-0.0, g, False, True) is None
    assert fx.check_double_sum(None, fx.Group(np.zeros(0), 3)) is None


@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("sql_type", [abi.kDOUBLE, abi.kFLOAT])
def test_oracle_agrees_on_the_merge_special_values(sql_type, nullable):
    """The groups test_gpu_multi_exact places across ranks (+-0 on two ranks, a NaN-only partial, +-inf, per-rank sums whose
    total overflows), whole-table, against the same rules.  Left out for the reference only: group 22 in the nullable form,
    whose first value is a NaN (the leading-NaN order dependence above), and the FLOAT group 30, which the reference adds in
    float (2^24 + 1 rounds back to 2^24) where the product narrows its double sum once."""
    import test_gpu_multi_exact as mx
    null = fx.NULL_FLOAT if sql_type == abi.kFLOAT else fx.NULL_DOUBLE
    spec = mx.fp_merge_groups(3, sql_type)
    if not nullable:
        spec = {key: {r: [1.0 if v == null else v for v in vals] for r, vals in pr.items()} for key, pr in spec.items()}
    t, keys, vals = mx.rank_table(spec, 3, sql_type, not nullable, null, abi.NUMPY_OF[sql_type])
    rows = oracle_lib.execute(sqlmini.parse(SPECIAL_SQL, t, ["k", "v"]), t, entry_guess=64, has_card=True).rows()
    skip = ((22,) if nullable else ()) + ((30,) if sql_type == abi.kFLOAT else ())
    assert check_special_rows(rows, keys, vals, sql_type, nullable, skip) == []
