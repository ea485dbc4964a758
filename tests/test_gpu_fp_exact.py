"""Floating-point aggregates of every scan kernel against the exact reference (fp_exact_ref): SUM / AVG within the error bound
of IEEE double summation in any order, MIN / MAX / COUNT exactly, NaN / inf / -0.0 / subnormals / NULL-sentinel neighbours
with the reference's semantics.  The bound is tight enough that one lost, doubled or sign-flipped row fails it on every
non-cancellation dataset (test_fp_exact_ref.py proves that on the CPU).  The plan still has to equal the oracle's.

ORDER BY over floating-point aggregates uses dyadic data whose sums are exact in double, so that the expected order is
unique; NaN is left out on purpose: the reference's `<` is not a strict weak order on NaN, so no order is "the" answer."""
import math

import numpy as np
import pytest

import fp_exact_ref as fx
import gpu_util as gu
import oracle_lib
import sqlmini
from heavydb_b200 import abi, executor
from test_fp_exact_ref import SPECIAL_DOUBLE, SPECIAL_SQL, check_special_rows, special_float

pytestmark = pytest.mark.gpu

AGGS = "SUM(v), AVG(v), MIN(v), MAX(v), COUNT(v), COUNT(*)"


def check_rows(rows, plan, groups):
    """Every target of every row against the exact group it belongs to; returns nothing, raises on the first mismatches."""
    targets = plan.targets[: plan.num_targets]
    grouped = plan.query_desc_type != abi.NonGroupedAggregate
    keys = [r[0] for r in rows] if grouped else [None] * len(rows)
    assert sorted(keys, key=lambda k: (k is None, k)) == sorted(groups, key=lambda k: (k is None, k)), (len(keys), len(groups))
    bad = []
    for k, r in zip(keys, rows):
        g = groups[k]
        for i, t in enumerate(targets):
            if not t.is_agg:
                continue
            is_float = t.agg_arg_type.type == abi.kFLOAT
            got = r[i]
            if t.agg_kind == abi.kCOUNT:
                want = g.rows if t.arg_col_id < 0 else g.n
                msg = None if got == want else f"COUNT {got} != {want}"
            elif t.agg_kind == abi.kSUM:
                msg = (fx.check_float_sum if is_float else fx.check_double_sum)(got, g)
            elif t.agg_kind == abi.kAVG:
                msg = (fx.check_float_avg if is_float else fx.check_double_avg)(got, g)
            else:
                msg = fx.check_minmax(got, g, t.agg_kind == abi.kMIN, bool(t.skip_null_val), is_float)
            if msg:
                bad.append((k, i, msg))
    assert not bad, f"{len(bad)} mismatches, first: {bad[:6]}"


def execute(unit, table, dev=None, entry_guess=0, has_card=False, force_kernel=0, output_columnar=False, result_on_device=False):
    """The CUDA path; asserts the plan equals the oracle's (the oracle plans only: the values come from fp_exact_ref)."""
    eo = executor.execution_options(force_kernel=force_kernel, output_columnar_hint=output_columnar, result_on_device=result_on_device)
    ex = executor.Executor()
    if dev is not None:
        rs = ex.executeWorkUnit(entry_guess, True, dev.table, unit, eo=eo, has_cardinality_estimation=has_card, memory_level=abi.GPU_LEVEL)
    else:
        rs = ex.executeWorkUnit(entry_guess, True, table, unit, eo=eo, has_cardinality_estimation=has_card, memory_level=abi.CPU_LEVEL)
    want = oracle_lib.plan(unit, table, entry_guess=entry_guess, has_card=has_card, output_columnar=output_columnar).as_dict()
    got = rs.getQueryMemDesc().as_dict()
    if unit.unit.num_order_entries or unit.unit.has_limit:      # the sorted result holds the LIMIT / OFFSET window only
        for k in ("entry_count", "buffer_size"):
            got.pop(k), want.pop(k)
    assert got == want
    return rs


def value_table(keys, vals, sql_type, nullable, frag_rows, key_type=abi.kINT, filt=None):
    """t(k, v[, f]) in fragments of frag_rows."""
    cols = [keys, vals] + ([filt] if filt is not None else [])
    types = [(key_type, True), (sql_type, not nullable)] + ([(abi.kINT, True)] if filt is not None else [])
    t = abi.Table(types)
    for b in range(0, len(keys), frag_rows):
        t.add_host_fragment([c[b:b + frag_rows] for c in cols])
    return t


def with_nulls(vals, sql_type, rng, p=0.05):
    v = vals.copy()
    v[rng.random(v.size) < p] = abi.NULL_OF[sql_type]
    return v


def dataset_table(name, nullable, seed=0, frag_rows=300_000):
    keys, vals = fx.make_dataset(name, seed)
    ty = abi.kFLOAT if fx.DATASETS[name][3] == "FLOAT" else abi.kDOUBLE
    rng = np.random.default_rng(seed + 100)
    if nullable:
        vals = with_nulls(vals, ty, rng)
    filt = rng.integers(0, 1000, keys.size).astype(np.int32)
    return value_table(keys, vals, ty, nullable, frag_rows, filt=filt), keys, vals, filt, ty


# ---- non-grouped: warp_sum_f64 + ballot "any", one slot fed by every CTA and replica --------------------------------------------
def test_non_grouped_one_hot_group_of_16m_rows():
    n = 16_000_000
    rng = np.random.default_rng(11)
    v = 1.0 + rng.random(n)
    f = rng.integers(0, 1000, n).astype(np.int32)
    t = abi.Table([(abi.kDOUBLE, True), (abi.kINT, True)])
    for b in range(0, n, 1 << 22):
        t.add_host_fragment([v[b:b + (1 << 22)], f[b:b + (1 << 22)]])
    dev = gu.DeviceTable(t)
    for sql, mask in [(f"SELECT {AGGS} FROM t;", None), (f"SELECT {AGGS} FROM t WHERE f < 999;", f < 999)]:
        unit = sqlmini.parse(sql, t, ["v", "f"])
        rs = execute(unit, t, dev)
        assert rs.getQueryMemDesc().kernel == abi.KERNEL_NON_GROUPED
        groups = fx.groups_of(None, v, mask=mask)
        assert fx.sensitive(groups[None])
        check_rows(rs.rows(), rs.getQueryMemDesc(), groups)


@pytest.mark.parametrize("name", sorted(fx.DATASETS))
def test_non_grouped_datasets(name):
    t, _keys, vals, filt, ty = dataset_table(name, nullable=True)
    dev = gu.DeviceTable(t)
    unit = sqlmini.parse(f"SELECT {AGGS} FROM t WHERE f < 700;", t, ["k", "v", "f"])
    rs = execute(unit, t, dev)
    assert rs.getQueryMemDesc().kernel == abi.KERNEL_NON_GROUPED
    check_rows(rs.rows(), rs.getQueryMemDesc(), fx.groups_of(None, vals, null=abi.NULL_OF[ty], mask=filt < 700))


# ---- perfect hash: shared-memory table (fused and general), HBM/L2 table ----------------------------------------------------------
@pytest.mark.parametrize("name", ["pos12", "pos2e20", "cancel"])
def test_perfect_hash_smem_fused_double_sum(name):
    """NOT NULL DOUBLE SUM + COUNT(*): the fused shared-memory path."""
    t, keys, vals, _f, ty = dataset_table(name, nullable=False)
    dev = gu.DeviceTable(t)
    unit = sqlmini.parse("SELECT k, SUM(v), COUNT(*) FROM t GROUP BY k;", t, ["k", "v", "f"])
    rs = execute(unit, t, dev)
    assert rs.getQueryMemDesc().kernel == abi.KERNEL_PERFECT_SMEM
    check_rows(rs.rows(), rs.getQueryMemDesc(), fx.groups_of(keys, vals))


@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("name", sorted(fx.DATASETS))
def test_perfect_hash_smem_and_global(name, nullable):
    t, keys, vals, filt, ty = dataset_table(name, nullable)
    dev = gu.DeviceTable(t)
    null = abi.NULL_OF[ty] if nullable else None
    unit = sqlmini.parse(f"SELECT k, {AGGS} FROM t WHERE f < 900 GROUP BY k;", t, ["k", "v", "f"])
    groups = fx.groups_of(keys, vals, null=null, mask=filt < 900)
    for force, kernel in [(0, abi.KERNEL_PERFECT_SMEM), (abi.KERNEL_PERFECT_GLOBAL, abi.KERNEL_PERFECT_GLOBAL)]:
        rs = execute(unit, t, dev, force_kernel=force)
        assert rs.getQueryMemDesc().kernel == kernel
        check_rows(rs.rows(), rs.getQueryMemDesc(), groups)


def test_perfect_hash_key_range_too_large_for_shared_memory():
    rng = np.random.default_rng(5)
    n = 1_000_000
    keys = rng.integers(0, 50_000, n).astype(np.int32)
    vals = with_nulls((1.0 + rng.random(n)) * 2.0 ** 20, abi.kDOUBLE, rng)
    t = value_table(keys, vals, abi.kDOUBLE, True, 1 << 21)
    unit = sqlmini.parse(f"SELECT k, {AGGS} FROM t GROUP BY k;", t, ["k", "v"])
    rs = execute(unit, t, gu.DeviceTable(t))
    assert rs.getQueryMemDesc().kernel == abi.KERNEL_PERFECT_GLOBAL
    check_rows(rs.rows(), rs.getQueryMemDesc(), fx.groups_of(keys, vals, null=abi.NULL_DOUBLE))


# ---- baseline hash: radix passes (DOUBLE) and the per-row probe (forced, and FLOAT arguments) -------------------------------------
@pytest.mark.parametrize("name,nullable", [("pos12", True), ("pos2e20", False), ("cancel", True), ("f32_pos", True), ("f32_subnormal", False)])
def test_baseline_hash(name, nullable):
    _t, keys, vals, _f, ty = dataset_table(name, nullable)
    sparse = keys.astype(np.int64) * 7919 * 10**9 + 12345
    t = value_table(sparse, vals, ty, nullable, 300_000, key_type=abi.kBIGINT)
    dev = gu.DeviceTable(t)
    unit = sqlmini.parse(f"SELECT k, {AGGS} FROM t GROUP BY k;", t, ["k", "v"])
    groups = fx.groups_of(sparse, vals, null=abi.NULL_OF[ty] if nullable else None)
    launches = {}
    for force in (0, abi.KERNEL_BASELINE_PROBE):          # the plan says BASELINE_GLOBAL either way; the executor picks the passes
        rs = execute(unit, t, dev, entry_guess=2 * len(groups), has_card=True, force_kernel=force)
        assert rs.getQueryMemDesc().kernel == abi.KERNEL_BASELINE_GLOBAL
        launches[force] = rs.stats()["kernel_launches"]
        check_rows(rs.rows(), rs.getQueryMemDesc(), groups)
    if ty == abi.kDOUBLE:
        assert launches[0] > launches[abi.KERNEL_BASELINE_PROBE], launches       # radix partition + aggregate passes
    else:
        assert launches[0] == launches[abi.KERNEL_BASELINE_PROBE], launches      # FLOAT arguments fall back to the probe


# ---- INNER / LEFT join: a DOUBLE column of the inner table ------------------------------------------------------------------------
@pytest.mark.parametrize("how", ["JOIN", "LEFT JOIN"])
def test_join_inner_double_column(how):
    rng = np.random.default_rng(21)
    dim_rows, n = 1000, 600_000
    dim_id = rng.permutation(dim_rows).astype(np.int32)
    w = (1.0 + rng.random(dim_rows)) * 2.0 ** 20
    w[rng.random(dim_rows) < 0.1] = abi.NULL_DOUBLE
    dim = abi.Table([(abi.kINT, True), (abi.kDOUBLE, False)])
    dim.add_host_fragment([dim_id, w])
    fk = rng.integers(-5, dim_rows + 60, n).astype(np.int32)
    x = rng.integers(0, 10, n).astype(np.int32)
    fact = abi.Table([(abi.kINT, True), (abi.kINT, True)])
    for b in range(0, n, 200_000):
        fact.add_host_fragment([fk[b:b + 200_000], x[b:b + 200_000]])
    unit = sqlmini.parse(f"SELECT t.x, SUM(d.w), AVG(d.w), MIN(d.w), MAX(d.w), COUNT(d.w), COUNT(*) FROM t {how} d ON t.fk = d.id "
                         "GROUP BY t.x;", fact, ["fk", "x"], inner=(dim, ["id", "w"]))
    row_of = np.full(dim_rows + 100, -1, np.int64)
    row_of[dim_id] = np.arange(dim_rows)
    hit = (fk >= 0) & (fk < dim_rows)
    r = np.where(hit, row_of[np.clip(fk, 0, dim_rows + 99)], -1)
    joined = np.where(r >= 0, w[np.maximum(r, 0)], abi.NULL_DOUBLE)     # LEFT: unmatched rows read the NULL placeholder
    mask = None if how == "LEFT JOIN" else r >= 0
    groups = fx.groups_of(x, joined, null=abi.NULL_DOUBLE, mask=mask)
    rs = execute(unit, fact, gu.DeviceTable(fact))
    check_rows(rs.rows(), rs.getQueryMemDesc(), groups)
    rs = execute(unit, fact)                                          # fact table streamed from the host
    check_rows(rs.rows(), rs.getQueryMemDesc(), groups)


# ---- host-resident tables: one launch per 16 Mi-row slice into the same accumulators -----------------------------------------------
@pytest.mark.parametrize("name", ["pos12", "f32_pos", "f32_subnormal"])
def test_host_resident(name):
    t, keys, vals, filt, ty = dataset_table(name, nullable=True, frag_rows=100_000)
    unit = sqlmini.parse(f"SELECT k, {AGGS} FROM t WHERE f < 900 GROUP BY k;", t, ["k", "v", "f"])
    rs = execute(unit, t)
    assert rs.stats()["h2d_bytes"] > 0
    check_rows(rs.rows(), rs.getQueryMemDesc(), fx.groups_of(keys, vals, null=abi.NULL_OF[ty], mask=filt < 900))


def test_float_sum_is_narrowed_once_across_host_slices():
    """2^24 + 1 FLOAT rows in one host fragment: slice 1 holds 2^24 rows summing to 2^24 + 2^-23, slice 2 one row of 1.0.
    Every partial sum is exact in double, so the one narrowing gives float(2^24 + 1 + 2^-23) = 2^24 + 2.  A float narrowing
    after slice 1 would give 2^24, and 2^24 + 1 then ties to 2^24 again."""
    n = (1 << 24) + 1
    v = np.ones(n, dtype=np.float32)
    v[12345] = np.float32(1.0 + 2.0 ** -23)
    t = abi.Table([(abi.kFLOAT, True)])
    t.add_host_fragment([v])
    unit = sqlmini.parse("SELECT SUM(v), AVG(v), COUNT(*) FROM t;", t, ["v"])
    rs = execute(unit, t)
    assert rs.stats()["h2d_bytes"] >= 4 * n
    s, avg, cnt = rs.rows()[0]
    assert cnt == n
    assert s == float(np.float32(2.0 ** 24 + 1 + 2.0 ** -23)) == 2.0 ** 24 + 2, s
    assert avg == (2.0 ** 24 + 2) / n


# ---- columnar output and the device hand-off ---------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["pos2e20", "f32_subnormal"])
def test_columnar_output_and_device_columns(name):
    t, keys, vals, filt, ty = dataset_table(name, nullable=True)
    dev = gu.DeviceTable(t)
    unit = sqlmini.parse(f"SELECT k, {AGGS} FROM t WHERE f < 900 GROUP BY k;", t, ["k", "v", "f"])
    groups = fx.groups_of(keys, vals, null=abi.NULL_OF[ty], mask=filt < 900)
    rs = execute(unit, t, dev, output_columnar=True, result_on_device=True)
    assert rs.getQueryMemDesc().output_columnar == 1
    cols = rs.deviceColumns().to_host()
    assert rs.stats()["result_d2h_bytes"] == 0                        # read where it lies
    rows = []
    for i in range(len(cols[0][2])):
        row = []
        for ty_c, _nn, values, validity, _nulls in cols:
            ok = validity is None or bool(validity[i >> 3] >> (i & 7) & 1)
            x = values[i]
            row.append(None if not ok else float(x) if ty_c in (abi.kDOUBLE, abi.kFLOAT) else int(x))
        rows.append(tuple(row))
    check_rows(rows, rs.getQueryMemDesc(), groups)
    check_rows(rs.rows(), rs.getQueryMemDesc(), groups)


# ---- IEEE special values on every kernel family ----------------------------------------------------------------------------------
@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("sql_type", [abi.kDOUBLE, abi.kFLOAT])
def test_special_values(sql_type, nullable):
    """NaN (quiet, negative, with a payload), +-inf, +-0, subnormals, DBL_MIN / FLT_MIN as NULL and their two neighbours as
    values, a sum past DBL_MAX / FLT_MAX, groups of only NaN, only NULL, only -0.0 — repeated so that replicas, warps and CTAs
    meet them in every arrangement (no group starts with a NaN: see test_fp_exact_ref for that order dependence)."""
    spec = SPECIAL_DOUBLE if sql_type == abi.kDOUBLE else special_float()
    rng = np.random.default_rng(8)
    k, v = [], []
    rep = 4000
    for g, vals in spec.items():
        body = [x for x in vals if not math.isnan(x)] or vals          # the group's first row is a number when it has one
        nan_rows = [x for x in vals if math.isnan(x)] if body is not vals else []
        if g == 7:                                                    # overflow: the double sum itself stays finite for FLOAT
            rows = list(vals) * 3
        elif g in (8, 9):                                             # sentinel neighbours / subnormals: small exact sums
            rows = list(vals) * 2
        elif g == 14:                                                 # two float subnormals summing to exactly FLT_MIN
            rows = list(vals)
        else:
            rows = body[:1] + list(rng.permutation(np.array((body + nan_rows) * rep, dtype=np.float64)))
        k += [g] * len(rows)
        v += rows
    keys = np.array(k, np.int32)
    dt = abi.NUMPY_OF[sql_type]
    null = fx.NULL_DOUBLE if sql_type == abi.kDOUBLE else fx.NULL_FLOAT
    vals = np.array([1.0 if (not nullable and x == null) else x for x in v], dtype=dt)
    perm = rng.permutation(keys.size)                                # groups interleaved, first rows kept first
    first = np.zeros(keys.size, bool)
    first[np.unique(keys, return_index=True)[1]] = True
    order = np.concatenate([np.flatnonzero(first), perm[~first[perm]]])
    keys, vals = keys[order], vals[order]
    t = value_table(keys, vals, sql_type, nullable, 7000)
    dev = gu.DeviceTable(t)
    skip = (14,) if sql_type == abi.kFLOAT else ()                   # FLT_MIN as a sum: checked below
    for sql, runs in [(SPECIAL_SQL, [(0, abi.KERNEL_PERFECT_SMEM), (abi.KERNEL_PERFECT_GLOBAL, abi.KERNEL_PERFECT_GLOBAL)])]:
        unit = sqlmini.parse(sql, t, ["k", "v"])
        for force, kernel in runs:
            for d in (dev, None):
                rs = execute(unit, t, d, entry_guess=32, has_card=True, force_kernel=force)
                assert rs.getQueryMemDesc().kernel == kernel
                rows = rs.rows()
                assert check_special_rows(rows, keys, vals, sql_type, nullable, skip) == []
                if sql_type == abi.kFLOAT:
                    r14 = {r[0]: r for r in rows}[14]
                    assert r14[1] is None and r14[5] == 2        # the narrowed sum IS FLT_MIN: reads as NULL
    # baseline (sparse keys): radix passes for DOUBLE, the per-row probe for FLOAT
    sparse = keys.astype(np.int64) * 7919 * 10**9
    ts = value_table(sparse, vals, sql_type, nullable, 7000, key_type=abi.kBIGINT)
    unit = sqlmini.parse(SPECIAL_SQL, ts, ["k", "v"])
    for force in (0, abi.KERNEL_BASELINE_PROBE):
        rs = execute(unit, ts, gu.DeviceTable(ts), entry_guess=64, has_card=True, force_kernel=force)
        assert rs.getQueryMemDesc().kernel == abi.KERNEL_BASELINE_GLOBAL
        rows = [(int(r[0]) // (7919 * 10**9),) + tuple(r[1:]) for r in rs.rows()]
        assert check_special_rows(rows, keys, vals, sql_type, nullable, skip) == []
    # non-grouped, one group at a time (the nullable form of every aggregate)
    for g in (0, 1, 3, 4, 7, 12):
        m = keys == g
        tg = value_table(keys[m], vals[m], sql_type, nullable, 5000)
        unit = sqlmini.parse(f"SELECT {AGGS} FROM t;", tg, ["k", "v"])
        rs = execute(unit, tg, gu.DeviceTable(tg))
        check_rows(rs.rows(), rs.getQueryMemDesc(), fx.groups_of(None, vals[m], null=null if nullable else None))


# ---- ORDER BY floating-point aggregates (sort.cu) ----------------------------------------------------------------------------------
def order_table(groups, rows_per_group, seed, nonneg=False):
    """Dyadic values (multiples of 1/4, |sum| < 2^40): every sum is exact in double.  Special groups: +inf, -inf, only -0.0,
    only +0.0, +-0 mixed, subnormals only, NULL only.  `nonneg`: no negative finite values, so that thousands of groups tie
    at a MIN of +-0 right behind the -inf group."""
    rng = np.random.default_rng(seed)
    n = groups * rows_per_group
    keys = rng.integers(0, groups, n).astype(np.int32)
    vals = rng.integers(0 if nonneg else -40, 40, n).astype(np.float64) * 0.25
    vals[rng.random(n) < 0.05] = abi.NULL_DOUBLE
    special = {0: math.inf, 1: -math.inf, 2: -0.0, 3: 0.0, 5: 5e-324, 6: abi.NULL_DOUBLE}
    for g, x in special.items():
        vals[keys == g] = x
    m = keys == 4
    vals[m] = np.where(np.arange(m.sum()) % 2 == 0, -0.0, 0.0)
    m = keys == 7
    vals[m] = np.arange(1, m.sum() + 1) * 5e-324                     # subnormals summing to a subnormal
    keys = np.concatenate([keys, np.arange(groups, dtype=np.int32)])  # every group present
    vals = np.concatenate([vals, np.where(np.isin(np.arange(groups), list(special)), [special.get(g, 0.0) for g in range(groups)], 0.25)])
    return keys, vals


def exact_rows(groups):
    """(k, SUM, AVG, MIN, MAX) of every group, exact (the sums of order_table are exact in double)."""
    rows = []
    for k, g in groups.items():
        s = None if g.n == 0 else g.exact_sum
        avg = None if g.n == 0 else (s / g.n if math.isfinite(s) else s)
        rows.append((k, s, avg, g.minmax(True, True), g.minmax(False, True)))
    return rows


def expected_order(rows, col, desc, nulls_first, limit, offset):
    """`rows` sorted by column `col` then the key, with the reference's `<` (-0.0 ties with +0.0)."""
    def key(r):
        v = r[col]
        null_rank = (0 if nulls_first else 2) if v is None else 1
        return (null_rank, 0.0 if v is None else (-v if desc else v), r[0])
    rows = sorted(rows, key=key)
    return rows[offset:offset + limit] if limit else rows[offset:]


@pytest.mark.parametrize("groups,limit,offset,nonneg", [(1000, 0, 0, False), (1000, 40, 3, False), (100_000, 10, 5, False),
                                                       (100_000, 12, 2, True)])
def test_order_by_floating_point_aggregates(groups, limit, offset, nonneg):
    """Over 65,536 groups with a small LIMIT the top-k bucket pre-filter runs first; with `nonneg` its window falls on groups
    whose MIN ties at -0.0 / +0.0, which the key (second order entry) must decide."""
    keys, vals = order_table(groups, 4, seed=groups, nonneg=nonneg)
    t = value_table(keys, vals, abi.kDOUBLE, True, 200_000)
    dev = gu.DeviceTable(t)
    exact = exact_rows(fx.groups_of(keys, vals, null=abi.NULL_DOUBLE))
    lim = (f" LIMIT {limit}" if limit else "") + (f" OFFSET {offset}" if offset else "")
    for col in (2, 3, 4, 5):
        for desc in (False, True):
            for nulls_first in (False, True):
                sql = (f"SELECT k, SUM(v), AVG(v), MIN(v), MAX(v) FROM t GROUP BY k ORDER BY {col} {'DESC' if desc else 'ASC'} "
                       f"NULLS {'FIRST' if nulls_first else 'LAST'}, 1 ASC{lim};")
                unit = sqlmini.parse(sql, t, ["k", "v"])
                rs = execute(unit, t, dev, entry_guess=groups + 1, has_card=True)
                got = rs.rows()
                want = expected_order(exact, col - 1, desc, nulls_first, limit, offset)
                assert [r[0] for r in got] == [r[0] for r in want], (sql, got[:5], want[:5])
                for a, b in zip(got, want):                           # the values are exact: == (either sign of zero)
                    assert all((x is None and y is None) or x == y for x, y in zip(a, b)), (sql, a, b)
