"""The exact integer reference (int_exact_ref) on the CPU: the oracle equals it on every edge table of every physical width
(this is also the only check of SUM / AVG over int64 wrap-around: SQLite raises where the reference wraps), the lowered
filter program (tests/cpp/filter_emulator.cpp) passes exactly the rows its predicate passes for every width x operator x
edge literal, and one dropped, duplicated or sign-flipped row changes a result on every dataset."""
import numpy as np
import pytest

import int_exact_ref as ix
import oracle_lib
import sqlmini
from heavydb_b200 import abi, executor
from test_filter_lowering import emu, passing_rows  # noqa: F401  (emu is a fixture)

FRAG_ROWS = 1500


def aggs_of(w: ix.Width) -> str:
    """COUNT(DISTINCT) where its bitmap spans the whole type (up to 16 bits; not over days-encoded dates): wider ranges are
    refused by design."""
    distinct = ", COUNT(DISTINCT v)" if w.bits <= 16 and not w.is_days else ""
    if w.is_dict:
        return "COUNT(*), COUNT(v)" + distinct
    if w.is_days:
        return "COUNT(*), COUNT(v), MIN(v), MAX(v)" + distinct
    return "COUNT(*), COUNT(v), SUM(v), MIN(v), MAX(v), AVG(v)" + distinct


def check_rows(rows, plan, groups, w: ix.Width, device=False):
    """Every target of every row (read with decimal_to_double=False) against the exact group.  Returns (mismatches, skipped):
    skipped counts the (group, target) pairs left out.  A 32-bit COUNT(col) is compared with IntGroup.count32.  For the
    oracle (device=False), SUM / AVG of a SENTINEL_SUM group are left out.  For the product (device=True) nothing is: its
    SUM is the wrapped sum in any order, which reads as NULL when it is INT64_MIN, and AVG divides that sum."""
    targets = plan.targets[: plan.num_targets]
    grouped = plan.query_desc_type != abi.NonGroupedAggregate
    keys = [r[0] for r in rows] if grouped else [None] * len(rows)
    assert sorted(keys, key=lambda k: (k is None, k)) == sorted(groups, key=lambda k: (k is None, k)), (len(keys), len(groups))
    bad, skipped = [], 0
    for k, r in zip(keys, rows):
        g = groups[k]
        for i, t in enumerate(targets):
            if not t.is_agg:
                continue
            got = r[i]
            if t.agg_kind == abi.kCOUNT:
                want = (g.rows if t.arg_col_id < 0 else g.count_distinct if t.is_distinct
                        else g.count if t.sql_type.type == abi.kBIGINT else g.count32)
            elif t.agg_kind in (abi.kSUM, abi.kAVG) and g.sentinel_sum and not device:
                skipped += 1
                continue
            elif t.agg_kind == abi.kSUM:
                want = None if g.sum == ix.INT64_MIN else g.sum
            elif t.agg_kind == abi.kAVG:
                want = g.avg(w.scale)
            else:
                want = g.min if t.agg_kind == abi.kMIN else g.max
            if got != want:
                bad.append((k, i, got, want))
    return bad, skipped


def edge_table(w, name, nullable, rows=6000, seed=0, frag_rows=FRAG_ROWS):
    keys, phys = ix.make_dataset(w, name, rows, nullable, seed=seed)
    t = w.table(notnull=not nullable)
    for b in range(0, keys.size, frag_rows):
        t.add_host_fragment([keys[b:b + frag_rows], phys[b:b + frag_rows]])
    return t, keys, phys


CASES = [(w.name, d, nn) for w in ix.WIDTHS for d in ix.dataset_names(w) for nn in (True, False)]


@pytest.mark.parametrize("width,dataset,nullable", CASES)
def test_oracle_equals_the_reference(width, dataset, nullable):
    w = ix.WIDTH[width]
    t, keys, phys = edge_table(w, dataset, nullable)
    aggs = aggs_of(w)
    drop_lo = ("cmp", "<>", w.logical(w.lo))          # the NULL sentinel's upper neighbour
    for sql, mask, grouped in [(f"SELECT k, {aggs} FROM t GROUP BY k;", None, True),
                               (f"SELECT k, {aggs} FROM t WHERE {ix.predicate_sql(w, drop_lo)} GROUP BY k;", drop_lo, True),
                               (f"SELECT {aggs} FROM t;", None, False)]:
        unit = sqlmini.parse(sql, t, ["k", "v"])
        res = oracle_lib.execute(unit, t, entry_guess=128, has_card=True)
        m = None if mask is None else ix.passing(w, phys, nullable, mask)
        groups = ix.groups_of(w, keys if grouped else None, phys, nullable, mask=m, frag_rows=FRAG_ROWS)
        bad, skipped = check_rows(res.rows(decimal_to_double=False), res.plan, groups, w)
        assert not bad, (sql, bad[:6], skipped)


def test_the_datasets_reach_the_edges():
    """What the edge tables are for: wrapped sums, sums of 0 mod 2^64 over non-zero values, carries in every add,
    sentinel neighbours, and DICT ids above 127 / 32767."""
    w = ix.WIDTH["INT64"]
    keys, phys = ix.make_dataset(w, "pool", 6000, False)
    vals = [int(v) for v in phys]
    assert ix.INT64_MIN + 1 in vals and ix.INT64_MAX in vals and 2 ** 53 + 1 in vals and 2 ** 32 - 1 in vals
    groups = ix.groups_of(w, keys, phys, False)
    assert any(sum(g.values) != g.sum for g in groups.values())                 # wrapped
    keys, phys = ix.make_dataset(w, "wrap_to_zero", 6000, False)
    groups = ix.groups_of(w, keys, phys, False)
    assert all(g.sum == 0 for g in groups.values()) and any(sum(g.values) != 0 for g in groups.values())
    keys, phys = ix.make_dataset(w, "carry_dense", 6000, False)
    assert set(phys.tolist()) == {2 ** 32 - 1}
    assert ix.pool(ix.WIDTH["DICT8"])[-2:] == [253, 254] and 65534 in ix.pool(ix.WIDTH["DICT16"])
    assert ix.pool(ix.WIDTH["INT8"])[:2] == [-127, -126] and ix.pool(ix.WIDTH["DAYS16"])[:2] == [-32767, -32766]
    assert ix.carry_value(ix.WIDTH["INT16"]) == -1
    keys, phys = ix.make_dataset(w, "pool", 6000, True)                 # COUNT32: 2^31 and -2^31 are not counted
    assert all(g.count32 < g.count for g in ix.groups_of(w, keys, phys, True).values() if 2 ** 31 in g.values)
    assert ix.groups_of(w, None, np.array([2 ** 31, -(2 ** 31), 5], np.int64), False)[None].count32 == 2


def test_sentinel_sum_is_named_not_tolerated():
    """A nullable group whose running sum meets INT64_MIN is excluded by name; the same values NOT NULL are not."""
    w = ix.WIDTH["INT64"]
    phys = np.array([-ix.INT64_MAX, -1, 5], dtype=np.int64)
    assert ix.groups_of(w, None, phys, True)[None].sentinel_sum
    assert ix.groups_of(w, None, phys[[2, 0]], True)[None].sentinel_sum is False


# ---- predicates: the lowered filter program against the reference ---------------------------------------------------------------
OPS = ["=", "<>", "<", ">", "<=", ">="]


def filter_table(w):
    """Every pool value twice and NULLs (nullable), two fragments."""
    p = ix.pool(w)
    phys = np.array(p + p[::-1] + [w.null] * 3, dtype=w.dtype)
    t = w.table(notnull=False)
    h = phys.size // 2
    keys = np.zeros(phys.size, np.int32)
    t.add_host_fragment([keys[:h], phys[:h]]).add_host_fragment([keys[h:], phys[h:]])
    return t, phys


def straddling(w):
    """IN lists and BETWEEN around the NULL sentinel, and a range that covers the whole type."""
    unit = ix.SECONDS_PER_DAY if w.is_days else 1
    s, lo, hi = w.null * unit, w.lo * unit, w.hi * unit
    near = [s - unit, s, s + unit, lo + unit] if not (w.is_dict and w.enc) else [s - 1, s, s + 1, 0]
    if w.scale:                                       # DECIMAL(18, s): the sentinel is out of the literal's reach
        near, lo, hi = [-ix.DECIMAL18_MAX, -ix.DECIMAL18_MAX + 1, 0], -ix.DECIMAL18_MAX, ix.DECIMAL18_MAX
    near = [x for x in near if ix.INT64_MIN <= x <= ix.INT64_MAX]
    ids = [("in", near), ("not", ("in", near)), ("or", ("isnull",), ("cmp", "=", lo)), ("in", [lo, hi, 0]), ("not", ("in", [lo, hi])),
           ("and", ("cmp", "<>", lo), ("not", ("isnull",)))]
    if w.is_dict:                                     # ids compare with = and <> only
        return ids
    return ids + [("between", min(near), max(near)), ("not", ("between", min(near), max(near))), ("between", lo, hi),
                  ("and", ("cmp", ">=", lo), ("cmp", "<", hi))]


@pytest.mark.parametrize("width", [w.name for w in ix.WIDTHS])
def test_filter_program_equals_the_reference(emu, width):  # noqa: F811
    w = ix.WIDTH[width]
    t, phys = filter_table(w)
    preds = [("cmp", op, lit) for op in (OPS[:2] if w.is_dict else OPS) for lit in ix.edge_literals(w)] + straddling(w)
    for p in preds:
        sql = f"SELECT COUNT(*) FROM t WHERE {ix.predicate_sql(w, p)};"
        unit = sqlmini.parse(sql, t, ["k", "v"])
        want = int(ix.passing(w, phys, True, p).sum())
        assert passing_rows(emu, unit, t) == want, sql
        assert oracle_lib.execute(unit, t).rows()[0][0] == want, sql


# ---- sensitivity ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("width,dataset", [(w.name, d) for w in ix.WIDTHS if w.summable for d in ix.dataset_names(w)])
def test_one_changed_row_changes_a_result(width, dataset):
    """For every group of every dataset: dropping, duplicating or sign-flipping one non-zero row makes check_rows report the
    exact answer of the changed rows as a mismatch — SUM moves unless the value is 0 mod 2^64, MIN / MAX / COUNT otherwise."""
    w = ix.WIDTH[width]
    keys, phys = ix.make_dataset(w, dataset, 3000, nullable=False, seed=1)
    t = w.table(notnull=True)
    t.add_host_fragment([keys, phys])
    plan = oracle_lib.plan(sqlmini.parse(f"SELECT k, {aggs_of(w)} FROM t GROUP BY k;", t, ["k", "v"]), t, entry_guess=128, has_card=True)
    groups = ix.groups_of(w, keys, phys, False)

    def row_of(k, g):
        return (k, g.rows, g.count, g.sum, g.min, g.max, g.avg(w.scale), g.count_distinct)
    for k, g in groups.items():
        i = next(j for j, v in enumerate(g.values) if v != 0)
        x = g.values[i]
        flipped = list(g.values)
        flipped[i] = -x
        for what, vals, rows in [("dropped", g.values[:i] + g.values[i + 1:], g.rows - 1), ("duplicated", g.values + [x], g.rows + 1),
                                 ("flipped", flipped, g.rows)]:
            changed = ix.IntGroup(vals, rows)
            assert check_rows([row_of(k, changed)], plan, {k: g}, w)[0], (width, dataset, k, what)
            assert changed.sum != g.sum, (width, dataset, k, what)           # the wrap never hides one row


def test_result_set_sort_refuses_dictionary_string_targets():
    """ResultSet::sort orders dictionary strings through the dictionary (ResultSet.cpp:1424-1436); the device sort would
    order ids.  Refused before any device work, so this runs without a GPU."""
    w = ix.WIDTH["DICT16"]
    t, _keys, _phys = edge_table(w, "pool", True, rows=500)
    t2 = abi.Table([(abi.kTEXT, False), (abi.kINT, True)], encoded_sizes=[2, 0])
    t2.add_host_fragment([_phys, _keys])
    ran = 0
    for table, sql, entries in [(t, "SELECT k, MIN(v), COUNT(*) FROM t GROUP BY k;", [(2, False, False)]),
                                (t2, "SELECT s, COUNT(*) FROM t GROUP BY s;", [(2, True, False), (1, False, True)])]:
        unit = sqlmini.parse(sql, table, ["k", "v"] if table is t else ["s", "k"])
        try:
            ref = oracle_lib.execute(unit, table, entry_guess=128, has_card=True)
        except oracle_lib.OracleError:
            continue
        rs = executor.Executor().resultSetFromStorage(ref.buffer(), unit, table, max_groups_buffer_entry_guess=128,
                                                      has_cardinality_estimation=True)
        with pytest.raises(executor.UnsupportedOnThisPath, match="dictionary"):
            rs.sort(entries)
        ran += 1
    assert ran


# ---- the datasets of the cross-device merge tests (test_gpu_multi_exact) ----------------------------------------------------------------
def fragment_prefix_sums(groups, t, w, nullable, grouped):
    """Record the running sums of fragments of unequal sizes (groups_of takes one fragment size), for SENTINEL_SUM."""
    totals = {}
    for f in t.fragments:
        run = {}
        for kk, x in zip(f.host_cols[0].tolist(), f.host_cols[1].tolist()):
            g = kk if grouped else None
            if nullable and x == w.null:
                continue
            run[g] = ix.wrap64(run.get(g, 0) + w.logical(x))
            groups[g].prefix_sums.add(run[g])
        for g, r in run.items():
            totals[g] = ix.wrap64(totals.get(g, 0) + r)
            groups[g].prefix_sums.add(totals[g])


@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("k", [2, 3, 8])
def test_oracle_equals_the_reference_on_the_merge_datasets(k, nullable):
    """Groups that only a merge creates (per-rank SUMs that wrap while the total does not and the reverse, a group on one
    rank only, NULL on one rank, MIN = MAX = INT64_MAX, values next to INT64_MIN) and the placement-edge table (skipped,
    filtered-out and fully deleted fragments), over the whole table."""
    import test_gpu_multi_exact as mx
    w = ix.WIDTH["INT64"]
    spec = mx.merge_edge_groups(k)
    if not nullable:
        spec = {key: {r: [1 if v is None else v for v in vals] for r, vals in pr.items()} for key, pr in spec.items()}
    t, keys, phys = mx.rank_table(spec, k, abi.kBIGINT, not nullable, w.null, np.int64)
    aggs = "COUNT(*), COUNT(v), SUM(v), MIN(v), MAX(v), AVG(v)"
    for sql, ks in [(f"SELECT k, {aggs} FROM t GROUP BY k;", keys), (f"SELECT {aggs} FROM t;", None)]:
        res = oracle_lib.execute(sqlmini.parse(sql, t, ["k", "v"]), t, entry_guess=64, has_card=True)
        groups = ix.groups_of(w, ks, phys, nullable)
        fragment_prefix_sums(groups, t, w, nullable, grouped=ks is not None)
        bad, _skipped = check_rows(res.rows(decimal_to_double=False), res.plan, groups, w)
        assert not bad, (sql, bad[:6])
    t, keys, v, _d, m = mx.placement_table(k)
    for sql, ks in [("SELECT k, COUNT(*), COUNT(v), SUM(v), MIN(v), MAX(v), AVG(v) FROM t WHERE k < 1000 AND (f > 0 OR f < 0) GROUP BY k;", keys),
                    ("SELECT COUNT(*), COUNT(v), SUM(v), MIN(v), MAX(v), AVG(v) FROM t WHERE k < 1000 AND (f > 0 OR f < 0);", None)]:
        res = oracle_lib.execute(sqlmini.parse(sql, t, ["k", "v", "d", "f", "del"]), t)
        bad, _skipped = check_rows(res.rows(decimal_to_double=False), res.plan, ix.groups_of(w, ks, v, True, mask=m), w)
        assert not bad, (sql, bad[:6])
    t, (keys, v, _s, _b) = mx.baseline_table(k)
    n_keys = len(set(keys.tolist()))
    res = oracle_lib.execute(sqlmini.parse("SELECT k, COUNT(*), COUNT(v), SUM(v), MIN(v), MAX(v), AVG(v) FROM t GROUP BY k;", t,
                                           ["k", "v", "s", "b"]), t, entry_guess=2 * n_keys, has_card=True)
    assert res.plan.query_desc_type == abi.GroupByBaselineHash
    groups = ix.groups_of(w, keys, v, True, frag_rows=mx.BASELINE_FRAG)
    groups = {None if kk == abi.NULL_BIGINT else kk: g for kk, g in groups.items()}
    bad, _skipped = check_rows(res.rows(decimal_to_double=False), res.plan, groups, w)
    assert not bad, bad[:6]
