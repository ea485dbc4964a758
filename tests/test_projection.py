"""Projection units (SELECT <columns> FROM t WHERE ... [ORDER BY ...] [LIMIT n [OFFSET m]]) on the host: the descriptor the
planner publishes, the read-out over a projection buffer, the refusals, and the scan limit sqlmini sets."""
from __future__ import annotations

import numpy as np
import pytest

import order_queries as oq
import ref_tables as rt
from heavydb_b200 import abi, executor, sqlmini
from projection_ref import (expected_buffer, load_sqlite, mixed_table, passing_rows, plan_matches, projected_cols,
                            restate_descriptor)

ALL = ", ".join(rt.TEST_NAMES)


@pytest.fixture(scope="module")
def golden():
    table = rt.make_table(rt.test_rows())
    return table, load_sqlite(table, rt.TEST_NAMES)


@pytest.mark.parametrize("columnar", [False, True])
@pytest.mark.parametrize("scan_limit", [0, 7])
def test_descriptor(golden, columnar, scan_limit):
    table, _ = golden
    sql = f"SELECT w, z, x, t, d, f FROM test WHERE x > 6" + (f" LIMIT {scan_limit}" if scan_limit else "")
    unit = sqlmini.parse(sql, table, rt.TEST_NAMES)
    assert unit.unit.scan_limit == scan_limit
    p = executor.Executor().plan(unit, table, eo=executor.execution_options(output_columnar_hint=columnar))
    n = scan_limit or 20
    plan_matches(p, restate_descriptor(table, projected_cols(unit), columnar, n))
    logical = [1, 2, 4, 8, 8, 4]   # pinned by hand as well: TINYINT, SMALLINT, INT, BIGINT, DOUBLE, FLOAT
    assert list(p.slot_logical_width[:6]) == logical
    assert list(p.slot_padded_width[:6]) == (logical if columnar else [8] * 6)
    assert (p.row_size, p.buffer_size) == ((32, p.slot_offset[5] + (4 * n + 7) // 8 * 8) if columnar else (56, 56 * n))
    for i in range(6):
        assert p.targets[i].is_agg == 0 and p.targets[i].first_slot == i


PARTS = [slice(1, 12), slice(9, 17)]   # at most 16 launch columns with the filter and $deleted$ columns


@pytest.mark.parametrize("part", PARTS)
@pytest.mark.parametrize("columnar", [False, True])
@pytest.mark.parametrize("limit", [0, 1, 37])
def test_descriptor_parity_encoded(mixed, columnar, limit, part):
    """Every encoding, both layouts, with and without a scan limit: the planner's descriptor equals the restatement."""
    table, names, _ = mixed
    sql = f"SELECT {', '.join(names[part])} FROM t WHERE k < 3000" + (f" LIMIT {limit}" if limit else "")
    unit = sqlmini.parse(sql, table, names)
    p = executor.Executor().plan(unit, table, eo=executor.execution_options(output_columnar_hint=columnar))
    plan_matches(p, restate_descriptor(table, projected_cols(unit), columnar, limit or sum(f.num_tuples for f in table.fragments)))


@pytest.fixture(scope="module")
def mixed():
    table, names = mixed_table(5000, 3, 1000, fragment_ids=[4, 0, 3, 1, 2])
    return table, names, load_sqlite(table, names)


@pytest.mark.parametrize("columnar", [False, True])
@pytest.mark.parametrize("sql", [f"SELECT {ALL} FROM test", f"SELECT {ALL} FROM test LIMIT 9",
                                 "SELECT ofq, dn, fn, w FROM test WHERE y = 43 LIMIT 3"])
def test_readout_over_storage(golden, columnar, sql):
    """b2q_rs_create_from_storage over the restated buffer reads back what SQLite selects, in scan order."""
    table, con = golden
    unit = sqlmini.parse(sql, table, rt.TEST_NAMES)
    eo = executor.execution_options(output_columnar_hint=columnar)
    ex = executor.Executor()
    plan = ex.plan(unit, table, eo=eo)
    where = sql.split(" WHERE ")[1].split(" LIMIT")[0] if " WHERE " in sql else None
    picks = passing_rows(con, where)[:plan.entry_count]
    assert len(picks) == plan.entry_count
    cols = projected_cols(unit)
    rs = ex.resultSetFromStorage(expected_buffer(table, cols, picks, columnar), unit, table, eo=eo)
    names = [rt.TEST_NAMES[c] for c in cols]
    want = [tuple(con.execute(f"SELECT {', '.join(names)} FROM t WHERE _id = ? AND _r = ?", pk).fetchone()) for pk in picks]
    got = rs.rows()
    assert rs.rowCount() == rs.entryCount() == len(want)
    assert not any(rs.isRowAtEmpty(i) for i in range(len(want))) and rs.isRowAtEmpty(len(want))
    for g, w in zip(got, want):
        for a, b in zip(g, w):
            assert (a is None) == (b is None) and (a is None or np.isclose(a, b, rtol=1e-6)), (g, w)
    cr = rs.columnarResults()
    for c, (ty, _nn, arr) in enumerate(cr):
        assert arr.size == len(want)
        null = abi.NULL_OF[ty]
        for v, w in zip(arr.tolist(), want):
            assert (v == null) == (w[c] is None)


@pytest.mark.parametrize("part", PARTS)
@pytest.mark.parametrize("columnar", [False, True])
def test_readout_encoded(mixed, columnar, part):
    """Decoded encodings read back through getNextRow (DECIMAL as scaled integers) and ColumnarResults, fragments given out
    of id order, deleted rows left out."""
    table, names, con = mixed
    unit = sqlmini.parse(f"SELECT {', '.join(names[part])} FROM t WHERE k < 4000", table, names)
    ex = executor.Executor()
    eo = executor.execution_options(output_columnar_hint=columnar)
    picks = passing_rows(con, "k < 4000")
    cols = projected_cols(unit)
    buf = expected_buffer(table, cols, picks, columnar)
    plan = ex.plan(unit, table, eo=eo)
    full = np.zeros(plan.buffer_size, dtype=np.uint8)   # the planned buffer: the rows, then empty entries
    n, cap = len(picks), plan.entry_count
    d_n = restate_descriptor(table, cols, columnar, n)
    if columnar:
        full[0:8 * cap] = np.full(cap, 2**63 - 1, dtype=np.int64).view(np.uint8)
        full[0:8 * n] = buf[0:8 * n]
        for s in range(len(cols)):
            w = plan.slot_padded_width[s]
            full[plan.slot_offset[s]:plan.slot_offset[s] + n * w] = buf[d_n["slot_offset"][s]:d_n["slot_offset"][s] + n * w]
    else:
        full[:buf.size] = buf
        full.reshape(cap, plan.row_size)[n:, 0:8] = np.full((cap - n, 1), 2**63 - 1, dtype=np.int64).view(np.uint8)
    rs = ex.resultSetFromStorage(full, unit, table, eo=eo)
    assert rs.rowCount() == n
    want = con.execute(f"SELECT {', '.join(names[part])} FROM t WHERE _del = 0 AND k < 4000 ORDER BY _id, _r").fetchall()
    got = rs.rows(decimal_to_double=False)
    for g, w in zip(got, want):
        for a, b in zip(g, w):
            assert (a is None) == (b is None) and (a is None or np.isclose(a, b, rtol=1e-6)), (g, w)
    assert len(got) == len(want)


@pytest.mark.parametrize("sql", [
    "SELECT x FROM test GROUP BY x",                 # GROUP BY without aggregates stays refused
    "SELECT x, COUNT(*) FROM test",                  # columns and aggregates mixed without GROUP BY
    "SELECT f, x FROM test ORDER BY f",              # ORDER BY a FLOAT target
])
def test_refusals(golden, sql):
    table, _ = golden
    unit = sqlmini.parse(sql, table, rt.TEST_NAMES)
    with pytest.raises(executor.UnsupportedOnThisPath):
        executor.Executor().plan(unit, table)


def test_refused_join_projection():
    import join_tables as jt
    fact, dim = jt.fact_table(1000, 3, 500), jt.dim_table()
    unit = sqlmini.parse("SELECT t.x FROM t JOIN d ON t.fk32 = d.id32", fact, jt.FACT_NAMES, inner=(dim, jt.DIM_NAMES))
    with pytest.raises(executor.UnsupportedOnThisPath):
        executor.Executor().plan(unit, fact)


def test_scan_limit_only_for_projections(golden):
    table, _ = golden
    def lim(sql):
        return sqlmini.parse(sql, table, rt.TEST_NAMES).unit.scan_limit
    assert lim("SELECT x, y FROM test LIMIT 5") == 5
    assert lim("SELECT x, y FROM test LIMIT 5 OFFSET 3") == 8
    assert lim("SELECT x, y FROM test ORDER BY y LIMIT 5") == 0        # ORDER BY: the sort needs every row
    assert lim("SELECT x FROM test") == 0
    assert lim("SELECT COUNT(*) FROM test LIMIT 5") == 0
    assert lim("SELECT x, COUNT(*) FROM test GROUP BY x LIMIT 5") == 0


def test_aggregate_units_unchanged(golden):
    """Aggregate units of the ORDER BY corpus carry no scan limit (bench.py builds its units the same way)."""
    table, _ = golden
    for sql in oq.GOLDEN_ORDER_QUERIES:
        assert sqlmini.parse(sql, table, rt.TEST_NAMES).unit.scan_limit == 0, sql


def test_limit_zero_plans_an_empty_scan(golden):
    table, _ = golden
    unit = sqlmini.parse("SELECT x FROM test LIMIT 0", table, rt.TEST_NAMES)
    assert unit.unit.has_limit == 1 and unit.unit.limit == 0
