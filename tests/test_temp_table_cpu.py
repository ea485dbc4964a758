"""Temporary tables without a GPU: the synthesize_metadata restatement on hand-checked columns, and the whole multi-step chain
(HAVING, subqueries in FROM, a join against an aggregated subquery) through the oracle and the host route:

  1. the oracle runs step 1;
  2. b2q_rs_create_from_storage + b2q_columnar_results_create turn its result into host columns;
  3. the restated metadata makes the host temporary table;
  4. the oracle runs step 2 over it (and so on for deeper nesting); a projection step, which the oracle does not run, is
     planned by the product's planner and its rows taken from SQLite over the temporary table;
  5. the final rows match SQLite running the original string.

Also: b2q_device_columns_chunk_stats is exported, refuses a NULL handle, and no B2QDeviceColumns exists without a device."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import oracle_lib
import ref_full_table as ft
import ref_tables as rt
import sqlmini
import temp_table_ref as tt
from gpu_util import has_gpu
from heavydb_b200 import abi, executor

HERE = os.path.dirname(os.path.abspath(__file__))
HARVEST = json.load(open(os.path.join(HERE, "golden", "executetest_steps_harvest.json")))
HARVESTED = [q["sql"] for q in HARVEST["queries"]]
GUESS = 48

F32 = np.finfo(np.float32)
F64 = np.finfo(np.float64)

# (sql_type, values, expected (min, max, has_nulls)) — NULL is the type's inline sentinel
HAND = [
    (abi.kTINYINT, [-128, -127, 127], (-127, 127, 1)),
    (abi.kTINYINT, [-127, 0, 126], (-127, 126, 0)),
    (abi.kSMALLINT, [-32768, -32767, 32767], (-32767, 32767, 1)),
    (abi.kINT, [-2**31, -2**31 + 1, 2**31 - 1], (-2**31 + 1, 2**31 - 1, 1)),
    (abi.kINT, [2**31 - 1, 2**31 - 1], (2**31 - 1, 2**31 - 1, 0)),
    (abi.kBIGINT, [-2**63, -2**63 + 1, 2**63 - 1], (-2**63 + 1, 2**63 - 1, 1)),
    (abi.kBIGINT, [2**63 - 1], (2**63 - 1, 2**63 - 1, 0)),
    (abi.kDECIMAL, [-2**63, 12345, -99999], (-99999, 12345, 1)),                     # scaled int64
    (abi.kDATE, [-2**63, 86400 * 19000, -86400], (-86400, 86400 * 19000, 1)),         # epoch seconds
    (abi.kTIMESTAMP, [0, -1], (-1, 0, 0)),
    (abi.kTEXT, [-2**31, 0, 2, 1], (0, 2, 1)),                                       # dictionary ids
    (abi.kFLOAT, [F32.tiny, np.nextafter(F32.tiny, np.float32(1)), 3.5], (float(np.nextafter(F32.tiny, np.float32(1))), 3.5, 1)),
    (abi.kFLOAT, [np.nan, -np.inf, np.inf, -0.0], (-np.inf, np.inf, 0)),
    (abi.kFLOAT, [np.nan, np.nan], (float(F32.max), -float(F32.max), 0)),
    (abi.kDOUBLE, [F64.tiny, -F64.tiny, 1.0], (-F64.tiny, 1.0, 1)),
    (abi.kDOUBLE, [np.nan, 2.0, np.nan, -7.25], (-7.25, 2.0, 0)),
    (abi.kDOUBLE, [0.0, -0.0], (0.0, 0.0, 0)),
]


@pytest.mark.parametrize("ty,vals,want", HAND, ids=[f"{i}-{t}" for i, (t, _, _) in enumerate(HAND)])
def test_restated_metadata(ty, vals, want):
    a = np.array(vals, dtype=abi.NUMPY_OF[ty])
    (st,) = tt.synthesize_metadata([(ty, False, a)])
    got = tt.stats_tuple(st, ty)[1:]
    assert got == want, (got, want)


@pytest.mark.parametrize("ty", [abi.kTINYINT, abi.kSMALLINT, abi.kINT, abi.kBIGINT, abi.kDECIMAL, abi.kTEXT, abi.kFLOAT, abi.kDOUBLE])
@pytest.mark.parametrize("all_null", [False, True])
def test_fresh_encoder_stats(ty, all_null):
    """No rows, or every value NULL: min = numeric_limits<T>::max(), max = lowest(); has_nulls as counted."""
    a = np.full(5 if all_null else 0, abi.NULL_OF[ty], dtype=abi.NUMPY_OF[ty])
    (st,) = tt.synthesize_metadata([(ty, False, a)])
    if ty in tt.FP:
        lim = float(np.finfo(abi.NUMPY_OF[ty]).max)
        assert (st.fp_min, st.fp_max) == (lim, -lim)
    else:
        info = np.iinfo(abi.NUMPY_OF[ty])
        assert (st.int_min, st.int_max) == (int(info.max), int(info.min))
    assert st.has_nulls == int(all_null)


def test_symbol_and_bad_arguments():
    L = executor.lib()
    fn = L.b2q_device_columns_chunk_stats
    st = abi.ChunkStats()
    assert fn(None, 0, C.byref(st)) == abi.ERR_INVALID_ARGUMENT
    assert fn(None, 0, None) == abi.ERR_INVALID_ARGUMENT
    assert L.b2q_abi_version() == abi.ABI_VERSION == 9


@pytest.mark.skipif(has_gpu(), reason="checks the behaviour of a machine without a CUDA device")
def test_no_device_columns_without_a_device():
    rows = ft.full_rows()
    table = ft.make_table(rows)
    unit = sqlmini.parse("SELECT x, COUNT(*) FROM test GROUP BY x;", table, ft.FULL_NAMES)
    res = oracle_lib.execute(unit, table, entry_guess=GUESS, has_card=True)
    rs = executor.Executor().resultSetFromStorage(res.buffer(), unit, table, max_groups_buffer_entry_guess=GUESS,
                                                  has_cardinality_estimation=True)
    with pytest.raises(executor.QueryExecutionError) as e:
        rs.deviceColumns()
    assert e.value.code == abi.ERR_NO_DEVICE


HAND_SQL = [
    # HAVING on keys and on each aggregate
    "SELECT x, COUNT(*) FROM test GROUP BY x HAVING x > 7;",
    "SELECT y, COUNT(*) FROM test GROUP BY y HAVING COUNT(*) > 5;",
    "SELECT x, SUM(y) FROM test GROUP BY x HAVING SUM(y) > 300;",
    "SELECT x, AVG(d) FROM test GROUP BY x HAVING AVG(d) > 2.3;",
    "SELECT z, MIN(t) FROM test GROUP BY z HAVING MIN(t) < 1002;",
    "SELECT x, MAX(y) FROM test GROUP BY x HAVING MAX(y) >= 43;",
    "SELECT x, COUNT(DISTINCT y) FROM test GROUP BY x HAVING COUNT(DISTINCT y) > 1;",
    "SELECT w, SUM(x) FROM test GROUP BY w HAVING MIN(z) > 100;",
    "SELECT x, COUNT(*) FROM test WHERE y > 42 GROUP BY x HAVING SUM(t) > 0;",
    "SELECT str, COUNT(*) FROM test GROUP BY str HAVING COUNT(*) > 5;",
    "SELECT smallint_nulls, COUNT(*) FROM test GROUP BY smallint_nulls HAVING COUNT(*) >= 5;",
    "SELECT x, MIN(dn) FROM test GROUP BY x HAVING MIN(dn) < -1000;",
    "SELECT y, COUNT(*) AS n FROM test GROUP BY y HAVING COUNT(*) > 1 ORDER BY n DESC, y DESC LIMIT 1;",
    "SELECT x, COUNT(*) FROM test GROUP BY x HAVING COUNT(*) > 1000;",                    # empty intermediate after the filter
    # derived tables
    "SELECT COUNT(*) FROM (SELECT x, COUNT(*) AS n FROM test GROUP BY x) WHERE n > 5;",
    "SELECT SUM(n), MAX(x) FROM (SELECT x, COUNT(*) AS n FROM test GROUP BY x) s;",
    "SELECT n, COUNT(*) FROM (SELECT y, COUNT(*) AS n FROM test GROUP BY y) GROUP BY n;",
    "SELECT COUNT(*), MIN(y) FROM (SELECT x, y FROM test WHERE y > 42) WHERE x < 8;",
    "SELECT COUNT(*) FROM (SELECT x, COUNT(*) AS n FROM test WHERE x > 100 GROUP BY x);",   # empty intermediate
    # a join against an aggregated subquery
    "SELECT s.n, COUNT(*) FROM test JOIN (SELECT y, COUNT(*) AS n FROM test GROUP BY y) s ON test.y = s.y GROUP BY s.n;",
    "SELECT COUNT(*), SUM(test.x) FROM test JOIN (SELECT x, MAX(y) AS m FROM test GROUP BY x) s ON test.x = s.x WHERE s.m > 42;",
    # three steps
    "SELECT COUNT(*) FROM (SELECT n, COUNT(*) AS c FROM (SELECT x, COUNT(*) AS n FROM test GROUP BY x) GROUP BY n) WHERE c > 0;",
    "SELECT n, COUNT(*) FROM (SELECT x, COUNT(*) AS n FROM test GROUP BY x HAVING COUNT(*) > 5) GROUP BY n;",
]


@pytest.fixture(scope="module")
def golden():
    rows = ft.full_rows()
    return ft.make_table(rows), ft.make_sqlite(rows), len(rows)


def run_chain_on_host(sql, table):
    """Every step on the oracle; every intermediate handed over as host ColumnarResults with restated stats."""
    steps = sqlmini.parse_steps(sql, table, ft.FULL_NAMES)

    def run(i, unit, tbl, names):
        return tt.run_step_on_host(steps[i], unit, tbl, names, GUESS)

    def to_table(_i, unit, tbl, res):
        return tt.host_table(tt.oracle_columns(unit, tbl, res, GUESS))

    return steps, tt.run_steps(steps, {"test": (table, ft.FULL_NAMES)}, run, to_table, dicts=ft.DICTS)


def check_against_sqlite(sql, steps, out, con, n_rows):
    unit, _tbl, res = out[-1]
    plan = res.getQueryMemDesc() if isinstance(res, executor.ResultSet) else res.plan
    got = tt.translate(res.rows(), plan, steps[-1].names, ft.DICTS)
    ref = [tuple(r) for r in con.execute(tt.sqlite_sql(sql, unit)).fetchall()]
    fp_abs = rt.float_sum_atol(n_rows) if tt.float_sum_query(sql) else 0.0
    if unit.unit.num_order_entries:
        from test_order_by import assert_ordered_rows_match
        assert_ordered_rows_match(got, ref, fp_abs=fp_abs)
    else:
        rt.assert_rows_match(got, ref, fp_abs=fp_abs)


@pytest.mark.parametrize("sql", HAND_SQL)
def test_host_chain_hand_written(golden, sql):
    table, con, n = golden
    steps, out = run_chain_on_host(sql, table)
    assert len(steps) >= 2
    check_against_sqlite(sql, steps, out, con, n)


def test_harvest_is_what_the_script_reports():
    assert HARVEST["stats"]["kept"] == len(HARVESTED) > 0 and len(set(HARVESTED)) == len(HARVESTED)


@pytest.mark.parametrize("sql", HARVESTED)
def test_host_chain_harvested(golden, sql):
    table, con, n = golden
    steps, out = run_chain_on_host(sql, table)
    check_against_sqlite(sql, steps, out, con, n)


def test_parse_steps_shapes():
    t = ft.make_table(ft.full_rows())
    s = sqlmini.parse_steps("SELECT x, SUM(y) FROM test GROUP BY x HAVING MAX(z) > 1 ORDER BY 2 LIMIT 3;", t, ft.FULL_NAMES)
    assert [st.source for st in s] == ["test", 0] and s[0].names == ["x", "agg0", "agg1"]
    assert s[1].sql.startswith("SELECT x, agg0 FROM tmp0 WHERE agg1 > 1 ORDER BY 2 LIMIT 3")
    s = sqlmini.parse_steps("SELECT COUNT(*) FROM (SELECT n, COUNT(*) AS c FROM (SELECT x, COUNT(*) AS n FROM test GROUP BY x) "
                            "GROUP BY n) WHERE c > 0;", t, ft.FULL_NAMES)
    assert [st.source for st in s] == ["test", 0, 1] and s[1].names == ["n", "c"]
    s = sqlmini.parse_steps("SELECT COUNT(*) FROM test JOIN (SELECT y, COUNT(*) AS n FROM test GROUP BY y) s ON test.y = s.y;",
                            t, ft.FULL_NAMES)
    assert [(st.source, st.inner) for st in s] == [("test", None), ("test", 0)]
    with pytest.raises(ValueError):
        sqlmini.parse_steps("SELECT x FROM test HAVING COUNT(*) > 1;", t, ft.FULL_NAMES)
