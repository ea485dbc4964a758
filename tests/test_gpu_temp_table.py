"""Temporary tables on the H100: the conversion kernel's chunk stats (b2q_device_columns_chunk_stats) against the
synthesize_metadata restatement over the host ColumnarResults of the same result, for every kernel family as step 1; and
second steps over DeviceColumns.as_table() that plan and answer exactly what the host route (host columns + host stats, the
reference's getResultSetColumn + synthesize_metadata) plans and answers, and what SQLite answers for the original string."""
import numpy as np
import pytest

import dec_tables as dect
import gpu_util as gu
import join_tables as jt
import order_queries as oq
import ref_full_table as ft
import ref_time_table as timet
import sqlmini
import str_tables as stt
import temp_table_ref as tt
from heavydb_b200 import abi, executor
from test_gpu_device_results import EMPTY_AND_NON_GROUPED, SPARSE
from test_gpu_parity import RAND_NAMES, RAND_QUERIES, random_table
from test_temp_table_cpu import GUESS, HAND_SQL, HARVESTED, check_against_sqlite

pytestmark = pytest.mark.gpu

PROJECTIONS = [
    "SELECT a8, a16, a32, a64, d, f32 FROM r WHERE k8 < 3;",
    "SELECT k64, sparse, dnn FROM r WHERE a32 > 500 LIMIT 100;",
    "SELECT a8, d FROM r WHERE k32 < -1000000;",                      # no row passes
]


def check_stats(rs):
    """Device stats of a device-resident result == the restatement over its host ColumnarResults; nothing crossed PCIe."""
    assert rs.stats()["result_d2h_bytes"] == 0
    dc = rs.deviceColumns()
    assert rs.stats()["result_d2h_bytes"] == 0
    got = [dc.chunk_stats(i) for i in range(dc.num_columns())]
    cols = rs.columnarResults(num_threads=4, with_scale=True)
    want = tt.synthesize_metadata(cols)
    for c, (g, w) in enumerate(zip(got, want)):
        assert tt.stats_tuple(g, cols[c][0]) == tt.stats_tuple(w, cols[c][0]), (c, cols[c][0])
    with pytest.raises(executor.QueryExecutionError):
        dc.chunk_stats(dc.num_columns())
    return dc


def run_stats_set(sqls, table, names, min_ran, inner=None, resident=True, entry_guess=0, has_card=False, **eo_kw):
    ex = executor.Executor()
    dev = gu.DeviceTable(table) if resident else None
    ran = 0
    for sql in sqls:
        unit = sqlmini.parse(sql, table, names, inner=inner)
        try:
            rs = ex.executeWorkUnit(entry_guess, True, dev.table if resident else table, unit,
                                    eo=executor.execution_options(**eo_kw), has_cardinality_estimation=has_card,
                                    memory_level=abi.GPU_LEVEL if resident else abi.CPU_LEVEL, result_on_device=True)
        except (executor.UnsupportedOnThisPath, executor.CardinalityEstimationRequired):
            continue
        try:
            check_stats(rs)
        except AssertionError as e:
            raise AssertionError(f"query: {sql}\n{e}") from e
        ran += 1
    assert ran >= min_ran


@pytest.fixture(scope="module")
def rand():
    return random_table(30000, seed=91, frag_rows=8000)


@pytest.mark.parametrize("columnar", [False, True])
def test_stats_every_kernel_family(rand, columnar):
    run_stats_set(RAND_QUERIES + EMPTY_AND_NON_GROUPED, rand, RAND_NAMES, 12, entry_guess=4001, has_card=True,
                  output_columnar_hint=columnar)
    run_stats_set(RAND_QUERIES[5:12], rand, RAND_NAMES, 4, entry_guess=4001, has_card=True,
                  force_kernel=abi.KERNEL_PERFECT_GLOBAL, output_columnar_hint=columnar)
    for fk in (0, abi.KERNEL_BASELINE_PROBE):
        run_stats_set([SPARSE], rand, RAND_NAMES, 1, entry_guess=45000, has_card=True, force_kernel=fk, output_columnar_hint=columnar)


def test_stats_host_resident_sorted_and_projection(rand):
    run_stats_set(RAND_QUERIES[:12], rand, RAND_NAMES, 6, resident=False, entry_guess=4001, has_card=True)
    run_stats_set(oq.RAND_ORDER_QUERIES, rand, RAND_NAMES, 3, entry_guess=3001, has_card=True)
    run_stats_set(PROJECTIONS, rand, RAND_NAMES, 3)


def test_stats_joins_dictionary_time_decimal():
    fact = jt.fact_table(40000, seed=13, frag_rows=9000)
    run_stats_set(jt.JOIN_QUERIES + jt.LEFT_JOIN_QUERIES, fact, jt.FACT_NAMES, 5, inner=(jt.dim_table(), jt.DIM_NAMES),
                  entry_guess=4000, has_card=True)
    table = stt.str_table(20000, seed=5, frag_rows=6000)
    run_stats_set(stt.STR_QUERIES, table, stt.STR_NAMES, 5)
    table = timet.make_table(timet.time_rows())
    run_stats_set(timet.TIME_QUERIES, table, timet.TIME_NAMES, 5)
    table = dect.make_table(dect.mixed_rows(), fragment_size=170)
    run_stats_set(dect.GOLDEN_QUERIES + dect.MORE_QUERIES, table, dect.DEC_NAMES, 5)


def test_stats_fp_edges():
    """NaN never enters the range, +-inf do, FLT_MIN / DBL_MIN are NULL, an all-NULL and a NaN-only group give the fresh
    encoder's stats."""
    n = 64
    f = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, np.finfo(np.float32).tiny, 1.5, -2.5] * 8, dtype=np.float32)
    d = f.astype(np.float64)
    d[d == np.finfo(np.float32).tiny] = np.finfo(np.float64).tiny
    g = np.repeat(np.arange(8, dtype=np.int32), 8)            # group g holds value g of the pattern 8 times
    table = abi.Table([(abi.kINT, True), (abi.kFLOAT, False), (abi.kDOUBLE, False)])
    table.add_host_fragment([g, f, d])
    names = ["g", "f", "d"]
    assert n == g.size
    run_stats_set(["SELECT f, d FROM t;",
                   "SELECT g, MIN(f), MAX(d), SUM(f) FROM t GROUP BY g;",
                   "SELECT g, MIN(d) FROM t WHERE g = 0 GROUP BY g;",        # NaN only
                   "SELECT g, MAX(f) FROM t WHERE g = 5 GROUP BY g;"],       # NULL only
                  table, names, 4)


class Chain:
    """Runs parse_steps' steps on the GPU: every intermediate result_on_device, converted with b2q_rs_device_columns and fed
    as DeviceColumns.as_table() to the next step.  Each step over a temporary table also runs over the host route's table (the
    same result's host ColumnarResults + restated stats): same plan, same rows."""

    def __init__(self, base, names, dicts=None, entry_guess=GUESS, name="test"):
        self.ex = executor.Executor()
        self.dev = gu.DeviceTable(base)
        self.names, self.dicts, self.guess, self.name = names, dicts, entry_guess, name
        self.host_of = {}          # id(device temp table) -> host-route table
        self.skipped = []
        self.pending = None

    def execute(self, unit, table, memory_level, on_device):
        return self.ex.executeWorkUnit(self.guess, True, table, unit, has_cardinality_estimation=True,
                                       memory_level=memory_level, result_on_device=on_device)

    def run(self, sql):
        steps = sqlmini.parse_steps(sql, self.dev.table, self.names)

        def run_one(i, unit, table, names):
            st = steps[i]
            last = i + 1 == len(steps)
            level = abi.GPU_LEVEL
            rs = self.execute(unit, table, level, not last)
            if not last:
                assert rs.stats()["result_d2h_bytes"] == 0
            self.skipped.append(rs.stats()["fragments_skipped"])
            if id(table) in self.host_of or isinstance(st.inner, int):
                self.pending = (st, unit, table, names, rs, steps)
                if last:      # an intermediate is compared once its device columns exist (no host accessor before them)
                    self.compare_pending()
            return rs

        def to_table(_i, _unit, _table, rs):
            dc = rs.deviceColumns()
            assert rs.stats()["result_d2h_bytes"] == 0
            t = dc.as_table()
            self.host_of[id(t)] = tt.host_table(rs.columnarResults(num_threads=4, with_scale=True))
            self.compare_pending()
            return t

        return steps, tt.run_steps(steps, {self.name: (self.dev.table, self.names)}, run_one, to_table, dicts=self.dicts)

    def compare_pending(self):
        if self.pending is not None:
            self.compare_host_route(*self.pending)
            self.pending = None

    def compare_host_route(self, st, unit, table, names, rs, steps):
        host = self.host_of.get(id(table), table)
        inner = None
        if st.inner is not None:
            dev_inner = unit.inner
            inner = (self.host_of.get(id(dev_inner), dev_inner), steps[st.inner].names if isinstance(st.inner, int) else self.names)
        hunit = sqlmini.parse(st.sql, host, names, inner=inner, dicts=self.dicts)
        level = abi.CPU_LEVEL if host is not table else abi.GPU_LEVEL
        hrs = self.execute(hunit, host, level, False)
        assert hrs.getQueryMemDesc().as_dict() == rs.getQueryMemDesc().as_dict()
        assert rs.stats()["fragments_skipped"] == hrs.stats()["fragments_skipped"]
        if unit.unit.num_order_entries:
            gu.rows_equal_ordered(rs.rows(), hrs.rows())
        else:
            gu.rows_equal(rs.rows(), hrs.rows())


@pytest.fixture(scope="module")
def golden():
    rows = ft.full_rows()
    return ft.make_table(rows), ft.make_sqlite(rows), len(rows)


EDGE_SQL = [
    "SELECT COUNT(*), MAX(m), MIN(m) FROM (SELECT x, MAX(u) AS m FROM test GROUP BY x);",        # an all-NULL column
    "SELECT COUNT(*), SUM(n) FROM (SELECT x, COUNT(*) AS n FROM test WHERE x > 100 GROUP BY x);",  # an empty intermediate
    "SELECT m, COUNT(*) FROM (SELECT x, MAX(u) AS m FROM test GROUP BY x) GROUP BY m;",           # GROUP BY an all-NULL key
    "SELECT x, COUNT(*) FROM (SELECT x, y FROM test WHERE y > 42) GROUP BY x ORDER BY x LIMIT 1 OFFSET 1;",
]


@pytest.mark.parametrize("sql", HAND_SQL + EDGE_SQL + HARVESTED)
def test_second_steps_against_host_route_and_sqlite(golden, sql):
    table, con, n = golden
    chain = Chain(table, ft.FULL_NAMES, ft.DICTS)
    steps, out = chain.run(sql)
    check_against_sqlite(sql, steps, out, con, n)


def test_having_constant_outside_the_range_skips_the_fragment(golden):
    table, con, n = golden
    sql = "SELECT x, COUNT(*) FROM test GROUP BY x HAVING COUNT(*) > 1000;"
    chain = Chain(table, ft.FULL_NAMES, ft.DICTS)
    steps, out = chain.run(sql)
    assert chain.skipped[-1] == 1 and out[-1][2].rowCount() == 0
    check_against_sqlite(sql, steps, out, con, n)


def test_temp_table_as_outer_and_inner_of_a_join(rand):
    """A larger intermediate: the temporary table as the scanned table and as the one-to-one join table."""
    names = RAND_NAMES
    chain = Chain(rand, names, entry_guess=4001, name="r")
    for sql in ["SELECT COUNT(*), SUM(n), MAX(s) FROM (SELECT nn32, COUNT(*) AS n, SUM(a64) AS s FROM r GROUP BY nn32) WHERE n > 90;",
                "SELECT n, COUNT(*) FROM (SELECT nn32, COUNT(*) AS n FROM r GROUP BY nn32) GROUP BY n;",
                "SELECT k8, SUM(a32) FROM r GROUP BY k8 HAVING COUNT(*) > 1500 ORDER BY 2 DESC LIMIT 5;",
                "SELECT nn32, COUNT(*), AVG(d) FROM r GROUP BY nn32 HAVING AVG(d) > 0 ORDER BY nn32 LIMIT 20 OFFSET 3;",
                "SELECT s.n, COUNT(*) FROM r JOIN (SELECT nn32, COUNT(*) AS n FROM r GROUP BY nn32) s ON r.nn32 = s.nn32 GROUP BY s.n;",
                "SELECT s.n, COUNT(*) FROM r LEFT JOIN (SELECT nn32, COUNT(*) AS n FROM r WHERE a8 > 0 GROUP BY nn32) s "
                "ON r.nn32 = s.nn32 GROUP BY s.n;"]:
        steps, out = chain.run(sql)
        assert len(steps) >= 2
        con = rt_sqlite(rand, names)
        unit, _t, rs = out[-1]
        ref = [tuple(r) for r in con.execute(tt.sqlite_sql(sql, unit)).fetchall()]
        if unit.unit.num_order_entries:
            gu.rows_equal_ordered(rs.rows(), ref)
        else:
            gu.rows_equal(rs.rows(), ref)


def rt_sqlite(table, names):
    import projection_ref
    return projection_ref.load_sqlite(table, names, name="r")
