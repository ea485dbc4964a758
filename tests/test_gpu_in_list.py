"""IN / NOT IN lists past the 16-leaf filter program on the GPU: one set term per list, a bitmap built on the device per call
(b2q_k_set_build) and read by every kernel that evaluates the filter.  Every query asserts its kernel and that
kernel_launches counts the build (the same query with a one-leaf filter launches one kernel less), and is checked against the
oracle; values at the edges of every width against int_exact_ref."""
import random

import numpy as np
import pytest

import gpu_util as gu
import int_exact_ref as ier
import join_tables as jt
import oracle_lib
import sqlmini
from heavydb_b200 import abi, executor
from test_gpu_parity import RAND_NAMES, random_table
from test_in_list_cpu import lst, scattered

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rand():
    table = random_table(300_000, seed=91, frag_rows=70_000)
    return table, gu.DeviceTable(table)


def long_list(rng, col, n=200):
    lo, hi = {"k8": (-150, 150), "k16": (60, 12000), "k32": (-3000, 60000), "k64": (10**9 - 500, 10**9 + 9000),
              "nn32": (-30, 5000), "a16": (-32768, 32767), "a32": (-50000, 50000), "a64": (-10**6, 10**6), "nn64": (-200, 9000)}[col]
    return scattered(rng, n, lo, hi)


def run_checked(sql, table, dev, names=RAND_NAMES, kernel=None, plain_where="k8 = 1", inner=None, **kw):
    """run_both (plan, rows, buffers against the oracle), the kernel, and one launch more than the same query with a one-leaf
    filter: the bitmap build."""
    unit = sqlmini.parse(sql, table, names, inner=inner)
    rs, ref = gu.run_both(unit, table, dev_table=dev, **kw)
    if kernel is not None:
        assert rs.getQueryMemDesc().kernel == kernel, sql[:200]
    where = sql[sql.index(" WHERE ") + 7:]
    tail = min([where.index(k) for k in (" GROUP BY ", ";") if k in where])
    plain = sqlmini.parse(sql.replace(where[:tail], plain_where), table, names, inner=inner)
    prs, _ = gu.run_both(plain, table, dev_table=dev, **kw)
    assert rs.stats()["kernel_launches"] == prs.stats()["kernel_launches"] + 1, sql[:200]
    return rs, ref


def test_table_modes(rand):
    """Non-grouped, the shared-memory perfect hash (fused COUNT / SUM and general), forced HBM/L2, and the baseline hash through
    the radix passes and through the probe kernel."""
    table, dev = rand
    rng = random.Random(1)
    a, b, c = long_list(rng, "k32"), long_list(rng, "a16", 3000), long_list(rng, "k64", 40)
    cases = [
        (f"SELECT COUNT(*), SUM(a64), MIN(k16), MAX(nn64) FROM r WHERE k32 IN ({lst(a)});", abi.KERNEL_NON_GROUPED, {}),
        (f"SELECT COUNT(*) FROM r WHERE k32 NOT IN ({lst(a)}) AND a16 IN ({lst(b)});", abi.KERNEL_NON_GROUPED, {}),
        (f"SELECT k8, COUNT(*), SUM(nn64) FROM r WHERE k32 IN ({lst(a)}) GROUP BY k8;", abi.KERNEL_PERFECT_SMEM, {}),
        (f"SELECT k8, COUNT(*), MIN(a32), MAX(d), AVG(a16) FROM r WHERE a16 NOT IN ({lst(b)}) OR k64 IN ({lst(c)}) GROUP BY k8;", abi.KERNEL_PERFECT_SMEM, {}),
        (f"SELECT k16, COUNT(*), SUM(a64) FROM r WHERE k32 IN ({lst(a)}) GROUP BY k16;", abi.KERNEL_PERFECT_GLOBAL,
         dict(force_kernel=abi.KERNEL_PERFECT_GLOBAL, entry_guess=3001, has_card=True)),
        (f"SELECT sparse, COUNT(*), SUM(a32) FROM r WHERE k64 NOT IN ({lst(c)}) AND k32 IN ({lst(a)}) GROUP BY sparse;", abi.KERNEL_BASELINE_GLOBAL,
         dict(entry_guess=400_000, has_card=True)),
        (f"SELECT sparse, COUNT(*), SUM(a32) FROM r WHERE a16 IN ({lst(b)}) GROUP BY sparse;", abi.KERNEL_BASELINE_GLOBAL,
         dict(entry_guess=400_000, has_card=True, force_kernel=abi.KERNEL_BASELINE_PROBE)),
    ]
    for sql, kernel, kw in cases:
        run_checked(sql, table, dev, kernel=kernel, **kw)


@pytest.mark.parametrize("left", ["", "LEFT "])
def test_join_outer_and_inner_columns(left):
    fact, dim = jt.fact_table(200_000, seed=92, frag_rows=60_000), jt.dim_table(seed=15)
    dev = gu.DeviceTable(fact)
    rng = random.Random(2)
    for where in [f"t.x IN ({lst(scattered(rng, 30, 0, 99))})", f"d.attr8 NOT IN ({lst(scattered(rng, 40, -100, 100))})",
                  f"d.big IN ({lst(scattered(rng, 50, -2**20, 2**20))}) OR t.fk16 IN ({lst(scattered(rng, 200, 0, 1009))})"]:
        sql = f"SELECT d.attr, COUNT(*), SUM(t.v) FROM t {left}JOIN d ON t.fk32 = d.id32 WHERE {where} GROUP BY d.attr;"
        run_checked(sql, fact, dev, names=jt.FACT_NAMES, inner=(dim, jt.DIM_NAMES), kernel=abi.KERNEL_PERFECT_SMEM,
                    plain_where="t.x = 1", entry_guess=4000, has_card=True)


def in_chain(b, col, vals, neg=False):
    e = b.cmp(col, abi.kEQ, vals[0])
    for v in vals[1:]:
        e = b.binop(abi.kOR, e, b.cmp(col, abi.kEQ, v))
    return b.uoper(abi.kNOT, e) if neg else e


def test_ndv_estimator(rand):
    table, dev = rand
    rng = random.Random(3)
    ex = executor.Executor()
    for neg in (False, True):
        b = abi.UnitBuilder(table)
        b.add_qual(in_chain(b, RAND_NAMES.index("k32"), long_list(rng, "k32", 300), neg))
        b.estimator([RAND_NAMES.index("a32"), RAND_NAMES.index("k8")])
        unit = b.build()
        ref = oracle_lib.execute(unit, table, num_threads=4)
        for t, lvl in ((dev.table, abi.GPU_LEVEL), (table, abi.CPU_LEVEL)):
            rs = ex.executeWorkUnit(1, True, t, unit, memory_level=lvl)
            assert rs.getQueryMemDesc().as_dict() == ref.plan.as_dict()
            assert np.array_equal(rs.getHostEstimatorBuffer(), ref.buffer().view(np.uint8))


@pytest.fixture(scope="module")
def big():
    from test_gpu_projection import _big
    t, cols = _big(3_000_000, 700_001)
    return t, gu.DeviceTable(t), cols


@pytest.mark.parametrize("columnar", [False, True])
@pytest.mark.parametrize("neg,limit", [(False, 0), (True, 0), (False, 1000), (True, 123_457)])
def test_projection(big, columnar, neg, limit):
    """Rows and their order from projection_ref, with and without LIMIT; the pre-flight count builds its own bitmap."""
    from test_gpu_projection import _run, _want_buffer
    table, dev, (c0, c1, g, s) = big
    rng = random.Random(4)
    vals = scattered(rng, 100, -300, 300) if neg else scattered(rng, 150_000, 0, 10**6)
    col = "s" if neg else "c0"
    mask = (~np.isin(s, vals) & (s != abi.NULL_OF[abi.kSMALLINT])) if neg else np.isin(c0, vals)
    sql = f"SELECT g, c1, s FROM t WHERE {col} {'NOT IN' if neg else 'IN'} ({lst(vals)})" + (f" LIMIT {limit}" if limit else "")
    unit = sqlmini.parse(sql, table, ["c0", "c1", "g", "s"])
    rs = _run(executor.Executor(), unit, dev.table, columnar, abi.GPU_LEVEL)
    want, idx = _want_buffer(rs.getQueryMemDesc(), table, [2, 1, 3], mask, 700_001, limit)
    assert rs.rowCount() == idx.size
    assert rs.getStorageBuffer().tobytes() == want.tobytes()
    plain = _run(executor.Executor(), sqlmini.parse(sql[:sql.index(" WHERE ")] + " WHERE c0 < 5" + (f" LIMIT {limit}" if limit else ""),
                                                    table, ["c0", "c1", "g", "s"]), dev.table, columnar, abi.GPU_LEVEL)
    assert rs.stats()["kernel_launches"] == plain.stats()["kernel_launches"] + (1 if limit else 2)


def test_host_resident_slices():
    """One fragment of 2^24 + 12 345 rows streamed in two slices: the bitmap is built once per call."""
    n = (1 << 24) + 12_345
    rng = np.random.default_rng(5)
    c0 = rng.integers(0, 10**6, n).astype(np.int64)
    g = rng.integers(0, 1000, n).astype(np.int32)
    v = rng.integers(-10**6, 10**6, n).astype(np.int64)
    t = abi.Table([(abi.kBIGINT, True), (abi.kINT, True), (abi.kBIGINT, True)])
    t.add_host_fragment([c0, g, v])
    vals = np.array(scattered(random.Random(6), 100_000, 0, 10**6), dtype=np.int64)
    ex = executor.Executor()
    for neg in (False, True):
        sql = f"SELECT g, COUNT(*), SUM(v) FROM t WHERE c0 {'NOT IN' if neg else 'IN'} ({lst(vals.tolist())}) GROUP BY g;"
        rs = ex.executeWorkUnit(0, True, t, sqlmini.parse(sql, t, ["c0", "g", "v"]), memory_level=abi.CPU_LEVEL)
        assert rs.getQueryMemDesc().kernel == abi.KERNEL_PERFECT_SMEM
        m = np.isin(c0, vals) != neg
        gm, vm = g[m], v[m]
        cnt = np.bincount(gm, minlength=1000)
        order = np.argsort(gm, kind="stable")
        bounds = np.searchsorted(gm[order], np.arange(1001))
        vs = vm[order]
        want = {k: (int(cnt[k]), int(vs[bounds[k]:bounds[k + 1]].sum())) for k in range(1000) if cnt[k]}
        assert {r[0]: (r[1], r[2]) for r in rs.rows()} == want
        plain = ex.executeWorkUnit(0, True, t, sqlmini.parse("SELECT g, COUNT(*), SUM(v) FROM t WHERE c0 < 5 GROUP BY g;", t, ["c0", "g", "v"]),
                                   memory_level=abi.CPU_LEVEL)
        assert rs.stats()["kernel_launches"] == plain.stats()["kernel_launches"] + 1


def test_columnar_output_and_result_on_device(rand):
    from test_gpu_device_results import run_pair
    table, dev = rand
    rng = random.Random(7)
    a = long_list(rng, "k32")
    for sql in [f"SELECT k8, COUNT(*), SUM(a64), MAX(d) FROM r WHERE k32 IN ({lst(a)}) GROUP BY k8;",
                f"SELECT COUNT(*), MIN(a16) FROM r WHERE k32 NOT IN ({lst(a)});"]:
        run_checked(sql, table, dev, output_columnar=True)
        for columnar in (False, True):
            run_pair(sqlmini.parse(sql, table, RAND_NAMES), dev, table.total_tuples(), output_columnar_hint=columnar)


def test_multi_device_in_process():
    from test_gpu_multi import device_views
    ndev = min(executor.lib().b2q_device_count(), 4)
    comms = executor.Comm.init_all(list(range(ndev)))
    try:
        table = random_table(120_000, seed=93, frag_rows=10_000)
        views, _keep = device_views(table, ndev)
        rng = random.Random(8)
        ex = executor.Executor()
        for sql in [f"SELECT k8, COUNT(*), SUM(a64) FROM r WHERE k32 IN ({lst(long_list(rng, 'k32'))}) GROUP BY k8;",
                    f"SELECT COUNT(*), SUM(nn64) FROM r WHERE a16 NOT IN ({lst(long_list(rng, 'a16', 1000))});"]:
            unit = sqlmini.parse(sql, table, RAND_NAMES)
            rs = executor.execute_work_unit_multi(comms, ex, 4000, True, views, unit, has_cardinality_estimation=True)
            ref = oracle_lib.execute(unit, table, entry_guess=4000, has_card=True, num_threads=4)
            gu.rows_equal(rs.rows(), ref.rows())
    finally:
        for c in comms:
            c.destroy()


def test_bitmap_sizes():
    """A one-word bitmap, values on both sides of word ends at an offset minimum, and a bitmap of about 100 MB."""
    n = 2_000_000
    rng = np.random.default_rng(9)
    near = np.array([5] + [5 + 32 * k + d for k in range(1, 13) for d in (-1, 1)], dtype=np.int64)   # bits 31 and 33, 63 and 65, ...
    wide = np.array(scattered(random.Random(10), 1000, 0, 800_000_000), dtype=np.int64)
    x = rng.integers(0, 40, n).astype(np.int32)
    y = rng.choice(np.concatenate([near, near + 1, np.arange(0, 200)]), n).astype(np.int64)
    z = rng.choice(np.concatenate([wide, wide + 1, rng.integers(0, 800_000_000, 5000)]), n).astype(np.int64)
    y[rng.random(n) < 0.05] = abi.NULL_BIGINT
    t = abi.Table([(abi.kINT, True), (abi.kBIGINT, False), (abi.kBIGINT, True), (abi.kTINYINT, True)])
    t.add_host_fragment([x, y, z, rng.integers(0, 10, n).astype(np.int8)])
    names = ["x", "y", "z", "k"]
    dev = gu.DeviceTable(t)
    one_word = lst(range(0, 32, 2))                              # 16 values: the set only when the program overflows
    overflow = " AND ".join(f"k <> {v}" for v in (11, 13))
    for where in [f"x IN ({one_word}) AND {overflow}", f"y IN ({lst(near.tolist())})", f"y NOT IN ({lst(near.tolist())})",
                  f"z IN ({lst(wide.tolist())})", f"z NOT IN ({lst(wide.tolist())}) AND y IN ({lst(near.tolist())})"]:
        run_checked(f"SELECT k, COUNT(*), SUM(z) FROM t WHERE {where} GROUP BY k;", t, dev, names=names, kernel=abi.KERNEL_PERFECT_SMEM,
                    plain_where="k = 1")


@pytest.mark.parametrize("w", [ier.WIDTH[n] for n in ("INT16", "INT32", "INT64", "BIGINT_FIXED16", "DICT8", "DICT16", "DAYS16", "DAYS32", "DECIMAL18_2")],
                         ids=lambda w: w.name)
def test_exact_at_width_edges(w):
    """COUNT(*), COUNT(v) (its 32-bit nullable form, IntGroup.count32), MIN / MAX per group of rows whose value sits at the width's edges, against int_exact_ref."""
    from test_in_list_cpu import edge_lists
    rng = np.random.default_rng(11)
    pool = ier.pool(w)
    unit_ = ier.SECONDS_PER_DAY if w.is_days else 1
    extra = sorted({v // unit_ for l in edge_lists(w) for v in l if v % unit_ == 0})
    extra = [x for x in extra if w.lo <= x <= w.hi and (w.sql_type != abi.kDECIMAL or abs(x) <= ier.DECIMAL18_MAX)]
    for nullable in (True, False):
        vals = np.array(pool + extra, dtype=object)
        phys = np.array([int(v) for v in rng.choice(vals, 200_000)], dtype=w.dtype)
        if nullable:
            phys[rng.random(phys.size) < 0.1] = w.null
        keys = rng.integers(0, 8, phys.size).astype(np.int32)
        t = w.table(not nullable)
        for b in range(0, phys.size, 70_000):
            t.add_host_fragment([keys[b:b + 70_000], phys[b:b + 70_000]])
        dev = gu.DeviceTable(t)
        ex = executor.Executor()
        minmax = "" if w.sql_type == abi.kDECIMAL or w.is_dict else ", MIN(v), MAX(v)"
        for l in edge_lists(w):
            for p in [("in", l), ("not", ("in", l))]:
                sql = f"SELECT k, COUNT(*), COUNT(v){minmax} FROM t WHERE {ier.predicate_sql(w, p)} GROUP BY k;"
                rs = ex.executeWorkUnit(0, True, dev.table, sqlmini.parse(sql, t, ["k", "v"]), memory_level=abi.GPU_LEVEL)
                assert rs.getQueryMemDesc().kernel == abi.KERNEL_PERFECT_SMEM
                groups = ier.groups_of(w, keys, phys, nullable, mask=ier.passing(w, phys, nullable, p))
                want = sorted((k, g.rows, g.count32) + ((g.min, g.max) if minmax else ()) for k, g in groups.items())
                assert sorted(tuple(r) for r in rs.rows()) == want, (w.name, nullable, p[0])


def test_interrupt_token_stops_a_query_with_a_set_term(rand):
    table, dev = rand
    rng = random.Random(12)
    unit = sqlmini.parse(f"SELECT k8, COUNT(*), SUM(a64) FROM r WHERE k32 IN ({lst(long_list(rng, 'k32'))}) GROUP BY k8;", table, RAND_NAMES)
    ex = executor.Executor()
    tok = ex.interrupt_token("s")
    ex.interrupt("s", "admin")
    eo = executor.execution_options(allow_runtime_query_interrupt=True, interrupt_token=tok)
    with pytest.raises(executor.QueryExecutionError) as ei:
        ex.executeWorkUnit(0, True, dev.table, unit, eo=eo, memory_level=abi.GPU_LEVEL)
    assert ei.value.code == abi.ERR_INTERRUPTED
    ex.resetInterrupt("s")
    rs = ex.executeWorkUnit(0, True, dev.table, unit, eo=eo, memory_level=abi.GPU_LEVEL)
    gu.rows_equal(rs.rows(), oracle_lib.execute(unit, table, num_threads=4).rows())
