"""Stopping a running call on the GPU: the runtime interrupt token and the dynamic watchdog (B2QExecutionOptions).

Every kernel family is stopped by a token interrupted before the call and returns INTERRUPTED; after b2q_interrupt_reset the
same call (same executor, same stream) matches the oracle bit for bit.  The watchdog stops a 1e9-row scan with a 1 ms budget
and leaves it alone with the reference's default 10 000 ms; watchdog + interrupt reports INTERRUPTED; a token interrupted from
another thread stops a 1e9-row c4-shaped call while it runs; a multi-device call with an interrupted token returns
INTERRUPTED on every device.  Each case runs once."""
from __future__ import annotations

import os
import sys
import threading
import time

import numpy as np
import pytest

import gpu_util as gu
import join_tables as jt
import oracle_lib
from heavydb_b200 import abi, executor, sqlmini

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not gu.has_gpu(), reason="needs a CUDA device")]

NAMES = ["k", "v", "d", "s", "f"]


def base_table(n=400_000, frag_rows=150_000, seed=17):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, 100, n).astype(np.int32)
    v = rng.integers(-10**6, 10**6, n).astype(np.int64)
    d = rng.normal(0, 10, n)
    s = ((rng.integers(0, 20_000, n).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)) >> np.uint64(1)).astype(np.int64)
    f = rng.integers(0, 1000, n).astype(np.int32)
    t = abi.Table([(abi.kINT, True), (abi.kBIGINT, True), (abi.kDOUBLE, True), (abi.kBIGINT, True), (abi.kINT, True)])
    for b in range(0, n, frag_rows):
        t.add_host_fragment([k[b:b + frag_rows], v[b:b + frag_rows], d[b:b + frag_rows], s[b:b + frag_rows], f[b:b + frag_rows]])
    return t


@pytest.fixture(scope="module")
def tables():
    t = base_table()
    fact, dim = jt.fact_table(300_000, 5, 120_000), jt.dim_table()
    return t, gu.DeviceTable(t), fact, gu.DeviceTable(fact), dim


def eo_of(token=None, watchdog=False, limit=10_000, **kw):
    return executor.execution_options(allow_runtime_query_interrupt=token is not None, interrupt_token=token,
                                      with_dynamic_watchdog=watchdog, dynamic_watchdog_time_limit=limit, **kw)


def expect_code(code, fn):
    with pytest.raises(executor.QueryExecutionError) as ei:
        fn()
    assert ei.value.code == code, ei.value
    return ei.value


def compare_with_oracle(rs, unit, table, entry_guess, has_card):
    ref = oracle_lib.execute(unit, table, entry_guess=entry_guess, has_card=has_card, num_threads=4)
    plan = rs.getQueryMemDesc()
    assert plan.as_dict() == ref.plan.as_dict()
    if plan.query_desc_type == abi.Estimator:
        assert np.array_equal(rs.getHostEstimatorBuffer(), ref.buffer().view(np.uint8))
        return
    n_rows = sum(f.num_tuples for f in table.fragments)
    gu.rows_equal(rs.rows(), ref.rows(), col_tol=gu.column_tolerances(plan, n_rows))
    if plan.query_desc_type != abi.GroupByBaselineHash:
        gu.buffers_equal(rs.getStorageBuffer(), ref.buffer(), plan)


# (name, sql, force_kernel, entry_guess, has_cardinality_estimation, kernel family of the plan)
AGG_CASES = [
    ("non_grouped", "SELECT COUNT(*), SUM(v), AVG(d) FROM t WHERE f < 700;", 0, 0, False, abi.KERNEL_NON_GROUPED),
    ("smem", "SELECT k, COUNT(*), SUM(v), MIN(d) FROM t WHERE f < 700 GROUP BY k;", 0, 0, False, abi.KERNEL_PERFECT_SMEM),
    ("hbm", "SELECT k, COUNT(*), SUM(v), MIN(d) FROM t WHERE f < 700 GROUP BY k;", abi.KERNEL_PERFECT_GLOBAL, 0, False,
     abi.KERNEL_PERFECT_GLOBAL),
    ("radix", "SELECT s, SUM(v), COUNT(*) FROM t GROUP BY s;", 0, 40_000, True, abi.KERNEL_BASELINE_GLOBAL),
    ("probe", "SELECT s, SUM(v), COUNT(*) FROM t GROUP BY s;", abi.KERNEL_BASELINE_PROBE, 40_000, True, abi.KERNEL_BASELINE_GLOBAL),
]


@pytest.mark.parametrize("level", [abi.GPU_LEVEL, abi.CPU_LEVEL])
@pytest.mark.parametrize("case", AGG_CASES, ids=[c[0] for c in AGG_CASES])
def test_preset_interrupt_then_reset(tables, case, level):
    _, sql, force, guess, has_card, kernel = case
    t, dev, *_ = tables
    unit = sqlmini.parse(sql, t, NAMES)
    ex = executor.Executor()
    tok = ex.interrupt_token("s1")
    ex.interrupt("s1", "admin")
    src = dev.table if level == abi.GPU_LEVEL else t
    run = lambda: ex.executeWorkUnit(guess, True, src, unit, eo=eo_of(tok, force_kernel=force), has_cardinality_estimation=has_card,
                                     memory_level=level)
    expect_code(abi.ERR_INTERRUPTED, run)
    ex.resetInterrupt("s1")
    rs = run()
    assert rs.getQueryMemDesc().kernel == kernel
    compare_with_oracle(rs, unit, t, guess, has_card)


@pytest.mark.parametrize("left", [False, True])
@pytest.mark.parametrize("level", [abi.GPU_LEVEL, abi.CPU_LEVEL])
def test_preset_interrupt_join(tables, left, level):
    *_, fact, fdev, dim = tables
    sql = f"SELECT d.attr, COUNT(*), SUM(t.v) FROM t {'LEFT ' if left else ''}JOIN d ON t.fk32 = d.id32 GROUP BY d.attr;"
    unit = sqlmini.parse(sql, fact, jt.FACT_NAMES, inner=(dim, jt.DIM_NAMES))
    tok = executor.InterruptToken()
    tok.interrupt()
    ex = executor.Executor()
    src = fdev.table if level == abi.GPU_LEVEL else fact
    run = lambda: ex.executeWorkUnit(4000, True, src, unit, eo=eo_of(tok), has_cardinality_estimation=True, memory_level=level)
    expect_code(abi.ERR_INTERRUPTED, run)
    tok.reset()
    compare_with_oracle(run(), unit, fact, 4000, True)


def test_preset_interrupt_ndv_estimator(tables):
    t, dev, *_ = tables
    b = abi.UnitBuilder(t)
    b.estimator([NAMES.index("s")])
    unit = b.build()
    tok = executor.InterruptToken()
    tok.interrupt()
    ex = executor.Executor()
    for src, level in ((dev.table, abi.GPU_LEVEL), (t, abi.CPU_LEVEL)):
        expect_code(abi.ERR_INTERRUPTED, lambda: ex.executeWorkUnit(1, True, src, unit, eo=eo_of(tok), memory_level=level))
    tok.reset()
    compare_with_oracle(ex.executeWorkUnit(1, True, dev.table, unit, eo=eo_of(tok), memory_level=abi.GPU_LEVEL), unit, t, 1, False)


@pytest.mark.parametrize("level", [abi.GPU_LEVEL, abi.CPU_LEVEL])
@pytest.mark.parametrize("sql", ["SELECT k, v, d FROM t WHERE f < 300", "SELECT k, v FROM t WHERE f < 300 LIMIT 1000"])
def test_preset_interrupt_projection(tables, sql, level):
    """Projections have no oracle run here: the reference answer is the same call without a token (tests/test_gpu_projection.py
    checks that one against the restated buffer)."""
    t, dev, *_ = tables
    unit = sqlmini.parse(sql, t, NAMES)
    src = dev.table if level == abi.GPU_LEVEL else t
    ex = executor.Executor()
    want = ex.executeWorkUnit(0, False, src, unit, memory_level=level).getStorageBuffer().copy()
    tok = executor.InterruptToken()
    tok.interrupt()
    run = lambda: ex.executeWorkUnit(0, False, src, unit, eo=eo_of(tok), memory_level=level)
    expect_code(abi.ERR_INTERRUPTED, run)
    tok.reset()
    assert np.array_equal(run().getStorageBuffer(), want)


def test_preset_interrupt_host_slices():
    """A host-resident table of three 16 Mi-row slices: the scans stop at their first chunk, and the host, which waits for the
    scan of slice 0 before it refills that staging set, enqueues no third slice."""
    n = 40_000_000
    rng = np.random.default_rng(3)
    g = rng.integers(0, 64, n).astype(np.int32)
    v = rng.integers(0, 1000, n).astype(np.int32)
    t = abi.Table([(abi.kINT, True), (abi.kINT, True)])
    t.add_host_fragment([g, v])
    unit = sqlmini.parse("SELECT g, SUM(v), COUNT(*) FROM t GROUP BY g;", t, ["g", "v"])
    tok = executor.InterruptToken()
    tok.interrupt()
    ex = executor.Executor()
    expect_code(abi.ERR_INTERRUPTED, lambda: ex.executeWorkUnit(0, True, t, unit, eo=eo_of(tok), memory_level=abi.CPU_LEVEL))
    tok.reset()
    rs = ex.executeWorkUnit(0, True, t, unit, eo=eo_of(tok), memory_level=abi.CPU_LEVEL)
    sums = np.bincount(g, weights=v, minlength=64).astype(np.int64)
    cnts = np.bincount(g, minlength=64)
    assert sorted(rs.rows()) == [(i, int(sums[i]), int(cnts[i])) for i in range(64) if cnts[i]]
    assert rs.stats()["h2d_bytes"] == n * 8


# ---- 1e9-row scans: tables generated in HBM by the bench's generator (a ring of 4 resident 32 Mi-row fragments) ----------
def _bench():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    import bench
    return bench


@pytest.fixture(scope="module")
def big():
    import torch
    bench = _bench()
    out = {}
    for cfg in ("c2all", "c4"):
        frags = bench.rank_fragments(10**9, 0, 1, ring=4)
        table, keep = bench.build_device_table(cfg, frags, torch)
        names = [c[0] for c in bench.CONFIGS[cfg][0]]
        out[cfg] = (table, keep, bench.make_unit(cfg, bench.CONFIGS[cfg][1], table, names))
    yield out
    out.clear()
    torch.cuda.empty_cache()


def _run_big(ex, big, cfg, eo):
    table, _, unit = big[cfg]
    return ex.executeWorkUnit(0, True, table, unit, eo=eo, memory_level=abi.GPU_LEVEL)


def test_watchdog(big):
    ex = executor.Executor()
    want = _run_big(ex, big, "c2all", None).getStorageBuffer().copy()
    err = expect_code(abi.ERR_OUT_OF_TIME, lambda: _run_big(ex, big, "c2all", eo_of(watchdog=True, limit=1)))
    assert "dynamic_watchdog_time_limit" in str(err)
    assert np.array_equal(_run_big(ex, big, "c2all", eo_of(watchdog=True, limit=10_000)).getStorageBuffer(), want)
    tok = executor.InterruptToken()
    tok.interrupt()
    expect_code(abi.ERR_INTERRUPTED, lambda: _run_big(ex, big, "c2all", eo_of(tok, watchdog=True, limit=1)))
    tok.reset()
    assert np.array_equal(_run_big(ex, big, "c2all", eo_of(tok, watchdog=True, limit=10_000)).getStorageBuffer(), want)


def test_interrupt_during_run(big, record_property):
    ex = executor.Executor()
    want = _run_big(ex, big, "c4", None).getStorageBuffer().copy()
    tok = ex.interrupt_token("q")
    fired = {}

    def fire():
        time.sleep(0.010)
        fired["t"] = time.perf_counter()
        ex.interrupt("q", "killer")

    th = threading.Thread(target=fire)
    t0 = time.perf_counter()
    th.start()
    expect_code(abi.ERR_INTERRUPTED, lambda: _run_big(ex, big, "c4", eo_of(tok)))
    t1 = time.perf_counter()
    th.join()
    latency_ms = (t1 - fired["t"]) * 1e3
    record_property("interrupt_to_return_ms", latency_ms)
    print(f"c4 1e9 rows: interrupt -> return {latency_ms:.2f} ms (call {1e3 * (t1 - t0):.1f} ms)")
    assert latency_ms < 1000
    ex.resetInterrupt("q")
    assert np.array_equal(_run_big(ex, big, "c4", eo_of(tok)).getStorageBuffer(), want)


def test_multi_device_preset_interrupt():
    """execute_work_unit_multi over the devices present (one on a single-GPU machine) with an interrupted token: every device
    stops, none waits in a collective, the call returns INTERRUPTED; after the reset the same call equals the oracle."""
    from test_gpu_multi import device_views
    n_dev = executor.lib().b2q_device_count()
    comms = executor.Comm.init_all(list(range(n_dev)))
    try:
        ex = executor.Executor()
        t = base_table(200_000, 25_000, seed=9)
        views, _keep = device_views(t, n_dev)
        unit = sqlmini.parse("SELECT k, COUNT(*), SUM(v) FROM t WHERE f < 500 GROUP BY k;", t, NAMES)
        tok = executor.InterruptToken()
        tok.interrupt()
        run = lambda: executor.execute_work_unit_multi(comms, ex, 0, True, views, unit, eo=eo_of(tok))
        expect_code(abi.ERR_INTERRUPTED, run)
        tok.reset()
        rs = run()
        ref = oracle_lib.execute(unit, t, num_threads=4)
        gu.rows_equal(rs.rows(), ref.rows())
    finally:
        for c in comms:
            c.destroy()
