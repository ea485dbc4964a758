"""Host-resident tables that take more than one 16 Mi-row slice, for the two scans the host stream serves besides the plain
aggregate: a projection (its chunk order, tickets and offset words run on across slices; a scan limit stops the copies) and a
LEFT JOIN aggregate (the inner columns stay resident across slices).  Each result is compared with the same query on the
HBM-resident copy of the table and with numpy."""
from __future__ import annotations

import numpy as np
import pytest

import join_tables as jt
from gpu_util import DeviceTable, has_gpu
from heavydb_b200 import abi, executor, sqlmini

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_gpu(), reason="needs a CUDA device")]

SLICE = 1 << 24
NAMES = ["c0", "c1"]


@pytest.fixture(scope="module")
def three_slices():
    """One fragment of 2^25 + 12 345 rows: two full slices and a short third one."""
    n = 2 * SLICE + 12_345
    rng = np.random.default_rng(11)
    c0 = rng.integers(0, 10**6, n).astype(np.int64)
    c1 = rng.integers(-2**31, 2**31 - 1, n).astype(np.int32)
    t = abi.Table([(abi.kBIGINT, True), (abi.kINT, True)])
    t.add_host_fragment([c0, c1])
    yield t, DeviceTable(t), (c0, c1)


def _run(table, sql, level, columnar):
    unit = sqlmini.parse(sql, table, NAMES)
    eo = executor.execution_options(output_columnar_hint=columnar)
    return executor.Executor().executeWorkUnit(0, False, table, unit, eo=eo, memory_level=level)


def _offset_words(rs, n):
    """the offset word of every row: the row's index in its fragment"""
    plan = rs.getQueryMemDesc()
    buf = rs.getStorageBuffer()
    if plan.output_columnar:
        return buf[:8 * n].view(np.int64)
    return buf.view(np.int64).reshape(n, plan.row_size // 8)[:, 0]


@pytest.mark.parametrize("columnar", [False, True])
def test_projection_over_three_slices(three_slices, columnar):
    host, dev, (c0, c1) = three_slices
    sql = "SELECT c1, c0 FROM t WHERE c0 < 300000"
    rs = _run(host, sql, abi.CPU_LEVEL, columnar)
    ref = _run(dev.table, sql, abi.GPU_LEVEL, columnar)
    idx = np.nonzero(c0 < 300_000)[0]
    assert rs.rowCount() == idx.size and idx[-1] >= 2 * SLICE
    assert rs.getStorageBuffer().tobytes() == ref.getStorageBuffer().tobytes()
    assert np.array_equal(_offset_words(rs, idx.size), idx)
    assert rs.stats()["rows_scanned"] == ref.stats()["rows_scanned"]


@pytest.mark.parametrize("columnar", [False, True])
def test_projection_limit_met_in_slice_0_stops_the_copies(three_slices, columnar):
    host, _, (c0, c1) = three_slices
    rs = _run(host, "SELECT c1 FROM t WHERE c0 < 300000 LIMIT 1000", abi.CPU_LEVEL, columnar)
    idx = np.nonzero(c0 < 300_000)[0][:1000]
    assert idx[-1] < SLICE
    assert rs.rows() == [(int(v),) for v in c1[idx]]
    assert rs.stats()["h2d_bytes"] == 2 * SLICE * (8 + 4)   # slices 0 and 1 of c0 and c1, nothing after them


def _left_join_reference(fact, dim):
    """{d.attr (None = NULL): (COUNT(*), SUM(t.v), COUNT(d.id32))} of the query below, in numpy"""
    fk32, _fk64, _x, v = fact.fragments[0].host_cols[:4]
    id32, _id64, attr = dim.fragments[0].host_cols[:3]
    lut = np.full(int(id32.max()) + 1, -1, np.int64)
    lut[id32] = np.arange(id32.size)
    inside = (fk32 >= 0) & (fk32 < lut.size)
    row = np.where(inside, lut[np.where(inside, fk32, 0)], -1)
    matched = row >= 0
    key = np.where(matched, attr[np.where(matched, row, 0)], abi.NULL_INT)
    v_ok = v != abi.NULL_BIGINT
    out = {}
    for k in np.unique(key):
        sel = key == k
        out[None if k == abi.NULL_INT else int(k)] = (int(sel.sum()), int(v[sel & v_ok].sum()), int((sel & matched).sum()))
    return out


def test_left_join_over_two_slices():
    n = SLICE + (1 << 20)
    fact, dim = jt.fact_table(n, 23, n), jt.dim_table()
    sql = "SELECT d.attr, COUNT(*), SUM(t.v), COUNT(d.id32) FROM t LEFT JOIN d ON t.fk32 = d.id32 GROUP BY d.attr;"
    unit = sqlmini.parse(sql, fact, jt.FACT_NAMES, inner=(dim, jt.DIM_NAMES))
    ex = executor.Executor()
    rs = ex.executeWorkUnit(4000, True, fact, unit, has_cardinality_estimation=True, memory_level=abi.CPU_LEVEL)
    got = {r[0]: r[1:] for r in rs.rows()}
    assert got == _left_join_reference(fact, dim)
    dev = DeviceTable(fact)
    ref = ex.executeWorkUnit(4000, True, dev.table, unit, has_cardinality_estimation=True, memory_level=abi.GPU_LEVEL)
    assert sorted(rs.rows(), key=repr) == sorted(ref.rows(), key=repr)
    assert rs.stats()["fragments_scanned"] == 1
