"""Projection units on the GPU (b2q_k_project): raw buffers bit for bit against the restated buffer (rows SQLite selects, in
(fragment, row) order), both layouts, HBM- and host-resident tables; the scan limit and its early exit; ORDER BY / LIMIT /
OFFSET; the device hand-off."""
from __future__ import annotations

import numpy as np
import pytest

import ref_tables as rt
from gpu_util import DeviceTable, has_gpu
from heavydb_b200 import abi, executor, sqlmini
from projection_ref import expected_buffer, load_sqlite, mixed_table, passing_rows, plan_matches, projected_cols, restate_descriptor

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_gpu(), reason="needs a CUDA device")]

ALL = ", ".join(rt.TEST_NAMES)
GOLDEN = [f"SELECT {ALL} FROM test", "SELECT x, y, z FROM test WHERE y = 43", "SELECT d, dn, f, fn FROM test WHERE dn IS NULL",
          "SELECT w, ofq, ufq FROM test WHERE z IN (101, 102) OR t > 1001", "SELECT t, u FROM test WHERE x BETWEEN 7 AND 7",
          f"SELECT {ALL} FROM test WHERE NOT (y <> 42) LIMIT 4", "SELECT x FROM test WHERE x > 100", "SELECT smallint_nulls, w FROM test LIMIT 13"]


def _run(ex, unit, table, columnar, level, on_device=False):
    eo = executor.execution_options(output_columnar_hint=columnar, result_on_device=on_device)
    return ex.executeWorkUnit(0, False, table, unit, eo=eo, memory_level=level)


@pytest.fixture(scope="module")
def golden():
    table = rt.make_table(rt.test_rows())
    return table, DeviceTable(table), load_sqlite(table, rt.TEST_NAMES)


@pytest.mark.parametrize("level", [abi.GPU_LEVEL, abi.CPU_LEVEL])
@pytest.mark.parametrize("columnar", [False, True])
@pytest.mark.parametrize("sql", GOLDEN)
def test_golden_buffers(golden, sql, columnar, level):
    table, dev, con = golden
    unit = sqlmini.parse(sql, table, rt.TEST_NAMES)
    ex = executor.Executor()
    rs = _run(ex, unit, dev.table if level == abi.GPU_LEVEL else table, columnar, level)
    where = sql.split(" WHERE ")[1].split(" LIMIT")[0] if " WHERE " in sql else None
    picks = passing_rows(con, where)
    if unit.unit.scan_limit:
        picks = picks[:unit.unit.scan_limit]
    plan = rs.getQueryMemDesc()
    assert plan.query_desc_type == abi.Projection and plan.entry_count == len(picks) == rs.rowCount() == rs.entryCount()
    got = rs.getStorageBuffer()
    plan_matches(plan, restate_descriptor(table, projected_cols(unit), columnar, len(picks)))
    want = expected_buffer(table, projected_cols(unit), picks, columnar)
    assert got.view(np.uint8).tobytes() == want.tobytes(), sql
    again = _run(ex, unit, dev.table, columnar, abi.GPU_LEVEL).getStorageBuffer()
    assert again.tobytes() == got.tobytes()


def _big(n, frag_rows, seed=5):
    rng = np.random.default_rng(seed)
    t = abi.Table([(abi.kBIGINT, True), (abi.kBIGINT, True), (abi.kINT, True), (abi.kSMALLINT, False)])
    c0 = rng.integers(0, 10**6, n).astype(np.int64)
    c1 = rng.integers(-10**9, 10**9, n).astype(np.int64)
    g = rng.integers(0, 10**4, n).astype(np.int32)
    s = rng.integers(-300, 300, n).astype(np.int16)
    s[rng.random(n) < 0.05] = abi.NULL_OF[abi.kSMALLINT]
    for b in range(0, n, frag_rows):
        t.add_host_fragment([c0[b:b + frag_rows], c1[b:b + frag_rows], g[b:b + frag_rows], s[b:b + frag_rows]])
    return t, (c0, c1, g, s)


@pytest.fixture(scope="module")
def big():
    t, cols = _big(3_000_000, 700_001)
    return t, DeviceTable(t), cols


def _want_buffer(plan, table, cols_idx, mask, frag_rows, limit=None):
    idx = np.nonzero(mask)[0]
    if limit:
        idx = idx[:limit]
    picks = [(int(i // frag_rows), int(i % frag_rows)) for i in idx]
    return expected_buffer(table, cols_idx, picks, plan.output_columnar == 1), idx


@pytest.mark.parametrize("columnar", [False, True])
@pytest.mark.parametrize("k,limit", [(10_000, 0), (500_000, 0), (10**6, 0), (500_000, 1000), (10_000, 123_457), (0, 0), (0, 10)])
def test_filter_and_limit(big, columnar, k, limit):
    table, dev, (c0, c1, g, s) = big
    sql = f"SELECT g, c1, s FROM t WHERE c0 < {k}" + (f" LIMIT {limit}" if limit else "")
    unit = sqlmini.parse(sql, table, ["c0", "c1", "g", "s"])
    ex = executor.Executor()
    rs = _run(ex, unit, dev.table, columnar, abi.GPU_LEVEL)
    plan = rs.getQueryMemDesc()
    want, idx = _want_buffer(plan, table, [2, 1, 3], c0 < k, 700_001, limit)
    assert rs.rowCount() == idx.size
    assert rs.getStorageBuffer().tobytes() == want.tobytes()
    if limit and idx.size == limit:
        assert rs.stats()["rows_scanned"] < c0.size


@pytest.mark.parametrize("columnar", [False, True])
@pytest.mark.parametrize("order,limit,offset", [("c1 DESC", 10, 0), ("g, c1", 50, 7), ("s NULLS FIRST, c1", 20, 100)])
def test_order_by(big, columnar, order, limit, offset):
    table, dev, (c0, c1, g, s) = big
    sql = f"SELECT g, c1, s FROM t WHERE c0 < 20000 ORDER BY {order}" + (f" LIMIT {limit}" if limit else "") + (f" OFFSET {offset}" if offset else "")
    unit = sqlmini.parse(sql, table, ["c0", "c1", "g", "s"])
    rs = _run(executor.Executor(), unit, dev.table, columnar, abi.GPU_LEVEL)
    con = load_sqlite(table, ["c0", "c1", "g", "s"])
    q = f"SELECT g, c1, s FROM t WHERE c0 < 20000 ORDER BY {order.replace('s NULLS FIRST', 's IS NOT NULL, s')}, _id, _r"
    want = con.execute(q + (f" LIMIT {limit if limit else -1} OFFSET {offset}")).fetchall()
    assert rs.rows() == [tuple(r) for r in want]
    rs2 = _run(executor.Executor(), sqlmini.parse("SELECT g, c1, s FROM t WHERE c0 < 20000", table, ["c0", "c1", "g", "s"]), dev.table, columnar, abi.GPU_LEVEL)
    rs2.sort([(2, True, True)], 5)
    rs2.keepFirstN(5)
    top = con.execute("SELECT g, c1, s FROM t WHERE c0 < 20000 ORDER BY c1 DESC, _id, _r LIMIT 5").fetchall()
    assert rs2.rows()[:5] == [tuple(r) for r in top]


@pytest.mark.parametrize("columnar", [False, True])
def test_device_handoff(big, columnar):
    table, dev, _ = big
    unit = sqlmini.parse("SELECT g, c1, s FROM t WHERE c0 < 300000", table, ["c0", "c1", "g", "s"])
    rs = _run(executor.Executor(), unit, dev.table, columnar, abi.GPU_LEVEL, on_device=True)
    assert rs.stats()["result_d2h_bytes"] == 0
    dc = rs.deviceColumns().to_host()
    assert rs.stats()["result_d2h_bytes"] == 0
    host = rs.columnarResults()
    for (ty, _nn, vals, _v, _n), (ty2, _nn2, arr) in zip(dc, host):
        assert ty == ty2 and np.array_equal(vals, arr)


def test_early_exit_large():
    import torch
    n = 200_000_000
    t = abi.Table([(abi.kBIGINT, True), (abi.kBIGINT, True)])
    c0 = torch.randint(0, 10**6, (n,), dtype=torch.int64, device="cuda")
    c1 = torch.arange(n, dtype=torch.int64, device="cuda")
    t.add_device_fragment(n, [c0.data_ptr(), c1.data_ptr()], [abi.ChunkStats(0, 10**6 - 1, 0.0, 0.0, 0), abi.ChunkStats(0, n - 1, 0.0, 0.0, 0)])
    torch.cuda.synchronize()
    unit = sqlmini.parse("SELECT c1 FROM t WHERE c0 < 500000 LIMIT 1000", t, ["c0", "c1"])
    rs = executor.Executor().executeWorkUnit(0, False, t, unit, memory_level=abi.GPU_LEVEL)
    want = torch.nonzero(c0 < 500000).flatten()[:1000].cpu().numpy()
    assert [r[0] for r in rs.rows()] == want.tolist()
    assert rs.stats()["rows_scanned"] <= 4 * 132 * 4 * 2048   # a few grid-widths of 2048-row chunks, not 2e8 rows
    full = executor.Executor().executeWorkUnit(0, False, t, sqlmini.parse("SELECT c1 FROM t WHERE c0 < 500000", t, ["c0", "c1"]),
                                               eo=executor.execution_options(output_columnar_hint=True), memory_level=abi.GPU_LEVEL)
    assert full.rowCount() == int((c0 < 500000).sum())
    cr = full.columnarResults()[0][2]
    want = c1[c0 < 500000].cpu().numpy()
    assert int(cr.sum()) == int(want.sum())
    assert np.array_equal(cr[:100_000], want[:100_000]) and np.array_equal(cr[-100_000:], want[-100_000:])


def test_split_forms_refuse(big):
    table, dev, _ = big
    unit = sqlmini.parse("SELECT g FROM t", table, ["c0", "c1", "g", "s"])
    with pytest.raises(executor.UnsupportedOnThisPath):
        executor.Executor().executePartial(0, False, dev.table, unit, memory_level=abi.GPU_LEVEL)


PARTS = [slice(1, 12), slice(9, 17)]   # at most 16 launch columns with the filter and $deleted$ columns


@pytest.fixture(scope="module")
def mixed():
    table, names = mixed_table(200_000, 11, 30_000, fragment_ids=[5, 0, 6, 2, 1, 4, 3])
    return table, names, DeviceTable(table), load_sqlite(table, names)


@pytest.mark.parametrize("level", [abi.GPU_LEVEL, abi.CPU_LEVEL])
@pytest.mark.parametrize("columnar", [False, True])
@pytest.mark.parametrize("part", PARTS)
@pytest.mark.parametrize("where,limit", [(None, 0), ("k < 4000 AND (i32f16 IS NULL OR s8 <> 3)", 0), ("k >= 2000", 5000),
                                         ("dt16 IS NOT NULL AND ti > 0", 17), ("k < 0", 0), ("k < 0", 10)])
def test_encoded_buffers(mixed, where, limit, part, columnar, level):
    """FIXED / DICT(8|16) / DAYS / DECIMAL / TIME columns decoded, deleted rows left out, fragments given out of id order,
    fragments skipped on chunk stats: raw buffers bit for bit, both layouts, HBM- and host-resident."""
    table, names, dev, con = mixed
    sql = f"SELECT {', '.join(names[part])} FROM t" + (f" WHERE {where}" if where else "") + (f" LIMIT {limit}" if limit else "")
    unit = sqlmini.parse(sql, table, names)
    rs = _run(executor.Executor(), unit, dev.table if level == abi.GPU_LEVEL else table, columnar, level)
    picks = passing_rows(con, where)
    if limit:
        picks = picks[:limit]
    cols = projected_cols(unit)
    plan_matches(rs.getQueryMemDesc(), restate_descriptor(table, cols, columnar, len(picks)))
    assert rs.getStorageBuffer().tobytes() == expected_buffer(table, cols, picks, columnar).tobytes(), sql
    st = rs.stats()
    if where == "k >= 2000":   # k // 1000 is the fragment position: the first two fragments are skipped
        assert st["fragments_skipped"] == 2 and st["fragments_scanned"] == 5
    if level == abi.CPU_LEVEL and where == "k >= 2000":
        assert st["h2d_bytes"] > 0


@pytest.mark.parametrize("seed", range(4))
def test_fuzz(mixed, seed):
    """Random filters x column lists x scan limits x layouts against the restatement."""
    import random
    table, names, dev, con = mixed
    rng = random.Random(seed)
    cents = rng.randint(-10**6, 10**6)
    # (engine text, SQLite text): SQLite holds a DECIMAL as its scaled integer, the engine folds the literal to the column's scale
    leaves = [("k < {}".format(rng.randint(0, 8000)),) * 2, ("i32f16 > {}".format(rng.randint(-3000, 3000)),) * 2, ("i64f8 IS NULL",) * 2,
              ("s16 <> {}".format(rng.randint(0, 60000)),) * 2, (f"dec32 >= {cents / 100:.2f}", f"dec32 >= {cents}"),
              ("d < {}".format(rng.random() * 100),) * 2, ("tm BETWEEN {} AND {}".format(rng.randint(0, 40000), rng.randint(40000, 86400)),) * 2,
              ("si IN (1, 2, 3) OR ti < {}".format(rng.randint(-127, 127)),) * 2]
    for _ in range(6):
        chosen = rng.sample(leaves, rng.randint(1, 3))
        where = " AND ".join(f"({x})" for x, _ in chosen)
        where_sqlite = " AND ".join(f"({y})" for _, y in chosen)
        cols = rng.sample(names[1:-1], rng.randint(1, 8))
        limit = rng.choice([0, 1, 100, 3000, 10**6])
        columnar = rng.random() < 0.5
        sql = f"SELECT {', '.join(cols)} FROM t WHERE {where}" + (f" LIMIT {limit}" if limit else "")
        unit = sqlmini.parse(sql, table, names)
        rs = _run(executor.Executor(), unit, dev.table, columnar, abi.GPU_LEVEL)
        picks = passing_rows(con, where_sqlite)
        if limit:
            picks = picks[:limit]
        assert rs.getStorageBuffer().tobytes() == expected_buffer(table, projected_cols(unit), picks, columnar).tobytes(), sql


def test_scan_limit_equal_to_count(big):
    """scan_limit == 0 (the COUNT(*) pre-flight sizes the buffer) gives the same bytes as a scan limit of exactly that count."""
    table, dev, (c0, *_r) = big
    n = int((c0 < 300_000).sum())
    for columnar in (False, True):
        a = _run(executor.Executor(), sqlmini.parse("SELECT g, c1, s FROM t WHERE c0 < 300000", table, ["c0", "c1", "g", "s"]), dev.table, columnar, abi.GPU_LEVEL)
        b = _run(executor.Executor(), sqlmini.parse(f"SELECT g, c1, s FROM t WHERE c0 < 300000 LIMIT {n}", table, ["c0", "c1", "g", "s"]), dev.table, columnar, abi.GPU_LEVEL)
        assert a.getStorageBuffer().tobytes() == b.getStorageBuffer().tobytes()
        huge = _run(executor.Executor(), sqlmini.parse("SELECT g FROM t WHERE c0 < 300000 LIMIT 1000000000000", table, ["c0", "c1", "g", "s"]), dev.table, columnar, abi.GPU_LEVEL)
        assert huge.rowCount() == n
        empty = _run(executor.Executor(), sqlmini.parse("SELECT g FROM t LIMIT 0", table, ["c0", "c1", "g", "s"]), dev.table, columnar, abi.GPU_LEVEL)
        assert empty.rowCount() == 0 and empty.stats()["rows_scanned"] == 0


@pytest.mark.parametrize("columnar", [False, True])
def test_arrow_export(mixed, columnar):
    """The Arrow C Device export of a projection equals toArrow()."""
    pa = pytest.importorskip("pyarrow")
    table, names, dev, _ = mixed
    unit = sqlmini.parse(f"SELECT {', '.join(names[1:9])} FROM t WHERE k < 5000", table, names)
    rs = _run(executor.Executor(), unit, dev.table, columnar, abi.GPU_LEVEL, on_device=True)
    dc = rs.deviceColumns()
    host = rs.toArrow()
    got = dc.to_host()
    for i, (ty, _nn, vals, valid, nulls) in enumerate(got):
        col = host.column(i)
        assert nulls == col.null_count
        if ty not in abi.DECIMAL_TYPES:
            assert np.array_equal(np.asarray(col.fill_null(0)), np.where(vals == abi.NULL_OF[ty], 0, vals))
    ex = dc.export_arrow(names[1:9])
    assert ex.array.device_type == 2   # ARROW_DEVICE_CUDA
    ex.release()


def test_multi_and_dist_refuse(big):
    import torch
    table, dev, _ = big
    unit = sqlmini.parse("SELECT g FROM t", table, ["c0", "c1", "g", "s"])
    comms = executor.Comm.init_all([0])
    try:
        with pytest.raises(executor.UnsupportedOnThisPath):
            executor.execute_work_unit_multi(comms, executor.Executor(), 0, False, [dev.table], unit)
    finally:
        for c in comms:
            c.destroy()
    comm = executor.Comm.init_rank(executor.Comm.unique_id(), 1, 0, torch.cuda.current_device())
    try:
        with pytest.raises(executor.UnsupportedOnThisPath):
            executor.execute_work_unit_dist(comm, executor.Executor(), 0, False, dev.table, unit)
    finally:
        comm.destroy()


def test_inner_entry_b2q_launch(big):
    """b2q_launch with a projection plan: rows at TOTAL_MATCHED up to MAX_MATCHED in (fragment, row) order."""
    import ctypes as C
    import torch
    table, dev, (c0, c1, g, s) = big
    L = executor.lib()
    unit = sqlmini.parse("SELECT c1, g FROM t WHERE c0 < 400000", table, ["c0", "c1", "g", "s"])
    bt = dev.table.build(abi.GPU_LEVEL)
    co, eo = executor.compilation_options(), executor.execution_options(output_columnar_hint=True)
    q = C.c_void_p()
    assert L.b2q_plan(C.byref(unit.unit), C.byref(bt.info), C.byref(co), C.byref(eo), 0, 0, C.byref(q)) == 0
    cap = 5000
    nf, nc = len(dev.table.fragments), dev.table.num_cols
    per_frag = [(C.c_void_p * nc)(*[p or None for p in f.dev_ptrs]) for f in dev.table.fragments]
    col_buffers = (C.POINTER(C.c_void_p) * nf)(*[C.cast(a, C.POINTER(C.c_void_p)) for a in per_frag])
    num_rows = (C.c_int64 * nf)(*[f.num_tuples for f in dev.table.fragments])
    num_frags, num_tables, max_matched = C.c_uint32(nf), C.c_uint32(1), C.c_int32(cap)
    d = restate_descriptor(table, [1, 2], True, cap)
    out = torch.zeros(d["buffer_size"], dtype=torch.uint8, device="cuda")
    gb = torch.tensor([out.data_ptr()], dtype=torch.int64, device="cuda")
    err = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    matched = torch.zeros(1, dtype=torch.int32, device="cuda")
    prm = abi.Params()
    prm.error_codes = err.data_ptr()
    prm.total_matched = matched.data_ptr()
    prm.group_by_buffers = gb.data_ptr()
    prm.num_fragments, prm.num_tables = C.pointer(num_frags), C.pointer(num_tables)
    prm.col_buffers = col_buffers
    prm.num_rows = num_rows
    prm.max_matched = C.addressof(max_matched)
    torch.cuda.synchronize()
    assert L.b2q_launch(q, C.byref(prm), None) == 0, L.b2q_last_error_message()
    torch.cuda.synchronize()
    L.b2q_query_free(q)
    assert int(err.item()) == 0 and int(matched.item()) == cap
    idx = np.nonzero(c0 < 400000)[0][:cap]
    buf = out.cpu().numpy()
    assert np.array_equal(buf[:8 * cap].view(np.int64), idx % 700_001)
    assert np.array_equal(buf[d["slot_offset"][0]:d["slot_offset"][0] + 8 * cap].view(np.int64), c1[idx])
    assert np.array_equal(buf[d["slot_offset"][1]:d["slot_offset"][1] + 4 * cap].view(np.int32), g[idx])
