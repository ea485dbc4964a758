"""Results handed over in device memory: every query runs twice, with `result_on_device` off and on.  The device columns
(b2q_rs_device_columns) must be exactly the host ColumnarResults of the same result set, with an Arrow validity bitmap that
marks the inline NULL sentinels; nothing crosses PCIe until a host accessor asks; and the device-resident run answers what
the default run answers."""
import ctypes as C
import gc

import numpy as np
import pytest

import dec_tables as dt
import gpu_util as gu
import join_tables as jt
import oracle_lib
import order_queries as oq
import ref_tables as rt
import ref_time_table as tt
import sqlmini
import str_tables as stt
from heavydb_b200 import abi, executor
from test_gpu_parity import RAND_NAMES, RAND_QUERIES, random_table
from test_oracle_golden import COUNT_DISTINCT_QUERIES, FLOAT_QUERIES, MULTI_KEY_QUERIES

pytestmark = pytest.mark.gpu

EMPTY_AND_NON_GROUPED = [
    "SELECT k8, COUNT(*), AVG(d) FROM r WHERE k32 < -1000000 GROUP BY k8;",
    "SELECT COUNT(*), SUM(a64), AVG(d), MIN(f32) FROM r;",
    "SELECT COUNT(*), MIN(a32), MAX(d) FROM r WHERE k32 < -1000000;",
]
SPARSE = "SELECT sparse, COUNT(*), SUM(a32), MIN(d), AVG(a16) FROM r GROUP BY sparse;"


def device_bytes(ptr, nbytes, device):
    import torch
    if not nbytes:
        return np.zeros(0, np.uint8)
    return torch.as_tensor(executor._CudaArray(None, ptr, nbytes, "|u1"), device=torch.device("cuda", device)).cpu().numpy()


def check_device_columns(rs, resident=True):
    """(a) + (b): the device columns of `rs`, copied back, are its host ColumnarResults byte for byte; the validity bitmap is
    packbits(~is_sentinel) and the NULL counts agree.  (c): a device-resident set crosses PCIe only at its first host
    accessor, which is the columnarResults() below."""
    if resident:
        assert rs.stats()["result_d2h_bytes"] == 0
    dc = rs.deviceColumns()
    if resident:
        assert rs.stats()["result_d2h_bytes"] == 0
    got = dc.to_host()
    want = rs.columnarResults(num_threads=4)
    if resident:
        assert rs.stats()["result_d2h_bytes"] == rs.getQueryMemDesc().buffer_size
    assert len(got) == len(want) == dc.num_columns() == rs.colCount()
    for (ty, nn, vals, mask, nulls), (wty, wnn, wa) in zip(got, want):
        assert (ty, nn) == (wty, wnn)
        assert vals.dtype == wa.dtype and vals.size == wa.size == dc.size()
        assert np.array_equal(vals.view(np.uint8), wa.view(np.uint8))
        sentinel = wa == abi.NULL_OF[ty]
        assert nulls == int(sentinel.sum())
        if nulls:
            assert np.array_equal(mask, np.packbits(~sentinel, bitorder="little"))
        else:
            assert mask is None
    return dc


def columns_close(got, want, tol, ordered):
    """Two runs' ColumnarResults: integer columns identical, floating-point ones within the sum tolerance."""
    assert len(got) == len(want)
    if not ordered:   # baseline-hash entry order depends on which thread claimed a slot first
        got = _sorted_columns(got)
        want = _sorted_columns(want)
    for (ty, _, a), (wty, _, b), (rtol, atol) in zip(got, want, tol):
        assert ty == wty and a.dtype == b.dtype and a.size == b.size
        if a.dtype.kind == "f":
            assert np.array_equal(a == abi.NULL_OF[ty], b == abi.NULL_OF[ty])
            assert np.all((a == b) | (np.abs(a - b) <= rtol * np.abs(b) + atol))
        else:
            assert np.array_equal(a, b)


def _sorted_columns(cols):
    keys = [c[2] for c in cols if c[2].dtype.kind != "f"]
    if not keys or not keys[0].size:
        return cols
    order = np.lexsort(keys[::-1])
    return [(t, nn, a[order]) for t, nn, a in cols]


def run_pair(unit, dev, n_rows, entry_guess=0, has_card=False, **eo_kw):
    """The same unit with result_on_device off and on; checks (a)-(c) and that both runs agree."""
    ex = executor.Executor()
    kw = dict(has_cardinality_estimation=has_card, memory_level=abi.GPU_LEVEL)
    host = ex.executeWorkUnit(entry_guess, True, dev.table, unit, eo=executor.execution_options(**eo_kw), **kw)
    drs = ex.executeWorkUnit(entry_guess, True, dev.table, unit, eo=executor.execution_options(result_on_device=True, **eo_kw), **kw)
    plan = drs.getQueryMemDesc()
    assert bytes(plan) == bytes(host.getQueryMemDesc())
    assert host.stats()["result_d2h_bytes"] == plan.buffer_size
    check_device_columns(drs)
    tol = gu.column_tolerances(plan, n_rows)
    sorted_unit = bool(unit.unit.num_order_entries or unit.unit.has_limit or unit.unit.offset)
    baseline = plan.query_desc_type == abi.GroupByBaselineHash
    if sorted_unit:
        gu.rows_equal(drs.rows(), host.rows(), col_tol=tol)
    else:
        columns_close(drs.columnarResults(), host.columnarResults(), tol, ordered=not baseline)
        gu.rows_equal(drs.rows(), host.rows(), col_tol=tol)
        if not baseline:
            gu.buffers_equal(drs.getStorageBuffer(), host.getStorageBuffer(), plan, float_atol=rt.float_sum_atol(n_rows))
    assert drs.rowCount() == host.rowCount()
    return host, drs


def run_set(sqls, table, names, dev, min_ran, inner=None, **kw):
    ran = 0
    for sql in sqls:
        unit = sqlmini.parse(sql, table, names, inner=inner)
        try:
            run_pair(unit, dev, table.total_tuples(), **kw)
        except (executor.UnsupportedOnThisPath, executor.CardinalityEstimationRequired):
            continue   # refused by the planner whatever the flag (the flag changes no plan: test_device_results_cpu)
        except Exception as e:
            raise AssertionError(f"query: {sql}\n{e}") from e
        ran += 1
    assert ran >= min_ran


@pytest.fixture(scope="module")
def rand():
    table = random_table(30000, seed=77, frag_rows=8000)
    return table, gu.DeviceTable(table)


def test_random_empty_and_non_grouped_queries(rand):
    table, dev = rand
    run_set(RAND_QUERIES + EMPTY_AND_NON_GROUPED, table, RAND_NAMES, dev, 12, entry_guess=4001, has_card=True)


def test_columnar_output_and_bigint_count(rand):
    table, dev = rand
    run_set(RAND_QUERIES, table, RAND_NAMES, dev, 5, entry_guess=4001, has_card=True, output_columnar_hint=True)
    run_set(RAND_QUERIES[:8], table, RAND_NAMES, dev, 4, entry_guess=4001, has_card=True, bigint_count=True)


def test_order_by_limit_offset(rand):
    table, dev = rand
    run_set(oq.RAND_ORDER_QUERIES + [oq.OFFSET_WITHOUT_LIMIT_QUIRK], table, RAND_NAMES, dev, 5, entry_guess=3001, has_card=True)
    run_set(oq.RAND_ORDER_QUERIES, table, RAND_NAMES, dev, 3, entry_guess=3001, has_card=True, output_columnar_hint=True)


def test_baseline_hash_radix_and_probe(rand):
    table, dev = rand
    for fk in (0, abi.KERNEL_BASELINE_PROBE):
        unit = sqlmini.parse(SPARSE, table, RAND_NAMES)
        _, drs = run_pair(unit, dev, table.total_tuples(), entry_guess=45000, has_card=True, force_kernel=fk)
        assert drs.getQueryMemDesc().query_desc_type == abi.GroupByBaselineHash


def test_dictionary_time_and_decimal_targets():
    table = stt.str_table(20000, seed=5, frag_rows=6000)
    run_set(stt.STR_QUERIES, table, stt.STR_NAMES, gu.DeviceTable(table), 5)
    table = tt.make_table(tt.time_rows())
    run_set(tt.TIME_QUERIES, table, tt.TIME_NAMES, gu.DeviceTable(table), 5)
    table = dt.make_table(dt.mixed_rows(), fragment_size=170)
    run_set(dt.GOLDEN_QUERIES + dt.MORE_QUERIES, table, dt.DEC_NAMES, gu.DeviceTable(table), 5)


def test_multi_key_count_distinct_and_float_targets():
    table = rt.make_table(rt.test_rows())
    run_set(MULTI_KEY_QUERIES + COUNT_DISTINCT_QUERIES + FLOAT_QUERIES, table, rt.TEST_NAMES, gu.DeviceTable(table), 15)


def test_joins():
    fact = jt.fact_table(40000, seed=11, frag_rows=9000)
    run_set(jt.JOIN_QUERIES + jt.LEFT_JOIN_QUERIES, fact, jt.FACT_NAMES, gu.DeviceTable(fact), 5, inner=(jt.dim_table(), jt.DIM_NAMES),
            entry_guess=4000, has_card=True)


@pytest.mark.parametrize("columnar", [False, True])
def test_sort_drop_keep_on_a_device_resident_set(rand, columnar):
    """(d): ResultSet.sort / dropFirstN / keepFirstN on a device-resident set sort the device buffer (still no D2H) and
    the device columns follow them, row for row like the host-resident set treated the same way."""
    table, dev = rand
    ex = executor.Executor()
    ran = 0
    # COUNT descending, ties by the group key(s): a total order, so both sets must list the same rows
    for sql, order in [("SELECT k16, COUNT(*), SUM(a32), AVG(d) FROM r GROUP BY k16;", [(2, True, False), (1, False, True)]),
                       ("SELECT k8, k32, COUNT(*), MIN(f32) FROM r GROUP BY k8, k32;", [(3, True, False), (1, False, True), (2, False, True)])]:
        unit = sqlmini.parse(sql, table, RAND_NAMES)
        for top_n, drop, keep in ((0, 3, 20), (15, 0, 0), (0, 10**6, 5)):
            try:
                rss = [ex.executeWorkUnit(4001, True, dev.table, unit, eo=executor.execution_options(output_columnar_hint=columnar),
                                          has_cardinality_estimation=True, memory_level=abi.GPU_LEVEL, result_on_device=on)
                       for on in (False, True)]
            except executor.UnsupportedOnThisPath:
                continue
            for rs in rss:
                rs.sort(order, top_n)
                rs.dropFirstN(drop)
                rs.keepFirstN(keep)
            assert rss[1].stats()["result_d2h_bytes"] == 0
            check_device_columns(rss[1])
            gu.rows_equal_ordered(rss[1].rows(), rss[0].rows())
            ran += 1
    assert ran >= 3


def test_storage_wrapped_from_the_oracle_converts_on_the_device(rand):
    """b2q_rs_create_from_storage over the oracle's buffers (row-wise and columnar; keyless, keyed, baseline): uploaded and
    converted on the device to exactly the host ColumnarResults."""
    table, _ = rand
    ex = executor.Executor()
    layouts = set()
    for sql, guess in [(q, 4001) for q in RAND_QUERIES] + [(SPARSE, 45000)]:
        unit = sqlmini.parse(sql, table, RAND_NAMES)
        for columnar in (False, True):
            try:
                ref = oracle_lib.execute(unit, table, entry_guess=guess, has_card=True, num_threads=4, output_columnar=columnar)
            except oracle_lib.OracleError:
                continue
            rs = ex.resultSetFromStorage(ref.buffer(), unit, table, eo=executor.execution_options(output_columnar_hint=columnar),
                                         max_groups_buffer_entry_guess=guess, has_cardinality_estimation=True)
            check_device_columns(rs, resident=False)
            p = rs.getQueryMemDesc()
            layouts.add((bool(p.output_columnar), "baseline" if p.query_desc_type == abi.GroupByBaselineHash else
                         "keyless" if p.keyless_hash else "non-grouped" if p.query_desc_type == abi.NonGroupedAggregate else "keyed"))
    assert {(False, "keyed"), (False, "baseline"), (True, "baseline")} <= layouts, layouts
    assert any(kind == "keyless" for _, kind in layouts), layouts


def _arrow_format(t):
    import pyarrow as pa
    if pa.types.is_decimal(t):
        return f"d:{t.precision},{t.scale}"
    return {pa.int8(): "c", pa.int16(): "s", pa.int32(): "i", pa.int64(): "l", pa.float32(): "f", pa.float64(): "g"}[t]


def _pool_used(device):
    """CU_MEMPOOL_ATTR_USED_MEM_CURRENT of the device's default stream-ordered pool (where libb2q allocates)."""
    cu = C.CDLL("libcuda.so.1")
    dev, pool, used = C.c_int(), C.c_void_p(), C.c_uint64()
    assert cu.cuDeviceGet(C.byref(dev), device) == 0
    assert cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    assert cu.cuMemPoolGetAttribute(pool, 7, C.byref(used)) == 0
    return used.value


def test_arrow_export_matches_toArrow_and_release_frees(rand):
    import torch
    table, dev = rand
    dtable = dt.make_table(dt.mixed_rows(), fragment_size=170)
    cases = [("SELECT k8, k16, COUNT(*), SUM(a64), AVG(d), MIN(f32), MAX(d) FROM r GROUP BY k8, k16;", table, RAND_NAMES, dev)]
    cases += [(q, dtable, dt.DEC_NAMES, gu.DeviceTable(dtable)) for q in dt.GOLDEN_QUERIES + dt.MORE_QUERIES if "ORDER" not in q.upper()]
    ex = executor.Executor()
    saw_decimal = saw_nulls = False
    for sql, tbl, names, dtab in cases:
        unit = sqlmini.parse(sql, tbl, names)
        try:
            rs = ex.executeWorkUnit(4001, True, dtab.table, unit, has_cardinality_estimation=True, memory_level=abi.GPU_LEVEL,
                                    result_on_device=True)
        except executor.UnsupportedOnThisPath:
            continue
        nc = rs.colCount()
        cols = [f"c{i}" for i in range(nc)]
        torch.cuda.synchronize()
        used0 = _pool_used(torch.cuda.current_device())
        dc = rs.deviceColumns()
        exp = dc.export_arrow(cols)
        batch = rs.toArrow(names=cols)
        s, a = exp.schema, exp.array
        assert s.format == b"+s" and s.n_children == nc
        assert a.device_type == abi.ARROW_DEVICE_CUDA and a.device_id == dc.device() and a.sync_event
        assert a.array.length == batch.num_rows and a.array.n_children == nc and a.array.null_count == 0
        for i in range(nc):
            cs, ca, col = s.children[i].contents, a.array.children[i].contents, batch.column(i)
            assert cs.name.decode() == cols[i] and cs.format.decode() == _arrow_format(col.type), (sql, i)
            assert ca.length == len(col) and ca.null_count == col.null_count and ca.n_buffers == 2
            saw_decimal |= cs.format.startswith(b"d:")
            saw_nulls |= col.null_count > 0
            width = col.type.bit_width // 8
            pa_bufs = col.buffers()
            assert np.array_equal(device_bytes(ca.buffers[1], len(col) * width, dc.device()),
                                  np.frombuffer(pa_bufs[1], np.uint8)[: len(col) * width]), (sql, i)
            if col.null_count:
                got = np.unpackbits(device_bytes(ca.buffers[0], (len(col) + 7) // 8, dc.device()), bitorder="little")[: len(col)]
                want = np.unpackbits(np.frombuffer(pa_bufs[0], np.uint8), bitorder="little")[: len(col)]
                assert np.array_equal(got, want), (sql, i)
            else:
                assert not ca.buffers[0]
        # shared ownership: the handle goes first, the export keeps the buffers; its release returns them to the pool
        del dc
        gc.collect()
        torch.cuda.synchronize()
        assert _pool_used(torch.cuda.current_device()) > used0
        exp.release()
        torch.cuda.synchronize()
        assert _pool_used(torch.cuda.current_device()) == used0
        assert not exp.array.array.release and not exp.schema.release
    assert saw_decimal and saw_nulls


def test_tensors_are_zero_copy_and_outlive_the_result_set(rand):
    import torch
    table, dev = rand
    unit = sqlmini.parse("SELECT k16, COUNT(*), SUM(a32), AVG(d), MIN(f32) FROM r GROUP BY k16;", table, RAND_NAMES)
    rs = executor.Executor().executeWorkUnit(4001, True, dev.table, unit, has_cardinality_estimation=True, memory_level=abi.GPU_LEVEL,
                                             result_on_device=True)
    dc = rs.deviceColumns()
    ts = dc.tensors()
    assert rs.stats()["result_d2h_bytes"] == 0
    for i, (vals, mask) in enumerate(ts):
        ptr, (ty, _, _), valid, nulls = dc.column(i)
        assert vals.is_cuda and vals.data_ptr() == ptr and vals.numel() == dc.size()
        assert vals.dtype == {np.int8: torch.int8, np.int16: torch.int16, np.int32: torch.int32, np.int64: torch.int64,
                              np.float32: torch.float32, np.float64: torch.float64}[abi.NUMPY_OF[ty]]
        assert (mask is None) == (nulls == 0) and (mask is None or mask.data_ptr() == valid)
    want = [a for _, _, a in rs.columnarResults()]
    del dc, rs
    gc.collect()
    torch.cuda.synchronize()
    for (vals, _), w in zip(ts, want):
        assert np.array_equal(vals.cpu().numpy().view(np.uint8), w.view(np.uint8))


def _generated_table(rows, key_span, key_stride):
    """key BIGINT (lo 0, span key_span, stride key_stride), v BIGINT in [0, 1e6): generated in HBM with b2q_gen_column."""
    import torch
    t = abi.Table([(abi.kBIGINT, True), (abi.kBIGINT, True)])
    keep, stats = [], []
    for tag, (span, stride) in enumerate([(key_span, key_stride), (10**6, 1)]):
        buf = torch.empty(rows * 8, dtype=torch.uint8, device="cuda")
        executor.gen_column_device(buf.data_ptr(), abi.kBIGINT, 0x5EED, tag, 0, rows, 0, span, stride=stride)
        keep.append(buf)
        st = abi.ChunkStats()
        st.int_min, st.int_max = 0, (span - 1) * stride
        stats.append(st)
    t.add_device_fragment(rows, [b.data_ptr() for b in keep], stats)
    torch.cuda.synchronize()
    return t, keep


@pytest.mark.parametrize("shape", ["dense_1e7_groups", "baseline"])
def test_high_cardinality_results(shape):
    rows, span, stride, guess = (20_000_000, 10**7, 1, 0) if shape == "dense_1e7_groups" else (4_000_000, 10**6, 900_000_000_007, 1_500_000)
    table, _keep = _generated_table(rows, span, stride)
    unit = sqlmini.parse("SELECT key, SUM(v), COUNT(*) FROM t GROUP BY key;", table, ["key", "v"])
    ex = executor.Executor()
    kw = dict(has_cardinality_estimation=guess > 0, memory_level=abi.GPU_LEVEL)
    host = ex.executeWorkUnit(guess, True, table, unit, **kw)
    drs = ex.executeWorkUnit(guess, True, table, unit, result_on_device=True, **kw)
    dc = check_device_columns(drs)
    assert dc.size() == host.rowCount() > span // 2
    columns_close(drs.columnarResults(), host.columnarResults(), [(0, 0)] * 3, ordered=shape != "baseline")


def test_multi_and_dist_entry_points_keep_the_result_on_device():
    """b2q_execute_work_unit_multi over every visible device (up to 2) and b2q_execute_work_unit_dist on a one-rank
    communicator: the flag reaches their finalize, the columns match the default run's."""
    import torch
    from test_gpu_multi import device_views
    ndev = min(executor.lib().b2q_device_count(), 2)
    table = random_table(40000, seed=29, frag_rows=5000)
    views, _keep = device_views(table, ndev)
    ex = executor.Executor()
    comms = executor.Comm.init_all(list(range(ndev)))
    try:
        for sql in RAND_QUERIES[:6] + oq.RAND_ORDER_QUERIES[:2]:
            unit = sqlmini.parse(sql, table, RAND_NAMES)
            base, res = [executor.execute_work_unit_multi(comms, ex, 4001, True, views, unit, has_cardinality_estimation=True,
                                                           eo=executor.execution_options(result_on_device=on)) for on in (False, True)]
            check_device_columns(res)
            gu.rows_equal(res.rows(), base.rows(), col_tol=gu.column_tolerances(base.getQueryMemDesc(), 40000))
    finally:
        for c in comms:
            c.destroy()
    uid = executor.Comm.unique_id()
    comm = executor.Comm.init_rank(uid, 1, 0, torch.cuda.current_device())
    try:
        dev = gu.DeviceTable(table)
        for sql in RAND_QUERIES[:4]:
            unit = sqlmini.parse(sql, table, RAND_NAMES)
            base, res = [executor.execute_work_unit_dist(comm, ex, 4001, True, dev.table, unit, has_cardinality_estimation=True,
                                                          eo=executor.execution_options(result_on_device=on)) for on in (False, True)]
            check_device_columns(res)
            gu.rows_equal(res.rows(), base.rows(), col_tol=gu.column_tolerances(base.getQueryMemDesc(), 40000))
    finally:
        comm.destroy()
