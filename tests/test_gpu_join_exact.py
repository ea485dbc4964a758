"""The hash-join probe on the device against the exact join reference (join_exact_ref), in every join-table layout.

The matrix is layout x join type (INNER, LEFT) x table mode (non-grouped, shared-memory perfect hash, forced HBM/L2 perfect
hash, baseline hash on an inner column) x outer key width (INT8 / INT16 / INT32 / BIGINT, FIXED(8|16|32), NOT NULL INT and
FIXED(16)).  Every aggregate is compared exactly with int_exact_ref over the rows the reference joined, and every query asserts
its kernel and the join table it probed (ResultSet.stats()["join_table"], B2Q_STAT_JOIN_TABLE).  The last test checks that
every layout was observed.

Also here: staged tables over 64 KB whose size is not a multiple of 16 bytes; the group table's replicas giving way to the
join table; fact tables in HBM and streamed from the host, 1 Mi rows; the inner table in device memory at element-aligned
(not 16-byte-aligned) offsets of one buffer; DOUBLE inner columns against fp_exact_ref; COUNT(DISTINCT) and the NDV estimator
over an inner column; b2q_launch with the caller's int32 table; stale chunk stats of the uint16 column; and each experiment
switch (B2Q_JOIN_SMEM / _PACK / _SLOT16 / _CG / _SMEM_KB) in a child pytest run."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import gpu_util as gu
import int_exact_ref as ix
import join_exact_ref as jr
import oracle_lib
import sqlmini
from heavydb_b200 import abi, executor
from test_int_exact_ref import check_rows
from test_join_exact_ref import FORCE, KERNEL, expected_layout, guess_of, parse, reference

pytestmark = pytest.mark.gpu

ROWS, FRAG = 1 << 16, 1 << 14
BIG_ROWS, BIG_FRAG = 1 << 20, 1 << 18
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# one case per staged / HBM layout runs the whole matrix; the other edge cases run INNER / LEFT x two modes
PRIMARY = ["int32_smem_multi_copy", "int32_hbm", "int2_smem_multi_copy", "int2_hbm", "uint16_span_65533"]
MATRIX = [(c, left, mode) for c in PRIMARY for left in (False, True) for mode in ("non_grouped", "smem", "global", "baseline")]
MATRIX += [(c.name, left, mode) for c in jr.CASES if c.name not in PRIMARY for left in (False, True) for mode in ("non_grouped", "smem")]
MATRIX += [("int2_smem_multi_copy", left, "smem_wide") for left in (False, True)]
# b2q_launch reads the caller's table (JOIN_TABLE_CALLER) for plans the planner stages as {row, value} and as uint16
LAUNCH_CASES = ["int2_smem_multi_copy", "uint16_span_65533"]
# the matrix targets every layout (under the default settings: a child run with a switch set targets fewer)
assert {expected_layout(jr.CASE[c], m) for c, _l, m in MATRIX} | {abi.JOIN_TABLE_CALLER} == set(range(1, 7)) or any(
    k in os.environ for k in ("B2Q_JOIN_SMEM", "B2Q_JOIN_PACK", "B2Q_JOIN_SLOT16"))

OBSERVED = set()
_TABLES = {}


def tables(name, rows=ROWS, frag=FRAG):
    """(fact, fact on the device, dim) of an edge case, built once per module."""
    key = (name, rows, frag)
    if key not in _TABLES:
        c = jr.CASE[name]
        fact = jr.fact_table(c, rows, frag, seed=11)
        _TABLES[key] = (fact, gu.DeviceTable(fact), jr.dim_table(c, seed=13))
    return _TABLES[key]


def execute(unit, fact, dev=None, guess=0, card=False, force=0):
    eo = executor.execution_options(force_kernel=force)
    ex = executor.Executor()
    if dev is not None:
        return ex.executeWorkUnit(guess, True, dev.table, unit, eo=eo, has_cardinality_estimation=card, memory_level=abi.GPU_LEVEL)
    return ex.executeWorkUnit(guess, True, fact, unit, eo=eo, has_cardinality_estimation=card, memory_level=abi.CPU_LEVEL)


def checked(rs, groups, w, kernel, layout):
    assert rs.getQueryMemDesc().kernel == kernel
    assert rs.stats()["join_table"] == layout
    OBSERVED.add(layout)
    bad, skipped = check_rows(rs.rows(decimal_to_double=False), rs.getQueryMemDesc(), groups, w, device=True)
    assert not bad and not skipped, bad[:6]


def run_case(name, left, mode, keys, fact, dev, dim, frag):
    c = jr.CASE[name]
    for key in keys:
        key_col = jr.KEY_NAMES.index(key)
        unit = parse(c, fact, dim, key_col, left, mode)
        groups, w, _j = reference(c, fact, dim, key_col, left, mode, frag_rows=frag)
        guess, card = guess_of(mode, groups)
        rs = execute(unit, fact, dev, guess, card, FORCE.get(mode, 0))
        checked(rs, groups, w, KERNEL[mode], expected_layout(c, mode))


@pytest.mark.parametrize("case,left,mode", MATRIX, ids=[f"{c}-{'left' if l else 'inner'}-{m}" for c, l, m in MATRIX])
def test_join_matrix(case, left, mode):
    fact, dev, dim = tables(case)
    keys = jr.KEY_NAMES if case in PRIMARY else ["k8", "k32", "k64", "f16", "f32"]
    run_case(case, left, mode, keys, fact, dev, dim, FRAG)


@pytest.mark.parametrize("case", ["int32_hbm", "int2_smem_multi_copy", "uint16_int8"])
def test_host_streamed_and_device_resident_facts_of_1mi_rows(case):
    fact, dev, dim = tables(case, BIG_ROWS, BIG_FRAG)
    for d in (dev, None):
        for left in (False, True):
            run_case(case, left, "smem", ["k64"], fact, d, dim, BIG_FRAG)


def device_inner(dim):
    """The inner table on the device: its columns in ONE buffer at element-aligned offsets that are not 16-byte aligned, as
    ColumnFetcher::getAllTableColumnFragments may hand them over."""
    import torch
    f = dim.fragments[0]
    offs, off = [], 0
    for a in f.host_cols:
        off = (off + a.itemsize - 1) // a.itemsize * a.itemsize
        if off % 16 == 0:
            off += a.itemsize
        offs.append(off)
        off += a.nbytes
    host = np.zeros(off, np.uint8)
    for a, o in zip(f.host_cols, offs):
        host[o:o + a.nbytes] = a.view(np.uint8)
    buf = torch.from_numpy(host).cuda()
    t = abi.Table(dim.col_types, encoded_sizes=dim.encoded_sizes)
    t.add_device_fragment(f.num_tuples, [buf.data_ptr() + o for o in offs], f.stats)
    torch.cuda.synchronize()
    assert any((buf.data_ptr() + o) % 16 for o in offs)
    return buf, t.build(abi.GPU_LEVEL)


@pytest.mark.parametrize("case", ["int32_hbm", "int2_smem_multi_copy", "int2_hbm", "uint16_dict8", "uint16_int8"])
def test_inner_table_in_device_memory(case):
    c = jr.CASE[case]
    fact, dev, dim = tables(case)
    buf, built = device_inner(dim)
    for left in (False, True):
        for mode in ("non_grouped", "smem"):
            key_col = jr.KEY_NAMES.index("k64")
            unit = parse(c, fact, dim, key_col, left, mode)
            unit.unit.inner_table = C.cast(C.pointer(built.info), C.c_void_p)
            groups, w, _j = reference(c, fact, dim, key_col, left, mode)
            checked(execute(unit, fact, dev), groups, w, KERNEL[mode], expected_layout(c, mode))
    del buf


@pytest.mark.parametrize("case", ["int32_smem_multi_copy", "int32_hbm", "int2_hbm"])
def test_double_inner_column_against_the_exact_sum(case):
    """SUM / AVG / MIN / MAX / COUNT of the inner DOUBLE w within fp_exact_ref's bound (an fp column is never packed)."""
    from test_gpu_fp_exact import check_rows as fp_check_rows
    c = jr.CASE[case]
    fact, dev, dim = tables(case)
    stage = os.environ.get("B2Q_JOIN_SMEM") != "0"
    for left in (False, True):
        how = "LEFT JOIN" if left else "JOIN"
        sql = f"SELECT t.x, SUM(d.w), AVG(d.w), MIN(d.w), MAX(d.w), COUNT(d.w), COUNT(*) FROM t {how} d ON t.k32 = d.id GROUP BY t.x;"
        unit = sqlmini.parse(sql, fact, jr.FACT_NAMES, inner=(dim, jr.DIM_NAMES))
        j = jr.join(fact, dim, jr.KEY_NAMES.index("k32"), 0, left)
        rs = execute(unit, fact, dev)
        assert rs.getQueryMemDesc().kernel == abi.KERNEL_PERFECT_SMEM
        layout = jr.layout(c.entries, False, False, True, 4096, 1, stage=stage)[0]
        assert rs.stats()["join_table"] == layout
        OBSERVED.add(layout)
        fp_check_rows(rs.rows(), rs.getQueryMemDesc(), jr.fp_groups(j, ("outer", len(jr.FACT_KEYS)), 3))


@pytest.mark.parametrize("case", ["uint16_dict8", "uint16_span_65533", "int2_hbm"])
def test_count_distinct_and_ndv_estimator_over_an_inner_column(case):
    """COUNT(DISTINCT d.a) on its bitmap (uint16 and {row, value} HBM tables), and the NDV estimator over d.a: its bitmap bit for
    bit with the oracle's, its estimate within linear counting's error of the exact distinct count of the joined values.  The
    estimator's program packs no column, so it probes int32 row tables: staged, or in HBM for the 60 000-entry table."""
    from test_ndv_estimator import estimator_unit
    c = jr.CASE[case]
    fact, dev, dim = tables(case)
    key_col = jr.KEY_NAMES.index("k32")
    for left in (False, True):
        how = "LEFT JOIN" if left else "JOIN"
        sql = f"SELECT t.x, COUNT(DISTINCT d.a), COUNT(*) FROM t {how} d ON t.k32 = d.id GROUP BY t.x;"
        unit = sqlmini.parse(sql, fact, jr.FACT_NAMES, inner=(dim, jr.DIM_NAMES))
        j = jr.join(fact, dim, key_col, 0, left)
        groups = jr.int_groups(j, ("outer", len(jr.FACT_KEYS)), 1, True)
        rs = execute(unit, fact, dev)
        checked(rs, groups, ix.WIDTH[c.packed], abi.KERNEL_PERFECT_SMEM, expected_layout(c, "smem"))
    unit = estimator_unit(fact, jr.FACT_NAMES, [(1, 1)], inner=(dim, key_col, 0))
    ref = oracle_lib.execute(unit, fact, num_threads=4)
    rs = executor.Executor().executeWorkUnit(1, True, dev.table, unit, memory_level=abi.GPU_LEVEL)
    # the estimator's program packs no inner column: its table holds int32 rows, staged where E * 4 B fits
    assert rs.stats()["join_table"] == jr.layout(c.entries, False, False, True, 4096, 1, stage=os.environ.get("B2Q_JOIN_SMEM") != "0")[0]
    OBSERVED.add(rs.stats()["join_table"])
    assert np.array_equal(rs.getHostEstimatorBuffer(), ref.buffer().view(np.uint8))
    a = jr.join(fact, dim, key_col, 0, False).inner(1)
    exact = len(set(a[a != dim.physical_null(1)].tolist()))
    assert abs(rs.getNDVEstimator() - exact) <= max(3, 0.01 * exact), (rs.getNDVEstimator(), exact)


def test_stale_chunk_stats_of_the_uint16_column():
    """A value of the packed column below its chunk-stats minimum: the uint16 table cannot encode it and the query fails with
    KEY_OUT_OF_RANGE; the {row, value} table of the same query (uint16 slots switched off), and the same table read with a
    second inner column, give the exact answer."""
    c = jr.CASE["uint16_span_65533"]
    fact, dev, _dim = tables(c.name)
    dim = jr.dim_table(c, seed=13)
    dim.fragments[0].stats[1].int_min += 1                            # stale: the column's least value is now below it
    key_col = jr.KEY_NAMES.index("k32")
    w = ix.WIDTH[c.packed]
    j = jr.join(fact, dim, key_col, 0, False)
    sql = "SELECT COUNT(*), COUNT(d.a), SUM(d.a), MIN(d.a), MAX(d.a), AVG(d.a) FROM t JOIN d ON t.k32 = d.id"
    unit = sqlmini.parse(sql + ";", fact, jr.FACT_NAMES, inner=(dim, jr.DIM_NAMES))
    groups = jr.int_groups(j, None, 1, True)
    layout = expected_layout(c, "non_grouped")
    if layout != abi.JOIN_TABLE_UINT16_SMEM:       # a child run with uint16 slots switched off
        checked(execute(unit, fact, dev), groups, w, abi.KERNEL_NON_GROUPED, layout)
    else:
        with pytest.raises(executor.QueryExecutionError) as e:
            execute(unit, fact, dev)
        assert e.value.code == abi.ERR_KEY_OUT_OF_RANGE
    unit = sqlmini.parse(sql + " WHERE d.b < 0;", fact, jr.FACT_NAMES, inner=(dim, jr.DIM_NAMES))
    mask = ix.passing(ix.WIDTH["INT64"], j.inner(2), True, ("cmp", "<", 0))
    packed = os.environ.get("B2Q_JOIN_PACK") != "0"
    checked(execute(unit, fact, dev), jr.int_groups(j, None, 1, True, mask=mask), w, abi.KERNEL_NON_GROUPED,
            abi.JOIN_TABLE_INT2_HBM if packed else abi.JOIN_TABLE_INT32_HBM)


# ---- b2q_launch: the caller's int32 table, read in place -------------------------------------------------------------------
def launch(q, fact_dev, inner_ptrs, join_table, out, err):
    import torch
    L = executor.lib()
    nf = len(fact_dev.table.fragments)
    per_frag = [(C.c_void_p * (fact_dev.table.num_cols + len(inner_ptrs)))(*([p or None for p in f.dev_ptrs] + inner_ptrs))
                for f in fact_dev.table.fragments]
    col_buffers = (C.POINTER(C.c_void_p) * nf)(*[C.cast(a, C.POINTER(C.c_void_p)) for a in per_frag])
    num_rows = (C.c_int64 * nf)(*[f.num_tuples for f in fact_dev.table.fragments])
    num_frags, num_tables = C.c_uint32(nf), C.c_uint32(2 if join_table is not None else 1)
    gb = torch.tensor([out.data_ptr()], dtype=torch.int64, device="cuda")
    prm = abi.Params()
    prm.error_codes = err.data_ptr()
    prm.group_by_buffers = gb.data_ptr()
    prm.num_fragments, prm.num_tables = C.pointer(num_frags), C.pointer(num_tables)
    prm.col_buffers = col_buffers
    prm.num_rows = num_rows
    jh = (C.c_int64 * 1)(join_table.data_ptr() if join_table is not None else 0)
    prm.join_hash_tables = C.cast(jh, C.c_void_p) if join_table is not None else None
    torch.cuda.synchronize()
    rc = L.b2q_launch(q, C.byref(prm), None)
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("case", LAUNCH_CASES)
@pytest.mark.parametrize("mode", ["non_grouped", "smem"])
def test_b2q_launch_reads_the_callers_int32_table(case, mode):
    import torch
    c = jr.CASE[case]
    fact, dev, dim = tables(case)
    key_col = jr.KEY_NAMES.index("k64")
    unit = parse(c, fact, dim, key_col, False, mode)
    groups, w, j = reference(c, fact, dim, key_col, False, mode)
    assert execute(unit, fact, dev).stats()["join_table"] == expected_layout(c, mode)    # what the planner stages
    L = executor.lib()
    bt = dev.table.build(abi.GPU_LEVEL)
    co, eo = executor.compilation_options(), executor.execution_options()
    q = C.c_void_p()
    assert L.b2q_plan(C.byref(unit.unit), C.byref(bt.info), C.byref(co), C.byref(eo), 0, 0, C.byref(q)) == 0, L.b2q_last_error_message()
    try:
        plan = L.b2q_query_plan(q).contents
        assert (plan.join_min_key, plan.join_entry_count) == (j.jt.min_key, j.jt.entry_count)
        # the reference's own one-to-one table: int32 slots, -1 = no row
        table = torch.from_numpy(j.jt.row_of.astype(np.int32)).cuda()
        dcols = [torch.from_numpy(a.view(np.uint8).copy()).cuda() for a in dim.fragments[0].host_cols]
        out = torch.zeros(max(int(plan.buffer_size), 8), dtype=torch.uint8, device="cuda")
        err = torch.zeros(1, dtype=torch.int32, device="cuda")
        rc = launch(q, dev, [t.data_ptr() for t in dcols], table, out, err)
        assert rc == 0, L.b2q_last_error_message()
        assert int(err.item()) == 0
        assert L.b2q_last_launch_stat(abi.STAT_JOIN_TABLE) == abi.JOIN_TABLE_CALLER
        assert L.b2q_last_launch_stat(abi.STAT_KERNEL_LAUNCHES) == -1
        OBSERVED.add(abi.JOIN_TABLE_CALLER)
        rs = executor.Executor().resultSetFromStorage(out.cpu().numpy()[: int(plan.buffer_size)], unit, fact)
        bad, skipped = check_rows(rs.rows(decimal_to_double=False), rs.getQueryMemDesc(), groups, w, device=True)
        assert not bad and not skipped, bad[:6]
        # a join level without JOIN_HASH_TABLES is refused
        assert launch(q, dev, [t.data_ptr() for t in dcols], None, out, err) == abi.ERR_INVALID_ARGUMENT
    finally:
        L.b2q_query_free(q)
    # ... and so is JOIN_HASH_TABLES for a plan without one
    plain = sqlmini.parse("SELECT t.x, COUNT(*) FROM t GROUP BY t.x;", fact, jr.FACT_NAMES)
    q = C.c_void_p()
    assert L.b2q_plan(C.byref(plain.unit), C.byref(bt.info), C.byref(co), C.byref(eo), 0, 0, C.byref(q)) == 0
    try:
        assert launch(q, dev, [], table, out, err) == abi.ERR_INVALID_ARGUMENT
    finally:
        L.b2q_query_free(q)


# ---- experiment switches: each read once per process, hence a child run -------------------------------------------------------
SWITCHES = [("B2Q_JOIN_SMEM", "0"), ("B2Q_JOIN_PACK", "0"), ("B2Q_JOIN_SLOT16", "0"), ("B2Q_JOIN_CG", "1"), ("B2Q_JOIN_SMEM_KB", "8")]


@pytest.mark.parametrize("var,value", SWITCHES, ids=[f"{k}={v}" for k, v in SWITCHES])
def test_experiment_switches(var, value):
    if var in os.environ:
        pytest.skip("already a child run")
    env = dict(os.environ, **{var: value})
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", "tests/test_gpu_join_exact.py",
                        "-k", "test_join_matrix and (int2_hbm- or uint16_span_65533 or int32_smem_multi_copy or int2_smem_multi_copy) "
                              "and (inner-smem or left-global or left-baseline or smem_wide) or test_stale_chunk_stats"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-1000:]
    assert " passed" in r.stdout


def test_zz_every_layout_was_observed(request):
    """Every B2Q_JOIN_TABLE_* value 1-6 came back from at least one passing query of this module."""
    names = {i.name for i in request.session.items}
    if not all(f"test_join_matrix[{c}-{'left' if l else 'inner'}-{m}]" in names for c, l, m in MATRIX) or any(
            k in os.environ for k in ("B2Q_JOIN_SMEM", "B2Q_JOIN_PACK", "B2Q_JOIN_SLOT16")):
        pytest.skip("only a run of the whole matrix under the default settings observes every layout")
    assert request.session.testsfailed == 0
    assert OBSERVED == set(range(1, 7)), OBSERVED
