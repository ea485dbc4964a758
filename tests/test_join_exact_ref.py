"""The join reference (join_exact_ref) on the CPU.

- The oracle equals the reference on every edge table, INNER and LEFT, for every outer key width: the aggregates of the joined
  rows come from int_exact_ref, so a wrong probe shows as a wrong group.
- The host emulation of the lowered join program (tests/cpp/filter_emulator.cpp), fed with the reference's own probe, gives
  the reference's groups.
- Each mutation of the probe in join_exact_ref.MUTATIONS changes at least one result on the edge tables.
- join_exact_ref.layout restates the planner's choice of join-table layout; over b2q_plan's join fields and group-table sizes
  it gives the layout the planner chose, for every case and table mode, and the cases reach all six layouts."""
import ctypes as C
import os

import numpy as np
import pytest

import int_exact_ref as ix
import join_exact_ref as jr
import oracle_lib
import sqlmini
from heavydb_b200 import abi, executor
from test_filter_lowering import emu  # noqa: F401  (emu is a fixture)
from test_int_exact_ref import aggs_of, check_rows

FRAG_ROWS = 2500
CPU_ROWS = 6000
X_COL, G_COL = len(jr.FACT_KEYS), len(jr.FACT_KEYS) + 1
MODES = ["non_grouped", "smem", "global", "baseline", "smem_wide"]
GROUP_KEY = {"non_grouped": None, "smem": ("outer", X_COL), "global": ("outer", X_COL), "smem_wide": ("outer", G_COL),
             "baseline": ("inner", 2)}
KERNEL = {"non_grouped": abi.KERNEL_NON_GROUPED, "smem": abi.KERNEL_PERFECT_SMEM, "smem_wide": abi.KERNEL_PERFECT_SMEM,
          "global": abi.KERNEL_PERFECT_GLOBAL, "baseline": abi.KERNEL_BASELINE_GLOBAL}
FORCE = {"global": abi.KERNEL_PERFECT_GLOBAL}
B_FILTER = ("cmp", "<", 0)


def arg_of(case: jr.Case):
    """(inner column, width) of the aggregates' argument: the attribute a where the case reads it, else the BIGINT b."""
    return (1, ix.WIDTH[case.packed]) if case.reads_a else (2, ix.WIDTH["INT64"])


def reads_b(case: jr.Case, mode: str) -> bool:
    return case.reads_b or mode == "baseline" or not case.reads_a


def query(case: jr.Case, key_col: int, left: bool, mode: str) -> str:
    """COUNT(*) and every integer aggregate of the argument, over t [LEFT] JOIN d ON t.<key> = d.id; a case that reads b
    filters on d.b < 0; baseline mode groups by d.b (an inner BIGINT: sparse, so baseline hash)."""
    arg, w = arg_of(case)
    aggs = aggs_of(w).replace("(v)", f"(d.{jr.DIM_NAMES[arg]})").replace("DISTINCT v)", f"DISTINCT d.{jr.DIM_NAMES[arg]})")
    key = GROUP_KEY[mode]
    sel = "" if key is None else ("d.b, " if key[0] == "inner" else f"t.{jr.FACT_NAMES[key[1]]}, ")
    where = " WHERE d.b < 0" if case.reads_b else ""
    group = "" if key is None else f" GROUP BY {sel[:-2]}"
    how = "LEFT JOIN" if left else "JOIN"
    return f"SELECT {sel}{aggs} FROM t {how} d ON t.{jr.KEY_NAMES[key_col]} = d.id{where}{group};"


def parse(case, fact, dim, key_col, left, mode):
    return sqlmini.parse(query(case, key_col, left, mode), fact, jr.FACT_NAMES, inner=(dim, jr.DIM_NAMES))


def reference(case, fact, dim, key_col, left, mode, probe=None, frag_rows=FRAG_ROWS):
    """(int_exact_ref groups, argument width, the Joined) of one query."""
    j = jr.join(fact, dim, key_col, 0, left, probe)
    arg, w = arg_of(case)
    mask = ix.passing(ix.WIDTH["INT64"], j.inner(2), True, B_FILTER) if case.reads_b else None
    return jr.int_groups(j, GROUP_KEY[mode], arg, True, mask=mask, frag_rows=frag_rows), w, j


def attr_span(case: jr.Case) -> int:
    """The chunk-stats span of the attribute a (attr_values puts both ends of its range in the table)."""
    w = ix.WIDTH[case.packed]
    return case.span or w.hi - w.lo


def expected_layout(case: jr.Case, mode: str, env=os.environ) -> int:
    """The layout a query of this case gets, by join_exact_ref.layout under the experiment switches in `env`
    (B2Q_JOIN_SMEM / _PACK / _SLOT16).  The group tables of these queries take a few KB: every case's join table is sized away
    from the thresholds by more than that (test_restated_layout_rule_matches_the_planner checks the exact rule)."""
    on = {k: env.get(k, "1") != "0" for k in ("B2Q_JOIN_SMEM", "B2Q_JOIN_PACK", "B2Q_JOIN_SLOT16")}
    packed = on["B2Q_JOIN_PACK"] and case.reads_a
    n_inner = int(case.reads_a) + int(reads_b(case, mode))
    slot16_ok = on["B2Q_JOIN_SLOT16"] and jr.slot16_eligible(packed, n_inner, attr_span(case))
    return jr.layout(case.entries, packed, slot16_ok, True, 4096, 1, stage=on["B2Q_JOIN_SMEM"])[0]


def guess_of(mode, groups):
    return (2 * len(groups) + 16, True) if mode == "baseline" else (0, False)


@pytest.fixture(scope="module")
def tables():
    return {c.name: (jr.fact_table(c, CPU_ROWS, FRAG_ROWS, seed=3), jr.dim_table(c, seed=5)) for c in jr.CASES}


# ---- the oracle -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("left", [False, True], ids=["inner", "left"])
@pytest.mark.parametrize("case", [c.name for c in jr.CASES])
def test_oracle_equals_the_reference(tables, case, left):
    c = jr.CASE[case]
    fact, dim = tables[case]
    for key_col in range(len(jr.FACT_KEYS)):
        for mode in ("non_grouped", "smem", "baseline"):
            unit = parse(c, fact, dim, key_col, left, mode)
            groups, w, _j = reference(c, fact, dim, key_col, left, mode)
            guess, card = guess_of(mode, groups)
            res = oracle_lib.execute(unit, fact, entry_guess=guess, has_card=card)
            bad, _skipped = check_rows(res.rows(decimal_to_double=False), res.plan, groups, w)
            assert not bad, (query(c, key_col, left, mode), bad[:6])


def test_the_edge_tables_reach_the_edges(tables):
    """Keys congruent mod 2^32 to an in-range key, min - 1 and min + E, NULL and FIXED-NULL outer keys, NULL inner keys, packed
    values at the NULL sentinel's neighbours, chunk stats wider than the keys."""
    c = jr.CASE["int2_smem_multi_copy"]
    fact, dim = tables[c.name]
    k64 = jr.column(fact, jr.KEY_NAMES.index("k64")).astype(np.int64)
    lo, hi = jr.stats_range(dim, 0)
    assert {lo - 1, hi + 1, lo + 2 ** 32, hi - 2 ** 32} <= set(k64.tolist())
    f16 = jr.column(fact, jr.KEY_NAMES.index("f16"))
    assert (f16 == -(2 ** 15)).any() and (f16 == -(2 ** 15) + 1).any()
    assert (jr.column(dim, 0) == abi.NULL_BIGINT).any()
    a = jr.column(dim, 1)
    assert {-(2 ** 15), -(2 ** 15) + 1, -(2 ** 15) + 2, 2 ** 15 - 1} <= set(a.tolist())
    padded = jr.CASE["uint16_int8"]
    lo, hi = jr.stats_range(tables[padded.name][1], 0)
    keys = jr.column(tables[padded.name][1], 0)
    keys = keys[keys != abi.NULL_BIGINT]
    assert lo < keys.min() and hi > keys.max() and hi - lo + 1 == padded.entries
    s = tables["uint16_span_65533"][1].fragments[0].stats[1]
    assert s.int_max - s.int_min == 65533
    s = tables["int2_hbm_span_65534"][1].fragments[0].stats[1]
    assert s.int_max - s.int_min == 65534


def test_duplicate_and_out_of_range_inner_keys_are_named():
    dim = abi.Table([(abi.kINT, True), (abi.kINT, True)])
    dim.add_host_fragment([np.array([3, 4, 3], np.int32), np.arange(3, dtype=np.int32)])
    with pytest.raises(jr.NotOneToOne):
        jr.Probe().build(dim, 0)
    dim = abi.Table([(abi.kINT, True), (abi.kINT, True)])
    dim.add_host_fragment([np.array([3, 4, 9], np.int32), np.arange(3, dtype=np.int32)])
    dim.fragments[0].stats[0].int_max = 8                            # stale stats: 9 is outside them
    with pytest.raises(jr.KeyOutOfRange):
        jr.Probe().build(dim, 0)


# ---- the host emulation of the lowered join program ----------------------------------------------------------------------------
def run_program_on_reference_probe(emu, unit, fact, dim, j, left, guess, card):
    """The whole lowered program over the rows the reference joined: inner columns gathered at the reference's inner row (the
    physical NULL where a LEFT row has no match) -> the result buffer, read back as a ResultSet."""
    emu.b2q_test_run_program_joined.restype = C.c_int32
    emu.b2q_test_run_program_joined.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.POINTER(C.c_void_p)), C.POINTER(C.c_int64),
                                                C.POINTER(C.POINTER(C.c_uint8)), C.c_void_p]
    L = executor.lib()
    bt = fact.build(abi.CPU_LEVEL)
    co, eo = executor.compilation_options(), executor.execution_options()
    h = C.c_void_p()
    assert L.b2q_plan(C.byref(unit.unit), C.byref(bt.info), C.byref(co), C.byref(eo), guess, int(card), C.byref(h)) == 0, L.b2q_last_error_message()
    plan = L.b2q_query_plan(h).contents
    full = jr.join(fact, dim, j.outer_col, 0, True)                 # every outer row with its inner row (or -1)
    keep, valids, base = [], [], 0
    for f in fact.fragments:
        idx = full.idx[base:base + f.num_tuples]
        base += f.num_tuples
        gathered = []
        for c in range(dim.num_cols):
            col = jr.column(dim, c)
            g = col[np.maximum(idx, 0)].copy()
            g[idx < 0] = dim.physical_null(c)
            gathered.append(g)
        arrays = list(f.host_cols) + gathered
        keep.append((arrays, (C.c_void_p * len(arrays))(*[x.ctypes.data for x in arrays])))
        valids.append(np.ascontiguousarray(np.ones(idx.size, np.uint8) if left else (idx >= 0).astype(np.uint8)))
    nf = len(keep)
    frag_cols = (C.POINTER(C.c_void_p) * nf)(*[C.cast(k[1], C.POINTER(C.c_void_p)) for k in keep])
    frag_rows = (C.c_int64 * nf)(*[f.num_tuples for f in fact.fragments])
    frag_valid = (C.POINTER(C.c_uint8) * nf)(*[v.ctypes.data_as(C.POINTER(C.c_uint8)) for v in valids])
    out = np.zeros(max(plan.buffer_size, 8), dtype=np.uint8)
    rc = emu.b2q_test_run_program_joined(h, nf, frag_cols, frag_rows, frag_valid, out.ctypes.data)
    L.b2q_query_free(h)
    assert rc == 0, rc
    return executor.Executor().resultSetFromStorage(out[:plan.buffer_size], unit, fact, max_groups_buffer_entry_guess=guess,
                                                    has_cardinality_estimation=card)


@pytest.mark.parametrize("left", [False, True], ids=["inner", "left"])
@pytest.mark.parametrize("case", ["int32_smem", "int2_smem_multi_copy", "uint16_int8", "uint16_dict8", "int2_smem_near_int32_max"])
def test_emulated_join_program_equals_the_reference(emu, tables, case, left):  # noqa: F811
    c = jr.CASE[case]
    fact, dim = tables[case]
    for key in ("k8", "k32", "k64", "f16", "f16nn"):
        key_col = jr.KEY_NAMES.index(key)
        for mode in ("non_grouped", "smem"):
            unit = parse(c, fact, dim, key_col, left, mode)
            groups, w, j = reference(c, fact, dim, key_col, left, mode)
            rs = run_program_on_reference_probe(emu, unit, fact, dim, j, left, 0, False)
            bad, _skipped = check_rows(rs.rows(decimal_to_double=False), rs.getQueryMemDesc(), groups, w)
            assert not bad, (query(c, key_col, left, mode), bad[:6])


# ---- the reference is sensitive ------------------------------------------------------------------------------------------------
def _results(case, fact, dim, probe):
    out = []
    for key_col in range(len(jr.FACT_KEYS)):
        for left in (False, True):
            groups, _w, j = reference(case, fact, dim, key_col, left, "smem", probe)
            out.append({k: (g.rows, g.count, g.sum, g.min, g.max) for k, g in groups.items()})
            if case.layout == abi.JOIN_TABLE_UINT16_SMEM:
                out.append(j.inner_via_slot16(1, int(dim.fragments[0].stats[1].int_min)).tolist())
    return out


@pytest.mark.parametrize("mutation", jr.MUTATIONS, ids=lambda m: m.__name__)
def test_every_mutation_of_the_probe_changes_a_result(tables, mutation):
    changed = []
    for c in jr.CASES:
        fact, dim = tables[c.name]
        if _results(c, fact, dim, mutation()) != _results(c, fact, dim, jr.Probe()):
            changed.append(c.name)
    assert changed, f"{mutation.__name__} changes nothing"


def test_uint16_slots_read_back_the_gathered_column(tables):
    for c in jr.CASES:
        if c.layout != abi.JOIN_TABLE_UINT16_SMEM:
            continue
        fact, dim = tables[c.name]
        vmin = int(dim.fragments[0].stats[1].int_min)
        for left in (False, True):
            j = jr.join(fact, dim, jr.KEY_NAMES.index("k32"), 0, left)
            assert np.array_equal(j.inner_via_slot16(1, vmin), j.inner(1)), c.name
            assert (j.inner(1) == dim.physical_null(1)).any() and (j.idx >= 0).any()


# ---- the layout rule ---------------------------------------------------------------------------------------------------------
def planned_layout(emu, unit, fact, guess, card, force=0):
    """(b2q_plan's Plan, [JOIN_TABLE_*, use_smem, replica_bytes, replicas, join_bytes]) of the planner's choice."""
    emu.b2q_test_join_layout.restype = C.c_int32
    emu.b2q_test_join_layout.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
    L = executor.lib()
    bt = fact.build(abi.CPU_LEVEL)
    co, eo = executor.compilation_options(), executor.execution_options(force_kernel=force)
    h = C.c_void_p()
    assert L.b2q_plan(C.byref(unit.unit), C.byref(bt.info), C.byref(co), C.byref(eo), guess, int(card), C.byref(h)) == 0, L.b2q_last_error_message()
    plan = abi.Plan()
    C.memmove(C.byref(plan), L.b2q_query_plan(h), C.sizeof(abi.Plan))
    out = (C.c_int64 * 5)()
    assert emu.b2q_test_join_layout(h, out) == 0
    L.b2q_query_free(h)
    return plan, list(out)


def replicas_before_the_join(replica_bytes: int) -> int:
    """Warp-private copies of a shared-memory group table (use_smem_table, 96 KB cap for the join kernels)."""
    rep = 1
    while rep < 32 and rep * 2 * replica_bytes <= 96 * 1024:
        rep *= 2
    return rep


def restated_layout(case, dim, plan, planned, mode):
    """join_exact_ref.layout over b2q_plan's join fields, the group table's size and the columns the query reads."""
    _kind, use_smem, replica_bytes, _rep, _jb = planned
    packed = case.reads_a and ix.WIDTH[case.packed].bits <= 32
    st = dim.fragments[0].stats[1]
    span = int(st.int_max) - int(st.int_min) if st.int_min <= st.int_max else None
    n_inner = int(case.reads_a) + int(reads_b(case, mode))
    assert plan.join_entry_count == plan.join_max_key - plan.join_min_key + 1
    return jr.layout(plan.join_entry_count, packed, jr.slot16_eligible(packed, n_inner, span), bool(use_smem), replica_bytes,
                     replicas_before_the_join(replica_bytes) if use_smem else 1)


def test_restated_layout_rule_matches_the_planner_and_reaches_every_layout(emu, tables):  # noqa: F811
    seen = set()
    for c in jr.CASES:
        assert expected_layout(c, "smem", env={}) == c.layout, c.name
        fact, dim = tables[c.name]
        lo, hi = jr.stats_range(dim, 0)
        for mode in MODES:
            unit = parse(c, fact, dim, jr.KEY_NAMES.index("k32"), False, mode)
            guess, card = (4096, True) if mode == "baseline" else (0, False)
            plan, planned = planned_layout(emu, unit, fact, guess, card, FORCE.get(mode, 0))
            assert (plan.join_min_key, plan.join_max_key, plan.join_entry_count) == (lo, hi, c.entries)
            assert plan.kernel == KERNEL[mode], (c.name, mode, plan.kernel)
            kind, rep, jb = restated_layout(c, dim, plan, planned, mode)
            assert [kind, rep, jb] == [planned[0], planned[3], planned[4]], (c.name, mode, planned)
            if mode != "smem_wide":
                assert kind == expected_layout(c, mode), (c.name, mode, kind)
            seen.add(kind)
    # the caller's table of b2q_launch: any plan with a join level, JOIN_HASH_TABLES given, is read in place
    seen.add(abi.JOIN_TABLE_CALLER)
    assert seen == set(range(1, 7)), seen


def test_replicas_give_way_to_the_staged_join_table(emu, tables):  # noqa: F811
    c = jr.CASE["int2_smem_multi_copy"]
    fact, dim = tables[c.name]
    unit = parse(c, fact, dim, jr.KEY_NAMES.index("k32"), False, "smem_wide")
    _plan, (kind, use_smem, replica_bytes, rep, jb) = planned_layout(emu, unit, fact, 0, False)
    assert kind == abi.JOIN_TABLE_INT2_SMEM and use_smem
    assert rep < replicas_before_the_join(replica_bytes), (rep, replica_bytes)
    assert jb > 2 * 65536 and (c.entries * 8) % 16 != 0                   # three bulk copies, the last one rounded up


def test_join_table_stat_mirrors_the_header(tmp_path):
    """B2Q_STAT_JOIN_TABLE and the B2Q_JOIN_TABLE_* values of include/b2q.h equal abi.py's; without a device, the last-launch
    statistic is the no-join value and every other statistic -1."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    names = ["NONE", "CALLER", "INT32_HBM", "INT2_HBM", "INT32_SMEM", "INT2_SMEM", "UINT16_SMEM"]
    prog = '#include <stdio.h>\n#include "b2q.h"\nint main(){\nprintf("STAT %d\\n", B2Q_STAT_JOIN_TABLE);\n'
    prog += "".join(f'printf("{n} %d\\n", B2Q_JOIN_TABLE_{n});\n' for n in names) + "return 0;}\n"
    src, exe = tmp_path / "join_table.c", tmp_path / "join_table"
    src.write_text(prog)
    subprocess.check_call(["gcc", "-I", os.path.join(root, "include"), "-o", str(exe), str(src)])
    out = dict(line.split() for line in subprocess.check_output([str(exe)]).decode().splitlines())
    assert int(out["STAT"]) == abi.STAT_JOIN_TABLE
    for n in names:
        assert int(out[n]) == getattr(abi, f"JOIN_TABLE_{n}"), n
    L = executor.lib()
    assert L.b2q_last_launch_stat(abi.STAT_JOIN_TABLE) == abi.JOIN_TABLE_NONE
    assert L.b2q_last_launch_stat(abi.STAT_KERNEL_LAUNCHES) == -1
