"""N > 1 host logic on CPU (world_size 2, gloo): the reference's fragment placement rule and the claim the whole
multi-GPU design rests on — that merging per-device partial tables (ResultSetStorage::reduce,
QueryEngine/ResultSetReduction.cpp:203-396,1496-1566) equals ONE all-reduce per dense identity-initialised array
with SUM / MIN / MAX — checked against the oracle's own host reduce over all fragments.

The dense-array model below mirrors the decomposition the CUDA library uses for its accumulators
(heavydb_b200/csrc/planner.cpp `lower`): COUNT and SUM as sums from 0, a non-NULL count next to every nullable
SUM/MIN/MAX (it decides the NULL sentinel at materialisation), MIN/MAX from +-identity, doubles as they are.  A merged
MIN / MAX equal to its identity (+inf, INT64_MAX) is a value, not NULL: EDGE_QUERIES hold such groups.
"""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import oracle_lib
import ref_tables as rt
from heavydb_b200 import abi, multigpu, sqlmini

I64_MAX, I64_MIN = np.iinfo(np.int64).max, np.iinfo(np.int64).min

QUERIES = [
    "SELECT x, COUNT(*), SUM(t), MIN(t), MAX(t), AVG(t) FROM test GROUP BY x;",
    "SELECT z, COUNT(*), SUM(ofd), MIN(ofd), MAX(ofd), COUNT(ofd), AVG(ofd) FROM test GROUP BY z;",
    "SELECT y, SUM(d), AVG(d), MIN(dn), MAX(dn), COUNT(dn) FROM test WHERE x = 7 GROUP BY y;",
    "SELECT smallint_nulls, COUNT(*), SUM(x) FROM test GROUP BY smallint_nulls;",
    "SELECT COUNT(*), SUM(t), MIN(z), MAX(w), AVG(y), SUM(u) FROM test WHERE z > 0;",
    "SELECT t, SUM(x) FROM test GROUP BY t;",
]
# over edge_table(): one row per fragment, so that both ranks hold part of every group
EDGE_QUERIES = ["SELECT k, MIN(d), MAX(d), MIN(b), MAX(b), COUNT(d), COUNT(b) FROM e GROUP BY k;",
                "SELECT MIN(d), MAX(d), MIN(b), MAX(b) FROM e WHERE k = 0;"]
EDGE_NAMES = ["k", "d", "b"]


def edge_table():
    """Group 0: MIN(d) = +inf and MIN(b) = MAX(b) = INT64_MAX, the MIN identities; 1: -inf and INT64_MIN + 1; 2: a NULL
    and a value on different ranks; 3: NULL only."""
    inf, nd, nb = np.inf, abi.NULL_DOUBLE, abi.NULL_BIGINT
    rows = [(0, inf, I64_MAX), (0, inf, I64_MAX), (1, -inf, I64_MIN + 1), (1, 5.0, 3), (2, 1.0, nb), (2, nd, 7), (3, nd, nb), (3, nd, nb)]
    t = abi.Table([(abi.kINT, True), (abi.kDOUBLE, False), (abi.kBIGINT, False)])
    for k, d, b in rows:
        t.add_host_fragment([np.array([k], np.int32), np.array([d]), np.array([b], np.int64)])
    return t


def test_fragment_placement_rule():
    """fragment_id % num_devices (InsertOrderFragmenter.cpp:435-443): every fragment on exactly one rank."""
    for world in (1, 2, 4, 8):
        frags = list(range(30))
        seen = []
        for r in range(world):
            mine = multigpu.shard_fragments(frags, r, world)
            assert all(f % world == r for f in mine)
            seen += mine
        assert sorted(seen) == frags


def _slot_views(plan, buf):
    rows = buf.view(np.int8).reshape(-1, plan.row_size)
    out = []
    for s in range(plan.num_slots):
        off = plan.slot_offset[s]
        out.append(np.ascontiguousarray(rows[:, off:off + 8]).view(np.int64).ravel().copy())
    return out


def dense_arrays(res):
    """oracle partial (reference row-wise layout, NULL-sentinel inits) -> identity-form dense arrays + reduce ops"""
    plan = res.plan
    n = res.entry_count()
    slots = _slot_views(plan, res.buffer())
    L = oracle_lib.lib()
    touched = np.array([not L.oracle_result_is_row_at_empty(res.h, i) for i in range(n)], dtype=np.int64)
    arrays = [("touched", touched, abi.RED_MAX)]
    for ti in range(plan.num_targets):
        t = plan.targets[ti]
        s = t.first_slot
        if not t.is_agg:
            continue
        v = slots[s]
        init = plan.init_vals[s]
        fp = t.agg_arg_type.type == abi.kDOUBLE
        if t.agg_kind == abi.kCOUNT:
            arrays.append((f"cnt{ti}", v.copy(), abi.RED_SUM))
        elif t.agg_kind in (abi.kSUM, abi.kAVG):
            is_null = (v == init) if t.skip_null_val else np.zeros(n, dtype=bool)
            if fp:
                d = v.view(np.float64).copy()
                d[is_null] = 0.0
                arrays.append((f"sum{ti}", d, abi.RED_SUM))
            else:
                w = v.copy()
                w[is_null] = 0
                arrays.append((f"sum{ti}", w, abi.RED_SUM))
            arrays.append((f"nn{ti}", (~is_null & (touched > 0)).astype(np.int64) if t.agg_kind == abi.kSUM else slots[s + 1].copy(), abi.RED_SUM))
        else:
            # MIN / MAX from +-identity, NULL decided by a non-NULL count (a real +inf or INT64_MAX is a value)
            ident = I64_MAX if t.agg_kind == abi.kMIN else I64_MIN
            nn = (touched > 0) & (v != init) if t.skip_null_val else touched > 0
            empty = ~nn
            arrays.append((f"nn{ti}", nn.astype(np.int64), abi.RED_SUM))
            if fp:
                d = v.view(np.float64).copy()
                d[empty] = np.inf if t.agg_kind == abi.kMIN else -np.inf
                arrays.append((f"mm{ti}", d, abi.RED_MIN if t.agg_kind == abi.kMIN else abi.RED_MAX))
            else:
                w = v.copy()
                w[empty] = ident
                arrays.append((f"mm{ti}", w, abi.RED_MIN if t.agg_kind == abi.kMIN else abi.RED_MAX))
    return arrays


def rebuild_rows(plan, merged, key_of_entry):
    """merged dense arrays -> rows (python values, None = NULL) for touched entries, like getNextRow"""
    m = {name: a for name, a, _ in merged}
    rows = []
    for i in np.nonzero(m["touched"] > 0)[0]:
        row = []
        for ti in range(plan.num_targets):
            t = plan.targets[ti]
            fp = t.agg_arg_type.type == abi.kDOUBLE
            if not t.is_agg:
                row.append(key_of_entry(int(i)))
            elif t.agg_kind == abi.kCOUNT:
                row.append(int(m[f"cnt{ti}"][i]))
            elif t.agg_kind == abi.kSUM:
                null = t.skip_null_val and m[f"nn{ti}"][i] == 0
                row.append(None if null else (float(m[f"sum{ti}"][i]) if fp else int(m[f"sum{ti}"][i])))
            elif t.agg_kind == abi.kAVG:
                c = int(m[f"nn{ti}"][i])
                row.append(None if c == 0 else float(m[f"sum{ti}"][i]) / c)
            else:
                v = m[f"mm{ti}"][i]
                null = t.skip_null_val and m[f"nn{ti}"][i] == 0
                row.append(None if null else (float(v) if fp else int(v)))
        rows.append(tuple(row))
    return rows


def _placed(table, rank, world):
    """This rank's fragments, the others as placeholders that carry only their chunk stats: chunk stats drive the plan
    (entry_count, keyless...), so every rank must plan on the WHOLE table's stats, exactly like the reference plans once for
    all devices."""
    plan_table = abi.Table(table.col_types)
    for fid, f in enumerate(table.fragments):
        if fid % world == rank:
            plan_table.fragments.append(f)
        else:
            plan_table.fragments.append(abi.Fragment(0, host_cols=[None] * len(f.host_cols), stats=f.stats, fragment_id=fid))
    return plan_table


def _worker(rank, world, port, out_q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        full = rt.make_table(rt.test_rows())                      # 10 fragments of 2 rows
        ok = True
        for sql, names, table in [(q, rt.TEST_NAMES, full) for q in QUERIES] + [(q, EDGE_NAMES, edge_table()) for q in EDGE_QUERIES]:
            plan_table = _placed(table, rank, world)
            unit = sqlmini.parse(sql, table, names)
            local = oracle_lib.execute(unit, plan_table)
            want = oracle_lib.execute(unit, table)
            assert local.plan.as_dict() == want.plan.as_dict()
            arrays = dense_arrays(local)
            tensors = [(torch.from_numpy(a), op) for _, a, op in arrays]
            multigpu.allreduce_tensors(tensors, dist)
            plan = want.plan

            def key_of_entry(i, plan=plan):
                if plan.has_nulls and i == plan.max_val - plan.min_val + 1:
                    return None
                return plan.min_val + i
            got = rebuild_rows(plan, arrays, key_of_entry)
            try:
                rt.assert_rows_match(got, want.rows(), fp_tol=1e-9)
            except AssertionError as e:  # noqa
                ok = False
                out_q.put((rank, sql, str(e)[:500]))
        # the estimator query: per-rank linear-counting bitmaps merge with OR (reduce_estimator_results)
        plan_table = _placed(full, rank, world)
        for cols in (["t"], ["x", "y"]):
            b = abi.UnitBuilder(full)
            b.estimator([rt.TEST_NAMES.index(c) for c in cols])
            eu = b.build()
            mine_bits = torch.from_numpy(oracle_lib.execute(eu, plan_table).buffer().view(np.uint8).copy())
            multigpu.allreduce_tensors([(mine_bits, abi.RED_BOR)], dist)
            want_bits = oracle_lib.execute(eu, full).buffer().view(np.uint8)
            if not np.array_equal(mine_bits.numpy(), want_bits):
                ok = False
                out_q.put((rank, f"estimator {cols}", "OR-merged bitmap differs from the whole-table bitmap"))
        out_q.put((rank, "done", ok))
    finally:
        dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.timeout(120)
def test_allreduce_merge_equals_host_reduce_world2():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    msgs = []
    for p in procs:
        p.join(100)
    while not q.empty():
        msgs.append(q.get())
    for p in procs:
        assert p.exitcode == 0, msgs
    done = [m for m in msgs if m[1] == "done"]
    assert len(done) == world and all(m[2] for m in done), msgs
