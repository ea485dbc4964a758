"""The cross-device merge of partial aggregate tables against the exact references, computed over the WHOLE table.

A multi-device query scans each device's fragments into a partial table and merges the partials (DESIGN.md section 5):
dense tables are position-aligned on every device and start at the identity of their reduction, so the merge is one
all-reduce per reduction class (integer SUM, double SUM, MIN, MAX, touched flags, bitmap OR); baseline-hash tables are
all-gathered and re-probed.  Two forms are checked here, on the same matrix of kernels, widths and edge data:

- the split form (always runs, one GPU): b2q_execute_partial once per view, then the caller's own reduction of every array
  b2q_partial_array reports, done here on the host in numpy with the array's reported dtype and redop, copied back into one
  partial and b2q_partial_finalize.  This checks the library's half of that contract (identities, the export of the split
  (lo | hi) words, the redops, finalize) without NCCL.
- the NCCL merge inside the library (b2q_execute_work_unit_multi, one device per view): needs two GPUs or more.  It also runs
  what the split form refuses: baseline hash (re-probe), a merged table that is exactly full or one entry over, and the
  estimator's bitmap.

Integer results are exact (int_exact_ref: SUM mod 2^64, COUNT32, MIN / MAX, pair_to_double AVG, COUNT(DISTINCT) as a set),
and byte-equal on every non-empty entry to one device scanning the whole table.  Floating-point results are checked with
fp_exact_ref's any-order bounds, unchanged: a merge is one more summation tree over the same values, and those bounds hold
for every order and every tree of the n - 1 additions, so the extra additions of a merge are already inside them.  The
split form adds the double partial sums in view order and again in reverse view order.

Nothing here is compared with the oracle.  The (group, target) pairs compared are counted and printed at the end of the
module (pytest -s); none is left out."""
import ctypes as C
import math
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import fp_exact_ref as fx
import gpu_util as gu
import int_exact_ref as ix
import sqlmini
from heavydb_b200 import abi, executor, multigpu
from test_fp_exact_ref import SPECIAL_SQL, check_special_rows
from test_gpu_fp_exact import check_rows as fp_check_rows
from test_gpu_int_exact import GPU_WIDTHS, expected_order, extreme_groups, no_distinct
from test_int_exact_ref import aggs_of, check_rows as int_check_rows

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not gu.has_gpu(), reason="needs a CUDA device")]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KS = (2, 3, 8)
ROWS = 1 << 15
FRAG_SIZES = (5000, 1, 3000, 777, 4096, 2)          # fragments of unequal sizes, cycled
INT_CASES = [(w, d) for w in GPU_WIDTHS for d in ix.dataset_names(ix.WIDTH[w])]
COMPARED = {"pairs": 0}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print(f"\nmulti-device exact: {COMPARED['pairs']} (group, target) pairs compared, 0 left out")


def device_count():
    return executor.lib().b2q_device_count() if gu.has_gpu() else 0


def nccl_devices():
    return min(device_count(), 8)


# ---- tables and placement ------------------------------------------------------------------------------------------------
def cut(table, cols, sizes=FRAG_SIZES):
    """Append the rows of `cols` to `table` in fragments whose sizes cycle through `sizes`."""
    n, b, i = len(cols[0]), 0, 0
    while b < n:
        s = sizes[i % len(sizes)]
        table.add_host_fragment([c[b:b + s] for c in cols])
        b, i = b + s, i + 1
    return table


class Views:
    """K views of one table: view r holds the fragments with fragment_id % K == r as its own (in the HBM of devices[r], or
    host-resident) and every other fragment as chunk stats only, so that every view plans on the whole table's stats."""

    def __init__(self, table, k, devices=None, level=abi.GPU_LEVEL):
        import torch
        devices = list(devices) if devices is not None else [0] * k
        self.tables, self.keep, self.level = [], [], level
        for r in range(k):
            v = abi.Table(table.col_types, encoded_sizes=table.encoded_sizes, deleted_column=table.deleted_column,
                          col_scales=table.col_scales)
            for f in table.fragments:
                if f.fragment_id % k != r:
                    v.add_remote_fragment(f.num_tuples, f.stats, f.fragment_id)
                elif level == abi.CPU_LEVEL:
                    v.fragments.append(f)
                else:
                    ptrs = []
                    for a in f.host_cols:
                        if a is None or a.size == 0:
                            ptrs.append(0)
                            continue
                        t = torch.from_numpy(a.view(np.uint8).copy()).cuda(devices[r])
                        self.keep.append(t)
                        ptrs.append(t.data_ptr())
                    v.add_device_fragment(f.num_tuples, ptrs, f.stats, fragment_id=f.fragment_id, device_id=devices[r])
            self.tables.append(v)
        for d in set(devices):
            torch.cuda.synchronize(d)


def plan_fields(x):
    """A plan (or a field of one) as plain Python values, every field but the padding."""
    if isinstance(x, C.Structure):
        return {name: plan_fields(getattr(x, name)) for name, *_ in x._fields_ if not name.endswith("_")}
    if isinstance(x, C.Array):
        return [plan_fields(e) for e in x]
    return x


def assert_same_plan(got, want):
    g, w = plan_fields(got), plan_fields(want)
    diff = {k: (g[k], w[k]) for k in w if g[k] != w[k]}
    assert not diff, f"partial plan differs from the whole-table plan: {diff}"


# ---- the two merge forms ---------------------------------------------------------------------------------------------------
_TYPESTR = {abi.DT_FLOAT64: "<f8", abi.DT_INT64: "<i8", abi.DT_UINT8: "|u1"}
# (dtype, redop) of every array kind b2q.h documents: COUNT / integer SUM, double SUM, MIN, MAX (doubles travel as
# order-preserving int64), "group touched" flags merged with MAX, bitmaps merged with OR
ARRAY_KINDS = {(abi.DT_INT64, abi.RED_SUM), (abi.DT_FLOAT64, abi.RED_SUM), (abi.DT_INT64, abi.RED_MIN), (abi.DT_INT64, abi.RED_MAX),
               (abi.DT_UINT8, abi.RED_MAX), (abi.DT_UINT8, abi.RED_BOR)}


def host_reduce(parts, dtype, redop):
    """What an outside caller's collective does to one array, in numpy: int64 SUM as uint64 (mod 2^64), f64 SUM in the order
    given, MIN / MAX, byte-wise OR."""
    if redop == abi.RED_BOR:
        return np.bitwise_or.reduce(np.stack(parts), axis=0)
    if redop == abi.RED_MIN:
        return np.minimum.reduce(np.stack(parts), axis=0)
    if redop == abi.RED_MAX:
        return np.maximum.reduce(np.stack(parts), axis=0)
    assert redop == abi.RED_SUM, redop
    if dtype == abi.DT_INT64:
        acc = parts[0].view(np.uint64).copy()
        for p in parts[1:]:
            acc += p.view(np.uint64)
        return acc.view(np.int64)
    assert dtype == abi.DT_FLOAT64, dtype
    acc = parts[0].copy()
    for p in parts[1:]:
        acc = acc + p
    return acc


def run_split(unit, table, views, guess=0, has_card=False, force_kernel=0):
    """Split form on the views' devices: one partial per view, plans checked against the whole table's, the arrays merged
    on the host into partial 0 (view order) and, when a double SUM is among them, into the last partial (reverse view
    order).  Returns the finalized result sets."""
    import torch
    ex = executor.Executor()
    eo = executor.execution_options(force_kernel=force_kernel)
    want_plan = ex.plan(unit, table, eo=eo, max_groups_buffer_entry_guess=guess, has_cardinality_estimation=has_card)
    parts = [ex.executePartial(guess, True, v, unit, eo=eo, has_cardinality_estimation=has_card, memory_level=views.level)
             for v in views.tables]
    for p in parts:
        assert_same_plan(p.plan(), want_plan)
        assert p.is_mergeable()
    arrays = [p.arrays() for p in parts]
    dev = f"cuda:{torch.cuda.current_device()}"

    def tensor(a):
        ptr, n, dt, _op = a
        return torch.as_tensor(multigpu.CudaArray(ptr, n, _TYPESTR[dt]), device=dev)
    shapes = [(n, dt, op) for _p, n, dt, op in arrays[0]]
    assert all([(n, dt, op) for _p, n, dt, op in a] == shapes for a in arrays)
    assert {(dt, op) for _n, dt, op in shapes} <= ARRAY_KINDS, shapes
    host = [[tensor(a).cpu().numpy().copy() for a in arr] for arr in arrays]
    runs = [(0, list(range(len(parts))))]
    if any(dt == abi.DT_FLOAT64 for _n, dt, _op in shapes):
        runs.append((len(parts) - 1, list(range(len(parts)))[::-1]))
    out = []
    for into, order in runs:
        for i, (_n, dt, op) in enumerate(shapes):
            merged = host_reduce([host[r][i] for r in order], dt, op)
            tensor(arrays[into][i]).copy_(torch.from_numpy(np.ascontiguousarray(merged)))
        torch.cuda.synchronize()
        out.append(parts[into].finalize())
    return out


_COMMS = {}


def comms():
    """One communicator per device 0..ndev-1, made once per process (NCCL communicators are costly to build)."""
    ndev = nccl_devices()
    if ndev < 2:
        pytest.skip(f"the NCCL merge needs 2 GPUs or more; this machine has {device_count()}")
    if "c" not in _COMMS:
        _COMMS["c"] = executor.Comm.init_all(list(range(ndev)))
    return _COMMS["c"]


@pytest.fixture(scope="module", autouse=True)
def _destroy_comms():
    yield
    for c in _COMMS.pop("c", []):
        c.destroy()


def run_nccl(unit, table, views, guess=0, has_card=False, force_kernel=0):
    ex = executor.Executor()
    eo = executor.execution_options(force_kernel=force_kernel)
    rs = executor.execute_work_unit_multi(comms(), ex, guess, True, views.tables, unit, eo=eo, has_cardinality_estimation=has_card,
                                          memory_level=views.level)
    assert_same_plan_parity(rs.getQueryMemDesc(), ex.plan(unit, table, eo=eo, max_groups_buffer_entry_guess=guess,
                                                          has_cardinality_estimation=has_card), unit)
    return [rs]


def assert_same_plan_parity(got, want, unit):
    g, w = plan_fields(got), plan_fields(want)
    if unit.unit.num_order_entries or unit.unit.has_limit:      # the sorted result holds the LIMIT / OFFSET window only
        for k in ("entry_count", "buffer_size"):
            g.pop(k), w.pop(k)
    assert g == w


class Form:
    """`split`: K views in {2, 3, 8} on device 0; `nccl`: one view per device."""

    def __init__(self, name):
        self.name = name

    def ks(self):
        if self.name == "split":
            return KS
        comms()
        return (nccl_devices(),)

    def views(self, table, k, level=abi.GPU_LEVEL):
        return Views(table, k, devices=None if self.name == "split" else range(k), level=level)

    def run(self, unit, table, views, **kw):
        return (run_split if self.name == "split" else run_nccl)(unit, table, views, **kw)


FORMS = ["split", "nccl"]


def whole_table(unit, table, dev, guess=0, has_card=False, force_kernel=0):
    eo = executor.execution_options(force_kernel=force_kernel)
    return executor.Executor().executeWorkUnit(guess, True, dev.table, unit, eo=eo, has_cardinality_estimation=has_card,
                                               memory_level=abi.GPU_LEVEL)


def same_bytes(rs, ref):
    """Integer targets: the merged storage equals one device's over the whole table on every non-empty entry, and the
    same entries are empty."""
    plan = rs.getQueryMemDesc()
    n = rs.entryCount()
    assert n == ref.entryCount()
    empty = np.array([rs.isRowAtEmpty(i) for i in range(n)], dtype=bool)
    assert np.array_equal(empty, np.array([ref.isRowAtEmpty(i) for i in range(n)], dtype=bool))
    gu.buffers_equal(rs.getStorageBuffer(), ref.getStorageBuffer(), plan, fp_rtol=0.0, empty=empty)


def count_pairs(rows, plan):
    COMPARED["pairs"] += len(rows) * sum(1 for t in plan.targets[: plan.num_targets] if t.is_agg)


def int_exact(rs, groups, w, kernel, ref=None):
    plan = rs.getQueryMemDesc()
    assert plan.kernel == kernel
    rows = rs.rows(decimal_to_double=False)
    bad, skipped = int_check_rows(rows, plan, groups, w, device=True)
    assert not bad and not skipped, bad[:6]
    count_pairs(rows, plan)
    if ref is not None:
        same_bytes(rs, ref)


def fp_exact(rs, groups, kernel):
    plan = rs.getQueryMemDesc()
    assert plan.kernel == kernel
    rows = rs.rows()
    fp_check_rows(rows, plan, groups)
    count_pairs(rows, plan)


# ---- integer widths and datasets ---------------------------------------------------------------------------------------------
def int_table(w, dataset, nullable):
    keys, phys = ix.make_dataset(w, dataset, ROWS, nullable)
    return cut(w.table(notnull=not nullable), [keys, phys]), keys, phys


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("width,dataset", INT_CASES)
def test_integer_widths(form, width, dataset, nullable):
    """Non-grouped, perfect hash in shared memory (keyless, the COUNT(*) slot as the empty marker; COUNT(DISTINCT) bitmaps
    OR-ed where the width has them) and the HBM table in the split layout."""
    form = Form(form)
    w = ix.WIDTH[width]
    t, keys, phys = int_table(w, dataset, nullable)
    dev = gu.DeviceTable(t)
    drop_lo = ("cmp", "<>", w.logical(w.lo))
    m = ix.passing(w, phys, nullable, drop_lo)
    where = ix.predicate_sql(w, drop_lo)
    runs = [(f"SELECT {no_distinct(w)} FROM t WHERE {where};", None, 0, abi.KERNEL_NON_GROUPED),
            (f"SELECT k, {aggs_of(w)} FROM t WHERE {where} GROUP BY k;", keys, 0, abi.KERNEL_PERFECT_SMEM),
            (f"SELECT k, {no_distinct(w)} FROM t WHERE {where} GROUP BY k;", keys, abi.KERNEL_PERFECT_GLOBAL, abi.KERNEL_PERFECT_GLOBAL)]
    for sql, ks, force, kernel in runs:
        unit = sqlmini.parse(sql, t, ["k", "v"])
        groups = ix.groups_of(w, ks, phys, nullable, mask=m)
        ref = whole_table(unit, t, dev, force_kernel=force)
        if ks is not None:
            assert ref.getQueryMemDesc().keyless_hash == 1
        for k in form.ks():
            for rs in form.run(unit, t, form.views(t, k), force_kernel=force):
                int_exact(rs, groups, w, kernel, ref)


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("width,dataset", [("INT64", "wrap_to_zero"), ("INT64", "cancelling"), ("DECIMAL18_2", "wrap_to_zero"),
                                           ("INT16", "cancelling")])
def test_touched_flag_and_avg_marker(form, width, dataset):
    """Keyed perfect hash (a touched flag per entry, merged with MAX) where a group's SUM is 0 mod 2^64, and keyless perfect
    hash whose empty marker is AVG's count slot."""
    form = Form(form)
    w = ix.WIDTH[width]
    for nullable, sql, keyless in [(False, "SELECT k, SUM(v) FROM t GROUP BY k;", False),
                                   (True, "SELECT k, MIN(v), MAX(v), SUM(v), COUNT(v) FROM t GROUP BY k;", False),
                                   (False, "SELECT k, AVG(v), SUM(v), MIN(v), MAX(v) FROM t GROUP BY k;", True)]:
        t, keys, phys = int_table(w, dataset, nullable)
        dev = gu.DeviceTable(t)
        unit = sqlmini.parse(sql, t, ["k", "v"])
        groups = ix.groups_of(w, keys, phys, nullable)
        for force, kernel in [(0, abi.KERNEL_PERFECT_SMEM), (abi.KERNEL_PERFECT_GLOBAL, abi.KERNEL_PERFECT_GLOBAL)]:
            ref = whole_table(unit, t, dev, force_kernel=force)
            p = ref.getQueryMemDesc()
            assert p.keyless_hash == int(keyless), sql
            if keyless:
                assert p.idx_target_as_key == p.targets[1].first_slot + 1         # AVG's count slot
            for k in form.ks():
                for rs in form.run(unit, t, form.views(t, k), force_kernel=force):
                    int_exact(rs, groups, w, kernel, ref)


# ---- cases only a merge creates: integers ---------------------------------------------------------------------------------------
I64_MAX, I64_MIN = ix.INT64_MAX, ix.INT64_MIN
NULL = None


def merge_edge_groups(k):
    """key -> {rank: values}: per-rank SUMs that wrap while the total does not (0) and the reverse (1), a group on the last
    rank only (2), NULL only on rank 0 and values on rank 1 (3), MIN = MAX = INT64_MAX, the MIN identity (4), values next to
    the MAX identity (5), carries on every rank (7); keys 10.. fill every rank."""
    g = {0: {0: [I64_MAX, 5], 1: [-I64_MAX, -10]},
         1: {0: [I64_MAX], 1: [2]},
         2: {k - 1: [7, 8]},
         3: {0: [NULL, NULL], 1: [3, -4]},
         4: {0: [I64_MAX, I64_MAX], 1: [I64_MAX]},
         5: {1: [I64_MIN + 1], 0: [I64_MIN + 1, I64_MIN + 1]},
         7: {0: [2 ** 32 - 1] * 3, 1: [2 ** 32 - 1] * 2}}
    rng = np.random.default_rng(k)
    pool = ix.pool(ix.WIDTH["INT64"])
    for key in range(10, 30):
        g[key] = {r: [pool[i] for i in rng.integers(0, len(pool), 5)] + ([NULL] if key % 3 == 0 else []) for r in range(k)}
    return g


def rank_table(groups_by_rank, k, sql_type, notnull, null, dtype, sentinel_group=None):
    """Fragment r (and r + k, the rank's second, one-row fragment) hold rank r's rows.  NULL becomes `null`."""
    t = abi.Table([(abi.kINT, True), (sql_type, notnull)])
    rows = {r: [] for r in range(k)}
    for key, per_rank in groups_by_rank.items():
        for r, vals in per_rank.items():
            rows[r] += [(key, null if v is None else v) for v in vals]
    if sentinel_group is not None:
        rows[0].append(sentinel_group)
    all_k, all_v = [], []
    for r in range(k):
        ks = np.array([a for a, _ in rows[r]], np.int32)
        vs = np.array([b for _, b in rows[r]], dtype)
        if ks.size > 1:
            t.add_host_fragment([ks[:-1], vs[:-1]], fragment_id=r)
            t.add_host_fragment([ks[-1:], vs[-1:]], fragment_id=r + k)
        elif ks.size:
            t.add_host_fragment([ks, vs], fragment_id=r)
        all_k.append(ks)
        all_v.append(vs)
    return t, np.concatenate(all_k), np.concatenate(all_v)


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("nullable", [True, False])
def test_integer_cases_only_a_merge_creates(form, nullable):
    """NOT NULL also holds a group whose only value is INT64_MIN, the MAX identity: it is BIGINT's NULL sentinel, which
    MIN / MAX / SUM read back as NULL (b2q_read_target, as the reference does) however the partials combine."""
    form = Form(form)
    w = ix.WIDTH["INT64"]
    aggs = "COUNT(*), COUNT(v), SUM(v), MIN(v), MAX(v), AVG(v)"
    for k in form.ks():
        spec = merge_edge_groups(k)
        if not nullable:
            spec = {key: {r: [1 if v is None else v for v in vals] for r, vals in pr.items()} for key, pr in spec.items()}
        t, keys, phys = rank_table(spec, k, abi.kBIGINT, not nullable, w.null, np.int64,
                                   sentinel_group=None if nullable else (6, I64_MIN))
        dev = gu.DeviceTable(t)
        views = form.views(t, k)
        sentinel = keys == 6
        for sql, grouped, force, kernel in [(f"SELECT k, {aggs} FROM t GROUP BY k;", True, 0, abi.KERNEL_PERFECT_SMEM),
                                            (f"SELECT k, {aggs} FROM t GROUP BY k;", True, abi.KERNEL_PERFECT_GLOBAL, abi.KERNEL_PERFECT_GLOBAL),
                                            (f"SELECT {aggs} FROM t WHERE k <> 6;", False, 0, abi.KERNEL_NON_GROUPED)]:
            unit = sqlmini.parse(sql, t, ["k", "v"])
            ref = whole_table(unit, t, dev, force_kernel=force)
            groups = ix.groups_of(w, keys[~sentinel] if grouped else None, phys[~sentinel], nullable)
            if grouped:
                assert (groups[0].sum, groups[1].sum) == (-5, I64_MIN + 1)
            for rs in form.run(unit, t, views, force_kernel=force):
                rows = rs.rows(decimal_to_double=False)
                if not nullable and grouped:
                    assert [r for r in rows if r[0] == 6] == [(6, 1, 1, None, None, None, float(I64_MIN))]
                    rows = [r for r in rows if r[0] != 6]
                plan = rs.getQueryMemDesc()
                assert plan.kernel == kernel
                bad, skipped = int_check_rows(rows, plan, groups, w, device=True)
                assert not bad and not skipped, bad[:6]
                count_pairs(rows, plan)
                same_bytes(rs, ref)


# ---- placement edges ----------------------------------------------------------------------------------------------------------
def placement_table(k, seed=0):
    """t(k INT, v BIGINT, d DOUBLE, f INT, del BOOLEAN) with $deleted$ = del.  Rank 0 holds three fragments of 9000, 1 and 4097
    rows; the other ranks take, in turn, a fragment that the simple qual `k < 1000` skips on its chunk stats, one whose rows
    all fail `(f > 0 OR f < 0)`, one that is fully deleted, and nothing (K = 8 is more ranks than fragments)."""
    rng = np.random.default_rng(seed)
    t = abi.Table([(abi.kINT, True), (abi.kBIGINT, False), (abi.kDOUBLE, False), (abi.kINT, True), (abi.kBOOLEAN, True)], deleted_column=4)
    pool = np.array(ix.pool(ix.WIDTH["INT64"]), np.int64)
    cols = []

    def frag(fid, n, role):
        kk = rng.integers(0, 40, n).astype(np.int32)
        v = pool[rng.integers(0, pool.size, n)]
        v[rng.random(n) < 0.1] = abi.NULL_BIGINT
        d = (1.0 + rng.random(n)) * 2.0 ** 20
        d[rng.random(n) < 0.1] = abi.NULL_DOUBLE
        f = rng.integers(0, 10, n).astype(np.int32)
        dl = (rng.random(n) < 0.2).astype(np.int8)
        if role == "skipped":
            kk += 1000
        elif role == "filtered":
            f[:] = 0
        elif role == "deleted":
            dl[:] = 1
        t.add_host_fragment([kk, v, d, f, dl], fragment_id=fid)
        cols.append((kk, v, d, f, dl))
    for i, n in enumerate((9000, 1, 4097)):
        frag(i * k, n, "normal")
    roles = ["skipped", "filtered", "deleted"]
    for r in range(1, min(k, 4)):
        frag(r, 3000, roles[r - 1])
    kk, v, d, f, dl = (np.concatenate(c) for c in zip(*cols))
    return t, kk, v, d, (kk < 1000) & (f != 0) & (dl == 0)


@pytest.mark.parametrize("form", FORMS)
def test_placement_edges(form):
    form = Form(form)
    w = ix.WIDTH["INT64"]
    for k in form.ks():
        t, keys, v, d, m = placement_table(k)
        dev = gu.DeviceTable(t)
        views = form.views(t, k)
        where = "WHERE k < 1000 AND (f > 0 OR f < 0)"
        names = ["k", "v", "d", "f", "del"]
        for sql, ks, kernel in [(f"SELECT k, COUNT(*), COUNT(v), SUM(v), MIN(v), MAX(v), AVG(v) FROM t {where} GROUP BY k;", keys, abi.KERNEL_PERFECT_SMEM),
                                (f"SELECT COUNT(*), COUNT(v), SUM(v), MIN(v), MAX(v), AVG(v) FROM t {where};", None, abi.KERNEL_NON_GROUPED)]:
            unit = sqlmini.parse(sql, t, names)
            ref = whole_table(unit, t, dev)
            if k >= 4:
                assert ref.stats()["fragments_skipped"] >= 2       # the skipped and the fully deleted fragment
            groups = ix.groups_of(w, ks, v, True, mask=m)
            for rs in form.run(unit, t, views):
                int_exact(rs, groups, w, kernel, ref)
        for sql, ks, kernel in [(f"SELECT k, SUM(d), AVG(d), MIN(d), MAX(d), COUNT(d), COUNT(*) FROM t {where} GROUP BY k;", keys, abi.KERNEL_PERFECT_SMEM),
                                (f"SELECT SUM(d), AVG(d), MIN(d), MAX(d), COUNT(d), COUNT(*) FROM t {where};", None, abi.KERNEL_NON_GROUPED)]:
            unit = sqlmini.parse(sql, t, names)
            groups = fx.groups_of(ks, d, null=abi.NULL_DOUBLE, mask=m)
            for rs in form.run(unit, t, views):
                fp_exact(rs, groups, kernel)


# ---- floating point -------------------------------------------------------------------------------------------------------------
FP_AGGS = "SUM(v), AVG(v), MIN(v), MAX(v), COUNT(v), COUNT(*)"


def fp_table(name, nullable, seed=0):
    keys, vals = fx.make_dataset(name, seed)
    ty = abi.kFLOAT if fx.DATASETS[name][3] == "FLOAT" else abi.kDOUBLE
    rng = np.random.default_rng(seed + 100)
    if nullable:
        vals = vals.copy()
        vals[rng.random(vals.size) < 0.05] = abi.NULL_OF[ty]
    filt = rng.integers(0, 1000, keys.size).astype(np.int32)
    t = abi.Table([(abi.kINT, True), (ty, not nullable), (abi.kINT, True)])
    step = keys.size // 8
    cut(t, [keys, vals, filt], sizes=(step + 1, step // 3, step * 2 - 5, 7))
    return t, keys, vals, filt, ty


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("name", sorted(fx.DATASETS))
def test_floating_point_datasets(form, name, nullable):
    form = Form(form)
    t, keys, vals, filt, ty = fp_table(name, nullable)
    null = abi.NULL_OF[ty] if nullable else None
    runs = [(f"SELECT {FP_AGGS} FROM t WHERE f < 700;", None, filt < 700, 0, abi.KERNEL_NON_GROUPED),
            (f"SELECT k, {FP_AGGS} FROM t WHERE f < 900 GROUP BY k;", keys, filt < 900, 0, abi.KERNEL_PERFECT_SMEM),
            (f"SELECT k, {FP_AGGS} FROM t WHERE f < 900 GROUP BY k;", keys, filt < 900, abi.KERNEL_PERFECT_GLOBAL, abi.KERNEL_PERFECT_GLOBAL)]
    if not nullable:
        runs.append(("SELECT k, SUM(v), COUNT(*) FROM t GROUP BY k;", keys, None, 0, abi.KERNEL_PERFECT_SMEM))   # fused
    for k in form.ks():
        views = form.views(t, k)
        for sql, ks, mask, force, kernel in runs:
            unit = sqlmini.parse(sql, t, ["k", "v", "f"])
            groups = fx.groups_of(ks, vals, null=null, mask=mask)
            for rs in form.run(unit, t, views, force_kernel=force):
                fp_exact(rs, groups, kernel)


NAN, INF = math.nan, math.inf


def fp_merge_groups(k, sql_type):
    """key -> {rank: values}: -0.0 on one rank and +0.0 on another (20, 21); a partial of only NaN on a rank other than the
    one holding numbers (22, 23); +inf / -inf as a real MAX / MIN (24, 25); per-rank sums that are finite while their total
    overflows (26); +inf and -inf on two ranks (27); NULL only on rank 0 (28); a group on the last rank only (29); FLOAT:
    a sum that narrowed per rank would round differently (30: 2^24 + 1 on rank 0 narrows to 2^24, but the merged double
    2^24 + 2 is a float)."""
    big = 3e38 if sql_type == abi.kFLOAT else 1e308
    null = fx.NULL_FLOAT if sql_type == abi.kFLOAT else fx.NULL_DOUBLE
    g = {20: {0: [-0.0], 1: [0.0]},
         21: {0: [0.0], 1: [-0.0, -0.0]},
         22: {0: [NAN, NAN], 1: [4.0, 2.0]},
         23: {1: [NAN], 0: [-3.0]},
         24: {0: [INF], 1: [1.0]},
         25: {0: [-INF], 1: [7.0]},
         26: {0: [big], 1: [big]},
         27: {0: [INF], 1: [-INF]},
         28: {0: [null, null], 1: [2.5]},
         29: {k - 1: [0.75, -0.25]}}
    if sql_type == abi.kFLOAT:
        g[30] = {0: [2.0 ** 24, 1.0], 1: [1.0]}
    rng = np.random.default_rng(k)
    for key in range(40, 56):
        g[key] = {r: list(rng.integers(-40, 40, 6) * 0.25) for r in range(k)}
    return g


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("sql_type", [abi.kDOUBLE, abi.kFLOAT])
def test_floating_point_cases_only_a_merge_creates(form, sql_type, nullable):
    """fp_exact_ref's special-value rules after the merge.  Where the reference's MIN / MAX depend on which value arrives
    first (a NaN before a number, group 22 in view order), the device must follow its own rule: NaN loses to every number."""
    form = Form(form)
    null = fx.NULL_FLOAT if sql_type == abi.kFLOAT else fx.NULL_DOUBLE
    dt = abi.NUMPY_OF[sql_type]
    for k in form.ks():
        spec = fp_merge_groups(k, sql_type)
        if not nullable:
            spec = {key: {r: [1.0 if v == null else v for v in vals] for r, vals in pr.items()} for key, pr in spec.items()}
        t, keys, vals = rank_table(spec, k, sql_type, not nullable, null, dt)
        views = form.views(t, k)
        unit = sqlmini.parse(SPECIAL_SQL, t, ["k", "v"])
        for force, kernel in [(0, abi.KERNEL_PERFECT_SMEM), (abi.KERNEL_PERFECT_GLOBAL, abi.KERNEL_PERFECT_GLOBAL)]:
            for rs in form.run(unit, t, views, force_kernel=force):
                assert rs.getQueryMemDesc().kernel == kernel
                rows = rs.rows()
                assert check_special_rows(rows, keys, vals, sql_type, nullable) == []
                count_pairs(rows, rs.getQueryMemDesc())
                by = {r[0]: r for r in rows}
                assert by[22][2:4] == (2.0, 4.0) and by[23][2:4] == (-3.0, -3.0)      # NaN loses to every number
                assert by[24][3] == INF and by[25][2] == -INF and by[26][1] == INF and math.isnan(by[27][1])
                if sql_type == abi.kFLOAT:
                    assert by[30][1] == 2.0 ** 24 + 2                              # narrowed once, after the merge


# ---- joins, composite keys, host-resident views ------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("how", ["JOIN", "LEFT JOIN"])
def test_join_inner_table_on_every_device(form, how):
    """The fact table is placed; the inner table travels whole with the unit (the library builds its join table on every
    device, as tools/multigpu_check.py does)."""
    form = Form(form)
    w = ix.WIDTH["INT64"]
    rng = np.random.default_rng(21)
    dim_rows, n = 1000, 300_000
    dim_id = rng.permutation(dim_rows).astype(np.int32)
    p = np.array(ix.pool(w), dtype=np.int64)
    dw = p[rng.integers(0, p.size, dim_rows)]
    dw[rng.random(dim_rows) < 0.1] = w.null
    dim = abi.Table([(abi.kINT, True), (abi.kBIGINT, False)])
    dim.add_host_fragment([dim_id, dw])
    fk = rng.integers(-5, dim_rows + 60, n).astype(np.int32)
    x = rng.integers(0, 10, n).astype(np.int32)
    fact = cut(abi.Table([(abi.kINT, True), (abi.kINT, True)]), [fk, x], sizes=(40_000, 3, 25_000))
    unit = sqlmini.parse(f"SELECT t.x, COUNT(*), COUNT(d.w), SUM(d.w), MIN(d.w), MAX(d.w), AVG(d.w) FROM t {how} d ON t.fk = d.id "
                         "GROUP BY t.x;", fact, ["fk", "x"], inner=(dim, ["id", "w"]))
    row_of = np.full(dim_rows + 100, -1, np.int64)
    row_of[dim_id] = np.arange(dim_rows)
    hit = (fk >= 0) & (fk < dim_rows)
    r = np.where(hit, row_of[np.clip(fk, 0, dim_rows + 99)], -1)
    joined = np.where(r >= 0, dw[np.maximum(r, 0)], w.null)
    groups = ix.groups_of(w, x, joined, True, mask=None if how == "LEFT JOIN" else r >= 0)
    ref = whole_table(unit, fact, gu.DeviceTable(fact))
    for k in form.ks():
        for level in (abi.GPU_LEVEL, abi.CPU_LEVEL):
            for rs in form.run(unit, fact, form.views(fact, k, level)):
                int_exact(rs, groups, w, abi.KERNEL_PERFECT_SMEM, ref)


@pytest.mark.parametrize("form", FORMS)
def test_composite_keys(form):
    form = Form(form)
    rng = np.random.default_rng(4)
    n = 100_000
    a = rng.choice(np.array([-127, -126, 0, 126, 127], np.int8), n)
    b = rng.choice(np.array([-32767, -32766, -32700], np.int16), n)
    v = np.full(n, 2 ** 32 - 1, np.int64)
    v[rng.random(n) < 0.5] = ix.INT64_MAX
    t = cut(abi.Table([(abi.kTINYINT, True), (abi.kSMALLINT, True), (abi.kBIGINT, True)]), [a, b, v])
    unit = sqlmini.parse("SELECT a, b, COUNT(*), SUM(v), MIN(v), MAX(v) FROM t GROUP BY a, b;", t, ["a", "b", "v"])
    want = {}
    for x, y, z in zip(a.tolist(), b.tolist(), v.tolist()):
        want.setdefault((x, y), []).append(z)
    want = {kk: (len(z), ix.wrap64(sum(z)), min(z), max(z)) for kk, z in want.items()}
    ref = whole_table(unit, t, gu.DeviceTable(t))
    for k in form.ks():
        for rs in form.run(unit, t, form.views(t, k)):
            assert rs.getQueryMemDesc().kernel == abi.KERNEL_PERFECT_GLOBAL         # 255 x 68 entries of four slots
            got = {(r[0], r[1]): tuple(r[2:]) for r in rs.rows()}
            assert got == want
            COMPARED["pairs"] += 4 * len(got)
            same_bytes(rs, ref)


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("case", ["INT64-pool", "INT64-carry_dense", "INT16-wrap_to_zero", "pos12", "f32_pos"])
def test_host_resident_views(form, case):
    """Every view streams its own fragments from host memory (CPU_LEVEL)."""
    form = Form(form)
    if case in fx.DATASETS:
        t, keys, vals, filt, ty = fp_table(case, True)
        unit = sqlmini.parse(f"SELECT k, {FP_AGGS} FROM t WHERE f < 900 GROUP BY k;", t, ["k", "v", "f"])
        groups = fx.groups_of(keys, vals, null=abi.NULL_OF[ty], mask=filt < 900)
        for k in form.ks():
            for rs in form.run(unit, t, form.views(t, k, abi.CPU_LEVEL)):
                fp_exact(rs, groups, abi.KERNEL_PERFECT_SMEM)
        return
    width, dataset = case.split("-")
    w = ix.WIDTH[width]
    t, keys, phys = int_table(w, dataset, True)
    unit = sqlmini.parse(f"SELECT k, {no_distinct(w)} FROM t GROUP BY k;", t, ["k", "v"])
    groups = ix.groups_of(w, keys, phys, True)
    ref = whole_table(unit, t, gu.DeviceTable(t))
    for k in form.ks():
        for rs in form.run(unit, t, form.views(t, k, abi.CPU_LEVEL)):
            int_exact(rs, groups, w, abi.KERNEL_PERFECT_SMEM, ref)


# ---- ORDER BY / LIMIT / OFFSET over merged aggregates ------------------------------------------------------------------------------
@pytest.mark.parametrize("form", FORMS)
def test_order_by_limit_offset_after_the_merge(form):
    form = Form(form)
    w = ix.WIDTH["INT64"]
    keys, v = extreme_groups(1000, seed=7)
    gs = ix.groups_of(w, keys, v, True)
    t = cut(w.table(notnull=False), [keys, v], sizes=(700, 1, 1300))
    exact = [(kk, g.sum, g.min, g.max, g.count) for kk, g in gs.items()]
    for k in form.ks():
        views = form.views(t, k)
        for col, desc, nf, limit, offset in [(2, False, True, 0, 0), (3, True, False, 30, 0), (4, False, False, 25, 7),
                                             (5, True, True, 40, 11), (2, True, False, 12, 990)]:
            lim = (f" LIMIT {limit}" if limit else "") + (f" OFFSET {offset}" if offset else "")
            sql = (f"SELECT k, SUM(v), MIN(v), MAX(v), COUNT(v) FROM t GROUP BY k ORDER BY {col} {'DESC' if desc else 'ASC'} "
                   f"NULLS {'FIRST' if nf else 'LAST'}, 1{lim};")
            unit = sqlmini.parse(sql, t, ["k", "v"])
            want = expected_order(exact, [(col - 1, desc, nf), (0, False, False)])[offset:]
            want = want[:limit] if limit else want
            for rs in form.run(unit, t, views, guess=1001, has_card=True):
                got = rs.rows()
                assert got == want, (sql, got[:4], want[:4])
                COMPARED["pairs"] += 4 * len(got)


# ---- estimator bitmaps --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", FORMS)
def test_estimator_bitmaps(form):
    form = Form(form)
    rng = np.random.default_rng(3)
    n = 200_000
    cols = [rng.integers(0, 50, n).astype(np.int32), rng.integers(-10 ** 12, 10 ** 12, n), rng.integers(0, 3000, n).astype(np.int16)]
    t = cut(abi.Table([(abi.kINT, True), (abi.kBIGINT, True), (abi.kSMALLINT, True)]), cols, sizes=(30_000, 5, 17_000))
    dev = gu.DeviceTable(t)
    for cs in ([0], [1], [0, 2]):
        b = abi.UnitBuilder(t)
        b.estimator(cs)
        unit = b.build()
        want = executor.Executor().executeWorkUnit(1, True, dev.table, unit, memory_level=abi.GPU_LEVEL)
        for k in form.ks():
            for rs in form.run(unit, t, form.views(t, k), guess=1):
                assert np.array_equal(rs.getHostEstimatorBuffer(), want.getHostEstimatorBuffer()), cs
                assert rs.getNDVEstimator() == want.getNDVEstimator()


# ---- the HBM table's plain-word layout ----------------------------------------------------------------------------------------------
def test_plain_word_layout_of_the_hbm_table():
    """B2Q_GLOBAL_SPLIT=0 (read once per process, hence the child): the HBM table's plain int64 words and the touched flag
    derived from them at materialise time, through both merge forms."""
    env = dict(os.environ, B2Q_GLOBAL_SPLIT="0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "tests/test_gpu_multi_exact.py", "-k",
                        "test_integer_widths and (INT64 or DECIMAL18_2 or INT8) or test_touched_flag_and_avg_marker "
                        "or test_integer_cases_only_a_merge_creates"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-1000:]
    assert " passed" in r.stdout


# ---- Part B only: baseline hash, a merged table that is exactly full -----------------------------------------------------------
BASELINE_FRAG = 4000


def baseline_table(k, seed=0):
    """t(k BIGINT nullable, v BIGINT nullable, s SMALLINT, b TINYINT): sparse keys, so baseline hash.  Keys 0.. are on every
    rank, keys 100.. on one rank only (the one of their fragment), plus NULL, INT64_MAX - 1 and INT64_MIN + 1 / + 2 as keys.
    COUNT(DISTINCT b) over [0, 20) is one bitmap word per entry, COUNT(DISTINCT s) over [0, 2000) 63 words."""
    rng = np.random.default_rng(seed)
    pool = np.array(ix.pool(ix.WIDTH["INT64"]), np.int64)
    t = abi.Table([(abi.kBIGINT, False), (abi.kBIGINT, False), (abi.kSMALLINT, True), (abi.kTINYINT, True)])
    edge = np.array([abi.NULL_BIGINT, I64_MAX - 1, I64_MIN + 1, I64_MIN + 2], np.int64)
    cols = []
    n = BASELINE_FRAG
    for fid in range(2 * k):
        common = rng.integers(0, 60, n) * 7919 * 10 ** 9 + 12345
        own = (100 + fid * 50 + rng.integers(0, 50, n)) * 7919 * 10 ** 9
        kk = np.where(rng.random(n) < 0.5, common, own)
        kk[:4] = edge if fid % 2 == 0 else edge[[0, 1, 1, 3]]
        v = pool[rng.integers(0, pool.size, n)]
        v[rng.random(n) < 0.1] = abi.NULL_BIGINT
        s = rng.integers(0, 2000, n).astype(np.int16)
        b = rng.integers(0, 20, n).astype(np.int8)
        t.add_host_fragment([kk, v, s, b], fragment_id=fid)
        cols.append((kk, v, s, b))
    return t, tuple(np.concatenate(c) for c in zip(*cols))


@pytest.mark.parametrize("force", [0, abi.KERNEL_BASELINE_PROBE])
def test_nccl_baseline_hash(force):
    form = Form("nccl")
    w = ix.WIDTH["INT64"]
    k = form.ks()[0]
    t, (keys, v, s, b) = baseline_table(k)
    views = form.views(t, k)
    dev = gu.DeviceTable(t)
    n_keys = len(set(keys.tolist()))
    unit = sqlmini.parse("SELECT k, COUNT(*), COUNT(v), SUM(v), MIN(v), MAX(v), AVG(v) FROM t GROUP BY k;", t, ["k", "v", "s", "b"])
    groups = ix.groups_of(w, keys, v, True)
    groups = {None if kk == abi.NULL_BIGINT else kk: g for kk, g in groups.items()}
    rs = form.run(unit, t, views, guess=2 * n_keys, has_card=True, force_kernel=force)[0]
    int_exact(rs, groups, w, abi.KERNEL_BASELINE_GLOBAL)
    # COUNT(DISTINCT): one bitmap word and 63 words per entry, re-probed across ranks
    unit = sqlmini.parse("SELECT k, COUNT(DISTINCT b), COUNT(DISTINCT s), COUNT(*) FROM t GROUP BY k;", t, ["k", "v", "s", "b"])
    rs = form.run(unit, t, views, guess=2 * n_keys, has_card=True, force_kernel=force)[0]
    assert rs.getQueryMemDesc().kernel == abi.KERNEL_BASELINE_GLOBAL
    want = {}
    for kk, bb, ss in zip(keys.tolist(), b.tolist(), s.tolist()):
        e = want.setdefault(None if kk == abi.NULL_BIGINT else kk, [set(), set(), 0])
        e[0].add(bb)
        e[1].add(ss)
        e[2] += 1
    got = {r[0]: tuple(r[1:]) for r in rs.rows()}
    assert got == {kk: (len(e[0]), len(e[1]), e[2]) for kk, e in want.items()}
    COMPARED["pairs"] += 3 * len(got)
    single = whole_table(unit, t, dev, guess=2 * n_keys, has_card=True, force_kernel=force)
    assert sorted(single.rows(), key=repr) == sorted(rs.rows(), key=repr)


def per_rank_codes(views, unit, guess, force):
    """b2q_execute_work_unit_dist on every rank at once (one host thread each): the error code each rank returns."""
    cs = comms()
    codes = [None] * len(cs)
    eo = executor.execution_options(force_kernel=force)

    def rank(r):
        try:
            executor.execute_work_unit_dist(cs[r], executor.Executor(), guess, True, views.tables[r], unit, eo=eo,
                                            has_cardinality_estimation=True)
            codes[r] = 0
        except executor.QueryExecutionError as e:
            codes[r] = e.code
    ths = [threading.Thread(target=rank, args=(r,)) for r in range(len(cs))]
    for th in ths:
        th.start()
    for th in ths:
        th.join(300)
    assert not any(th.is_alive() for th in ths), "a rank did not return"
    return codes


@pytest.mark.parametrize("force", [0, abi.KERNEL_BASELINE_PROBE])
def test_nccl_merged_baseline_table_exactly_full(force):
    """Keys whose union across ranks is exactly the plan's entry count E: the merge succeeds.  One key more, with every rank's
    own table still fitting: every rank reports OUT_OF_SLOTS (the error word all-reduced after the re-probe) and no result
    is returned."""
    form = Form("nccl")
    k = form.ks()[0]
    guess = 4096
    probe = abi.Table([(abi.kBIGINT, True), (abi.kBIGINT, True)])
    probe.add_host_fragment([np.array([0, 10 ** 15], np.int64), np.array([1, 2], np.int64)])
    unit0 = sqlmini.parse("SELECT k, COUNT(*), SUM(v) FROM t GROUP BY k;", probe, ["k", "v"])
    e = executor.Executor().plan(unit0, probe, max_groups_buffer_entry_guess=guess, has_cardinality_estimation=True).entry_count
    assert e >= k + 1
    for extra in (0, 1):
        n_keys = e + extra
        key_vals = (np.arange(n_keys, dtype=np.int64) * 1_000_003 + 17) * 999_983
        t = abi.Table([(abi.kBIGINT, True), (abi.kBIGINT, True)])
        per = np.array_split(key_vals, k)                                  # rank r's own keys: about E / k of them
        for r in range(k):
            kk = np.repeat(per[r], 3)
            t.add_host_fragment([kk, np.full(kk.size, 2, np.int64)], fragment_id=r)
        unit = sqlmini.parse("SELECT k, COUNT(*), SUM(v) FROM t GROUP BY k;", t, ["k", "v"])
        plan = executor.Executor().plan(unit, t, max_groups_buffer_entry_guess=guess, has_cardinality_estimation=True)
        assert plan.entry_count == e and plan.kernel == abi.KERNEL_BASELINE_GLOBAL
        views = form.views(t, k)
        if extra == 0:
            rs = form.run(unit, t, views, guess=guess, has_card=True, force_kernel=force)[0]
            assert sorted(rs.rows()) == [(int(x), 3, 6) for x in sorted(key_vals)]
            COMPARED["pairs"] += 2 * n_keys
        else:
            with pytest.raises(executor.QueryExecutionError) as ei:
                form.run(unit, t, views, guess=guess, has_card=True, force_kernel=force)
            assert ei.value.code == abi.ERR_OUT_OF_SLOTS
            assert per_rank_codes(views, unit, guess, force) == [abi.ERR_OUT_OF_SLOTS] * k
