"""Integer aggregates, filters, group keys and sort orders of every scan kernel against the exact reference (int_exact_ref):
COUNT / SUM mod 2^64 / MIN / MAX / AVG / COUNT(DISTINCT) bit for bit on edge tables of every physical width (type extremes,
the NULL sentinel's neighbours, 2^31, 2^32 - 1, 2^53 + 1, +-(2^63 - 1)), carry-dense, wrap-to-zero and cancelling data.  The
plan still has to equal the oracle's, and every aggregate query of the kernel-family tests asserts the kernel it ran on.
Nothing is excluded: the device's SUM is the wrapped sum whatever the order of the adds (int_exact_ref, SENTINEL_SUM), and
its 32-bit COUNT(col) is IntGroup.count32.

ORDER BY and ResultSet.sort() are checked against a plain Python sort with the reference comparator's rules: NULLs first or
last, DESC, ties passed on to the next order entry (every order below ends in the unique group key)."""
import os
import subprocess
import sys

import numpy as np
import pytest

import gpu_util as gu
import int_exact_ref as ix
import oracle_lib
import sqlmini
from heavydb_b200 import abi, executor
from test_int_exact_ref import aggs_of, check_rows, edge_table

pytestmark = pytest.mark.gpu

FRAG = 1 << 15
ROWS = 1 << 18
GPU_WIDTHS = ["INT8", "INT16", "INT32", "INT64", "INT_FIXED16", "BIGINT_FIXED8", "BIGINT_FIXED32", "DECIMAL18_2", "DAYS32", "DICT16"]
CASES = [(w, d) for w in GPU_WIDTHS for d in ix.dataset_names(ix.WIDTH[w])]


def execute(unit, table, dev=None, entry_guess=0, has_card=False, force_kernel=0, output_columnar=False, result_on_device=False):
    """The CUDA path; asserts the plan equals the oracle's (the oracle plans only: the values come from int_exact_ref)."""
    eo = executor.execution_options(force_kernel=force_kernel, output_columnar_hint=output_columnar, result_on_device=result_on_device)
    ex = executor.Executor()
    if dev is not None:
        rs = ex.executeWorkUnit(entry_guess, True, dev.table, unit, eo=eo, has_cardinality_estimation=has_card, memory_level=abi.GPU_LEVEL)
    else:
        rs = ex.executeWorkUnit(entry_guess, True, table, unit, eo=eo, has_cardinality_estimation=has_card, memory_level=abi.CPU_LEVEL)
    want = oracle_lib.plan(unit, table, entry_guess=entry_guess, has_card=has_card, output_columnar=output_columnar).as_dict()
    got = rs.getQueryMemDesc().as_dict()
    if unit.unit.num_order_entries or unit.unit.has_limit:      # the sorted result holds the LIMIT / OFFSET window only
        for k in ("entry_count", "buffer_size"):
            got.pop(k), want.pop(k)
    assert got == want
    return rs


def exact(rows, rs, groups, w):
    bad, skipped = check_rows(rows, rs.getQueryMemDesc(), groups, w, device=True)
    assert not bad and not skipped, bad[:6]


def checked(rs, groups, w, kernel):
    assert rs.getQueryMemDesc().kernel == kernel
    exact(rs.rows(decimal_to_double=False), rs, groups, w)


def no_distinct(w):
    return aggs_of(w).replace(", COUNT(DISTINCT v)", "")


# ---- non-grouped (WAGG) and perfect hash: shared-memory general, HBM/L2 split ------------------------------------------------------
@pytest.mark.parametrize("nullable", [True, False])
@pytest.mark.parametrize("width,dataset", CASES)
def test_non_grouped_and_perfect_hash(width, dataset, nullable):
    w = ix.WIDTH[width]
    t, keys, phys = edge_table(w, dataset, nullable, rows=ROWS, frag_rows=FRAG)
    dev = gu.DeviceTable(t)
    aggs = no_distinct(w)
    drop_lo = ("cmp", "<>", w.logical(w.lo))
    m = ix.passing(w, phys, nullable, drop_lo)
    where = ix.predicate_sql(w, drop_lo)
    unit = sqlmini.parse(f"SELECT {aggs} FROM t WHERE {where};", t, ["k", "v"])
    checked(execute(unit, t, dev), ix.groups_of(w, None, phys, nullable, mask=m, frag_rows=FRAG), w, abi.KERNEL_NON_GROUPED)
    unit = sqlmini.parse(f"SELECT k, {aggs} FROM t WHERE {where} GROUP BY k;", t, ["k", "v"])
    groups = ix.groups_of(w, keys, phys, nullable, mask=m, frag_rows=FRAG)
    for force, kernel in [(0, abi.KERNEL_PERFECT_SMEM), (abi.KERNEL_PERFECT_GLOBAL, abi.KERNEL_PERFECT_GLOBAL)]:
        checked(execute(unit, t, dev, force_kernel=force), groups, w, kernel)


@pytest.mark.parametrize("width,dataset", [(w, d) for w, d in CASES if ix.WIDTH[w].summable])
def test_fused_shared_memory_sum_and_count(width, dataset):
    """NOT NULL SUM + COUNT(*): the fused shared-memory path (8-byte and sign-extended 1/2/4-byte arguments), with 8 keys
    (many warp-private replicas) and with 16 384 keys: 8 bytes per entry make one 128 KiB replica, past the 100 KiB at which
    the scan runs one CTA of 1024 threads per SM (scan_config) instead of two of 512."""
    w = ix.WIDTH[width]
    t, keys, phys = edge_table(w, dataset, False, rows=ROWS, frag_rows=FRAG)
    dev = gu.DeviceTable(t)
    for sql, ks in [("SELECT k, SUM(v), COUNT(*) FROM t GROUP BY k;", keys),
                    ("SELECT k, SUM(v), COUNT(*) FROM t WHERE k < 8 GROUP BY k;", None)]:
        unit = sqlmini.parse(sql, t, ["k", "v"])
        groups = ix.groups_of(w, keys, phys, False, mask=None if ks is not None else keys < 8)
        checked(execute(unit, t, dev), groups, w, abi.KERNEL_PERFECT_SMEM)
    wide = (np.arange(keys.size) % 16384).astype(np.int32)             # 16 384 keys, 16 rows each
    tw = w.table(notnull=True)
    for b in range(0, keys.size, FRAG):
        tw.add_host_fragment([wide[b:b + FRAG], phys[b:b + FRAG]])
    unit = sqlmini.parse("SELECT k, SUM(v), COUNT(*) FROM t GROUP BY k;", tw, ["k", "v"])
    groups = ix.groups_of(w, wide, phys, False)
    assert len(groups) == 16384
    checked(execute(unit, tw, gu.DeviceTable(tw)), groups, w, abi.KERNEL_PERFECT_SMEM)


def test_large_key_range_of_the_hbm_table():
    """50 000 keys: too many for shared memory; INT64 edge values into the split (lo | hi) words."""
    w = ix.WIDTH["INT64"]
    _t, _k, phys = edge_table(w, "pool", True, rows=ROWS)
    keys = np.random.default_rng(3).integers(0, 50_000, phys.size).astype(np.int32)
    t = w.table(notnull=False)
    for b in range(0, keys.size, FRAG):
        t.add_host_fragment([keys[b:b + FRAG], phys[b:b + FRAG]])
    unit = sqlmini.parse(f"SELECT k, {no_distinct(w)} FROM t GROUP BY k;", t, ["k", "v"])
    checked(execute(unit, t, gu.DeviceTable(t)), ix.groups_of(w, keys, phys, True, frag_rows=FRAG), w, abi.KERNEL_PERFECT_GLOBAL)


@pytest.mark.parametrize("width", ["INT64", "DECIMAL18_2", "INT16"])
def test_wrap_to_zero_groups_stay_groups(width):
    """SUM as the only accumulator: a group whose values sum to 0 mod 2^64 can only be told from an empty entry by its
    touched flag (in the plain-word layout derived at materialise time from flag | sum != 0)."""
    w = ix.WIDTH[width]
    t, keys, phys = edge_table(w, "wrap_to_zero", False, rows=ROWS, frag_rows=FRAG)
    dev = gu.DeviceTable(t)
    unit = sqlmini.parse("SELECT k, SUM(v) FROM t GROUP BY k;", t, ["k", "v"])
    groups = ix.groups_of(w, keys, phys, False, frag_rows=FRAG)
    assert len(groups) == 64 and all(g.sum == 0 for g in groups.values())
    for force, kernel in [(0, abi.KERNEL_PERFECT_SMEM), (abi.KERNEL_PERFECT_GLOBAL, abi.KERNEL_PERFECT_GLOBAL)]:
        checked(execute(unit, t, dev, force_kernel=force), groups, w, kernel)


def test_plain_word_layout_of_the_hbm_table_kernels():
    """B2Q_GLOBAL_SPLIT=0 (read once per process, hence the child): the touched flag derived at materialise must keep
    wrap-to-zero and cancelling groups, and the plain words must carry."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, B2Q_GLOBAL_SPLIT="0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "tests/test_gpu_int_exact.py", "-k",
                        "test_non_grouped_and_perfect_hash and (INT64 or DECIMAL18_2) or test_large_key_range or test_wrap_to_zero_groups "
                        "or test_count_and_sum_over_more_than_2_32_rows"],
                       cwd=root, env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-1000:]
    assert " passed" in r.stdout


# ---- baseline hash: radix passes and the forced per-row probe ------------------------------------------------------------------------
@pytest.mark.parametrize("width,dataset", [("INT64", "pool"), ("INT64", "carry_dense"), ("INT64", "wrap_to_zero"), ("INT32", "cancelling"),
                                           ("INT8", "pool"), ("DECIMAL18_2", "wrap_to_zero")])
def test_baseline_hash(width, dataset):
    w = ix.WIDTH[width]
    _t, keys, phys = edge_table(w, dataset, True, rows=ROWS)
    sparse = keys.astype(np.int64) * 7919 * 10 ** 9 + 12345
    t = abi.Table([(abi.kBIGINT, True), (w.sql_type, False)], encoded_sizes=[0, w.enc], col_scales={1: w.scale} if w.scale else None)
    for b in range(0, keys.size, FRAG):
        t.add_host_fragment([sparse[b:b + FRAG], phys[b:b + FRAG]])
    dev = gu.DeviceTable(t)
    unit = sqlmini.parse(f"SELECT k, {no_distinct(w)} FROM t GROUP BY k;", t, ["k", "v"])
    groups = ix.groups_of(w, sparse, phys, True, frag_rows=FRAG)
    launches = {}
    for force in (0, abi.KERNEL_BASELINE_PROBE):
        rs = execute(unit, t, dev, entry_guess=2 * len(groups), has_card=True, force_kernel=force)
        launches[force] = rs.stats()["kernel_launches"]
        checked(rs, groups, w, abi.KERNEL_BASELINE_GLOBAL)
    assert launches[0] > launches[abi.KERNEL_BASELINE_PROBE], launches       # radix partition + aggregate passes


# ---- INNER / LEFT join: an edge-valued BIGINT column of the inner table ----------------------------------------------------------------
@pytest.mark.parametrize("how", ["JOIN", "LEFT JOIN"])
def test_join_inner_edge_column(how):
    w = ix.WIDTH["INT64"]
    rng = np.random.default_rng(21)
    dim_rows, n = 1000, 600_000
    dim_id = rng.permutation(dim_rows).astype(np.int32)
    p = np.array(ix.pool(w), dtype=np.int64)
    dw = p[rng.integers(0, p.size, dim_rows)]
    dw[rng.random(dim_rows) < 0.1] = w.null
    dim = abi.Table([(abi.kINT, True), (abi.kBIGINT, False)])
    dim.add_host_fragment([dim_id, dw])
    fk = rng.integers(-5, dim_rows + 60, n).astype(np.int32)
    x = rng.integers(0, 10, n).astype(np.int32)
    fact = abi.Table([(abi.kINT, True), (abi.kINT, True)])
    for b in range(0, n, 200_000):
        fact.add_host_fragment([fk[b:b + 200_000], x[b:b + 200_000]])
    unit = sqlmini.parse(f"SELECT t.x, COUNT(*), COUNT(d.w), SUM(d.w), MIN(d.w), MAX(d.w), AVG(d.w) FROM t {how} d ON t.fk = d.id "
                         "GROUP BY t.x;", fact, ["fk", "x"], inner=(dim, ["id", "w"]))
    row_of = np.full(dim_rows + 100, -1, np.int64)
    row_of[dim_id] = np.arange(dim_rows)
    hit = (fk >= 0) & (fk < dim_rows)
    r = np.where(hit, row_of[np.clip(fk, 0, dim_rows + 99)], -1)
    joined = np.where(r >= 0, dw[np.maximum(r, 0)], w.null)
    groups = ix.groups_of(w, x, joined, True, mask=None if how == "LEFT JOIN" else r >= 0)
    for d in (gu.DeviceTable(fact), None):
        checked(execute(unit, fact, d), groups, w, abi.KERNEL_PERFECT_SMEM)


# ---- host-resident slices, columnar output, device columns ------------------------------------------------------------------------------
def test_host_resident_over_16mi_rows_carries_across_slices():
    """(2^24 + 2^20) INT64 rows streamed from the host in 16 Mi-row slices: carry-dense values (every add carries out of the
    low word) and the pool's extremes; sums computed per (group, value) count in Python ints."""
    w = ix.WIDTH["INT64"]
    n = (1 << 24) + (1 << 20)
    rng = np.random.default_rng(5)
    p = np.array(ix.pool(w) + [2 ** 32 - 1] * 8, dtype=np.int64)       # carry-dense: half of the rows are 2^32 - 1
    idx = rng.integers(0, p.size, n)
    keys = rng.integers(0, 16, n).astype(np.int32)
    phys = p[idx]
    t = w.table(notnull=True)
    for b in range(0, n, 1 << 22):
        t.add_host_fragment([keys[b:b + (1 << 22)], phys[b:b + (1 << 22)]])
    unit = sqlmini.parse("SELECT k, COUNT(*), SUM(v), MIN(v), MAX(v) FROM t GROUP BY k;", t, ["k", "v"])
    rs = execute(unit, t)
    assert rs.getQueryMemDesc().kernel == abi.KERNEL_PERFECT_SMEM
    assert rs.stats()["h2d_bytes"] >= 8 * n
    counts = np.zeros((16, p.size), np.int64)
    np.add.at(counts, (keys, idx), 1)
    for k, cnt, s, mn, mx in rs.rows():
        c = counts[k]
        assert cnt == int(c.sum())
        assert s == ix.wrap64(sum(int(a) * int(v) for a, v in zip(c, p)))
        assert (mn, mx) == (int(p[c > 0].min()), int(p[c > 0].max()))


@pytest.mark.parametrize("width", ["INT64", "INT16", "DECIMAL18_2"])
def test_columnar_output_and_device_columns(width):
    w = ix.WIDTH[width]
    t, keys, phys = edge_table(w, "pool", True, rows=ROWS, frag_rows=FRAG)
    unit = sqlmini.parse(f"SELECT k, {no_distinct(w)} FROM t GROUP BY k;", t, ["k", "v"])
    groups = ix.groups_of(w, keys, phys, True, frag_rows=FRAG)
    rs = execute(unit, t, gu.DeviceTable(t), output_columnar=True, result_on_device=True)
    assert rs.getQueryMemDesc().output_columnar == 1 and rs.getQueryMemDesc().kernel == abi.KERNEL_PERFECT_SMEM
    cols = rs.deviceColumns().to_host()
    rows = []
    for i in range(len(cols[0][2])):
        row = []
        for ty_c, _nn, values, validity, _nulls in cols:
            ok = validity is None or bool(validity[i >> 3] >> (i & 7) & 1)
            row.append(None if not ok else float(values[i]) if ty_c in (abi.kDOUBLE, abi.kFLOAT) else int(values[i]))
        rows.append(tuple(row))
    exact(rows, rs, groups, w)
    exact(rs.rows(decimal_to_double=False), rs, groups, w)
    checked(execute(unit, t), groups, w, abi.KERNEL_PERFECT_SMEM)      # host-resident, row-wise


# ---- projections of edge values, bit for bit ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("width", ["INT8", "INT32", "INT64", "BIGINT_FIXED16", "DICT8", "DAYS16", "DECIMAL18_2"])
def test_projection_of_edge_values(width):
    w = ix.WIDTH[width]
    t, keys, phys = edge_table(w, "pool", True, rows=1 << 16, frag_rows=5000)
    p = ("not", ("in", [w.logical(w.lo), w.logical(w.hi)]))
    unit = sqlmini.parse(f"SELECT k, v FROM t WHERE {ix.predicate_sql(w, p)};", t, ["k", "v"])
    m = ix.passing(w, phys, True, p)
    want = [(int(k), w.logical(int(v))) for k, v in zip(keys[m], phys[m])]
    for d in (gu.DeviceTable(t), None):
        rs = executor.Executor().executeWorkUnit(0, False, d.table if d else t, unit, memory_level=abi.GPU_LEVEL if d else abi.CPU_LEVEL)
        assert rs.getQueryMemDesc().query_desc_type == abi.Projection
        assert rs.rows(decimal_to_double=False) == want


# ---- COUNT(DISTINCT): bitmap ends, negative minima, DATE buckets --------------------------------------------------------------------------
def test_count_distinct_at_the_bitmap_ends():
    rng = np.random.default_rng(9)
    n = 300_000
    keys = rng.integers(0, 32, n).astype(np.int32)
    lo = -(2 ** 31) + 1                                                # the INT minimum above NULL, 1000 bits of bitmap
    v = (lo + rng.integers(0, 1000, n)).astype(np.int32)
    v[keys == 0] = lo                                                  # bm_min only
    v[keys == 1] = lo + 999                                            # bm_min + bits - 1 only
    v[rng.random(n) < 0.05] = abi.NULL_INT
    days = (rng.integers(-400, 400, n) * 86400 + rng.integers(0, 86400, n)).astype(np.int64)   # DATE on both sides of 1970
    t = abi.Table([(abi.kINT, True), (abi.kINT, False), (abi.kDATE, True)])
    for b in range(0, n, FRAG):
        t.add_host_fragment([keys[b:b + FRAG], v[b:b + FRAG], (days[b:b + FRAG] // 86400) * 86400])
    dt = (days // 86400) * 86400
    unit = sqlmini.parse("SELECT k, COUNT(DISTINCT v), COUNT(DISTINCT d), COUNT(v) FROM t GROUP BY k;", t, ["k", "v", "d"])
    dev = gu.DeviceTable(t)
    for d in (dev, None):
        rs = execute(unit, t, d)
        assert rs.getQueryMemDesc().kernel == abi.KERNEL_PERFECT_SMEM
        for k, cd, cdd, cnt in rs.rows():
            m = keys == k
            vals = v[m][v[m] != abi.NULL_INT]
            assert (cd, cdd, cnt) == (len(set(vals.tolist())), len(set(dt[m].tolist())), vals.size), k


# ---- group keys: both ends of the perfect-hash range, 32-bit keys near +-2^31, composite keys -------------------------------------------
@pytest.mark.parametrize("lo", [-(2 ** 31) + 1, 2 ** 31 - 1001, -1])
def test_group_keys_at_the_ends_of_the_range(lo):
    """INT keys in [lo, lo + 999] (INT32_MAX itself is EMPTY_KEY of a 4-byte key slot and never a key here)."""
    rng = np.random.default_rng(lo & 0xFFFF)
    n = 400_000
    k = (lo + rng.integers(0, 1000, n)).astype(np.int32)
    k[:2] = [lo, lo + 999]
    p = np.array(ix.pool(ix.WIDTH["INT64"]), np.int64)
    v = p[rng.integers(0, p.size, n)]
    t = abi.Table([(abi.kINT, True), (abi.kBIGINT, True)])
    for b in range(0, n, FRAG):
        t.add_host_fragment([k[b:b + FRAG], v[b:b + FRAG]])
    w = ix.WIDTH["INT64"]
    unit = sqlmini.parse("SELECT k, COUNT(*), SUM(v), MIN(v), MAX(v) FROM t GROUP BY k;", t, ["k", "v"])
    groups = ix.groups_of(w, k, v, False)
    dev = gu.DeviceTable(t)
    for force, kernel in [(0, abi.KERNEL_PERFECT_SMEM), (abi.KERNEL_PERFECT_GLOBAL, abi.KERNEL_PERFECT_GLOBAL)]:
        checked(execute(unit, t, dev, force_kernel=force), groups, w, kernel)


def test_composite_keys_at_type_extremes():
    rng = np.random.default_rng(4)
    n = 300_000
    a = rng.choice(np.array([-127, -126, 0, 126, 127], np.int8), n)
    b = rng.choice(np.array([-32767, -32766, -32700], np.int16), n)       # a perfect-hash range: 255 x 68 entries
    v = np.full(n, 2 ** 32 - 1, np.int64)
    v[rng.random(n) < 0.5] = ix.INT64_MAX
    t = abi.Table([(abi.kTINYINT, True), (abi.kSMALLINT, True), (abi.kBIGINT, True)])
    for s in range(0, n, FRAG):
        t.add_host_fragment([a[s:s + FRAG], b[s:s + FRAG], v[s:s + FRAG]])
    unit = sqlmini.parse("SELECT a, b, COUNT(*), SUM(v) FROM t GROUP BY a, b;", t, ["a", "b", "v"])
    want = {}
    for x, y, z in zip(a.tolist(), b.tolist(), v.tolist()):
        c, s = want.get((x, y), (0, 0))
        want[(x, y)] = (c + 1, s + z)
    rs = execute(unit, t, gu.DeviceTable(t))
    assert rs.getQueryMemDesc().kernel == abi.KERNEL_PERFECT_SMEM
    got = {(r[0], r[1]): (r[2], r[3]) for r in rs.rows()}
    assert got == {kk: (c, ix.wrap64(s)) for kk, (c, s) in want.items()}


# ---- more than 2^32 device-resident rows: 64-bit COUNT slots and the forced split ---------------------------------------------------------
def test_count_and_sum_over_more_than_2_32_rows():
    """5 x 2^30 TINYINT rows in device memory: COUNT(*) needs 8-byte slots (tuples > UINT32_MAX) and SUM / COUNT exceed 2^32 in
    the non-grouped, shared-memory and HBM-table kernels.  Run again with B2Q_GLOBAL_SPLIT=0 by
    test_plain_word_layout_of_the_hbm_table_kernels, where the HBM table must fall back to the split layout at 2^32 rows
    (split_layout): the touched flag of the plain words is only sound below that.  The layout chosen is not visible through
    the ABI; the exact results are what is checked."""
    import torch
    frag, n_frags = 1 << 30, 5
    need = frag * n_frags + 3 * (frag * 4)
    if torch.cuda.mem_get_info()[0] < need + (4 << 30):
        pytest.skip("not enough free device memory for 5.4e9 TINYINT rows")
    keep, t = [], abi.Table([(abi.kTINYINT, True)])
    for f in range(n_frags):
        col = (torch.arange(frag, dtype=torch.int32, device="cuda") % 4).to(torch.int8)
        keep.append(col)
        st = abi.ChunkStats()
        st.int_min, st.int_max, st.has_nulls = 0, 3, 0
        t.add_device_fragment(frag, [col.data_ptr()], [st])
    torch.cuda.synchronize()
    n = frag * n_frags
    assert n > 2 ** 32
    ex = executor.Executor()
    unit = sqlmini.parse("SELECT COUNT(*), SUM(v), MIN(v), MAX(v) FROM t;", t, ["v"])
    rs = ex.executeWorkUnit(0, True, t, unit, memory_level=abi.GPU_LEVEL)
    assert rs.getQueryMemDesc().kernel == abi.KERNEL_NON_GROUPED
    assert rs.rows() == [(n, n // 4 * 6, 0, 3)]
    unit = sqlmini.parse("SELECT v, COUNT(*), SUM(v) FROM t GROUP BY v;", t, ["v"])
    for force, kernel in [(0, abi.KERNEL_PERFECT_SMEM), (abi.KERNEL_PERFECT_GLOBAL, abi.KERNEL_PERFECT_GLOBAL)]:
        rs = ex.executeWorkUnit(0, True, t, unit, eo=executor.execution_options(force_kernel=force), memory_level=abi.GPU_LEVEL)
        p = rs.getQueryMemDesc()
        assert p.kernel == kernel
        assert p.slot_padded_width[p.targets[1].first_slot] == 8              # COUNT(*) of more than UINT32_MAX tuples
        assert sorted(rs.rows()) == [(x, n // 4, x * (n // 4)) for x in range(4)]
    unit = sqlmini.parse("SELECT v, SUM(v) FROM t GROUP BY v;", t, ["v"])   # the touched flag rides on the SUM
    rs = ex.executeWorkUnit(0, True, t, unit, eo=executor.execution_options(force_kernel=abi.KERNEL_PERFECT_GLOBAL), memory_level=abi.GPU_LEVEL)
    assert rs.getQueryMemDesc().kernel == abi.KERNEL_PERFECT_GLOBAL
    assert sorted(rs.rows()) == [(x, x * (n // 4)) for x in range(4)]
    del keep


# ---- ORDER BY over integer aggregates: a plain Python sort ---------------------------------------------------------------------------------
def expected_order(rows, entries):
    """rows sorted by [(0-based column, desc, nulls_first)]: NULLs first / last, DESC, ties to the next entry."""
    def key(r):
        out = []
        for col, desc, nulls_first in entries:
            v = r[col]
            out.append(((0 if nulls_first else 2) if v is None else 1, 0 if v is None else (-v if desc else v)))
        return out
    return sorted(rows, key=key)


def extreme_groups(groups_n, seed):
    """Values up to 2^53 + 1 in magnitude, NULLs, and four groups at the edges: 0 holds INT64_MAX alone, 1 -INT64_MAX alone,
    2 sums INT64_MAX + 2 to INT64_MIN + 1 (the value next to the NULL sentinel), 3 is NULL only."""
    w = ix.WIDTH["INT64"]
    rng = np.random.default_rng(seed)
    n = groups_n * 4
    keys = rng.integers(4, groups_n, n).astype(np.int32)
    p = np.array([x for x in ix.pool(w) if abs(x) <= 2 ** 53 + 1 and x & 0xFFFFFFFF != 2 ** 31], np.int64)   # no COUNT32_SENTINEL
    v = p[rng.integers(0, p.size, n)]
    v[rng.random(n) < 0.1] = w.null
    edge_k = np.array([0, 1, 2, 2, 3], np.int32)
    edge_v = np.array([ix.INT64_MAX, -ix.INT64_MAX, ix.INT64_MAX, 2, w.null], np.int64)
    return np.concatenate([edge_k, keys, np.arange(4, groups_n, dtype=np.int32)]), np.concatenate([edge_v, v, np.ones(groups_n - 4, np.int64)])


@pytest.mark.parametrize("groups_n,limit", [(1000, 0), (1000, 30), (100_000, 12)])
def test_order_by_integer_aggregates_at_the_extremes(groups_n, limit):
    w = ix.WIDTH["INT64"]
    keys, v = extreme_groups(groups_n, seed=groups_n + limit)
    gs = ix.groups_of(w, keys, v, True, frag_rows=200_000)
    t = w.table(notnull=False)
    for b in range(0, keys.size, 200_000):
        t.add_host_fragment([keys[b:b + 200_000], v[b:b + 200_000]])
    dev = gu.DeviceTable(t)
    exact = [(k, g.sum, g.min, g.max, g.count) for k, g in gs.items()]
    assert not any(g.sentinel_sum for g in gs.values())
    orders = [(c, d, nf) for c in (2, 3, 4, 5) for d in (False, True) for nf in (False, True)]
    if groups_n > 1000:                                               # the top-k pre-filter: one order per column
        orders = [(2, False, True), (3, True, False), (4, False, False), (5, True, True)]
    for col, desc, nf in orders:
        sql = (f"SELECT k, SUM(v), MIN(v), MAX(v), COUNT(v) FROM t GROUP BY k ORDER BY {col} {'DESC' if desc else 'ASC'} "
               f"NULLS {'FIRST' if nf else 'LAST'}, 1{f' LIMIT {limit}' if limit else ''};")
        rs = execute(sqlmini.parse(sql, t, ["k", "v"]), t, dev, entry_guess=groups_n + 1, has_card=True)
        want = expected_order(exact, [(col - 1, desc, nf), (0, False, False)])
        want = want[:limit] if limit else want
        assert rs.rows() == want, (sql, rs.rows()[:4], want[:4])


def sort_result(keys, vals, sql_type=abi.kBIGINT, nullable=True, aggs="SUM(v), MIN(v), MAX(v)"):
    t = abi.Table([(abi.kINT, True), (sql_type, not nullable)])
    for b in range(0, keys.size, 1 << 20):
        t.add_host_fragment([keys[b:b + (1 << 20)], vals[b:b + (1 << 20)]])
    unit = sqlmini.parse(f"SELECT k, {aggs} FROM t GROUP BY k;", t, ["k", "v"])
    rs = execute(unit, t, gu.DeviceTable(t), entry_guess=int(keys.max()) + 2, has_card=True)
    return rs, rs.rows()


def check_sort(rs, rows, entries, top_n):
    """ResultSet.sort(entries, top_n) == the Python order's first top_n rows."""
    rs.sort([(c + 1, d, nf) for c, d, nf in entries], top_n=top_n)
    want = expected_order(rows, entries)
    want = want[:top_n] if top_n else want
    got = rs.rows()
    assert got == want, (entries, top_n, got[:5], want[:5])


def test_topk_prefilter_edges():
    """> 65 536 groups and top_n * 8 <= n: the top-k pre-filter (sort.cu) runs on the primary key before the full sort."""
    rng = np.random.default_rng(12)
    g = 70_000
    keys = np.arange(g, dtype=np.int32)
    # primary keys that differ only below bit 13 (shift 0), with heavy ties
    v = rng.integers(0, 1 << 12, g).astype(np.int64)
    rs, rows = sort_result(keys, v, nullable=False, aggs="SUM(v)")
    for top_n in (1, 10, 8000):
        check_sort(rs, rows, [(1, False, False), (0, True, False)], top_n)
        check_sort(rs, rows, [(1, True, False), (0, False, False)], top_n)
    # keys spanning the whole 64-bit image (msb 63), NULL ranks on both sides
    p = np.array(ix.pool(ix.WIDTH["INT64"]), np.int64)
    v = p[rng.integers(0, p.size, g)]
    v[rng.random(g) < 0.3] = abi.NULL_BIGINT
    rs, rows = sort_result(keys, v)
    for col in (1, 2, 3):
        for desc in (False, True):
            for nf in (False, True):
                check_sort(rs, rows, [(col, desc, nf), (0, False, False)], 25)
    # a bucket that ends exactly at top_n: 100 groups at each of 700 distinct values, top_n = 300
    v = (np.arange(g) // 100).astype(np.int64) << 40
    rs, rows = sort_result(keys, rng.permutation(v), nullable=False, aggs="SUM(v)")
    for top_n in (300, 301, 299):
        check_sort(rs, rows, [(1, False, False), (0, False, False)], top_n)
    # n == 65536 and top_n * 8 == n
    keys = np.arange(65536, dtype=np.int32)
    rs, rows = sort_result(keys, rng.integers(-(2 ** 62), 2 ** 62, 65536).astype(np.int64), nullable=False, aggs="SUM(v)")
    check_sort(rs, rows, [(1, True, False), (0, False, False)], 8192)


def test_digit_skipping_sort_paths():
    """All primary keys equal (every digit pass is skipped; the next entry decides), and keys that differ only in the sign
    bit (one pass, on the top digit)."""
    keys = np.arange(5000, dtype=np.int32)
    rs, rows = sort_result(keys, np.full(5000, -7, np.int64), nullable=False, aggs="SUM(v)")
    check_sort(rs, rows, [(1, False, False), (0, True, False)], 0)
    v = np.where(np.arange(5000) % 3 == 0, 5, ix.INT64_MIN + 5).astype(np.int64)
    rs, rows = sort_result(keys, v, nullable=False, aggs="MIN(v)")
    for desc in (False, True):
        check_sort(rs, rows, [(1, desc, False), (0, False, False)], 0)


# ---- ResultSet.sort() over every target type --------------------------------------------------------------------------------------------
def test_result_set_sort_over_float_targets():
    """FLOAT MIN / MAX / SUM / AVG: ordered by value (negative floats too), NULL_FLOAT recognised as NULL, AVG's sum read as
    a float.  Dyadic values keep every sum exact, so the order is unique."""
    rng = np.random.default_rng(2)
    g = 3000
    keys = rng.integers(0, g, g * 6).astype(np.int32)
    vals = (rng.integers(-4000, 4000, keys.size) * 0.25).astype(np.float32)
    vals[rng.random(keys.size) < 0.05] = abi.NULL_FLOAT
    vals[keys == 5] = abi.NULL_FLOAT                                   # NULL only
    keys = np.concatenate([keys, np.arange(g, dtype=np.int32)])
    vals = np.concatenate([vals, np.where(np.arange(g) == 5, abi.NULL_FLOAT, 0.5).astype(np.float32)])
    rs, rows = sort_result(keys, vals, abi.kFLOAT, aggs="SUM(v), MIN(v), MAX(v), AVG(v)")
    assert any(r[2] is not None and r[2] < 0 for r in rows) and any(r[1] is None for r in rows)
    for col in (1, 2, 3, 4):
        for desc in (False, True):
            for nf in (False, True):
                check_sort(rs, rows, [(col, desc, nf), (0, False, False)], 0)
                check_sort(rs, rows, [(col, desc, nf), (0, True, False)], 40)


def test_result_set_sort_over_double_and_projection_float_columns():
    rng = np.random.default_rng(3)
    n = 20_000
    keys = np.arange(n, dtype=np.int32)
    d = rng.integers(-10 ** 6, 10 ** 6, n) * 0.125
    d[rng.random(n) < 0.05] = abi.NULL_DOUBLE
    rs, rows = sort_result(keys, d, abi.kDOUBLE, aggs="MIN(v)")
    check_sort(rs, rows, [(1, True, True), (0, False, False)], 0)
    f = (rng.integers(-10 ** 6, 10 ** 6, n) * 0.25).astype(np.float32)
    f[rng.random(n) < 0.05] = abi.NULL_FLOAT
    t = abi.Table([(abi.kINT, True), (abi.kFLOAT, False)])
    t.add_host_fragment([keys, f])
    dev = gu.DeviceTable(t)
    for columnar in (False, True):
        unit = sqlmini.parse("SELECT k, v FROM t WHERE k >= 0;", t, ["k", "v"])
        rs = executor.Executor().executeWorkUnit(0, False, dev.table, unit, eo=executor.execution_options(output_columnar_hint=columnar),
                                                 memory_level=abi.GPU_LEVEL)
        rows = rs.rows()
        for desc, nf in [(False, False), (True, True), (True, False)]:
            check_sort(rs, rows, [(1, desc, nf), (0, False, False)], 0)


# (sum, count) pairs of DECIMAL(18, 2) AVG groups found by a search over sums in [2^48, 2^54] and counts below 10: the two
# groups' sum / count round to the same double but sum / (count * 100) do not (first pair), or the other way round (second
# pair).  Every sum is exact in double, so each quotient is one rounding: 9069919065288332 is above 2^53 but even.
# The reference compares pair_to_double, which divides by count x 10^scale.
DECIMAL_NEAR_TIES = [((9069919065288332, 7), (5182810894450475, 4)), ((575410806117919, 5), (1035739451012254, 9))]


def test_result_set_sort_decimal_avg_near_ties():
    for (sa, ca), (sb, cb) in DECIMAL_NEAR_TIES:
        assert (sa / ca == sb / cb) != (sa / (ca * 100.0) == sb / (cb * 100.0))
        keys, vals = [], []
        for k, (s, c) in ((1, (sa, ca)), (2, (sb, cb))):
            parts = [s // c] * (c - 1) + [s - (s // c) * (c - 1)]
            keys += [k] * c
            vals += parts
        keys += [3, 3]
        vals += [1, 2]
        t = abi.Table([(abi.kINT, True), (abi.kDECIMAL, True)], col_scales={1: 2})
        t.add_host_fragment([np.array(keys, np.int32), np.array(vals, np.int64)])
        dev = gu.DeviceTable(t)
        exact = {1: ix.pair_to_double(sa, ca, 2), 2: ix.pair_to_double(sb, cb, 2), 3: ix.pair_to_double(3, 2, 2)}
        for desc in (False, True):
            for kdesc in (False, True):
                want = [k for k, _ in expected_order([(k, a) for k, a in exact.items()], [(1, desc, False), (0, kdesc, False)])]
                sql = (f"SELECT k, AVG(v) FROM t GROUP BY k ORDER BY 2 {'DESC' if desc else 'ASC'}, 1 {'DESC' if kdesc else 'ASC'};")
                rs = execute(sqlmini.parse(sql, t, ["k", "v"]), t, dev, entry_guess=8, has_card=True)
                assert [r[0] for r in rs.rows()] == want, (sql, (sa, ca), (sb, cb))
                rs = execute(sqlmini.parse("SELECT k, AVG(v) FROM t GROUP BY k;", t, ["k", "v"]), t, dev, entry_guess=8, has_card=True)
                rs.sort([(2, desc, False), (1, kdesc, False)])
                assert [r[0] for r in rs.rows()] == want, ((sa, ca), (sb, cb), desc, kdesc)
