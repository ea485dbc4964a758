"""Temporary tables on the host: synthesize_metadata (QueryEngine/InputMetadata.cpp:381-470) restated over host ColumnarResults
columns, the host table the reference's route builds from them (getResultSetColumn: host columns + host stats), and a driver
that runs the steps of sqlmini.parse_steps one after another.

The restatement follows the encoder Encoder::Create(nullptr, getColType(i)) picks (DataMgr/NoneEncoder.h:93-117, 219-223):
  * integer-meta columns (integers, DECIMAL as scaled int64, TIME / TIMESTAMP / DATE, dictionary ids): a value is NULL iff it
    equals the type's inline sentinel; min / max of static_cast<T>(value) over the others;
  * FLOAT / DOUBLE: NULL is inline_fp_null_val (FLT_MIN widened / DBL_MIN); std::min / std::max never take a NaN;
  * has_nulls = a NULL was seen;
  * no value in range (no rows, every value NULL or NaN): the fresh encoder's stats, min = numeric_limits<T>::max() and
    max = numeric_limits<T>::lowest()."""
import re

import numpy as np

import oracle_lib
import projection_ref
import sqlmini
from heavydb_b200 import abi, executor

FP = (abi.kFLOAT, abi.kDOUBLE)


def synthesize_metadata(cols):
    """cols = [(sql_type, notnull, ndarray[, scale])] -> [abi.ChunkStats]"""
    out = []
    for c in cols:
        ty, a = c[0], np.asarray(c[2])
        st = abi.ChunkStats()
        if ty in FP:
            dt = np.float32 if ty == abi.kFLOAT else np.float64
            a = a.astype(dt, copy=False)
            null = np.finfo(dt).tiny            # FLT_MIN / DBL_MIN: NULL_FLOAT / NULL_DOUBLE
            is_null = a == null
            vals = a[~is_null & ~np.isnan(a)]
            lim = float(np.finfo(dt).max)
            st.fp_min = float(vals.min()) if vals.size else lim
            st.fp_max = float(vals.max()) if vals.size else -lim
        else:
            dt = np.dtype(abi.NUMPY_OF[ty])
            is_null = a == abi.NULL_OF[ty]
            vals = a[~is_null].astype(dt, copy=False)
            info = np.iinfo(dt)
            st.int_min = int(vals.min()) if vals.size else int(info.max)
            st.int_max = int(vals.max()) if vals.size else int(info.min)
        st.has_nulls = int(bool(is_null.any()))
        out.append(st)
    return out


def stats_tuple(st: abi.ChunkStats, sql_type: int):
    """The fields of one ChunkStats that carry meaning for a column of this type (fp as floats, compared with ==)."""
    if sql_type in FP:
        return ("fp", st.fp_min, st.fp_max, st.has_nulls)
    return ("int", st.int_min, st.int_max, st.has_nulls)


def host_table(cols) -> abi.Table:
    """The host route's temporary table: one CPU fragment over host columns [(sql_type, notnull, ndarray, scale)] with the
    restated stats (a zero-row column passes a NULL pointer)."""
    t = abi.Table([(c[0], c[1]) for c in cols], col_scales={i: c[3] for i, c in enumerate(cols) if len(c) > 3 and c[3]})
    t.add_host_fragment([np.ascontiguousarray(c[2], dtype=abi.NUMPY_OF[c[0]]) for c in cols], fragment_id=0)
    t.fragments[0].stats = synthesize_metadata(cols)
    return t


def columns_from_rows(rows, col_types):
    """Host columns of rows given as python values (None = NULL), col_types = [(sql_type, notnull, scale)]."""
    cols = []
    for i, (ty, nn, scale) in enumerate(col_types):
        vals = [abi.NULL_OF[ty] if r[i] is None else r[i] for r in rows]
        cols.append((ty, bool(nn), np.array(vals, dtype=abi.NUMPY_OF[ty]), scale))
    return cols


def oracle_columns(unit, table, res, entry_guess, has_card=True):
    """Host ColumnarResults of an oracle result: b2q_rs_create_from_storage over its buffer, then b2q_columnar_results_create.
    A sorted or projected result is read through the oracle's own iteration (the host has no device to sort on)."""
    u = unit.unit
    if isinstance(res, HostProjection) or u.num_order_entries or u.has_limit or u.offset:
        return columns_from_rows(res.rows(decimal_to_double=False), [res.col_type(i) for i in range(res.col_count())])
    rs = executor.Executor().resultSetFromStorage(res.buffer(), unit, table, max_groups_buffer_entry_guess=entry_guess,
                                                  has_cardinality_estimation=has_card)
    return rs.columnarResults(with_scale=True)


class HostProjection:
    """A projection step on the host, where the oracle has no projection: the product's planner plans it (b2q_plan) and the
    rows are the step run by SQLite over its input table, in scan order (the GPU path is held to the same rows)."""

    def __init__(self, step, unit, table, names, entry_guess=0, has_card=True):
        self.plan = executor.Executor().plan(unit, table, max_groups_buffer_entry_guess=entry_guess,
                                             has_cardinality_estimation=has_card)
        assert self.plan.query_desc_type == abi.Projection
        if "'" in step.sql:
            raise ValueError("string literals against dictionary ids: SQLite holds the ids here, not the strings")
        toks = step.sql.rstrip(";").split()
        name = toks[toks.index("FROM") + 1]
        con = projection_ref.load_sqlite(table, names, name=name)
        sql = sqlite_sql(step.sql, unit)
        if not unit.unit.num_order_entries:
            m = re.search(r"\s(LIMIT|OFFSET)\s", sql, re.I)
            k = m.start() if m else len(sql)
            sql = f"{sql[:k]} ORDER BY _id, _r{sql[k:]}"
            if re.search(r"\sOFFSET\s", sql, re.I) and not re.search(r"\sLIMIT\s", sql, re.I):
                sql = sql.replace(" OFFSET ", " LIMIT -1 OFFSET ")
        self._rows = [tuple(r) for r in con.execute(sql).fetchall()]

    def rows(self, decimal_to_double=True):
        return self._rows

    def col_count(self):
        return self.plan.num_targets

    def col_type(self, i):
        t = self.plan.targets[i].sql_type
        return (t.type, t.notnull, t.scale)


def run_step_on_host(step, unit, table, names, entry_guess, has_card=True):
    """The oracle for aggregate steps, HostProjection for projection steps."""
    plan = executor.Executor().plan(unit, table, max_groups_buffer_entry_guess=entry_guess, has_cardinality_estimation=has_card)
    if plan.query_desc_type == abi.Projection:
        return HostProjection(step, unit, table, names, entry_guess, has_card)
    return oracle_lib.execute(unit, table, entry_guess=entry_guess, has_card=has_card, num_threads=2)


def run_steps(steps, tables, run, to_table, dicts=None, bigint_count=False):
    """Run parse_steps' steps in order.  tables = {name: (abi.Table, [names])}; run(i, unit, table, names) -> result;
    to_table(i, unit, table, result) -> the temporary table of an intermediate result.  Returns [(unit, table, result)]."""
    temps, out = [], []
    for i, st in enumerate(steps):
        def resolve(src):
            return tables[src] if isinstance(src, str) else (temps[src], steps[src].names)
        table, names = resolve(st.source)
        inner = resolve(st.inner) if st.inner is not None else None
        unit = sqlmini.parse(st.sql, table, names, bigint_count=bigint_count, inner=inner, dicts=dicts)
        res = run(i, unit, table, names)
        out.append((unit, table, res))
        temps.append(to_table(i, unit, table, res) if i + 1 < len(steps) else None)
    return out


def sqlite_sql(sql: str, unit) -> str:
    """The query for SQLite with the final ORDER BY's NULL placement made explicit (HeavyDB's NULLs are the largest values)."""
    s = sql.rstrip(";")
    u = unit.unit
    if not u.num_order_entries:
        return s
    up = s.upper()
    k = up.rindex(" ORDER BY ")
    head, tail = s[:k], s[k + 10:]
    m = re.search(r"\s(LIMIT|OFFSET)\s", tail, re.I)
    rest = tail[m.start():] if m else ""
    items = [f"{u.order_entries[i].tle_no} {'DESC' if u.order_entries[i].is_desc else 'ASC'} NULLS "
             f"{'FIRST' if u.order_entries[i].nulls_first else 'LAST'}" for i in range(u.num_order_entries)]
    if re.search(r"\sOFFSET\s", rest, re.I) and not re.search(r"\sLIMIT\s", rest, re.I):
        rest = " LIMIT -1" + rest
    return f"{head} ORDER BY {', '.join(items)}{rest}"


def translate(rows, plan, names, dicts):
    """Dictionary ids of the final step's string targets back to strings, by the target's column name."""
    idx = [(i, dicts[names[i]]) for i, t in enumerate(plan.targets[: plan.num_targets])
           if not t.is_agg and t.sql_type.type in (abi.kTEXT, abi.kVARCHAR, abi.kCHAR) and names[i] in dicts]
    if not idx:
        return rows
    out = []
    for r in rows:
        r = list(r)
        for i, d in idx:
            if r[i] is not None:
                r[i] = d[r[i]] if 0 <= r[i] < len(d) else None
        out.append(tuple(r))
    return out


def float_sum_query(sql: str) -> bool:
    """SUM / AVG over a FLOAT column of the golden table: float-precision accumulation, compared with an absolute bound."""
    return re.search(r"\b(SUM|AVG)\s*\(\s*(f|ff|fn)\s*\)", sql, re.I) is not None
