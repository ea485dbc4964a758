"""Restatement of a projection unit for the tests, independent of the planner under test.

Descriptor (QueryMemoryDescriptor::init, Projection branch, QueryMemoryDescriptor.cpp:394-418, without lazy fetch): one slot
per target of the column's logical size (ColSlotContext, ColSlotContext.cpp:35-97).  Row-wise every slot is padded to 8 bytes
(setAllUnsetSlotsPaddedSize(8)) behind the int64 offset word (get_scan_output_slot, GroupByRuntime.cpp:242-254); columnar the
slots stay logical-sized (isLogicalSizedColumnsAllowed) behind the int64 offsets column (get_columnar_scan_output_offset,
:256-266), every column padded to 8 bytes.

Values: what the chunk decoders hand to agg_id — ENCODING FIXED and DICT(8|16) NULLs become the logical NULL, DATE DAYS values are
days * 86400 (NULL: the logical NULL); integer slots hold the logical value sign-extended, DOUBLE its bits, FLOAT its 4 bytes
(upper word 0 in a row-wise slot).

Rows: those SQLite selects (SQL three-valued logic) over the decoded rows, deleted rows left out, in (fragment id, row) order;
under a scan limit the first scan_limit of them."""
from __future__ import annotations

import sqlite3

import numpy as np

from heavydb_b200 import abi

LOGICAL_SIZE = {abi.kTINYINT: 1, abi.kSMALLINT: 2, abi.kINT: 4, abi.kFLOAT: 4, abi.kTEXT: 4, abi.kVARCHAR: 4, abi.kCHAR: 4}


def logical_size(t):
    return LOGICAL_SIZE.get(t, 8)


def align8(x):
    return (x + 7) // 8 * 8


def restate_descriptor(table: abi.Table, cols, columnar: bool, entry_count: int) -> dict:
    logical = [logical_size(table.col_types[c][0]) for c in cols]
    padded = logical if columnar else [8] * len(cols)
    offs, off = [], align8(8 * entry_count) if columnar else 8
    for w in padded:
        offs.append(off)
        off += align8(w * entry_count) if columnar else 8
    row_size = align8(sum(padded)) if columnar else off
    return {"query_desc_type": abi.Projection, "entry_count": entry_count, "output_columnar": int(columnar),
            "num_targets": len(cols), "num_slots": len(cols), "effective_key_width": 8, "key_col_id": -1,
            "slot_logical_width": logical, "slot_padded_width": padded, "slot_offset": offs, "row_size": row_size,
            "buffer_size": off if columnar else row_size * entry_count}


def plan_matches(plan: abi.Plan, d: dict):
    n = d["num_slots"]
    for k, v in d.items():
        got = list(getattr(plan, k)[:n]) if isinstance(v, list) else getattr(plan, k)
        assert got == v, (k, got, v)


def decode(table: abi.Table, c: int, phys: np.ndarray):
    """(logical values, NULL mask) of a chunk's physical elements."""
    t, nn = table.col_types[c]
    enc = table.encoded_sizes[c]
    pnull = table.physical_null(c)
    isnull = (phys == pnull) if (not nn or enc <= 0) else np.zeros(phys.shape, dtype=bool)   # an unencoded sentinel reads as NULL
    if t in (abi.kFLOAT, abi.kDOUBLE):
        return phys.copy(), phys == abi.NULL_OF[t]
    vals = phys.astype(np.int64)
    if enc < 0:
        vals = vals * 86400
    vals = np.where(isnull, np.int64(abi.NULL_OF[t]), vals)
    return vals, isnull


def load_sqlite(table: abi.Table, names, name="t"):
    """The decoded rows (NULL as SQL NULL) plus _id / _r (fragment id, row in fragment) and _del (1 = deleted row)."""
    con = sqlite3.connect(":memory:")
    decl = ", ".join(f"{n} {'double' if t in (abi.kDOUBLE, abi.kFLOAT) else 'bigint'}" for n, (t, _nn) in zip(names, table.col_types))
    con.execute(f"CREATE TABLE {name}(_id bigint, _r bigint, _del bigint, {decl})")
    for f in table.fragments:
        cols = []
        for c in range(table.num_cols):
            v, isnull = decode(table, c, f.host_cols[c])
            cols.append([None if m else x for x, m in zip(v.tolist(), isnull.tolist())])
        dc = table.deleted_column
        rows = [(f.fragment_id, r, int(dc is not None and (cols[dc][r] or 0) > 0)) + tuple(col[r] for col in cols) for r in range(f.num_tuples)]
        con.executemany(f"INSERT INTO {name} VALUES({','.join('?' * (len(names) + 3))})", rows)
    return con


def passing_rows(con, where: str | None, name="t"):
    """[(fragment id, row)] of the rows that pass, in scan order."""
    w = f" AND ({where})" if where else ""
    return con.execute(f"SELECT _id, _r FROM {name} WHERE _del = 0{w} ORDER BY _id, _r").fetchall()


def expected_buffer(table: abi.Table, cols, picks, columnar: bool) -> np.ndarray:
    """The buffer of len(picks) entries laid out as the restated descriptor says."""
    d = restate_descriptor(table, cols, columnar, len(picks))
    n = len(picks)
    frag = {f.fragment_id: f for f in table.fragments}
    buf = np.zeros(d["buffer_size"], dtype=np.uint8)
    rows = buf.reshape(n, d["row_size"]) if not columnar else None
    offs = np.array([r for _f, r in picks], dtype=np.int64)
    for s, c in enumerate(cols):
        t = table.col_types[c][0]
        phys = np.array([frag[f].host_cols[c][r] for f, r in picks], dtype=table.physical_dtype(c))
        vals, _ = decode(table, c, phys)
        w = d["slot_padded_width"][s]
        if t == abi.kFLOAT:
            img = vals.astype(np.float32).view(np.uint32)
            img = img.astype(np.uint64) if w == 8 else img
        elif t == abi.kDOUBLE:
            img = vals.astype(np.float64).view(np.int64)
        else:
            img = vals.astype({1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}[w])
        img = np.ascontiguousarray(img).view(np.uint8)
        off = d["slot_offset"][s]
        if columnar:
            buf[off:off + n * w] = img
        elif n:
            rows[:, off:off + 8] = img.reshape(n, 8)
    if columnar:
        buf[0:8 * n] = offs.view(np.uint8)
    elif n:
        rows[:, 0:8] = offs.view(np.uint8).reshape(n, 8)
    return buf


def projected_cols(unit: abi.BuiltUnit):
    u = unit.unit
    return [u.exprs[u.target_exprs[i]].col_id for i in range(u.num_target_exprs)]


def mixed_table(n, seed, frag_rows, fragment_ids=None, deleted_frac=0.1):
    """Every encoding a projection decodes: ENCODING FIXED, DICT(8|16), DATE DAYS(32|16), DECIMAL (plain and FIXED(32)),
    TIME / TIMESTAMP, TINYINT / SMALLINT, FLOAT / DOUBLE, NULLs in each nullable column, and a $deleted$ column."""
    rng = np.random.default_rng(seed)
    spec = [  # name, type, notnull, encoded size, scale, generator of physical values
        ("k", abi.kBIGINT, True, 0, 0, lambda: rng.integers(0, 1000, n) + np.arange(n) // frag_rows * 1000),  # k // 1000 = fragment
        ("i32f16", abi.kINT, False, 2, 0, lambda: rng.integers(-3000, 3000, n)),
        ("i64f8", abi.kBIGINT, False, 1, 0, lambda: rng.integers(-100, 100, n)),
        ("i64f32nn", abi.kBIGINT, True, 4, 0, lambda: rng.integers(-2**31 + 1, 2**31 - 1, n)),
        ("s8", abi.kTEXT, False, 1, 0, lambda: rng.integers(0, 250, n)),
        ("s16", abi.kTEXT, False, 2, 0, lambda: rng.integers(0, 60000, n)),
        ("s32", abi.kTEXT, False, 0, 0, lambda: rng.integers(0, 10**6, n)),
        ("dt", abi.kDATE, False, -4, 0, lambda: rng.integers(-20000, 20000, n)),
        ("dt16", abi.kDATE, False, -2, 0, lambda: rng.integers(-20000, 20000, n)),
        ("dec", abi.kDECIMAL, False, 0, 2, lambda: rng.integers(-10**9, 10**9, n)),
        ("dec32", abi.kDECIMAL, False, 4, 2, lambda: rng.integers(-10**8, 10**8, n)),
        ("tm", abi.kTIME, False, 0, 0, lambda: rng.integers(0, 86400, n)),
        ("ts32", abi.kTIMESTAMP, False, 4, 0, lambda: rng.integers(0, 2**31 - 1, n)),
        ("ti", abi.kTINYINT, False, 0, 0, lambda: rng.integers(-127, 128, n)),
        ("si", abi.kSMALLINT, False, 0, 0, lambda: rng.integers(-32767, 32768, n)),
        ("f", abi.kFLOAT, False, 0, 0, lambda: rng.random(n) * 100),
        ("d", abi.kDOUBLE, False, 0, 0, lambda: rng.random(n) * 100),
        ("del", abi.kBOOLEAN, True, 0, 0, lambda: rng.random(n) < deleted_frac),
    ]
    t = abi.Table([(ty, nn) for _, ty, nn, *_ in spec], encoded_sizes=[e for _, _, _, e, _, _ in spec],
                  deleted_column=len(spec) - 1, col_scales={c: sc for c, (_, _, _, _, sc, _) in enumerate(spec) if sc})
    cols = []
    for c, (_name, ty, nn, _e, _sc, gen) in enumerate(spec):
        a = np.asarray(gen()).astype(t.physical_dtype(c))
        if not nn and ty != abi.kBOOLEAN:
            a[rng.random(n) < 0.1] = t.physical_null(c)
        cols.append(a)
    starts = list(range(0, n, frag_rows))
    ids = fragment_ids or list(range(len(starts)))
    for fid, b in zip(ids, starts):
        t.add_host_fragment([a[b:b + frag_rows] for a in cols], fragment_id=fid)
    return t, [s[0] for s in spec]
