"""IN / NOT IN lists past the 16-leaf filter program, checked on the CPU: the planner lowers each such list to ONE set term
(a bitmap over [min, max] of the values on the device), and only when the leaf program does not fit.

tests/cpp/in_list_emulator.cpp (the host reading of tests/cpp/filter_emulator.cpp, extended) reads the set term as a search
in the term's value list, so the lowered program is compared
row for row with the oracle, SQLite and int_exact_ref's three-valued predicates.  Programs that fit the leaf program are
compared byte for byte with the ones the planner emitted before set terms existed (tests/golden/in_list_leaf_programs.json,
recorded from that planner over the corpus below)."""
import ctypes as C
import hashlib
import json
import os
import random
import sqlite3
import subprocess

import numpy as np
import pytest

import int_exact_ref as ier
import join_tables as jt
import oracle_lib
import ref_time_table as tt
import sqlmini
import str_tables as stt
from heavydb_b200 import abi, build, executor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "in_list_leaf_programs.json")


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    build.build()
    so = tmp_path_factory.mktemp("emu_in") / "libfilter_emulator.so"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "in_list_emulator.cpp"), "-o", str(so)])
    return load_emulator(str(so))


class WithSets:
    """What test_filter_lowering's run_program / run_join_program call, with set terms (same arguments and results)."""
    def __init__(self, E):
        self.b2q_test_run_program = E.b2q_test_run_program_sets
        self.b2q_test_run_program_joined = E.b2q_test_run_program_joined_sets


def load_emulator(path):
    E = C.CDLL(path)
    for name, res, args in [("b2q_test_eval_filter_sets", C.c_int32, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int64]),
                            ("b2q_test_filter_terms", C.c_int32, [C.c_void_p]),
                            ("b2q_test_set_terms", C.c_int32, [C.c_void_p]),
                            ("b2q_test_filter_bytes", C.c_int64, [C.c_void_p, C.c_void_p, C.c_int64])]:
        getattr(E, name).restype = res
        getattr(E, name).argtypes = args
    return E


class Planned:
    """A query planned on the host (b2q_plan), freed on exit; rc != 0: refused."""
    def __init__(self, unit, table, guess=0, has_card=False):
        self.L = executor.lib()
        self.bt = table.build(abi.CPU_LEVEL)
        co, eo = executor.compilation_options(), executor.execution_options()
        self.h = C.c_void_p()
        self.rc = self.L.b2q_plan(C.byref(unit.unit), C.byref(self.bt.info), C.byref(co), C.byref(eo), guess, int(has_card), C.byref(self.h))
        self.err = self.L.b2q_last_error_message().decode() if self.rc else None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        if not self.rc:
            self.L.b2q_query_free(self.h)


def filter_digest(E, unit, table):
    """sha256 of the lowered filter's bytes (b2q_test_filter_bytes), or "rc<code>" when the planner refuses the query."""
    with Planned(unit, table) as p:
        if p.rc:
            return f"rc{p.rc}"
        buf = (C.c_uint8 * 8192)()
        n = E.b2q_test_filter_bytes(p.h, buf, 8192)
        return hashlib.sha256(bytes(buf[:n])).hexdigest()[:20]


def set_terms(E, unit, table):
    """(set terms, all terms) of the planned filter; raises with the planner's message when it refuses."""
    with Planned(unit, table) as p:
        assert p.rc == 0, p.err
        return E.b2q_test_set_terms(p.h), E.b2q_test_filter_terms(p.h)


def where_of(sql):
    import re
    m = re.search(r" WHERE (.*?)( GROUP BY | ORDER BY |;)", sql)
    return m.group(1) if m else None


# ---- the lowering corpora: every program the planner emitted before set terms must come out the same ------------------------
FOLD_CASES = [
    "k8 IN (1, 2, 3, 7, 8, 20)", "NOT (k8 IN (5, 4, 3) OR k16 = 7)", "k16 IN (100, 101, 102) AND a8 NOT IN (-1, 0, 1, 2)",
    "nn32 IN (3, 4, 5) OR nn32 IN (6, 7) OR d < 0.5", "k8 = 2 OR (k32 < 10 AND k16 > 5) OR k8 = 3 OR k8 = 4 OR a16 IS NULL",
    "k64 IN (1000000001, 1000000002, 1000000004)", "a8 IN (5, 5, 6) OR a8 = 127", "NOT (a16 <> 10 AND a16 <> 11 AND a16 <> 12)",
    "k16 BETWEEN 100 AND 130", "k16 >= 100 AND k16 <= 130 AND k16 < 125 AND k16 > 90", "k16 NOT BETWEEN 100 AND 130",
    "k16 < 100 OR k16 > 130 OR k16 = 110", "a8 > 5 AND d < 0.5 AND a8 <= 60 AND nn32 <> 7", "k8 >= 2 AND k8 <= 9 AND k8 NOT IN (4, 5, 6)",
    "(a16 > 100 AND a16 < 20000) OR (a16 > -20000 AND a16 < -100)", "a16 < 100 OR a16 > 99", "dnn < 0.3 OR dnn > 0.6 OR dnn = 0.45",
    "a16 IS NOT NULL AND a16 > 100", "a64 IS NOT NULL AND a64 IN (5, 6, 7) AND nn64 IS NOT NULL",
    "k32 IN (" + ", ".join(str(v) for v in range(-40, 200, 15)) + ")",                      # 16 scattered values: 16 leaves
    "k32 NOT IN (" + ", ".join(str(v) for v in range(-40, 200, 15)) + ")",
    "k8 IN (" + ", ".join(str(v) for v in range(-3, 27)) + ")",                             # dense: one range
    "a32 IN (" + ", ".join(str(v) for v in list(range(0, 40)) + [77, 99]) + ")",            # a run and two leaves
]
STR_FOLD_CASES = ["dd IN (1555286400, 1555372800, 1555459200)", "dd16 NOT IN (864000000, 864086400, 863913600, 5)",
                  "s8 IN (3, 4, 5, 6, 200) OR str = 7 OR str = 8", "dt IN (1555200000, 1555286400) OR dt = 1555372801",
                  "dd NOT IN (1555286400, 1555372800, 5)", "ts <= 1600000100 AND s8 <> 200 AND NOT (s16 = 7)"]


def lowering_corpus():
    """(label, table, names, sql, inner) of the lowering tests' queries: hand-written IN / range cases, the random filter
    trees, dense IN lists and range chains, the fuzz generator's queries, the reference-shaped query lists and joins."""
    from test_gpu_fuzz import rand_join_query, rand_query
    from test_gpu_parity import RAND_NAMES, RAND_QUERIES, random_table
    out = []
    r = random_table(900, seed=61, frag_rows=250)
    out += [(f"fold{i}", r, RAND_NAMES, f"SELECT COUNT(*) FROM r WHERE {w};", None) for i, w in enumerate(FOLD_CASES)]
    s = stt.str_table(1500, seed=9, frag_rows=400)
    out += [(f"strfold{i}", s, stt.STR_NAMES, f"SELECT COUNT(*) FROM s WHERE {w};", None) for i, w in enumerate(STR_FOLD_CASES)]
    out += [(f"str{i}", s, stt.STR_NAMES, q, None) for i, q in enumerate(stt.STR_QUERIES)]
    t = tt.make_table(tt.time_rows())
    out += [(f"time{i}", t, tt.TIME_NAMES, q, None) for i, q in enumerate(tt.TIME_QUERIES)]
    out += [(f"rand{i}", r, RAND_NAMES, q, None) for i, q in enumerate(RAND_QUERIES)]
    for seed in range(3):
        rng = random.Random(4400 + seed)
        for i in range(150):
            w = where_of(rand_query(rng))
            if w:
                out.append((f"tree{seed}.{i}", r, RAND_NAMES, f"SELECT COUNT(*) FROM r WHERE {w};", None))
    for seed in range(3):
        rng = random.Random(31000 + seed)
        for i in range(70):
            out.append((f"fuzz{seed}.{i}", r, RAND_NAMES, rand_query(rng, multi_key=(i % 3 == 0)), None))
    cols = {"k8": (-2, 12), "k16": (90, 140), "nn32": (0, 40), "a8": (-128, 127), "k64": (1000000000, 1000000040), "nn64": (-50, 50)}
    for seed in range(2):
        rng = random.Random(880 + seed)
        for i in range(120):
            parts = []
            for _ in range(rng.randint(1, 3)):
                c = rng.choice(sorted(cols))
                lo, hi = cols[c]
                start = rng.randint(lo, hi)
                vals = [start + k for k in range(rng.randint(1, 6))] + [rng.randint(lo, hi) for _ in range(rng.randint(0, 2))]
                rng.shuffle(vals)
                parts.append(f"{c} {'NOT IN' if rng.random() < 0.4 else 'IN'} ({', '.join(map(str, vals))})")
            where = parts[0]
            for p in parts[1:]:
                where = f"({where}) {rng.choice(['AND', 'OR'])} {'NOT ' if rng.random() < 0.2 else ''}({p})"
            out.append((f"dense{seed}.{i}", r, RAND_NAMES, f"SELECT COUNT(*) FROM r WHERE {where};", None))
    rcols = dict(cols, a16=(-32768, 32767), big=(-2**62, 2**62))
    for seed in range(2):
        rng = random.Random(990 + seed)
        for i in range(150):
            leaves = []
            for _ in range(rng.randint(2, 6)):
                c = rng.choice(sorted(rcols))
                lo, hi = rcols[c]
                leaves.append(f"{'NOT ' if rng.random() < 0.15 else ''}({c} {rng.choice(['<', '<=', '>', '>=', '=', '<>'])} {rng.randint(lo, hi)})")
            where = leaves[0]
            for lf in leaves[1:]:
                where = f"{where} {rng.choice(['AND', 'AND', 'OR'])} {lf}" if rng.random() < 0.7 else f"({where}) {rng.choice(['AND', 'OR'])} {lf}"
            out.append((f"chain{seed}.{i}", r, RAND_NAMES, f"SELECT COUNT(*) FROM r WHERE {where};", None))
    fact, dim = jt.fact_table(1500, seed=41, frag_rows=600), jt.dim_table(seed=13)
    rng = random.Random(77)
    joins = jt.JOIN_QUERIES + jt.LEFT_JOIN_QUERIES + [rand_join_query(rng) for _ in range(60)]
    out += [(f"join{i}", fact, jt.FACT_NAMES, q, (dim, jt.DIM_NAMES)) for i, q in enumerate(joins)]
    return out


def corpus_digests(E):
    out = {}
    for label, table, names, sql, inner in lowering_corpus():
        try:
            unit = sqlmini.parse(sql, table, names, inner=inner)
        except ValueError:
            continue
        out[label] = [hashlib.sha256(sql.encode()).hexdigest()[:8], filter_digest(E, unit, table)]
    return out


def test_programs_that_fit_the_leaf_program_are_unchanged(emu):
    """Byte for byte: term count, ops and every term's fields, for every query of the corpus; a refusal keeps its code."""
    want = json.load(open(GOLDEN))
    got = corpus_digests(emu)
    assert len(got) == len(want) >= 1000
    diff = [k for k in want if got.get(k) != want[k]]
    assert not diff, [(k, want[k], got.get(k)) for k in diff[:5]]
    for label, table, names, sql, inner in lowering_corpus()[:len(FOLD_CASES)]:
        assert set_terms(emu, sqlmini.parse(sql, table, names, inner=inner), table)[0] == 0, sql


# ---- which lists become set terms --------------------------------------------------------------------------------------------
def scattered(rng, n, lo, hi, step_min=2):
    """min(n, what fits) distinct values in [lo, hi], no two closer than step_min (no folding into runs), in random order."""
    cands = range(lo + rng.randrange(step_min), hi + 1, step_min)
    return rng.sample(cands, min(n, len(cands)))


def lst(vals):
    return ", ".join(str(v) for v in vals)


def test_lists_past_the_leaf_program_become_set_terms(emu):
    from test_gpu_parity import RAND_NAMES, random_table
    table = random_table(600, seed=81, frag_rows=200)
    rng = random.Random(5)
    a, b = scattered(rng, 17, -1000, 1000), scattered(rng, 40, 0, 30000)
    cases = [
        (f"k32 IN ({lst(a)})", 1, 1), (f"k32 NOT IN ({lst(a)})", 1, 1), (f"NOT (k32 IN ({lst(a)}))", 1, 1),
        (f"k32 IN ({lst(a)}) AND a16 IN ({lst(b)})", 2, 2), (f"k32 IN ({lst(a)}) OR a16 NOT IN ({lst(b)}) OR d < 0.5", 2, 3),
        (f"k32 IN ({lst(a)}) AND k16 > 5 AND k16 < 100", 1, 2), (f"k32 IN ({lst(a[:16])})", 0, 16),
        (f"k64 IN ({lst(a)}) AND nn32 = 4", 1, 2), (f"k32 IN ({lst(a)}) OR k32 < -5000", 1, 2),
        (f"(k32 IN ({lst(a[:9])}) AND k8 = 1) OR (k32 IN ({lst(a[9:])}) AND k8 = 2)", 2, 4),
    ]
    for where, n_sets, n_terms in cases:
        unit = sqlmini.parse(f"SELECT COUNT(*) FROM r WHERE {where};", table, RAND_NAMES)
        assert set_terms(emu, unit, table) == (n_sets, n_terms), where


def set_values(emu, unit, table, k=0):
    emu.b2q_test_set_values.restype = C.c_int64
    emu.b2q_test_set_values.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64]
    with Planned(unit, table) as p:
        assert p.rc == 0, p.err
        out = np.zeros(1 << 16, np.int64)
        n = emu.b2q_test_set_values(p.h, k, out.ctypes.data, out.size)
        return out[:n].tolist()


def test_set_values_are_logical_sorted_and_in_the_register_class(emu):
    """Duplicates go, days-encoded DATE values are days (off-grid seconds dropped), a 4-byte column keeps only int32 values."""
    from test_gpu_parity import RAND_NAMES, random_table
    table = random_table(300, seed=82, frag_rows=100)
    rng = random.Random(6)
    a = scattered(rng, 20, -100, 100)
    got = set_values(emu, sqlmini.parse(f"SELECT COUNT(*) FROM r WHERE k32 IN ({lst(a + a[:5] + [2**31, -2**31 - 1, 2**40])});", table, RAND_NAMES), table)
    assert got == sorted(a)
    got = set_values(emu, sqlmini.parse(f"SELECT COUNT(*) FROM r WHERE k64 IN ({lst(a + [2**31, -2**31 - 1])});", table, RAND_NAMES), table)
    assert got == sorted(a + [2**31, -2**31 - 1])
    s = stt.str_table(200, seed=3, frag_rows=100)
    days = scattered(rng, 20, 17990, 18070)
    secs = [d * 86400 for d in days] + [days[0] * 86400 + 1, 5]
    got = set_values(emu, sqlmini.parse(f"SELECT COUNT(*) FROM s WHERE dd IN ({lst(secs)});", s, stt.STR_NAMES), s)
    assert got == sorted(days)


def test_a_bitmap_at_the_memory_limit_is_not_built(emu):
    """[min, max] of 8e9 values or more (g_bitmap_memory_limit bits): the group keeps its leaves, and a list of more than 16
    of them is refused as before.  The OR chain is a binary tree, so a subtree whose values do fit still becomes a set."""
    from test_gpu_parity import RAND_NAMES, random_table
    table = random_table(300, seed=83, frag_rows=100)
    rng = random.Random(7)
    base = [v for v in scattered(rng, 19, 1, 10**6)]
    fits = [0] + base + [8_000_000_000 - 2]
    assert set_terms(emu, sqlmini.parse(f"SELECT COUNT(*) FROM r WHERE k64 IN ({lst(fits)});", table, RAND_NAMES), table) == (1, 1)
    far = 8_000_000_000 - 1
    with Planned(sqlmini.parse(f"SELECT COUNT(*) FROM r WHERE k64 IN ({lst([far, 0] + base)});", table, RAND_NAMES), table) as p:
        assert p.rc == abi.ERR_UNSUPPORTED and p.err == "filter too large", (p.rc, p.err)
    assert set_terms(emu, sqlmini.parse(f"SELECT COUNT(*) FROM r WHERE k64 IN ({lst([0] + base + [far])});", table, RAND_NAMES), table) == (1, 2)
    # the set term does not help when the program still does not fit: the first error stands
    many = " AND ".join(f"k{w} <> {v}" for w in (8, 16, 32, 64) for v in (3, 7, 11, 15, 19))
    with Planned(sqlmini.parse(f"SELECT COUNT(*) FROM r WHERE k32 IN ({lst(base)}) AND {many} AND a8 > 1 AND a16 > 1 AND a32 > 1 AND a64 > 1 AND nn32 > 1 AND nn64 > 1 AND big > 1 AND d > 1 AND dnn > 1 AND f32 > 1 AND fnn > 1 AND k8 < 100 AND k16 < 1000;", table, RAND_NAMES), table) as p:
        assert p.rc == abi.ERR_UNSUPPORTED and p.err == "filter too large", (p.rc, p.err)


# ---- row for row against the oracle and SQLite -------------------------------------------------------------------------------
def logical_columns(table):
    """Per column: Python values (None = NULL), DATE ENCODING DAYS as seconds, DECIMAL as scaled integers."""
    cols = []
    for c, (ty, nn) in enumerate(table.col_types):
        a = np.concatenate([f.host_cols[c] for f in table.fragments])
        null = table.physical_null(c)
        days = table.encoded_sizes[c] < 0
        vals = []
        for x in a.tolist():
            if not nn and x == null:
                vals.append(None)
            else:
                vals.append(float(x) if ty in (abi.kDOUBLE, abi.kFLOAT) else int(x) * (86400 if days else 1))
        cols.append(vals)
    return cols


def sqlite_of(table, names, name):
    con = sqlite3.connect(":memory:")
    cols = logical_columns(table)
    con.execute(f"CREATE TABLE {name}({', '.join(f'{n} {'double' if t in (abi.kDOUBLE, abi.kFLOAT) else 'integer'}' for n, (t, _) in zip(names, table.col_types))})")
    con.executemany(f"INSERT INTO {name} VALUES({','.join('?' * len(names))})", list(zip(*cols)))
    return con


def emulated_rows(emu, unit, table):
    """Indices (in fragment order) of the rows the lowered program passes."""
    with Planned(unit, table) as p:
        assert p.rc == 0, p.err
        out, base = [], 0
        for f in table.fragments:
            ptrs = (C.c_void_p * table.num_cols)(*[a.ctypes.data for a in f.host_cols])
            for row in range(f.num_tuples):
                r = emu.b2q_test_eval_filter_sets(p.h, ptrs, row)
                assert r >= 0
                if r:
                    out.append(base + row)
            base += f.num_tuples
        return out


def check_rows(emu, table, names, name, where, con, sqlite_where=None, min_sets=1):
    unit = sqlmini.parse(f"SELECT COUNT(*) FROM {name} WHERE {where};", table, names, dicts=getattr(table, "_dicts", None))
    assert set_terms(emu, unit, table)[0] >= min_sets, where
    got = emulated_rows(emu, unit, table)
    want = [r[0] - 1 for r in con.execute(f"SELECT rowid FROM {name} WHERE {sqlite_where or where} ORDER BY rowid")]
    assert got == want, where
    assert oracle_lib.execute(unit, table).rows()[0][0] == len(got), where


def random_where(rng, cols, n_lo=17, n_hi=300):
    c = rng.choice(sorted(cols))
    lo, hi = cols[c]
    vals = scattered(rng, min(rng.randint(n_lo, n_hi), (hi - lo) // 4), lo, hi)
    if rng.random() < 0.3:
        vals += [rng.randint(lo, hi) for _ in range(3)]                         # duplicates
    return f"{c} {'NOT IN' if rng.random() < 0.4 else 'IN'} ({lst(vals)})"


@pytest.fixture(scope="module")
def rand_env():
    from test_gpu_parity import RAND_NAMES, random_table
    table = random_table(2500, seed=84, frag_rows=700)
    return table, RAND_NAMES, sqlite_of(table, RAND_NAMES, "r")


INT_COLS = {"k8": (-150, 150), "k16": (60, 12000), "k32": (-3000, 60000), "k64": (10**9 - 500, 10**9 + 9000), "nn32": (-30, 5000),
            "nn64": (-200, 9000), "a8": (-128, 127), "a16": (-32768, 32767), "a32": (-50000, 50000), "a64": (-10**6, 10**6)}


@pytest.mark.parametrize("seed", range(3))
def test_long_lists_with_other_leaves_row_for_row(emu, rand_env, seed):
    """Random IN / NOT IN lists of 17 to 5 000 scattered values, alone, several in one query, and under AND / OR / NOT with
    other leaves: the rows the emulated program passes are SQLite's, their count the oracle's."""
    table, names, con = rand_env
    rng = random.Random(600 + seed)
    for i in range(12):
        parts = [random_where(rng, INT_COLS, 17, 5000 if i == 0 else 300) for _ in range(rng.randint(1, 3))]
        parts += [rng.choice(["d < 0.3", "k8 = 3", "a16 IS NULL", "nn32 BETWEEN 100 AND 900", "k32 <> 7", "dnn >= 0.5", "big > 0"])
                  for _ in range(rng.randint(0, 3))]
        rng.shuffle(parts)
        where = parts[0]
        for p in parts[1:]:
            where = f"({where}) {rng.choice(['AND', 'OR'])} {'NOT ' if rng.random() < 0.25 else ''}({p})"
        if rng.random() < 0.2:
            where = f"NOT ({where})"
        check_rows(emu, table, names, "r", where, con)


def test_list_values_at_the_null_sentinel(emu):
    """A list value equal to the column's NULL sentinel (and its neighbours) never matches a NULL row, for IN and NOT IN,
    on plain, FIXED and DICT(8|16) columns."""
    import enc_tables as et
    e = et.enc_table(3000, seed=4, frag_rows=800)
    con = sqlite_of(e, et.ENC_NAMES, "e")
    rng = random.Random(8)
    for col, null in [("k_i32_f16", -2**15), ("a_i64_f8", -2**7), ("a_i32_f8", -2**7), ("plain64", -2**63)]:
        vals = [null, null + 1, null + 2, null - 1] + [null + 4 + 3 * k for k in range(20)]
        if null > -2**63:
            vals += scattered(rng, 20, -120, 120)                                # values the data holds
        vals = [v for v in vals if v >= -2**63]
        for neg in ("", "NOT "):
            where = f"{col} {neg}IN ({lst(vals)})"
            check_rows(emu, e, et.ENC_NAMES, "e", where, con, sqlite_where=f"({where}) AND deleted = 0")
    s = stt.str_table(3000, seed=5, frag_rows=700)
    scon = sqlite_of(s, stt.STR_NAMES, "s")
    for col, null, hi in [("s8", 255, 254), ("s16", 65535, 39999), ("str", -2**31, 49)]:
        vals = sorted({null, null - 1, 0, 1} | set(scattered(rng, 20, 2, hi)))
        for neg in ("", "NOT "):
            check_rows(emu, s, stt.STR_NAMES, "s", f"{col} {neg}IN ({lst(vals)})", scon)


def test_encodings_dictionary_strings_days_decimal_and_time(emu):
    """FIXED, DICT(8|16|32) ids and dictionary strings (an unknown string is id -1), DAYS(16|32) dates with values off the day
    grid, TIMESTAMP FIXED(32), 8-byte DATE and DECIMAL columns."""
    import dec_tables as dt
    import enc_tables as et
    rng = random.Random(9)
    e = et.enc_table(2500, seed=6, frag_rows=700)
    econ = sqlite_of(e, et.ENC_NAMES, "e")
    for where in [f"k_i32_f16 IN ({lst(scattered(rng, 30, -60, 80))})",
                  f"k_i64_f32 NOT IN ({lst(scattered(rng, 60, 1000, 1400))})", f"a_i64_f16 IN ({lst(scattered(rng, 900, -30000, 30000))}) AND d < 0.7"]:
        check_rows(emu, e, et.ENC_NAMES, "e", where, econ, sqlite_where=f"({where}) AND deleted = 0")
    s = stt.str_table(3000, seed=7, frag_rows=800)
    scon = sqlite_of(s, stt.STR_NAMES, "s")
    days = scattered(rng, 25, 17995, 18065)
    d16 = scattered(rng, 20, 9980, 10020)
    ts = scattered(rng, 40, 1_600_000_000 - 20, 1_600_000_320)
    dts = scattered(rng, 20, 17990, 18050)
    for where in [f"dd IN ({lst([d * 86400 for d in days] + [days[0] * 86400 + 7])})",
                  f"dd NOT IN ({lst([d * 86400 for d in days] + [3])})", f"dd16 IN ({lst([d * 86400 for d in d16])})",
                  f"ts IN ({lst(ts)}) OR dd16 NOT IN ({lst([d * 86400 for d in d16])})", f"dt IN ({lst([d * 86400 for d in dts] + [dts[1] * 86400 + 1])})",
                  f"str NOT IN ({lst(scattered(rng, 20, -5, 60))})", f"s8 IN ({lst(scattered(rng, 40, 0, 254))}) AND s16 NOT IN ({lst(scattered(rng, 100, 0, 40000))})"]:
        check_rows(emu, s, stt.STR_NAMES, "s", where, scon)
    words = [f"w{i}" for i in range(50)]
    s._dicts = {"str": words}
    known = [words[i] for i in scattered(rng, 19, 0, 49)]
    strs = known + ["nope", "also-missing"]
    ids = [words.index(w) if w in words else -1 for w in strs]
    for neg in ("", "NOT "):
        check_rows(emu, s, stt.STR_NAMES, "s", f"str {neg}IN ({', '.join(repr(w) for w in strs)})", scon, sqlite_where=f"str {neg}IN ({lst(ids)})")
    rows = dt.mixed_rows(1500, seed=3)
    d = dt.make_table(rows, fragment_size=400)
    dcon = sqlite_of(d, dt.DEC_NAMES, "test")
    scaled = scattered(rng, 60, -5000, 5000)
    pv = scattered(rng, 30, -9999, 9999)
    for where, sq in [(f"dd IN ({', '.join(f'{v / 100:.2f}' for v in scaled)})", f"dd IN ({lst(scaled)})"),
                      (f"q NOT IN ({', '.join(f'{v / 100:.2f}' for v in pv)})", f"q NOT IN ({lst(pv)})"),
                      (f"dd_notnull IN ({', '.join(f'{v / 100:.2f}' for v in scattered(rng, 20, 0, 40) )})", None)]:
        if sq is None:
            vals = [int(round(float(x) * 100)) for x in where[where.index('(') + 1:-1].split(', ')]
            sq = f"dd_notnull IN ({lst(vals)})"
        check_rows(emu, d, dt.DEC_NAMES, "test", where, dcon, sqlite_where=sq)


def test_inner_columns_under_inner_and_left_joins(emu):
    """Long lists on outer and on inner columns of a join level: the whole lowered program on the denormalised rows (the probe
    done in numpy) gives the oracle's buffer, INNER and LEFT."""
    from test_filter_lowering import assert_buffers_match, run_join_program
    fact, dim = jt.fact_table(3000, seed=42, frag_rows=900), jt.dim_table(seed=14)
    rng = random.Random(10)
    ran = 0
    for left in ("", "LEFT "):
        for where in [f"d.attr IN ({lst(scattered(rng, 9, 0, 19, 1))}) OR d.big IN ({lst(scattered(rng, 30, -2**20, 2**20))})",
                      f"d.attr8 NOT IN ({lst(scattered(rng, 40, -100, 100))})", f"t.x IN ({lst(scattered(rng, 30, 0, 99))}) AND d.attr8 IN ({lst(scattered(rng, 25, -100, 100))})",
                      f"NOT (d.attr8 IN ({lst(scattered(rng, 20, -100, 100))}) AND t.fk16 IN ({lst(scattered(rng, 30, 0, 1000))}))"]:
            sql = f"SELECT d.attr, COUNT(*), SUM(t.v) FROM t {left}JOIN d ON t.fk32 = d.id32 WHERE {where} GROUP BY d.attr;"
            unit = sqlmini.parse(sql, fact, jt.FACT_NAMES, inner=(dim, jt.DIM_NAMES))
            assert set_terms(emu, unit, fact)[0] >= 1, sql
            res = oracle_lib.execute(unit, fact, entry_guess=4000, has_card=True)
            rc, got = run_join_program(WithSets(emu), unit, fact, dim, left=bool(left))
            assert rc == 0, sql
            assert_buffers_match(got, res.buffer(), sql)
            ran += 1
    assert ran == 8


def test_grouped_programs_reproduce_the_oracles_buffer(emu, rand_env):
    """filter (with set terms) -> entry -> accumulators -> materialise, on the host: the oracle's buffer, both layouts."""
    from test_filter_lowering import assert_buffers_match, run_program
    table, names, _ = rand_env
    rng = random.Random(11)
    ran = 0
    for i in range(6):
        w = random_where(rng, INT_COLS)
        sql = rng.choice([f"SELECT k8, COUNT(*), SUM(a64), MIN(k16), MAX(a32) FROM r WHERE {w} GROUP BY k8;",
                          f"SELECT COUNT(*), SUM(nn64), AVG(a16) FROM r WHERE {w} AND d < 0.8;",
                          f"SELECT k16, COUNT(DISTINCT a8), SUM(d) FROM r WHERE ({w}) OR k32 < 0 GROUP BY k16;"])
        unit = sqlmini.parse(sql, table, names)
        for columnar in (False, True):
            try:
                res = oracle_lib.execute(unit, table, entry_guess=3001, has_card=True, output_columnar=columnar)
            except oracle_lib.OracleError:
                continue
            ran += 1
            rc, got = run_program(WithSets(emu), unit, table, output_columnar=columnar, entry_guess=3001, has_card=True)
            assert rc == 0, sql
            assert_buffers_match(got, res.buffer(), sql)
    assert ran >= 8


# ---- int_exact_ref: the edges of every width --------------------------------------------------------------------------------
def edge_lists(w):
    """Scattered lists (>= 17 runs, so set terms) around the width's low edge (the NULL sentinel and its neighbours), its high
    edge and zero, in the column's logical unit; values the width cannot hold are kept (they match nothing)."""
    unit = ier.SECONDS_PER_DAY if w.is_days else 1
    lists = []
    for centre in (w.null, w.hi, 0):
        vals = sorted({centre + d for d in (-2, -1, 0, 1)} | {centre + k for k in range(3, 60, 3)} | {centre - k for k in range(4, 60, 3)})
        vals = [v * unit for v in vals if -(2**63) <= v * unit < 2**63]
        if w.is_days:
            vals += [vals[3] + 1, vals[-1] - 1]                                  # off the day grid
        if w.sql_type == abi.kDECIMAL:
            vals = [v for v in vals if abs(v) <= ier.DECIMAL18_MAX]
        if len(vals) >= 17:
            lists.append(vals)
    return lists


@pytest.mark.parametrize("w", ier.WIDTHS, ids=lambda w: w.name)
def test_exact_predicates_at_the_edges_of_every_width(emu, w):
    rng = np.random.default_rng(12)
    for nullable in (True, False):
        pool = ier.pool(w)
        extra = sorted({v // (ier.SECONDS_PER_DAY if w.is_days else 1) for lst_ in edge_lists(w) for v in lst_} )
        extra = [x for x in extra if w.lo <= x <= w.hi]
        if w.sql_type == abi.kDECIMAL:
            extra = [x for x in extra if abs(x) <= ier.DECIMAL18_MAX]
        vals = np.array(pool + extra, dtype=object)
        phys = np.array([int(v) for v in rng.choice(vals, 1500)], dtype=w.dtype)
        if nullable:
            phys[rng.random(phys.size) < 0.1] = w.null
        t = w.table(not nullable)
        keys = np.zeros(phys.size, np.int32)
        for b in range(0, phys.size, 400):
            t.add_host_fragment([keys[b:b + 400], phys[b:b + 400]])
        for vals_ in edge_lists(w):
            for p in [("in", vals_), ("not", ("in", vals_)), ("or", ("in", vals_), ("isnull",)), ("or", ("not", ("in", vals_)), ("isnull",))]:
                sql = f"SELECT COUNT(*) FROM t WHERE {ier.predicate_sql(w, p)};"
                unit = sqlmini.parse(sql, t, ["k", "v"])
                assert set_terms(emu, unit, t)[0] == 1, (w.name, sql[:120])
                want = np.flatnonzero(ier.passing(w, phys, nullable, p)).tolist()
                assert emulated_rows(emu, unit, t) == want, (w.name, nullable, p[0])


# ---- b2q_launch --------------------------------------------------------------------------------------------------------------
def test_b2q_launch_refuses_a_plan_with_a_set_term(emu):
    """b2q_launch runs on caller memory only, so a plan whose filter needs a bitmap is refused with a clear message (checked
    before the device: the same code with or without one)."""
    from test_gpu_parity import RAND_NAMES, random_table
    table = random_table(300, seed=85, frag_rows=100)
    rng = random.Random(13)
    unit = sqlmini.parse(f"SELECT k8, COUNT(*) FROM r WHERE k32 IN ({lst(scattered(rng, 30, -500, 500))}) GROUP BY k8;", table, RAND_NAMES)
    L = executor.lib()
    with Planned(unit, table, guess=3001, has_card=True) as p:
        assert p.rc == 0, p.err
        prm = abi.Params()
        assert L.b2q_launch(p.h, C.byref(prm), None) == abi.ERR_UNSUPPORTED
        assert "value set" in str(L.b2q_last_error_message())
