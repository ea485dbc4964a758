#!/usr/bin/env python
"""TEST INFRASTRUCTURE (fixture generator; never imported by the product, tests, smoke() or bench.py — it is the committed script that
made tests/golden/executetest_harvest.json).  Harvest the reference's own golden query strings for this path (run where the heavydb source tree exists; the result is
committed as tests/golden/executetest_harvest.json and replayed by tests/test_oracle_golden_harvest.py without the reference).

    python tools/harvest_executetest.py <heavydb source tree> > tests/golden/executetest_harvest.json
    python tools/harvest_executetest.py --steps <heavydb source tree> > tests/golden/executetest_steps_harvest.json

Tests/ExecuteTest.cpp holds ~1350 `c("SELECT ...", dt)` comparisons against SQLite.  A string is kept when
  * it reads only table `test` and only the columns tests/ref_full_table.py models (the numeric, dictionary-string and FIXED columns
    of the golden table),
  * heavydb_b200.sqlmini parses it (one table, AND/OR/NOT of column-vs-constant / column-vs-column / IS NULL / IN / BETWEEN,
    GROUP BY columns, COUNT / SUM / MIN / MAX / AVG / COUNT(DISTINCT) of a column, ORDER BY / LIMIT / OFFSET),
  * the oracle plans it (the path's own refusals drop the rest), and
  * SQLite evaluates the same string.
With --steps it keeps instead the strings of more than one work unit (HAVING, a subquery in FROM) that sqlmini.parse_steps splits
and the oracle plans at EVERY step, each intermediate read as a host temporary table (tests/temp_table_ref.py); they are replayed by
tests/test_temp_table_cpu.py and tests/test_gpu_temp_table.py.
Only the query string and the reference line it came from are stored: the expected rows are recomputed with SQLite at test time,
exactly as the reference's SQLiteComparator does (ExecuteTest.cpp:383-520)."""
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import oracle_lib  # noqa: E402
import ref_full_table as ft  # noqa: E402
import ref_tables as rt  # noqa: E402
import sqlmini  # noqa: E402
from heavydb_b200 import abi, executor  # noqa: E402

def accepts_steps(sql, table):
    """parse_steps splits it into two or more steps and the oracle plans and runs every one of them."""
    import temp_table_ref as tt
    steps = sqlmini.parse_steps(sql, table, ft.FULL_NAMES)
    if len(steps) < 2:
        return False
    tt.run_steps(steps, {"test": (table, ft.FULL_NAMES)},
                 lambda i, unit, tbl, names: tt.run_step_on_host(steps[i], unit, tbl, names, 48),
                 lambda _i, unit, tbl, res: tt.host_table(tt.oracle_columns(unit, tbl, res, 48)), dicts=ft.DICTS)
    return True


def main():
    steps_mode = "--steps" in sys.argv[1:]
    args = [a for a in sys.argv[1:] if a != "--steps"]
    text = open(os.path.join(args[0], "Tests", "ExecuteTest.cpp")).read()
    rows = ft.full_rows()
    table = ft.make_table(rows)
    con = ft.make_sqlite(rows)
    seen, out, stats = set(), [], {"strings": 0, "table_test": 0, "parsed": 0, "planned": 0, "kept": 0}
    # c("..." "..." , dt) with adjacent literals concatenated, or c(R"(...)", dt); comparisons wrapped in EXPECT_THROW are negative tests
    pat = re.compile(r'\bc\(\s*(?:R"\((.*?)\)"|((?:"(?:[^"\\]|\\.)*"\s*)+))\s*,', re.S)
    for _ in (0,):
        for m in pat.finditer(text):
            if re.search(r"EXPECT_(ANY_)?THROW\(\s*$", text[max(0, m.start() - 40):m.start()]):
                continue
            q = m.group(1) if m.group(1) is not None else "".join(re.findall(r'"((?:[^"\\]|\\.)*)"', m.group(2)))
            q = re.sub(r"\s+", " ", q).strip()
            if not q.upper().startswith("SELECT"):
                continue
            ln = text.count("\n", 0, m.start()) + 1
            stats["strings"] += 1
            if steps_mode:
                if not re.search(r"\bFROM test\b", q) or not re.search(r"\bHAVING\b|\bFROM\s*\(\s*SELECT\b", q, re.I) or \
                        re.search(r"\b(JOIN|UNION|OVER|CASE|EXTRACT|CAST|LIKE|DISTINCT ON)\b|,\s*test\b", q, re.I):
                    continue
            elif not re.search(r"\bFROM test\b", q) or re.search(r"\b(JOIN|UNION|OVER|CASE|HAVING|EXTRACT|CAST|LIKE|DISTINCT ON)\b|,\s*test\b|\(SELECT", q, re.I):
                continue
            stats["table_test"] += 1
            sql = q if q.endswith(";") else q + ";"
            if sql in seen:
                continue
            if steps_mode:
                try:
                    sqlmini.parse_steps(sql, table, ft.FULL_NAMES)
                except Exception:
                    continue
                stats["parsed"] += 1
                try:
                    if not accepts_steps(sql, table):
                        continue
                except (oracle_lib.OracleError, executor.QueryExecutionError, ValueError, AssertionError, KeyError, IndexError):
                    continue
                res = None
            else:
                try:
                    unit = sqlmini.parse(sql, table, ft.FULL_NAMES, dicts=ft.DICTS)
                except Exception:
                    continue
                stats["parsed"] += 1
                try:
                    res = oracle_lib.execute(unit, table, entry_guess=48, has_card=True, num_threads=2)
                except oracle_lib.OracleError:
                    continue
            stats["planned"] += 1
            try:
                con.execute(sql.rstrip(";")).fetchall()
            except Exception:
                continue
            del res
            seen.add(sql)
            out.append({"sql": sql, "line": ln})
    stats["kept"] = len(out)
    how = "tools/harvest_executetest.py --steps" if steps_mode else "tools/harvest_executetest.py"
    json.dump({"source": "Tests/ExecuteTest.cpp", "how": how, "stats": stats, "queries": out}, sys.stdout, indent=0)
    print()
    print(stats, file=sys.stderr)


if __name__ == "__main__":
    main()
